// sbg_device.cuh -- device-side data layout and kernels of the H100 (sm_90a) 3-LUT search.
//
// Everything here is integer/bitwise work on 256-bit truth tables (no tensor cores: there is no
// contraction to map to them).  The reference functions being replaced are lut.c:34-66
// (check_n_lut_possible), lut.c:79-109 (get_lut_function), lut.c:116-249 (search_5lut) and
// lut.c:256-487 (search_7lut); see DESIGN.md for how the loops were restructured.
//
// Data layout in HBM (DevProblem; the uncompressed tables stay resident, the rest is derived on the
// device whenever gates, target or mask change):
//   * tables are compressed to the masked positions only: bit i of a compressed table is the
//     table's value at the i-th set position of the mask, so a search under a mask of popcount m
//     touches NW = ceil(m/32) words per table instead of 8 (every test in the reference is
//     "under the mask", lut.c:38-42,86, so positions outside it never matter);
//   * word-major (tabs[w][gate]) so that a warp whose lanes hold different gates reads
//     consecutive shared-memory banks.
// Kernels stage the tables into shared memory with cp.async (LDGSTS) and keep them there; the
// per-launch DRAM traffic is the 16.5 KB problem block plus the hit list.
#pragma once

#if defined(SBG_COUNT_STAGE1) || defined(SBG_COUNT_FILTER)
#include <cstdio>
#endif
#include <cuda_pipeline.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

namespace sbg {

constexpr int kMaxGatesPad = 512;
constexpr int kThreads = 256;
constexpr int kWarpsPerCta = kThreads / 32;
constexpr unsigned kFull = 0xffffffffu;
constexpr uint64_t kDeal = 16;  // prefixes per block dealt to one part of a sharded search

struct DevProblem {
  uint32_t tabs[8][kMaxGatesPad];  // [word][gate], compressed + pre-ANDed with the mask
  uint32_t T[8];                   // target & mask, compressed
  uint32_t M[8];                   // compressed mask = low popcount(mask) bits set
  int32_t n;                       // number of gates
  int32_t nw;                      // words in use: 1, 2, 4 or 8
  uint32_t inmask;                 // bit g set: gate g (< 8) is excluded (lut.c:177-185)
  int32_t m;                       // popcount(mask) = number of (compressed) positions
  // Position-major copy: row p (compressed position) holds one bit per gate, bit g = value of
  // gate g at position p, the whole row complemented where the target is 0.  So "gate g takes
  // the target's value on every position of a set S" <=> bit g of AND_{p in S} xr[p], and "gate g
  // takes the opposite value on all of S" <=> bit g of ~OR_{p in S} xr[p].
  uint32_t xr[256][16];
  // The device-resident copy of the state's gate tables (state.h:72-88, 256 bits per gate,
  // gate-major) with the target and mask they were last compressed under.  A call ships only the
  // gates that differ from what is here (kernel arguments, or one copy for a large change); tabs,
  // T, M and xr above are derived from it on the device (prepare_problem).
  uint32_t full[kMaxGatesPad][8];
  uint32_t target_full[8];
  uint32_t mask_full[8];
};

struct DevCtl {
  // The work dispenser gets a cache line of its own: every warp of a sweep takes a ticket with an
  // atomic on it every few microseconds, and everything else in this block (hit counter, minimum
  // key, statistics) would otherwise queue up behind those atomics in the same L2 slice.
  unsigned long long ticket;       // next work item
  unsigned long long pad0[15];
  unsigned long long hit_count;    // filter7 / two-kernel search5: slots reserved in the hit buffer
  unsigned long long pad1[15];
  unsigned long long best;         // minimum key found so far by the running stage
  unsigned long long stop_ticket;  // search5: tickets above this cannot improve `best`
  unsigned long long swept;        // tuples put through the feasibility test
  unsigned long long feasible;     // search5: feasible tuples met
  unsigned long long ticket2;      // decomp5 / decomp7: next list entry
  unsigned long long seq;          // sequence number of the call (echoed to the host with each result)
  unsigned int overflow;           // 1: hit buffer too small, 2: ticket table too small
  unsigned int list_count;         // written by k_offsets: entries of the ordered list (<= cap)
  unsigned int ctas_done;          // last-CTA detection of the stage-closing kernels
  unsigned int skip5, skip7;       // stages not asked for (node calls)
  // seq << 8 | code once a stage of chain `seq` matched (code 3 / 5 / 7) or was left incomplete
  // (0xff): the later stages of that chain return at once.  Tagged with the sequence number so that
  // nobody has to reset it -- the 3-LUT scan runs inside the chain's first kernel, next to the
  // block that installs the other control words.
  unsigned long long found;
  // the 3-LUT scan's own words; its closing block leaves them as it found them (~0 and 0)
  unsigned long long best3;
  unsigned int scan_done;
  unsigned int pad2;
};

// What the device tells the host, in MAPPED PINNED host memory, one block per lane: the last CTA of
// a stage's closing kernel stores the stage's numbers, fences system-wide, then stores the call's
// sequence number into seq[stage]; the host spins on that word -- no copy, no stream
// synchronisation.  Stages: 0 = 3-LUT scan (lut.c:501-523), 1 = search_5lut, 2 = search_7lut.
struct HostOut {
  unsigned long long key[3];
  unsigned long long swept[3];
  unsigned long long feasible[3];   // stage 1: feasible 5-tuples met; stage 2: list length
  unsigned long long tuple;         // stage 2: the winning list entry ...
  unsigned long long tuple_prev;    // ... and the one before it (stale-cache quirk, lut.c:432-435)
  unsigned int overflow[3];
  unsigned int pad;
  unsigned long long seq[3];
};

// Per-call parameters of the 7-LUT decomposition.  The host supplies where each function sits in
// the two shuffled orders; k_prepare7 derives from the middle order the table
//   minpos3[code(S,V)] = min { pm : (middle_order[pm] & S) == V },   V subset of S,
// indexed in base 3 (digit j = 0: bit j unconstrained, 1: forced 0, 2: forced 1), i.e.
// code(S,V) = p3(S) + p3(V) with p3(x) = sum of 3^j over the set bits of x.  6,561 entries.
constexpr int kMinpos3 = 6561;
struct DevParams7 {
  uint8_t pos_outer[256];
  uint8_t pos_middle[256];
  uint8_t minpos3[kMinpos3 + 3];   // device-built; not part of the upload
};

// Lane-indexed lookup tables live in global memory (coalesced, L1-resident): a constant-memory load
// whose address differs per lane is replayed once per distinct address.
struct DevTables {
  uint8_t src5[10][32];    // search5: ordering k, lane (u,v2) -> canonical cell
  uint32_t src7[25][32];   // decomp7: outer triple j, lane (u0,v4) -> 4 cells (u2,u1)
  // k_begin: the 6,561 entries of DevParams7::minpos3 listed by number of unconstrained bits
  // (level l = entries m3_level[l] .. m3_level[l+1]-1); info = entry | (level 0: the function,
  // else: 3^j of its lowest unconstrained bit j) << 16
  uint32_t m3_info[6561];
  int32_t m3_level[10];
};

__constant__ uint64_t c_binom[501][8];   // C(m, r), 0 <= m <= 500, 0 <= r <= 7
__constant__ uint8_t c_j_first_k[25];    // first ordering row of outer triple j
__constant__ uint8_t c_j_rows[25];       // rows sharing that outer triple (4 or 1)
__constant__ uint8_t c_row_b[70];        // bit of v4 that is the g input in ordering row k

// One LOP3 with the given truth table (inputs a = 0xF0, b = 0xCC, c = 0xAA), opaque to the
// compiler so that it keeps the operand grouping chosen here.
template <int LUT>
__device__ __forceinline__ uint32_t lop3(uint32_t a, uint32_t b, uint32_t c) {
  uint32_t d;
  asm("lop3.b32 %0, %1, %2, %3, %4;" : "=r"(d) : "r"(a), "r"(b), "r"(c), "n"(LUT));
  return d;
}

__device__ __forceinline__ unsigned lanemask_lt() {
  unsigned m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}

// Item t of one part of a sharded sweep, as an item of the whole: items are dealt to the parts in
// blocks of kDeal consecutive items, part p owning blocks p, p + nparts, ...
__device__ __forceinline__ uint64_t dealt_item(uint64_t t, int part, int nparts) {
  return (t / kDeal) * kDeal * (uint64_t)nparts + (uint64_t)part * kDeal + t % kDeal;
}

// Stages `rows` rows of `npad` words of the problem's tables into shared memory with cp.async.
__device__ __forceinline__ void stage_tables(uint32_t *s_tabs, const DevProblem *prob, int rows,
    int npad) {
  const int chunks_per_row = npad >> 2;  // 16-byte chunks
  for (int i = threadIdx.x; i < rows * chunks_per_row; i += blockDim.x) {
    const int w = i / chunks_per_row;
    const int c = i - w * chunks_per_row;
    __pipeline_memcpy_async(s_tabs + w * npad + 4 * c, &prob->tabs[w][4 * c], 16);
  }
  __pipeline_commit();
  __pipeline_wait_prior(0);
  __syncthreads();
}

// C(a, r) for 0 <= a <= 512, r <= 5, by arithmetic (exact at every step: a product of k consecutive
// integers is divisible by k!).  r is a compile-time constant wherever this is called from an
// unrolled loop, the chain below then folds to the one case.  The table c_binom sits in constant
// memory, which serves one address per warp at a time -- lanes that each need a different entry
// compute it instead.
__device__ __forceinline__ uint64_t binom_arith(uint32_t a, int r) {
  if (r <= 0) return 1ull;
  if (r == 1) return a;
  const uint32_t c2 = (a * (a - 1u)) >> 1;                 // <= 130,816
  if (r == 2) return c2;
  const uint32_t c3 = (c2 * (a - 2u)) * 0xaaaaaaabu;       // exact division by 3 (inverse mod 2^32)
  if (r == 3) return c3;
  const uint64_t c4 = ((uint64_t)c3 * (uint64_t)(a - 3u)) >> 2;
  if (r == 4) return c4;                                   // (a < r: some factor above is zero)
  return (c4 * (uint64_t)(a - 4u)) / 5ull;
}

// Work item t of the P-element prefixes of K-combinations over n gates, lexicographic order, and
// (RANK) the rank in C(n,K) order (lut.c:635-662) of the first combination with that prefix --
// unranked by the whole warp: per element, lane l asks "do at most t prefixes have a smaller
// element here than x0 + l?" -- the number that do is C(np - x0, r) - C(np - y, r) with r elements
// still to place (hockey stick) -- and one ballot counts the lanes that say yes.  Three or four
// ballots instead of a loop that walks the gates one constant-memory load at a time (which was a
// tenth of phase 1's instructions at n = 40).  All lanes must call; all receive the result.
template <int P, int K, bool RANK>
__device__ __forceinline__ void unrank_prefix_warp(uint64_t t64, int n, int *pre, uint64_t &base_rank,
    int lane) {
  static_assert(P <= 5 && (!RANK || K <= 5), "binom_arith covers r <= 5");
  // the number of P-prefixes fits 32 bits up to P = 4 (C(509, 4) = 2.77e9)
  using T = typename std::conditional<(P <= 4), uint32_t, uint64_t>::type;
  const int np = n - (K - P);
  T t = (T)t64;
  int x0 = 0;
  base_rank = 0;
#pragma unroll
  for (int pos = 0; pos < P; pos++) {
    const int r = P - pos;
    int e;
    if (r == 1) {
      e = x0 + (int)t;
    } else {
      const T total = (T)binom_arith((uint32_t)(np - x0), r);
      int cnt = 0;
      for (int y0 = x0;; y0 += 32) {
        const int y = y0 + lane;
        const bool le = y <= np - r && (T)(total - (T)binom_arith((uint32_t)max(np - y, 0), r)) <= t;
        const uint32_t bal = __ballot_sync(kFull, le);
        cnt += __popc(bal);
        if (bal != 0xffffffffu) break;
      }
      e = x0 + cnt - 1;
      t -= (T)(total - (T)binom_arith((uint32_t)(np - e), r));
    }
    if (RANK) {
      base_rank += binom_arith((uint32_t)(n - x0), K - pos) - binom_arith((uint32_t)(n - e), K - pos);
    }
    pre[pos] = e;
    x0 = e + 1;
  }
}

// q-th pair (i < j) of {0..r-1} in lexicographic order.
__device__ __forceinline__ void unrank_pair(uint32_t q, int r, int &i, int &j) {
  const float b = 2.0f * r - 1.0f;
  int ii = (int)((b - sqrtf(fmaxf(b * b - 8.0f * (float)q, 0.0f))) * 0.5f);
  ii = max(0, min(ii, r - 2));
  // offset(i) = i*(2r-i-1)/2 pairs precede row i
  while (ii > 0 && (uint32_t)(ii * (2 * r - ii - 1) / 2) > q) ii--;
  while ((uint32_t)((ii + 1) * (2 * r - ii - 2) / 2) <= q) ii++;
  i = ii;
  j = ii + 1 + (int)(q - (uint32_t)(ii * (2 * r - ii - 1) / 2));
}

// Leading zeros of a non-zero word in one instruction (FLO.SH); __clz pays a subtraction for x == 0.
__device__ __forceinline__ int clz_nonzero(uint32_t x) {
  int c;
  asm("bfind.shiftamt.u32 %0, %1;" : "=r"(c) : "r"(x));
  return c;
}

// Each byte of x replaced by its top bit spread over the whole byte (0x00 or 0xff), in one PRMT:
// selector nibbles with the high bit set replicate the sign of the selected byte.
__device__ __forceinline__ uint32_t prmt_sign_bytes(uint32_t x) {
  uint32_t d;
  asm("prmt.b32 %0, %1, 0, 0xba98;" : "=r"(d) : "r"(x));
  return d;
}

// Shared-memory load from a 32-bit shared-window address (one address instruction in the caller).
__device__ __forceinline__ uint32_t lds_u32(uint32_t saddr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(saddr) : "memory");
  return v;
}

__device__ __forceinline__ uint2 lds_v2(uint32_t saddr) {
  uint2 v;
  asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(saddr) : "memory");
  return v;
}

__device__ __forceinline__ unsigned long long volatile_load(const unsigned long long *p) {
  return *reinterpret_cast<const volatile unsigned long long *>(p);
}

__device__ __forceinline__ uint32_t volatile_load32(const unsigned int *p) {
  return *reinterpret_cast<const volatile unsigned int *>(p);
}

// Programmatic dependent launch (sm_90+): a kernel launched with the programmatic-serialisation
// attribute starts while its predecessor in the stream is still draining; everything before this
// call (staging the problem's tables into shared memory, which no kernel of a chain writes) overlaps
// the predecessor's tail, everything after it sees the predecessor's memory.  Without the attribute
// both calls are no-ops.
__device__ __forceinline__ void wait_for_predecessor() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
}
__device__ __forceinline__ void let_successor_start() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

// Has an earlier stage of this chain matched (or been left incomplete)?
__device__ __forceinline__ bool chain_is_over(const DevCtl *ctl) {
  const unsigned long long f = volatile_load(&ctl->found);
  return (f >> 8) == volatile_load(&ctl->seq) && (f & 0xffull) != 0;
}

// End of a stage-closing kernel.  Every CTA calls it (no early returns in those kernels); exactly one
// -- the last to arrive -- gets `true`, with every other CTA's global writes visible to it.
__device__ __forceinline__ bool last_cta_of_grid(DevCtl *ctl) {
  __shared__ int s_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned int prev = atomicAdd(&ctl->ctas_done, 1u);
    s_last = prev == gridDim.x - 1;
    if (s_last) {
      ctl->ctas_done = 0;   // the next kernel of the chain counts from zero
      __threadfence();
    }
  }
  __syncthreads();
  return s_last != 0;
}

// The closing CTA's thread 0: stage results -> mapped host memory, sequence number last; then the
// control words the stages share are made ready for the next stage of the chain (its kernels cannot
// pass their wait_for_predecessor() / stream order before this kernel has completed).
__device__ __forceinline__ void close_stage(DevCtl *ctl, HostOut *out, int stage,
    unsigned long long key, unsigned long long feasible, unsigned long long tuple,
    unsigned long long tuple_prev) {
  const unsigned int overflow = volatile_load32(&ctl->overflow);
  out->key[stage] = key;
  out->swept[stage] = volatile_load(&ctl->swept);
  out->feasible[stage] = feasible;
  out->overflow[stage] = overflow;
  if (stage == 2) {
    out->tuple = tuple;
    out->tuple_prev = tuple_prev;
  }
  const unsigned long long tag = ctl->seq << 8;
  if (key != ~0ull) ctl->found = tag | (unsigned long long)(3 + 2 * stage);   // later stages return at once
  else if (overflow != 0) ctl->found = tag | 0xffull;      // incomplete stage: the host redoes it
  ctl->ticket = 0;
  ctl->ticket2 = 0;
  ctl->hit_count = 0;
  ctl->swept = 0;
  ctl->feasible = 0;
  ctl->best = ~0ull;
  ctl->stop_ticket = ~0ull;
  ctl->overflow = 0;
  __threadfence_system();
  *reinterpret_cast<volatile unsigned long long *>(&out->seq[stage]) = ctl->seq;
}

// ------------------------------------------------------------------------------------------------
// search_5lut's inner loops for ONE feasible 5-tuple (lut.c:189-230), whole warp: the 10 orderings x
// 256 outer functions decided from the tuple's 32-cell summary H1/H0 (cells that contain a masked
// 1 / a masked 0 of the target).  Returns the first (ordering, position in the shuffled function
// order) that decomposes, as k<<8 | pos, or 0xffffffff.

// The tuple's 32-cell summary (lane = cell, first gate = most significant bit): bit l of H1 / H0 is
// set iff cell l holds a masked position with target 1 / 0.
template <int NW>
__device__ __forceinline__ void summary5(const uint32_t *s_tabs, int npad, const int *g,
    const uint32_t *T, const uint32_t *M, int lane, uint32_t &H1, uint32_t &H0) {
  uint32_t ones = 0, zeros = 0;
#pragma unroll
  for (int w = 0; w < NW; w++) {
    uint32_t tt = M[w];
#pragma unroll
    for (int i = 0; i < 5; i++) {
      const uint32_t tv = s_tabs[w * npad + g[i]];
      tt &= ((lane >> (4 - i)) & 1) ? tv : ~tv;
    }
    ones |= tt & T[w];
    zeros |= tt & ~T[w];
  }
  H1 = __ballot_sync(kFull, ones != 0);
  H0 = __ballot_sync(kFull, zeros != 0);
}

// Ordering k of a tuple with summary H1 / H0: ok[hi] bit lane and ok[7 - hi] bit 31 - lane both
// set <=> outer function hi*32+lane decomposes.
__device__ __forceinline__ void outer_ok5(uint32_t H1, uint32_t H0, int k, int lane,
    const DevTables *__restrict__ tab, uint32_t *ok) {
  const int s = tab->src5[k][lane];
  const uint32_t b1 = __ballot_sync(kFull, (H1 >> s) & 1u);
  const uint32_t b0 = __ballot_sync(kFull, (H0 >> s) & 1u);
  // wv(u): bits 0-3 = inner cells (x, d, e) with a masked 1 contributed by outer pattern u,
  // bits 4-7 = the same for masked 0.
#define SBG_W5(u) (((b1 >> (4 * (u))) & 0xfu) | (((b0 >> (4 * (u))) & 0xfu) << 4))
  uint32_t L = 0;
#pragma unroll
  for (int u = 0; u < 5; u++) {
    if ((lane >> u) & 1) L |= SBG_W5(u);
  }
#pragma unroll
  for (int hi = 0; hi < 8; hi++) {
    uint32_t rr = L;
    if (hi & 1) rr |= SBG_W5(5);
    if (hi & 2) rr |= SBG_W5(6);
    if (hi & 4) rr |= SBG_W5(7);
    ok[hi] = __ballot_sync(kFull, ((rr & (rr >> 4)) & 0xfu) == 0);
  }
#undef SBG_W5
}

template <int NW>
__device__ __forceinline__ uint32_t decomp5_tuple(const uint32_t *s_tabs, int npad, const int *g,
    const uint32_t *T, const uint32_t *M, int lane, const uint8_t *s_pos,
    const DevTables *__restrict__ tab) {
  uint32_t H1, H0;
  summary5<NW>(s_tabs, npad, g, T, M, lane, H1, H0);
  for (int k = 0; k < 10; k++) {
    uint32_t ok[8];
    outer_ok5(H1, H0, k, lane, tab, ok);
    // Outer function fo = hi*32+lane maps pattern u to x = bit u of fo; it works iff neither
    // {u: x=1} nor {u: x=0} merges a masked 1 and a masked 0 into one inner cell.
    uint32_t best_pos = 256;
#pragma unroll
    for (int hi = 0; hi < 8; hi++) {
      const uint32_t surv = ok[hi] & __brev(ok[7 - hi]);
      if ((surv >> lane) & 1u) best_pos = min(best_pos, (uint32_t)s_pos[hi * 32 + lane]);
    }
    best_pos = __reduce_min_sync(kFull, best_pos);
    if (best_pos < 256) return ((uint32_t)k << 8) | best_pos;
  }
  return 0xffffffffu;
}

// ------------------------------------------------------------------------------------------------
// Sweep kernel of search_5lut.  One warp per 3-gate prefix; lanes take the (d,e) pairs that complete
// it: search_5lut's loop over C(n,5) (lut.c:174-245), either with the 10 x 256 decomposition
// attempts fused (large searches; result = minimum key in ctl->best) or only recording the feasible
// tuples for k_decomp5 (small ones).
//
// Feasibility (lut.c:34-66) of prefix + (d,e): no cell of the 32-cell partition may hold both a
// masked 1 and a masked 0 of the target.  A prefix cell that is already pure stays pure however it
// is split, so only the "mixed" prefix cells are kept (their ones C1 = C & T and zeros C0 = C & ~T,
// in shared memory); each must be split by d and e into four parts none of which meets both C1 and
// C0.  A pair is dropped at the first cell it fails on.
// Chunk tickets (see k_sweep / k_filter7_pm): the t-th P-gate prefix made of allowed gates only, as
// gate numbers, with its rank among all prefixes (for the stop rule) and the rank of its first
// combination (for the key).  Kept out of line: it runs once per chunk ticket, and inlined it
// changes the code of the sweep loop around it for the worse.
template <int P, int K>
__device__ __noinline__ void chunk_ticket_prefix(uint64_t t, int n, uint32_t inmask, int *pre,
    uint64_t &prefix_rank, uint64_t &base_rank, int lane) {
  uint64_t unused_rank;
  unrank_prefix_warp<P, K, false>(t, n - __popc(inmask & 0xffu), pre, unused_rank, lane);
  prefix_rank = 0;
  base_rank = 0;
  int prev = -1;
  for (int i = 0; i < P; i++) {
    int g = pre[i];   // index among the allowed gates -> gate number (excluded gates are < 8)
    for (int bit = 0; bit < 8; bit++) g += (((inmask >> bit) & 1u) != 0 && bit <= g) ? 1 : 0;
    pre[i] = g;
    for (int x = prev + 1; x < g; x++) {
      prefix_rank += c_binom[n - (K - P) - x - 1][P - i - 1];
      base_rank += c_binom[n - x - 1][K - i - 1];
    }
    prev = g;
  }
}

// closes = this launch ends the search_5lut stage (fused form): its last CTA publishes the result.
template <int NW>
__global__ void __launch_bounds__(kThreads) k_sweep(const DevProblem *__restrict__ prob,
    DevCtl *__restrict__ ctl, HostOut *__restrict__ out, const uint8_t *__restrict__ pos_of,
    uint64_t *__restrict__ hits, unsigned long long hits_cap, int part, int nparts, int batch,
    bool emit5, const DevTables *__restrict__ tab, unsigned long long t_offset,
    unsigned long long chunk_items, int chunks_per_prefix, unsigned long long chunk_tickets) {
  constexpr int P = 3, K = 5, NC = 1 << P;
  extern __shared__ uint32_t smem[];
  __shared__ uint8_t s_pos[256];
  __shared__ uint32_t s_TM[16];   // T[0..7], M[0..7]: indexed by a lane-dependent word number

  wait_for_predecessor();   // the chain's first kernel derives the problem block
  const int n = prob->n;
  const int npad = (n + 3) & ~3;
  uint32_t *s_tabs = smem;
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  uint32_t *cells = smem + NW * npad + warp * (NC * 2 * NW);  // per mixed cell: C1[NW], C0[NW]

  stage_tables(s_tabs, prob, NW, npad);
  const bool skip = chain_is_over(ctl) || volatile_load32(&ctl->skip5) != 0;
  if (!skip) {
  for (int i = threadIdx.x; i < 256; i += blockDim.x) s_pos[i] = pos_of[i];
  if (threadIdx.x < 16) {
    const int w = threadIdx.x & 7;
    s_TM[threadIdx.x] = w < NW ? (threadIdx.x < 8 ? prob->T[w] : prob->M[w]) : 0u;
  }
  __syncthreads();

  uint32_t T[NW], M[NW];
#pragma unroll
  for (int w = 0; w < NW; w++) {
    T[w] = prob->T[w];
    M[w] = prob->M[w];
  }
  const uint32_t inmask = prob->inmask;
  const uint64_t total = c_binom[n - 2][P];

  // Work items (prefixes) are handed out in lexicographic order in batches of `batch` consecutive
  // prefixes: one global atomic per batch, issued one batch ahead so that its latency (and that of
  // the stop-flag read) overlaps the previous batch's work; inside a batch the prefix and the rank
  // of its first combination advance incrementally instead of being unranked again.
  unsigned long long swept_local = 0;
  unsigned long long next_b = 0, next_stop = ~0ull;
  auto fetch = [&]() {
    if (lane == 0) {
      next_stop = volatile_load(&ctl->stop_ticket);
      next_b = atomicAdd(&ctl->ticket, 1ull);
    }
  };
  fetch();
  bool warp_finished = false;
  while (!warp_finished) {
    const unsigned long long b = __shfl_sync(kFull, next_b, 0);
    const unsigned long long stop_at = __shfl_sync(kFull, next_stop, 0);
    // Prefixes are dealt to the parts of a sharded search in blocks of kDeal consecutive prefixes
    // (part p owns blocks p, p + nparts, ...), independently of the batch size, which is a power
    // of two <= kDeal so that a batch never straddles two blocks.
    // The first chunk_tickets tickets (search_5lut on large states) are (prefix, chunk of 32 pairs)
    // items over the first prefixes made of allowed gates only, as in k_filter7_pm: on a dense
    // state the tuples in front of the first match are then decomposed by many warps, not one.
    const bool chunked = b < chunk_tickets;
    const uint64_t lt = chunked ? b : (b - chunk_tickets) * (uint64_t)batch;
    const uint64_t dealt = dealt_item(lt, part, nparts);
    uint64_t t_first, t_end;
    uint32_t q_begin = 0, q_limit = 0xffffffffu;
    int pre[P];
    uint64_t base_rank;
    if (chunked) {
      if (dealt >= chunk_items) {   // the last deal block is shorter for some parts
        fetch();
        continue;
      }
      q_begin = (uint32_t)(dealt % (uint64_t)chunks_per_prefix) * 32u;
      q_limit = q_begin + 32u;
      fetch();
      chunk_ticket_prefix<P, K>(dealt / (uint64_t)chunks_per_prefix, n, inmask, pre, t_first,
          base_rank, lane);
      t_end = t_first + 1;
      if (t_first > stop_at) break;
    } else {
      t_first = t_offset + dealt;
      if (t_first >= total) break;
      if (t_first > stop_at) break;
      fetch();
      t_end = min(t_first + (uint64_t)batch, total);
      unrank_prefix_warp<P, K, true>(t_first, n, pre, base_rank, lane);
    }
   for (uint64_t gt = t_first; gt < t_end && !warp_finished; gt++) {
    if (gt != t_first) {
      // successor of the prefix among the P-subsets of {0..n-3}; the combinations sharing the
      // previous prefix were contiguous in rank
      const int rprev = n - pre[P - 1] - 1;
      base_rank += (uint64_t)(rprev * (rprev - 1) / 2);
      int i = P - 1;
      while (i > 0 && pre[i] + (P - i) >= n - 2) i--;
      pre[i]++;
      for (int k2 = i + 1; k2 < P; k2++) pre[k2] = pre[k2 - 1] + 1;
    }
    const int last = pre[P - 1];
    const int r = n - last - 1;
    const uint32_t Q = (uint32_t)(r * (r - 1) / 2);
    if (q_begin >= max(Q, 1u)) continue;   // chunk ticket beyond this prefix's pairs
    // T-units (lut.c:174-187): the combinations of the pair chunks this ticket goes through
    swept_local += (uint64_t)(min(Q, q_limit) - q_begin);
    bool rejected = false;
#pragma unroll
    for (int i = 0; i < P; i++) rejected |= (pre[i] < 8) && ((inmask >> pre[i]) & 1u);
    if (rejected) continue;

    // Prefix cells: lane = cell index, first prefix gate = most significant bit (lut.c:46-49).
    // The warp's four groups of 8 lanes share the table words among them (G groups, NWG words each).
    uint32_t mixed_ballot;
    {
      constexpr int G = NW >= 4 ? 4 : NW, NWG = NW / G;
      const int cell = lane & (NC - 1);
      const int group = (lane >> 3) & (G - 1);
      uint32_t c1[NWG], c0[NWG];
      uint32_t ones = 0, zeros = 0;
#pragma unroll
      for (int k = 0; k < NWG; k++) {
        const int w = group * NWG + k;
        uint32_t tt = s_TM[8 + w];
        const uint32_t tw = s_TM[w];
#pragma unroll
        for (int i = 0; i < P; i++) {
          const uint32_t tv = s_tabs[w * npad + pre[i]];
          tt &= ((cell >> (P - 1 - i)) & 1) ? tv : ~tv;
        }
        c1[k] = tt & tw;
        c0[k] = tt & ~tw;
        ones |= c1[k];
        zeros |= c0[k];
      }
      if (G >= 2) {
        ones |= __shfl_xor_sync(kFull, ones, 8);
        zeros |= __shfl_xor_sync(kFull, zeros, 8);
      }
      if (G >= 4) {
        ones |= __shfl_xor_sync(kFull, ones, 16);
        zeros |= __shfl_xor_sync(kFull, zeros, 16);
      }
      const bool mixed = ones != 0 && zeros != 0;   // the same in every group
      mixed_ballot = __ballot_sync(kFull, mixed) & ((1u << NC) - 1u);
      __syncwarp();
      if (mixed) {
        const int slot = __popc(mixed_ballot & ((1u << cell) - 1u));
#pragma unroll
        for (int k = 0; k < NWG; k++) {
          cells[slot * 2 * NW + group * NWG + k] = c1[k];
          cells[slot * 2 * NW + NW + group * NWG + k] = c0[k];
        }
      }
      __syncwarp();
    }
    const int mc = __popc(mixed_ballot);

    bool warp_done = false;
    // the lane's pair: unranked once per prefix, then moved on by 32 places per chunk (row i of the
    // pairs of {0..r-1} holds j = i+1 .. r-1)
    int run_i = 0, run_j = 1;
    if (q_begin + (uint32_t)lane < Q) unrank_pair(q_begin + (uint32_t)lane, r, run_i, run_j);
    for (uint32_t q0 = q_begin; q0 < min(Q, q_limit) && !warp_done; q0 += 32) {
      const uint32_t q = q0 + lane;
      bool alive = q < Q;
      if (q0 != q_begin) {
        run_j += 32;
        while (run_j >= r && run_i < r - 2) {
          run_i++;
          run_j += run_i + 1 - r;
        }
      }
      const int pi = alive ? run_i : 0, pj = alive ? run_j : 1;   // past the end: pair (0, 1)
      const int gf = last + 1 + pi;
      const int gg = last + 1 + pj;
      if ((gf < 8 && ((inmask >> gf) & 1u)) || (gg < 8 && ((inmask >> gg) & 1u))) alive = false;

      if (mc > 0) {
        uint32_t m11[NW], m10[NW], m01[NW], m00[NW];  // the four (d,e) minterms
#pragma unroll
        for (int w = 0; w < NW; w++) {
          const uint32_t tf = s_tabs[w * npad + gf];
          const uint32_t tg = s_tabs[w * npad + gg];
          m11[w] = tf & tg;
          m10[w] = tf & ~tg;
          m01[w] = ~tf & tg;
          m00[w] = ~(tf | tg);
        }
        for (int cj = 0; cj < mc; cj++) {
          if (!__any_sync(kFull, alive)) break;
          uint32_t a11 = 0, a10 = 0, a01 = 0, a00 = 0, b11 = 0, b10 = 0, b01 = 0, b00 = 0;
#pragma unroll
          for (int w = 0; w < NW; w++) {
            const uint32_t c1 = cells[cj * 2 * NW + w];
            const uint32_t c0 = cells[cj * 2 * NW + NW + w];
            a11 |= c1 & m11[w]; b11 |= c0 & m11[w];
            a10 |= c1 & m10[w]; b10 |= c0 & m10[w];
            a01 |= c1 & m01[w]; b01 |= c0 & m01[w];
            a00 |= c1 & m00[w]; b00 |= c0 & m00[w];
          }
          if ((a11 != 0 && b11 != 0) || (a10 != 0 && b10 != 0) || (a01 != 0 && b01 != 0)
              || (a00 != 0 && b00 != 0)) {
            alive = false;
          }
        }
      }

      uint32_t fb = __ballot_sync(kFull, alive);
      if (fb == 0) continue;

      if (emit5) {
        // Two-kernel form for small searches: feasible 5-tuples are only recorded here (rank and
        // packed gates) and decomposed by k_decomp5, one warp per tuple, so that a warp meeting
        // several of them does not become the kernel's critical path.
        const int cnt = __popc(fb);
        unsigned long long base_slot = 0;
        if (lane == 0) base_slot = atomicAdd(&ctl->hit_count, (unsigned long long)cnt);
        base_slot = __shfl_sync(kFull, base_slot, 0);
        if (alive) {
          const unsigned long long slot = base_slot + __popc(fb & lanemask_lt());
          uint64_t packed = 0;
#pragma unroll
          for (int i = 0; i < 3; i++) packed = (packed << 9) | (uint64_t)pre[i];
          packed = (packed << 18) | ((uint64_t)gf << 9) | (uint64_t)gg;
          if (2 * slot + 1 < hits_cap) {
            hits[2 * slot] = base_rank + q;
            hits[2 * slot + 1] = packed;
          } else {
            atomicExch(&ctl->overflow, 1u);
          }
        }
        continue;
      }
      // search_5lut: try the 10 orderings x 256 outer functions on each feasible tuple
      // (lut.c:189-230), here, one after the other -- unless a match in an earlier prefix is
      // already known (dense states: every warp of the first wave sits on feasible tuples).
      {
        unsigned long long st = 0;
        if (lane == 0) st = volatile_load(&ctl->stop_ticket);
        if (gt > __shfl_sync(kFull, st, 0)) warp_done = true;
      }
      while (fb != 0 && !warp_done) {
        const int src = __ffs(fb) - 1;
        fb &= fb - 1;
        int g5[5];
        g5[0] = pre[0];
        g5[1] = pre[1];
        g5[2] = pre[2];
        g5[3] = __shfl_sync(kFull, gf, src);
        g5[4] = __shfl_sync(kFull, gg, src);
        if (lane == 0) atomicAdd(&ctl->feasible, 1ull);
        const uint32_t hit = decomp5_tuple<NW>(s_tabs, npad, g5, T, M, lane, s_pos, tab);
        if (hit != 0xffffffffu) {
          const uint64_t key = ((base_rank + q0 + src) << 12) | (uint64_t)hit;
          if (lane == 0) {
            atomicMin(&ctl->best, (unsigned long long)key);
            atomicMin(&ctl->stop_ticket, (unsigned long long)gt);
          }
          warp_done = true;
        }
      }
    }
    if (warp_done) warp_finished = true;  // every later prefix has a larger key
   }
  }
  if (lane == 0 && swept_local != 0) atomicAdd(&ctl->swept, swept_local);
  }  // !skip
  let_successor_start();
  if (!emit5 && last_cta_of_grid(ctl) && threadIdx.x == 0 && !skip) {
    close_stage(ctl, out, 1, volatile_load(&ctl->best), volatile_load(&ctl->feasible), 0, 0);
  }
}

// ------------------------------------------------------------------------------------------------
// Second kernel of the two-kernel search_5lut: one warp per recorded feasible 5-tuple.  Closes the
// stage: its last CTA publishes the result.
template <int NW>
__global__ void __launch_bounds__(kThreads) k_decomp5(const DevProblem *__restrict__ prob,
    DevCtl *__restrict__ ctl, HostOut *__restrict__ out, const uint8_t *__restrict__ pos_of,
    const uint64_t *__restrict__ hits, const DevTables *__restrict__ tab) {
  extern __shared__ uint32_t smem[];
  __shared__ uint8_t s_pos[256];
  wait_for_predecessor();
  const int n = prob->n;
  const int npad = (n + 3) & ~3;
  uint32_t *s_tabs = smem;
  const int lane = threadIdx.x & 31;
  stage_tables(s_tabs, prob, NW, npad);
  const bool skip = chain_is_over(ctl) || volatile_load32(&ctl->skip5) != 0;
  const unsigned long long count = ctl->hit_count;
  if (!skip && ctl->overflow == 0 && (unsigned long long)blockIdx.x * kWarpsPerCta < count) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) s_pos[i] = pos_of[i];
    __syncthreads();
    uint32_t T[NW], M[NW];
#pragma unroll
    for (int w = 0; w < NW; w++) {
      T[w] = prob->T[w];
      M[w] = prob->M[w];
    }
    for (;;) {
      unsigned long long t = 0;
      if (lane == 0) t = atomicAdd(&ctl->ticket2, 1ull);
      t = __shfl_sync(kFull, t, 0);
      if (t >= count) break;
      const uint64_t rank = hits[2 * t];
      if ((volatile_load(&ctl->best) >> 12) < rank) continue;  // a smaller combination matched
      const uint64_t packed = hits[2 * t + 1];
      int g5[5];
#pragma unroll
      for (int i = 0; i < 5; i++) g5[i] = (int)((packed >> (9 * (4 - i))) & 0x1ffu);
      const uint32_t hit = decomp5_tuple<NW>(s_tabs, npad, g5, T, M, lane, s_pos, tab);
      if (hit != 0xffffffffu && lane == 0) {
        atomicMin(&ctl->best, (unsigned long long)((rank << 12) | (uint64_t)hit));
      }
    }
  }
  let_successor_start();
  if (last_cta_of_grid(ctl) && threadIdx.x == 0 && !skip) {
    close_stage(ctl, out, 1, volatile_load(&ctl->best), count, 0, 0);
  }
}

// ------------------------------------------------------------------------------------------------
// Weighted tickets (phase 1, 4-gate prefixes, n <= kWeightedMaxGates).  A whole prefix as one ticket
// is too coarse where a warp's balanced share of the sweep is short: prefix (a,b,c,d) has
// C(n-d-2, 2) pairs -- 19 chunks of 32 for the first prefixes at n = 40 -- and such prefixes recur
// all through the lexicographic order (every (a,b,c) block starts with a small d).  So a prefix is
// cut into groups of `group_pairs` pairs, f(d) = ceil(pairs / group_pairs) tickets, numbered in
// lexicographic order of (prefix, group): ticket numbers stay monotone in the order of the list, which
// is all the ordered emission and the stop rule need.  Ticket -> (prefix, group) is the same ballot
// search as unrank_prefix_warp with f-weighted counts in place of binomials:
//   w[r-1][x] = total tickets of the sequences of r more prefix elements whose first is >= x
// (host-built suffix sums, travelling as a kernel argument).
constexpr int kWeightedMaxGates = 72;
constexpr int kWeightedRow = 76;
struct WeightedTickets {
  uint32_t group_pairs;   // 0 = not in use
  uint32_t total;         // tickets of the whole sweep = w[3][0]
  uint32_t w[4][kWeightedRow];
};

__device__ __forceinline__ void unrank_weighted_warp(uint32_t t, int np,
    const uint32_t (*__restrict__ w)[kWeightedRow], int *pre, uint32_t &group, int lane) {
  int x0 = 0;
#pragma unroll
  for (int pos = 0; pos < 4; pos++) {
    const int r = 4 - pos;
    const uint32_t *wr = w[r - 1];
    const uint32_t total = wr[x0];
    int cnt = 0;
    for (int y0 = x0;; y0 += 32) {
      const int y = y0 + lane;
      const bool le = y <= np - r && total - wr[min(y, kWeightedRow - 1)] <= t;
      const uint32_t bal = __ballot_sync(kFull, le);
      cnt += __popc(bal);
      if (bal != 0xffffffffu) break;
    }
    const int e = x0 + cnt - 1;
    t -= total - wr[e];
    pre[pos] = e;
    x0 = e + 1;
  }
  group = t;
}

// ------------------------------------------------------------------------------------------------
// Phase 1 of search_7lut, position-major form (lut.c:294-327).
//
// One warp per 4-gate prefix (a,b,c,d); lanes take the (e,f) pairs; the last gate g is not
// enumerated at all: each lane computes the SET of feasible g as a bit vector over gates.
// For a mixed cell C of the prefix and each of the four (e,f)-parts of it, let A / B be the part's
// positions with target 1 / 0.  If both are non-empty, g is admissible for that part iff it is
// constant on A, constant on B and different between them, i.e. iff bit g of
//     AND_{p in part} xr[p]   |   ~OR_{p in part} xr[p]
// is set (xr = position-major rows, complemented where the target is 0).  Intersecting over parts and
// cells gives exactly the g for which check_n_lut_possible(7, ...) holds (lut.c:34-66); the vector
// usually empties after the first cell.  Cost per lane: ~30 instructions per visited position for
// up to 64 candidate g, against ~100 per (pair, cell) in k_sweep.
// W = 32-bit words of candidate gates handled per pass: 1 when n <= 32, else 2.
// P = gates in the prefix a warp owns: 4 (lanes take (e,f) pairs, four parts per cell) or 5 (lanes
// take single gates f, two parts per cell: half the masked-accumulate work per position and half
// the positions per cell, at the price of fewer busy lanes -- it wins once n - 7 approaches a warp).
// FS ("free seen"): when all candidate gates fit one pass and leave the top bit of the last word
// unused (n <= 31 with W = 1, n <= 63 with W = 2), the host stores the position's target bit there;
// the AND / OR accumulators then also tell which targets a part has seen (OR = some 1, AND = only 1s)
// and the separate bookkeeping disappears from the inner loop.
// SH ("shifted window", n <= 63, W = 1, FS): at small n a lane has few candidate last gates -- all of
// them above the prefix -- so instead of aligned 64-gate windows the CTA keeps, for every possible
// first g (= window base 6 .. n-1), a copy of the rows shifted down to it (31 gates per word, the
// target bit on top; (n - 6) * m words of shared memory, built once at the start of the kernel); one
// word per position then covers every candidate of nearly every prefix and the position loop does
// half the accumulates.  A chunk's windows start at the smallest candidate g of its live lanes, so
// they are often much shorter than the prefix's range: windows with <= 15 gates use the PACKED form
// and windows with <= 7 gates the QUAD form (see the cell loop).
// CTAs per SM the register allocation aims at: 3 for the shifted-window form (about 80 registers,
// against 2 CTAs with about 113; the gain measured for 3 was small, and it has not been re-measured
// on the H100), 2 for the two-word forms of larger n (a cap of 80 spills there).
#ifndef SBG_FILTER_MIN_CTAS
#define SBG_FILTER_MIN_CTAS (SH ? 3 : 2)
#endif
constexpr int kQuadGates = 7;   // QUAD windows: 7 candidate gates + the target bit per byte
// SIEVE (SH only): a 7-tuple is feasible iff every masked (target 1, target 0) pair of positions is
// told apart by one of its gates.  Within a mixed cell of the prefix a, b, c and d agree on every
// such pair, so (e,f,g) must separate all of the cell's pairs; the gates that separate pair
// (p,q) are S = ~(xr[p] ^ xr[q]) over the gate bits.  Per prefix the warp takes up to 64 such pairs
// (each position of a mixed cell with the first position of the other target in its cell) and
// keeps, per warp, S[u] for each pair u and
// sep[x] = the pairs gate x separates.  A lane with pair (e,f) then only has to intersect its
// candidate g with S[u] for the pairs u neither e nor f separates -- a necessary condition, usually
// empty after a few pairs.  Lanes and chunks that keep candidates go through the exact cell loop,
// seeded with what the sieve left.
constexpr int kSievePairs = 64;
constexpr int kSieveWords = 4 * kSievePairs;   // per warp: S[64] and sep[64], 64-bit words
// SV: the sieve is compiled in (SH only); without it the shifted form is the plain cell loop.
template <int NW, int W, int P, bool FS, bool SH = false, bool SV = false>
__global__ void __launch_bounds__(kThreads, SBG_FILTER_MIN_CTAS) k_filter7_pm(const DevProblem *__restrict__ prob,
    DevCtl *__restrict__ ctl, uint64_t *__restrict__ hits, uint64_t *__restrict__ aux,
    uint32_t *__restrict__ tcount, uint32_t *__restrict__ gcount, unsigned long long hits_cap,
    unsigned long long tickets_cap, int part, int nparts, unsigned long long list_cap, int batch,
    int max_warps, unsigned long long t_offset, unsigned long long chunk_items,
    int chunks_per_prefix, unsigned long long chunk_tickets, unsigned long long seg_base,
    int packed_gates, const WeightedTickets wt) {
  constexpr int K = 7, NC = 1 << P, NP = P == 4 ? 4 : 2;
  extern __shared__ uint32_t smem[];
  __shared__ uint32_t s_wt[4][kWeightedRow];
  // Work is handed out through one ordered ticket counter, in lexicographic order, under one stop
  // rule (no new ticket once the list cap is reached; what was handed out is finished).  Two kinds
  // of ticket:
  //  * the first chunk_tickets tickets are (prefix, chunk of 32 lane items) pairs over the first
  //    prefixes made of ALLOWED gates only (inbits skipped in the enumeration).  They are the
  //    heaviest prefixes, so this spreads the kernel's longest items over many warps; and because
  //    little work is in flight, a list that fills from the first prefixes -- small masks, where
  //    most combinations are feasible -- ends the sweep after microseconds, whatever n is;
  //  * the rest are batches of whole prefixes from prefix rank t_offset on (the first prefix the
  //    chunk tickets do not cover): less bookkeeping per combination, the form for sweeps that
  //    have to cover everything.
  //
  // ORDERED EMISSION.  The reference's list is in lexicographic order for free (lut.c:316-349); here
  // hits are produced by thousands of warps at once.  Ticket numbers are monotone in lexicographic
  // order, a ticket is worked on by one warp, and that warp meets the ticket's hits in increasing
  // order.  So every hit is stored (anywhere: one atomic reserves the slots of a chunk) together
  // with (ticket b, index j among the ticket's hits), the warp leaves the ticket's hit count in
  // tcount[b], and the place of the hit in the ordered list is  prefix_sum(tcount)[b] + j  --
  // k_offsets does the prefix sum, k_scatter the move.  No sort.
  wait_for_predecessor();   // the chain's first kernel derives the problem block and its rows
  const int n = prob->n;
  const int m = prob->m;
  const int npad = (n + 3) & ~3;
  const int ngw = (((n + 31) >> 5) + 1) & ~1;      // gate words per row, even
  uint32_t *s_tabs = smem;                         // NW * npad   gate-major
  uint32_t *s_xr = smem + NW * npad;               // m * ngw     position-major
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  uint32_t *cells = s_xr + ((m * ngw + 3) & ~3) + warp * (NC * NW);
  // per warp: the surviving-g vectors of one chunk, word-major (vs[word * 32 + lane])
  uint32_t *vs = s_xr + ((m * ngw + 3) & ~3) + kWarpsPerCta * (NC * NW) + warp * (ngw * 32);
  // SV only: the warp's sieve tables, S[u] at s_sieve[u] and sep[x] at s_sieve[kSievePairs + x]
  uint64_t *s_sieve = reinterpret_cast<uint64_t *>(s_xr + ((m * ngw + 3) & ~3)
      + kWarpsPerCta * (NC * NW + ngw * 32) + warp * kSieveWords);
  // SH only: the shifted rows for EVERY window base 6 .. n-1 (a prefix's first window starts at its
  // last gate + 3 >= 6), sxt[(base - 6) * m + p]; built once per CTA, read by all its warps
  uint32_t *sxt = s_xr + ((m * ngw + 3) & ~3)
      + kWarpsPerCta * (NC * NW + ngw * 32 + (SV ? kSieveWords : 0));
  static_assert(!SH || (W == 1 && P == 4 && FS), "shifted windows: one word, 4-gate prefixes, n <= 63");
  static_assert(!SV || SH, "the sieve is part of the shifted-window form");
  const uint32_t sxt_top = (uint32_t)__cvta_generic_to_shared(sxt + 31);   // row 31 of base 6
  const uint32_t xr_base = (uint32_t)__cvta_generic_to_shared(s_xr);
  const uint32_t neg_row_bytes = 0u - (uint32_t)ngw * 4u;   // one multiply-add per address
  // 0x7fffffff held in a register: as a literal the compiler re-creates it at every position, and
  // as a warp-uniform value it copies it from a uniform register at every position (max_warps is
  // never negative; the arithmetic only hides the constant from constant folding and uniformity)
  const uint32_t low31 = 0x7fffffffu ^ (((uint32_t)max_warps >> 31) & (uint32_t)lane);

  if (chain_is_over(ctl) || volatile_load32(&ctl->skip7) != 0) return;
  // position-major rows: 8-byte cp.async chunks, one row per warp at a time (no division); they
  // complete together with the gate-major tables (stage_tables commits and waits for both)
  for (int p = warp; p < m; p += kWarpsPerCta) {
    if (lane < (ngw >> 1)) {
      __pipeline_memcpy_async(s_xr + p * ngw + 2 * lane, &prob->xr[p][2 * lane], 8);
    }
  }
  if (P == 4 && wt.group_pairs != 0) {
    for (int i = threadIdx.x; i < 4 * kWeightedRow; i += blockDim.x) {
      s_wt[i / kWeightedRow][i % kWeightedRow] = wt.w[i / kWeightedRow][i % kWeightedRow];
    }
  }
  stage_tables(s_tabs, prob, NW, npad);
  if constexpr (SH) {
    // Window `base` = gates base .. base+30 in bits 0..30 and the row's target bit on top -- or, where
    // at most packed_gates gates remain (PACKED, below), 15 gates + the target bit, twice over; or,
    // where at most kQuadGates remain as well (QUAD), 7 gates + the target bit, four times over.
    for (int base = 6 + warp; base < n; base += kWarpsPerCta) {
      const bool packed_b = n - base <= packed_gates;
      const bool quad_b = packed_b && n - base <= kQuadGates;
      for (int pp = lane; pp < m; pp += 32) {
        const uint32_t lo = s_xr[pp * ngw], hi = s_xr[pp * ngw + 1];
        const uint32_t tb = (n <= 31 ? lo : hi) & 0x80000000u;   // the row's target bit
        const uint32_t v = base < 32 ? __funnelshift_r(lo, hi, base) : (hi >> (base - 32));
        const uint32_t half = (v & 0x7fffu) | (tb >> 16);
        const uint32_t quarter = (v & 0x7fu) | (tb >> 24);
        sxt[(base - 6) * m + pp] = quad_b ? quarter * 0x01010101u
            : packed_b ? (half | (half << 16)) : ((v & 0x7fffffffu) | tb);
      }
    }
    __syncthreads();
  }
  // overflow retry: only the first max_warps warps work (bounds the hits in flight)
  if (max_warps > 0 && (int)(blockIdx.x * kWarpsPerCta + warp) >= max_warps) return;

  uint32_t T[NW], M[NW];
#pragma unroll
  for (int w = 0; w < NW; w++) {
    T[w] = prob->T[w];
    M[w] = prob->M[w];
  }
  const uint32_t inmask = prob->inmask;
  const uint64_t total = c_binom[n - (K - P)][P];
  unsigned long long swept_lane = 0;   // T-units this lane put through the test (summed at the end)
#ifndef SBG_FETCH_DEPTH
#define SBG_FETCH_DEPTH 1   // tickets fetched ahead; 2 was slower on bench.py's step (n = 40)
#endif
  // tickets in flight per warp: with every warp of the machine taking tickets from one counter,
  // the latency of the atomic under load is of the order of one ticket's work
  constexpr int kDepth = SBG_FETCH_DEPTH;
  unsigned long long q_b[kDepth], q_hc[kDepth];
  unsigned long long next_b = 0, next_hc = 0;
  // A ticket and the hit count as it stood when the ticket was taken -- two independent requests to
  // the same cache line, the load first, so neither waits for the other and both have arrived when
  // they are looked at one ticket later.  The stop rule is evaluated on that pair: a ticket taken
  // when the cap was already reached is dropped, and (tickets being handed out in order) every hit
  // counted at that moment came from a lower ticket, so nothing that belongs to the first list_cap
  // entries is lost.
  auto fetch = [&]() {
    if (lane == 0) {
      next_hc = volatile_load(&ctl->hit_count);
      next_b = atomicAdd(&ctl->ticket, 1ull);
    }
  };
  // In the overflow retry (max_warps > 0) tickets are taken synchronously: a ticket fetched ahead
  // would be worked on even if the cap was reached meanwhile, doubling the hits in flight.
  const bool ahead = max_warps == 0;
  const int n_allowed = n - __popc(inmask & 0xffu);
  if (ahead) {
#pragma unroll
    for (int i = 0; i < kDepth; i++) {
      fetch();
      q_b[i] = next_b;
      q_hc[i] = next_hc;
    }
  }
  for (;;) {
    if (!ahead) {
      fetch();
      q_b[0] = next_b;
      q_hc[0] = next_hc;
    }
    const unsigned long long b = __shfl_sync(kFull, q_b[0], 0);
    const unsigned long long hc_then = __shfl_sync(kFull, q_hc[0], 0);
    if (b >= tickets_cap) {   // the ticket table is too small for this sweep: the host continues it
      if (lane == 0 && hc_then < list_cap) atomicMax(&ctl->overflow, 2u);
      break;
    }
    if (hc_then >= list_cap) {   // the list was complete before this ticket was handed out
      if (lane == 0) tcount[b] = 0;
      break;
    }
    uint32_t tj = 0;          // hits of this ticket so far
    uint64_t t_first, t_end;
    uint32_t q_begin = 0, q_limit = 0xffffffffu;
    // A sweep whose tickets outnumber the ticket table runs as several launches ("segments"); this
    // one hands out tickets seg_base, seg_base + 1, ... and indexes its table from zero.
    // Dealt to the parts of a sharded search in blocks of kDeal consecutive items, see k_sweep.
    const unsigned long long bg = seg_base + b;
    const bool weighted = P == 4 && wt.group_pairs != 0;   // every ticket = (prefix, group of pairs)
    const bool chunked = !weighted && bg < chunk_tickets;
    const uint64_t lt = (chunked || weighted) ? bg : (bg - chunk_tickets) * (uint64_t)batch;
    const uint64_t dealt = dealt_item(lt, part, nparts);
    bool valid = true;
    if (weighted) {
      if (dealt >= (uint64_t)wt.total) {   // past the end: every later ticket is, too
        if (lane == 0) tcount[b] = 0;
        break;
      }
      t_first = 0;
      t_end = 1;
    } else if (chunked) {
      valid = dealt < chunk_items;   // the last deal block is shorter for some parts
      t_first = dealt / (uint64_t)chunks_per_prefix;
      t_end = t_first + 1;
      q_begin = (uint32_t)(dealt % (uint64_t)chunks_per_prefix) * 32u;
      q_limit = q_begin + 32u;
    } else {
      t_first = t_offset + dealt;
      if (t_first >= total) {        // past the end: every later ticket is, too
        if (lane == 0) tcount[b] = 0;
        break;
      }
      t_end = min(t_first + (uint64_t)batch, total);
    }
    if (ahead) {   // the queue moves up, a new ticket is requested for its end
#pragma unroll
      for (int i = 0; i + 1 < kDepth; i++) {
        q_b[i] = q_b[i + 1];
        q_hc[i] = q_hc[i + 1];
      }
      fetch();
      q_b[kDepth - 1] = next_b;
      q_hc[kDepth - 1] = next_hc;
    }
    if (valid) {
    int pre[P];
    uint64_t unused_rank;
    if constexpr (P == 4) {
      if (weighted) {
        uint32_t group;
        unrank_weighted_warp((uint32_t)dealt, n - (K - P), s_wt, pre, group, lane);
        q_begin = group * wt.group_pairs;
        q_limit = q_begin + wt.group_pairs;
      }
    }
    if (!weighted) {
      unrank_prefix_warp<P, K, false>(t_first, chunked ? n_allowed : n, pre, unused_rank, lane);
    }
    if (chunked) {   // index among the allowed gates -> gate number (excluded gates are < 8)
#pragma unroll
      for (int i = 0; i < P; i++) {
        int g = pre[i];
#pragma unroll
        for (int bit = 0; bit < 8; bit++) g += (((inmask >> bit) & 1u) != 0 && bit <= g) ? 1 : 0;
        pre[i] = g;
      }
    }
    for (uint64_t gt = t_first; gt < t_end; gt++) {
      if (gt != t_first) {
        int i = P - 1;
        while (i > 0 && pre[i] + (P - i) >= n - (K - P)) i--;
        pre[i]++;
        for (int k2 = i + 1; k2 < P; k2++) pre[k2] = pre[k2 - 1] + 1;
      }
      const int last = pre[P - 1];
      const int r = n - last - 2;                   // candidates for (e,)f: last+1 .. n-2
      const uint32_t Q = P == 4 ? (uint32_t)(r * (r - 1) / 2) : (uint32_t)r;
      if (q_begin >= max(Q, 1u)) continue;          // head launch: no such chunk in this prefix
      bool rejected = false;
#pragma unroll
      for (int i = 0; i < P; i++) rejected |= (pre[i] < 8) && ((inmask >> pre[i]) & 1u);
      if (rejected) {
        // the reference steps through these one by one (lut.c:294-305): T-units all the same
        if (q_begin == 0 && lane == 0) swept_lane += c_binom[n - last - 1][K - P];
        continue;
      }

      // mixed cells of the prefix (cell = lane mod NC, first gate most significant).  With 16 cells
      // and several table words the two half-warps take half the words each.
      uint32_t mixed_ballot;
      {
        constexpr bool kSplit = NC == 16 && NW >= 2;
        constexpr int NWH = kSplit ? NW / 2 : NW;
        const bool upper = kSplit && lane >= 16;
        const int cell = lane & (NC - 1);
        const uint32_t *tabs_h = s_tabs + (upper ? NWH * npad : 0);
        uint32_t c[NWH];
        uint32_t ones = 0, zeros = 0;
#pragma unroll
        for (int k = 0; k < NWH; k++) {
          uint32_t tt = upper ? M[kSplit ? k + NWH : k] : M[k];
          const uint32_t tw = upper ? T[kSplit ? k + NWH : k] : T[k];
#pragma unroll
          for (int i = 0; i < P; i++) {
            const uint32_t tv = tabs_h[k * npad + pre[i]];
            tt &= ((cell >> (P - 1 - i)) & 1) ? tv : ~tv;
          }
          c[k] = tt;
          ones |= tt & tw;
          zeros |= tt & ~tw;
        }
        if (kSplit) {
          ones |= __shfl_xor_sync(kFull, ones, 16);
          zeros |= __shfl_xor_sync(kFull, zeros, 16);
        }
        const bool mixed = ones != 0 && zeros != 0;   // both halves of a split warp agree
        mixed_ballot = __ballot_sync(kFull, mixed) & (NC == 32 ? 0xffffffffu : ((1u << (NC & 31)) - 1u));
        __syncwarp();
        if (mixed) {
          const int slot = __popc(mixed_ballot & ((1u << cell) - 1u));
#pragma unroll
          for (int k = 0; k < NWH; k++) cells[slot * NW + (upper ? NWH : 0) + k] = c[k];
        }
        __syncwarp();
      }
      const int mc = __popc(mixed_ballot);
#ifdef SBG_COUNT_FILTER
      unsigned long long dbg_chunks = 0, dbg_windows = 0, dbg_cells = 0, dbg_pos = 0, dbg_packed = 0;
      unsigned long long dbg_quad = 0, dbg_sieve = 0, dbg_exact = 0;
      unsigned long long dbg_mc = (unsigned long long)mc;
#endif
      if constexpr (SV) {
        {
          // the sieve's pairs, all mixed cells at once: every masked position p of a mixed cell is
          // paired with the first position of the other target in its cell (lane j < mc holds those
          // of mixed cell j), except the first target-0 position, whose pair the first target-1
          // position already has; positions in order, word by word, up to 64 pairs.  No loop over
          // cells and no dependent shared-memory round trips per cell.
          const uint64_t gmask = (1ull << n) - 1u;   // gate bits: no target bit, no padding
          int rep1 = 0, rep0 = 0;
          if (lane < mc) {
            bool f1 = false, f0 = false;
#pragma unroll
            for (int w = 0; w < NW; w++) {
              const uint32_t c = cells[lane * NW + w];
              const uint32_t a = c & T[w], bq = c & ~T[w];
              if (!f1 && a != 0) rep1 = w * 32 + __ffs(a) - 1;
              if (!f0 && bq != 0) rep0 = w * 32 + __ffs(bq) - 1;
              f1 |= a != 0;
              f0 |= bq != 0;
            }
          }
          int npairs = 0;
#pragma unroll
          for (int w = 0; w < NW; w++) {
            if (npairs < kSievePairs) {   // warp-uniform
              const int p = w * 32 + lane;
              uint32_t cell = 0;
#pragma unroll
              for (int i = 0; i < P; i++) cell = (cell << 1) | ((s_tabs[w * npad + pre[i]] >> lane) & 1u);
              const bool t1 = ((T[w] >> lane) & 1u) != 0;
              const int slot = __popc(mixed_ballot & ((1u << cell) - 1u));
              const int r1 = __shfl_sync(kFull, rep1, slot), r0 = __shfl_sync(kFull, rep0, slot);
              const int q = t1 ? r0 : r1;
              const bool paired = ((M[w] >> lane) & 1u) != 0 && ((mixed_ballot >> cell) & 1u) != 0
                  && (t1 || p != r0);
              const uint32_t bal = __ballot_sync(kFull, paired);
              const int u = npairs + __popc(bal & lanemask_lt());
              if (paired && u < kSievePairs) {
                const uint64_t xp = *reinterpret_cast<const uint64_t *>(s_xr + p * ngw);
                const uint64_t xq = *reinterpret_cast<const uint64_t *>(s_xr + q * ngw);
                s_sieve[u] = ~(xp ^ xq) & gmask;
              }
              npairs = min(kSievePairs, npairs + __popc(bal));
            }
          }
          __syncwarp();
          // entries past npairs are stale; their bits are masked below and never read
          const uint64_t s_lo = s_sieve[lane], s_hi = s_sieve[lane + 32];
          // sep[x] for the gates that can be e or f; pairs past npairs count as separated, so that
          // a prefix without mixed cells (npairs = 0) passes everything
          const uint64_t unused = npairs >= kSievePairs ? 0ull : ~0ull << npairs;
          for (int x = last + 1; x <= n - 2; x++) {
            const uint32_t lo = __ballot_sync(kFull, ((s_lo >> x) & 1u) != 0);
            const uint32_t hi = npairs > 32 ? __ballot_sync(kFull, ((s_hi >> x) & 1u) != 0) : 0u;
            if (lane == 0) s_sieve[kSievePairs + x] = (((uint64_t)hi << 32) | lo) | unused;
          }
          __syncwarp();
        }
      }

      unsigned long long emitted = 0;
      bool prefix_done = false;
      // the lane's pair (e, f) = (last+1+run_i, last+1+run_j): unranked once (square root), then
      // moved on by 32 places per chunk
      int run_i = 0, run_j = 1;
      if (P == 4 && q_begin + (uint32_t)lane < Q) unrank_pair(q_begin + (uint32_t)lane, r, run_i, run_j);
      for (uint32_t q0 = q_begin; q0 < min(Q, q_limit) && !prefix_done; q0 += 32) {
        const uint32_t q = q0 + lane;
        bool lane_ok = q < Q;
#ifdef SBG_COUNT_FILTER
        dbg_chunks++;
#endif
        int pi = 0, pj = 0;
        if (P == 4) {
          if (q0 != q_begin) {
            run_j += 32;
            while (run_j >= r && run_i < r - 2) {   // into the next row(s): row i holds j = i+1 .. r-1
              run_i++;
              run_j += run_i + 1 - r;
            }
          }
          pi = lane_ok ? run_i : 0;   // lanes past the end read the tables of pair (0, 1)
          pj = lane_ok ? run_j : 1;
        } else {
          pj = lane_ok ? (int)q : 0;
        }
        const int ge = P == 4 ? last + 1 + pi : pre[P - 1];   // P == 5: e is the prefix's last gate
        const int gf = last + 1 + pj;
        if (lane_ok) swept_lane += (unsigned long long)(n - 1 - gf);   // T-units: every g > f
        if (P == 4 && ge < 8 && ((inmask >> ge) & 1u)) lane_ok = false;
        if (gf < 8 && ((inmask >> gf) & 1u)) lane_ok = false;
        // the lane's e / f tables are read from shared memory word by word where they are used
        // (once per cell and word) instead of living in 2 x NW registers across the whole chunk
        const uint32_t *tab_e = s_tabs + ge, *tab_f = s_tabs + gf;
        // windows of 32*W candidate gates g, from the first that can hold the smallest possible g
        // (SH: windows of 31 gates starting AT the chunk's smallest candidate g, wb counts them)
        int first_g = last + (K - P);
        uint64_t cand = 0;   // SV: the lane's candidate g, gf < g < n, excluded gates out, sieved
        if constexpr (SV) {
          if (lane_ok) cand = ((1ull << n) - 1u) & (~0ull << (gf + 1)) & ~(uint64_t)(inmask & 0xffu);
          {
            const uint64_t sepd = s_sieve[kSievePairs + ge] | s_sieve[kSievePairs + gf];
            // the pairs neither e nor f separates, in two halves taken a pair each per step: two
            // independent load chains instead of one
            uint32_t u_lo = ~(uint32_t)sepd, u_hi = ~(uint32_t)(sepd >> 32);
#ifdef SBG_COUNT_FILTER
            uint32_t its = 0;
#endif
            while ((u_lo | u_hi) != 0 && cand != 0) {
              const uint64_t s_a = u_lo != 0 ? s_sieve[__ffs(u_lo) - 1] : ~0ull;
              const uint64_t s_b = u_hi != 0 ? s_sieve[31 + __ffs(u_hi)] : ~0ull;
              cand &= s_a & s_b;
              u_lo &= u_lo - 1;
              u_hi &= u_hi - 1;
#ifdef SBG_COUNT_FILTER
              its++;
#endif
            }
#ifdef SBG_COUNT_FILTER
            dbg_sieve += __reduce_max_sync(kFull, its);
#endif
          }
          // a lane needs only its candidates: the chunk's windows start at the lowest of its lanes
          // (often well above the prefix's last + 3), so that more of them take the packed forms
          const uint32_t lo = __reduce_min_sync(kFull, cand != 0 ? (uint32_t)(__ffsll((long long)cand) - 1)
                                                                 : (uint32_t)n);
          if (lo >= (uint32_t)n) continue;   // no candidate left in any lane: nothing to test or emit
          first_g = (int)lo;
#ifdef SBG_COUNT_FILTER
          dbg_exact++;
#endif
        } else if constexpr (SH) {
          // a lane needs only g > f: the chunk's windows start at the lowest gf + 1 of its live lanes
          // (often well above the prefix's last + 3), so that more of them take the packed forms
          const uint32_t lo = __reduce_min_sync(kFull, lane_ok ? (uint32_t)(gf + 1) : (uint32_t)n);
          if (lo >= (uint32_t)n) continue;   // no live lane: nothing to test or emit
          first_g = (int)lo;
        }
        const int wb0 = SH ? 0 : ((first_g >> 5) & ~(W - 1));
        int nvw = 0;      // words of surviving-g vectors stored for this chunk
        bool chunk_live = false;   // some lane kept a candidate in some window
        for (int wb = wb0; SH ? (first_g + 31 * wb < n) : (wb < ((n + 31) >> 5)); wb += W) {
          const int base = SH ? first_g + 31 * wb : 0;
          // PACKED (SH only): a window with at most 15 candidate last gates keeps TWO parts in one
          // accumulator register -- halves of 15 gates + the target bit each, the shifted rows stored
          // twice over -- so a position costs 2 part masks + 4 accumulates instead of 4 + 8.
          // QUAD: at most 7 candidates, all FOUR parts in one register, a byte each: 2 + 2.
          const bool packed = SH && n - base <= packed_gates;   // 15, or 0 = never
          const bool quad = packed && n - base <= kQuadGates;
          const uint32_t sx_top = sxt_top + (uint32_t)((base - 6) * m) * 4u;
          uint32_t V[W];
          if constexpr (SV) {
            V[0] = (uint32_t)(cand >> base) & 0x7fffffffu;   // gates base .. base+30
          } else if constexpr (SH) {
            uint32_t v = 0x7fffffffu;                // gates base .. base+30: keep gf < g < n
            if (n - base < 31) v = 0x7fffffffu >> (31 - (n - base));
            if (gf + 1 - base >= 31) v = 0u;
            else if (gf + 1 - base > 0) v &= 0xffffffffu << (gf + 1 - base);
            if (base < 8) v &= ~(inmask >> base);
            V[0] = lane_ok ? v : 0u;
          } else {
#pragma unroll
            for (int j = 0; j < W; j++) {
              const int g0 = (wb + j) * 32;           // gates g0 .. g0+31: keep gf < g < n
              uint32_t v = 0xffffffffu;
              if (n - g0 < 32) v = (n - g0 <= 0) ? 0u : (0xffffffffu >> (32 - (n - g0)));
              if (gf + 1 - g0 >= 32) v = 0u;
              else if (gf + 1 - g0 > 0) v &= 0xffffffffu << (gf + 1 - g0);
              if (g0 == 0) v &= ~inmask;
              V[j] = lane_ok ? v : 0u;
            }
          }
          bool alive = false;
#pragma unroll
          for (int j = 0; j < W; j++) alive |= V[j] != 0;
#ifdef SBG_COUNT_FILTER
          dbg_windows++;
          if (packed && !quad) dbg_packed++;
          if (quad) dbg_quad++;
#endif
          bool any_alive = __any_sync(kFull, alive);
          for (int cj = 0; cj < mc && any_alive; cj++) {
#ifdef SBG_COUNT_FILTER
            dbg_cells++;
            for (int w = 0; w < NW; w++) dbg_pos += __popc(cells[cj * NW + w]);
#endif
            if constexpr (SH) {
              if (quad) {
                // part 2e + f in byte 2e + f of (aq, oq): e picks the half, f the byte within it
                uint32_t aq = 0xffffffffu, oq = 0u;
#pragma unroll
                for (int w = 0; w < NW; w++) {
                  uint32_t bits = cells[cj * NW + w];
                  const uint32_t tf_w = tab_f[w * npad];
                  const uint32_t te_w = tab_e[w * npad];
                  while (bits != 0) {
                    const int c = clz_nonzero(bits);
                    bits &= low31 >> c;
                    const uint32_t fb = (uint32_t)((int32_t)(tf_w << c) >> 31);
                    const uint32_t eb = (uint32_t)((int32_t)(te_w << c) >> 31);
                    const uint32_t x = lds_u32(sx_top + (uint32_t)(w * 128) - 4u * (uint32_t)c);
                    const uint32_t mq = lop3<0x60>(eb ^ 0x0000ffffu, fb, 0x00ff00ffu);   // a & (b ^ c)
                    aq = lop3<0xd0>(aq, x, mq);
                    oq = lop3<0xf8>(oq, x, mq);
                  }
                }
                // per byte: admissible g = constant over the part, or the part lacks a target value
                // (bit 7 of a byte: OR = some target 1 seen, AND = only target 1 seen); the sign
                // of each byte of z spread over the byte, then the four bytes ANDed into the low one
                uint32_t t = prmt_sign_bytes(oq & ~aq);
                t = aq | ~oq | ~t;
                t &= t >> 16;
                t &= t >> 8;
                V[0] &= t;
                alive = V[0] != 0;
                any_alive = __any_sync(kFull, alive);
                continue;
              }
              if (packed) {
                // parts 0 | 1 in the low | high half of (and01, or01), parts 2 | 3 of (and23, or23)
                uint32_t and01 = 0xffffffffu, or01 = 0u, and23 = 0xffffffffu, or23 = 0u;
                const uint32_t low_half = 0x0000ffffu ^ ((uint32_t)max_warps >> 31);
#pragma unroll
                for (int w = 0; w < NW; w++) {
                  uint32_t bits = cells[cj * NW + w];
                  const uint32_t tf_w = tab_f[w * npad];
                  const uint32_t te_w = tab_e[w * npad];
                  while (bits != 0) {
                    const int c = clz_nonzero(bits);
                    bits &= low31 >> c;
                    const uint32_t fb = (uint32_t)((int32_t)(tf_w << c) >> 31);
                    const uint32_t eb = (uint32_t)((int32_t)(te_w << c) >> 31);
                    const uint32_t x = lds_u32(sx_top + (uint32_t)(w * 128) - 4u * (uint32_t)c);
                    // the half this position's part lives in: f picks the half, e the register
                    const uint32_t m01 = lop3<0x06>(eb, fb, low_half);   // ~eb & (fb ^ low_half)
                    const uint32_t m23 = lop3<0x60>(eb, fb, low_half);   //  eb & (fb ^ low_half)
                    and01 = lop3<0xd0>(and01, x, m01);
                    or01 = lop3<0xf8>(or01, x, m01);
                    and23 = lop3<0xd0>(and23, x, m23);
                    or23 = lop3<0xf8>(or23, x, m23);
                  }
                }
                // per half: admissible g = constant over the part, or the part lacks a target value
                // (bit 15 of a half: OR = some target 1 seen, AND = only target 1 seen)
                uint32_t v = V[0];
                {
                  const uint32_t z = or01 & ~and01, adm = and01 | ~or01;
                  v &= (adm | ~(uint32_t)((int32_t)(z << 16) >> 31))
                      & ((adm >> 16) | ~(uint32_t)((int32_t)z >> 31));
                }
                {
                  const uint32_t z = or23 & ~and23, adm = and23 | ~or23;
                  v &= (adm | ~(uint32_t)((int32_t)(z << 16) >> 31))
                      & ((adm >> 16) | ~(uint32_t)((int32_t)z >> 31));
                }
                V[0] = v;
                alive = v != 0;
                any_alive = __any_sync(kFull, alive);
                continue;
              }
            }
            uint32_t a_and[NP][W], a_or[NP][W];
#pragma unroll
            for (int k = 0; k < NP; k++) {
#pragma unroll
              for (int j = 0; j < W; j++) {
                a_and[k][j] = 0xffffffffu;
                a_or[k][j] = 0u;
              }
            }
            uint32_t seen1[NP], seen0[NP];
#pragma unroll
            for (int k = 0; k < NP; k++) seen1[k] = seen0[k] = 0u;
#pragma unroll
            for (int w = 0; w < NW; w++) {
              uint32_t bits = cells[cj * NW + w];
              const uint32_t tf_w = tab_f[w * npad];
              const uint32_t te_w = P == 4 ? tab_e[w * npad] : 0u;
              // shared-window address of row w*32+31 of this window (aligned two-word windows)
              const uint32_t row_top = xr_base + (uint32_t)((w * 32 + 31) * ngw + wb) * 4u;
              while (bits != 0) {                     // warp-uniform loop over the cell's positions
                // from the top bit down: the leading-zero count is at once the shift that brings
                // the position's bit of a table to the sign position
                const int c = clz_nonzero(bits);
                bits &= low31 >> c;
                const int p = w * 32 + 31 - c;
                const uint32_t tp = (T[w] << c) >> 31;
                // eb / fb = bit j of the lane's e / f table spread over a whole word (shift it to
                // the sign position, arithmetic shift back): all-ones / zero masks without a
                // predicate, so that every masked accumulate below is ONE three-input LOP3.
                const uint32_t fb = (uint32_t)((int32_t)(tf_w << c) >> 31);
                const uint32_t eb = P == 4 ? (uint32_t)((int32_t)(te_w << c) >> 31) : 0u;
                uint32_t x[W];
                if (W == 2) {
                  const uint2 xx = lds_v2(row_top + neg_row_bytes * (uint32_t)c);
                  x[0] = xx.x;
                  x[W - 1] = xx.y;
                } else if (SH) {
                  x[0] = lds_u32(sx_top + (uint32_t)(w * 128) - 4u * (uint32_t)c);
                } else {
                  x[0] = s_xr[p * ngw + wb];
                }
                uint32_t mk[NP];   // mk[k] = all-ones iff this position lies in part k
                if (P == 4) {   // materialised, so that each accumulate below stays one LOP3
                  mk[0] = lop3<0x03>(eb, fb, 0u);        // ~(eb | fb)
                  mk[1] = lop3<0x0c>(eb, fb, 0u);        // ~eb & fb
                  mk[NP - 2] = lop3<0x30>(eb, fb, 0u);   // eb & ~fb
                  mk[NP - 1] = lop3<0xc0>(eb, fb, 0u);   // eb & fb
                } else {
                  mk[0] = ~fb;
                  mk[NP - 1] = fb;
                }
                // which targets each part has seen: whole-word flags, updated under a warp-uniform
                // branch (tp belongs to the position, not to the lane)
                if (!FS) {
                  if (tp) {
#pragma unroll
                    for (int k = 0; k < NP; k++) seen1[k] |= mk[k];
                  } else {
#pragma unroll
                    for (int k = 0; k < NP; k++) seen0[k] |= mk[k];
                  }
                }
#pragma unroll
                for (int k = 0; k < NP; k++) {
#pragma unroll
                  for (int jw = 0; jw < W; jw++) {
                    a_and[k][jw] = lop3<0xd0>(a_and[k][jw], x[jw], mk[k]);   // a & (x | ~m)
                    a_or[k][jw] = lop3<0xf8>(a_or[k][jw], x[jw], mk[k]);     // a | (x & m)
                  }
                }
              }
            }
#pragma unroll
            for (int k = 0; k < NP; k++) {
              // all-ones iff the part has both targets
              const uint32_t both = FS
                  ? (uint32_t)((int32_t)(a_or[k][W - 1] & ~a_and[k][W - 1]) >> 31)
                  : (seen1[k] & seen0[k]);
#pragma unroll
              for (int jw = 0; jw < W; jw++) V[jw] &= a_and[k][jw] | ~a_or[k][jw] | ~both;
            }
            alive = false;
#pragma unroll
            for (int jw = 0; jw < W; jw++) alive |= V[jw] != 0;
            any_alive = __any_sync(kFull, alive);
          }
          chunk_live |= any_alive;
          // park this window's survivors; the chunk is emitted once all its windows are done, so
          // that a lane's hits come out in increasing g whatever the window they were found in
#pragma unroll
          for (int jw = 0; jw < W; jw++) vs[(nvw + jw) * 32 + lane] = V[jw];
          nvw += W;
        }
        // emit the chunk: lane-major (= (e,f) order), then g ascending
        if (!chunk_live) continue;   // the common case: nothing survived
        int cnt = 0;
        for (int i = 0; i < nvw; i++) cnt += __popc(vs[i * 32 + lane]);
        int incl = cnt;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const int up = __shfl_up_sync(kFull, incl, d);
          if (lane >= d) incl += up;
        }
        const int warp_total = __shfl_sync(kFull, incl, 31);
        unsigned long long base_slot = 0;
        if (lane == 0) base_slot = atomicAdd(&ctl->hit_count, (unsigned long long)warp_total);
        base_slot = __shfl_sync(kFull, base_slot, 0) + (unsigned long long)(incl - cnt);
        uint64_t where = (b << 22) | (uint64_t)(tj + (uint32_t)(incl - cnt));   // (ticket, index in it)
        uint64_t head = 0;
#pragma unroll
        for (int i = 0; i < P; i++) head = (head << 9) | (uint64_t)pre[i];
        if (P == 4) {
          head = (head << 27) | ((uint64_t)ge << 18) | ((uint64_t)gf << 9);
        } else {
          head = (head << 18) | ((uint64_t)gf << 9);
        }
        if (cnt != 0) {
          for (int i = 0; i < nvw; i++) {
            uint32_t v = vs[i * 32 + lane];
            const int g0 = SH ? first_g + 31 * i : (wb0 + i) * 32;
            while (v != 0) {
              const int gbit = __ffs(v) - 1;
              v &= v - 1;
              if (base_slot < hits_cap) {
                hits[base_slot] = head | (uint64_t)(g0 + gbit);
                aux[base_slot] = where;
              } else {
                atomicExch(&ctl->overflow, 1u);
              }
              base_slot++;
              where++;
            }
          }
        }
        tj += (uint32_t)warp_total;
        emitted += (unsigned long long)warp_total;
        // One prefix never needs to contribute more than the list cap (lut.c:316-318); checked only
        // between chunks, when every pair up to here has all its g emitted.
        if (emitted >= list_cap) prefix_done = true;
      }
#ifdef SBG_COUNT_FILTER
      if (lane == 0) {
        atomicAdd(&ctl->pad1[0], 1ull);
        atomicAdd(&ctl->pad1[1], dbg_chunks);
        atomicAdd(&ctl->pad1[2], dbg_windows);
        atomicAdd(&ctl->pad1[3], dbg_cells);
        atomicAdd(&ctl->pad1[4], dbg_pos);
        atomicAdd(&ctl->pad1[5], dbg_packed);
        atomicAdd(&ctl->pad1[6], dbg_mc);
        atomicAdd(&ctl->pad1[7], dbg_quad);
        atomicAdd(&ctl->pad1[8], dbg_sieve);
        atomicAdd(&ctl->pad1[9], dbg_exact);
      }
#endif
    }
    }  // valid
    if (lane == 0) {
      tcount[b] = tj;
      if (tj != 0) atomicAdd(&gcount[b >> 10], tj);
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) swept_lane += __shfl_xor_sync(kFull, swept_lane, d);
  if (lane == 0 && swept_lane != 0) atomicAdd(&ctl->swept, swept_lane);
}

// ------------------------------------------------------------------------------------------------
// Ordered list from ticket-tagged hits (see k_filter7_pm).  k_offsets: exclusive prefix sum of the
// per-ticket hit counts, one CTA per group of 1,024 tickets (the group totals were accumulated by
// the filter itself); k_scatter: every stored hit to its place, cut at the list cap
// (lut.c:291,316-318).
constexpr int kTicketGroup = 1024;

__global__ void __launch_bounds__(256) k_offsets(DevCtl *__restrict__ ctl,
    const uint32_t *__restrict__ tcount, const uint32_t *__restrict__ gcount,
    uint32_t *__restrict__ toffset, unsigned long long tickets_cap, unsigned int list_cap,
    unsigned int list_base) {
  __shared__ unsigned long long s_part[8];
  __shared__ uint32_t s_scan[8];
  wait_for_predecessor();
  if (chain_is_over(ctl) || volatile_load32(&ctl->skip7) != 0) return;
  const unsigned long long handed = min(volatile_load(&ctl->ticket), tickets_cap);
  const unsigned long long first = (unsigned long long)blockIdx.x * kTicketGroup;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const unsigned long long total = (unsigned long long)list_base
        + min(volatile_load(&ctl->hit_count), (unsigned long long)0xffffffffu);
    ctl->list_count = (unsigned int)min(total, (unsigned long long)list_cap);
#ifdef SBG_COUNT_FILTER
    // windows = single (31 gates) + packed (two parts of 15) + quad (four parts of 7); sieve = the
    // slowest lane's sieve iterations summed over chunks, exact = chunks the cell loop still ran on
    printf("F1 prefixes %llu chunks %llu windows %llu cells %llu positions %llu packed %llu mixed %llu hits %llu quad %llu sieve %llu exact %llu\n",
        ctl->pad1[0], ctl->pad1[1], ctl->pad1[2], ctl->pad1[3], ctl->pad1[4], ctl->pad1[5],
        ctl->pad1[6], ctl->hit_count, ctl->pad1[7], ctl->pad1[8], ctl->pad1[9]);
    for (int i = 0; i < 10; i++) ctl->pad1[i] = 0;
#endif
  }
  if (first >= handed) return;
  // hits in front of this group
  unsigned long long before = 0;
  for (unsigned int g = threadIdx.x; g < blockIdx.x; g += blockDim.x) before += gcount[g];
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) before += __shfl_xor_sync(kFull, before, d);
  if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = before;
  __syncthreads();
  before = list_base;
#pragma unroll
  for (int i = 0; i < 8; i++) before += s_part[i];
  // local scan: 4 consecutive tickets per thread
  const unsigned long long t0 = first + 4ull * threadIdx.x;
  uint32_t c[4];
#pragma unroll
  for (int i = 0; i < 4; i++) c[i] = t0 + i < handed ? tcount[t0 + i] : 0u;
  const uint32_t mine = c[0] + c[1] + c[2] + c[3];
  uint32_t incl = mine;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t up = __shfl_up_sync(kFull, incl, d);
    if ((threadIdx.x & 31) >= d) incl += up;
  }
  if ((threadIdx.x & 31) == 31) s_scan[threadIdx.x >> 5] = incl;
  __syncthreads();
  uint32_t warp_base = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) warp_base += i < (int)(threadIdx.x >> 5) ? s_scan[i] : 0u;
  unsigned long long off = before + warp_base + (incl - mine);
#pragma unroll
  for (int i = 0; i < 4; i++) {
    if (t0 + i < handed) toffset[t0 + i] = (uint32_t)min(off, (unsigned long long)0xffffffffu);
    off += c[i];
  }
}

__global__ void __launch_bounds__(256) k_scatter(DevCtl *__restrict__ ctl,
    const uint64_t *__restrict__ hits, const uint64_t *__restrict__ aux,
    const uint32_t *__restrict__ toffset, uint64_t *__restrict__ sorted,
    unsigned long long hits_cap, unsigned int list_cap) {
  wait_for_predecessor();
  if (chain_is_over(ctl) || volatile_load32(&ctl->skip7) != 0) return;
  if (volatile_load32(&ctl->overflow) == 1u) return;   // incomplete hit buffer: the host retries
  const unsigned long long count = min(volatile_load(&ctl->hit_count), hits_cap);
  for (unsigned long long s = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; s < count;
       s += (unsigned long long)gridDim.x * blockDim.x) {
    const uint64_t where = aux[s];
    const unsigned long long pos = (unsigned long long)toffset[where >> 22] + (where & 0x3fffffu);
    if (pos < list_cap) sorted[pos] = hits[s];
  }
}

// Merge of `nruns` ascending runs of packed tuples (the per-part lists of a sharded phase 1, laid
// out run r at src + r * stride, counts[r] entries) into one ascending list cut at list_cap: an
// entry's place is its index in its own run plus the number of smaller entries in every other run
// (binary searches; entries are distinct).  The device-side counterpart of lut.c:329-349.
constexpr int kMaxRuns = 64;
struct RunCounts { uint32_t n[kMaxRuns]; };

__global__ void __launch_bounds__(256) k_merge_runs(const uint64_t *__restrict__ src,
    unsigned long long stride, RunCounts counts, int nruns, uint64_t *__restrict__ dst,
    unsigned int list_cap, DevCtl *__restrict__ ctl) {
  unsigned long long total = 0;
  for (int r = 0; r < nruns; r++) total += counts.n[r];
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    ctl->list_count = (unsigned int)min(total, (unsigned long long)list_cap);
  }
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    int r = 0;
    unsigned long long idx = i;
    while (idx >= counts.n[r]) {
      idx -= counts.n[r];
      r++;
    }
    const uint64_t v = src[(unsigned long long)r * stride + idx];
    unsigned long long pos = idx;
    for (int o = 0; o < nruns; o++) {
      if (o == r) continue;
      const uint64_t *run = src + (unsigned long long)o * stride;
      uint32_t lo = 0, hi = counts.n[o];
      while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (run[mid] < v) lo = mid + 1; else hi = mid;
      }
      pos += lo;
    }
    if (pos < list_cap) dst[pos] = v;
  }
}

// ------------------------------------------------------------------------------------------------
// First kernel of every call chain.
//
// Per-call inputs travel as kernel arguments, not as separate host->device copies: a copy-engine
// transfer of a few hundred bytes costs several microseconds of stream latency, and a real run is
// thousands of searches that last tens of microseconds each.
constexpr int kArgGates = 40;   // gate tables that fit the kernel arguments next to everything else
struct BeginArgs {
  uint8_t pos5[256];       // search_5lut: position of each function in the shuffled order
  uint8_t pos_outer[256];  // search_7lut
  uint8_t pos_middle[256];
  uint16_t order3[512];    // 3-LUT scan: the caller's shuffled gate order (lut.c:501-507)
  unsigned long long seq;
  uint32_t flags;          // kBegin* bits
  uint32_t gcount_n;       // ticket-group counters to clear
  // problem delta (kBeginProblem): the state is n gates under (target, mask, inmask); gates
  // a_first .. a_first + a_count - 1 travel in newg (the others are resident, or were copied into
  // DevProblem::full before the launch); gates from c_first on are (re)compressed.
  int32_t n;
  uint32_t inmask;
  int32_t a_first, a_count;
  int32_t c_first;
  uint32_t target[8];
  uint32_t mask[8];
  uint32_t newg[kArgGates][8];
};
constexpr int kScanKeyBits = 28;                       // stage-0 word: seq << 28 | key
constexpr unsigned long long kScanKeyNone = (1ull << kScanKeyBits) - 1;
constexpr uint32_t kBeginScan3 = 1, kBeginSearch5 = 2, kBeginSearch7 = 4, kBeginRows = 8,
    kBeginKeepCtl = 16, kBeginOrder3 = 32, kBeginProblem = 64;

// Derives the search's working set from the resident uncompressed tables (CTAs of k_begin, or all
// CTAs of k_prepare_problem): tables compressed to the masked positions (word-major tabs, T, M;
// every test of the path is "under the mask", lut.c:38-42,86), the header, and -- when asked -- the
// position-major rows xr: bit g of row p = gate g at masked position p, the row complemented where
// the target is 0; with n <= 31 / n <= 63 the top bit of word 0 / 1 is no gate and carries the
// position's target bit.  One warp builds one 32-bit word at a time (lane = bit, one ballot).  No CTA
// depends on another's output: a gate is read from the arguments if it travels there, else from
// DevProblem::full (which this launch writes for the travelling gates only).
__device__ __forceinline__ uint32_t arg_or_resident(const DevProblem *prob, const BeginArgs &a, int g,
    int w) {
  const int k = g - a.a_first;
  return (k >= 0 && k < a.a_count) ? a.newg[k][w] : prob->full[g][w];
}

__device__ __forceinline__ void prepare_problem(DevProblem *__restrict__ prob, const BeginArgs &a,
    int cta, int nctas) {
  __shared__ uint8_t s_posn[256];   // i-th masked position
  __shared__ uint32_t s_mask[8], s_target[8];
  if (threadIdx.x < 8) {
    s_mask[threadIdx.x] = a.mask[threadIdx.x];
    s_target[threadIdx.x] = a.target[threadIdx.x];
  }
  __syncthreads();
  int m = 0;
#pragma unroll
  for (int w = 0; w < 8; w++) m += __popc(s_mask[w]);
  if (threadIdx.x < 256) {
    const int p = threadIdx.x, w = p >> 5, j = p & 31;
    if ((s_mask[w] >> j) & 1u) {
      int idx = __popc(s_mask[w] & ((1u << j) - 1u));
      for (int k = 0; k < w; k++) idx += __popc(s_mask[k]);
      s_posn[idx] = (uint8_t)p;
    }
  }
  __syncthreads();
  const int n = a.n;
  const int nw = m <= 32 ? 1 : m <= 64 ? 2 : m <= 128 ? 4 : 8;
  const int lane = threadIdx.x & 31;
  const int warps = blockDim.x >> 5;
  const int wid = cta * warps + (threadIdx.x >> 5);
  const int nwarps = nctas * warps;
  if (cta == 0 && threadIdx.x < 8) {
    const int w = threadIdx.x;
    uint32_t t = 0, mm = 0;
    for (int i = 0; i < 32; i++) {
      const int ci = w * 32 + i;
      if (ci < m) {
        const int p = s_posn[ci];
        t |= ((s_target[p >> 5] >> (p & 31)) & 1u) << i;
        mm |= 1u << i;
      }
    }
    prob->T[w] = t;
    prob->M[w] = mm;
    prob->target_full[w] = s_target[w];
    prob->mask_full[w] = s_mask[w];
    if (w == 0) {
      prob->n = n;
      prob->nw = nw;
      prob->inmask = a.inmask;
      prob->m = m;
    }
  }
  // compressed tables: warp item = (gate, word); all 8 words are written (zero above nw) so that no
  // stale bits survive a change of mask
  for (int it = wid; it < (n - a.c_first) * 8; it += nwarps) {
    const int g = a.c_first + (it >> 3), w = it & 7;
    const int ci = w * 32 + lane;
    uint32_t bit = 0;
    if (w < nw && ci < m) {
      const int p = s_posn[ci];
      bit = (arg_or_resident(prob, a, g, p >> 5) >> (p & 31)) & 1u;
    }
    const uint32_t out = __ballot_sync(kFull, bit != 0);
    if (lane == 0) prob->tabs[w][g] = out;
    // the travelling gates become resident
    if (lane == 1 && g >= a.a_first && g < a.a_first + a.a_count) {
      prob->full[g][w] = a.newg[g - a.a_first][w];
    }
  }
  if (a.flags & kBeginRows) {
    const int spare = n <= 31 ? 31 : (n <= 63 ? 63 : -1);
    const int ngw = (n + 31) >> 5;             // gate words that hold gates
    for (int it = wid; it < m * 16; it += nwarps) {
      const int p = it >> 4, gw = it & 15;
      uint32_t word = 0;
      const int pp = s_posn[p];
      const bool t1 = ((s_target[pp >> 5] >> (pp & 31)) & 1u) != 0;
      if (gw < ngw) {
        const int g = gw * 32 + lane;
        uint32_t bit = 0;
        if (g < n) bit = (arg_or_resident(prob, a, g, pp >> 5) >> (pp & 31)) & 1u;
        word = __ballot_sync(kFull, bit != 0);
      }
      if (!t1) word = ~word;
      if (spare >= 0 && gw == (spare >> 5)) word = t1 ? (word | 0x80000000u) : (word & 0x7fffffffu);
      if (lane == 0) prob->xr[p][gw] = word;
    }
  }
}

// sbg_stage_problem: makes a state resident AND ready (derived data built) ahead of the searches.
__global__ void __launch_bounds__(1024) k_prepare_problem(DevProblem *__restrict__ prob,
    const BeginArgs a) {
  prepare_problem(prob, a, blockIdx.x, gridDim.x);
}

// The 3-LUT scan of lut_search (lut.c:501-523): the first triple (i < k < m, as positions in the
// caller's shuffled gate order) whose three gates admit SOME 3-input function equal to the target
// under the mask (check_n_lut_possible(3, ...); get_lut_function then always succeeds).  Runs in the
// scan blocks of k_begin, on the uncompressed tables (arguments / resident copy), so that it needs
// nothing the same launch derives.  One warp per position pair (i, k), lanes over m; the minimum of
// the packed position triple i << 18 | k << 9 | m goes to ctl->best3; the last scan block to finish
// closes stage 0 (result to the host) and leaves best3 / scan_done as it found them.
__device__ __forceinline__ void scan3_blocks(const DevProblem *__restrict__ prob,
    DevCtl *__restrict__ ctl, HostOut *__restrict__ out, const BeginArgs &a, int blk, int nblks,
    uint32_t *s_full) {
  __shared__ uint16_t s_order[512];
  __shared__ uint32_t s_t[8], s_nt[8];
  __shared__ int s_last;
  const int n = a.n;
  for (int i = threadIdx.x; i < n * 8; i += blockDim.x) {
    s_full[i] = arg_or_resident(prob, a, i >> 3, i & 7);
  }
  for (int i = threadIdx.x; i < n; i += blockDim.x) s_order[i] = a.order3[i];
  if (threadIdx.x < 8) {
    s_t[threadIdx.x] = a.mask[threadIdx.x] & a.target[threadIdx.x];
    s_nt[threadIdx.x] = a.mask[threadIdx.x] & ~a.target[threadIdx.x];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warps = blockDim.x >> 5;
  const uint32_t pairs = (uint32_t)(n * (n - 1) / 2);
  for (uint32_t pq = (uint32_t)(blk * warps + (threadIdx.x >> 5)); pq < pairs;
       pq += (uint32_t)(nblks * warps)) {
    int pi, pk;
    unrank_pair(pq, n, pi, pk);
    const unsigned long long key0 = ((unsigned long long)pi << 18) | ((unsigned long long)pk << 9);
    // an earlier triple already matched?  Only worth a trip to L2 when a warp has many pairs to go
    if (pairs > 4096u && volatile_load(&ctl->best3) < key0) break;
    const uint32_t *ta = s_full + 8 * s_order[pi], *tb = s_full + 8 * s_order[pk];
    for (int m0 = pk + 1; m0 < n; m0 += 32) {
      const int pm = m0 + lane;
      const uint32_t *tc = s_full + 8 * s_order[pm < n ? pm : pk];
      uint32_t ones[8], zeros[8];
#pragma unroll
      for (int c = 0; c < 8; c++) ones[c] = zeros[c] = 0;
#pragma unroll
      for (int w = 0; w < 8; w++) {
        const uint32_t va = ta[w], vb = tb[w], vc = tc[w];
#pragma unroll
        for (int c = 0; c < 8; c++) {
          const uint32_t ab = ((c & 4) ? va : ~va) & ((c & 2) ? vb : ~vb);   // warp-uniform
          const uint32_t cell = ab & ((c & 1) ? vc : ~vc);
          ones[c] |= cell & s_t[w];
          zeros[c] |= cell & s_nt[w];
        }
      }
      bool ok = pm < n;
#pragma unroll
      for (int c = 0; c < 8; c++) ok &= !(ones[c] != 0 && zeros[c] != 0);
      const uint32_t hit = __ballot_sync(kFull, ok);
      if (hit != 0) {
        if (lane == 0) {
          atomicMin(&ctl->best3, key0 | (unsigned long long)(m0 + __ffs(hit) - 1));
        }
        break;   // later m of this pair are larger
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    s_last = atomicAdd(&ctl->scan_done, 1u) == (unsigned int)(nblks - 1);
  }
  __syncthreads();
  if (s_last != 0 && threadIdx.x == 0) {
    __threadfence();
    const unsigned long long key = volatile_load(&ctl->best3);
    if (key != ~0ull) ctl->found = (a.seq << 8) | 3ull;   // the rest of the chain returns at once
    ctl->best3 = ~0ull;
    ctl->scan_done = 0;
    // Stage 0 has one result, the 27-bit key: it travels INSIDE the sequence word (one 8-byte
    // store, no fence across the bus to order it after anything else).
    *reinterpret_cast<volatile unsigned long long *>(&out->seq[0]) =
        (a.seq << kScanKeyBits) | (key == ~0ull ? kScanKeyNone : key);
  }
}

// First kernel of every chain, three kinds of blocks:
//   block 0: control words, position tables, ticket-group counters, and minpos3 (see DevParams7) by
//            dynamic programming over the number of unconstrained bits: an entry with a free bit j
//            is the minimum of the two entries that force bit j (entries are visited level by level
//            through DevTables::m3_info, which lists them by number of free bits);
//   then prep_blocks blocks: the problem block (prepare_problem) when the state changed or its
//            rows are needed;
//   then the scan blocks: the 3-LUT scan (scan3_blocks), when the call asks for it.
__global__ void __launch_bounds__(1024) k_begin(DevProblem *__restrict__ prob,
    DevCtl *__restrict__ ctl, HostOut *__restrict__ out, DevParams7 *__restrict__ par,
    uint8_t *__restrict__ pos5, uint32_t *__restrict__ gcount, const DevTables *__restrict__ tab,
    int prep_blocks, const BeginArgs a) {
  extern __shared__ uint32_t smem[];
  if (blockIdx.x != 0) {
    const int b = (int)blockIdx.x - 1;
    if (b < prep_blocks) {
      prepare_problem(prob, a, b, prep_blocks);
    } else {
      scan3_blocks(prob, ctl, out, a, b - prep_blocks, (int)gridDim.x - 1 - prep_blocks, smem);
    }
    return;
  }
  __shared__ uint8_t posm[256];
  __shared__ uint8_t s_min[kMinpos3 + 3];
  uint32_t *s_info = smem;   // kMinpos3 words
  __shared__ int s_level[10];
  // the visiting order of minpos3 (26 KB): all loads in flight at once, instead of one dependent
  // round trip to L2 per level of the sweep below
  if (a.flags & kBeginSearch7) {
    for (int i = threadIdx.x; i < kMinpos3; i += blockDim.x) s_info[i] = tab->m3_info[i];
    if (threadIdx.x < 10) s_level[threadIdx.x] = tab->m3_level[threadIdx.x];
  }
  if (threadIdx.x == 0) {
    if (a.flags & kBeginKeepCtl) {   // phase 2 on an installed list: keep the list, restart the rest
      ctl->best = ~0ull;
      ctl->ticket2 = 0;
      ctl->ctas_done = 0;
      ctl->overflow = 0;
      ctl->skip7 = 0;
      ctl->seq = a.seq;
    } else {
      ctl->ticket = 0;
      ctl->hit_count = 0;
      ctl->best = ~0ull;
      ctl->stop_ticket = ~0ull;
      ctl->swept = 0;
      ctl->feasible = 0;
      ctl->ticket2 = 0;
      ctl->seq = a.seq;
      ctl->overflow = 0;
      ctl->list_count = 0;
      ctl->ctas_done = 0;
      ctl->skip5 = (a.flags & kBeginSearch5) ? 0u : 1u;
      ctl->skip7 = (a.flags & kBeginSearch7) ? 0u : 1u;
    }
  }
  if (!(a.flags & kBeginKeepCtl)) {
    for (uint32_t i = threadIdx.x; i < a.gcount_n; i += blockDim.x) gcount[i] = 0;
  }
  if (a.flags & kBeginSearch5) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) pos5[i] = a.pos5[i];
  }
  if (!(a.flags & kBeginSearch7)) return;
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    posm[i] = a.pos_middle[i];
    par->pos_middle[i] = a.pos_middle[i];
    par->pos_outer[i] = a.pos_outer[i];
  }
  __syncthreads();
  int lo = 0;
  for (int level = 0; level <= 8; level++) {
    const int hi = s_level[level + 1];
    for (int i = lo + threadIdx.x; i < hi; i += blockDim.x) {
      const uint32_t info = s_info[i];
      const uint32_t e = info & 0x1fffu;
      if (level == 0) {
        s_min[e] = posm[info >> 16];
      } else {
        const uint32_t step = info >> 16;   // 3^j of the lowest free bit j
        s_min[e] = min(s_min[e + step], s_min[e + 2 * step]);
      }
    }
    lo = hi;
    __syncthreads();
  }
  for (int e = threadIdx.x; e < kMinpos3; e += blockDim.x) par->minpos3[e] = s_min[e];
}

// ------------------------------------------------------------------------------------------------
// Phase 2 of search_7lut (lut.c:416-484): one warp per feasible 7-tuple.

__device__ __forceinline__ uint32_t compress16x2(uint32_t r, int b, int z) {
  // r holds two 16-bit sets over v4 (low and high half).  Of each, keeps the 8 bits whose index has
  // bit b equal to z, in order: results in bits 0..7 and 16..23.
  uint32_t t;
  switch (b) {
    case 3:
      return (r >> (8 * z)) & 0x00ff00ffu;
    case 2:
      t = r >> (4 * z);
      return (t & 0x000f000fu) | ((t >> 4) & 0x00f000f0u);
    case 1:
      t = r >> (2 * z);
      return (t & 0x00030003u) | ((t >> 2) & 0x000c000cu) | ((t >> 4) & 0x00300030u)
          | ((t >> 6) & 0x00c000c0u);
    default:
      t = (r >> z) & 0x55555555u;
      t = (t | (t >> 1)) & 0x33333333u;
      t = (t | (t >> 2)) & 0x0f0f0f0fu;
      return (t | (t >> 4)) & 0x00ff00ffu;
  }
}

// 128-cell summary of a 7-tuple: word fg (= f<<1|g) bit l (= a<<4|b<<3|c<<2|d<<1|e) of H1 / H0 is
// set iff the cell holds a masked position with target 1 / 0.  Written to sH[0..3] / sH[4..7].
template <int NW>
__device__ __forceinline__ void tuple_summary(const uint32_t *s_tabs, int npad, const int *g,
    const uint32_t *T, const uint32_t *M, int lane, uint32_t *sH) {
  uint32_t h1[4] = {0, 0, 0, 0}, h0[4] = {0, 0, 0, 0};
#pragma unroll
  for (int w = 0; w < NW; w++) {
    uint32_t tt = M[w];
#pragma unroll
    for (int i = 0; i < 5; i++) {
      const uint32_t tv = s_tabs[w * npad + g[i]];
      tt &= ((lane >> (4 - i)) & 1) ? tv : ~tv;
    }
    const uint32_t tf = s_tabs[w * npad + g[5]];
    const uint32_t tg = s_tabs[w * npad + g[6]];
    const uint32_t s3 = tt & tf & tg, s2 = tt & tf & ~tg, s1 = tt & ~tf & tg, s0 = tt & ~tf & ~tg;
    h1[0] |= s0 & T[w]; h0[0] |= s0 & ~T[w];
    h1[1] |= s1 & T[w]; h0[1] |= s1 & ~T[w];
    h1[2] |= s2 & T[w]; h0[2] |= s2 & ~T[w];
    h1[3] |= s3 & T[w]; h0[3] |= s3 & ~T[w];
  }
  __syncwarp();
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const uint32_t b1 = __ballot_sync(kFull, h1[j] != 0);
    const uint32_t b0 = __ballot_sync(kFull, h0[j] != 0);
    if (lane == 0) {
      sH[j] = b1;
      sH[4 + j] = b0;
    }
  }
  __syncwarp();
}

// ------------------------------------------------------------------------------------------------
// Phase 2, stage 1 as a FILTER with one lane per outer triple.
//
// For an outer triple the 128 cells of the tuple's summary fall into 8 groups of 16 (one group per
// pattern u of the three outer gates, 16 cells over the other four gates).  An outer function fo is
// a 2-colouring of the groups; it leaves a decomposable remainder iff no two groups of the same
// colour hold, in the same place, one a masked 1 and the other a masked 0 -- i.e. iff fo properly
// 2-colours the "conflict graph" on the 8 groups.  Most (tuple, outer triple) pairs have NO proper
// colouring (measured on bench.py's states: 87-100 %), and deciding that needs neither the order of
// the groups nor the order of the cells inside them.  So lane j < 25 takes outer triple j of the
// warp's tuple: it permutes the summary's index bits (at most two word<->bit exchanges, done
// without branches since every lane has its own triple) until the three outer gates select (word,
// half word), tests the 28 pairs of groups with one AND each, and ANDs a 128-bit set of colourings
// (those with group 7 = 0; the set is closed under complement) with one mask per conflict.  About
// 350 warp instructions decide all 25 triples of a tuple; the ballot form below (~170 per triple)
// only sees the triples that pass.
//
// Summary layout (tuple_summary): word = f << 1 | g, bit = a << 4 | b << 3 | c << 2 | d << 1 | e.

// Exchanges index bit i (inside the words) with word-index bit wb of a 4-word set; on == false
// makes it a no-op.  Branch-free: i, wb and on differ from lane to lane.
__device__ __forceinline__ void swap_bit_with_word(uint32_t *h, int i, int wb, bool on) {
  uint32_t m = i == 0 ? 0x55555555u : i == 1 ? 0x33333333u : i == 2 ? 0x0f0f0f0fu : 0x00ff00ffu;
  if (!on) m = 0;
  const int d = 1 << i;
  // word pairs: wb == 0: (0,1) (2,3); wb == 1: (0,2) (1,3) -- bring them to the first form
  const uint32_t a1 = wb ? h[2] : h[1];
  const uint32_t a2 = wb ? h[1] : h[2];
  uint32_t lo0 = h[0], hi0 = a1, lo1 = a2, hi1 = h[3];
  uint32_t t = ((lo0 >> d) ^ hi0) & m;
  hi0 ^= t;
  lo0 ^= t << d;
  t = ((lo1 >> d) ^ hi1) & m;
  hi1 ^= t;
  lo1 ^= t << d;
  h[0] = lo0;
  h[1] = wb ? lo1 : hi0;
  h[2] = wb ? hi0 : lo1;
  h[3] = hi1;
}

// colourings x < 128 as 4 words (x = 32 * wd + bit): those in which group u has colour 1
__host__ __device__ constexpr uint32_t colour_pattern(int u, int wd) {
  return u == 0 ? 0xAAAAAAAAu : u == 1 ? 0xCCCCCCCCu : u == 2 ? 0xF0F0F0F0u : u == 3 ? 0xFF00FF00u
      : u == 4 ? 0xFFFF0000u : u == 5 ? ((wd & 1) ? 0xffffffffu : 0u)
      : u == 6 ? ((wd & 2) ? 0xffffffffu : 0u) : 0u;
}

// Bit j of the result: outer triple j (in the order of lut.c:396-415: the 15 triples {a, x, y}, then
// the 10 triples {b, x, y} without a) of the tuple whose summary is sH[0..7] may have survivors.
__device__ __forceinline__ uint32_t triples_with_colourings(const uint32_t *sH, int lane) {
  const int j = lane < 25 ? lane : 0;
  // the triple's two other positions x < y (1 = b .. 6 = g): pairs in lexicographic order
  int x, y;
  {
    int q = j < 15 ? j : j - 15;
    x = j < 15 ? 1 : 2;
    int row = 6 - x;
#pragma unroll
    for (int step = 0; step < 4; step++) {
      const bool more = q >= row;
      q -= more ? row : 0;
      x += more ? 1 : 0;
      row -= more ? 1 : 0;
    }
    y = x + 1 + q;
  }
  uint32_t h1[4], h0[4];
#pragma unroll
  for (int i = 0; i < 4; i++) {
    h1[i] = sH[i];
    h0[i] = sH[4 + i];
    if (j >= 15) {
      // the triples with b and without a: exchange index bits 4 (a) and 3 (b) inside the words,
      // so that b selects the half word; a becomes one of the four inner gates
      uint32_t t = ((h1[i] >> 8) ^ h1[i]) & 0x0000ff00u;
      h1[i] ^= t | (t << 8);
      t = ((h0[i] >> 8) ^ h0[i]) & 0x0000ff00u;
      h0[i] ^= t | (t << 8);
    }
  }
  // bring x and y to the word-index bits (f = bit 1, g = bit 0 of the word index); the in-word
  // index bit of position p (1 = b .. 4 = e) is 4 - p.  x goes to f's place unless f is the other
  // outer gate (then to g's); y, if it is an in-word gate as well, to g's place.
  const int ix = x <= 4 ? 4 - x : 0, iy = y <= 4 ? 4 - y : 0;
  swap_bit_with_word(h1, ix, y == 5 ? 0 : 1, x <= 4);
  swap_bit_with_word(h0, ix, y == 5 ? 0 : 1, x <= 4);
  swap_bit_with_word(h1, iy, 0, y <= 4);
  swap_bit_with_word(h0, iy, 0, y <= 4);
  // group u = word * 2 + half: gx[u] = ones | zeros << 16, gr[u] = zeros | ones << 16
  uint32_t gx[8], gr[8];
#pragma unroll
  for (int w = 0; w < 4; w++) {
    gx[2 * w] = __byte_perm(h1[w], h0[w], 0x5410);
    gx[2 * w + 1] = __byte_perm(h1[w], h0[w], 0x7632);
    gr[2 * w] = __byte_perm(h0[w], h1[w], 0x5410);
    gr[2 * w + 1] = __byte_perm(h0[w], h1[w], 0x7632);
  }
  uint32_t v[4] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu};
#pragma unroll
  for (int a = 0; a < 8; a++) {
#pragma unroll
    for (int b = a + 1; b < 8; b++) {
      const uint32_t e = (gx[a] & gr[b]) != 0 ? 0xffffffffu : 0u;   // groups a and b conflict
#pragma unroll
      for (int wd = 0; wd < 4; wd++) {
        const uint32_t differ = colour_pattern(a, wd) ^ colour_pattern(b, wd);
        v[wd] &= differ | ~e;
      }
    }
  }
  return __ballot_sync(kFull, lane < 25 && (v[0] | v[1] | v[2] | v[3]) != 0);
}

// Phase 2, stage 1 for outer triple j of a tuple with summary Hs (srcw = DevTables::src7[j][lane]):
// W[u] = low half: the 16 cells (over the four non-outer gates) in which outer pattern u holds a
// masked 1, high half: the same for a masked 0; ok[hi] bit lane and ok[7 - hi] bit 31 - lane both
// set <=> outer function hi*32+lane leaves a conflict-free 5-input remainder.
__device__ __forceinline__ void outer_ok7(const uint32_t *Hs, uint32_t srcw, int lane, uint32_t *W,
    uint32_t *ok) {
  uint32_t P1[4], P0[4];
#pragma unroll
  for (int t4 = 0; t4 < 4; t4++) {
    const uint32_t c = (srcw >> (8 * t4)) & 0x7fu;
    P1[t4] = __ballot_sync(kFull, (Hs[c >> 5] >> (c & 31u)) & 1u);
    P0[t4] = __ballot_sync(kFull, (Hs[4 + (c >> 5)] >> (c & 31u)) & 1u);
  }
#pragma unroll
  for (int u = 0; u < 8; u++) {
    W[u] = ((P1[u >> 1] >> (16 * (u & 1))) & 0xffffu)
        | (((P0[u >> 1] >> (16 * (u & 1))) & 0xffffu) << 16);
  }
  uint32_t L = 0;
#pragma unroll
  for (int u = 0; u < 5; u++) {
    if ((lane >> u) & 1) L |= W[u];
  }
#pragma unroll
  for (int hi = 0; hi < 8; hi++) {
    uint32_t rr = L;
    if (hi & 1) rr |= W[5];
    if (hi & 2) rr |= W[6];
    if (hi & 4) rr |= W[7];
    ok[hi] = __ballot_sync(kFull, ((rr & (rr >> 16)) & 0xffffu) == 0);
  }
}

// Stage 2 for one surviving outer function (r1 / r0 = OR of W[u] over the patterns u it sends to 1
// / 0) and one ordering row (b = bit of v4 that is the g input): the middle functions that work are
// the union, over the (c0, c1) with hok[0][c0] && hok[1][c1] && ((hv[0][c0] ^ hv[1][c1]) & ov) == 0,
// of the cubes { fm : (fm & S) == (hv[0][c0] | hv[1][c1]) }.
__device__ __forceinline__ void middle_cubes(uint32_t r1, uint32_t r0, int b, uint32_t (*hv)[4],
    bool (*hok)[4], uint32_t &S, uint32_t &ov) {
  // The four inner cells (x, g): A = middle patterns with a masked 1, B = with a masked 0
  // (both compressed at once: they are the two halves of r1 / r0).
  // If both are non-empty, fm must send A to one value and B to the other: fm & S in {A, B}.
  uint32_t cs[4], ca[4], cb[4];
#pragma unroll
  for (int ci = 0; ci < 4; ci++) {
    const uint32_t AB = compress16x2((ci & 2) ? r1 : r0, b, ci & 1);
    const uint32_t A = AB & 0xffu, B = AB >> 16;
    const bool act = A != 0 && B != 0;
    cs[ci] = act ? (A | B) : 0u;   // inactive: empty support, both choices identical
    ca[ci] = act ? A : 0u;
    cb[ci] = act ? B : 0u;
  }
  // Combine constraints 0,1 and 2,3 (4 choices each), then cross the two halves; a
  // combination is consistent iff its forced values agree wherever supports overlap.
  uint32_t hs[2];
#pragma unroll
  for (int h2 = 0; h2 < 2; h2++) {
    const int i = 2 * h2;
    hs[h2] = cs[i] | cs[i + 1];
    const uint32_t ov2 = cs[i] & cs[i + 1];
#pragma unroll
    for (int c = 0; c < 4; c++) {
      const uint32_t v0 = (c & 1) ? cb[i] : ca[i];
      const uint32_t v1 = (c & 2) ? cb[i + 1] : ca[i + 1];
      hok[h2][c] = ((v0 ^ v1) & ov2) == 0;
      hv[h2][c] = v0 | v1;
    }
  }
  S = hs[0] | hs[1];
  ov = hs[0] & hs[1];
}

// Moves index bit b of both 16-bit halves of r to bit 3, bits b+1..3 one place down (the other
// bits keep their order), so that compress16x2(r, b, z) == compress16x2(index_bit_to_top(r, b), 3, z).
// Branch-free: b differs from lane to lane in k_decomp7's stage 2.
__device__ __forceinline__ uint32_t index_bit_to_top(uint32_t r, int b) {
  uint32_t t = ((r >> 1) ^ r) & (b <= 0 ? 0x22222222u : 0u);   // exchange index bits 0 and 1
  r ^= t ^ (t << 1);
  t = ((r >> 2) ^ r) & (b <= 1 ? 0x0c0c0c0cu : 0u);            // 1 and 2
  r ^= t ^ (t << 2);
  t = ((r >> 4) ^ r) & (b <= 2 ? 0x00f000f0u : 0u);            // 2 and 3
  return r ^ t ^ (t << 4);
}

// k_decomp7's stage 2 for entries p0 .. min(p0 + 32, nent) - 1 of a tuple's entry list, one lane
// each.  Entry = j << 9 | row << 7 | fo: outer function fo (bit 7 clear; it stands for fo and ~fo)
// of outer triple j, ordering row `row` of that triple.  sW[9 j + u] = W[u] of triple j (outer_ok7),
// sW[9 j + 8] = its first ordering number | (bit of v4 that is the g input, 2 bits per row) << 8.
// Complementing fo swaps r1 and r0, which middle_cubes answers with the same S, ov and set of cubes,
// so both members of a pair have the same best middle position and the pair's outer position is the
// smaller of the two (s_pmin).  Returns the smallest k << 16 | po << 8 | pm with a match over the
// warp's entries, 0xffffffff if none.
__device__ __forceinline__ uint32_t decomp7_entries(const uint16_t *ent, int p0, int nent,
    const uint32_t *sW, const uint8_t *s_pmin, const uint8_t *s_minpos, const uint16_t *s_p3,
    int lane) {
  const bool have = p0 + lane < nent;
  const uint32_t e = have ? ent[p0 + lane] : 0u;
  const uint32_t fo = e & 0x7fu, row = (e >> 7) & 3u;
  const uint32_t *w = sW + 9 * (e >> 9);   // stride 9: lanes on different triples, different banks
  uint32_t r1 = 0, r0 = 0;
#pragma unroll
  for (int u = 0; u < 8; u++) {
    const uint32_t wu = w[u];
    if ((fo >> u) & 1) r1 |= wu; else r0 |= wu;
  }
  const uint32_t info = w[8];
  const int b = (int)((info >> (8 + 2 * row)) & 3u);
  uint32_t hv[2][4], S, ov;
  bool hok[2][4];
  middle_cubes(index_bit_to_top(r1, b), index_bit_to_top(r0, b), 3, hv, hok, S, ov);
  // which of the 16 ways to pick are consistent; every consistent way is a non-empty cube, i.e. a
  // match.  Entries of dense lists almost never match, so the warp looks positions up only when
  // one of its lanes has a match.
  uint32_t picks = 0;
#pragma unroll
  for (int c0 = 0; c0 < 4; c0++) {
#pragma unroll
    for (int c1 = 0; c1 < 4; c1++) {
      const bool ok2 = hok[0][c0] && hok[1][c1] && ((hv[0][c0] ^ hv[1][c1]) & ov) == 0;
      if (ok2) picks |= 1u << (4 * c0 + c1);
    }
  }
  if (!have) picks = 0;
  if (!__any_sync(kFull, picks != 0)) return 0xffffffffu;
  const uint32_t p3s = s_p3[S];
  uint32_t best_pm = 256;
#pragma unroll
  for (int c0 = 0; c0 < 4; c0++) {
#pragma unroll
    for (int c1 = 0; c1 < 4; c1++) {
      if ((picks >> (4 * c0 + c1)) & 1u) {
        const uint32_t V = hv[0][c0] | hv[1][c1];
        best_pm = min(best_pm, (uint32_t)s_minpos[p3s + s_p3[V]]);
      }
    }
  }
  uint32_t cand = 0xffffffffu;
  if (picks != 0) cand = (((info & 0x7fu) + row) << 16) | ((uint32_t)s_pmin[fo] << 8) | best_pm;
  return __reduce_min_sync(kFull, cand);
}

// k_decomp7's per-warp entry list: at most 31 entries carried over + 128 pairs x 4 rows of a triple
constexpr int kDecompEntries = 31 + 128 * 4;

template <int NW>
__global__ void __launch_bounds__(kThreads) k_decomp7(const DevProblem *__restrict__ prob,
    DevCtl *__restrict__ ctl, HostOut *__restrict__ out, const DevParams7 *__restrict__ par,
    const uint64_t *__restrict__ list, int part, int nparts, const DevTables *__restrict__ tab,
    int use_filter) {
  extern __shared__ uint32_t smem[];
  __shared__ uint8_t s_minpos[kMinpos3 + 3];
  __shared__ uint16_t s_p3[256];
  __shared__ uint8_t s_pmin[128];        // fo < 128 -> smaller shuffled position of fo and ~fo
  __shared__ uint32_t s_src7[25 * 32];   // copy of DevTables::src7
  __shared__ uint32_t s_H[kWarpsPerCta][16];
  __shared__ uint32_t s_W[kWarpsPerCta][25 * 9];            // per outer triple: W[8], row info
  __shared__ uint16_t s_ent[kWarpsPerCta][kDecompEntries];  // (triple, row, outer pair) entries

  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  // independent of the chain's earlier kernels: overlaps their tail under programmatic launch
  for (int i = threadIdx.x; i < 25 * 32; i += blockDim.x) s_src7[i] = tab->src7[i >> 5][i & 31];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    int p3 = 0, w3 = 1;
    for (int j = 0; j < 8; j++) {
      if ((i >> j) & 1) p3 += w3;
      w3 *= 3;
    }
    s_p3[i] = (uint16_t)p3;
  }
  wait_for_predecessor();
  const int n = prob->n;
  const int npad = (n + 3) & ~3;
  uint32_t *s_tabs = smem;
  stage_tables(s_tabs, prob, NW, npad);

  // the list length is on the device (k_offsets / k_merge_runs); this part's share is
  // ceil((count - part) / nparts) entries, surplus CTAs have nothing to do
  const bool skip = chain_is_over(ctl) || volatile_load32(&ctl->skip7) != 0
      || volatile_load32(&ctl->overflow) != 0;
  const unsigned int count = skip ? 0u : ctl->list_count;
  const unsigned int share = count > (unsigned int)part
      ? (count - (unsigned int)part + (unsigned int)nparts - 1) / (unsigned int)nparts : 0u;
  if (blockIdx.x * kWarpsPerCta < share) {
  for (int i = threadIdx.x; i < kMinpos3; i += blockDim.x) s_minpos[i] = par->minpos3[i];
  for (int i = threadIdx.x; i < 128; i += blockDim.x) {
    s_pmin[i] = min(par->pos_outer[i], par->pos_outer[255 - i]);
  }
  __syncthreads();

  uint32_t T[NW], M[NW];
#pragma unroll
  for (int w = 0; w < NW; w++) {
    T[w] = prob->T[w];
    M[w] = prob->M[w];
  }
  uint32_t *sH = s_H[warp];

  for (;;) {
    unsigned long long t = 0;
    if (lane == 0) t = atomicAdd(&ctl->ticket2, 1ull);
    t = __shfl_sync(kFull, t, 0);
    const uint64_t idx = t * (uint64_t)nparts + (uint64_t)part;
    if (idx >= count) break;
    if ((volatile_load(&ctl->best) >> 23) < idx) break;  // a smaller list index already matched

    const uint64_t cur = list[idx];
    int g[7];
#pragma unroll
    for (int i = 0; i < 7; i++) g[i] = (int)((cur >> (9 * (6 - i))) & 0x1ffu);

    // The reference's outer-table cache is keyed by a truncated value (lut.c:379,432-435): rows
    // 0-3 of a tuple whose first gate is 0 reuse the previous tuple's last outer tables when that
    // tuple ended in the same two gates this one continues with.  Reproduce it: those rows see
    // gate prev[1] in place of gate 0.
    bool stale = false;
    int sub = 0;
    if (idx > 0) {
      const uint64_t prev = list[idx - 1];
      stale = g[0] == 0 && (int)((prev >> 9) & 0x1ffu) == g[1] && (int)(prev & 0x1ffu) == g[2];
      sub = (int)((prev >> 45) & 0x1ffu);
    }
    tuple_summary<NW>(s_tabs, npad, g, T, M, lane, sH);
    // outer triples worth the ballot form (all of them for a stale-cache tuple, whose first triple
    // is decided on a second summary)
    const uint32_t pass_i = (use_filter != 0 && !stale) ? triples_with_colourings(sH, lane)
                                                        : 0x1ffffffu;
    if (stale) {
      int g2[7];
#pragma unroll
      for (int i = 0; i < 7; i++) g2[i] = g[i];
      g2[0] = sub;
      tuple_summary<NW>(s_tabs, npad, g2, T, M, lane, sH + 8);
    }

    // Stage 1 proper per passing outer triple, in order j; its survivors come in complementary
    // pairs (fo, ~fo), and each pair goes on the warp's entry list once per ordering row of the
    // triple.  Stage 2 then takes 32 (pair, row) entries at a time, one lane each, so that rows and
    // triples with few survivors share passes.  Ordering numbers grow with j, so the smallest
    // k << 16 | po << 8 | pm over all entries is the first match: full passes run as the list
    // fills, and once one of them matches, the entries left over and nothing after them decide.
    uint32_t *sW = s_W[warp];
    uint16_t *ent = s_ent[warp];
    uint32_t best = 0xffffffffu;
    int nent = 0;
#ifdef SBG_COUNT_STAGE1
    unsigned long long n_pairs = 0, n_passes = 0, n_row_passes = 0;
#endif
    for (int j = 0; j < 25; j++) {
      if (((pass_i >> j) & 1u) == 0) continue;   // the filter found no admissible outer function
      const uint32_t *Hs = (stale && j == 0) ? sH + 8 : sH;
      uint32_t W[8], ok[8];
      outer_ok7(Hs, s_src7[j * 32 + lane], lane, W, ok);
      uint32_t sv[4], any = 0;
#pragma unroll
      for (int hi = 0; hi < 4; hi++) {   // the pair's member without bit 7
        sv[hi] = ok[hi] & __brev(ok[7 - hi]);
        any |= sv[hi];
      }
#ifdef SBG_COUNT_STAGE1
      if (lane == 0) atomicAdd(&ctl->pad0[0], 1ull);                    // (tuple, outer triple) pairs
      if (lane == 0 && any != 0) atomicAdd(&ctl->pad0[1], 1ull);        // ... with survivors
#endif
      if (any == 0) continue;  // no outer function leaves a conflict-free 5-input remainder
      const int k0 = c_j_first_k[j];
      const int nrows = c_j_rows[j];
      uint32_t mine = 0;
#pragma unroll
      for (int u = 0; u < 8; u++) {
        if (lane == u) mine = W[u];
      }
      if (lane == 8) {
        mine = (uint32_t)k0;
#pragma unroll
        for (int row = 0; row < 4; row++) {
          if (row < nrows) mine |= (uint32_t)c_row_b[k0 + row] << (8 + 2 * row);
        }
      }
      __syncwarp();
      if (lane < 9) sW[9 * j + lane] = mine;
#pragma unroll
      for (int hi = 0; hi < 4; hi++) {
        if ((sv[hi] >> lane) & 1u) {
          const int at = nent + __popc(sv[hi] & lanemask_lt()) * nrows;
          const uint32_t e = (uint32_t)j << 9 | (uint32_t)(hi * 32 + lane);
          for (int row = 0; row < nrows; row++) ent[at + row] = (uint16_t)(e | (uint32_t)row << 7);
        }
        nent += __popc(sv[hi]) * nrows;
      }
#ifdef SBG_COUNT_STAGE1
      {
        const int np = __popc(sv[0]) + __popc(sv[1]) + __popc(sv[2]) + __popc(sv[3]);
        n_pairs += np;
        n_row_passes += (unsigned long long)((2 * np + 31) / 32 * nrows);  // one lane per fo and row
      }
#endif
      if (nent < 32) continue;
      __syncwarp();
      const int full = nent & ~31;
      for (int p0 = 0; p0 < full; p0 += 32) {
        best = min(best, decomp7_entries(ent, p0, nent, sW, s_pmin, s_minpos, s_p3, lane));
#ifdef SBG_COUNT_STAGE1
        n_passes++;
#endif
      }
      if (best != 0xffffffffu) break;
      // carry the partial pass over to the front
      const int rest = nent - full;
      const uint16_t e = lane < rest ? ent[full + lane] : (uint16_t)0;
      __syncwarp();
      if (lane < rest) ent[lane] = e;
      nent = rest;
    }
    if (nent & 31) {
      __syncwarp();
      best = min(best, decomp7_entries(ent, nent & ~31, nent, sW, s_pmin, s_minpos, s_p3, lane));
#ifdef SBG_COUNT_STAGE1
      n_passes++;
#endif
    }
#ifdef SBG_COUNT_STAGE1
    if (lane == 0) {
      atomicAdd(&ctl->pad0[2], n_pairs);        // complementary pairs of survivors
      atomicAdd(&ctl->pad0[3], n_passes);       // 32-lane passes of stage 2
      atomicAdd(&ctl->pad0[4], n_row_passes);   // the same triples one lane per fo, row by row
    }
#endif
    if (best != 0xffffffffu) {
      if (lane == 0) atomicMin(&ctl->best, (unsigned long long)((idx << 23) | best));
      break;  // later tickets of this warp have larger list indices
    }
  }
  }  // this CTA has a share
  let_successor_start();
  if (last_cta_of_grid(ctl) && threadIdx.x == 0
      && !chain_is_over(ctl) && volatile_load32(&ctl->skip7) == 0) {
    const unsigned long long key = volatile_load(&ctl->best);
    unsigned long long tuple = 0, tuple_prev = 0;
    if (key != ~0ull) {
      const unsigned long long idx = key >> 23;
      tuple = list[idx];
      if (idx > 0) tuple_prev = list[idx - 1];
    }
#ifdef SBG_COUNT_STAGE1
    printf("S1 list %u pairs %llu with_survivors %llu outer_pairs %llu passes %llu row_passes %llu\n",
        ctl->list_count, ctl->pad0[0], ctl->pad0[1], ctl->pad0[2], ctl->pad0[3], ctl->pad0[4]);
    for (int i = 0; i < 5; i++) ctl->pad0[i] = 0;
#endif
    close_stage(ctl, out, 2, key, ctl->list_count, tuple, tuple_prev);
  }
}

// ------------------------------------------------------------------------------------------------
// Enumeration (sbg_enum3 / sbg_enum5 / sbg_enum7): every match of lut_search's 3-LUT scan /
// search_5lut / search_7lut, not only the first.  The same decisions as the searches above with
// nothing thrown away, in two passes over the same tickets -- a position pair of the gate order, a
// 3-gate prefix of C(n,5) (dealt to the parts as k_sweep deals them) or one list entry:
//   count: the number of matches of each ticket, and their sum;
//   k_enum_scan: exclusive prefix sum of those counts = where each ticket's matches start in the
//     ascending key order;
//   emit: the tickets whose matches start below K write them there, in key order, decoded into
//     DevMatch records.
// Tickets are numbered in key order, so the order needs no sort.  Both passes run the identical
// sweep, so a ticket emits exactly the matches it counted: each kernel holds one sweep of a ticket,
// enum_tickets runs it for every pass, and every ballot of matches goes through emit_step.
//
// After a count, any rank of the share can be emitted again from counts and offsets alone
// (sbg_enum_fetch / sbg_enum_pick): the emit pass of the same sweep, run over the tickets that hold
// the wanted ranks only (k_enum_locate finds them).  The pass's mode (template parameter MODE):
//   kEnumCount  the count pass;
//   kEnumFirst  the first K (max_out = K), ranks [0, K) to out[rank];
//   kEnumRange  ranks [sel.lo, max_out) to out[rank - sel.lo];
//   kEnumPick   one warp per ticket of sel.tickets, writing each rank of its slice of sel.ranks to
//               out[sel.slots[...]] (duplicate ranks: every slot that asked for it).
// The kernels keep one parameter list for all modes; sel reaches the range and pick forms in the
// lane's EnumCtl block.
enum EnumMode : int { kEnumCount = 0, kEnumFirst = 1, kEnumRange = 2, kEnumPick = 3 };

struct EnumSel {
  unsigned long long lo;                  // kEnumRange: first rank of the window
  const unsigned long long *ranks;        // kEnumPick: the requested ranks, ascending, duplicates kept
  const unsigned int *slots;              //   the output slot of each of them
  const unsigned long long *tickets;      //   the distinct tickets holding them, ascending
  const unsigned int *first;              //   ticket j's ranks: ranks[first[j] .. first[j+1]-1]
};

// Where a pass stands in the ticket a warp sweeps (warp-uniform).
struct EnumTicket {
  EnumSel sel;                   // range / pick: what to emit
  unsigned long long max_out;    // first / range: the end of the wanted ranks
  unsigned long long base;       // emit: rank of the ticket's first match
  uint32_t count;                // matches met so far (count pass: the ticket's count)
  unsigned int req, req_end;     // pick: the ticket's requests not yet met
};

// One ballot of a sweep: the lanes with hit hold the next matches of the ticket, in lane order.  The
// ballot covers ranks [step_end - popc(ballot), step_end), the lane's own match has rank `at`, and
// write(i) writes the lane's match to out[i].  Pick: the requests of this step are consumed in
// order from req, each written by the lane that holds its rank.  Returns whether the ticket has
// nothing more to emit (never in the count pass).
template <int MODE, class Write>
__device__ __forceinline__ bool emit_step(bool hit, EnumTicket &tk, Write write) {
  const uint32_t bal = __ballot_sync(kFull, hit);
  const unsigned long long at = tk.base + tk.count + __popc(bal & lanemask_lt());
  const unsigned long long step_end = tk.base + tk.count + __popc(bal);
  if (MODE == kEnumPick) {
    for (; tk.req < tk.req_end; tk.req++) {
      const unsigned long long r = tk.sel.ranks[tk.req];
      if (r >= step_end) break;
      if (hit && at == r) write((unsigned long long)tk.sel.slots[tk.req]);
    }
  } else if (MODE != kEnumCount && hit && at < tk.max_out
             && (MODE != kEnumRange || at >= tk.sel.lo)) {
    write(MODE == kEnumRange ? at - tk.sel.lo : at);
  }
  tk.count += __popc(bal);
  if (MODE == kEnumCount) return false;
  return MODE == kEnumPick ? tk.req >= tk.req_end : tk.base + tk.count >= tk.max_out;
}

// The layout of sbg_match (include/sboxgates_b200.h; sbg_api.cu checks that the two agree).
struct DevMatch {
  unsigned long long key;
  uint16_t gates[7];
  uint8_t func_outer, func_middle, func_inner, inner_seen;
  uint8_t width;
  uint8_t pad[5];
};

struct EnumCtl {
  unsigned long long total;     // matches counted so far (all windows of the call)
  unsigned long long feasible;  // 5-LUT: feasible tuples met
  unsigned long long carry;     // k_enum_scan: matches in front of the next window
  EnumSel sel;                  // range / pick emit: what to emit (set by the host before the pass)
  unsigned long long gtotal;    // k_enum_globalize: the whole's total
  unsigned int gbad;            //   1 if the share's own row of block sums differs from its own
};

// The ticket loop of the enumeration kernels: one warp per ticket of t_begin .. t_end-1 (pick: per
// entry j of sel.tickets, ticket sel.tickets[j]); the emit passes skip the tickets that hold no
// wanted rank.  sweep(t, tk, feasible) sweeps ticket t, passing every ballot of matches to
// emit_step.  In the count pass it leaves the ticket's matches in tk.count (and the 5-LUT sweep adds
// the feasible tuples it met to feasible); the tickets' counts and both sums are written back here.
template <int MODE, class Sweep>
__device__ __forceinline__ void enum_tickets(EnumCtl *__restrict__ ectl,
    uint32_t *__restrict__ counts, const unsigned long long *__restrict__ offsets,
    unsigned long long max_out, unsigned long long t_begin, unsigned long long t_end, Sweep sweep) {
  EnumTicket tk = {};
  if (MODE == kEnumRange || MODE == kEnumPick) tk.sel = ectl->sel;
  tk.max_out = max_out;
  const int lane = threadIdx.x & 31;
  const unsigned long long nwarps = (unsigned long long)gridDim.x * kWarpsPerCta;
  unsigned long long matches_local = 0, feasible_local = 0;
  for (unsigned long long j = t_begin + (unsigned long long)blockIdx.x * kWarpsPerCta
           + (threadIdx.x >> 5);
       j < t_end; j += nwarps) {
    const unsigned long long t = MODE == kEnumPick ? tk.sel.tickets[j] : j;
    if (MODE != kEnumCount) {
      if (MODE != kEnumPick && (counts[t] == 0 || offsets[t] >= max_out)) continue;
      if (MODE == kEnumRange && offsets[t] + counts[t] <= tk.sel.lo) continue;
      if (MODE == kEnumPick) {
        tk.req = tk.sel.first[j];
        tk.req_end = tk.sel.first[j + 1];
      }
      tk.base = offsets[t];
    }
    tk.count = 0;
    sweep(t, tk, feasible_local);
    if (MODE == kEnumCount) {
      if (lane == 0) counts[t] = tk.count;
      matches_local += tk.count;
    }
  }
  if (MODE == kEnumCount && lane == 0) {
    if (matches_local != 0) atomicAdd(&ectl->total, matches_local);
    if (feasible_local != 0) atomicAdd(&ectl->feasible, feasible_local);
  }
}

struct EnumOrders {
  uint8_t order[2][256];   // the shuffled function order(s): [0] outer (5-LUT: the only one), [1] middle
};

__constant__ uint8_t c_rows5[10][5];   // ordering rows (lut.c:189,224-229 and lut.c:396-415)
__constant__ uint8_t c_rows7[70][7];

// Output of LUT(func; x, y, z) on one table word (state.c:202-230).
__device__ __forceinline__ uint32_t lut_word(uint32_t func, uint32_t x, uint32_t y, uint32_t z) {
  uint32_t r = 0;
#pragma unroll
  for (int m = 0; m < 8; m++) {
    if ((func >> m) & 1u) r |= ((m & 4) ? x : ~x) & ((m & 2) ? y : ~y) & ((m & 1) ? z : ~z);
  }
  return r;
}

// A match's record of width 3, 5 or 7: the first WIDTH gates of G, zeros in the fields the width
// does not use (func_outer at width 3, func_middle below width 7).
template <int WIDTH>
__device__ __forceinline__ void store_match(DevMatch *__restrict__ dst, unsigned long long key,
    const int *G, uint32_t fo, uint32_t fm, uint32_t inner, uint32_t seen) {
  DevMatch m;
  m.key = key;
#pragma unroll
  for (int i = 0; i < 7; i++) m.gates[i] = i < WIDTH ? (uint16_t)G[i] : (uint16_t)0;
  m.func_outer = WIDTH > 3 ? (uint8_t)fo : (uint8_t)0;
  m.func_middle = WIDTH == 7 ? (uint8_t)fm : (uint8_t)0;
  m.func_inner = (uint8_t)inner;
  m.inner_seen = (uint8_t)seen;
  m.width = (uint8_t)WIDTH;
#pragma unroll
  for (int i = 0; i < 5; i++) m.pad[i] = 0;
  *dst = m;
}

// A 5- or 7-LUT match's record: gates in reference order (tuple positions of ordering row k),
// func_inner = solved bits only and inner_seen = cells with a masked position (sbg_solve_inner's
// closed form, on the compressed tables; a match has no conflicting cell).
template <int NW, int WIDTH>
__device__ __forceinline__ void write_match(DevMatch *__restrict__ dst, unsigned long long key,
    const int *tuple, int k, uint32_t fo, uint32_t fm, const uint32_t *s_tabs, int npad,
    const uint32_t *T, const uint32_t *M) {
  int G[WIDTH];
#pragma unroll
  for (int i = 0; i < WIDTH; i++) G[i] = tuple[WIDTH == 5 ? c_rows5[k][i] : c_rows7[k][i]];
  uint32_t ones = 0, seen = 0;
#pragma unroll
  for (int w = 0; w < NW; w++) {
    const uint32_t *t = s_tabs + w * npad;
    const uint32_t x = lut_word(fo, t[G[0]], t[G[1]], t[G[2]]);
    const uint32_t y = WIDTH == 7 ? lut_word(fm, t[G[3]], t[G[4]], t[G[5]]) : t[G[3]];
    const uint32_t z = t[G[WIDTH - 1]];
#pragma unroll
    for (int c = 0; c < 8; c++) {
      const uint32_t in_cell = M[w] & ((c & 4) ? x : ~x) & ((c & 2) ? y : ~y) & ((c & 1) ? z : ~z);
      if (in_cell & T[w]) ones |= 1u << c;
      if (in_cell) seen |= 1u << c;
    }
  }
  store_match<WIDTH>(dst, key, G, fo, fm, ones, seen);
}

// The 5-LUT sweep of one part, tickets t_begin .. t_end-1 of it: the warp's prefix, its (d,e) pairs
// 32 at a time with the feasibility test of k_sweep (mixed prefix cells split by d and e), then per
// feasible tuple and ordering the set of working outer functions from outer_ok5.
template <int NW, int MODE>
__global__ void __launch_bounds__(kThreads) k_enum5(const DevProblem *__restrict__ prob,
    EnumCtl *__restrict__ ectl, const EnumOrders ord, uint32_t *__restrict__ counts,
    const unsigned long long *__restrict__ offsets, DevMatch *__restrict__ out,
    unsigned long long max_out, unsigned long long t_begin, unsigned long long t_end, int part,
    int nparts, const DevTables *__restrict__ tab) {
  constexpr int P = 3, K = 5, NC = 1 << P;
  extern __shared__ uint32_t smem[];
  __shared__ uint8_t s_ord[256];
  const int n = prob->n;
  const int npad = (n + 3) & ~3;
  uint32_t *s_tabs = smem;
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  uint32_t *cells = smem + NW * npad + warp * (NC * 2 * NW);  // per prefix cell: C1[NW], C0[NW]
  stage_tables(s_tabs, prob, NW, npad);
  for (int i = threadIdx.x; i < 256; i += blockDim.x) s_ord[i] = ord.order[0][i];
  __syncthreads();
  uint32_t T[NW], M[NW];
#pragma unroll
  for (int w = 0; w < NW; w++) {
    T[w] = prob->T[w];
    M[w] = prob->M[w];
  }
  const uint32_t inmask = prob->inmask;
  const uint64_t total = c_binom[n - 2][P];

  enum_tickets<MODE>(ectl, counts, offsets, max_out, t_begin, t_end,
      [&](unsigned long long t, EnumTicket &tk, unsigned long long &feasible) {
    const uint64_t dealt = dealt_item(t, part, nparts);   // as k_sweep deals its prefixes
    if (dealt < total) {
      int pre[P];
      uint64_t base_rank;
      unrank_prefix_warp<P, K, true>(dealt, n, pre, base_rank, lane);
      bool rejected = false;
#pragma unroll
      for (int i = 0; i < P; i++) rejected |= (pre[i] < 8) && ((inmask >> pre[i]) & 1u);
      const int last = pre[P - 1];
      const int r = n - last - 1;
      const uint32_t Q = rejected ? 0u : (uint32_t)(r * (r - 1) / 2);
      uint32_t mixed = 0;
      if (Q != 0) {
        // prefix cell `lane` (first prefix gate = most significant bit), kept if mixed
        bool mx = false;
        if (lane < NC) {
          uint32_t ones = 0, zeros = 0;
#pragma unroll
          for (int w = 0; w < NW; w++) {
            uint32_t tt = M[w];
#pragma unroll
            for (int i = 0; i < P; i++) {
              const uint32_t tv = s_tabs[w * npad + pre[i]];
              tt &= ((lane >> (P - 1 - i)) & 1) ? tv : ~tv;
            }
            cells[lane * 2 * NW + w] = tt & T[w];
            cells[lane * 2 * NW + NW + w] = tt & ~T[w];
            ones |= tt & T[w];
            zeros |= tt & ~T[w];
          }
          mx = ones != 0 && zeros != 0;
        }
        mixed = __ballot_sync(kFull, mx);
        __syncwarp();
      }
      bool done = false;
      for (uint32_t q0 = 0; q0 < Q && !done; q0 += 32) {
        const uint32_t q = q0 + lane;
        bool alive = q < Q;
        int pi = 0, pj = 1;
        if (alive) unrank_pair(q, r, pi, pj);
        const int gf = last + 1 + pi, gg = last + 1 + pj;
        if ((gf < 8 && ((inmask >> gf) & 1u)) || (gg < 8 && ((inmask >> gg) & 1u))) alive = false;
        for (uint32_t mc = mixed; mc != 0 && alive; mc &= mc - 1) {
          const int cj = __ffs(mc) - 1;
          uint32_t a11 = 0, a10 = 0, a01 = 0, a00 = 0, b11 = 0, b10 = 0, b01 = 0, b00 = 0;
#pragma unroll
          for (int w = 0; w < NW; w++) {
            const uint32_t tf = s_tabs[w * npad + gf], tg = s_tabs[w * npad + gg];
            const uint32_t c1 = cells[cj * 2 * NW + w], c0 = cells[cj * 2 * NW + NW + w];
            a11 |= c1 & tf & tg; b11 |= c0 & tf & tg;
            a10 |= c1 & tf & ~tg; b10 |= c0 & tf & ~tg;
            a01 |= c1 & ~tf & tg; b01 |= c0 & ~tf & tg;
            a00 |= c1 & ~(tf | tg); b00 |= c0 & ~(tf | tg);
          }
          if ((a11 && b11) || (a10 && b10) || (a01 && b01) || (a00 && b00)) alive = false;
        }
        for (uint32_t fb = __ballot_sync(kFull, alive); fb != 0 && !done; fb &= fb - 1) {
          const int src = __ffs(fb) - 1;
          int g5[5] = {pre[0], pre[1], pre[2], __shfl_sync(kFull, gf, src),
                       __shfl_sync(kFull, gg, src)};
          feasible++;
          uint32_t H1, H0;
          summary5<NW>(s_tabs, npad, g5, T, M, lane, H1, H0);
          for (int k = 0; k < 10 && !done; k++) {
            uint32_t ok[8], surv_mine = 0;
            outer_ok5(H1, H0, k, lane, tab, ok);
            uint32_t c = 0;
#pragma unroll
            for (int hi = 0; hi < 8; hi++) {
              const uint32_t surv = ok[hi] & __brev(ok[7 - hi]);
              c += __popc(surv);
              if (lane == hi) surv_mine = surv;
            }
            if (MODE == kEnumCount) {
              tk.count += c;
              continue;
            }
            if (c == 0) continue;
            // positions in ascending order: lane takes position 32 * w + lane
            const unsigned long long key_hi = ((base_rank + q0 + src) << 12) | ((uint64_t)k << 8);
#pragma unroll 1
            for (int w = 0; w < 8; w++) {
              const uint32_t pos = 32u * w + lane;
              const uint32_t fo = s_ord[pos];
              const bool hit = (__shfl_sync(kFull, surv_mine, fo >> 5) >> (fo & 31u)) & 1u;
              done = emit_step<MODE>(hit, tk, [&](unsigned long long i) {
                write_match<NW, 5>(out + i, key_hi | pos, g5, k, fo, 0, s_tabs, npad, T, M);
              });
            }
          }
        }
      }
    }
  });
}

// Middle functions of one cube set (see middle_cubes) as a 256-bit set over fm, word wd = fm >> 5.
__device__ __forceinline__ void cube_union(const uint32_t (*hv)[4], const bool (*hok)[4],
    uint32_t S, uint32_t ov, uint32_t *bits) {
#pragma unroll
  for (int wd = 0; wd < 8; wd++) bits[wd] = 0;
#pragma unroll
  for (int c0 = 0; c0 < 4; c0++) {
#pragma unroll
    for (int c1 = 0; c1 < 4; c1++) {
      if (!(hok[0][c0] && hok[1][c1] && ((hv[0][c0] ^ hv[1][c1]) & ov) == 0)) continue;
      const uint32_t V = hv[0][c0] | hv[1][c1];
      uint32_t low = 0xffffffffu;   // fm & 31 with (fm & S & 31) == (V & 31)
#pragma unroll
      for (int i = 0; i < 5; i++) {
        if ((S >> i) & 1u) low &= ((V >> i) & 1u) ? colour_pattern(i, 0) : ~colour_pattern(i, 0);
      }
#pragma unroll
      for (int wd = 0; wd < 8; wd++) {
        if ((((uint32_t)wd << 5) & S) == (V & 0xe0u)) bits[wd] |= low;
      }
    }
  }
}

// The 7-LUT sweep of one part over the list, tickets t_begin .. t_end-1 of it (entry idx = t *
// nparts + part), one warp per entry: the summary and stage-1 filter of k_decomp7 on the TRUE gate
// tables (no stale outer cache), then per surviving outer function and ordering row the union of
// the middle-function cubes.  Count: one lane per outer function; emit: positions in ascending
// order, outer position in the loop, middle position across the lanes.
template <int NW, int MODE>
__global__ void __launch_bounds__(kThreads) k_enum7(const DevProblem *__restrict__ prob,
    EnumCtl *__restrict__ ectl, const EnumOrders ord, const uint64_t *__restrict__ list,
    unsigned int list_count, uint32_t *__restrict__ counts,
    const unsigned long long *__restrict__ offsets, DevMatch *__restrict__ out,
    unsigned long long max_out, unsigned long long t_begin, unsigned long long t_end, int part,
    int nparts, const DevTables *__restrict__ tab) {
  constexpr bool EMIT = MODE != kEnumCount;
  extern __shared__ uint32_t smem[];
  __shared__ uint8_t s_ord[2][256];      // position -> outer / middle function
  __shared__ uint8_t s_fo[kWarpsPerCta][256];
  __shared__ uint32_t s_src7[25 * 32];
  __shared__ uint32_t s_H[kWarpsPerCta][16];
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int n = prob->n;
  const int npad = (n + 3) & ~3;
  uint32_t *s_tabs = smem;
  stage_tables(s_tabs, prob, NW, npad);
  for (int i = threadIdx.x; i < 25 * 32; i += blockDim.x) s_src7[i] = tab->src7[i >> 5][i & 31];
  for (int i = threadIdx.x; i < 512; i += blockDim.x) s_ord[i >> 8][i & 255] = ord.order[i >> 8][i & 255];
  __syncthreads();
  uint32_t T[NW], M[NW];
#pragma unroll
  for (int w = 0; w < NW; w++) {
    T[w] = prob->T[w];
    M[w] = prob->M[w];
  }
  uint32_t *sH = s_H[warp];
  uint8_t *fo_list = s_fo[warp];

  enum_tickets<MODE>(ectl, counts, offsets, max_out, t_begin, t_end,
      [&](unsigned long long t, EnumTicket &tk, unsigned long long &) {
    const uint64_t idx = t * (uint64_t)nparts + (uint64_t)part;
    if (idx < list_count) {
      const uint64_t cur = list[idx];
      int g[7];
#pragma unroll
      for (int i = 0; i < 7; i++) g[i] = (int)((cur >> (9 * (6 - i))) & 0x1ffu);
      tuple_summary<NW>(s_tabs, npad, g, T, M, lane, sH);
      const uint32_t pass_j = triples_with_colourings(sH, lane);
      bool done = false;
      for (int j = 0; j < 25 && !done; j++) {
        if (((pass_j >> j) & 1u) == 0) continue;
        uint32_t W[8], ok[8];
        outer_ok7(sH, s_src7[j * 32 + lane], lane, W, ok);
        uint32_t any = 0, surv_mine = 0;
#pragma unroll
        for (int hi = 0; hi < 8; hi++) {
          const uint32_t sv = ok[hi] & __brev(ok[7 - hi]);
          any |= sv;
          if (lane == hi) surv_mine = sv;
        }
        if (any == 0) continue;
        const int k0 = c_j_first_k[j];
        const int nrows = c_j_rows[j];
        if (!EMIT) {
          int ns = 0;
          __syncwarp();
#pragma unroll
          for (int hi = 0; hi < 8; hi++) {
            const uint32_t sv = __shfl_sync(kFull, surv_mine, hi);
            if ((sv >> lane) & 1u) fo_list[ns + __popc(sv & lanemask_lt())] = (uint8_t)(hi * 32 + lane);
            ns += __popc(sv);
          }
          __syncwarp();
          for (int i0 = 0; i0 < ns; i0 += 32) {
            const bool have = i0 + lane < ns;
            const int fo = have ? fo_list[i0 + lane] : 0;
            uint32_t r1 = 0, r0 = 0;
#pragma unroll
            for (int u = 0; u < 8; u++) {
              if ((fo >> u) & 1) r1 |= W[u]; else r0 |= W[u];
            }
            uint32_t c = 0;
#pragma unroll 1
            for (int row = 0; row < nrows; row++) {
              uint32_t hv[2][4], S, ov, bits[8];
              bool hok[2][4];
              middle_cubes(r1, r0, c_row_b[k0 + row], hv, hok, S, ov);
              cube_union(hv, hok, S, ov, bits);
#pragma unroll
              for (int wd = 0; wd < 8; wd++) c += __popc(bits[wd]);
            }
            tk.count += __reduce_add_sync(kFull, have ? c : 0u);
          }
        }
#pragma unroll 1
        for (int row = 0; EMIT && row < nrows && !done; row++) {
          const int k = k0 + row;
#pragma unroll 1
          for (int po = 0; po < 256 && !done; po++) {
            const uint32_t fo = s_ord[0][po];
            if (((__shfl_sync(kFull, surv_mine, fo >> 5) >> (fo & 31u)) & 1u) == 0) continue;
            uint32_t r1 = 0, r0 = 0;
#pragma unroll
            for (int u = 0; u < 8; u++) {
              if ((fo >> u) & 1) r1 |= W[u]; else r0 |= W[u];
            }
            uint32_t hv[2][4], S, ov;
            bool hok[2][4];
            middle_cubes(r1, r0, c_row_b[k], hv, hok, S, ov);
            const unsigned long long key_hi = (idx << 23) | ((uint64_t)k << 16) | ((uint64_t)po << 8);
#pragma unroll 1
            for (int w = 0; w < 8; w++) {
              const uint32_t pm = 32u * w + lane;
              const uint32_t fm = s_ord[1][pm];
              bool hit = false;
#pragma unroll
              for (int c0 = 0; c0 < 4; c0++) {
#pragma unroll
                for (int c1 = 0; c1 < 4; c1++) {
                  hit |= hok[0][c0] && hok[1][c1] && ((hv[0][c0] ^ hv[1][c1]) & ov) == 0
                      && (fm & S) == (hv[0][c0] | hv[1][c1]);
                }
              }
              done = emit_step<MODE>(hit, tk, [&](unsigned long long i) {
                write_match<NW, 7>(out + i, key_hi | pm, g, k, fo, fm, s_tabs, npad, T, M);
              });
            }
          }
        }
      }
    }
  });
}


// The caller's shuffled gate order of the 3-LUT enumeration: position -> gate.
struct EnumGateOrder {
  uint16_t order[kMaxGatesPad];
};

// The 3-LUT scan of lut_search (lut.c:501-523) with nothing thrown away, tickets t_begin .. t_end-1
// of one part: a ticket is a position pair (i, k) of the gate order in lexicographic order (dealt to
// the parts in blocks of kDeal, as k_enum5 deals its prefixes), one warp per pair, lanes over the
// third position m.  The triple matches iff no cell a<<2 | b<<1 | c holds a masked 1 and a masked 0
// of the target (scan3_blocks' test, here on the compressed tables).  Key i << 18 | k << 9 | m, so a
// ticket's matches are consecutive keys in the order of its lanes.  A match's record: the gates in
// position order, func_inner = cells holding a masked 1, inner_seen = cells holding a masked
// position (sbg_solve_inner's closed form).
template <int NW, int MODE>
__global__ void __launch_bounds__(kThreads) k_enum3(const DevProblem *__restrict__ prob,
    EnumCtl *__restrict__ ectl, const EnumGateOrder go, uint32_t *__restrict__ counts,
    const unsigned long long *__restrict__ offsets, DevMatch *__restrict__ out,
    unsigned long long max_out, unsigned long long t_begin, unsigned long long t_end, int part,
    int nparts) {
  extern __shared__ uint32_t smem[];
  __shared__ uint16_t s_order[kMaxGatesPad];
  const int lane = threadIdx.x & 31;
  const int n = prob->n;
  const int npad = (n + 3) & ~3;
  uint32_t *s_tabs = smem;
  stage_tables(s_tabs, prob, NW, npad);
  for (int i = threadIdx.x; i < n; i += blockDim.x) s_order[i] = go.order[i];
  __syncthreads();
  uint32_t T[NW], Z[NW];   // masked positions with target 1 / with target 0
#pragma unroll
  for (int w = 0; w < NW; w++) {
    T[w] = prob->T[w];
    Z[w] = prob->M[w] & ~prob->T[w];
  }
  const uint64_t pairs = (uint64_t)(n * (n - 1) / 2);

  enum_tickets<MODE>(ectl, counts, offsets, max_out, t_begin, t_end,
      [&](unsigned long long t, EnumTicket &tk, unsigned long long &) {
    const uint64_t dealt = dealt_item(t, part, nparts);
    if (dealt < pairs) {
      int pi, pk;
      unrank_pair((uint32_t)dealt, n, pi, pk);
      const uint32_t *ta = s_tabs + s_order[pi], *tb = s_tabs + s_order[pk];
      bool done = false;
      for (int m0 = pk + 1; m0 < n && !done; m0 += 32) {
        const int pm = m0 + lane;
        const uint32_t *tc = s_tabs + s_order[pm < n ? pm : pk];
        uint32_t one[8], zero[8];
#pragma unroll
        for (int c = 0; c < 8; c++) one[c] = zero[c] = 0;
#pragma unroll
        for (int w = 0; w < NW; w++) {
          const uint32_t va = ta[w * npad], vb = tb[w * npad], vc = tc[w * npad];
#pragma unroll
          for (int c = 0; c < 8; c++) {
            const uint32_t ab = ((c & 4) ? va : ~va) & ((c & 2) ? vb : ~vb);   // warp-uniform
            const uint32_t cell = ab & ((c & 1) ? vc : ~vc);
            one[c] |= cell & T[w];
            zero[c] |= cell & Z[w];
          }
        }
        uint32_t ones = 0, seen = 0;   // bit c: cell c holds a masked 1 / any masked position
        bool ok = pm < n;
#pragma unroll
        for (int c = 0; c < 8; c++) {
          ok &= !(one[c] != 0 && zero[c] != 0);
          if (one[c] != 0) ones |= 1u << c;
          if ((one[c] | zero[c]) != 0) seen |= 1u << c;
        }
        done = emit_step<MODE>(ok, tk, [&](unsigned long long i) {
          const int G[3] = {s_order[pi], s_order[pk], s_order[pm]};
          store_match<3>(out + i, ((unsigned long long)pi << 18) | ((unsigned long long)pk << 9)
              | (unsigned)pm, G, 0, 0, ones, seen);
        });
      }
    }
  });
}


// k_enum_locate's mark for a rank no ticket of the share holds (global ranks only).
constexpr unsigned long long kEnumUnowned = ~0ull;

// The ticket of each requested rank (ranks[i] < the count pass's total): the last t < tickets with
// offsets[t] <= ranks[i], by binary search over the count pass's offsets.  A ticket without matches
// has its successor's offset, so it is never the answer.
// Global offsets (k_enum_rebase) hold the share's ranks only, so the answer's range
// [offsets[t], offsets[t] + counts[t]) may miss the rank, and offsets[0] may exceed it (the search
// then ends at lo = 0); given counts, such a rank gets kEnumUnowned instead.  A global fetch passes
// no counts: its launch runs from the first rank's ticket (0 if the rank lies below offsets[0]) to
// the last rank's, and the range emit skips every ticket whose matches lie outside the window.
__global__ void __launch_bounds__(256) k_enum_locate(const unsigned long long *__restrict__ offsets,
    unsigned long long tickets, const unsigned long long *__restrict__ ranks,
    unsigned long long nranks, unsigned long long *__restrict__ ticket_of,
    const uint32_t *__restrict__ counts) {
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < nranks;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned long long r = ranks[i];
    // offsets[lo] <= r (local offsets: offsets[0] = 0; global ones: unless lo = 0), offsets[hi] > r
    unsigned long long lo = 0, hi = tickets;
    while (hi - lo > 1) {
      const unsigned long long mid = lo + (hi - lo) / 2;
      if (offsets[mid] <= r) lo = mid; else hi = mid;
    }
    const bool owned = counts == nullptr || (r >= offsets[lo] && r - offsets[lo] < counts[lo]);
    ticket_of[i] = owned ? lo : kEnumUnowned;
  }
}

// ---- global ranks across shares (sbg_enum_block_sums / sbg_enum_set_global) ----------------------
// A share's tickets fall into deal blocks of B tickets: B = kDeal for widths 3 and 5 (local block j
// is the whole's block j * nparts + part, the `dealt` numbering of the kernels above), B = 1 for
// width 7 (local ticket t is list entry t * nparts + part).  The whole's blocks are in key order, so
// a ticket's global offset is the whole's exclusive prefix of block sums at its block plus its
// offset within the block.

// The match count of each of the share's deal blocks: out[j] = counts[j*B .. j*B + B-1] summed (a
// widening copy for B = 1).  tickets is a multiple of B.
__global__ void __launch_bounds__(256) k_enum_block_sums(const uint32_t *__restrict__ counts,
    unsigned long long nblocks, unsigned int B, unsigned long long *__restrict__ out) {
  for (unsigned long long j = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; j < nblocks;
       j += (unsigned long long)gridDim.x * blockDim.x) {
    unsigned long long s = 0;
    for (unsigned int i = 0; i < B; i++) s += counts[j * B + i];
    out[j] = s;
  }
}

// One tile of an exclusive prefix sum over the CTA's threads (blockDim.x a multiple of 32, at most
// 1,024), one value c per thread, every thread taking part: returns carry plus the sum of the tile's
// values in front of this thread's, and advances carry by the tile's sum.
__device__ __forceinline__ unsigned long long tile_scan(unsigned long long c,
    unsigned long long &carry) {
  __shared__ unsigned long long s_warp[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long incl = c;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned long long up = __shfl_up_sync(kFull, incl, d);
    if (lane >= d) incl += up;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  unsigned long long before = 0;
  for (int i = 0; i < warp; i++) before += s_warp[i];
  unsigned long long tile = 0;
  for (int i = 0; i < (int)(blockDim.x >> 5); i++) tile += s_warp[i];
  __syncthreads();   // s_warp is free for the next tile
  const unsigned long long excl = carry + before + incl - c;
  carry += tile;
  return excl;
}

// Exclusive prefix sum over the whole's deal blocks g = 0 .. nblocks-1, block g being part
// q = g % nparts's local block g / nparts with sums[q * stride + g / nparts] matches.  For this
// share's blocks (q == part): delta[j] = (global start of block j) - offsets[j * B], the amount
// k_enum_rebase adds to the block's local offsets; ectl->gbad = 1 if the share's row of sums differs
// from its own block sums `own` (a gather in the wrong part order), ectl->gtotal = the whole's total.
// One CTA of 1,024 threads, a tile of 1,024 blocks at a time.
__global__ void __launch_bounds__(1024) k_enum_globalize(EnumCtl *__restrict__ ectl,
    const unsigned long long *__restrict__ sums, unsigned long long stride,
    unsigned long long nblocks, int part, int nparts, const unsigned long long *__restrict__ own,
    const unsigned long long *__restrict__ offsets, unsigned int B,
    unsigned long long *__restrict__ delta) {
  __shared__ unsigned int s_bad;
  if (threadIdx.x == 0) s_bad = 0;
  unsigned long long carry = 0;
  for (unsigned long long g0 = 0; g0 < nblocks; g0 += blockDim.x) {
    const unsigned long long g = g0 + threadIdx.x;
    const unsigned long long j = g / (unsigned long long)nparts;
    const int q = (int)(g % (unsigned long long)nparts);
    const unsigned long long c = g < nblocks ? sums[(unsigned long long)q * stride + j] : 0ull;
    const unsigned long long start = tile_scan(c, carry);
    if (g < nblocks && q == part) {
      delta[j] = start - offsets[j * B];
      if (c != own[j]) s_bad = 1;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    ectl->gtotal = carry;
    ectl->gbad = s_bad;
  }
}

// offsets[t] += delta[t / B]: the share's local offsets become global ones.  delta is computed
// beforehand so that no thread reads a block-start offset another thread has already rebased.
__global__ void __launch_bounds__(256) k_enum_rebase(unsigned long long *__restrict__ offsets,
    unsigned long long tickets, unsigned int B, const unsigned long long *__restrict__ delta) {
  for (unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; t < tickets;
       t += (unsigned long long)gridDim.x * blockDim.x) {
    offsets[t] += delta[t / B];
  }
}

// Exclusive prefix sum of counts[t_begin .. t_end-1] into offsets, continuing from ectl->carry
// (the matches of earlier windows), which it advances.  One CTA of 1,024 threads, a tile of 1,024
// tickets at a time.
__global__ void __launch_bounds__(1024) k_enum_scan(EnumCtl *__restrict__ ectl,
    const uint32_t *__restrict__ counts, unsigned long long *__restrict__ offsets,
    unsigned long long t_begin, unsigned long long t_end) {
  unsigned long long carry = ectl->carry;
  for (unsigned long long t0 = t_begin; t0 < t_end; t0 += blockDim.x) {
    const unsigned long long t = t0 + threadIdx.x;
    const unsigned long long start = tile_scan(t < t_end ? counts[t] : 0ull, carry);
    if (t < t_end) offsets[t] = start;
  }
  if (threadIdx.x == 0) ectl->carry = carry;
}

}  // namespace sbg
