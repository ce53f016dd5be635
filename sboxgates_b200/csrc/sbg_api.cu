// sbg_api.cu -- host side of libsboxgates_b200.so: the C ABI declared in
// include/sboxgates_b200.h.  No search logic runs on the CPU here except the O(256) decode of the
// winning key into the reference's ret[] vocabulary (sbg_finish5 / sbg_finish7); there is no CPU
// fallback -- without a CUDA device sbg_create() fails.
#include "sbg_device.cuh"

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <map>
#include <type_traits>
#include <utility>
#include <vector>

#include "../../include/sboxgates_b200.h"

using namespace sbg;

namespace {

// ---- combinatorics and ordering tables (host copies) -------------------------------------------

uint64_t h_binom[501][8];
int h_rows7[70][7];
int h_rows7c[210][7];
int h_rows4s[12][5];
int h_rows5[10][5];
bool g_tables_ready = false;

void build_host_tables() {
  if (g_tables_ready) return;
  for (int m = 0; m <= 500; m++) {
    for (int r = 0; r < 8; r++) {
      if (r > m) {
        h_binom[m][r] = 0;
      } else if (r == 0) {
        h_binom[m][r] = 1;
      } else {
        h_binom[m][r] = h_binom[m - 1][r - 1] + (r <= m - 1 ? h_binom[m - 1][r] : 0);
      }
    }
  }
  // lut.c:189,224-229: outer = 3-subsets of {0..4} in lexicographic order, rest ascending.
  int k = 0;
  for (int a = 0; a < 5; a++) for (int b = a + 1; b < 5; b++) for (int c = b + 1; c < 5; c++) {
    int w = 3;
    h_rows5[k][0] = a; h_rows5[k][1] = b; h_rows5[k][2] = c;
    for (int i = 0; i < 5; i++) {
      if (i != a && i != b && i != c) h_rows5[k][w++] = i;
    }
    k++;
  }
  // lut.c:396-415: outer = 3-subsets of {0..6} (lexicographic), middle = 3-subsets of the other
  // four (lexicographic), kept iff min(outer) < min(middle); last = the leftover position.
  k = 0;
  for (int a = 0; a < 7; a++) for (int b = a + 1; b < 7; b++) for (int c = b + 1; c < 7; c++) {
    int rest[4], r = 0;
    for (int i = 0; i < 7; i++) {
      if (i != a && i != b && i != c) rest[r++] = i;
    }
    for (int skip = 3; skip >= 0; skip--) {
      int mid[3], m = 0;
      for (int i = 0; i < 4; i++) {
        if (i != skip) mid[m++] = rest[i];
      }
      if (a >= mid[0]) continue;
      h_rows7[k][0] = a; h_rows7[k][1] = b; h_rows7[k][2] = c;
      h_rows7[k][3] = mid[0]; h_rows7[k][4] = mid[1]; h_rows7[k][5] = mid[2];
      h_rows7[k][6] = rest[skip];
      k++;
    }
  }
  // chain rows (sbg_chain_row): k = 6 j + q, j = the outer triple's lexicographic index, q = that
  // of the pair {d, e} among the four other positions; f, g = the other two, ascending.
  k = 0;
  for (int a = 0; a < 7; a++) for (int b = a + 1; b < 7; b++) for (int c = b + 1; c < 7; c++) {
    int rest[4], r = 0;
    for (int i = 0; i < 7; i++) {
      if (i != a && i != b && i != c) rest[r++] = i;
    }
    for (int d = 0; d < 4; d++) for (int e = d + 1; e < 4; e++) {
      int *row = h_rows7c[k++];
      row[0] = a; row[1] = b; row[2] = c; row[3] = rest[d]; row[4] = rest[e];
      int w = 5;
      for (int i = 0; i < 4; i++) {
        if (i != d && i != e) row[w++] = rest[i];
      }
    }
  }
  // shared-input rows (sbg_shared_row): k = 3 j + q, j = the position of d (the gate L1 does not
  // read), q = the index of the shared gate s among L1's three positions; record order: L1's
  // positions ascending, then {s, d} ascending.
  k = 0;
  for (int j = 0; j < 4; j++) {
    int l1[3], r = 0;
    for (int i = 0; i < 4; i++) {
      if (i != j) l1[r++] = i;
    }
    for (int q = 0; q < 3; q++) {
      int *row = h_rows4s[k++];
      row[0] = l1[0]; row[1] = l1[1]; row[2] = l1[2];
      row[3] = std::min(l1[q], j);
      row[4] = std::max(l1[q], j);
    }
  }
  g_tables_ready = true;
}

void unrank_combination(uint64_t rank, int n, int t, uint16_t *out) {
  int x = 0;
  for (int pos = 0; pos < t; pos++) {
    for (;; x++) {
      const uint64_t cnt = h_binom[n - x - 1][t - pos - 1];
      if (rank < cnt) break;
      rank -= cnt;
    }
    out[pos] = (uint16_t)x++;
  }
}

int popcount256(const uint64_t *m) {
  return __builtin_popcountll(m[0]) + __builtin_popcountll(m[1]) + __builtin_popcountll(m[2])
      + __builtin_popcountll(m[3]);
}

}  // namespace

// ---- handle ----------------------------------------------------------------------------------

namespace {
constexpr int kSlots = SBG_PROBLEM_SLOTS;
constexpr int kLanes = SBG_LANES;
constexpr size_t kPerPrefixMax = SBG_LIST_CAP + 32 * 512;  // hits one prefix can emit
constexpr size_t kPerChunkMax = 32 * 512;                  // hits one (prefix, chunk) item can emit
constexpr size_t kDefaultHitsCap = (size_t)4 << 20;        // entries; grown once on overflow
constexpr size_t kGrownHitsCap = (size_t)32 << 20;
constexpr uint64_t kTicketTableMax = (uint64_t)1 << 24;    // tickets per launch (table entries)
constexpr uint64_t kTicketSlack = 16384;                   // tickets fetched past the end (one per warp)
}  // namespace

// A device array the handle owns: cap elements at p (none until the first grow), freed with its
// owner.  The handle's device is current whenever an owner is destroyed (sbg_destroy); a handle
// that never bound a device holds no array, so destroying it makes no CUDA call.
template <class T>
struct DevArray {
  T *p = nullptr;
  uint64_t cap = 0;
  DevArray() = default;
  DevArray(const DevArray &) = delete;
  DevArray &operator=(const DevArray &) = delete;
  ~DevArray() {
    if (p != nullptr) cudaFree(p);
  }
  int grow(sbg_handle *h, cudaStream_t stream, uint64_t need);
};

// One lane = one CUDA stream with its own control words, parameter block, hit buffers and result
// block: the unit a search chain runs on.  Single calls use lane 0; sbg_search_batch() spreads
// independent searches over the lanes so that their kernels overlap on the device.
struct sbg_lane {
  cudaStream_t own_stream = nullptr;
  cudaStream_t stream = nullptr;
  DevArray<DevCtl> d_ctl;
  DevArray<DevParams7> d_par7;
  DevArray<uint8_t> d_pos5;
  HostOut *h_out = nullptr;      // mapped pinned: written by the device, polled here
  HostOut *d_out = nullptr;      // the same block through its device address
  DevCtl *h_ctl = nullptr;       // pinned: control words read back by the step-by-step calls
  // d_hits and d_aux grow together: d_hits.cap is the hit buffers' capacity
  DevArray<uint64_t> d_hits;     // unordered hits (filter7) / (rank, tuple) pairs (two-kernel search5)
  DevArray<uint64_t> d_aux;      // (ticket, index in ticket) of each hit
  DevArray<uint64_t> d_sorted;   // the ordered, capped list (SBG_LIST_CAP entries)
  DevArray<uint32_t> d_tcount;   // hits per ticket
  DevArray<uint32_t> d_toffset;  // their exclusive prefix sum
  DevArray<uint32_t> d_gcount;   // hits per group of 1,024 tickets
  DevArray<uint64_t> d_sieve3;   // phase 1's pair sieve per 3-gate prefix (k_sieve3)
  cudaEvent_t ev[8] = {};        // timing (only with sbg_set_timing)
  cudaEvent_t ev_done = nullptr; // end of the lane's last chain
  bool ev_ready = false;
  // sbg_search_batch, one slot on several lanes of a wave: the lane's last k_begin brought the
  // slot's problem block or rows up to date (prepared); ev_begun follows it when mark_begun is set
  bool prepared = false;
  bool mark_begun = false;
  cudaEvent_t ev_begun = nullptr;
  uint64_t seq = 0;
  // what the host adds to the sweep counters of the lane's last search_5lut / phase-1 launch (see
  // head_skipped)
  uint64_t skipped5 = 0, skipped7 = 0;
  int slot = -1;                 // problem the lane's chain works on
  bool timed5 = false, timed7 = false;
  float ms[4] = {0, 0, 0, 0};
};

// The handle's 7-LUT list and what the last sbg_decomp7_part found in it.  Lane 0's d_sorted is the
// list's storage; the other lanes' d_sorted serve only their own chains in sbg_search_batch.
struct List7 {
  uint32_t count = 0;
  bool whole = false;   // the problem's full list, which phase 2 may use (else one part's)
  int slot = -1;        // the problem it was built for: a slot and that slot's version (-1: none)
  uint64_t version = 0;
  uint64_t swept = 0;   // this device's phase-1 sweep behind the list (sbg_finish7's tuples_swept)
  uint64_t last_key = SBG_KEY_NONE;   // sbg_decomp7_part's result and the two list entries behind it
  uint64_t last_tuple = 0, last_tuple_prev = 0;
};

// The enumeration's device buffers, each allocated on its first need.  Enumerations run on lane 0
// only, so the handle holds one set and grows it on lane 0's stream.
struct EnumBuffers {
  DevArray<EnumCtl> d_ectl;
  DevArray<uint32_t> d_ecount;             // matches per ticket
  DevArray<unsigned long long> d_eoffset;  // their exclusive prefix sum
  DevArray<DevMatch> d_ematch;             // the emitted records
  DevArray<unsigned long long> d_ehist;    // filtered count: matches per depth (kDepthBins)
  // fetch and pick on an enumeration cursor
  DevArray<unsigned long long> d_pranks;   // requested ranks, ascending
  DevArray<unsigned int> d_pslots;         // their output slots
  DevArray<unsigned long long> d_ptickets; // ticket of each rank, then the distinct tickets
  DevArray<unsigned int> d_pfirst;         // each distinct ticket's first rank in d_pranks
  DevArray<unsigned long long> d_psizes;   // group sizes of the requested ranks, by slot
  // global ranks (sbg_enum_block_sums / sbg_enum_set_global)
  DevArray<unsigned long long> d_bsums;    // the share's block sums
  DevArray<unsigned long long> d_delta;    // what k_enum_rebase adds to each of its blocks
  DevArray<unsigned long long> d_gsums;    // every share's block sums, one row per part
};

// What the enumeration kernels of one width read besides the problem block: the function order(s)
// (widths 5 and 7) or the gate order (width 3), the kernel form (EnumForm), the 7-LUT ticket source
// (Enum7Source; kSrcList at the other widths), the 7-LUT shape (Enum7Shape; the chain over the list
// in the plain form only) and, for the filtered and grouped forms, the filter block (take_filter;
// its histogram pointer is the lane's, set at launch).
struct EnumInputs {
  EnumOrders ord;
  EnumGateOrder gates;
  int form;
  int source;
  int shape = kShapeTree;
  EnumFilter filter;
};

// The depth filter of a handle (sbg_enum_set_depth): the depths of n gates and the bound.
struct DepthFilter {
  bool on = false;
  int n = 0;
  uint32_t max_depth = 0;
  uint16_t depth[SBG_MAX_GATES] = {};
};

// The function filter of a handle (sbg_enum_set_functions): the sets and inner_all of EnumFilter,
// ready for the kernels.
struct FunctionFilter {
  bool on = false;
  uint32_t sets[16 + kInnerWords] = {};
  int inner_all = 0;
};

// The enumeration cursor: what sbg_enum_fetch / sbg_enum_pick need of the last counted enumeration
// besides the counts and offsets it left in the handle's EnumBuffers.  Valid while seq equals the
// handle's api_seq.
struct EnumCursor {
  bool made = false;
  uint64_t seq = 0;
  int width = 0, part = 0, nparts = 1, slot = -1;
  EnumInputs in;
  uint64_t tickets = 0, total = 0;
  uint32_t list_count = 0;   // width 7 over the list
  uint64_t blocks = 0;       // the whole's deal blocks (every part's)
  bool global = false;       // sbg_enum_set_global ran: offsets and total are the whole's
};

struct sbg_handle {
  int device = 0;
  int sm_count = 0;
  sbg_lane lane[kLanes];
  cudaStream_t user_stream = nullptr;

  DevArray<DevProblem> d_slots;  // kSlots device-resident problems
  uint64_t *h_stage = nullptr;   // pinned staging block for large table changes
  DevArray<DevTables> d_tab;     // lane-indexed ordering tables
  DevArray<uint32_t> d_scratch;  // sbg_alu_peak
  EnumBuffers ebuf;
  List7 list7;

  // host copies of the staged problems (for sbg_finish*)
  struct HostProblem {
    uint64_t tables[SBG_MAX_GATES][4];
    uint64_t target[4];
    uint64_t mask[4];
    int n = 0;
    int nw = 0;
    int m = 0;
    uint32_t inmask = 0;
    bool ready = false;
    bool rows_ready = false;     // DevProblem::xr built on the device
    int busy_lane = -1;          // lane whose chain may still be reading the slot
    cudaEvent_t uploaded = nullptr;
    // what the device holds of this state: gates [0, dev_n) of `tables` are in DevProblem::full,
    // gates [0, comp_n) are compressed under the current target/mask, the header is current
    int dev_n = 0;
    int comp_n = 0;
    bool header_valid = false;
    uint64_t version = 0;        // bumped by every staged change (not by an identical restage)
  };
  HostProblem *slots = nullptr;  // kSlots entries
  int cur_slot = 0;
  bool problem_ready = false;

  uint64_t swept5 = 0;      // the last sbg_search5_part's work counters, read by sbg_finish5
  uint64_t feasible5 = 0;
  std::map<std::pair<const void *, size_t>, int> occupancy;  // grid_for's cache
  std::map<const void *, size_t> smem_attr;                  // largest dynamic smem opted into
  // Kernel-form switches, read from the environment when the handle is created.  Each forces one
  // form of a kernel that the automatic choice would not pick for the same state, so that tests can
  // compare the forms with each other and with the oracle.  SBG_TICKET_TABLE and SBG_HITS_CAP (below)
  // shrink the ticket table and the hit buffer to reach the segment and overflow-retry paths.
  int opt_pm_prefix = 0;    // SBG_PM_PREFIX: 4 or 5 (0 = by n)
  int opt_search5 = 0;      // SBG_SEARCH5: 0 by size, 1 fused, 2 two kernels
  int opt_head = -1;        // SBG_HEAD: chunked phase of the 7-LUT filter, 0 none, 1 first prefixes,
                            // 2 everything (-1 = by n and mask size)
  int opt_shift = -1;       // SBG_SHIFT: phase-1 shifted single-word windows, 0 never, 1 whenever n <= 63
  int opt_packed = 1;       // SBG_PACKED: phase 1 keeps two parts per register where <= 15 last gates remain
  int opt_sieve = 1;        // SBG_SIEVE: phase 1 (shifted windows) rules out last gates with the pair sieve
                            // first: 0 never, 1 above kSieveMinPositions masked positions, 2 always
  int opt_decomp_filter = 1;  // SBG_DECOMP_FILTER: lane-parallel stage-1 filter of phase 2 (0 = ballot form only)
  bool concurrent = false;  // set while sbg_search_batch enqueues more than one chain
  bool hits_cap_forced = false;
  size_t hits_cap_default = kDefaultHitsCap;
  uint64_t ticket_table_max = kTicketTableMax;
  bool timing = false;
  uint64_t launches = 0;
  uint64_t uploads_full = 0, uploads_incremental = 0, uploads_skipped = 0;
  uint64_t h2d_bytes = 0, d2h_bytes = 0;   // problem data shipped / results read, over the handle's life
  float last_ms[4] = {0, 0, 0, 0};         // kernel families of the last call (timing mode)
  double host_s[2] = {0, 0};               // host seconds: enqueueing chains, waiting + decoding
  double wait_s[3] = {0, 0, 0};            // of the waiting: for the 3-LUT scan, search_5lut, search_7lut
  char err[512] = {0};
  // bumped by every entry point that launches device work or changes a problem, a list or the
  // enumeration buffers; the enumeration cursor lives as long as it does not change
  uint64_t api_seq = 0;
  EnumCursor cursor;
  DepthFilter filter;   // read by sbg_enum3 / sbg_enum5 / sbg_enum7 only
  FunctionFilter functions;   // likewise
  int grouping = SBG_GROUP_NONE;   // likewise (sbg_enum_set_grouping)
};

namespace {

int fail(sbg_handle *h, int code, const char *fmt, ...) {
  if (h != nullptr) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(h->err, sizeof(h->err), fmt, ap);
    va_end(ap);
  }
  return code;
}

#define SBG_CUDA(h, call)                                                                  \
  do {                                                                                     \
    cudaError_t e_ = (call);                                                               \
    if (e_ != cudaSuccess) {                                                               \
      return fail((h), SBG_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), \
          __FILE__, __LINE__);                                                             \
    }                                                                                      \
  } while (0)

}  // namespace

// Grows the array to `need` elements.  Work queued on `stream` may still read the old array, so
// growing waits for it; the contents are not kept.
template <class T>
int DevArray<T>::grow(sbg_handle *h, cudaStream_t stream, uint64_t need) {
  if (cap >= need) return SBG_OK;
  SBG_CUDA(h, cudaStreamSynchronize(stream));
  cudaFree(p);
  p = nullptr;
  cap = 0;
  SBG_CUDA(h, cudaMalloc(&p, need * sizeof(T)));
  cap = need;
  return SBG_OK;
}

namespace {

template <int NW>
size_t sweep_smem(int n) {
  const int npad = (n + 3) & ~3;
  return sizeof(uint32_t) * (size_t)(NW * npad + kWarpsPerCta * 8 * 2 * NW);
}

template <int NW>
size_t decomp_smem(int n) {
  const int npad = (n + 3) & ~3;
  return sizeof(uint32_t) * (size_t)(NW * npad);
}

// k_enum7_all and k_enum7_chain: the tables and each warp's prefix cells.
template <int NW>
size_t enum7_all_smem(int n) {
  return decomp_smem<NW>(n) + sizeof(uint32_t) * (size_t)(kWarpsPerCta * kPrefix7Cells * NW);
}

// Kernels whose dynamic shared memory can exceed the 48 KB default opt in once per size class.
template <typename Kernel>
int ensure_smem(sbg_handle *h, Kernel kernel, size_t smem) {
  if (smem <= 48 * 1024) return SBG_OK;
  const void *key = reinterpret_cast<const void *>(kernel);
  auto it = h->smem_attr.find(key);
  if (it != h->smem_attr.end() && it->second >= smem) return SBG_OK;
  SBG_CUDA(h, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  h->smem_attr[key] = smem;
  return SBG_OK;
}

// Persistent grid: as many CTAs as are resident at once, but no more than there is work for.
template <typename Kernel>
int grid_for(sbg_handle *h, Kernel kernel, size_t smem, uint64_t work_items_in_warps) {
  // the occupancy query costs a few microseconds; a search makes several launches and a graph
  // build makes tens of thousands of searches, so remember the answer per (kernel, smem size)
  auto &cache = h->occupancy;   // per handle: handles may be driven from different threads
  const auto key = std::make_pair(reinterpret_cast<const void *>(kernel), smem);
  int per_sm = 1;
  auto it = cache.find(key);
  if (it != cache.end()) {
    per_sm = it->second;
  } else {
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kThreads, smem);
    cache[key] = per_sm;
  }
  if (per_sm < 1) per_sm = 1;
  uint64_t want = (work_items_in_warps + kWarpsPerCta - 1) / kWarpsPerCta;
  uint64_t cap = (uint64_t)per_sm * (uint64_t)h->sm_count;
  if (want < 1) want = 1;
  return (int)std::min(want, cap);
}

// One launch of a chain.  pdl: the kernel may start while its predecessor in the stream drains
// (programmatic dependent launch); it calls wait_for_predecessor() before touching anything the
// predecessor writes.
template <typename... KArgs, typename... Args>
cudaError_t launch(sbg_handle *h, void (*kernel)(KArgs...), int grid, int block, size_t smem,
    cudaStream_t stream, bool pdl, Args &&...args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)grid, 1, 1);
  cfg.blockDim = dim3((unsigned)block, 1, 1);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  h->launches++;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// f(nw_c) with the problem's table width in 32-bit words (1, 2, 4 or 8) as the compile-time
// constant decltype(nw_c)::value, for the kernels templated on it.
template <class F>
auto with_nw(int nw, F &&f) {
  switch (nw) {
    case 1: return f(std::integral_constant<int, 1>());
    case 2: return f(std::integral_constant<int, 2>());
    case 4: return f(std::integral_constant<int, 4>());
    default: return f(std::integral_constant<int, 8>());
  }
}

// f(form_c) with the enumeration kernel form (EnumForm) as the compile-time constant
// decltype(form_c)::value.  Width 3 has no grouped form (take_filter never picks it there).  The
// count, range and pick passes (MODE kEnumCount, kEnumRange, kEnumPick) run in every form of the
// width; the sizes pass (kEnumSizes) runs on grouped cursors of widths 5 and 7 only, so it has the
// grouped form alone.
template <int WIDTH, int MODE, class F>
auto with_form(int form, F &&f) {
  static_assert(MODE != kEnumSizes || WIDTH != 3, "width 3 has no sizes pass");
  if constexpr (MODE == kEnumSizes) {
    return f(std::integral_constant<int, kFormGrouped>());
  } else {
    if constexpr (WIDTH != 3) {
      if (form == kFormGrouped) return f(std::integral_constant<int, kFormGrouped>());
    }
    if (form == kFormFiltered) return f(std::integral_constant<int, kFormFiltered>());
    return f(std::integral_constant<int, kFormPlain>());
  }
}

// Prefixes per ticket batch.  One batch costs one global atomic; batches should hold enough pairs
// to hide its latency (~64 chunks of 32), leave several batches per resident warp, and never hold
// more work than a warp's fair share (prefixes are dealt heaviest first, so the tail evens out).
//
// The batch size also defines how work is dealt to the parts of a sharded search (part p takes
// batches p, p + nparts, ...), so it must be the same on every rank: it is a function of the
// problem and a nominal warp count only, never of the device a rank happens to run on: two CTAs on
// each of the H100 SXM's 132 SMs.
constexpr uint64_t kNominalWarps = 132 * 2 * kWarpsPerCta;

constexpr int kSinglePrefixMaxGates = 72;
// Shifted single-word windows in phase 1 up to here (SBG_SHIFT=0|1 overrides): faster than the
// aligned two-word windows under a full mask, by less as n grows (scripts/sweep_shift.sh compares
// the two).
constexpr int kShiftMaxGates = 60;
// Phase 1's pair sieve (shifted windows) above this many masked positions (SBG_SIEVE=0|1|2
// overrides).  On one H100 at n = 40 it took the launches under 256 / 128 / 64 positions from
// 0.393 / 0.277 / 0.231 ms to 0.264 / 0.231 / 0.212 ms (0.212 / 0.199 / 0.212 ms with its pairs
// built once per 3-gate prefix, k_sieve3); under 32 positions the cell loop visits about 10
// positions per chunk, fewer than the sieve and its table cost (0.220 -> 0.249 ms forced on).
constexpr int kSieveMinPositions = 32;
// Phase-1 prefixes per ticket (4-gate prefixes, n <= kSinglePrefixMaxGates) while several chains
// share the device (sbg_search_batch).
constexpr uint64_t kConcurrentBatch = 2;
uint64_t pick_batch(const sbg_handle *h, uint64_t tickets, int n, int P) {
  const uint64_t warps = kNominalWarps;
  // work per ticket in lane-items: (d,e) pairs for the 5-LUT sweep (P = 3), (e,f) pairs for the
  // position-major kernel with 4-gate prefixes (P = 4), single f for its 5-gate form (P = 6)
  const bool pm = P == 4 || P == 6;
  // position-major kernel, 4-gate prefixes: single prefixes up to n = 72 (faster than the formula
  // below at n = 48 and 64 under a full mask; from n = 80 on the formula's 4 is as good or better)
  // ... when the kernel has the device to itself.  Several chains at once (sbg_search_batch) fill
  // each other's tails, and what counts is fewer trips to the ticket counter: on bench.py's step
  // (n = 40, 8 states) pairs of prefixes beat single prefixes and fours.
  if (P == 4 && n <= kSinglePrefixMaxGates) return h->concurrent ? kConcurrentBatch : 1;
  const uint64_t total = pm ? h_binom[n - 1][6] : h_binom[n][P + 2];
  const uint64_t avg_pairs = std::max<uint64_t>(1, total / std::max<uint64_t>(1, tickets));
  const uint64_t qmax = P == 6 ? (uint64_t)std::max(1, n - 7) : h_binom[n - P - (P == 4 ? 1 : 0)][2];
  uint64_t b = (64 * 32 + avg_pairs - 1) / avg_pairs;
  b = std::min<uint64_t>(b, std::max<uint64_t>(1, tickets / (warps * 4)));
  b = std::min<uint64_t>(b, std::max<uint64_t>(1, total / (warps * std::max<uint64_t>(1, qmax))));
  b = std::max<uint64_t>(1, std::min<uint64_t>(16, b));
  while (b & (b - 1)) b &= b - 1;   // power of two: a batch must not straddle two deal blocks
  return b;
}

// Chunked phase of phase 1 (see k_filter7_pm): a head of kHeadWaves waves of (prefix, chunk) items
// in front of the prefix form.  A list that fills early -- small masks make most combinations
// feasible -- then costs microseconds instead of the first wave of whole-prefix batches, which at
// large n is enormous (n = 200 - 500 with 16-32 masked positions: seconds to minutes through the
// overflow retry without the head, well under a millisecond with it; scripts/dense_cases.py).
// Sweeping EVERYTHING in chunk items is much slower where the sweep has to cover the space (n = 128,
// 64 positions: about 15 times), so that form is kept for the overflow retry.  Below
// kHeadAlwaysMinGates the head is used for small masks only, below kHeadMinGates never (the
// rijndael -o 0 run and bench.py at n = 40 are indifferent to it).
constexpr int kHeadAlwaysMinGates = 128;
constexpr int kHeadMaxPositions = 64;
constexpr int kHeadMinGates = 48;
constexpr uint64_t kHeadWaves = 64;
constexpr uint64_t kHeadWaves5 = 16;   // search_5lut: the first match is what ends it, a short head does

struct ChunkPlan {
  unsigned long long items = 0;     // (prefix, chunk) items of the chunked phase
  int chunks = 0;                   // chunks per prefix
  unsigned long long t_offset = 0;  // rank of the first prefix left to the prefix form
  bool all = false;                 // the chunked phase covers everything
};

// K = size of the combinations, P = gates per prefix, mode: 0 none, 1 a head of `waves` waves of chunk
// tickets, 2 everything in chunk tickets.
template <int P, int K>
ChunkPlan plan_chunks_mode(int n, uint32_t inmask, int mode, uint64_t waves, uint64_t qmax) {
  ChunkPlan pl;
  const int na = n - __builtin_popcount(inmask & 0xffu);   // allowed gates
  const uint64_t total_c = na >= K ? h_binom[na - (K - P)][P] : 0;
  if (mode == 0 || total_c == 0) return pl;
  // qmax = lane items of the first (largest) prefix
  pl.chunks = (int)std::max<uint64_t>(1, (qmax + 31) / 32);
  uint64_t prefixes = total_c;
  if (mode == 1) {
    prefixes = std::min<uint64_t>(total_c,
        std::max<uint64_t>(1, waves * kNominalWarps / (uint64_t)pl.chunks));
  }
  pl.items = prefixes * (uint64_t)pl.chunks;
  pl.all = prefixes == total_c;
  if (!pl.all) {
    // the first allowed prefix not covered: index `prefixes` among the P-subsets of the allowed
    // gates, as gate numbers, ranked among the P-subsets of all gates
    int c[P];
    uint64_t t = prefixes;
    const int np = na - (K - P);
    int x = 0;
    for (int pos = 0; pos < P; pos++) {
      for (;; x++) {
        const uint64_t cnt = h_binom[np - x - 1][P - pos - 1];
        if (t < cnt) break;
        t -= cnt;
      }
      c[pos] = x++;
    }
    for (int i = 0; i < P; i++) {
      int g = c[i];
      for (int bit = 0; bit < 8; bit++) g += (((inmask >> bit) & 1u) != 0 && bit <= g) ? 1 : 0;
      c[i] = g;
    }
    const int nr = n - (K - P);
    uint64_t rank = 0;
    int prev = -1;
    for (int pos = 0; pos < P; pos++) {
      for (int y = prev + 1; y < c[pos]; y++) rank += h_binom[nr - y - 1][P - pos - 1];
      prev = c[pos];
    }
    pl.t_offset = rank;
  }
  return pl;
}

// The combinations of the P-gate prefixes in front of the first prefix the prefix tickets take
// (all prefixes when the chunk tickets cover everything) that hold an excluded gate.  The chunk
// tickets walk the allowed gates only, so no ticket meets these prefixes and no kernel credits
// them; the reference steps through them one by one (lut.c:174-187, 294-305), so the host adds them
// to the sweep of part 0.  Each prefix weighs the C(n-1-last, K-P) combinations that complete it.
template <int P, int K>
uint64_t head_skipped(int n, uint32_t inmask, const ChunkPlan &pl) {
  inmask &= 0xffu;
  if (pl.items == 0 || inmask == 0) return 0;
  const int nr = n - (K - P);   // prefix gates are < nr
  const uint64_t end = h_binom[nr][P];
  const uint64_t t_end = pl.all ? end : pl.t_offset;
  // the prefix at rank t_end (the first one left to the prefix tickets: made of allowed gates)
  int t[P];
  if (t_end < end) {
    uint64_t r = t_end;
    int x = 0;
    for (int pos = 0; pos < P; pos++) {
      for (;; x++) {
        const uint64_t cnt = h_binom[nr - x - 1][P - pos - 1];
        if (r < cnt) break;
        r -= cnt;
      }
      t[pos] = x++;
    }
  }
  // weight of the prefixes below t_end, over all gates (excl = 0) or over the allowed ones:
  // f[r][v] = the weight of the r more gates above v (gates above v allowed), summed
  auto below = [&](uint32_t excl) {
    static thread_local uint64_t f[P][SBG_MAX_GATES + 1];
    for (int v = nr - 1; v >= 0; v--) f[0][v] = h_binom[n - 1 - v][K - P];
    for (int r = 1; r < P; r++) {
      uint64_t acc = 0;
      for (int v = nr - 1; v >= 0; v--) {
        f[r][v] = acc;
        if (!(v < 8 && ((excl >> v) & 1u))) acc += f[r - 1][v];
      }
    }
    uint64_t w = 0;
    int lo = 0;
    for (int pos = 0; pos < P; pos++) {
      const int hi = t_end < end ? t[pos] : nr;
      for (int u = lo; u < hi; u++) {
        if (!(u < 8 && ((excl >> u) & 1u))) w += f[P - 1 - pos][u];
      }
      if (t_end >= end) break;
      lo = t[pos] + 1;
    }
    return w;
  };
  return below(0) - below(inmask);
}

sbg_handle::HostProblem &cur(sbg_handle *h) { return h->slots[h->cur_slot]; }

// ---- lane resources (allocated on first need: most graphs never run a large 7-LUT search) ------

int ensure_hits(sbg_handle *h, sbg_lane &L, uint64_t cap) {
  int rc;
  if ((rc = L.d_hits.grow(h, L.stream, cap)) != SBG_OK) return rc;
  if ((rc = L.d_aux.grow(h, L.stream, cap)) != SBG_OK) return rc;
  return L.d_sorted.grow(h, L.stream, SBG_LIST_CAP);
}

int ensure_tickets(sbg_handle *h, sbg_lane &L, uint64_t tickets) {
  uint64_t want = L.d_tcount.cap;
  if (want < tickets) {
    // grow generously: reallocation synchronises the lane
    want = std::max<uint64_t>(tickets, (uint64_t)1 << 18);
    want = std::min<uint64_t>(std::max<uint64_t>(want, 2 * L.d_tcount.cap),
        h->ticket_table_max + kTicketSlack);
    want = std::max<uint64_t>(want, tickets);
  }
  int rc;
  if ((rc = L.d_tcount.grow(h, L.stream, want)) != SBG_OK) return rc;
  if ((rc = L.d_toffset.grow(h, L.stream, want)) != SBG_OK) return rc;
  return L.d_gcount.grow(h, L.stream, want / kTicketGroup + 2);
}

// The k_sieve3 table for n gates: C(n - 4, 3) entries of kSieve3Words words, 7.3 MB at n = 40,
// 28.4 MB at n = 60 (the shifted windows' limit).  Entry ranks do not depend on n, so a table
// allocated for a larger n serves every smaller one.
int ensure_sieve3(sbg_handle *h, sbg_lane &L, int n) {
  return L.d_sieve3.grow(h, L.stream, h_binom[n - 4][3] * kSieve3Words);
}

// The chain about to be enqueued on lane L reads problem slot `slot`: order it after the slot's
// upload (when that went through another stream) and remember who is reading.
int lane_uses_slot(sbg_handle *h, sbg_lane &L, int slot) {
  sbg_handle::HostProblem &hp = h->slots[slot];
  if (L.stream != h->lane[0].stream && hp.uploaded != nullptr) {
    SBG_CUDA(h, cudaStreamWaitEvent(L.stream, hp.uploaded, 0));
  }
  L.slot = slot;
  hp.busy_lane = (int)(&L - h->lane);
  return SBG_OK;
}

void record_done(sbg_handle *h, sbg_lane &L) {
  if (&L != &h->lane[0]) {
    cudaEventRecord(L.ev_done, L.stream);
    L.ev_ready = true;
  }
}

// ---- waiting for a stage ---------------------------------------------------------------------

double wall_now() {
  struct timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}

// Spins on the lane's mapped result block until the device has stored this call's sequence number
// for `stage`.  No CUDA call on the fast path; every ~2 ms of waiting the stream is queried so that
// a failed launch turns into an error instead of a hang.
int wait_stage(sbg_handle *h, sbg_lane &L, int stage) {
  // stage 0 (the 3-LUT scan) publishes seq << 28 | key in one word, see scan3_blocks
  volatile unsigned long long *flag = &L.h_out->seq[stage];
  const int shift = stage == 0 ? kScanKeyBits : 0;
  uint64_t spins = 0;
  const double t_wait = wall_now();
  while ((*flag >> shift) != L.seq) {
    __builtin_ia32_pause();
    if ((++spins & 0x3ffff) == 0) {
      const cudaError_t e = cudaStreamQuery(L.stream);
      if (e != cudaSuccess && e != cudaErrorNotReady) {
        return fail(h, SBG_ERR_CUDA, "search chain failed: %s", cudaGetErrorString(e));
      }
      if (e == cudaSuccess && (*flag >> shift) != L.seq) {
        return fail(h, SBG_ERR_STATE, "internal: chain ended without publishing stage %d", stage);
      }
    }
  }
  __atomic_thread_fence(__ATOMIC_ACQUIRE);
  if (stage == 0) {
    const unsigned long long key = *flag & kScanKeyNone;
    L.h_out->key[0] = key == kScanKeyNone ? SBG_KEY_NONE : key;
  }
  h->wait_s[stage] += wall_now() - t_wait;
  return SBG_OK;
}

// Control words of the lane, by copy (the step-by-step calls, which do not close a stage).
int fetch_ctl(sbg_handle *h, sbg_lane &L) {
  SBG_CUDA(h, cudaMemcpyAsync(L.h_ctl, L.d_ctl.p, sizeof(DevCtl), cudaMemcpyDeviceToHost,
      L.stream));
  SBG_CUDA(h, cudaStreamSynchronize(L.stream));
  return SBG_OK;
}

float elapsed(cudaEvent_t a, cudaEvent_t b) {
  float ms = 0.f;
  if (cudaEventElapsedTime(&ms, a, b) != cudaSuccess) {
    (void)cudaGetLastError();  // do not leave a sticky "last error" behind
    return 0.f;
  }
  return ms;
}

// ---- chain pieces ----------------------------------------------------------------------------

struct CallInputs {
  const uint8_t *order5 = nullptr;
  const uint8_t *outer = nullptr;
  const uint8_t *middle = nullptr;
  const uint16_t *gate_order = nullptr;
};

int enqueue_begin(sbg_handle *h, sbg_lane &L, uint32_t flags, const CallInputs &in, uint32_t gcount_n);

// search_5lut.  Small searches (the bulk of a real run) use two kernels -- a sweep that only
// records feasible tuples, then one warp per recorded tuple -- so that the decomposition of several
// feasible tuples met by one warp is not serialised; large ones use the fused kernel, whose ordered
// early exit matters there.
bool search5_two_kernels(const sbg_handle *h, int n) {
  const uint64_t two_kernel_max = 4000000;  // C(n,5) up to n = 52
  return h->opt_search5 != 0 ? h->opt_search5 == 2 : h_binom[n][5] <= two_kernel_max;
}

// head = false keeps the fused form on the prefix deal (see sbg_search5_part's fallback).
int enqueue_search5(sbg_handle *h, sbg_lane &L, int part, int nparts, bool two, bool head = true) {
  const sbg_handle::HostProblem &hp = h->slots[L.slot];
  const int n = hp.n;
  constexpr int P = 3;
  const uint64_t total = h_binom[n - 2][P];
  int rc;
  if (two && (rc = ensure_hits(h, L, h->hits_cap_default)) != SBG_OK) return rc;
  // search_5lut on a large state (fused kernel): a head of chunk tickets, so that on a dense state
  // the feasible-but-not-decomposable tuples in front of the first match are spread over the
  // machine instead of being decomposed by the one warp that owns their prefix
  ChunkPlan pl;
  if (!two && head && h->opt_head != 0 && n >= kHeadAlwaysMinGates) {
    pl = plan_chunks_mode<P, P + 2>(n, hp.inmask, 1, kHeadWaves5, h_binom[n - 3][2]);
  }
  L.skipped5 = part == 0 ? head_skipped<P, P + 2>(n, hp.inmask, pl) : 0;
  const uint64_t tickets = pl.all ? 0 : (total - pl.t_offset + nparts - 1) / nparts;
  const uint64_t chunk_tickets = (pl.items + kDeal * nparts - 1) / (kDeal * nparts) * kDeal;
  if (h->timing) cudaEventRecord(L.ev[6], L.stream);
  const cudaError_t e = with_nw(hp.nw, [&](auto nw_c) {
    constexpr int NW = decltype(nw_c)::value;
    const size_t smem = sweep_smem<NW>(n);
    const int grid = grid_for(h, k_sweep<NW>, smem, tickets + chunk_tickets);
    const uint64_t bsz = pick_batch(h, tickets, n, P);
    cudaError_t e = launch(h, k_sweep<NW>, grid, kThreads, smem, L.stream, !h->timing,
        h->d_slots.p + L.slot, L.d_ctl.p, L.d_out, L.d_pos5.p, L.d_hits.p,
        (unsigned long long)L.d_hits.cap, part, nparts, (int)bsz, two, h->d_tab.p,
        pl.all ? (unsigned long long)total : pl.t_offset, pl.items, std::max(1, pl.chunks),
        (unsigned long long)chunk_tickets);
    if (e == cudaSuccess && two) {
      e = launch(h, k_decomp5<NW>, 2 * h->sm_count, kThreads, decomp_smem<NW>(n), L.stream, true,
          h->d_slots.p + L.slot, L.d_ctl.p, L.d_out, L.d_pos5.p, L.d_hits.p, h->d_tab.p);
    }
    return e;
  });
  if (e != cudaSuccess) return fail(h, SBG_ERR_CUDA, "search5 launch: %s", cudaGetErrorString(e));
  if (h->timing) {
    cudaEventRecord(L.ev[7], L.stream);
    L.timed5 = true;
  }
  return SBG_OK;
}

template <int NW, int P>
size_t filter_pm_smem(int n, int m, bool shifted = false, bool sieve = false) {
  const int npad = (n + 3) & ~3;
  const int ngw = (((n + 31) >> 5) + 1) & ~1;
  return sizeof(uint32_t) * (size_t)(NW * npad + ((m * ngw + 3) & ~3)
      + kWarpsPerCta * ((1 << P) * NW + ngw * 32 + (sieve ? kSieveWords : 0))
      + (shifted ? std::max(n - 6, 1) * m : 0));
}

// Position-major phase 1 (k_filter7_pm): work items are 4- or 5-gate prefixes.  The 5-gate form does
// half the work per visited position but keeps only n-7-ish lanes of a warp busy, so it is used
// from n = kPm5MinGates on (the measured cross-over; scripts/sweep_pm_prefix.sh); SBG_PM_PREFIX=4|5
// overrides.
constexpr int kPm5MinGates = 128;
template <int P>
ChunkPlan plan_chunks(const sbg_handle *h, const sbg_handle::HostProblem &hp, bool retry) {
  const int n = hp.n;
  int mode = h->opt_head;
  if (mode < 0) {
    mode = n >= kHeadAlwaysMinGates || (hp.m <= kHeadMaxPositions && n >= kHeadMinGates) ? 1 : 0;
  }
  // overflow retry: one form for everything, so that the bound on the hits in flight is simple --
  // chunk items where a prefix is large, whole prefixes otherwise
  if (retry) mode = n >= kHeadAlwaysMinGates ? 2 : 0;
  // lane items: (e,f) pairs out of the n-5 gates that leave room for g; single f for 5-gate prefixes
  const uint64_t qmax = P == 4 ? h_binom[n - 5][2] : (uint64_t)(n - 6);
  return plan_chunks_mode<P, 7>(n, hp.inmask, mode, kHeadWaves, qmax);
}

// How one phase-1 launch is cut into tickets: everything the filter, k_offsets and k_begin must
// agree on.
struct FilterPlan {
  ChunkPlan pl;
  uint64_t total = 0;          // prefixes
  uint64_t tickets = 0;        // whole-prefix tickets' prefixes of this part
  uint64_t chunk_tickets = 0;
  uint64_t batch = 1;
  uint64_t ticket_bound = 0;   // tickets this part can be handed (incl. the overshoot)
  uint64_t tickets_cap = 0;    // ticket table entries in use by the launch
  int max_warps = 0;
  bool five = false;
  uint64_t seg_base = 0;       // first ticket of this launch (sweeps larger than the ticket table)
  uint32_t list_base = 0;      // list entries earlier segments produced
  WeightedTickets wt;          // group_pairs != 0: every ticket is a (prefix, group of pairs)
};

// Ticket tables of the weighted form (see WeightedTickets): f(d) tickets for a prefix whose last
// gate is d, suffix sums level by level.
void build_weighted(int n, uint32_t group_pairs, WeightedTickets *wt) {
  memset(wt, 0, sizeof *wt);
  const int np = n - 3;   // prefix elements are < np (three more gates follow)
  if (np < 4 || np >= kWeightedRow || group_pairs == 0) return;
  wt->group_pairs = group_pairs;
  uint64_t prev[kWeightedRow + 1] = {0}, cur[kWeightedRow + 1];
  // level 1: first (= only) element d >= x
  for (int x = np - 1; x >= 0; x--) {
    const uint64_t r = (uint64_t)(n - x - 2);
    const uint64_t pairs = r >= 2 ? r * (r - 1) / 2 : 0;
    const uint64_t f = std::max<uint64_t>(1, (pairs + group_pairs - 1) / group_pairs);
    prev[x] = prev[x + 1] + f;
  }
  for (int x = 0; x < kWeightedRow; x++) wt->w[0][x] = (uint32_t)prev[x];
  for (int r = 2; r <= 4; r++) {   // level r: first element a in [x, np - r], then r-1 more above it
    memset(cur, 0, sizeof cur);
    for (int x = np - r; x >= 0; x--) cur[x] = cur[x + 1] + prev[x + 1];
    for (int x = 0; x < kWeightedRow; x++) wt->w[r - 1][x] = (uint32_t)cur[x];
    memcpy(prev, cur, sizeof cur);
  }
  wt->total = wt->w[3][0];
}

// Chunks of 32 pairs per weighted ticket.
constexpr uint32_t kGroupChunks = 6;

template <int P>
FilterPlan plan_filter_p(const sbg_handle *h, const sbg_lane &L, const sbg_handle::HostProblem &hp,
    int nparts, bool retry, uint64_t seg_base) {
  FilterPlan fp;
  fp.seg_base = seg_base;
  const int n = hp.n;
  fp.five = P == 5;
  fp.total = h_binom[n - (7 - P)][P];
  fp.pl = plan_chunks<P>(h, hp, retry);
  // No item is handed out once the list cap is reached, so with w warps at work the buffer holds
  // fewer than cap + w x (hits one item can emit) entries; a whole prefix stops by itself after
  // cap + one chunk.
  fp.max_warps = !retry ? 0 : (int)std::max<size_t>(1, fp.pl.all
      ? (L.d_hits.cap - SBG_LIST_CAP) / kPerChunkMax : L.d_hits.cap / kPerPrefixMax - 1);
  fp.tickets = fp.pl.all ? 0 : (fp.total - fp.pl.t_offset + nparts - 1) / nparts;
  // chunk tickets of one part: whole deal blocks, the same count for every part
  fp.chunk_tickets = (fp.pl.items + kDeal * nparts - 1) / (kDeal * nparts) * kDeal;
  fp.batch = fp.pl.all ? 1 : pick_batch(h, fp.tickets, n, P == 4 ? 4 : 6);
  if (fp.max_warps > 0) fp.batch = 1;
  fp.wt.group_pairs = 0;
  // Weighted tickets: a chain that has the device to itself, 4-gate prefixes, no head, no retry
  // (chains that share the device fill each other's tails and prefer fewer, larger tickets: whole
  // prefixes, see pick_batch).
  if (P == 4 && !retry && !h->concurrent && fp.pl.items == 0 && n >= 7 && n <= kWeightedMaxGates) {
    build_weighted(n, 32u * kGroupChunks, &fp.wt);
    if (fp.wt.group_pairs != 0) {
      fp.tickets = ((uint64_t)fp.wt.total + nparts - 1) / nparts;
      fp.batch = 1;
    }
  }
  fp.ticket_bound = fp.chunk_tickets + (fp.tickets + 2 * kDeal) / fp.batch + 2 + kTicketSlack;
  const uint64_t left = fp.ticket_bound > seg_base ? fp.ticket_bound - seg_base : kTicketSlack;
  fp.tickets_cap = std::min<uint64_t>(left, h->ticket_table_max + kTicketSlack);
  return fp;
}

bool filter_uses_five(const sbg_handle *h, int n) {
  return h->opt_pm_prefix != 0 ? h->opt_pm_prefix == 5 : n >= kPm5MinGates;
}

FilterPlan plan_filter(const sbg_handle *h, const sbg_lane &L, const sbg_handle::HostProblem &hp,
    int nparts, bool retry, uint64_t seg_base = 0) {
  return filter_uses_five(h, hp.n) ? plan_filter_p<5>(h, L, hp, nparts, retry, seg_base)
                                   : plan_filter_p<4>(h, L, hp, nparts, retry, seg_base);
}

// build_sieve3: the sieve's form first fills the lane's k_sieve3 table; a later launch of the same
// search (the next segment, the overflow retry) finds it filled.
template <int P>
int launch_filter7_pm_p(sbg_handle *h, sbg_lane &L, const FilterPlan &fp, int part, int nparts,
    unsigned long long list_cap, bool build_sieve3) {
  const sbg_handle::HostProblem &hp = h->slots[L.slot];
  const int n = hp.n;
  const int m = hp.m;
  const ChunkPlan &pl = fp.pl;
  const bool shifted = P == 4 && (h->opt_shift >= 0 ? h->opt_shift != 0 && n <= 63
                                                     : n <= kShiftMaxGates);
  // the pair sieve where it pays: it costs a fixed set-up per prefix, and under the smallest masks
  // the cell loop it replaces visits too few positions per chunk (SBG_SIEVE=2: always)
  const bool sieve = h->opt_sieve == 2 || (h->opt_sieve == 1 && m > kSieveMinPositions);
  return with_nw(hp.nw, [&](auto nw_c) {
    constexpr int NW = decltype(nw_c)::value;
    // one form of the kernel: the shifted / sieve flags also size its shared memory
    auto run = [&](auto kernel, bool sh, bool sv) {
      const size_t smem = filter_pm_smem<NW, P>(n, m, sh, sv);
      int rc;
      if ((rc = ensure_smem(h, kernel, smem)) != SBG_OK) return rc;
      int grid = grid_for(h, kernel, smem, fp.tickets + fp.chunk_tickets);
      if (fp.max_warps > 0) grid = std::min(grid, (fp.max_warps + kWarpsPerCta - 1) / kWarpsPerCta);
      const cudaError_t e = launch(h, kernel, grid, kThreads, smem, L.stream, !h->timing,
          h->d_slots.p + L.slot, L.d_ctl.p, L.d_hits.p, L.d_aux.p, L.d_tcount.p, L.d_gcount.p,
          (unsigned long long)L.d_hits.cap, (unsigned long long)fp.tickets_cap, part, nparts,
          list_cap, (int)fp.batch, fp.max_warps,
          pl.all ? (unsigned long long)fp.total : pl.t_offset, pl.items, std::max(1, pl.chunks),
          (unsigned long long)fp.chunk_tickets, (unsigned long long)fp.seg_base,
          h->opt_packed ? 15 : 0, fp.wt, (const uint64_t *)L.d_sieve3.p);
      if (e != cudaSuccess) return fail(h, SBG_ERR_CUDA, "k_filter7_pm: %s", cudaGetErrorString(e));
      return SBG_OK;
    };
    if constexpr (P == 4) {
      if (shifted && sieve) {
        if (build_sieve3) {
          int rc;
          if ((rc = ensure_sieve3(h, L, n)) != SBG_OK) return rc;
          const int grid = (int)((h_binom[n - 4][3] + kWarpsPerCta - 1) / kWarpsPerCta);
          const cudaError_t e = launch(h, k_sieve3<NW>, grid, kThreads, 0, L.stream, !h->timing,
              h->d_slots.p + L.slot, (const DevCtl *)L.d_ctl.p, L.d_sieve3.p);
          if (e != cudaSuccess) return fail(h, SBG_ERR_CUDA, "k_sieve3: %s", cudaGetErrorString(e));
        }
        return run(k_filter7_pm<NW, 1, P, true, true, true>, true, true);
      }
      // one word of 31 candidate gates from the first possible g on
      if (shifted) return run(k_filter7_pm<NW, 1, P, true, true, false>, true, false);
    }
    // one word of candidate gates per pass, its top bit free
    if (n <= 31) return run(k_filter7_pm<NW, 1, P, true, false, false>, false, false);
    // two words, one pass, top bit free
    if (n <= 63) return run(k_filter7_pm<NW, 2, P, true, false, false>, false, false);
    return run(k_filter7_pm<NW, 2, P, false, false, false>, false, false);
  });
}

// Phase 1 on lane L: the filter, then the ordered, capped list in L.d_sorted (ctl->list_count).
// The caller has enqueued k_begin (which cleared fp.tickets_cap / kTicketGroup + 1 group counters).
int enqueue_filter7(sbg_handle *h, sbg_lane &L, const FilterPlan &fp, int part, int nparts,
    bool build_sieve3) {
  int rc;
  const sbg_handle::HostProblem &hp = h->slots[L.slot];
  L.skipped7 = part != 0 ? 0 : fp.five ? head_skipped<5, 7>(hp.n, hp.inmask, fp.pl)
                                       : head_skipped<4, 7>(hp.n, hp.inmask, fp.pl);
  if (h->timing) cudaEventRecord(L.ev[0], L.stream);
  const unsigned long long room = (unsigned long long)SBG_LIST_CAP - fp.list_base;
  rc = fp.five ? launch_filter7_pm_p<5>(h, L, fp, part, nparts, room, build_sieve3)
               : launch_filter7_pm_p<4>(h, L, fp, part, nparts, room, build_sieve3);
  if (rc != SBG_OK) return rc;
  if (h->timing) cudaEventRecord(L.ev[1], L.stream);
  const uint64_t groups = (fp.tickets_cap + kTicketGroup - 1) / kTicketGroup;
  // the grid covers the tickets that can have been handed out; CTAs past the counter return at once
  cudaError_t e = launch(h, k_offsets, (int)groups, 256, 0, L.stream, !h->timing, L.d_ctl.p,
      L.d_tcount.p, L.d_gcount.p, L.d_toffset.p, (unsigned long long)fp.tickets_cap,
      (unsigned int)SBG_LIST_CAP, (unsigned int)fp.list_base);
  if (e == cudaSuccess) {
    e = launch(h, k_scatter, 2 * h->sm_count, 256, 0, L.stream, true, L.d_ctl.p, L.d_hits.p,
        L.d_aux.p, L.d_toffset.p, L.d_sorted.p, (unsigned long long)L.d_hits.cap,
        (unsigned int)SBG_LIST_CAP);
  }
  if (e != cudaSuccess) return fail(h, SBG_ERR_CUDA, "ordering launch: %s", cudaGetErrorString(e));
  if (h->timing) {
    cudaEventRecord(L.ev[2], L.stream);
    L.timed7 = true;
  }
  return SBG_OK;
}

// Phase 2 on the lane's list (length on the device).  Closes stage 2.
int enqueue_decomp7(sbg_handle *h, sbg_lane &L, int part, int nparts, uint64_t items_hint) {
  const sbg_handle::HostProblem &hp = h->slots[L.slot];
  const int n = hp.n;
  const cudaError_t e = with_nw(hp.nw, [&](auto nw_c) {
    constexpr int NW = decltype(nw_c)::value;
    const size_t smem = decomp_smem<NW>(n);
    const int grid = grid_for(h, k_decomp7<NW>, smem, items_hint);
    return launch(h, k_decomp7<NW>, grid, kThreads, smem, L.stream, !h->timing,
        h->d_slots.p + L.slot, L.d_ctl.p, L.d_out, L.d_par7.p, L.d_sorted.p, part, nparts,
        h->d_tab.p, h->opt_decomp_filter);
  });
  if (e != cudaSuccess) return fail(h, SBG_ERR_CUDA, "k_decomp7: %s", cudaGetErrorString(e));
  if (h->timing) cudaEventRecord(L.ev[3], L.stream);
  return SBG_OK;
}

void collect_times(sbg_handle *h, sbg_lane &L) {
  if (!h->timing) return;
  for (int i = 0; i < 4; i++) L.ms[i] = 0.f;
  if (L.timed5) {
    cudaEventSynchronize(L.ev[7]);
    L.ms[0] = elapsed(L.ev[6], L.ev[7]);
  }
  if (L.timed7) {
    cudaEventSynchronize(L.ev[3]);
    L.ms[1] = elapsed(L.ev[0], L.ev[1]);
    L.ms[2] = elapsed(L.ev[1], L.ev[2]);
    L.ms[3] = elapsed(L.ev[2], L.ev[3]);
  }
  L.timed5 = L.timed7 = false;
}

bool valid_order(const uint8_t *order) {
  if (order == nullptr) return false;
  bool seen[256] = {false};
  for (int i = 0; i < 256; i++) {
    if (seen[order[i]]) return false;
    seen[order[i]] = true;
  }
  return true;
}

// ---- phase 1, step by step (sharded calls, overflow handling, very large sweeps) ---------------

// Runs phase 1 of this part to completion on lane L and leaves the ordered list (<= SBG_LIST_CAP)
// in L.d_sorted, its length in *count_out.  Handles the hit buffer overflowing (grow once, then the
// bounded-parallelism retry) and sweeps with more tickets than the ticket table holds (several
// launches, each appending to the list: later tickets only hold larger tuples).  *swept_out = the
// combinations the part's sweep put through the feasibility test, summed over the segments.
int run_filter7(sbg_handle *h, sbg_lane &L, int part, int nparts, uint32_t *count_out,
    uint64_t *swept_out, bool overflowed_already = false) {
  sbg_handle::HostProblem &hp = h->slots[L.slot];
  int rc;
  bool retry = false;
  if (overflowed_already) {
    // the caller's own launch (the fused chain) has just overflowed this buffer: do not repeat it
    if (!h->hits_cap_forced && L.d_hits.cap < kGrownHitsCap) {
      if ((rc = ensure_hits(h, L, kGrownHitsCap)) != SBG_OK) return rc;
    } else {
      retry = true;
    }
  }
  uint64_t seg_base = 0, swept = 0;
  uint32_t list_base = 0;
  float ms_filter = 0.f, ms_order = 0.f;
  for (int overflows = 0;;) {
    if ((rc = ensure_hits(h, L, std::max(L.d_hits.cap, h->hits_cap_default))) != SBG_OK) return rc;
    FilterPlan fp = plan_filter(h, L, hp, nparts, retry, seg_base);
    fp.list_base = list_base;
    if ((rc = ensure_tickets(h, L, fp.tickets_cap)) != SBG_OK) return rc;
    L.seq++;
    CallInputs none;
    if ((rc = enqueue_begin(h, L, kBeginSearch7 | kBeginRows, none,
        (uint32_t)(fp.tickets_cap / kTicketGroup + 1))) != SBG_OK) return rc;
    // the sieve's table once per search; the fused chain that overflowed has built it already
    const bool first_launch = seg_base == 0 && overflows == 0 && !overflowed_already;
    if ((rc = enqueue_filter7(h, L, fp, part, nparts, first_launch)) != SBG_OK) return rc;
    if ((rc = fetch_ctl(h, L)) != SBG_OK) return rc;
    if (h->timing) {
      ms_filter += elapsed(L.ev[0], L.ev[1]);
      ms_order += elapsed(L.ev[1], L.ev[2]);
      L.timed7 = false;
    }
    if (L.h_ctl->overflow == 1) {
      // hit buffer overflowed: a larger buffer first (unless its size was forced), then bounded
      // parallelism: a prefix stops contributing once it has emitted SBG_LIST_CAP hits and items
      // are handed out in order, so with w warps at work (w + 1) * (hits per item) entries suffice
      if (++overflows > 2) {
        return fail(h, SBG_ERR_OVERFLOW, "7-LUT hit buffer (%zu entries) overflowed", L.d_hits.cap);
      }
      if (!h->hits_cap_forced && L.d_hits.cap < kGrownHitsCap && !retry) {
        if ((rc = ensure_hits(h, L, kGrownHitsCap)) != SBG_OK) return rc;
      } else {
        retry = true;
      }
      continue;   // the same segment again
    }
    swept += L.h_ctl->swept;
    list_base = L.h_ctl->list_count;
    if (L.h_ctl->overflow == 0 || list_base >= SBG_LIST_CAP) break;
    seg_base += fp.tickets_cap;   // ticket table exhausted: the next segment
  }
  if (h->timing) {
    L.ms[1] = ms_filter;
    L.ms[2] = ms_order;
    L.ms[3] = 0.f;
  }
  *swept_out = swept + L.skipped7;
  *count_out = list_base;
  return SBG_OK;
}

}  // namespace

namespace {

// ---- problem staging -------------------------------------------------------------------------

// Fills the problem part of a chain's first-kernel arguments from the slot's pending change and
// marks it applied.  A change of more than kArgGates gates goes through one copy into
// DevProblem::full first (rare: the first state of a run, or a jump between unrelated states).
int apply_pending(sbg_handle *h, int slot, cudaStream_t stream, BeginArgs &a, bool want_rows) {
  sbg_handle::HostProblem &hp = h->slots[slot];
  a.n = hp.n;
  a.inmask = hp.inmask;
  memcpy(a.target, hp.target, 32);
  memcpy(a.mask, hp.mask, 32);
  a.a_first = hp.n;
  a.a_count = 0;
  a.c_first = hp.n;
  bool need = false;
  if (hp.dev_n < hp.n || hp.comp_n < hp.n || !hp.header_valid) {
    const int changed = hp.n - hp.dev_n;
    if (changed > kArgGates) {
      SBG_CUDA(h, cudaStreamSynchronize(stream));   // the staging block may still be in flight
      memcpy(h->h_stage, hp.tables[hp.dev_n], (size_t)changed * 32);
      SBG_CUDA(h, cudaMemcpyAsync(&h->d_slots.p[slot].full[hp.dev_n][0], h->h_stage,
          (size_t)changed * 32, cudaMemcpyHostToDevice, stream));
      h->uploads_full++;
      h->h2d_bytes += (uint64_t)changed * 32;
    } else {
      a.a_first = hp.dev_n;
      a.a_count = changed;
      for (int k = 0; k < changed; k++) memcpy(a.newg[k], hp.tables[hp.dev_n + k], 32);
      if (changed > 0) h->uploads_incremental++;
      h->h2d_bytes += (uint64_t)changed * 32;
    }
    h->h2d_bytes += 64 + 16;
    a.c_first = hp.comp_n;
    hp.dev_n = hp.n;
    hp.comp_n = hp.n;
    hp.header_valid = true;
    need = true;
  }
  if (want_rows && !hp.rows_ready && hp.m > 0) {
    a.flags |= kBeginRows;
    hp.rows_ready = true;
    need = true;
  }
  if (need) a.flags |= kBeginProblem;
  return SBG_OK;
}

int prep_ctas(const sbg_handle::HostProblem &hp, const BeginArgs &a) {
  if (!(a.flags & kBeginProblem)) return 0;
  // warp items (one 32-bit word each): compressed tables, position-major rows; 32 warps per block,
  // a few items per warp
  const int items = std::max((hp.n - a.c_first) * 8, (a.flags & kBeginRows) ? hp.m * 16 : 0);
  return std::max(1, std::min(64, (items + 127) / 128));
}

int scan_ctas(const sbg_handle *h, int n) {
  const int pairs = n * (n - 1) / 2;
  // one position pair per warp (32 warps per block) while the device has room: the scan's result is
  // the first thing a node's host code waits for
  return std::max(1, std::min(4 * h->sm_count, (pairs + 31) / 32));
}

int stage_problem(sbg_handle *h, int slot, const uint64_t *tables, int n, const uint64_t *target,
    const uint64_t *mask, const int8_t *inbits, bool eager) {
  if (slot < 0 || slot >= kSlots) return fail(h, SBG_ERR_ARG, "slot %d out of range", slot);
  if (tables == nullptr || target == nullptr || mask == nullptr || inbits == nullptr) {
    return fail(h, SBG_ERR_ARG, "null argument");
  }
  if (n < 1 || n > SBG_MAX_GATES) return fail(h, SBG_ERR_ARG, "n = %d out of range", n);
  sbg_handle::HostProblem &hp = h->slots[slot];
  uint32_t inmask = 0;
  for (int k = 0; k < 8 && inbits[k] != -1; k++) {
    if (inbits[k] >= 0 && inbits[k] < 8) inmask |= 1u << inbits[k];
  }
  // The device keeps the gate tables of the slot's last state.  Successive states of a graph build
  // share a prefix of gates (state.h:87: gates are only ever appended; a sibling branch replaces a
  // suffix), so only the gates after the common prefix are shipped; target, mask and the selector
  // bits are 72 bytes of kernel arguments.
  const bool same_tm = hp.ready && memcmp(hp.target, target, 32) == 0
      && memcmp(hp.mask, mask, 32) == 0;
  int lcp = 0;
  if (hp.ready) {
    const int lim = std::min(hp.n, n);
    while (lcp < lim && memcmp(hp.tables[lcp], tables + 4 * lcp, 32) == 0) lcp++;
  }
  if (same_tm && hp.inmask == inmask && hp.n == n && lcp == n) {
    // lut_search calls search_5lut and then search_7lut on the same state (lut.c:553,593)
    h->uploads_skipped++;
    return SBG_OK;
  }
  // A chain on another lane may still be reading the slot (an early return from a node call leaves
  // the rest of the chain draining): order this change after it.
  if (hp.busy_lane > 0 && h->lane[hp.busy_lane].ev_ready) {
    SBG_CUDA(h, cudaStreamWaitEvent(h->lane[0].stream, h->lane[hp.busy_lane].ev_done, 0));
  }
  memcpy(hp.tables[lcp], tables + 4 * lcp, (size_t)(n - lcp) * 32);
  hp.version++;   // a list built for the slot's previous state no longer belongs to it
  memcpy(hp.target, target, 32);
  memcpy(hp.mask, mask, 32);
  hp.dev_n = std::min(hp.dev_n, lcp);
  hp.comp_n = same_tm ? std::min(hp.comp_n, lcp) : 0;
  if (hp.inmask != inmask || hp.n != n || !same_tm) hp.header_valid = false;
  hp.inmask = inmask;
  hp.n = n;
  hp.m = popcount256(mask);
  hp.nw = hp.m <= 32 ? 1 : hp.m <= 64 ? 2 : hp.m <= 128 ? 4 : 8;
  hp.ready = true;
  hp.rows_ready = false;
  if (eager) {
    BeginArgs a;
    a.flags = 0;
    int rc = apply_pending(h, slot, h->lane[0].stream, a, false);
    if (rc != SBG_OK) return rc;
    const int ctas = prep_ctas(hp, a);
    if (ctas > 0) {
      const cudaError_t e = launch(h, k_prepare_problem, ctas, 1024, 0, h->lane[0].stream, false,
          h->d_slots.p + slot, a);
      if (e != cudaSuccess) return fail(h, SBG_ERR_CUDA, "k_prepare_problem: %s", cudaGetErrorString(e));
    }
    if (hp.uploaded != nullptr) SBG_CUDA(h, cudaEventRecord(hp.uploaded, h->lane[0].stream));
  }
  return SBG_OK;
}

// ---- whole chains ------------------------------------------------------------------------------

constexpr int kDoScan3 = SBG_DO_SCAN3, kDoSearch5 = SBG_DO_SEARCH5, kDoSearch7 = SBG_DO_SEARCH7;

// First kernel of a chain: control words, position tables, minpos3, ticket-group counters, and
// whatever of the problem block has to be (re)derived.
int enqueue_begin(sbg_handle *h, sbg_lane &L, uint32_t flags, const CallInputs &in, uint32_t gcount_n) {
  sbg_handle::HostProblem &hp = h->slots[L.slot];
  BeginArgs a;
  a.seq = L.seq;
  a.gcount_n = gcount_n;
  a.flags = flags & ~(kBeginRows | kBeginProblem);
  if (flags & kBeginSearch5) {
    for (int pos = 0; pos < 256; pos++) a.pos5[in.order5[pos]] = (uint8_t)pos;
  }
  if (flags & kBeginSearch7) {
    if (in.outer != nullptr) {
      for (int pos = 0; pos < 256; pos++) {
        a.pos_outer[in.outer[pos]] = (uint8_t)pos;
        a.pos_middle[in.middle[pos]] = (uint8_t)pos;
      }
    } else {
      memset(a.pos_outer, 0, 256);
      memset(a.pos_middle, 0, 256);
    }
  }
  if (flags & kBeginScan3) memcpy(a.order3, in.gate_order, sizeof(uint16_t) * (size_t)hp.n);
  int rc = apply_pending(h, L.slot, L.stream, a, (flags & kBeginRows) != 0);
  if (rc != SBG_OK) return rc;
  const int prep = prep_ctas(hp, a);
  const int scan = (flags & kBeginScan3) ? scan_ctas(h, hp.n) : 0;
  // block 0 keeps the minpos3 visiting order, the scan blocks the uncompressed tables, in dynamic
  // shared memory
  const size_t smem = std::max<size_t>(sizeof(uint32_t) * kMinpos3, (size_t)hp.n * 32);
  const cudaError_t e = launch(h, k_begin, 1 + prep + scan, 1024, smem, L.stream, false,
      h->d_slots.p + L.slot, L.d_ctl.p, L.d_out, L.d_par7.p, L.d_pos5.p, L.d_gcount.p, h->d_tab.p,
      prep, a);
  if (e != cudaSuccess) return fail(h, SBG_ERR_CUDA, "k_begin: %s", cudaGetErrorString(e));
  L.prepared = (a.flags & kBeginProblem) != 0;
  if (L.prepared && L.mark_begun) SBG_CUDA(h, cudaEventRecord(L.ev_begun, L.stream));
  return SBG_OK;
}

// Enqueues scan3 -> search_5lut -> search_7lut (whichever `what` asks for) of the lane's problem,
// every stage predicated on the device on the earlier ones not having matched.  One launch chain,
// no host synchronisation inside.
int enqueue_chain(sbg_handle *h, sbg_lane &L, int what, const CallInputs &in) {
  sbg_handle::HostProblem &hp = h->slots[L.slot];
  int rc;
  L.seq++;
  L.skipped5 = L.skipped7 = 0;
  uint32_t flags = 0;
  if ((what & kDoScan3) && hp.n >= 3) flags |= kBeginScan3;
  if ((what & kDoSearch5) && hp.n >= 5) flags |= kBeginSearch5;
  if ((what & kDoSearch7) && hp.n >= 7) flags |= kBeginSearch7 | kBeginRows;
  uint32_t gcount_n = 0;
  FilterPlan fp;
  if (flags & kBeginSearch7) {
    if ((rc = ensure_hits(h, L, std::max(L.d_hits.cap, h->hits_cap_default))) != SBG_OK) return rc;
    fp = plan_filter(h, L, hp, 1, false);
    if ((rc = ensure_tickets(h, L, fp.tickets_cap)) != SBG_OK) return rc;
    gcount_n = (uint32_t)(fp.tickets_cap / kTicketGroup + 1);
  }
  if ((rc = enqueue_begin(h, L, flags, in, gcount_n)) != SBG_OK) return rc;
  // How far ahead of the results to launch.  A batch launches whole chains: its lanes keep the
  // device busy.  Half of a graph build's nodes end at the 3-LUT scan, which runs inside that first
  // kernel: the kernels of the later stages would return at once, but launching and draining
  // hundreds of empty blocks still occupies the stream for 15-20 us, which the NEXT node's chain then
  // waits behind.  So a single call looks at the scan's result before it launches search_5lut +
  // search_7lut (one idle launch latency for the nodes that go on, against the drain for the ones
  // that do not).
  const volatile HostOut *o = L.h_out;
  if ((flags & kBeginScan3) && !h->concurrent && (flags & (kBeginSearch5 | kBeginSearch7))) {
    if ((rc = wait_stage(h, L, 0)) != SBG_OK) return rc;
  }
  auto over = [&]() {
    const unsigned long long word = o->seq[0];   // seq << 28 | key, see scan3_blocks
    return (flags & kBeginScan3) && (word >> kScanKeyBits) == L.seq
        && (word & kScanKeyNone) != kScanKeyNone;
  };
  if ((flags & kBeginSearch5) && !over()
      && (rc = enqueue_search5(h, L, 0, 1, search5_two_kernels(h, hp.n))) != SBG_OK) return rc;
  if ((flags & kBeginSearch7) && !over()) {
    if ((rc = enqueue_filter7(h, L, fp, 0, 1, true)) != SBG_OK) return rc;
    if (!over() && (rc = enqueue_decomp7(h, L, 0, 1, SBG_LIST_CAP)) != SBG_OK) return rc;
  }
  record_done(h, L);
  return SBG_OK;
}

// What lane 0's d_sorted now holds: the whole list of `slot`'s problem as it is staged now, one
// part's list of it (sbg_filter7_part with nparts > 1), or no list.  Each replaces the whole record:
// the key and list entries the last sbg_decomp7_part left behind belong to the list it searched
// (sbg_finish7 would otherwise decode an equal key of a new list with the old list's entries).
// `swept` is this device's phase-1 sweep behind the list, which sbg_finish7 reports.
void install_list(sbg_handle *h, int slot, uint32_t count, uint64_t swept) {
  h->list7 = {count, true, slot, h->slots[slot].version, swept};
}
void record_part_list(sbg_handle *h, int slot, uint32_t count, uint64_t swept) {
  h->list7 = {count, false, slot, h->slots[slot].version, swept};
}
void drop_list(sbg_handle *h) { h->list7 = {}; }

// Whether the handle's list belongs to the current problem as it is staged now, and is whole unless
// part_ok.  A batch leaves on lane 0 the list of its last wave's first job, whatever slot that job
// searched, and restaging a slot changes its problem under the list; the list's consumers check this.
bool list_is_current(const sbg_handle *h, bool part_ok) {
  const List7 &l = h->list7;
  return (l.whole || part_ok) && h->problem_ready && l.slot == h->cur_slot
      && l.version == h->slots[h->cur_slot].version;
}

int check_job(sbg_handle *h, const sbg_job *job) {
  if (job->slot < 0 || job->slot >= kSlots || !h->slots[job->slot].ready) {
    return fail(h, SBG_ERR_STATE, "slot %d holds no problem", job->slot);
  }
  if ((job->flags & (kDoScan3 | kDoSearch5 | kDoSearch7)) == 0) {
    return fail(h, SBG_ERR_ARG, "job asks for no search");
  }
  if ((job->flags & kDoScan3) && job->gate_order == nullptr) return fail(h, SBG_ERR_ARG, "no gate order");
  if ((job->flags & kDoSearch5) && !valid_order(job->order5)) {
    return fail(h, SBG_ERR_ARG, "func_order is not a permutation");
  }
  if ((job->flags & kDoSearch7) && (!valid_order(job->outer7) || !valid_order(job->middle7))) {
    return fail(h, SBG_ERR_ARG, "function order is not a permutation");
  }
  return SBG_OK;
}

void decode3(const sbg_handle::HostProblem &hp, uint64_t key, const uint16_t *gate_order,
    sbg_node_result *res) {
  const int pos[3] = {(int)((key >> 18) & 0x1ff), (int)((key >> 9) & 0x1ff), (int)(key & 0x1ff)};
  for (int i = 0; i < 3; i++) res->gates3[i] = gate_order[pos[i]];
  res->key3 = key;
  // check_n_lut_possible(3, ...) held, so get_lut_function cannot fail (lut.c:510-516)
  sbg_solve_inner(hp.tables[res->gates3[0]], hp.tables[res->gates3[1]], hp.tables[res->gates3[2]],
      hp.target, hp.mask, &res->func3, &res->seen3);
}

int finish5_slot(sbg_handle *h, const sbg_handle::HostProblem &hp, uint64_t key,
    const uint8_t *func_order, uint64_t feasible, uint64_t swept, sbg_result *res);
int finish7_slot(sbg_handle *h, const sbg_handle::HostProblem &hp, uint64_t key,
    const uint8_t *outer_order, const uint8_t *middle_order, uint64_t tuple, uint64_t tuple_prev,
    uint64_t list_count, uint64_t swept, sbg_result *res);

// search_5lut of the lane's problem, redone with the fused kernel: the two-kernel form met more
// feasible tuples than its buffer holds.
int redo_search5_fused(sbg_handle *h, sbg_lane &L, const uint8_t *order5) {
  int rc;
  L.seq++;
  CallInputs in;
  in.order5 = order5;
  if ((rc = enqueue_begin(h, L, kBeginSearch5, in, 0)) != SBG_OK) return rc;
  if ((rc = enqueue_search5(h, L, 0, 1, false)) != SBG_OK) return rc;
  record_done(h, L);
  return wait_stage(h, L, 1);
}

// search_7lut of the lane's problem through the step-by-step path (overflow handling, segments).
// *swept = its phase-1 sweep.
int redo_search7_steps(sbg_handle *h, sbg_lane &L, const uint8_t *outer, const uint8_t *middle,
    bool hit_buffer_overflowed, uint64_t *swept) {
  int rc;
  uint32_t keep = 0;
  if ((rc = run_filter7(h, L, 0, 1, &keep, swept, hit_buffer_overflowed)) != SBG_OK) return rc;
  if (&L == &h->lane[0]) install_list(h, L.slot, keep, *swept);
  L.seq++;
  CallInputs in;
  in.outer = outer;
  in.middle = middle;
  if ((rc = enqueue_begin(h, L, kBeginSearch7 | kBeginKeepCtl, in, 0)) != SBG_OK) return rc;
  if ((rc = enqueue_decomp7(h, L, 0, 1, std::max<uint32_t>(keep, 1))) != SBG_OK) return rc;
  record_done(h, L);
  if ((rc = wait_stage(h, L, 2)) != SBG_OK) return rc;
  if (h->timing) L.ms[3] = elapsed(L.ev[2], L.ev[3]);
  return SBG_OK;
}

// Waits for the lane's chain stage by stage and fills the result.  Returns as soon as a stage
// matched (the rest of the chain drains as no-ops).
int collect_chain(sbg_handle *h, sbg_lane &L, const sbg_job *job, sbg_node_result *res) {
  const sbg_handle::HostProblem &hp = h->slots[L.slot];
  const HostOut *o = L.h_out;
  int rc;
  bool redone7 = false;
  uint64_t swept7 = 0;   // the redone phase 1's sweep
  memset(res, 0, sizeof(*res));
  res->key3 = SBG_KEY_NONE;
  res->r5.key = SBG_KEY_NONE;
  res->r7.key = SBG_KEY_NONE;
  if ((job->flags & kDoScan3) && hp.n >= 3) {
    if ((rc = wait_stage(h, L, 0)) != SBG_OK) return rc;
    h->d2h_bytes += 48;
    if (o->key[0] != SBG_KEY_NONE) {
      decode3(hp, o->key[0], job->gate_order, res);
      res->found_stage = 3;
      return SBG_OK;
    }
  }
  if ((job->flags & kDoSearch5) && hp.n >= 5) {
    if ((rc = wait_stage(h, L, 1)) != SBG_OK) return rc;
    h->d2h_bytes += 48;
    bool redone = false;
    if (o->overflow[1] != 0) {
      if ((rc = redo_search5_fused(h, L, job->order5)) != SBG_OK) return rc;
      redone = true;
    }
    if ((rc = finish5_slot(h, hp, o->key[1], job->order5, o->feasible[1],
        o->swept[1] + L.skipped5, &res->r5)) != SBG_OK) return rc;
    if (res->r5.found) {
      res->found_stage = 5;
      return SBG_OK;
    }
    if (redone && (job->flags & kDoSearch7) && hp.n >= 7) {
      // the chain's 7-LUT stage was cancelled together with the incomplete 5-LUT stage
      if ((rc = redo_search7_steps(h, L, job->outer7, job->middle7, false, &swept7)) != SBG_OK) {
        return rc;
      }
      redone7 = true;
    }
  }
  if ((job->flags & kDoSearch7) && hp.n >= 7) {
    if ((rc = wait_stage(h, L, 2)) != SBG_OK) return rc;
    h->d2h_bytes += 64;
    if (o->overflow[2] != 0 || redone7) {
      if (!redone7 && (rc = redo_search7_steps(h, L, job->outer7, job->middle7,
          o->overflow[2] == 1, &swept7)) != SBG_OK) return rc;
    } else {
      swept7 = o->swept[2] + L.skipped7;
    }
    if (&L == &h->lane[0]) install_list(h, L.slot, (uint32_t)o->feasible[2], swept7);
    if ((rc = finish7_slot(h, hp, o->key[2], job->outer7, job->middle7, o->tuple, o->tuple_prev,
        o->feasible[2], swept7, &res->r7)) != SBG_OK) return rc;
    if (res->r7.found) res->found_stage = 7;
  }
  return SBG_OK;
}

int finish5_slot(sbg_handle *h, const sbg_handle::HostProblem &hp, uint64_t key,
    const uint8_t *func_order, uint64_t feasible, uint64_t swept, sbg_result *res) {
  memset(res, 0, sizeof(*res));
  res->key = key;
  res->tuples_feasible = feasible;
  res->tuples_swept = swept;
  if (key == SBG_KEY_NONE) return SBG_OK;
  const uint64_t rank = key >> 12;
  const int k = (int)((key >> 8) & 0xf);
  const int pos = (int)(key & 0xff);
  if (k >= 10 || rank >= h_binom[hp.n][5]) return fail(h, SBG_ERR_STATE, "corrupt 5-LUT key");
  uint16_t comb[5];
  unrank_combination(rank, hp.n, 5, comb);
  const int *o = h_rows5[k];
  for (int i = 0; i < 5; i++) res->gates[i] = comb[o[i]];
  res->found = 1;
  res->ordering = k;
  res->pos_outer = pos;
  res->func_outer = func_order[pos];
  res->index = rank;
  uint64_t t_outer[4];
  sbg_lut_table(res->func_outer, hp.tables[res->gates[0]], hp.tables[res->gates[1]],
      hp.tables[res->gates[2]], t_outer);
  if (!sbg_solve_inner(t_outer, hp.tables[res->gates[3]], hp.tables[res->gates[4]], hp.target,
      hp.mask, &res->func_inner, &res->inner_seen)) {
    return fail(h, SBG_ERR_STATE, "internal: winning 5-LUT key does not decompose");
  }
  return SBG_OK;
}

int finish7_slot(sbg_handle *h, const sbg_handle::HostProblem &hp, uint64_t key,
    const uint8_t *outer_order, const uint8_t *middle_order, uint64_t cur, uint64_t prev,
    uint64_t list_count, uint64_t swept, sbg_result *res) {
  memset(res, 0, sizeof(*res));
  res->key = key;
  res->tuples_feasible = list_count;
  res->tuples_swept = swept;
  if (key == SBG_KEY_NONE) return SBG_OK;
  const uint64_t idx = key >> 23;
  const int k = (int)((key >> 16) & 0x7f);
  const int po = (int)((key >> 8) & 0xff);
  const int pm = (int)(key & 0xff);
  if (idx >= list_count || k >= 70) return fail(h, SBG_ERR_STATE, "corrupt 7-LUT key");
  uint16_t t[7];
  for (int i = 0; i < 7; i++) t[i] = (uint16_t)((cur >> (9 * (6 - i))) & 0x1ff);
  const int *o = h_rows7[k];
  for (int i = 0; i < 7; i++) res->gates[i] = t[o[i]];
  res->found = 1;
  res->ordering = k;
  res->pos_outer = po;
  res->pos_middle = pm;
  res->func_outer = outer_order[po];
  res->func_middle = middle_order[pm];
  res->index = idx;
  // lut.c:432-435 quirk (see k_decomp7): rows 0-3 may have been evaluated with the previous
  // tuple's outer tables; the solved inner function must come from the same tables.
  uint16_t outer_a = res->gates[0];
  if (idx > 0 && k < 4 && t[0] == 0) {
    if ((uint16_t)((prev >> 9) & 0x1ff) == t[1] && (uint16_t)(prev & 0x1ff) == t[2]) {
      outer_a = (uint16_t)((prev >> 45) & 0x1ff);
      res->stale_outer = 1;
    }
  }
  uint64_t t_outer[4], t_middle[4];
  sbg_lut_table(res->func_outer, hp.tables[outer_a], hp.tables[res->gates[1]],
      hp.tables[res->gates[2]], t_outer);
  sbg_lut_table(res->func_middle, hp.tables[res->gates[3]], hp.tables[res->gates[4]],
      hp.tables[res->gates[5]], t_middle);
  if (!sbg_solve_inner(t_outer, t_middle, hp.tables[res->gates[6]], hp.target, hp.mask,
      &res->func_inner, &res->inner_seen)) {
    return fail(h, SBG_ERR_STATE, "internal: winning 7-LUT key does not decompose");
  }
  return SBG_OK;
}

// ---- enumeration (sbg_enum3 / sbg_enum5 / sbg_enum7) -------------------------------------------

static_assert(kDepthBins == SBG_DEPTH_BINS && SBG_MAX_DEPTH + 2 < SBG_DEPTH_BINS,
    "every match depth has a histogram bin");
static_assert(sizeof(sbg_match) == 32 && sizeof(DevMatch) == sizeof(sbg_match)
    && offsetof(sbg_match, gates) == offsetof(DevMatch, gates)
    && offsetof(sbg_match, func_outer) == offsetof(DevMatch, func_outer)
    && offsetof(sbg_match, inner_seen) == offsetof(DevMatch, inner_seen)
    && offsetof(sbg_match, width) == offsetof(DevMatch, width)
    && offsetof(sbg_match, shape) == offsetof(DevMatch, pad), "sbg_match and DevMatch agree");
// The largest enumeration form, the filtered k_enum3: the gate order and the filter block, plus at
// most 128 bytes of pointers and scalars, within the 4 KB kernel-parameter limit.
static_assert(sizeof(EnumGateOrder) + sizeof(EnumFilter) + 128 <= 4096,
    "the filtered k_enum3's parameters fit in 4 KB");
static_assert(kEnum7AllMaxGates == SBG_ENUM7_ALL_MAX_GATES,
    "one limit of the whole-space 7-LUT sweep");

// Count-free windows start at this many tickets and double: a first-match search then costs a few
// windows of work past the first match, a search without one about twice the counting sweep's
// launches (log2 of the tickets) and no more work.
constexpr uint64_t kEnumWindow3 = kNominalWarps;
constexpr uint64_t kEnumWindow5 = kNominalWarps;
constexpr uint64_t kEnumWindow7 = kNominalWarps / 4;
// A whole-space ticket is a 6-gate prefix, up to n - 7 combinations: a window's work past the first
// match stays near a list window's with fewer tickets per window.
constexpr uint64_t kEnumWindow7All = kNominalWarps / 16;

// The first n emitted records to the caller's out.
int copy_matches(sbg_handle *h, sbg_lane &L, sbg_match *out, uint64_t n) {
  SBG_CUDA(h, cudaMemcpyAsync(out, h->ebuf.d_ematch.p, n * sizeof(sbg_match),
      cudaMemcpyDeviceToHost, L.stream));
  SBG_CUDA(h, cudaStreamSynchronize(L.stream));
  h->d2h_bytes += n * sizeof(sbg_match);
  return SBG_OK;
}

// One enumeration pass (MODE: count, range or pick emit, or sizes) of width 3, 4 (the shared-input
// two-LUT circuits of sbg_enum4_shared), 5 or 7 over tickets [a, b) of the lane's problem (pick and
// sizes: entries [a, b) of the ticket list in EnumCtl::sel).
template <int WIDTH, int MODE>
int launch_enum(sbg_handle *h, sbg_lane &L, const EnumInputs &in, int part, int nparts,
    uint64_t max_out, uint64_t a, uint64_t b) {
  static_assert(WIDTH == 3 || WIDTH == 4 || WIDTH == 5 || WIDTH == 7,
      "enumeration widths are 3, 4, 5 and 7");
  const sbg_handle::HostProblem &hp = h->slots[L.slot];
  const int n = hp.n;
  const DevProblem *prob = h->d_slots.p + L.slot;
  const EnumBuffers &E = h->ebuf;
  const int rc = with_nw(hp.nw, [&](auto nw_c) {
    constexpr int NW = decltype(nw_c)::value;
    auto run = [&](auto kernel, size_t smem, auto... args) {
      int rc;
      if ((rc = ensure_smem(h, kernel, smem)) != SBG_OK) return rc;
      const cudaError_t e = launch(h, kernel, grid_for(h, kernel, smem, b - a), kThreads, smem,
          L.stream, false, args...);
      if (e != cudaSuccess) return fail(h, SBG_ERR_CUDA, "enumeration launch: %s", cudaGetErrorString(e));
      return SBG_OK;
    };
    return with_form<WIDTH, MODE>(in.form, [&](auto form_c) {
      constexpr int FORM = decltype(form_c)::value;
      EnumFilterOf<FORM> flt = {};
      if constexpr (FORM != kFormPlain) {
        flt = in.filter;
        flt.hist = E.d_ehist.p;
      }
      if constexpr (WIDTH == 3) {
        return run(k_enum3<NW, MODE, FORM>, decomp_smem<NW>(n), prob, E.d_ectl.p, in.gates,
            E.d_ecount.p, E.d_eoffset.p, E.d_ematch.p, max_out, a, b, part, nparts, flt);
      } else if constexpr (WIDTH == 4) {
        return run(k_enum4s<NW, MODE, FORM>, sweep_smem<NW>(n), prob, E.d_ectl.p, in.ord,
            E.d_ecount.p, E.d_eoffset.p, E.d_ematch.p, max_out, a, b, part, nparts, h->d_tab.p,
            flt);
      } else if constexpr (WIDTH == 5) {
        return run(k_enum5<NW, MODE, FORM>, sweep_smem<NW>(n), prob, E.d_ectl.p, in.ord,
            E.d_ecount.p, E.d_eoffset.p, E.d_ematch.p, max_out, a, b, part, nparts, h->d_tab.p,
            flt);
      } else {
        if (in.shape == kShapeChain && in.source == kSrcList) {
          // sbg_search7_chain's first match: the plain count and range passes only
          if constexpr (FORM == kFormPlain && (MODE == kEnumCount || MODE == kEnumRange)) {
            return run(k_enum7_chain_list<NW, MODE>, decomp_smem<NW>(n), prob, E.d_ectl.p, in.ord,
                L.d_sorted.p, h->list7.count, E.d_ecount.p, E.d_eoffset.p, E.d_ematch.p, max_out,
                a, b, part, nparts, h->d_tab.p, flt);
          } else {
            return fail(h, SBG_ERR_STATE, "internal: the list-form chain has no form %d, pass %d",
                FORM, MODE);
          }
        }
        if (in.shape == kShapeChain) {
          return run(k_enum7_chain<NW, MODE, FORM>, enum7_all_smem<NW>(n), prob, E.d_ectl.p,
              in.ord, E.d_ecount.p, E.d_eoffset.p, E.d_ematch.p, max_out, a, b, part, nparts,
              h->d_tab.p, flt);
        }
        if (in.source == kSrcWhole) {
          return run(k_enum7_all<NW, MODE, FORM>, enum7_all_smem<NW>(n), prob, E.d_ectl.p,
              in.ord, E.d_ecount.p, E.d_eoffset.p, E.d_ematch.p, max_out, a, b, part, nparts,
              h->d_tab.p, flt);
        }
        return run(k_enum7<NW, MODE, FORM>, decomp_smem<NW>(n), prob, E.d_ectl.p, in.ord,
            L.d_sorted.p, h->list7.count, E.d_ecount.p, E.d_eoffset.p, E.d_ematch.p, max_out, a, b,
            part, nparts, h->d_tab.p, flt);
      }
    });
  });
  if (rc != SBG_OK) return rc;
  if (MODE == kEnumCount) {
    const cudaError_t e = launch(h, k_enum_scan, 1, 1024, 0, L.stream, false, E.d_ectl.p,
        (const uint32_t *)E.d_ecount.p, E.d_eoffset.p, (unsigned long long)a,
        (unsigned long long)b);
    if (e != cudaSuccess) return fail(h, SBG_ERR_CUDA, "k_enum_scan: %s", cudaGetErrorString(e));
  }
  return SBG_OK;
}

// Deal blocks part q of nparts holds out of `blocks` (blocks q, q + nparts, ...).
uint64_t deal_share(uint64_t blocks, int q, int nparts) {
  return blocks > (uint64_t)q ? (blocks - q + nparts - 1) / nparts : 0;
}

// Tickets per deal block of an enumeration of `width` from `source` (Enum7Source): kDeal position
// pairs, 3-gate prefixes (widths 4 and 5) or 6-gate prefixes, or one 7-LUT list entry.
unsigned int enum_block_size(int width, int source) {
  return width == 7 && source == kSrcList ? 1u : (unsigned)kDeal;
}

// sbg_enum3 / sbg_enum4_shared / sbg_enum5 / sbg_enum7 / sbg_enum7_all / sbg_enum7_chain once their
// arguments are checked.  Lane 0
// takes the current problem slot, and k_begin (flags, begin_in) brings its problem block up to date;
// a 7-LUT enumeration over the list without an installed one runs phase 1 instead, which does that
// and installs the list.  Then the part's tickets are counted (in windows when only the first
// max_matches are wanted), their offsets taken, and the first max_matches emitted and copied out.
// *swept (may be NULL): the tickets the count went through, all of the part's when counting.
template <int WIDTH>
int run_enum(sbg_handle *h, uint32_t flags, const CallInputs &begin_in, const EnumInputs &in,
    int part, int nparts, uint64_t max_matches, sbg_match *out, uint64_t *n_out, uint64_t *total,
    uint64_t *feasible, uint64_t *swept = nullptr) {
  SBG_CUDA(h, cudaSetDevice(h->device));
  sbg_lane &L = h->lane[0];
  EnumBuffers &E = h->ebuf;
  int rc;
  if ((rc = lane_uses_slot(h, L, h->cur_slot)) != SBG_OK) return rc;
  const bool whole = WIDTH == 7 && in.source == kSrcWhole;
  if (WIDTH == 7 && !whole && !list_is_current(h, false)) {
    uint32_t count = 0;
    uint64_t swept = 0;
    if ((rc = run_filter7(h, L, 0, 1, &count, &swept)) != SBG_OK) return rc;
    install_list(h, L.slot, count, swept);
  } else {
    L.seq++;
    if ((rc = enqueue_begin(h, L, flags, begin_in, 0)) != SBG_OK) return rc;
  }
  // this part's tickets: its deal blocks (the last one may be cut short)
  const int n = h->slots[L.slot].n;
  const uint64_t B = enum_block_size(WIDTH, in.source);
  const uint64_t items = WIDTH == 3 ? h_binom[n][2] : WIDTH == 4 ? h_binom[n - 1][3]
      : WIDTH == 5 ? h_binom[n - 2][3] : whole ? h_binom[n - 1][6] : h->list7.count;
  const uint64_t blocks = (items + B - 1) / B;
  const uint64_t tickets = deal_share(blocks, part, nparts) * B;
  if ((rc = E.d_ectl.grow(h, L.stream, 1)) != SBG_OK) return rc;
  const uint64_t room = std::max<uint64_t>(tickets, 1);
  if ((rc = E.d_ecount.grow(h, L.stream, room)) != SBG_OK) return rc;
  if ((rc = E.d_eoffset.grow(h, L.stream, room)) != SBG_OK) return rc;
  // also sets EnumCtl::sel.lo = 0, which the first-K range pass below relies on
  SBG_CUDA(h, cudaMemsetAsync(E.d_ectl.p, 0, sizeof(EnumCtl), L.stream));
  if (in.form != kFormPlain) {
    if ((rc = E.d_ehist.grow(h, L.stream, (uint64_t)kDepthBins)) != SBG_OK) return rc;
    SBG_CUDA(h, cudaMemsetAsync(E.d_ehist.p, 0, kDepthBins * sizeof(unsigned long long), L.stream));
  }
  const bool count_all = total != nullptr;
  uint64_t window = count_all ? tickets
      : (WIDTH == 3 ? kEnumWindow3 : WIDTH == 4 || WIDTH == 5 ? kEnumWindow5
         : whole ? kEnumWindow7All : kEnumWindow7);
  uint64_t done = 0;
  EnumCtl ec;
  memset(&ec, 0, sizeof(ec));
  while (done < tickets) {
    const uint64_t end = std::min(tickets, done + window);
    if ((rc = launch_enum<WIDTH, kEnumCount>(h, L, in, part, nparts, 0, done, end)) != SBG_OK) return rc;
    done = end;
    window *= 2;
    if (!count_all) {
      // ordered stop: every later ticket holds larger keys only
      SBG_CUDA(h, cudaMemcpyAsync(&ec, E.d_ectl.p, sizeof(ec), cudaMemcpyDeviceToHost, L.stream));
      SBG_CUDA(h, cudaStreamSynchronize(L.stream));
      if (ec.carry >= max_matches) break;
    }
  }
  SBG_CUDA(h, cudaMemcpyAsync(&ec, E.d_ectl.p, sizeof(ec), cudaMemcpyDeviceToHost, L.stream));
  SBG_CUDA(h, cudaStreamSynchronize(L.stream));
  const uint64_t emit = std::min<uint64_t>(max_matches, ec.carry);
  if (emit > 0) {
    if ((rc = E.d_ematch.grow(h, L.stream, emit)) != SBG_OK) return rc;
    // ranks [0, emit): the range pass with sel.lo = 0 from the memset above (not emit_sel, which
    // needs the cursor a count-free call does not set)
    if ((rc = launch_enum<WIDTH, kEnumRange>(h, L, in, part, nparts, emit, 0, done)) != SBG_OK) return rc;
    if ((rc = copy_matches(h, L, out, emit)) != SBG_OK) return rc;
  }
  *n_out = emit;
  if (swept != nullptr) *swept = done;
  if (count_all) {
    // every ticket counted: any rank of the share can be emitted again from counts and offsets
    EnumCursor &c = h->cursor;
    c.made = true;
    c.seq = h->api_seq;
    c.width = WIDTH;
    c.part = part;
    c.nparts = nparts;
    c.slot = L.slot;
    c.in = in;
    c.tickets = tickets;
    c.total = ec.carry;
    c.list_count = h->list7.count;
    c.blocks = blocks;
    c.global = false;
  }
  if (total != nullptr) *total = ec.carry;
  if (feasible != nullptr) {
    // width 3: every feasible triple is a match (the filtered form counts them apart)
    *feasible = WIDTH == 7 && !whole ? (uint64_t)h->list7.count
        : WIDTH == 3 && in.form == kFormPlain ? ec.total : ec.feasible;
  }
  return SBG_OK;
}

// The checks every sbg_enum3 / sbg_enum5 / sbg_enum7 call starts with.  The call ends the
// enumeration cursor, whether it succeeds or not.
int check_enum_args(sbg_handle *h, int part, int nparts, uint64_t max_matches, sbg_match *out,
    uint64_t *n_out) {
  if (h == nullptr) return SBG_ERR_ARG;
  h->api_seq++;
  if (n_out == nullptr || (max_matches > 0 && out == nullptr)) return fail(h, SBG_ERR_ARG, "null output");
  if (max_matches > SBG_ENUM_MAX_MATCHES) {
    return fail(h, SBG_ERR_ARG, "max_matches %llu above %u", (unsigned long long)max_matches,
        SBG_ENUM_MAX_MATCHES);
  }
  if (nparts < 1 || part < 0 || part >= nparts) return fail(h, SBG_ERR_ARG, "bad part %d/%d", part, nparts);
  if (!h->problem_ready) return fail(h, SBG_ERR_STATE, "no problem loaded");
  return SBG_OK;
}

// A function filter's sets (host memory, 4 words each; NULL = all 256 functions) as the kernels read
// them (EnumFilter::sets and inner_all); all three NULL gives the filter that keeps every match.
void make_functions(const uint64_t *outer, const uint64_t *middle, const uint64_t *inner,
    FunctionFilter &fn) {
  memset(fn.sets, 0, sizeof(fn.sets));
  const uint64_t *sets[2] = {outer, middle};
  for (int r = 0; r < 2; r++) {
    for (int w = 0; w < 8; w++) {
      fn.sets[8 * r + w] = sets[r] == nullptr ? 0xffffffffu
          : (uint32_t)(sets[r][w >> 1] >> (32 * (w & 1)));
    }
  }
  uint8_t table[kMinpos3];
  sbg_inner_table(inner, table);
  for (int c = 0; c < kMinpos3; c++) fn.sets[16 + (c >> 5)] |= (uint32_t)table[c] << (c & 31);
  fn.inner_all = inner == nullptr
      || (inner[0] & inner[1] & inner[2] & inner[3]) == ~0ull;
}

// The function filter that keeps every match, built once (the inner table takes 65,536 steps).
const FunctionFilter &neutral_functions() {
  static const FunctionFilter all = [] {
    FunctionFilter f;
    make_functions(nullptr, nullptr, nullptr, f);
    return f;
  }();
  return all;
}

// The handle's depth and function filters and its grouping, for an sbg_enum* call of `width` on the
// current problem, into the kernel form and its filter block.  Any setting picks the filtered form
// (grouped at widths 5 and 7 under a grouping), with the neutral filter in place of one not
// installed; none picks the plain form.
int take_filter(sbg_handle *h, int width, EnumInputs &in) {
  const DepthFilter &f = h->filter;
  const FunctionFilter &fn = h->functions;
  const int grouping = width == 3 ? SBG_GROUP_NONE : h->grouping;   // the identity at width 3
  in.form = grouping != SBG_GROUP_NONE ? kFormGrouped
      : f.on || fn.on ? kFormFiltered : kFormPlain;
  EnumFilter &flt = in.filter;
  memset(&flt, 0, sizeof(flt));
  if (in.form == kFormPlain) return SBG_OK;
  if (f.on) {
    const int n = cur(h).n;
    if (f.n != n) {
      return fail(h, SBG_ERR_ARG, "the depth filter holds %d gates, the problem has %d", f.n, n);
    }
    memcpy(flt.d, f.depth, sizeof(uint16_t) * (size_t)n);
    // no match is deeper than kDepthBins - 2, so a larger bound filters nothing more
    flt.max_depth = (int)std::min<uint32_t>(f.max_depth, kDepthBins - 1);
  } else {
    flt.max_depth = kDepthBins - 1;   // the neutral depth filter: every gate at depth 0
  }
  flt.hist_on = f.on;
  const FunctionFilter &use = fn.on ? fn : neutral_functions();
  memcpy(flt.sets, use.sets, sizeof(flt.sets));
  flt.inner_all = use.inner_all;
  flt.grouping = grouping;
  return SBG_OK;
}

// ---- fetch and pick on the enumeration cursor (sbg_enum_fetch / sbg_enum_pick) ---------------------

// The cursor, if it is still valid (nothing has run on the handle since the count that made it).
int check_cursor(sbg_handle *h) {
  const EnumCursor &c = h->cursor;
  if (!c.made || c.seq != h->api_seq) {
    return fail(h, SBG_ERR_STATE, "no enumeration cursor: fetch and pick follow a counted "
        "sbg_enum3 / sbg_enum5 / sbg_enum7 call with nothing in between");
  }
  if (h->lane[0].slot != c.slot || h->ebuf.d_ecount.cap < c.tickets
      || (c.width == 7 && c.in.source == kSrcList && h->list7.count != c.list_count)) {
    return fail(h, SBG_ERR_STATE, "internal: enumeration cursor out of step with its buffers");
  }
  return SBG_OK;
}

// Ticket of each of ranks[0..nranks-1] (already in d_pranks) into d_ptickets.  owned: ranks
// outside their ticket's range (global ranks other shares hold) get kEnumUnowned.
int locate_tickets(sbg_handle *h, sbg_lane &L, uint64_t nranks, bool owned = false) {
  const EnumBuffers &E = h->ebuf;
  const int grid = (int)std::max<uint64_t>(1, std::min<uint64_t>((nranks + 255) / 256,
      (uint64_t)h->sm_count * 8));
  const cudaError_t e = launch(h, k_enum_locate, grid, 256, 0, L.stream, false,
      (const unsigned long long *)E.d_eoffset.p, (unsigned long long)h->cursor.tickets,
      (const unsigned long long *)E.d_pranks.p, (unsigned long long)nranks, E.d_ptickets.p,
      owned ? (const uint32_t *)E.d_ecount.p : (const uint32_t *)nullptr);
  if (e != cudaSuccess) return fail(h, SBG_ERR_CUDA, "k_enum_locate: %s", cudaGetErrorString(e));
  return SBG_OK;
}

// ---- global ranks across shares (sbg_enum_block_sums / sbg_enum_set_global) ---------------------

// The cursor's block sums into d_bsums (and room for as many deltas in d_delta).
int block_sums(sbg_handle *h, sbg_lane &L, uint64_t nblocks) {
  EnumBuffers &E = h->ebuf;
  int rc;
  if ((rc = E.d_bsums.grow(h, L.stream, nblocks)) != SBG_OK) return rc;
  if ((rc = E.d_delta.grow(h, L.stream, nblocks)) != SBG_OK) return rc;
  const int grid = (int)std::max<uint64_t>(1, std::min<uint64_t>((nblocks + 255) / 256,
      (uint64_t)h->sm_count * 8));
  const cudaError_t e = launch(h, k_enum_block_sums, grid, 256, 0, L.stream, false,
      (const uint32_t *)E.d_ecount.p, (unsigned long long)nblocks,
      enum_block_size(h->cursor.width, h->cursor.in.source),
      E.d_bsums.p);
  if (e != cudaSuccess) return fail(h, SBG_ERR_CUDA, "k_enum_block_sums: %s", cudaGetErrorString(e));
  return SBG_OK;
}

// A range or pick emit pass of the cursor's width over tickets [a, b) (pick: entries [a, b) of
// sel.tickets) into d_ematch, or the sizes pass over entries [a, b) of sel.tickets into d_psizes
// (grouped cursors of widths 4, 5 and 7 only); sel and the sizes pointer travel in the EnumCtl block.
template <int MODE>
int emit_sel(sbg_handle *h, sbg_lane &L, uint64_t max_out, uint64_t a, uint64_t b,
    const EnumSel &sel) {
  const EnumCursor &c = h->cursor;
  char *ectl = reinterpret_cast<char *>(h->ebuf.d_ectl.p);
  SBG_CUDA(h, cudaMemcpyAsync(ectl + offsetof(EnumCtl, sel), &sel, sizeof(sel),
      cudaMemcpyHostToDevice, L.stream));
  if constexpr (MODE == kEnumSizes) {
    unsigned long long *sizes = h->ebuf.d_psizes.p;
    SBG_CUDA(h, cudaMemcpyAsync(ectl + offsetof(EnumCtl, sizes), &sizes, sizeof(sizes),
        cudaMemcpyHostToDevice, L.stream));
    if (c.width == 4) return launch_enum<4, MODE>(h, L, c.in, c.part, c.nparts, max_out, a, b);
    if (c.width == 5) return launch_enum<5, MODE>(h, L, c.in, c.part, c.nparts, max_out, a, b);
    return launch_enum<7, MODE>(h, L, c.in, c.part, c.nparts, max_out, a, b);
  } else {
    switch (c.width) {
      case 3: return launch_enum<3, MODE>(h, L, c.in, c.part, c.nparts, max_out, a, b);
      case 4: return launch_enum<4, MODE>(h, L, c.in, c.part, c.nparts, max_out, a, b);
      case 5: return launch_enum<5, MODE>(h, L, c.in, c.part, c.nparts, max_out, a, b);
      default: return launch_enum<7, MODE>(h, L, c.in, c.part, c.nparts, max_out, a, b);
    }
  }
}

// The checks sbg_enum_pick and sbg_enum_group_sizes start with: ranks and out given unless nranks
// is 0, nranks <= SBG_ENUM_MAX_MATCHES, a cursor, and every rank below its total.
int check_ranks(sbg_handle *h, const uint64_t *ranks, uint64_t nranks, const void *out) {
  if (nranks > 0 && (ranks == nullptr || out == nullptr)) return fail(h, SBG_ERR_ARG, "null ranks or output");
  if (nranks > SBG_ENUM_MAX_MATCHES) {
    return fail(h, SBG_ERR_ARG, "nranks %llu above %u", (unsigned long long)nranks,
        SBG_ENUM_MAX_MATCHES);
  }
  int rc;
  if ((rc = check_cursor(h)) != SBG_OK) return rc;
  const EnumCursor &c = h->cursor;
  for (uint64_t i = 0; i < nranks; i++) {
    if (ranks[i] >= c.total) {
      return fail(h, SBG_ERR_ARG, "ranks[%llu] = %llu is not below the total %llu",
          (unsigned long long)i, (unsigned long long)ranks[i], (unsigned long long)c.total);
    }
  }
  return SBG_OK;
}

// The selection a pick or sizes pass runs over: the distinct tickets (sel.tickets) holding the
// share's ranks of ranks[0 .. nranks-1] (checked, nranks > 0), with their slices of those ranks
// (sel.ranks, ascending, sel.first) and the slots that asked for them (sel.slots), uploaded.
struct RankSelection {
  EnumSel sel = {};
  uint64_t tickets = 0;              // distinct tickets (0: the share owns none of the ranks)
  std::vector<unsigned int> slots;   // the slots of the share's ranks, by ascending rank
};

int select_ranks(sbg_handle *h, sbg_lane &L, const uint64_t *ranks, uint64_t nranks,
    RankSelection &rs) {
  const EnumCursor &c = h->cursor;
  // a share without tickets (global ranks only) owns no rank
  if (c.tickets == 0) return SBG_OK;
  // host: the ranks in ascending order with the slots that asked for them
  std::vector<std::pair<uint64_t, uint32_t>> req(nranks);
  for (uint64_t i = 0; i < nranks; i++) req[i] = std::make_pair(ranks[i], (uint32_t)i);
  std::sort(req.begin(), req.end());
  std::vector<unsigned long long> sorted(nranks);
  std::vector<unsigned int> &slots = rs.slots;
  slots.resize(nranks);
  for (uint64_t i = 0; i < nranks; i++) {
    sorted[i] = req[i].first;
    slots[i] = req[i].second;
  }
  EnumBuffers &E = h->ebuf;
  int rc;
  if ((rc = E.d_pranks.grow(h, L.stream, nranks)) != SBG_OK) return rc;
  if ((rc = E.d_pslots.grow(h, L.stream, nranks)) != SBG_OK) return rc;
  if ((rc = E.d_ptickets.grow(h, L.stream, nranks)) != SBG_OK) return rc;
  if ((rc = E.d_pfirst.grow(h, L.stream, nranks + 1)) != SBG_OK) return rc;
  // device: the ticket of every rank; host: the distinct tickets and their slices of the ranks.
  // Global ranks another share owns are dropped here, so that no warp sweeps a ticket for a rank
  // it never meets.
  SBG_CUDA(h, cudaMemcpyAsync(E.d_pranks.p, sorted.data(), nranks * sizeof(unsigned long long),
      cudaMemcpyHostToDevice, L.stream));
  if ((rc = locate_tickets(h, L, nranks, c.global)) != SBG_OK) return rc;
  std::vector<unsigned long long> tickets(nranks);
  SBG_CUDA(h, cudaMemcpyAsync(tickets.data(), E.d_ptickets.p, nranks * sizeof(unsigned long long),
      cudaMemcpyDeviceToHost, L.stream));
  SBG_CUDA(h, cudaStreamSynchronize(L.stream));
  std::vector<unsigned int> firsts;
  uint64_t d = 0, m = 0;   // distinct tickets, owned ranks
  for (uint64_t i = 0; i < nranks; i++) {
    if (tickets[i] == kEnumUnowned) continue;
    if (m == 0 || tickets[i] != tickets[d - 1]) {
      tickets[d++] = tickets[i];
      firsts.push_back((unsigned int)m);
    }
    sorted[m] = sorted[i];
    slots[m] = slots[i];
    m++;
  }
  firsts.push_back((unsigned int)m);
  slots.resize(m);
  if (m < nranks) {
    SBG_CUDA(h, cudaMemcpyAsync(E.d_pranks.p, sorted.data(), m * sizeof(unsigned long long),
        cudaMemcpyHostToDevice, L.stream));
  }
  SBG_CUDA(h, cudaMemcpyAsync(E.d_ptickets.p, tickets.data(), d * sizeof(unsigned long long),
      cudaMemcpyHostToDevice, L.stream));
  SBG_CUDA(h, cudaMemcpyAsync(E.d_pfirst.p, firsts.data(), (d + 1) * sizeof(unsigned int),
      cudaMemcpyHostToDevice, L.stream));
  SBG_CUDA(h, cudaMemcpyAsync(E.d_pslots.p, slots.data(), m * sizeof(unsigned int),
      cudaMemcpyHostToDevice, L.stream));
  rs.sel.lo = 0;
  rs.sel.ranks = E.d_pranks.p;
  rs.sel.slots = E.d_pslots.p;
  rs.sel.tickets = E.d_ptickets.p;
  rs.sel.first = E.d_pfirst.p;
  rs.tickets = d;
  return SBG_OK;
}

// LOP3 issue-rate microbenchmark (sbg_alu_peak): CHAINS independent dependent chains per thread.
template <int CHAINS>
__global__ void k_lop3_peak(uint32_t *out, int iters, uint32_t seed) {
  uint32_t a[CHAINS];
#pragma unroll
  for (int i = 0; i < CHAINS; i++) a[i] = seed + threadIdx.x * 31u + i;
  uint32_t b = seed ^ 0x9e3779b9u, c = seed * 0x85ebca6bu + blockIdx.x;
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int r = 0; r < 8; r++) {
#pragma unroll
      for (int i = 0; i < CHAINS; i++) {
        asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(b), "r"(c));
      }
    }
  }
  uint32_t x = 0;
#pragma unroll
  for (int i = 0; i < CHAINS; i++) x ^= a[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = x;
}

}  // namespace

// ---- C ABI -------------------------------------------------------------------------------------

extern "C" {

int sbg_plan_tickets(int width, int prefix_gates, int n, uint32_t excluded, int mode,
    uint64_t waves, uint64_t *out) {
  build_host_tables();
  if (out == nullptr || n < width || n > SBG_MAX_GATES) return SBG_ERR_ARG;
  ChunkPlan pl;
  uint64_t total = 0;
  if (width == 7 && prefix_gates == 4 && n >= 8) {
    pl = plan_chunks_mode<4, 7>(n, excluded, mode, waves, h_binom[n - 5][2]);
    total = h_binom[n - 3][4];
  } else if (width == 7 && prefix_gates == 5 && n >= 8) {
    pl = plan_chunks_mode<5, 7>(n, excluded, mode, waves, (uint64_t)(n - 6));
    total = h_binom[n - 2][5];
  } else if (width == 5 && prefix_gates == 3 && n >= 8) {
    pl = plan_chunks_mode<3, 5>(n, excluded, mode, waves, h_binom[n - 3][2]);
    total = h_binom[n - 2][3];
  } else {
    return SBG_ERR_ARG;
  }
  out[0] = pl.items;
  out[1] = (uint64_t)pl.chunks;
  out[2] = pl.items == 0 ? 0 : (pl.all ? total : pl.t_offset);
  out[3] = total;
  return SBG_OK;
}

int sbg_weighted_tickets(int n, uint32_t group_pairs, uint32_t *out) {
  static_assert(SBG_WEIGHTED_ROW == kWeightedRow, "header and device code agree on the row length");
  if (out == nullptr || n < 7 || n > kWeightedMaxGates || group_pairs == 0) return SBG_ERR_ARG;
  WeightedTickets wt;
  build_weighted(n, group_pairs, &wt);
  if (wt.group_pairs == 0) return SBG_ERR_ARG;
  out[0] = wt.total;
  for (int r = 0; r < 4; r++) {
    for (int x = 0; x < kWeightedRow; x++) out[1 + kWeightedRow * r + x] = wt.w[r][x];
  }
  return SBG_OK;
}

int sbg_ordering_row(int width, int k, int *row) {
  build_host_tables();
  if (row == nullptr) return SBG_ERR_ARG;
  if (width == 5 && k >= 0 && k < 10) {
    for (int i = 0; i < 5; i++) row[i] = h_rows5[k][i];
    return SBG_OK;
  }
  if (width == 7 && k >= 0 && k < 70) {
    for (int i = 0; i < 7; i++) row[i] = h_rows7[k][i];
    return SBG_OK;
  }
  return SBG_ERR_ARG;
}

int sbg_chain_row(int k, int *row) {
  build_host_tables();
  if (row == nullptr || k < 0 || k >= 210) return SBG_ERR_ARG;
  for (int i = 0; i < 7; i++) row[i] = h_rows7c[k][i];
  return SBG_OK;
}

int sbg_shared_row(int k, int *row) {
  build_host_tables();
  if (row == nullptr || k < 0 || k >= 12) return SBG_ERR_ARG;
  for (int i = 0; i < 5; i++) row[i] = h_rows4s[k][i];
  return SBG_OK;
}

void sbg_lut_table(uint8_t func, const uint64_t *in1, const uint64_t *in2, const uint64_t *in3,
    uint64_t *out) {
  for (int v = 0; v < 4; v++) {
    uint64_t r = 0;
    for (int m = 0; m < 8; m++) {
      if ((func >> m) & 1) {
        r |= ((m & 4) ? in1[v] : ~in1[v]) & ((m & 2) ? in2[v] : ~in2[v])
            & ((m & 1) ? in3[v] : ~in3[v]);
      }
    }
    out[v] = r;
  }
}

int sbg_solve_inner(const uint64_t *in1, const uint64_t *in2, const uint64_t *in3,
    const uint64_t *target, const uint64_t *mask, uint8_t *func, uint8_t *seen) {
  uint8_t f = 0, s = 0;
  for (int cell = 0; cell < 8; cell++) {
    uint64_t ones = 0, zeros = 0;
    for (int v = 0; v < 4; v++) {
      const uint64_t in_cell = ((cell & 4) ? in1[v] : ~in1[v]) & ((cell & 2) ? in2[v] : ~in2[v])
          & ((cell & 1) ? in3[v] : ~in3[v]) & mask[v];
      ones |= in_cell & target[v];
      zeros |= in_cell & ~target[v];
    }
    if (ones != 0 && zeros != 0) return 0;
    if (ones != 0) f |= (uint8_t)(1u << cell);
    if ((ones | zeros) != 0) s |= (uint8_t)(1u << cell);
  }
  *func = f;
  *seen = s;
  return 1;
}

int sbg_create(sbg_handle **out, int device) {
  if (out == nullptr) return SBG_ERR_ARG;
  *out = nullptr;
  build_host_tables();
  sbg_handle *h = new sbg_handle();
  *out = h;  // returned even on failure so the caller can read the error text
  h->device = device;
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev <= 0) {
    return fail(h, SBG_ERR_CUDA, "no CUDA device available (%s); sboxgates_b200 has no CPU path",
        e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
  }
  if (device < 0 || device >= ndev) return fail(h, SBG_ERR_ARG, "device %d out of range", device);
  SBG_CUDA(h, cudaSetDevice(device));
  SBG_CUDA(h, cudaFree(nullptr));
  cudaDeviceProp prop;
  SBG_CUDA(h, cudaGetDeviceProperties(&prop, device));
  h->sm_count = prop.multiProcessorCount;
  if (getenv("SBG_PM_PREFIX") != nullptr) h->opt_pm_prefix = atoi(getenv("SBG_PM_PREFIX"));
  if (getenv("SBG_HEAD") != nullptr) h->opt_head = std::max(0, std::min(2, atoi(getenv("SBG_HEAD"))));
  if (getenv("SBG_PACKED") != nullptr) h->opt_packed = atoi(getenv("SBG_PACKED")) != 0;
  if (getenv("SBG_SHIFT") != nullptr) h->opt_shift = atoi(getenv("SBG_SHIFT")) != 0;
  if (getenv("SBG_SIEVE") != nullptr) h->opt_sieve = std::max(0, std::min(2, atoi(getenv("SBG_SIEVE"))));
  if (getenv("SBG_DECOMP_FILTER") != nullptr) {   // 0 ballot form only, 1 lane-parallel filter first
    h->opt_decomp_filter = atoi(getenv("SBG_DECOMP_FILTER")) > 0;
  }
  if (getenv("SBG_TIMING") != nullptr) h->timing = atoi(getenv("SBG_TIMING")) != 0;
  if (getenv("SBG_SEARCH5") != nullptr) {
    h->opt_search5 = strcmp(getenv("SBG_SEARCH5"), "two") == 0 ? 2 : 1;
  }
  if (getenv("SBG_TICKET_TABLE") != nullptr) {
    h->ticket_table_max = std::max<uint64_t>(4096, strtoull(getenv("SBG_TICKET_TABLE"), nullptr, 10));
  }
  const char *cap_env = getenv("SBG_HITS_CAP");
  if (cap_env != nullptr) {
    h->hits_cap_default = std::max<size_t>((size_t)strtoull(cap_env, nullptr, 10), 3 * kPerPrefixMax);
    h->hits_cap_forced = true;
  }
  int rc;
  for (int i = 0; i < kLanes; i++) {
    sbg_lane &L = h->lane[i];
    SBG_CUDA(h, cudaStreamCreateWithFlags(&L.own_stream, cudaStreamNonBlocking));
    L.stream = L.own_stream;
    for (int k = 0; k < 8; k++) SBG_CUDA(h, cudaEventCreate(&L.ev[k]));
    SBG_CUDA(h, cudaEventCreateWithFlags(&L.ev_done, cudaEventDisableTiming));
    SBG_CUDA(h, cudaEventCreateWithFlags(&L.ev_begun, cudaEventDisableTiming));
    if ((rc = L.d_ctl.grow(h, L.stream, 1)) != SBG_OK) return rc;
    {
      DevCtl init;
      memset(&init, 0, sizeof(init));
      init.best3 = ~0ull;   // the 3-LUT scan expects (and leaves) ~0 here
      SBG_CUDA(h, cudaMemcpy(L.d_ctl.p, &init, sizeof(init), cudaMemcpyHostToDevice));
    }
    if ((rc = L.d_par7.grow(h, L.stream, 1)) != SBG_OK) return rc;
    if ((rc = L.d_pos5.grow(h, L.stream, 256)) != SBG_OK) return rc;
    SBG_CUDA(h, cudaHostAlloc(&L.h_out, sizeof(HostOut), cudaHostAllocMapped));
    memset(L.h_out, 0, sizeof(HostOut));
    SBG_CUDA(h, cudaHostGetDevicePointer(&L.d_out, L.h_out, 0));
    SBG_CUDA(h, cudaMallocHost(&L.h_ctl, sizeof(DevCtl)));
  }

  SBG_CUDA(h, cudaMemcpyToSymbol(c_binom, h_binom, sizeof(h_binom)));
  {
    // search5: lane = u<<2 | v2, canonical cell bit of slot s is 4-s.
    uint8_t src5[10][32];
    for (int k = 0; k < 10; k++) {
      const int *o = h_rows5[k];
      for (int lane = 0; lane < 32; lane++) {
        const int u = lane >> 2, v = lane & 3;
        int c = 0;
        c |= ((u >> 2) & 1) << (4 - o[0]);
        c |= ((u >> 1) & 1) << (4 - o[1]);
        c |= (u & 1) << (4 - o[2]);
        c |= ((v >> 1) & 1) << (4 - o[3]);
        c |= (v & 1) << (4 - o[4]);
        src5[k][lane] = (uint8_t)c;
      }
    }
    DevTables *host_tab = new DevTables();
    memcpy(host_tab->src5, src5, sizeof(src5));

    // decomp7: group the 70 rows by outer triple; canonical cell bit of slot s (tuple_summary):
    // a..e -> 4..0, f -> 6, g -> 5.
    static const int cb[7] = {4, 3, 2, 1, 0, 6, 5};
    uint32_t src7[25][32];
    uint8_t first_k[25], nrows[25], row_b[70];
    int nj = 0;
    for (int k = 0; k < 70;) {
      const int *o = h_rows7[k];
      int rows = 1;
      while (k + rows < 70 && h_rows7[k + rows][0] == o[0] && h_rows7[k + rows][1] == o[1]
          && h_rows7[k + rows][2] == o[2]) {
        rows++;
      }
      int rest[4], r = 0;
      for (int s = 0; s < 7; s++) {
        if (s != o[0] && s != o[1] && s != o[2]) rest[r++] = s;
      }
      for (int i = 0; i < rows; i++) {
        const int gslot = h_rows7[k + i][6];
        int m = 0;
        while (rest[m] != gslot) m++;
        row_b[k + i] = (uint8_t)(3 - m);
      }
      for (int lane = 0; lane < 32; lane++) {
        const int u0 = lane >> 4, v4 = lane & 15;
        uint32_t packed = 0;
        for (int t4 = 0; t4 < 4; t4++) {
          int c = 0;
          c |= ((t4 >> 1) & 1) << cb[o[0]];
          c |= (t4 & 1) << cb[o[1]];
          c |= u0 << cb[o[2]];
          for (int m = 0; m < 4; m++) c |= ((v4 >> (3 - m)) & 1) << cb[rest[m]];
          packed |= (uint32_t)c << (8 * t4);
        }
        src7[nj][lane] = packed;
      }
      first_k[nj] = (uint8_t)k;
      nrows[nj] = (uint8_t)rows;
      nj++;
      k += rows;
    }
    if (nj != 25) {
      delete host_tab;
      return fail(h, SBG_ERR_STATE, "internal: %d outer triples (expected 25)", nj);
    }
    memcpy(host_tab->src7, src7, sizeof(src7));
    // the chain's other 10 outer triples (positions 2..6), in src7's layout
    for (int j = 0; j < 10; j++) {
      const int *o = h_rows7c[6 * (25 + j)];
      for (int lane = 0; lane < 32; lane++) {
        const int u0 = lane >> 4, v4 = lane & 15;
        uint32_t packed = 0;
        for (int t4 = 0; t4 < 4; t4++) {
          int c = 0;
          c |= ((t4 >> 1) & 1) << cb[o[0]];
          c |= (t4 & 1) << cb[o[1]];
          c |= u0 << cb[o[2]];
          for (int m = 0; m < 4; m++) c |= ((v4 >> (3 - m)) & 1) << cb[o[3 + m]];
          packed |= (uint32_t)c << (8 * t4);
        }
        host_tab->src7x[j][lane] = packed;
      }
    }
    // minpos3 entries by number of unconstrained bits (k_begin)
    {
      int fill = 0;
      for (int level = 0; level <= 8; level++) {
        host_tab->m3_level[level] = fill;
        for (int e = 0; e < kMinpos3; e++) {
          int rest = e, nfree = 0, low = -1, step = 1, low_step = 0;
          uint32_t forced = 0;
          for (int j = 0; j < 8; j++) {
            const int d = rest % 3;
            rest /= 3;
            if (d == 0) {
              nfree++;
              if (low < 0) {
                low = j;
                low_step = step;
              }
            }
            if (d == 2) forced |= 1u << j;
            step *= 3;
          }
          if (nfree != level) continue;
          host_tab->m3_info[fill++] = (uint32_t)e | ((level == 0 ? forced : (uint32_t)low_step) << 16);
        }
      }
      host_tab->m3_level[9] = fill;
    }
    if ((rc = h->d_tab.grow(h, h->lane[0].stream, 1)) != SBG_OK) return rc;
    SBG_CUDA(h, cudaMemcpy(h->d_tab.p, host_tab, sizeof(DevTables), cudaMemcpyHostToDevice));
    delete host_tab;
    SBG_CUDA(h, cudaMemcpyToSymbol(c_j_first_k, first_k, sizeof(first_k)));
    SBG_CUDA(h, cudaMemcpyToSymbol(c_j_rows, nrows, sizeof(nrows)));
    SBG_CUDA(h, cudaMemcpyToSymbol(c_row_b, row_b, sizeof(row_b)));
    uint8_t rows5[10][5], rows7[70][7];
    for (int k = 0; k < 10; k++) for (int i = 0; i < 5; i++) rows5[k][i] = (uint8_t)h_rows5[k][i];
    for (int k = 0; k < 70; k++) for (int i = 0; i < 7; i++) rows7[k][i] = (uint8_t)h_rows7[k][i];
    SBG_CUDA(h, cudaMemcpyToSymbol(c_rows5, rows5, sizeof(rows5)));
    SBG_CUDA(h, cudaMemcpyToSymbol(c_rows7, rows7, sizeof(rows7)));
    uint8_t rows7c[210][7];
    for (int k = 0; k < 210; k++) for (int i = 0; i < 7; i++) rows7c[k][i] = (uint8_t)h_rows7c[k][i];
    SBG_CUDA(h, cudaMemcpyToSymbol(c_rows7c, rows7c, sizeof(rows7c)));
    uint8_t rows4s[12][5];
    for (int k = 0; k < 12; k++) for (int i = 0; i < 5; i++) rows4s[k][i] = (uint8_t)h_rows4s[k][i];
    SBG_CUDA(h, cudaMemcpyToSymbol(c_rows4s, rows4s, sizeof(rows4s)));
  }

  if ((rc = h->d_slots.grow(h, h->lane[0].stream, kSlots)) != SBG_OK) return rc;
  h->slots = new sbg_handle::HostProblem[kSlots];
  for (int i = 0; i < kSlots; i++) {
    SBG_CUDA(h, cudaEventCreateWithFlags(&h->slots[i].uploaded, cudaEventDisableTiming));
  }
  SBG_CUDA(h, cudaMallocHost(&h->h_stage, (size_t)SBG_MAX_GATES * 32));
  SBG_CUDA(h, cudaStreamSynchronize(h->lane[0].stream));
  return SBG_OK;
}

void sbg_destroy(sbg_handle *h) {
  if (h == nullptr) return;
  const bool bound = h->sm_count != 0;   // a device was bound: release whatever was created
  if (bound) {
    cudaSetDevice(h->device);
    cudaDeviceSynchronize();
    for (int i = 0; i < kLanes; i++) {
      sbg_lane &L = h->lane[i];
      if (L.h_out != nullptr) cudaFreeHost(L.h_out);
      if (L.h_ctl != nullptr) cudaFreeHost(L.h_ctl);
      for (int k = 0; k < 8; k++) if (L.ev[k] != nullptr) cudaEventDestroy(L.ev[k]);
      if (L.ev_done != nullptr) cudaEventDestroy(L.ev_done);
      if (L.ev_begun != nullptr) cudaEventDestroy(L.ev_begun);
      if (L.own_stream != nullptr) cudaStreamDestroy(L.own_stream);
    }
    if (h->h_stage != nullptr) cudaFreeHost(h->h_stage);
    if (h->slots != nullptr) {
      for (int i = 0; i < kSlots; i++) if (h->slots[i].uploaded != nullptr) cudaEventDestroy(h->slots[i].uploaded);
    }
  }
  delete[] h->slots;
  delete h;   // the handle's DevArrays free its device memory, on the device still current
  if (bound) (void)cudaGetLastError();
}

const char *sbg_last_error(const sbg_handle *h) { return h != nullptr ? h->err : "null handle"; }

int sbg_set_stream(sbg_handle *h, void *cuda_stream) {
  if (h == nullptr) return SBG_ERR_ARG;
  // work already enqueued on the old stream (uploads, a draining chain) must not be overtaken
  SBG_CUDA(h, cudaSetDevice(h->device));
  SBG_CUDA(h, cudaStreamSynchronize(h->lane[0].stream));
  h->lane[0].stream = cuda_stream != nullptr ? (cudaStream_t)cuda_stream : h->lane[0].own_stream;
  return SBG_OK;
}

int sbg_set_timing(sbg_handle *h, int on) {
  if (h == nullptr) return SBG_ERR_ARG;
  h->timing = on != 0;
  return SBG_OK;
}

uint64_t sbg_launch_count(const sbg_handle *h) { return h != nullptr ? h->launches : 0; }

int sbg_host_seconds(const sbg_handle *h, double *out) {
  if (h == nullptr || out == nullptr) return SBG_ERR_ARG;
  out[0] = h->host_s[0];
  out[1] = h->host_s[1];
  out[2] = h->wait_s[0];
  out[3] = h->wait_s[1];
  out[4] = h->wait_s[2];
  return SBG_OK;
}

int sbg_transfer_stats(const sbg_handle *h, uint64_t *out) {
  if (h == nullptr || out == nullptr) return SBG_ERR_ARG;
  out[0] = h->h2d_bytes;
  out[1] = h->d2h_bytes;
  out[2] = h->uploads_full;
  out[3] = h->uploads_incremental;
  out[4] = h->uploads_skipped;
  return SBG_OK;
}

float sbg_last_kernel_ms(const sbg_handle *h, int which) {
  if (h == nullptr || which < 0 || which > 3) return 0.f;
  return h->last_ms[which];
}

int sbg_alu_peak(sbg_handle *h, double *warp_instr_per_s) {
  if (h == nullptr || warp_instr_per_s == nullptr) return SBG_ERR_ARG;
  h->api_seq++;   // ends the enumeration cursor
  SBG_CUDA(h, cudaSetDevice(h->device));
  const int blocks = h->sm_count * 8, threads = 256, iters = 2048;
  constexpr int CH = 8;
  sbg_lane &L = h->lane[0];
  const int rc = h->d_scratch.grow(h, L.stream, (uint64_t)blocks * threads);
  if (rc != SBG_OK) return rc;
  double best = 0.0;
  for (int rep = 0; rep < 4; rep++) {
    cudaEventRecord(L.ev[4], L.stream);
    k_lop3_peak<CH><<<blocks, threads, 0, L.stream>>>(h->d_scratch.p, iters, 12345u + rep);
    cudaEventRecord(L.ev[5], L.stream);
    SBG_CUDA(h, cudaStreamSynchronize(L.stream));
    const float ms = elapsed(L.ev[4], L.ev[5]);
    if (ms > 0.f) {
      const double instr = (double)blocks * threads / 32.0 * (double)iters * 8 * CH;
      best = std::max(best, instr / (ms * 1e-3));
    }
  }
  *warp_instr_per_s = best;
  return SBG_OK;
}

int sbg_use_problem(sbg_handle *h, int slot) {
  if (h == nullptr) return SBG_ERR_ARG;
  h->api_seq++;   // ends the enumeration cursor
  if (slot < 0 || slot >= kSlots) return fail(h, SBG_ERR_ARG, "slot %d out of range", slot);
  if (!h->slots[slot].ready) return fail(h, SBG_ERR_STATE, "slot %d holds no problem", slot);
  h->cur_slot = slot;
  h->problem_ready = true;
  drop_list(h);
  return SBG_OK;
}

int sbg_stage_problem(sbg_handle *h, int slot, const uint64_t *tables, int n,
    const uint64_t *target, const uint64_t *mask, const int8_t *inbits) {
  if (h == nullptr) return SBG_ERR_ARG;
  h->api_seq++;   // ends the enumeration cursor
  SBG_CUDA(h, cudaSetDevice(h->device));
  return stage_problem(h, slot, tables, n, target, mask, inbits, true);
}

int sbg_load_problem(sbg_handle *h, const uint64_t *tables, int n, const uint64_t *target,
    const uint64_t *mask, const int8_t *inbits) {
  if (h == nullptr) return SBG_ERR_ARG;
  h->api_seq++;   // ends the enumeration cursor
  SBG_CUDA(h, cudaSetDevice(h->device));
  // lazily: the difference to the resident state rides in the next chain's first kernel
  int rc = stage_problem(h, 0, tables, n, target, mask, inbits, false);
  if (rc != SBG_OK) return rc;
  return sbg_use_problem(h, 0);
}

int sbg_search5_part(sbg_handle *h, int part, int nparts, const uint8_t *func_order,
    uint64_t *key) {
  if (h == nullptr || key == nullptr) return SBG_ERR_ARG;
  h->api_seq++;   // ends the enumeration cursor
  if (!h->problem_ready) return fail(h, SBG_ERR_STATE, "no problem loaded");
  const sbg_handle::HostProblem &hp = cur(h);
  if (hp.n < 5) return fail(h, SBG_ERR_ARG, "search_5lut needs n >= 5 (lut.c:119)");
  if (nparts < 1 || part < 0 || part >= nparts) return fail(h, SBG_ERR_ARG, "bad part %d/%d", part, nparts);
  if (!valid_order(func_order)) return fail(h, SBG_ERR_ARG, "func_order is not a permutation");
  SBG_CUDA(h, cudaSetDevice(h->device));
  sbg_lane &L = h->lane[0];
  int rc;
  if ((rc = lane_uses_slot(h, L, h->cur_slot)) != SBG_OK) return rc;
  const bool two_first = search5_two_kernels(h, hp.n);
  bool two = two_first;
  CallInputs in;
  in.order5 = func_order;
  for (;;) {
    L.seq++;
    if ((rc = enqueue_begin(h, L, kBeginSearch5, in, 0)) != SBG_OK) return rc;
    // A part that falls back from the two-kernel form keeps the prefix deal: the chunk head deals
    // its items differently, and the other parts, which may not have overflowed, cut their shares
    // by the prefix deal.  With the head this part's share would overlap theirs and leave ranks out.
    // A whole search (one part) shares with nobody and keeps the head.
    if ((rc = enqueue_search5(h, L, part, nparts, two, !two_first || nparts == 1)) != SBG_OK) return rc;
    if ((rc = wait_stage(h, L, 1)) != SBG_OK) return rc;
    if (two && L.h_out->overflow[1] != 0) {
      two = false;   // more feasible tuples than the buffer holds: let the fused kernel do it
      continue;
    }
    break;
  }
  collect_times(h, L);
  h->last_ms[0] = L.ms[0];
  h->d2h_bytes += 48;
  h->swept5 = L.h_out->swept[1] + L.skipped5;
  h->feasible5 = L.h_out->feasible[1];
  *key = L.h_out->key[1];
  return SBG_OK;
}

int sbg_finish5(sbg_handle *h, uint64_t key, const uint8_t *func_order, sbg_result *res) {
  if (h == nullptr || res == nullptr || func_order == nullptr) return SBG_ERR_ARG;
  h->api_seq++;   // ends the enumeration cursor
  if (!h->problem_ready) return fail(h, SBG_ERR_STATE, "no problem loaded");
  return finish5_slot(h, cur(h), key, func_order, h->feasible5, h->swept5, res);
}

int sbg_search5(sbg_handle *h, const uint8_t *func_order, sbg_result *res) {
  uint64_t key = SBG_KEY_NONE;
  int rc = sbg_search5_part(h, 0, 1, func_order, &key);
  if (rc != SBG_OK) return rc;
  return sbg_finish5(h, key, func_order, res);
}

int sbg_filter7_part(sbg_handle *h, int part, int nparts, uint64_t *list, int *count) {
  if (h == nullptr || count == nullptr) return SBG_ERR_ARG;
  h->api_seq++;   // ends the enumeration cursor
  if (!h->problem_ready) return fail(h, SBG_ERR_STATE, "no problem loaded");
  if (cur(h).n < 7) return fail(h, SBG_ERR_ARG, "search_7lut needs n >= 7 (lut.c:259)");
  if (nparts < 1 || part < 0 || part >= nparts) return fail(h, SBG_ERR_ARG, "bad part %d/%d", part, nparts);
  SBG_CUDA(h, cudaSetDevice(h->device));
  sbg_lane &L = h->lane[0];
  int rc;
  if ((rc = lane_uses_slot(h, L, h->cur_slot)) != SBG_OK) return rc;
  uint32_t keep = 0;
  uint64_t swept = 0;
  drop_list(h);
  if ((rc = run_filter7(h, L, part, nparts, &keep, &swept)) != SBG_OK) return rc;
  for (int i = 0; i < 4; i++) h->last_ms[i] = L.ms[i];
  *count = (int)keep;
  if (list != nullptr && keep > 0) {
    SBG_CUDA(h, cudaMemcpyAsync(list, L.d_sorted.p, (size_t)keep * sizeof(uint64_t),
        cudaMemcpyDeviceToHost, L.stream));
    SBG_CUDA(h, cudaStreamSynchronize(L.stream));
    h->d2h_bytes += (uint64_t)keep * 8;
  }
  // The part's own ordered list stays on the device; when it is the whole space (nparts == 1) it
  // IS the list, and phase 2 may follow without sbg_set_list7().
  if (nparts == 1) {
    install_list(h, h->cur_slot, keep, swept);
  } else {
    record_part_list(h, h->cur_slot, keep, swept);
  }
  return SBG_OK;
}

int sbg_list7_device(sbg_handle *h, const uint64_t **list, int *count) {
  if (h == nullptr || list == nullptr || count == nullptr) return SBG_ERR_ARG;
  h->api_seq++;   // ends the enumeration cursor
  *list = h->lane[0].d_sorted.p;
  *count = list_is_current(h, true) ? (int)h->list7.count : 0;
  return SBG_OK;
}

// Merge of ascending runs that already sit in device memory (run r at runs + r * stride).
int sbg_set_list7_device(sbg_handle *h, const uint64_t *runs, uint64_t stride, const int *counts,
    int nruns) {
  if (h == nullptr || counts == nullptr || nruns < 0 || nruns > kMaxRuns) return SBG_ERR_ARG;
  h->api_seq++;   // ends the enumeration cursor
  SBG_CUDA(h, cudaSetDevice(h->device));
  sbg_lane &L = h->lane[0];
  int rc;
  if ((rc = ensure_hits(h, L, std::max(L.d_hits.cap, h->hits_cap_default))) != SBG_OK) return rc;
  RunCounts rcnt;
  memset(&rcnt, 0, sizeof(rcnt));
  uint64_t total = 0;
  for (int r = 0; r < nruns; r++) {
    if (counts[r] < 0 || (uint64_t)counts[r] > stride) return fail(h, SBG_ERR_ARG, "bad run %d", r);
    rcnt.n[r] = (uint32_t)counts[r];
    total += (uint64_t)counts[r];
  }
  if (total > 0 && runs == nullptr) return SBG_ERR_ARG;
  // the merged list's sweep on this device: the part's that this handle's own phase 1 left for the
  // current problem (what an all-gather of the parts' lists follows), else none
  const uint64_t swept = list_is_current(h, true) ? h->list7.swept : 0;
  const int grid = (int)std::max<uint64_t>(1, std::min<uint64_t>((total + 255) / 256,
      (uint64_t)h->sm_count * 8));
  const cudaError_t e = launch(h, k_merge_runs, grid, 256, 0, L.stream, false, runs,
      (unsigned long long)stride, rcnt, nruns, L.d_sorted.p, (unsigned int)SBG_LIST_CAP, L.d_ctl.p);
  if (e != cudaSuccess) return fail(h, SBG_ERR_CUDA, "k_merge_runs: %s", cudaGetErrorString(e));
  install_list(h, h->cur_slot, (uint32_t)std::min<uint64_t>(total, SBG_LIST_CAP), swept);
  return SBG_OK;
}

int sbg_set_list7(sbg_handle *h, const uint64_t *list, int count) {
  if (h == nullptr || count < 0 || (count > 0 && list == nullptr)) return SBG_ERR_ARG;
  h->api_seq++;   // ends the enumeration cursor
  SBG_CUDA(h, cudaSetDevice(h->device));
  sbg_lane &L = h->lane[0];
  int rc;
  if ((rc = ensure_hits(h, L, std::max(L.d_hits.cap, h->hits_cap_default))) != SBG_OK) return rc;
  if ((size_t)count > L.d_hits.cap) return fail(h, SBG_ERR_ARG, "list of %d entries too long", count);
  // the list must be a concatenation of ascending runs (what gathering the parts' ordered lists
  // gives); they are merged on the device
  int counts[kMaxRuns];
  int nruns = 0, start = 0;
  for (int i = 1; i <= count; i++) {
    if (i == count || list[i] <= list[i - 1]) {
      if (nruns == kMaxRuns) {
        return fail(h, SBG_ERR_ARG, "list is not a concatenation of at most %d ascending runs", kMaxRuns);
      }
      counts[nruns++] = i - start;
      start = i;
    }
  }
  if (count > 0) {
    SBG_CUDA(h, cudaMemcpyAsync(L.d_hits.p, list, (size_t)count * sizeof(uint64_t),
        cudaMemcpyHostToDevice, L.stream));
    h->h2d_bytes += (uint64_t)count * 8;
  }
  // k_merge_runs takes the runs at a common stride: spread them out inside d_aux
  uint64_t stride = 0;
  for (int r = 0; r < nruns; r++) stride = std::max<uint64_t>(stride, (uint64_t)counts[r]);
  if (nruns > 1) {
    if ((uint64_t)nruns * stride > L.d_hits.cap) {
      return fail(h, SBG_ERR_ARG, "list too long to stage (%d runs of up to %llu)", nruns,
          (unsigned long long)stride);
    }
    uint64_t off = 0;
    for (int r = 0; r < nruns; r++) {
      SBG_CUDA(h, cudaMemcpyAsync(L.d_aux.p + (uint64_t)r * stride, L.d_hits.p + off,
          (size_t)counts[r] * sizeof(uint64_t), cudaMemcpyDeviceToDevice, L.stream));
      off += (uint64_t)counts[r];
    }
    return sbg_set_list7_device(h, L.d_aux.p, stride, counts, nruns);
  }
  return sbg_set_list7_device(h, L.d_hits.p, stride, counts, nruns);
}

int sbg_allgather_merge7(sbg_handle *const *hs, int nh, int *total) {
  if (hs == nullptr || nh < 1 || nh > kMaxRuns || total == nullptr) return SBG_ERR_ARG;
  int counts[kMaxRuns];
  uint64_t stride = 1;
  *total = 0;
  for (int i = 0; i < nh; i++) {
    if (hs[i] == nullptr) return SBG_ERR_ARG;
    hs[i]->api_seq++;   // ends the enumeration cursor
    counts[i] = (int)hs[i]->list7.count;
    stride = std::max<uint64_t>(stride, (uint64_t)counts[i]);
    *total += counts[i];
  }
  *total = std::min(*total, SBG_LIST_CAP);
  // 1. every device pulls every part's list into its staging area (d_aux); the lists are complete
  //    (sbg_filter7_part returns after its device finished)
  for (int d = 0; d < nh; d++) {
    sbg_handle *h = hs[d];
    sbg_lane &L = h->lane[0];
    SBG_CUDA(h, cudaSetDevice(h->device));
    int rc = ensure_hits(h, L, std::max<size_t>(std::max(L.d_hits.cap, h->hits_cap_default),
        (size_t)nh * stride));
    if (rc != SBG_OK) return rc;
    for (int s = 0; s < nh; s++) {
      if (counts[s] == 0) continue;
      if (hs[s]->device != h->device) {
        int can = 0;
        cudaDeviceCanAccessPeer(&can, h->device, hs[s]->device);
        if (can) {
          const cudaError_t e = cudaDeviceEnablePeerAccess(hs[s]->device, 0);
          if (e != cudaSuccess) (void)cudaGetLastError();   // already enabled
        }
      }
      SBG_CUDA(h, cudaMemcpyPeerAsync(L.d_aux.p + (uint64_t)s * stride, h->device,
          hs[s]->lane[0].d_sorted.p, hs[s]->device, (size_t)counts[s] * sizeof(uint64_t),
          L.stream));
    }
  }
  // 2. only when every copy has landed may a device overwrite its own list with the merged one
  for (int d = 0; d < nh; d++) {
    SBG_CUDA(hs[d], cudaSetDevice(hs[d]->device));
    SBG_CUDA(hs[d], cudaStreamSynchronize(hs[d]->lane[0].stream));
  }
  for (int d = 0; d < nh; d++) {
    int rc = sbg_set_list7_device(hs[d], hs[d]->lane[0].d_aux.p, stride, counts, nh);
    if (rc != SBG_OK) return rc;
  }
  return SBG_OK;
}

int sbg_decomp7_part(sbg_handle *h, int part, int nparts, const uint8_t *outer_order,
    const uint8_t *middle_order, uint64_t *key) {
  if (h == nullptr || key == nullptr) return SBG_ERR_ARG;
  h->api_seq++;   // ends the enumeration cursor
  if (!h->problem_ready) return fail(h, SBG_ERR_STATE, "no problem loaded");
  sbg_lane &L = h->lane[0];
  List7 &list = h->list7;
  if (!list_is_current(h, false)) {
    return fail(h, SBG_ERR_STATE, "no 7-LUT list installed for the current problem");
  }
  if (nparts < 1 || part < 0 || part >= nparts) return fail(h, SBG_ERR_ARG, "bad part %d/%d", part, nparts);
  if (!valid_order(outer_order) || !valid_order(middle_order)) {
    return fail(h, SBG_ERR_ARG, "function order is not a permutation");
  }
  SBG_CUDA(h, cudaSetDevice(h->device));
  int rc;
  *key = SBG_KEY_NONE;
  h->last_ms[3] = 0.f;
  if (list.count == 0) return SBG_OK;
  if ((rc = lane_uses_slot(h, L, h->cur_slot)) != SBG_OK) return rc;
  // k_decomp7 takes the list's length from the control words, which k_begin keeps here; but the
  // k_begin of a search_5lut or a 5-LUT enumeration since the list was installed has cleared them
  L.h_ctl->list_count = list.count;
  SBG_CUDA(h, cudaMemcpyAsync(&L.d_ctl.p->list_count, &L.h_ctl->list_count, sizeof(uint32_t),
      cudaMemcpyHostToDevice, L.stream));
  L.seq++;
  CallInputs in;
  in.outer = outer_order;
  in.middle = middle_order;
  if ((rc = enqueue_begin(h, L, kBeginSearch7 | kBeginKeepCtl, in, 0)) != SBG_OK) return rc;
  if (h->timing) cudaEventRecord(L.ev[2], L.stream);
  if ((rc = enqueue_decomp7(h, L, part, nparts, (list.count + nparts - 1) / nparts)) != SBG_OK) {
    return rc;
  }
  if ((rc = wait_stage(h, L, 2)) != SBG_OK) return rc;
  if (h->timing) h->last_ms[3] = L.ms[3] = elapsed(L.ev[2], L.ev[3]);
  h->d2h_bytes += 64;
  *key = L.h_out->key[2];
  list.last_tuple = L.h_out->tuple;
  list.last_tuple_prev = L.h_out->tuple_prev;
  list.last_key = *key;
  return SBG_OK;
}

int sbg_finish7(sbg_handle *h, uint64_t key, const uint8_t *outer_order,
    const uint8_t *middle_order, sbg_result *res) {
  if (h == nullptr || res == nullptr || outer_order == nullptr || middle_order == nullptr) {
    return SBG_ERR_ARG;
  }
  h->api_seq++;   // ends the enumeration cursor
  if (!h->problem_ready) return fail(h, SBG_ERR_STATE, "no problem loaded");
  sbg_lane &L = h->lane[0];
  if (!list_is_current(h, false)) {
    return fail(h, SBG_ERR_STATE, "no 7-LUT list installed for the current problem");
  }
  uint64_t pair[2] = {0, 0};
  if (key != SBG_KEY_NONE) {
    const uint64_t idx = key >> 23;
    if (idx >= h->list7.count) return fail(h, SBG_ERR_STATE, "corrupt 7-LUT key");
    if (key == h->list7.last_key) {   // this device found it: the tuples came with the result
      pair[0] = h->list7.last_tuple_prev;
      pair[1] = h->list7.last_tuple;
    } else {                   // another part's key: read the two list entries
      SBG_CUDA(h, cudaSetDevice(h->device));
      const size_t first = idx > 0 ? idx - 1 : 0;
      uint64_t tmp[2] = {0, 0};
      SBG_CUDA(h, cudaMemcpyAsync(tmp, L.d_sorted.p + first, (idx > 0 ? 2 : 1) * sizeof(uint64_t),
          cudaMemcpyDeviceToHost, L.stream));
      SBG_CUDA(h, cudaStreamSynchronize(L.stream));
      pair[0] = idx > 0 ? tmp[0] : 0;
      pair[1] = idx > 0 ? tmp[1] : tmp[0];
    }
  }
  return finish7_slot(h, cur(h), key, outer_order, middle_order, pair[1], pair[0], h->list7.count,
      h->list7.swept, res);
}

// ---- one call per node / per batch of nodes -----------------------------------------------------

int sbg_search_node(sbg_handle *h, const sbg_job *job, sbg_node_result *res) {
  if (h == nullptr || job == nullptr || res == nullptr) return SBG_ERR_ARG;
  h->api_seq++;   // ends the enumeration cursor
  int rc;
  const double t0 = wall_now();
  if ((rc = check_job(h, job)) != SBG_OK) return rc;
  SBG_CUDA(h, cudaSetDevice(h->device));
  sbg_lane &L = h->lane[0];
  if ((rc = lane_uses_slot(h, L, job->slot)) != SBG_OK) return rc;
  h->cur_slot = job->slot;
  h->problem_ready = true;
  CallInputs in;
  in.order5 = job->order5;
  in.outer = job->outer7;
  in.middle = job->middle7;
  in.gate_order = job->gate_order;
  drop_list(h);
  if ((rc = enqueue_chain(h, L, job->flags, in)) != SBG_OK) return rc;
  const double t1 = wall_now();
  if ((rc = collect_chain(h, L, job, res)) != SBG_OK) return rc;
  h->host_s[0] += t1 - t0;
  h->host_s[1] += wall_now() - t1;
  if (h->timing) {
    // timing events sit behind the whole chain: wait for it (the timed mode is for measurements)
    SBG_CUDA(h, cudaStreamSynchronize(L.stream));
    collect_times(h, L);
    for (int i = 0; i < 4; i++) h->last_ms[i] = L.ms[i];
  }
  return SBG_OK;
}

int sbg_search_batch(sbg_handle *h, int njobs, const sbg_job *jobs, sbg_node_result *results) {
  if (h == nullptr || njobs < 0 || (njobs > 0 && (jobs == nullptr || results == nullptr))) {
    return SBG_ERR_ARG;
  }
  h->api_seq++;   // ends the enumeration cursor
  int rc;
  for (int j = 0; j < njobs; j++) {
    if ((rc = check_job(h, &jobs[j])) != SBG_OK) return rc;
  }
  SBG_CUDA(h, cudaSetDevice(h->device));
  for (int i = 0; i < 4; i++) h->last_ms[i] = 0.f;
  // fork: the lanes' chains start after whatever the caller's stream (lane 0) holds so far --
  // staged problems, the caller's own events -- and the caller's stream continues after them
  cudaStream_t main_stream = h->lane[0].stream;
  for (int base = 0; base < njobs; base += kLanes) {
    const int wave = std::min(kLanes, njobs - base);
    h->concurrent = wave > 1;
    if (wave > 1) SBG_CUDA(h, cudaEventRecord(h->lane[0].ev_done, main_stream));
    for (int k = 0; k < wave; k++) {
      sbg_lane &L = h->lane[k];
      const sbg_job &job = jobs[base + k];
      if (k > 0) SBG_CUDA(h, cudaStreamWaitEvent(L.stream, h->lane[0].ev_done, 0));
      // A slot on several lanes: the first lane's k_begin applies the slot's pending change, and the
      // first with search_7lut builds its rows; the later lanes skip that work and would read the
      // problem block while it is being written.  Each starts after the last such k_begin of an
      // earlier lane (which itself started after the one before).  Distinct slots wait on nothing.
      for (int j = k - 1; j >= 0; j--) {
        if (jobs[base + j].slot == job.slot && h->lane[j].prepared) {
          SBG_CUDA(h, cudaStreamWaitEvent(L.stream, h->lane[j].ev_begun, 0));
          break;
        }
      }
      L.mark_begun = false;
      for (int j = k + 1; j < wave; j++) L.mark_begun |= jobs[base + j].slot == job.slot;
      L.slot = job.slot;
      h->slots[job.slot].busy_lane = k;
      CallInputs in;
      in.order5 = job.order5;
      in.outer = job.outer7;
      in.middle = job.middle7;
      in.gate_order = job.gate_order;
      if (k == 0) drop_list(h);
      rc = enqueue_chain(h, L, job.flags, in);
      L.mark_begun = false;
      if (rc != SBG_OK) {
        h->concurrent = false;
        return rc;
      }
    }
    h->concurrent = false;
    for (int k = 0; k < wave; k++) {
      sbg_lane &L = h->lane[k];
      if ((rc = collect_chain(h, L, &jobs[base + k], &results[base + k])) != SBG_OK) return rc;
    }
    // join: the caller's stream waits for every lane's chain (including chains still draining)
    for (int k = 1; k < wave; k++) {
      SBG_CUDA(h, cudaStreamWaitEvent(main_stream, h->lane[k].ev_done, 0));
    }
    if (h->timing) {
      for (int k = 0; k < wave; k++) {
        sbg_lane &L = h->lane[k];
        SBG_CUDA(h, cudaStreamSynchronize(L.stream));
        collect_times(h, L);
        for (int i = 0; i < 4; i++) h->last_ms[i] += L.ms[i];
      }
    }
  }
  return SBG_OK;
}

// Whole search_7lut on one device: one launch chain, no host synchronisation inside, the result
// read from mapped memory.
int sbg_search7(sbg_handle *h, const uint8_t *outer_order, const uint8_t *middle_order,
    sbg_result *res) {
  if (h == nullptr || res == nullptr) return SBG_ERR_ARG;
  h->api_seq++;   // ends the enumeration cursor
  if (!h->problem_ready) return fail(h, SBG_ERR_STATE, "no problem loaded");
  if (cur(h).n < 7) return fail(h, SBG_ERR_ARG, "search_7lut needs n >= 7 (lut.c:259)");
  sbg_job job;
  memset(&job, 0, sizeof(job));
  job.slot = h->cur_slot;
  job.flags = SBG_DO_SEARCH7;
  job.outer7 = outer_order;
  job.middle7 = middle_order;
  sbg_node_result nr;
  int rc = sbg_search_node(h, &job, &nr);
  if (rc != SBG_OK) return rc;
  *res = nr.r7;
  return SBG_OK;
}

int sbg_enum5(sbg_handle *h, int part, int nparts, const uint8_t *func_order, uint64_t max_matches,
    sbg_match *out, uint64_t *n_out, uint64_t *total, uint64_t *feasible) {
  int rc;
  if ((rc = check_enum_args(h, part, nparts, max_matches, out, n_out)) != SBG_OK) return rc;
  if (cur(h).n < 5) return fail(h, SBG_ERR_ARG, "search_5lut needs n >= 5 (lut.c:119)");
  if (!valid_order(func_order)) return fail(h, SBG_ERR_ARG, "func_order is not a permutation");
  CallInputs in;
  in.order5 = func_order;
  EnumInputs in5;
  memcpy(in5.ord.order[0], func_order, 256);
  memset(in5.ord.order[1], 0, 256);
  in5.source = kSrcList;
  if ((rc = take_filter(h, 5, in5)) != SBG_OK) return rc;
  return run_enum<5>(h, kBeginSearch5, in, in5, part, nparts, max_matches, out, n_out, total,
      feasible);
}

int sbg_enum7(sbg_handle *h, int part, int nparts, const uint8_t *outer_order,
    const uint8_t *middle_order, uint64_t max_matches, sbg_match *out, uint64_t *n_out,
    uint64_t *total, uint64_t *feasible) {
  int rc;
  if ((rc = check_enum_args(h, part, nparts, max_matches, out, n_out)) != SBG_OK) return rc;
  if (cur(h).n < 7) return fail(h, SBG_ERR_ARG, "search_7lut needs n >= 7 (lut.c:259)");
  if (!valid_order(outer_order) || !valid_order(middle_order)) {
    return fail(h, SBG_ERR_ARG, "function order is not a permutation");
  }
  EnumInputs in7;
  memcpy(in7.ord.order[0], outer_order, 256);
  memcpy(in7.ord.order[1], middle_order, 256);
  in7.source = kSrcList;
  if ((rc = take_filter(h, 7, in7)) != SBG_OK) return rc;
  // the installed list: only bring the problem block up to date
  return run_enum<7>(h, kBeginKeepCtl, CallInputs(), in7, part, nparts, max_matches, out, n_out,
      total, feasible);
}

int sbg_enum7_all(sbg_handle *h, int part, int nparts, const uint8_t *outer_order,
    const uint8_t *middle_order, uint64_t max_matches, sbg_match *out, uint64_t *n_out,
    uint64_t *total, uint64_t *feasible) {
  int rc;
  if ((rc = check_enum_args(h, part, nparts, max_matches, out, n_out)) != SBG_OK) return rc;
  const int n = cur(h).n;
  if (n < 7 || n > SBG_ENUM7_ALL_MAX_GATES) {
    return fail(h, SBG_ERR_ARG, "the whole-space 7-LUT enumeration needs 7 <= n <= %d, not %d",
        SBG_ENUM7_ALL_MAX_GATES, n);
  }
  if (!valid_order(outer_order) || !valid_order(middle_order)) {
    return fail(h, SBG_ERR_ARG, "function order is not a permutation");
  }
  EnumInputs in7;
  memcpy(in7.ord.order[0], outer_order, 256);
  memcpy(in7.ord.order[1], middle_order, 256);
  in7.source = kSrcWhole;
  if ((rc = take_filter(h, 7, in7)) != SBG_OK) return rc;
  // no list: only bring the problem block up to date, so an installed list and its control words
  // stay as they are
  return run_enum<7>(h, kBeginKeepCtl, CallInputs(), in7, part, nparts, max_matches, out, n_out,
      total, feasible);
}

int sbg_enum7_chain(sbg_handle *h, int part, int nparts, const uint8_t *outer_order,
    const uint8_t *middle_order, uint64_t max_matches, sbg_match *out, uint64_t *n_out,
    uint64_t *total, uint64_t *feasible) {
  int rc;
  if ((rc = check_enum_args(h, part, nparts, max_matches, out, n_out)) != SBG_OK) return rc;
  const int n = cur(h).n;
  if (n < 7 || n > SBG_ENUM7_ALL_MAX_GATES) {
    return fail(h, SBG_ERR_ARG, "the 7-LUT chain enumeration needs 7 <= n <= %d, not %d",
        SBG_ENUM7_ALL_MAX_GATES, n);
  }
  if (!valid_order(outer_order) || !valid_order(middle_order)) {
    return fail(h, SBG_ERR_ARG, "function order is not a permutation");
  }
  EnumInputs in7;
  memcpy(in7.ord.order[0], outer_order, 256);
  memcpy(in7.ord.order[1], middle_order, 256);
  in7.source = kSrcWhole;
  in7.shape = kShapeChain;
  if ((rc = take_filter(h, 7, in7)) != SBG_OK) return rc;
  // as sbg_enum7_all: no list is built or touched
  return run_enum<7>(h, kBeginKeepCtl, CallInputs(), in7, part, nparts, max_matches, out, n_out,
      total, feasible);
}

// The first chain match over the list: run_enum's count-free first K with K = 1 (windows of list
// entries that double until a match is known), then the record turned into an sbg_result.
int sbg_search7_chain(sbg_handle *h, const uint8_t *outer_order, const uint8_t *middle_order,
    sbg_result *res) {
  if (h == nullptr || res == nullptr) return SBG_ERR_ARG;
  h->api_seq++;   // ends the enumeration cursor
  if (!h->problem_ready) return fail(h, SBG_ERR_STATE, "no problem loaded");
  if (cur(h).n < 7) return fail(h, SBG_ERR_ARG, "the 7-LUT chain needs n >= 7");
  if (!valid_order(outer_order) || !valid_order(middle_order)) {
    return fail(h, SBG_ERR_ARG, "function order is not a permutation");
  }
  EnumInputs in7;
  memcpy(in7.ord.order[0], outer_order, 256);
  memcpy(in7.ord.order[1], middle_order, 256);
  in7.form = kFormPlain;   // the depth, function and grouping settings are not read
  in7.source = kSrcList;
  in7.shape = kShapeChain;
  memset(&in7.filter, 0, sizeof(in7.filter));
  sbg_match m;
  uint64_t found = 0;
  // the installed list, else phase 1 runs and installs it (as for sbg_enum7)
  int rc = run_enum<7>(h, kBeginKeepCtl, CallInputs(), in7, 0, 1, 1, &m, &found, nullptr, nullptr);
  if (rc != SBG_OK) return rc;
  memset(res, 0, sizeof(*res));
  res->key = SBG_KEY_NONE;
  res->tuples_feasible = h->list7.count;
  res->tuples_swept = h->list7.swept;
  if (found == 0) return SBG_OK;
  res->found = 1;
  res->key = m.key;
  res->index = m.key >> 24;
  res->ordering = (int)((m.key >> 16) & 0xff);
  res->pos_outer = (int)((m.key >> 8) & 0xff);
  res->pos_middle = (int)(m.key & 0xff);
  res->func_outer = m.func_outer;
  res->func_middle = m.func_middle;
  for (int i = 0; i < 7; i++) res->gates[i] = m.gates[i];
  // L3's solved bits from the host's tables, as finish7_slot does for the tree
  const sbg_handle::HostProblem &hp = cur(h);
  uint64_t x1[4], x2[4];
  sbg_lut_table(m.func_outer, hp.tables[m.gates[0]], hp.tables[m.gates[1]], hp.tables[m.gates[2]],
      x1);
  sbg_lut_table(m.func_middle, x1, hp.tables[m.gates[3]], hp.tables[m.gates[4]], x2);
  if (!sbg_solve_inner(x2, hp.tables[m.gates[5]], hp.tables[m.gates[6]], hp.target, hp.mask,
      &res->func_inner, &res->inner_seen) || res->func_inner != m.func_inner
      || res->inner_seen != m.inner_seen) {
    return fail(h, SBG_ERR_STATE, "internal: the first chain match does not decompose");
  }
  return SBG_OK;
}

// The shared-input two-LUT enumeration's inputs: the 5-LUT function order, no middle order.
int shared_inputs(sbg_handle *h, const uint8_t *func_order, EnumInputs &in4) {
  if (cur(h).n < 4) return fail(h, SBG_ERR_ARG, "the shared-input two-LUT circuits need n >= 4");
  if (!valid_order(func_order)) return fail(h, SBG_ERR_ARG, "func_order is not a permutation");
  memcpy(in4.ord.order[0], func_order, 256);
  memset(in4.ord.order[1], 0, 256);
  in4.source = kSrcList;
  in4.shape = kShapeShared;
  return SBG_OK;
}

int sbg_enum4_shared(sbg_handle *h, int part, int nparts, const uint8_t *func_order,
    uint64_t max_matches, sbg_match *out, uint64_t *n_out, uint64_t *total, uint64_t *feasible) {
  int rc;
  if ((rc = check_enum_args(h, part, nparts, max_matches, out, n_out)) != SBG_OK) return rc;
  EnumInputs in4;
  if ((rc = shared_inputs(h, func_order, in4)) != SBG_OK) return rc;
  if ((rc = take_filter(h, 4, in4)) != SBG_OK) return rc;
  // only bring the problem block up to date: an installed 7-LUT list and its control words stay
  return run_enum<4>(h, kBeginKeepCtl, CallInputs(), in4, part, nparts, max_matches, out, n_out,
      total, feasible);
}

// The first shared-input match: run_enum's count-free first K with K = 1 (windows of 3-gate
// prefixes that double until a match is known), then the record turned into an sbg_result.
int sbg_search4_shared(sbg_handle *h, const uint8_t *func_order, sbg_result *res) {
  if (h == nullptr || res == nullptr) return SBG_ERR_ARG;
  h->api_seq++;   // ends the enumeration cursor
  if (!h->problem_ready) return fail(h, SBG_ERR_STATE, "no problem loaded");
  EnumInputs in4;
  int rc;
  if ((rc = shared_inputs(h, func_order, in4)) != SBG_OK) return rc;
  in4.form = kFormPlain;   // the depth, function and grouping settings are not read
  memset(&in4.filter, 0, sizeof(in4.filter));
  sbg_match m;
  uint64_t found = 0, feasible = 0, prefixes = 0;
  rc = run_enum<4>(h, kBeginKeepCtl, CallInputs(), in4, 0, 1, 1, &m, &found, nullptr, &feasible,
      &prefixes);
  if (rc != SBG_OK) return rc;
  const sbg_handle::HostProblem &hp = cur(h);
  const int n = hp.n;
  memset(res, 0, sizeof(*res));
  res->key = SBG_KEY_NONE;
  res->tuples_feasible = feasible;
  // the 4-combinations of the prefixes swept: those ranked below the first one of prefix
  // `prefixes` (the prefixes are the 3-combinations of 0..n-2 in lexicographic order)
  res->tuples_swept = h_binom[n][4];
  if (prefixes < h_binom[n - 1][3]) {
    uint16_t pre[3];
    unrank_combination(prefixes, n - 1, 3, pre);
    uint64_t rank = 0;
    int x = 0;
    for (int pos = 0; pos < 3; pos++) {
      for (; x < pre[pos]; x++) rank += h_binom[n - x - 1][3 - pos];
      x++;
    }
    res->tuples_swept = rank;
  }
  if (found == 0) return SBG_OK;
  res->found = 1;
  res->key = m.key;
  res->index = m.key >> 12;
  res->ordering = (int)((m.key >> 8) & 0xf);
  res->pos_outer = (int)(m.key & 0xff);
  res->func_outer = m.func_outer;
  for (int i = 0; i < 5; i++) res->gates[i] = m.gates[i];
  // L2's solved bits from the host's tables, as finish5 does for search_5lut
  uint64_t x1[4];
  sbg_lut_table(m.func_outer, hp.tables[m.gates[0]], hp.tables[m.gates[1]], hp.tables[m.gates[2]],
      x1);
  if (!sbg_solve_inner(x1, hp.tables[m.gates[3]], hp.tables[m.gates[4]], hp.target, hp.mask,
      &res->func_inner, &res->inner_seen) || res->func_inner != m.func_inner
      || res->inner_seen != m.inner_seen) {
    return fail(h, SBG_ERR_STATE, "internal: the first shared-input match does not decompose");
  }
  return SBG_OK;
}

int sbg_enum3(sbg_handle *h, int part, int nparts, const uint16_t *gate_order,
    uint64_t max_matches, sbg_match *out, uint64_t *n_out, uint64_t *total, uint64_t *feasible) {
  int rc;
  if ((rc = check_enum_args(h, part, nparts, max_matches, out, n_out)) != SBG_OK) return rc;
  const int n = cur(h).n;
  if (n < 3) return fail(h, SBG_ERR_ARG, "the 3-LUT enumeration needs n >= 3 gates");
  if (gate_order == nullptr) return fail(h, SBG_ERR_ARG, "no gate order");
  // unlike the scan of sbg_search_node, which takes the order as given, the enumeration checks it
  bool seen[SBG_MAX_GATES] = {};
  for (int i = 0; i < n; i++) {
    if (gate_order[i] >= n || seen[gate_order[i]]) {
      return fail(h, SBG_ERR_ARG, "gate_order is not a permutation of 0..%d", n - 1);
    }
    seen[gate_order[i]] = true;
  }
  EnumInputs in3;
  memset(&in3, 0, sizeof(in3));
  memcpy(in3.gates.order, gate_order, sizeof(uint16_t) * (size_t)n);
  if ((rc = take_filter(h, 3, in3)) != SBG_OK) return rc;
  // only bring the problem block up to date: the control words of an installed 7-LUT list stay
  return run_enum<3>(h, kBeginKeepCtl, CallInputs(), in3, part, nparts, max_matches, out, n_out,
      total, feasible);
}

int sbg_enum_fetch(sbg_handle *h, uint64_t first, uint64_t count, sbg_match *out, uint64_t *n_out) {
  if (h == nullptr) return SBG_ERR_ARG;
  if (n_out == nullptr || (count > 0 && out == nullptr)) return fail(h, SBG_ERR_ARG, "null output");
  if (count > SBG_ENUM_MAX_MATCHES) {
    return fail(h, SBG_ERR_ARG, "count %llu above %u", (unsigned long long)count,
        SBG_ENUM_MAX_MATCHES);
  }
  int rc;
  if ((rc = check_cursor(h)) != SBG_OK) return rc;
  const EnumCursor &c = h->cursor;
  *n_out = 0;
  if (first >= c.total || count == 0) return SBG_OK;
  const uint64_t n = std::min(count, c.total - first);
  SBG_CUDA(h, cudaSetDevice(h->device));
  sbg_lane &L = h->lane[0];
  EnumBuffers &E = h->ebuf;
  if ((rc = E.d_pranks.grow(h, L.stream, 2)) != SBG_OK) return rc;
  if ((rc = E.d_ptickets.grow(h, L.stream, 2)) != SBG_OK) return rc;
  if ((rc = E.d_ematch.grow(h, L.stream, n)) != SBG_OK) return rc;
  // global ranks: the share writes the ranks it owns, zero records elsewhere
  if (c.global) SBG_CUDA(h, cudaMemsetAsync(E.d_ematch.p, 0, n * sizeof(sbg_match), L.stream));
  // the tickets of the window's first and last rank; the launch covers them and those between
  // (global: the range emit skips the tickets whose ranks lie outside the window)
  const unsigned long long ends[2] = {first, first + n - 1};
  unsigned long long tk[2] = {0, 0};
  SBG_CUDA(h, cudaMemcpyAsync(E.d_pranks.p, ends, sizeof(ends), cudaMemcpyHostToDevice, L.stream));
  if ((rc = locate_tickets(h, L, 2)) != SBG_OK) return rc;
  SBG_CUDA(h, cudaMemcpyAsync(tk, E.d_ptickets.p, sizeof(tk), cudaMemcpyDeviceToHost, L.stream));
  SBG_CUDA(h, cudaStreamSynchronize(L.stream));
  EnumSel sel;
  memset(&sel, 0, sizeof(sel));
  sel.lo = first;
  if (c.tickets > 0 && (rc = emit_sel<kEnumRange>(h, L, first + n, tk[0], tk[1] + 1, sel)) != SBG_OK) {
    return rc;
  }
  if ((rc = copy_matches(h, L, out, n)) != SBG_OK) return rc;
  *n_out = n;
  return SBG_OK;
}

int sbg_enum_pick(sbg_handle *h, const uint64_t *ranks, uint64_t nranks, sbg_match *out) {
  if (h == nullptr) return SBG_ERR_ARG;
  int rc;
  if ((rc = check_ranks(h, ranks, nranks, out)) != SBG_OK) return rc;
  if (nranks == 0) return SBG_OK;
  const EnumCursor &c = h->cursor;
  SBG_CUDA(h, cudaSetDevice(h->device));
  sbg_lane &L = h->lane[0];
  EnumBuffers &E = h->ebuf;
  if ((rc = E.d_ematch.grow(h, L.stream, nranks)) != SBG_OK) return rc;
  // global ranks: the share writes the ranks it owns, zero records elsewhere
  if (c.global) SBG_CUDA(h, cudaMemsetAsync(E.d_ematch.p, 0, nranks * sizeof(sbg_match), L.stream));
  RankSelection rs;
  if ((rc = select_ranks(h, L, ranks, nranks, rs)) != SBG_OK) return rc;
  if (rs.tickets > 0 && (rc = emit_sel<kEnumPick>(h, L, 0, 0, rs.tickets, rs.sel)) != SBG_OK) {
    return rc;
  }
  return copy_matches(h, L, out, nranks);
}

int sbg_enum_group_sizes(sbg_handle *h, const uint64_t *ranks, uint64_t nranks, uint64_t *sizes) {
  if (h == nullptr) return SBG_ERR_ARG;
  int rc;
  if ((rc = check_ranks(h, ranks, nranks, sizes)) != SBG_OK) return rc;
  if (nranks == 0) return SBG_OK;
  const EnumCursor &c = h->cursor;
  // ungrouped (or width 3, where every grouping is the identity): every group is one match
  const bool grouped = c.in.form == kFormGrouped;
  if (!grouped && !c.global) {
    std::fill(sizes, sizes + nranks, (uint64_t)1);
    return SBG_OK;
  }
  SBG_CUDA(h, cudaSetDevice(h->device));
  sbg_lane &L = h->lane[0];
  EnumBuffers &E = h->ebuf;
  RankSelection rs;
  if ((rc = select_ranks(h, L, ranks, nranks, rs)) != SBG_OK) return rc;
  if (!grouped) {
    // a global cursor: 1 at the ranks the share owns, 0 elsewhere
    std::fill(sizes, sizes + nranks, (uint64_t)0);
    for (const unsigned int s : rs.slots) sizes[s] = 1;
    return SBG_OK;
  }
  if ((rc = E.d_psizes.grow(h, L.stream, nranks)) != SBG_OK) return rc;
  // global ranks: the share writes the ranks it owns, zeros elsewhere
  SBG_CUDA(h, cudaMemsetAsync(E.d_psizes.p, 0, nranks * sizeof(unsigned long long), L.stream));
  if (rs.tickets > 0 && (rc = emit_sel<kEnumSizes>(h, L, 0, 0, rs.tickets, rs.sel)) != SBG_OK) {
    return rc;
  }
  SBG_CUDA(h, cudaMemcpyAsync(sizes, E.d_psizes.p, nranks * sizeof(uint64_t),
      cudaMemcpyDeviceToHost, L.stream));
  SBG_CUDA(h, cudaStreamSynchronize(L.stream));
  h->d2h_bytes += nranks * sizeof(uint64_t);
  return SBG_OK;
}

int sbg_enum_block_sums(sbg_handle *h, uint64_t *out, uint64_t *nblocks) {
  if (h == nullptr) return SBG_ERR_ARG;
  if (nblocks == nullptr) return fail(h, SBG_ERR_ARG, "null nblocks");
  int rc;
  if ((rc = check_cursor(h)) != SBG_OK) return rc;
  const EnumCursor &c = h->cursor;
  const uint64_t nb = c.tickets / enum_block_size(c.width, c.in.source);
  *nblocks = nb;
  if (out == nullptr || nb == 0) return SBG_OK;
  SBG_CUDA(h, cudaSetDevice(h->device));
  sbg_lane &L = h->lane[0];
  if ((rc = block_sums(h, L, nb)) != SBG_OK) return rc;
  SBG_CUDA(h, cudaMemcpyAsync(out, h->ebuf.d_bsums.p, nb * sizeof(uint64_t), cudaMemcpyDefault,
      L.stream));
  SBG_CUDA(h, cudaStreamSynchronize(L.stream));
  return SBG_OK;
}

int sbg_enum_set_global(sbg_handle *h, const uint64_t *sums, uint64_t stride,
    const uint64_t *counts, int nparts, uint64_t *total) {
  if (h == nullptr) return SBG_ERR_ARG;
  int rc;
  if ((rc = check_cursor(h)) != SBG_OK) return rc;
  EnumCursor &c = h->cursor;
  if (c.global) return fail(h, SBG_ERR_STATE, "the enumeration cursor is already global");
  if (total == nullptr || counts == nullptr) return fail(h, SBG_ERR_ARG, "null counts or total");
  if (nparts != c.nparts) {
    return fail(h, SBG_ERR_ARG, "nparts %d, but the cursor's share is part %d of %d", nparts,
        c.part, c.nparts);
  }
  uint64_t widest = 0;
  for (int q = 0; q < nparts; q++) {
    const uint64_t want = deal_share(c.blocks, q, nparts);
    if (counts[q] != want) {
      return fail(h, SBG_ERR_ARG, "counts[%d] = %llu, but part %d of %d holds %llu deal blocks", q,
          (unsigned long long)counts[q], q, nparts, (unsigned long long)want);
    }
    widest = std::max(widest, want);
  }
  if (stride < widest) {
    return fail(h, SBG_ERR_ARG, "stride %llu below the widest row (%llu blocks)",
        (unsigned long long)stride, (unsigned long long)widest);
  }
  if (sums == nullptr && widest > 0) return fail(h, SBG_ERR_ARG, "null sums");
  SBG_CUDA(h, cudaSetDevice(h->device));
  sbg_lane &L = h->lane[0];
  EnumBuffers &E = h->ebuf;
  const unsigned int B = enum_block_size(c.width, c.in.source);
  const uint64_t nb = c.tickets / B;
  uint64_t whole = 0;
  if (c.blocks > 0) {
    // the rows, packed at stride `widest` on the device
    if ((rc = E.d_gsums.grow(h, L.stream, (uint64_t)nparts * widest)) != SBG_OK) return rc;
    for (int q = 0; q < nparts; q++) {
      if (counts[q] == 0) continue;
      SBG_CUDA(h, cudaMemcpyAsync(E.d_gsums.p + (uint64_t)q * widest, sums + (uint64_t)q * stride,
          counts[q] * sizeof(uint64_t), cudaMemcpyDefault, L.stream));
    }
    if (nb > 0 && (rc = block_sums(h, L, nb)) != SBG_OK) return rc;
    cudaError_t e = launch(h, k_enum_globalize, 1, 1024, 0, L.stream, false, E.d_ectl.p,
        (const unsigned long long *)E.d_gsums.p, (unsigned long long)widest,
        (unsigned long long)c.blocks, c.part, nparts, (const unsigned long long *)E.d_bsums.p,
        (const unsigned long long *)E.d_eoffset.p, B, E.d_delta.p);
    if (e != cudaSuccess) return fail(h, SBG_ERR_CUDA, "k_enum_globalize: %s", cudaGetErrorString(e));
    EnumCtl ec;
    SBG_CUDA(h, cudaMemcpyAsync(&ec, E.d_ectl.p, sizeof(ec), cudaMemcpyDeviceToHost, L.stream));
    SBG_CUDA(h, cudaStreamSynchronize(L.stream));
    if (ec.gbad != 0) {
      return fail(h, SBG_ERR_ARG, "row %d of sums is not this share's block sums (rows gathered "
          "out of part order?)", c.part);
    }
    // only now, with the check passed: the local offsets become global
    if (nb > 0) {
      const int grid = (int)std::max<uint64_t>(1, std::min<uint64_t>((c.tickets + 255) / 256,
          (uint64_t)h->sm_count * 8));
      e = launch(h, k_enum_rebase, grid, 256, 0, L.stream, false, E.d_eoffset.p,
          (unsigned long long)c.tickets, B, (const unsigned long long *)E.d_delta.p);
      if (e != cudaSuccess) return fail(h, SBG_ERR_CUDA, "k_enum_rebase: %s", cudaGetErrorString(e));
      SBG_CUDA(h, cudaStreamSynchronize(L.stream));
    }
    whole = ec.gtotal;
  }
  c.global = true;
  c.total = whole;
  *total = whole;
  return SBG_OK;
}

int sbg_enum_set_depth(sbg_handle *h, const uint16_t *depth, int n, uint32_t max_depth) {
  if (h == nullptr) return SBG_ERR_ARG;
  h->api_seq++;   // ends the enumeration cursor
  if (depth == nullptr) {
    h->filter.on = false;
    return SBG_OK;
  }
  if (n < 1 || n > SBG_MAX_GATES) return fail(h, SBG_ERR_ARG, "n = %d outside 1..%d", n, SBG_MAX_GATES);
  for (int g = 0; g < n; g++) {
    if (depth[g] > SBG_MAX_DEPTH) {
      return fail(h, SBG_ERR_ARG, "depth[%d] = %u above %d", g, (unsigned)depth[g], SBG_MAX_DEPTH);
    }
  }
  DepthFilter &f = h->filter;
  memcpy(f.depth, depth, sizeof(uint16_t) * (size_t)n);
  f.n = n;
  f.max_depth = max_depth;
  f.on = true;
  return SBG_OK;
}

int sbg_enum_depth_counts(sbg_handle *h, uint64_t *out, uint32_t nbins) {
  if (h == nullptr) return SBG_ERR_ARG;
  if (nbins > SBG_DEPTH_BINS) return fail(h, SBG_ERR_ARG, "nbins %u above %d", nbins, SBG_DEPTH_BINS);
  if (out == nullptr && nbins > 0) return fail(h, SBG_ERR_ARG, "null output");
  int rc;
  if ((rc = check_cursor(h)) != SBG_OK) return rc;
  if (!h->cursor.in.filter.hist_on) {
    return fail(h, SBG_ERR_STATE, "the enumeration cursor was counted without a depth filter");
  }
  if (nbins == 0) return SBG_OK;
  SBG_CUDA(h, cudaSetDevice(h->device));
  sbg_lane &L = h->lane[0];
  SBG_CUDA(h, cudaMemcpyAsync(out, h->ebuf.d_ehist.p, nbins * sizeof(uint64_t),
      cudaMemcpyDeviceToHost, L.stream));
  SBG_CUDA(h, cudaStreamSynchronize(L.stream));
  h->d2h_bytes += nbins * sizeof(uint64_t);
  return SBG_OK;
}

int sbg_inner_table(const uint64_t *inner, uint8_t *out) {
  if (out == nullptr) return SBG_ERR_ARG;
  memset(out, 0, kMinpos3);
  int p3[256];
  for (int x = 0; x < 256; x++) {
    p3[x] = 0;
    for (int c = 7; c >= 0; c--) p3[x] = 3 * p3[x] + ((x >> c) & 1);
  }
  for (int f = 0; f < 256; f++) {
    if (inner != nullptr && ((inner[f >> 6] >> (f & 63)) & 1u) == 0) continue;
    for (int seen = 0; seen < 256; seen++) out[p3[seen] + p3[f & seen]] = 1;
  }
  return SBG_OK;
}

int sbg_enum_set_functions(sbg_handle *h, const uint64_t *outer, const uint64_t *middle,
    const uint64_t *inner) {
  if (h == nullptr) return SBG_ERR_ARG;
  h->api_seq++;   // ends the enumeration cursor
  FunctionFilter &f = h->functions;
  if (outer == nullptr && middle == nullptr && inner == nullptr) {
    f.on = false;
    return SBG_OK;
  }
  make_functions(outer, middle, inner, f);
  f.on = true;
  return SBG_OK;
}

int sbg_enum_set_grouping(sbg_handle *h, int grouping) {
  if (h == nullptr) return SBG_ERR_ARG;
  h->api_seq++;   // ends the enumeration cursor
  if (grouping != SBG_GROUP_NONE && grouping != SBG_GROUP_SHAPE && grouping != SBG_GROUP_TUPLE) {
    return fail(h, SBG_ERR_ARG, "grouping %d is none of SBG_GROUP_NONE, _SHAPE, _TUPLE", grouping);
  }
  h->grouping = grouping;
  return SBG_OK;
}

}  // extern "C"
