/* sboxgates_b200.h -- C ABI of the H100-native 3-LUT exhaustive search.
 *
 * This is the drop-in boundary for the `--lut` path of dansarie/sboxgates: plain pointers and
 * sizes, no torch / C++ / vector types.  Each entry point names the reference interface it
 * replaces (paths are relative to the reference checkout).
 *
 *   reference                                      here
 *   ---------------------------------------------  ----------------------------------------------
 *   search_5lut(st,target,mask,inbits,ret,v)       sbg_search5()         (lut.h:46-47, lut.c:116-249)
 *   search_7lut(st,target,mask,inbits,ret,v)       sbg_search7()         (lut.h:54-55, lut.c:256-487)
 *   MPI_Bcast(&work,...) of the search state       sbg_load_problem()    (lut.c:533-540,
 *                                                                         sboxgates.c:625-627)
 *   the per-rank slice of C(n,5) / C(n,7)          sbg_search5_part(), sbg_filter7_part()
 *                                                                        (lut.c:137-149, 265-277)
 *   MPI_Allgather(v) of the 7-LUT hit lists        sbg_set_list7()       (lut.c:329-349)
 *   the per-rank slice of the hit list             sbg_decomp7_part()    (lut.c:351-360, 416-484)
 *   get_search_result(): first finder wins         min over ranks of the 64-bit keys the *_part
 *                                                  calls return (one all-reduce(MIN) per phase),
 *                                                  then sbg_finish5()/sbg_finish7()  (lut.c:665-740)
 *
 * Semantics are those of the reference at MPI size == 1: the result is the FIRST match in the
 * reference's enumeration order (combination in lexicographic order, then ordering, then position
 * in the shuffled function order(s)), whatever the number of GPUs.  The shuffled function orders
 * are inputs because the caller owns the RNG (lut.c:125-135, 362-378 consume the host's
 * xorshift1024); likewise the random fill of don't-care LUT bits (lut.c:104-106) is left to the
 * caller: results carry the solved inner function and its `seen` mask.
 *
 * Truth tables are 4 x uint64_t per gate, gate-major: bit b of word v = value at S-box input
 * 64*v+b -- the memory image of the reference's `ttable` (state.h:64-68).
 *
 * All functions return SBG_OK (0) or a negative error code; sbg_last_error() gives the text.
 * A handle is bound to one CUDA device and is not thread-safe (the reference's functions are not
 * re-entrant either, lut.h / SURVEY.md section 8b).
 */
#ifndef SBOXGATES_B200_H
#define SBOXGATES_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SBG_OK 0
#define SBG_ERR_ARG (-1)       /* bad argument (n out of range, null pointer, ...) */
#define SBG_ERR_CUDA (-2)      /* a CUDA call failed; see sbg_last_error() */
#define SBG_ERR_OVERFLOW (-3)  /* hit buffer too small even for the serial retry */
#define SBG_ERR_STATE (-4)     /* call sequence error (e.g. no problem loaded) */

#define SBG_MAX_GATES 500      /* state.h:26 */
#define SBG_LIST_CAP 100000    /* lut.c:291,316-318: at most this many feasible 7-tuples are tried */
#define SBG_KEY_NONE UINT64_MAX
#define SBG_PROBLEM_SLOTS 64    /* device-resident search states per handle */
#define SBG_LANES 8             /* searches of one sbg_search_batch() call that run concurrently */

typedef struct sbg_handle sbg_handle;

/* What a search returns; the caller turns it into the reference's ret[10] (lut.c:202-211,
   453-462) after applying the random don't-care fill. */
typedef struct {
  int32_t found;
  int32_t ordering;        /* k: 0..9 (lut.c:189-229) or 0..69 (lut.c:396-415); sbg_search7_chain:
                              the chain row, 0..209 (sbg_chain_row); sbg_search4_shared: the
                              shared-input row, 0..11 (sbg_shared_row) */
  int32_t pos_outer;       /* position of func_outer in the shuffled order */
  int32_t pos_middle;      /* 7-LUT only */
  uint8_t func_outer;
  uint8_t func_middle;     /* 7-LUT only */
  uint8_t func_inner;      /* solved bits only; don't-care bits are 0 */
  uint8_t inner_seen;      /* bit c set = inner cell c occurs under the mask (0xff: no fill) */
  uint16_t gates[7];       /* LUT inputs in reference order: a,b,c,d,e[,f,g] */
  uint16_t stale_outer;    /* 7-LUT: 1 if the reference would have evaluated this row with its
                              stale outer cache (lut.c:432-435); func_inner then follows suit */
  uint64_t index;          /* 5-LUT: lexicographic rank of the combination; 7-LUT: list index */
  uint64_t key;            /* the packed minimum key (SBG_KEY_NONE if nothing matched) */
  uint64_t tuples_feasible;/* 5-LUT: feasible combinations met; 7-LUT: length of the hit list */
  uint64_t tuples_swept;   /* combinations put through the feasibility test by this device,
                              inbits rejections included: this part's share in a sharded search
                              (summed over the parts, the whole's).  5-LUT: C(n,5) on a miss, at
                              least index + 1 on a hit (a match stops the sweep).  7-LUT: the phase-1
                              sweep behind the installed list, C(n,7) for an uncapped list; one that
                              reached SBG_LIST_CAP stops between the reference's count (the last
                              entry's rank + 1) and C(n,7).  sbg_finish5 reports the last
                              sbg_search5_part's; sbg_finish7 the installed list's: that of the
                              sbg_filter7_part, sbg_search7 / node / batch or sbg_enum7 phase 1 that
                              built it, carried over by sbg_set_list7, sbg_set_list7_device and
                              sbg_allgather_merge7 from this handle's own list of the current
                              problem (0 where the handle held none) */
} sbg_result;

/* ---- lifecycle ------------------------------------------------------------------------------ */
int sbg_create(sbg_handle **out, int device);
void sbg_destroy(sbg_handle *h);
const char *sbg_last_error(const sbg_handle *h);
/* Run on an externally owned stream (a cudaStream_t, e.g. torch's current stream); NULL restores
   the handle's own stream. */
int sbg_set_stream(sbg_handle *h, void *cuda_stream);
/* Number of kernels the handle has launched so far (all of them this library's own; bench.py
   reports it). */
uint64_t sbg_launch_count(const sbg_handle *h);
/* Kernel timing is off by default (an event between two kernels of a chain forbids their
   overlap); sbg_set_timing(h, 1) or SBG_TIMING=1 turns it on.  sbg_last_kernel_ms() then gives the
   CUDA-event time (ms) of the named kernel family in the last call (summed over the searches of a
   batch): 0 = search5, 1 = filter7 (phase 1), 2 = ordering the hit list, 3 = decomp7. */
int sbg_set_timing(sbg_handle *h, int on);
float sbg_last_kernel_ms(const sbg_handle *h, int which);
/* Bytes this handle has shipped so far: out[0] = problem data host->device (gate tables that
   changed, target, mask; as kernel arguments or copies), out[1] = results device->host (mapped
   memory and copies), out[2..4] = state changes that took a bulk copy / travelled as kernel
   arguments / were no change at all. */
int sbg_transfer_stats(const sbg_handle *h, uint64_t *out /*5*/);
/* Host seconds sbg_search_node() has spent so far: out[0] = enqueueing the chains (launch calls),
   out[1] = waiting for and decoding their results; out[2..4] = the waiting alone, per stage
   (3-LUT scan, search_5lut, search_7lut; all calls of the handle). */
int sbg_host_seconds(const sbg_handle *h, double *out /*5*/);
/* Measures the device's LOP3 issue rate (warp instructions per second, whole chip): the ceiling
   the search kernels are bound by (SURVEY.md section 8d). */
int sbg_alu_peak(sbg_handle *h, double *warp_instr_per_s);

/* ---- problem -------------------------------------------------------------------------------- */
/* Makes one search state the current problem: n gate tables, target, mask, and the -1 terminated
   list of input-bit gates already used as multiplexer selectors (lut.c:177-185).  Host pointers.
   The gate tables stay resident on the device between calls (the replacement of the `state`
   array the reference re-broadcasts per call): only the gates that differ from the previous state
   of the slot are shipped -- a graph build only ever appends gates (state.h:87) or replaces a
   suffix when it backtracks -- together with target and mask, as arguments of the next search's
   first kernel; compression to the masked positions happens on the device. */
int sbg_load_problem(sbg_handle *h, const uint64_t *tables, int n, const uint64_t *target,
    const uint64_t *mask, const int8_t *inbits);
/* The same in two steps, for callers that keep several search states resident in HBM: stage a
   state into slot 0..SBG_PROBLEM_SLOTS-1 (upload), later make a staged slot the current problem
   (no transfer).  sbg_load_problem() = stage + use of slot 0.  This is the device-resident
   replacement of the `state` array the reference re-broadcasts per call (lut.c:533-540).
   A 7-LUT list belongs to the slot and the state it was built or installed for: staging a different
   state into that slot, the current one included, leaves the list to no problem (sbg_enum7 then
   runs phase 1 again, sbg_decomp7_part / sbg_finish7 return SBG_ERR_STATE); staging the state the
   slot already holds ships nothing and keeps the list.  sbg_use_problem drops the list. */
int sbg_stage_problem(sbg_handle *h, int slot, const uint64_t *tables, int n,
    const uint64_t *target, const uint64_t *mask, const int8_t *inbits);
int sbg_use_problem(sbg_handle *h, int slot);

/* ---- whole searches on one device (host buffers in, result out) ----------------------------- */
int sbg_search5(sbg_handle *h, const uint8_t *func_order /*256*/, sbg_result *res);
int sbg_search7(sbg_handle *h, const uint8_t *outer_order /*256*/, const uint8_t *middle_order
    /*256*/, sbg_result *res);
/* The first 7-LUT chain L3(L2(L1(a,b,c), d, e), f, g) (the wiring of sbg_enum7_chain, which
   search_7lut never tries) over the combinations search_7lut tries: the 7-LUT list of the current
   problem, taken as sbg_enum7 takes it (the installed list when it belongs to the current problem as
   staged now, else phase 1 runs here and its list stays installed), so the SBG_LIST_CAP cut applies
   and any n >= 7 works.  Candidates are those of sbg_enum7_chain: chain row k < 210, L1 =
   outer_order[po], L2 = middle_order[pm], L3 solvable without a random fill, decided on the true
   gate tables.  The result is the candidate with the smallest key idx << 24 | k << 16 | po << 8 | pm,
   idx being the list index; over an uncut list that is sbg_enum7_chain's first match with its rank
   replaced by the list index.  res: found, key, ordering = k, pos_outer = po, pos_middle = pm,
   func_outer = L1, func_middle = L2, func_inner / inner_seen = L3's solved bits and seen cells
   (cells x2<<2 | f<<1 | g), gates a..g in chain-row order, index = idx, stale_outer = 0,
   tuples_feasible = the list's length, tuples_swept = the installed list's sweep (as sbg_finish7
   reports it); nothing matched: found = 0, key = SBG_KEY_NONE.  The caller applies L3's random fill
   and adds L1, then L2 over (L1, d, e), then L3 over (L2, f, g).  The depth, function and grouping
   settings are not read.  The installed list and the current problem stay as they were, unless
   phase 1 had to run.  SBG_ERR_ARG: n < 7 or an order that is not a permutation; SBG_ERR_STATE: no
   problem loaded. */
int sbg_search7_chain(sbg_handle *h, const uint8_t *outer_order /*256*/,
    const uint8_t *middle_order /*256*/, sbg_result *res);
/* The first shared-input two-LUT circuit L2(L1(a,b,c), u, v), {u, v} = {s, d} with s one of a, b, c
   (the shape of sbg_enum4_shared, which search_5lut never tries: its five gates are distinct), over
   every 4-combination of the current problem, any n >= 4.  The result is sbg_enum4_shared's first
   match (smallest key rank << 12 | k << 8 | po).  res: found, key, ordering = the row k (0..11),
   pos_outer = po, func_outer = L1, func_inner / inner_seen = L2's solved bits and seen cells (cells
   x1<<2 | u<<1 | v), gates[0..4] = a, b, c, u, v (add_lut's argument order, as for a 5-LUT result),
   index = rank, tuples_feasible = the feasible 4-combinations met, tuples_swept = the
   4-combinations of the 3-gate prefixes swept, inbits rejections included (C(n,4) on a miss; the
   sweep stops in windows of prefixes once a match is known); nothing matched: found = 0, key =
   SBG_KEY_NONE.  The caller applies L2's random fill and adds L1, then L2 over (L1, u, v).  The
   depth, function and grouping settings are not read; the installed 7-LUT list stays as it was.
   SBG_ERR_ARG: n < 4 or an order that is not a permutation; SBG_ERR_STATE: no problem loaded. */
int sbg_search4_shared(sbg_handle *h, const uint8_t *func_order /*256*/, sbg_result *res);

/* ---- one call per node, batches of independent nodes ----------------------------------------- */
/* A job is what lut_search() does for one node (lut.c:489-631): the 3-LUT scan over the caller's
   shuffled gate order (lut.c:501-523), search_5lut (lut.c:553) and search_7lut (lut.c:593), each
   stage only if the earlier ones found nothing -- as ONE launch chain on the device, the stages
   predicated there, no host round trip in between.  The caller says which stages it wants
   (lut_search skips search_5lut / search_7lut when the gate budget forbids two / three more gates,
   lut.c:525-527, 582-586). */
#define SBG_DO_SCAN3 1
#define SBG_DO_SEARCH5 2
#define SBG_DO_SEARCH7 4
typedef struct {
  int32_t slot;                /* staged problem (sbg_stage_problem / sbg_load_problem = slot 0) */
  int32_t flags;               /* SBG_DO_* */
  const uint8_t *order5;       /* 256: shuffled function order of search_5lut (lut.c:125-135) */
  const uint8_t *outer7;       /* 256 + 256: the two orders of search_7lut (lut.c:362-378) */
  const uint8_t *middle7;
  const uint16_t *gate_order;  /* n: create_circuit's shuffled gate order (sboxgates.c:285-299) */
} sbg_job;
typedef struct {
  int32_t found_stage;         /* 0 nothing, else 3 / 5 / 7 */
  uint16_t gates3[3];          /* stage 3: LUT inputs in gate_order order (gi, gk, gm) */
  uint8_t func3, seen3;        /* solved function bits / cells seen under the mask (fill as below) */
  uint64_t key3;               /* the position triple in gate_order, i << 18 | k << 9 | m, or
                                  SBG_KEY_NONE */
  sbg_result r5;               /* as sbg_search5 (found = 0 if the stage did not run) */
  sbg_result r7;               /* as sbg_search7 */
} sbg_node_result;
/* One node; returns as soon as a stage has matched.  The job's slot becomes the current problem;
   the installed 7-LUT list is dropped, and when the search_7lut stage ran, its list is installed
   for that slot. */
int sbg_search_node(sbg_handle *h, const sbg_job *job, sbg_node_result *result);
/* Independent nodes (the first children of a create_circuit node, sboxgates.c:458-607; the output
   bits of generate_graph, sboxgates.c:701-788; the -i iterations): their chains run concurrently
   on up to SBG_LANES streams, results are read once per job.  Jobs may repeat a slot (lanes that
   share one are ordered where the slot's problem block is brought up to date).  The current
   problem does not change.  The installed 7-LUT list is dropped; the list of the first job of the
   last wave of SBG_LANES jobs is left installed for that job's slot when its search_7lut stage
   ran, so list consumers use it only when that slot is the current problem. */
int sbg_search_batch(sbg_handle *h, int njobs, const sbg_job *jobs, sbg_node_result *results);

/* ---- sharded building blocks (one process per GPU; part = rank, nparts = world size) -------- */
/* 5-LUT: this part's share of C(n,5); *key = local minimum key or SBG_KEY_NONE. */
int sbg_search5_part(sbg_handle *h, int part, int nparts, const uint8_t *func_order,
    uint64_t *key);
int sbg_finish5(sbg_handle *h, uint64_t key, const uint8_t *func_order, sbg_result *res);

/* 7-LUT phase 1: this part's share of C(n,7).  Writes this part's feasible combinations, sorted,
   at most SBG_LIST_CAP of them, as packed 63-bit words (9 bits per gate, first gate in the most
   significant position, so integer order = lexicographic order) to `list` (host memory, room for
   SBG_LIST_CAP entries) and their number to *count.  `list` may be NULL (no copy).  With
   nparts == 1 the device-resident result is installed as the list, so sbg_decomp7_part() may follow
   directly. */
int sbg_filter7_part(sbg_handle *h, int part, int nparts, uint64_t *list, int *count);
/* Installs the merged hit list: `list` is the concatenation of the parts' ascending lists (at most
   64 ascending runs, no duplicates); the runs are merged on the device and cut at SBG_LIST_CAP,
   which reproduces lut.c:316-349 for size == 1. */
int sbg_set_list7(sbg_handle *h, const uint64_t *list, int count);
/* The same without touching the host: this part's ordered list as a device pointer (valid until the
   next search on the handle; count 0 when the handle holds no list of the current problem as it is
   staged now), and the merge of `nruns` ascending runs that already sit in device
   memory, run r at runs + r * stride with counts[r] entries (what an all-gather of the parts'
   lists into one buffer gives). */
int sbg_list7_device(sbg_handle *h, const uint64_t **list, int *count);
int sbg_set_list7_device(sbg_handle *h, const uint64_t *runs, uint64_t stride, const int *counts,
    int nruns);
/* One process driving several devices (handles hs[0..nh-1], one per device, each holding its part's
   ordered list from sbg_filter7_part(part = i, nparts = nh)): gathers every part's list onto every
   device (peer copies over NVLink) and merges them there; afterwards every handle has the same
   installed list.  *total = its length.  The in-process counterpart of the all-gather
   (lut.c:329-349). */
int sbg_allgather_merge7(sbg_handle *const *hs, int nh, int *total);
/* 7-LUT phase 2 over list indices congruent to part modulo nparts.  sbg_finish7 decodes any part's
   key against the installed list; it reuses the entries sbg_decomp7_part returned with its key only
   while that list is still installed.  Both return SBG_ERR_STATE unless a list is installed for the
   current problem as it is staged now (see sbg_stage_problem, sbg_search_batch). */
int sbg_decomp7_part(sbg_handle *h, int part, int nparts, const uint8_t *outer_order,
    const uint8_t *middle_order, uint64_t *key);
int sbg_finish7(sbg_handle *h, uint64_t key, const uint8_t *outer_order,
    const uint8_t *middle_order, sbg_result *res);

/* ---- enumeration: every match, not only the first -------------------------------------------- */
/* The matches of search_5lut / search_7lut are the keys (as in sbg_result::key, so ascending key
   order is the reference's enumeration order) of the candidates that get_lut_function accepts
   without its random fill (lut.c:79-103), after the inbits rejection (lut.c:177-185) and
   check_n_lut_possible (lut.c:34-66):
     5-LUT: rank<<12 | k<<8 | pos over all combinations of C(n,5);
     7-LUT: idx<<23 | k<<16 | po<<8 | pm over the phase-1 list (the first SBG_LIST_CAP feasible
            7-combinations in lexicographic order), decided on the TRUE gate tables.  The reference's
            stale outer cache (lut.c:432-435, sbg_result::stale_outer) is not reproduced; it can only
            act on a list entry whose first gate is 0, so where inbits excludes gate 0 the smallest
            7-LUT match is the key sbg_search7 returns.
   One record per match, decoded on the device; nothing consumes the caller's RNG (the random fill
   of func_inner's don't-care bits stays with the caller, as for sbg_result).  32 bytes: */
typedef struct {
  uint64_t key;            /* offset 0 */
  uint16_t gates[7];       /* 8: LUT inputs in reference order a..c (3-LUT), a..e (5-LUT; then 0)
                              or a..g */
  uint8_t func_outer;      /* 22: the function at position (key >> 8) & 0xff of the outer order
                              (3-LUT: 0) */
  uint8_t func_middle;     /* 23: 7-LUT: the function at position key & 0xff of the middle order */
  uint8_t func_inner;      /* 24: solved bits only; don't-care bits are 0 (3-LUT: the LUT) */
  uint8_t inner_seen;      /* 25: bit c set = inner cell c occurs under the mask */
  uint8_t width;           /* 26: 3, 5 or 7; 4 for a shared-input circuit (sbg_enum4_shared) */
  uint8_t shape;           /* 27: how a 7-LUT match wires its LUTs, SBG_SHAPE_TREE (every call but
                              sbg_enum7_chain and sbg_enum4_shared, and widths 3 and 5),
                              SBG_SHAPE_CHAIN or SBG_SHAPE_SHARED */
  uint8_t pad[4];          /* 28: 0 */
} sbg_match;
#define SBG_SHAPE_TREE 0    /* L3(L1(a,b,c), L2(d,e,f), g): search_7lut's wiring */
#define SBG_SHAPE_CHAIN 1   /* L3(L2(L1(a,b,c), d, e), f, g) */
#define SBG_SHAPE_SHARED 2  /* L2(L1(a,b,c), u, v) over four gates, {u, v} = {s, d}, s in {a, b, c} */
#define SBG_ENUM_MAX_MATCHES (1u << 24)   /* largest max_matches of one call */

/* Enumerates the matches of the current problem in this part's share of the work (part/nparts as
   for sbg_search5_part / sbg_decomp7_part: the parts' totals add up to the whole, and merging their
   first-K lists and cutting at K gives the whole's first K).  Writes the first
   n = min(max_matches, matches) of them, in ascending key order, to out[0..n-1] and n to *n_out.
   total != NULL: *total = the exact number of matches of the share.  total == NULL: the sweep may
   stop as soon as the first max_matches matches are known (max_matches = 1: a first-match search).
   *feasible (may be NULL): 5-LUT: feasible combinations met (all of the share's when counting);
   7-LUT: the length of the list.  max_matches may be 0 (counting only), at most
   SBG_ENUM_MAX_MATCHES.  The match and count buffers are allocated on the first call. */
int sbg_enum5(sbg_handle *h, int part, int nparts, const uint8_t *func_order, uint64_t max_matches,
    sbg_match *out, uint64_t *n_out, uint64_t *total, uint64_t *feasible);
/* The 7-LUT list: the one installed for the current problem (sbg_set_list7 / sbg_set_list7_device /
   sbg_allgather_merge7, sbg_filter7_part with nparts == 1, or an earlier sbg_search7, sbg_search_node
   or sbg_search_batch of it, with the problem not staged anew since), else phase 1 runs here over
   the whole space and its list stays installed. */
int sbg_enum7(sbg_handle *h, int part, int nparts, const uint8_t *outer_order,
    const uint8_t *middle_order, uint64_t max_matches, sbg_match *out, uint64_t *n_out,
    uint64_t *total, uint64_t *feasible);
/* The matches sbg_enum7 would return if phase 1 had no list cap: every 7-combination of the current
   problem that has no gate excluded by inbits and passes check_n_lut_possible(7), decided on the
   true gate tables with the same ordering rows, orders and inner solve as sbg_enum7 (the stale
   outer cache is not reproduced either).  Key rank<<23 | k<<16 | po<<8 | pm, rank being the
   combination's lexicographic rank among all C(n,7) (as for the 5-LUT key and sbg_result::index;
   below 2^30 at n <= 64), so decode_key7 and the grouping key prefixes read it as they read a list
   index.  Records are byte-identical to the ones sbg_enum7 emits for the same combination, row and
   positions; only the key differs.  *feasible = the share's feasible 7-combinations (under a depth
   filter: those with an ordering within the bound, as for sbg_enum5) -- at width 7 the number the
   list cap hides.  part/nparts, max_matches, the count-free first K, the cursor (fetch, pick, group
   sizes, depth counts, global ranks) and the depth, function and grouping settings behave as for
   the other widths; a share's tickets are 6-gate prefixes dealt in blocks of 16.  The call builds
   no list: an installed 7-LUT list and what sbg_search7 / sbg_enum7 see of it stay as they were.
   The count buffers take 12 bytes per 6-gate prefix, C(n-1, 6) of them (815 MB at n = 64).
   SBG_ERR_ARG: n < 7, n > SBG_ENUM7_ALL_MAX_GATES, an order that is not a permutation, or a depth
   filter of another n; SBG_ERR_STATE: no problem loaded.  The call ends the cursor, whatever it
   returns. */
#define SBG_ENUM7_ALL_MAX_GATES 64
int sbg_enum7_all(sbg_handle *h, int part, int nparts, const uint8_t *outer_order,
    const uint8_t *middle_order, uint64_t max_matches, sbg_match *out, uint64_t *n_out,
    uint64_t *total, uint64_t *feasible);
/* The 7-LUT realisations search_7lut never tries: three LUTs wired as a chain,
   L3(L2(L1(a,b,c), d, e), f, g), over the 7-combinations sbg_enum7_all takes (no gate excluded by
   inbits, check_n_lut_possible(7) passed; *feasible as there, under a depth filter the ones with a
   chain row within the bound).  Row k = 6 j + q (sbg_chain_row): j = the lexicographic index of
   L1's position triple among the 3-subsets of 0..6 of the ascending combination, q = that of the
   pair {d, e} among the 2-subsets of the four other positions; f, g = the other two.  Inside each
   LUT the inputs are in ascending position, the first the cell's high bit: L2's cells are
   x1<<2 | d<<1 | e, L3's x2<<2 | f<<1 | g.  A match is (combination, k, po, pm) with L1 =
   outer_order[po] and L2 = middle_order[pm] for which L3 is solvable without a random fill,
   decided on the true gate tables.  Key rank<<24 | k<<16 | po<<8 | pm (rank as for sbg_enum7_all).
   Record: width 7, shape SBG_SHAPE_CHAIN, gates a..g in row order, func_outer = L1, func_middle
   = L2, func_inner / inner_seen = L3's solved bits and seen cells.  Depth (sbg_enum_set_depth)
   1 + max(1 + max(1 + max(Da, Db, Dc), Dd, De), Df, Dg); function filter: outer = L1, middle = L2,
   inner = L3; groupings: SBG_GROUP_SHAPE key >> 16, SBG_GROUP_TUPLE key >> 24.  Arguments, limits,
   tickets, deal blocks, the cursor and its calls, the count buffers and the errors are those of
   sbg_enum7_all; the call builds no list and leaves an installed one alone. */
int sbg_enum7_chain(sbg_handle *h, int part, int nparts, const uint8_t *outer_order,
    const uint8_t *middle_order, uint64_t max_matches, sbg_match *out, uint64_t *n_out,
    uint64_t *total, uint64_t *feasible);
/* The two-LUT realisations search_5lut never tries: L2 reads one of L1's inputs again,
   L2(L1(a,b,c), s, d) with s in {a, b, c}.  For each value of s, L1 may then compute a different
   function of the other two, so the shape covers more than any circuit over five distinct gates.
   Combinations: every 4-combination r0 < r1 < r2 < r3 in lexicographic order with no gate excluded
   by inbits that passes check_n_lut_possible(4) (no cell of 16 holds a masked 1 and a masked 0).
   Row k = 3 j + q (sbg_shared_row): j = the position of d, the gate L1 does not read; q = the index
   of s among L1's three positions, ascending.  L1's cells are a<<2 | b<<1 | c, L1's gates
   ascending; L2's are x1<<2 | u<<1 | v with (u, v) = {s, d} ascending.  A match is (combination, k,
   po) with L1 = func_order[po] (search_5lut's shuffled order) for which L2 is solvable without a
   random fill.  Key rank << 12 | k << 8 | po, rank = the combination's lexicographic rank among
   C(n,4) (below 2^32 at n <= 500, so it reads as a 5-LUT key).  Record: width 4, shape
   SBG_SHAPE_SHARED, gates[0..2] = a, b, c and gates[3..4] = u, v (add_lut's argument order: the
   record reads as a 5-LUT one with s repeated), gates[5..6] = 0, func_outer = L1, func_inner /
   inner_seen = L2's solved bits and seen cells.  Depth (sbg_enum_set_depth) 1 + max(1 + max(Da,
   Db, Dc), Du, Dv); function filter: outer = L1, inner = L2 (middle plays no part); groupings:
   SBG_GROUP_SHAPE key >> 8, SBG_GROUP_TUPLE key >> 12.  *feasible = the share's feasible
   4-combinations (under a depth filter, those with a row within the bound).  part/nparts,
   max_matches, the count-free first K, the cursor and its calls (fetch, pick, group sizes, depth
   counts, global ranks) behave as for sbg_enum5; a share's tickets are 3-gate prefixes dealt in
   blocks of 16, and the count buffers take 12 bytes per prefix, C(n-1, 3) of them (248 MB at
   n = 500).  The call builds no list and leaves an installed one alone.  SBG_ERR_ARG: n < 4, an
   order that is not a permutation, or a depth filter of another n; SBG_ERR_STATE: no problem
   loaded.  The call ends the cursor, whatever it returns. */
int sbg_enum4_shared(sbg_handle *h, int part, int nparts, const uint8_t *func_order,
    uint64_t max_matches, sbg_match *out, uint64_t *n_out, uint64_t *total, uint64_t *feasible);
/* The matches of lut_search's 3-LUT scan (lut.c:501-523) over the caller's shuffled gate order
   (n entries): the position triples i < k < m whose gates gate_order[i], gate_order[k],
   gate_order[m] pass check_n_lut_possible(3, ...) under the mask (get_lut_function then cannot
   fail, so each feasible triple is exactly one match).  inbits plays no part, as in the scan.
   Key i << 18 | k << 9 | m, as sbg_node_result::key3, so the first match is the triple the scan of
   sbg_search_node(SBG_DO_SCAN3) returns.  Record: width 3; gates[0..2] = gate_order[i],
   gate_order[k], gate_order[m] (add_lut's argument order, as sbg_node_result::gates3), gates[3..6]
   = 0; func_outer = func_middle = 0; func_inner / inner_seen as sbg_solve_inner gives them, cell
   a<<2 | b<<1 | c with a the gate at position i.  The work is the n(n-1)/2 position pairs (i, k);
   part/nparts, max_matches, total and the count-free stop behave as for sbg_enum5, and *feasible =
   the feasible triples met, which is the number of matches counted.  The call does not touch the
   installed 7-LUT list: an sbg_search7 / sbg_enum7 after it sees what it would have seen without
   it.  sbg_search_node takes its gate order as given; sbg_enum3 checks that gate_order is a
   permutation of 0..n-1 (as every order create_circuit builds is, sboxgates.c:285-299) and returns
   SBG_ERR_ARG otherwise, or when n < 3. */
int sbg_enum3(sbg_handle *h, int part, int nparts, const uint16_t *gate_order,
    uint64_t max_matches, sbg_match *out, uint64_t *n_out, uint64_t *total, uint64_t *feasible);

/* ---- matches at any rank: the enumeration cursor ---------------------------------------------- */
/* The cursor is the last sbg_enum3 / sbg_enum4_shared / sbg_enum5 / sbg_enum7 / sbg_enum7_all /
   sbg_enum7_chain call
   on the handle that counted
   (total != NULL; max_matches may be 0).  Ranks are positions in that call's share (part/nparts),
   in ascending key order: 0 .. total-1.  The device keeps what that count found (matches per
   ticket and where each ticket's matches start), so a fetch or pick emits the matches of the
   tickets it touches and counts nothing again; records are byte-identical to the ones the counted
   call emits at the same ranks.  Neither call consumes RNG or changes the problem, the installed
   7-LUT list or the cursor: any number of them may follow one count.  The cursor keeps the orders
   it was counted with; the caller's buffers of that call are not read again.  Cursor lifetime:
     - a counted sbg_enum* call replaces it; a count-free one ends it;
     - any call of sbg_load_problem, sbg_stage_problem, sbg_use_problem, sbg_search5, sbg_search7,
       sbg_search7_chain, sbg_search4_shared, sbg_search_node, sbg_search_batch, sbg_search5_part, sbg_finish5, sbg_filter7_part,
       sbg_set_list7, sbg_list7_device, sbg_set_list7_device, sbg_allgather_merge7 (every handle
       given), sbg_decomp7_part, sbg_finish7 or sbg_alu_peak ends it, whatever the call returns;
     - sbg_last_error, sbg_launch_count, sbg_transfer_stats, sbg_host_seconds, sbg_last_kernel_ms,
       sbg_set_timing, sbg_set_stream, sbg_enum_fetch, sbg_enum_pick, sbg_enum_block_sums,
       sbg_enum_set_global, sbg_enum_depth_counts and sbg_enum_group_sizes keep it;
     - sbg_enum_set_depth ends it, whatever the call returns.
     - sbg_enum_set_functions ends it, whatever the call returns.
     - sbg_enum_set_grouping ends it, whatever the call returns.
   Without a cursor both calls return SBG_ERR_STATE.
   A fetch or pick does the emit work of every ticket it touches up to the last wanted rank in it:
   a ticket is a position pair (3-LUT, up to n - 2 matches), a 3-gate prefix (5-LUT; shared-input:
   up to n - 3 combinations of 12 * 256 matches), a list
   entry (7-LUT, up to 70 * 65,536 matches) or a 6-gate prefix (sbg_enum7_all, up to n - 7
   combinations of that many; sbg_enum7_chain, of 210 * 65,536), so one deep rank can cost a whole
   ticket's sweep. */
/* The matches at ranks first .. min(first + count, total) - 1, in key order, to out[0..]; *n_out =
   how many (0 when first >= total).  count <= SBG_ENUM_MAX_MATCHES; out may be NULL iff count ==
   0. */
int sbg_enum_fetch(sbg_handle *h, uint64_t first, uint64_t count, sbg_match *out, uint64_t *n_out);
/* out[i] = the match at rank ranks[i], i < nranks <= SBG_ENUM_MAX_MATCHES.  The ranks may come in
   any order and repeat.  A rank >= total: SBG_ERR_ARG and nothing written.  (The ranks are sorted
   on the host and located on the device; each ticket holding one is swept once.) */
int sbg_enum_pick(sbg_handle *h, const uint64_t *ranks, uint64_t nranks, sbg_match *out);

/* ---- global ranks across shares --------------------------------------------------------------- */
/* A share's tickets fall into deal blocks, in the order the parts are dealt them: blocks of 16
   position pairs (3-LUT), 3-gate prefixes (5-LUT) or 6-gate prefixes (sbg_enum7_all,
   sbg_enum7_chain), local block j
   being the whole's block j * nparts + part; or single list entries (sbg_enum7), local entry t
   being list entry t * nparts + part.  The whole's blocks are in key order, so from every share's
   block sums each share can turn its ranks into ranks of the whole (a global cursor):
     1. every share counts (sbg_enum* with part = its part, nparts, total != NULL);
     2. sbg_enum_block_sums on each; the rows are gathered in part order;
     3. sbg_enum_set_global on each with all the rows;
     4. sbg_enum_fetch / sbg_enum_pick on each with the same ranks; the shares' outputs, summed (or
        OR-ed) as 64-bit words, are the records one handle's whole-share cursor (part 0 of 1)
        returns for those ranks.
   Both calls need a counted cursor (SBG_ERR_STATE without one) and keep it, whatever they return.
   On a global cursor fetch and pick take ranks of the whole; the first >= total checks and *n_out
   use the whole's total, so every share returns the same n_out.  Each share writes the records of
   the ranks it owns and an all-zero record (width == 0) at every other slot of out[0 .. n_out)
   (fetch) or out[0 .. nranks) (pick); it sweeps only the tickets holding the ranks it owns.  The
   calls that end a cursor end a global one. */
/* *nblocks = the number of the share's deal blocks; out != NULL: out[j] = the matches of its local
   block j.  out may be host or device memory (the copy is cudaMemcpyDefault). */
int sbg_enum_block_sums(sbg_handle *h, uint64_t *out, uint64_t *nblocks);
/* Makes the cursor global and sets *total (and the cursor's total) to the whole's total.  Part q's
   block sums are sums[q * stride .. q * stride + counts[q] - 1]; sums may be host or device memory,
   counts is host memory.  SBG_ERR_ARG, with the cursor left local and usable: nparts is not the
   cursor's nparts, a counts[q] is not the number of blocks the dealing gives part q, stride is below
   the largest counts[q], or the row of the cursor's own part is not its block sums (compared on the
   device: catches a gather in the wrong part order).  SBG_ERR_STATE: no cursor, or it is already
   global.  nparts == 1 is allowed and changes nothing observable. */
int sbg_enum_set_global(sbg_handle *h, const uint64_t *sums, uint64_t stride,
    const uint64_t *counts, int nparts, uint64_t *total);

/* ---- depth filter: the realisations at or below a circuit depth ------------------------------ */
/* The caller gives a depth for every gate of the problem, D[g] for g < n (any values up to
   SBG_MAX_DEPTH; they need not come from a real graph, and a large D[g] excludes gate g), and a
   bound max_depth.  A match's depth is that of the output gate it would add, from its record's
   gates in reference order:
     3-LUT a,b,c:     1 + max(Da, Db, Dc);
     5-LUT a..e:      1 + max(1 + max(Da, Db, Dc), Dd, De)            (outer LUT over a,b,c);
     7-LUT a..g:      1 + max(1 + max(Da, Db, Dc), 1 + max(Dd, De, Df), Dg);
     7-LUT chain a..g: 1 + max(1 + max(1 + max(Da, Db, Dc), Dd, De), Df, Dg) (sbg_enum7_chain);
     shared-input a..c, u, v: 1 + max(1 + max(Da, Db, Dc), Du, Dv)    (sbg_enum4_shared).
   Under a filter the matches of sbg_enum3 / sbg_enum5 / sbg_enum7 are exactly the unfiltered
   matches of depth <= max_depth: keys, key order and records are unchanged, only the set shrinks,
   and ranks are ranks within it.  The 7-LUT list is still the phase-1 list (the first
   SBG_LIST_CAP feasible 7-combinations whatever their depths).  *feasible of sbg_enum5 then counts
   the feasible combinations with an ordering within the bound (sbg_enum3: the matches counted,
   sbg_enum7: the list length, as without a filter).  The cursor keeps the filter it was counted
   under, so fetch, pick, sbg_enum_block_sums and sbg_enum_set_global serve the filtered set.
   Searches (sbg_search*, sbg_search_node / batch, the *_part and finish calls) never read it. */
#define SBG_MAX_DEPTH 1020     /* largest gate depth of a filter */
#define SBG_DEPTH_BINS 1024    /* bins of the depth histogram (a match is at most 1,023 deep) */
/* Installs the filter (n depths, host memory) for the later sbg_enum3 / sbg_enum5 / sbg_enum7
   calls on the handle; depth == NULL clears it.  SBG_ERR_ARG, with the filter left as it was: n
   outside 1..SBG_MAX_GATES or a depth above SBG_MAX_DEPTH.  An sbg_enum* call whose problem does
   not have n gates returns SBG_ERR_ARG.  The call ends the cursor. */
int sbg_enum_set_depth(sbg_handle *h, const uint16_t *depth, int n, uint32_t max_depth);
/* out[d] = the number of the cursor's counted matches of depth d, d < nbins <= SBG_DEPTH_BINS
   (deeper bins are not reported).  Per share, as totals are: the shares' arrays add up to the
   whole's.  The minimum depth: count with max_depth = SBG_DEPTH_BINS - 1, take the first non-empty
   bin, count again with that bound.  SBG_ERR_STATE without a cursor or when it was counted without
   a filter; SBG_ERR_ARG for nbins > SBG_DEPTH_BINS.  Keeps the cursor. */
int sbg_enum_depth_counts(sbg_handle *h, uint64_t *out, uint32_t nbins);

/* ---- function filter: the realisations whose LUTs lie in given sets of functions ------------- */
/* The caller gives three sets of 3-input functions, outer, middle and inner, each 4 words: bit f of
   word f >> 6 set = function f allowed, functions numbered as for sbg_lut_table (bit index
   in1<<2 | in2<<1 | in3).  A match is kept iff
     7-LUT: func_outer is in outer, func_middle is in middle, and the inner LUT can be completed
            inside inner;
     5-LUT: func_outer is in outer, and the inner LUT can be completed inside inner (middle plays
            no part);
     3-LUT: the LUT can be completed inside inner (outer and middle play no part);
   where "can be completed inside inner" means some f in inner has (f & inner_seen) == func_inner,
   from the match's record (not from a random fill, so the result is deterministic).  Under a
   filter the matches of sbg_enum3 / sbg_enum5 / sbg_enum7 are exactly the unfiltered matches that
   pass it: keys, key order and records are unchanged, only the set shrinks, and ranks are ranks
   within it.  The 7-LUT list is still the phase-1 list, and *feasible keeps its meaning (with a
   depth filter, its depth-filtered one).  Together with a depth filter both tests apply, and
   sbg_enum_depth_counts reports the matches that pass both.  The cursor keeps the filter it was
   counted under, so fetch, pick, sbg_enum_block_sums and sbg_enum_set_global serve the filtered
   set.  Searches (sbg_search*, sbg_search_node / batch, the *_part and finish calls) never read
   it.  A filtered 7-LUT count with a restricted inner set visits every (outer, middle) pair of
   each cube union instead of counting the union's bits, so it costs more than the others. */
/* Installs the filter (host memory; NULL = all 256 functions) for the later sbg_enum3 /
   sbg_enum5 / sbg_enum7 calls on the handle; all three NULL clears it.  An empty set is valid and
   leaves no match.  The call ends the cursor. */
int sbg_enum_set_functions(sbg_handle *h, const uint64_t *outer, const uint64_t *middle,
    const uint64_t *inner);
/* Test hook, no device needed: the inner table the kernels read.  out[code(seen, ones)] = 1 iff
   some f in inner (4 words; NULL = all 256) has (f & seen) == ones, else 0, for every seen and
   every ones within seen; code(S, V) = p3(S) + p3(V), p3(x) = the sum of 3^j over the set bits j
   of x (6,561 entries). */
int sbg_inner_table(const uint64_t *inner, uint8_t *out);

/* ---- grouping: the distinct gate sets and wirings that realise a state ----------------------- */
/* A realisation (one key) fixes the gates, the ordering row and the functions of the LUTs.  Under a
   grouping, sbg_enum3 / sbg_enum5 / sbg_enum7 enumerate groups of matches instead: the matches
   sharing a key prefix,
     SBG_GROUP_SHAPE: the gates and the ordering row (the wiring): 5-LUT key >> 8, 7-LUT key >> 16;
     SBG_GROUP_TUPLE: the gate set: 5-LUT key >> 12, 7-LUT key >> 23 (chain: key >> 24).
   A shared-input key (sbg_enum4_shared) groups as a 5-LUT key: >> 8 (shape), >> 12 (tuple).
   A 3-LUT key already is its gate set and wiring, so at width 3 every grouping is the identity.
   The total is the number of groups holding at least one match (after the depth and function
   filters); each group has one record, its first match (smallest key), byte-identical to the
   ungrouped record of that key, in ascending key order; ranks count groups.  The cursor keeps the
   grouping it was counted under, so fetch, pick, the count-free first K, sbg_enum_block_sums and
   sbg_enum_set_global serve the grouped set.  *feasible keeps its meaning, the 7-LUT list is still
   the phase-1 list, and searches never read the setting.  sbg_enum_depth_counts bins each group
   once, at the depth of its record: every match of a shape has the same depth, but a gate set's
   record is its first match, which need not be its shallowest (a histogram by shallowest gate set
   needs no grouping or shape grouping).  How many matches a group holds: sbg_enum_group_sizes. */
#define SBG_GROUP_NONE 0    /* every match (the default) */
#define SBG_GROUP_SHAPE 1   /* one per (gates, ordering row) */
#define SBG_GROUP_TUPLE 2   /* one per gate set */
/* Sets the grouping of the later sbg_enum3 / sbg_enum5 / sbg_enum7 calls on the handle.  Any other
   value: SBG_ERR_ARG, with the setting left as it was.  The call ends the cursor. */
int sbg_enum_set_grouping(sbg_handle *h, int grouping);
/* sizes[i] = the number of matches in the group at rank ranks[i] of the cursor, i < nranks <=
   SBG_ENUM_MAX_MATCHES: the matches the ungrouped enumeration, under the cursor's depth and
   function filters, would count with that group's id (match_group).  5-LUT shape: the outer
   functions that survive for that (tuple, row); 5-LUT tuple: their sum over the tuple's rows within
   the depth bound; 7-LUT shape: the (outer, middle) pairs of that (entry, row) that pass the
   filters; 7-LUT tuple: their sum over the entry's rows.  Every size is at least 1 and at most
   2,560 (5-LUT tuple) or 70 * 65,536 = 4,587,520 (7-LUT tuple; chain: 65,536 for a shape and
   210 * 65,536 for a tuple); the sizes of all ranks add up to
   the ungrouped total.  On an ungrouped cursor, or at width 3, every size is 1.  The ranks may
   come in any order and repeat.  A rank >= total: SBG_ERR_ARG and nothing written; ranks or sizes
   NULL with nranks > 0: SBG_ERR_ARG; no cursor: SBG_ERR_STATE.  Keeps the cursor, and changes
   neither the problem, the installed 7-LUT list nor the depth histogram.  On a global cursor each
   share writes the sizes of the ranks it owns and 0 at every other slot, so the shares' arrays,
   summed, are the whole's sizes.  Cost: the grouped pick's walk of every ticket holding a wanted
   rank, plus, per wanted group, the ungrouped count of its rows (a tuple group: its whole ticket's
   count; a 7-LUT count with a restricted inner set visits every (outer, middle) pair). */
int sbg_enum_group_sizes(sbg_handle *h, const uint64_t *ranks, uint64_t nranks, uint64_t *sizes);

/* ---- helpers shared with the host side ------------------------------------------------------ */
/* Test hook, no device needed: how a sweep's work is cut into tickets (DESIGN.md section 2, "Dense
   states").  width = 7 with prefix_gates = 4 or 5 (search_7lut phase 1), width = 5 with
   prefix_gates = 3 (search_5lut, fused kernel); n >= 8 gates, `excluded` = bit g set for an excluded
   gate g < 8 (lut.c:177-185); mode 0 = whole-prefix tickets only, 1 = a head of `waves` waves of
   (prefix, chunk) tickets over the allowed gates, 2 = chunk tickets throughout.
   out[0] = chunk tickets' items, out[1] = chunks per prefix, out[2] = lexicographic rank, among all
   prefixes, of the first prefix left to the whole-prefix tickets (= out[3] if none is left),
   out[3] = number of prefixes. */
int sbg_plan_tickets(int width, int prefix_gates, int n, uint32_t excluded, int mode,
                     uint64_t waves, uint64_t *out);

/* Test hook, no device needed: the ticket tables of search_7lut phase 1's weighted form (4-gate
   prefixes cut into groups of `group_pairs` (e,f) pairs, tickets numbered in lexicographic order of
   (prefix, group); 7 <= n <= 72).  out[0] = tickets of the whole sweep, out[1 + 76 * (r-1) + x] =
   tickets of all ways to choose r more prefix gates the first of which is >= x (r = 1..4). */
#define SBG_WEIGHTED_ROW 76
int sbg_weighted_tickets(int n, uint32_t group_pairs, uint32_t *out);

/* Row k of the ordering tables (lut.c:189-229 for width 5, lut.c:396-415 for width 7). */
int sbg_ordering_row(int width, int k, int *row);
/* Chain row k < 210 of sbg_enum7_chain: the seven positions in record order a..g. */
int sbg_chain_row(int k, int *row);
/* Shared-input row k < 12 of sbg_enum4_shared: the five positions (0..3 in the combination) in
   record order a, b, c, u, v; one of u, v repeats one of a, b, c. */
int sbg_shared_row(int k, int *row);
/* Closed form of get_lut_function without the random fill (lut.c:79-103): returns 1 and the
   solved function / seen mask, or 0 on conflict. */
int sbg_solve_inner(const uint64_t *in1, const uint64_t *in2, const uint64_t *in3,
    const uint64_t *target, const uint64_t *mask, uint8_t *func, uint8_t *seen);
/* generate_lut_ttable (state.c:202-230). */
void sbg_lut_table(uint8_t func, const uint64_t *in1, const uint64_t *in2, const uint64_t *in3,
    uint64_t *out);

#ifdef __cplusplus
}
#endif
#endif /* SBOXGATES_B200_H */
