/* lut_shim.c -- see lut_shim.h.  Plain C, compiled by gcc; everything CUDA is behind
 * include/sboxgates_b200.h. */
#define _POSIX_C_SOURCE 200809L
#include "lut_shim.h"

#include <pthread.h>
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include "sboxgates_b200.h"

_Static_assert(sizeof(sbg_ttable) == 32, "ttable must be 32 bytes (state.h:64-68)");
_Static_assert(sizeof(sbg_gate) == 64, "gate must be 64 bytes (state.h:72-79)");
_Static_assert(offsetof(sbg_gate, type) == 32 && offsetof(sbg_gate, in1) == 36
    && offsetof(sbg_gate, function) == 42, "gate field offsets (state.h:72-79)");
_Static_assert(offsetof(sbg_state, num_gates) == 10 && offsetof(sbg_state, gates) == 32,
    "state field offsets (state.h:81-88)");
_Static_assert(sizeof(sbg_state) == 32032, "state must be 32,032 bytes (state.h:81-88)");
_Static_assert(sizeof(sbg_boolfunc) == 24, "boolfunc must be 24 bytes (boolfunc.h:28-40)");
_Static_assert(offsetof(sbg_options, randomize) == 2019 && offsetof(sbg_options, verbosity) == 9756
    && sizeof(sbg_options) == 9760, "options field offsets (sboxgates.h:49-66)");

/* Devices: SBG_GPUS=N (default 1) drives CUDA devices SBG_DEVICE .. SBG_DEVICE+N-1 from this one
   process.  Searches above the size thresholds are sharded over them (one persistent host thread
   per device around the sbg_*_part calls; minimum key over the devices, per-device hit lists
   gathered and merged on the devices -- the in-process counterpart of the all-reduce(MIN) /
   all-gather that sboxgates_b200/distributed.py does over NCCL); smaller ones run on the first
   device only.
   SBG_LUT_CHAIN=1 (node variant; default off) adds a stage the reference does not have to
   lut_search: when search_7lut ran and found nothing, the first three-LUT chain
   L3(L2(L1(a,b,c), d, e), f, g) over the same 7-combinations and function orders
   (sbg_search7_chain) is built from three add_lut calls, where the reference would go on to
   multiplexer recursion.  A node without a chain leaves the state and the random stream exactly as
   without the variable; a node with one takes only L3's don't-care fill from the generator.
   SBG_LUT_SHARED=1 (node variant; default off) adds another such stage, between search_5lut and
   search_7lut: when search_5lut ran and found nothing, the first two-LUT circuit whose L2 reads one
   of L1's inputs again, L2(L1(a,b,c), u, v) with {u, v} = {s, d} and s in {a, b, c}
   (sbg_search4_shared, over every 4-combination, under search_5lut's function order), is built
   from two add_lut calls.  search_7lut (and the chain stage) then run only if it finds nothing, so
   with the variable set a node's device call stops after search_5lut.  A node without such a
   circuit leaves the state and the random stream exactly as without the variable; a node with one
   takes only L2's don't-care fill from the generator (search_7lut's 512 draws do not happen). */
#define SBG_SHIM_MAX_GPUS 8
static sbg_handle *g_handles[SBG_SHIM_MAX_GPUS];
static int g_ngpus = 0;
static double g_shard_min5 = 5e7, g_shard_min7 = 2e8;
static int g_shard_min_list = 8192;
static uint64_t g_sharded_calls = 0;
#define g_handle (g_handles[0])
static uint64_t g_calls[3] = {0, 0, 0};          /* search_5lut, search_7lut, lut_search */
static double g_seconds[3] = {0.0, 0.0, 0.0};
static uint64_t g_node_stage[6] = {0, 0, 0, 0, 0, 0};  /* node calls that ended at: nothing, 3, 5,
                                                         7, the 7-LUT chain, the shared-input pair */
static int g_lut_chain = 0;                         /* SBG_LUT_CHAIN */
static uint64_t g_chain_calls = 0;                  /* sbg_search7_chain calls and their seconds */
static double g_chain_seconds = 0.0;
static int g_lut_shared = 0;                        /* SBG_LUT_SHARED */
static uint64_t g_shared_calls = 0;                 /* sbg_search4_shared calls and their seconds */
static double g_shared_seconds = 0.0;
static double g_kernel_ms[4] = {0.0, 0.0, 0.0, 0.0}; /* search5, filter7, ordering, decomp7 */
static int g_stats = 0;

static double g_init_seconds = 0.0;   /* sbg_create: CUDA start-up + buffers, once */

static double now(void) {
  struct timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}

/* Errors are fatal, as in the reference, whose internal inconsistencies are assert()s
   (lut.c:118-119, 201, 452; sboxgates.h:31-44). */
static void die(const char *what, int rc, const sbg_handle *h) {
  fprintf(stderr, "sboxgates_b200: %s failed (%d): %s\n", what, rc,
      h != NULL ? sbg_last_error(h) : "no handle");
  abort();
}

/* ---- one persistent host thread per additional device ----------------------------------------- */

typedef struct {
  int part;
  int phase;                 /* 5: search5_part; 71: load + filter7_part; 72: decomp7_part */
  const uint64_t *flat;      /* problem (phases 5 and 71; device 0 is loaded by the caller) */
  int n;
  const uint64_t *target, *mask;
  const int8_t *inbits;
  const uint8_t *order_a, *order_b;
  int count;                 /* 71: out */
  uint64_t key;              /* 5, 72: out */
  int rc;
} shard_job;

static pthread_t g_threads[SBG_SHIM_MAX_GPUS];
static pthread_mutex_t g_mu = PTHREAD_MUTEX_INITIALIZER;
static pthread_cond_t g_cv_work = PTHREAD_COND_INITIALIZER, g_cv_done = PTHREAD_COND_INITIALIZER;
static shard_job *g_jobs = NULL;
static uint64_t g_epoch = 0;
static int g_pending = 0, g_quit = 0;

static void shard_run(shard_job *j) {
  sbg_handle *h = g_handles[j->part];
  j->rc = SBG_OK;
  if (j->part != 0 && (j->phase == 5 || j->phase == 71)) {
    j->rc = sbg_load_problem(h, j->flat, j->n, j->target, j->mask, j->inbits);
    if (j->rc != SBG_OK) return;
  }
  if (j->phase == 5) {
    j->rc = sbg_search5_part(h, j->part, g_ngpus, j->order_a, &j->key);
  } else if (j->phase == 71) {
    j->rc = sbg_filter7_part(h, j->part, g_ngpus, NULL, &j->count);
  } else {
    j->rc = sbg_decomp7_part(h, j->part, g_ngpus, j->order_a, j->order_b, &j->key);
  }
}

static void *shard_thread(void *arg) {
  const int part = (int)(intptr_t)arg;
  uint64_t seen = 0;
  pthread_mutex_lock(&g_mu);
  for (;;) {
    while (!g_quit && g_epoch == seen) pthread_cond_wait(&g_cv_work, &g_mu);
    if (g_quit) break;
    seen = g_epoch;
    shard_job *j = &g_jobs[part];
    pthread_mutex_unlock(&g_mu);
    shard_run(j);
    pthread_mutex_lock(&g_mu);
    if (--g_pending == 0) pthread_cond_signal(&g_cv_done);
  }
  pthread_mutex_unlock(&g_mu);
  return NULL;
}

static void run_shards(shard_job *jobs) {
  pthread_mutex_lock(&g_mu);
  g_jobs = jobs;
  g_pending = g_ngpus - 1;
  g_epoch++;
  pthread_cond_broadcast(&g_cv_work);
  pthread_mutex_unlock(&g_mu);
  shard_run(&jobs[0]);
  pthread_mutex_lock(&g_mu);
  while (g_pending > 0) pthread_cond_wait(&g_cv_done, &g_mu);
  pthread_mutex_unlock(&g_mu);
  for (int i = 0; i < g_ngpus; i++) {
    if (jobs[i].rc != SBG_OK) {
      fprintf(stderr, "sboxgates_b200: sharded phase %d failed on device %d\n", jobs[i].phase, i);
      die("sharded phase", jobs[i].rc, g_handles[i]);
    }
  }
  g_sharded_calls++;
}

static void shim_exit(void) {
  if (g_handle == NULL) return;
  if (g_ngpus > 1) {
    pthread_mutex_lock(&g_mu);
    g_quit = 1;
    pthread_cond_broadcast(&g_cv_work);
    pthread_mutex_unlock(&g_mu);
    for (int i = 1; i < g_ngpus; i++) pthread_join(g_threads[i], NULL);
  }
  if (g_stats) {
    uint64_t tr[5] = {0, 0, 0, 0, 0};
    sbg_transfer_stats(g_handle, tr);
    /* only with SBG_LUT_CHAIN / SBG_LUT_SHARED, so the default line stays as it was */
    char chain_col[64] = "", shared_col[64] = "";
    if (g_lut_chain) {
      snprintf(chain_col, sizeof(chain_col), ", 7-LUT chain %llu",
          (unsigned long long)g_node_stage[4]);
    }
    if (g_lut_shared) {
      snprintf(shared_col, sizeof(shared_col), ", shared-input pair %llu",
          (unsigned long long)g_node_stage[5]);
    }
    fprintf(stderr, "[sbg] start-up (sbg_create) %.3f s, inside the first call; "
        "lut_search: %llu calls %.3f s (ended at: 3-LUT %llu, 5-LUT %llu%s, 7-LUT %llu%s, nothing %llu); "
        "search_5lut: %llu calls %.3f s; search_7lut: %llu calls %.3f s; "
        "%llu kernel launches; state changes: %llu bulk copies, %llu as kernel arguments, %llu none; "
        "%llu B host->device, %llu B device->host\n", g_init_seconds,
        (unsigned long long)g_calls[2], g_seconds[2], (unsigned long long)g_node_stage[1],
        (unsigned long long)g_node_stage[2], shared_col, (unsigned long long)g_node_stage[3],
        chain_col,
        (unsigned long long)g_node_stage[0], (unsigned long long)g_calls[0], g_seconds[0],
        (unsigned long long)g_calls[1], g_seconds[1],
        (unsigned long long)sbg_launch_count(g_handle), (unsigned long long)tr[2],
        (unsigned long long)tr[3], (unsigned long long)tr[4], (unsigned long long)tr[0],
        (unsigned long long)tr[1]);
    double hs[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
    sbg_host_seconds(g_handle, hs);
    if (g_calls[2] != 0) {
      fprintf(stderr, "[sbg] node calls: %.3f s enqueueing chains, %.3f s waiting for results, "
          "%.3f s around them (flattening the state, shuffles, add_lut)\n", hs[0], hs[1],
          g_seconds[2] - g_init_seconds - hs[0] - hs[1]);
    }
    fprintf(stderr, "[sbg] waiting by stage: 3-LUT scan %.3f s, search_5lut %.3f s, search_7lut "
        "%.3f s\n", hs[2], hs[3], hs[4]);
    if (g_lut_shared) {
      fprintf(stderr, "[sbg] shared-input stage: %llu calls %.3f s, %llu nodes took a pair\n",
          (unsigned long long)g_shared_calls, g_shared_seconds, (unsigned long long)g_node_stage[5]);
    }
    if (g_lut_chain) {
      fprintf(stderr, "[sbg] 7-LUT chain stage: %llu calls %.3f s, %llu nodes took a chain\n",
          (unsigned long long)g_chain_calls, g_chain_seconds, (unsigned long long)g_node_stage[4]);
    }
    if (getenv("SBG_TIMING") != NULL) {
      fprintf(stderr, "[sbg] kernel time: search5 %.3f s, filter7 %.3f s, ordering %.3f s, "
          "decomp7 %.3f s\n", 1e-3 * g_kernel_ms[0], 1e-3 * g_kernel_ms[1], 1e-3 * g_kernel_ms[2],
          1e-3 * g_kernel_ms[3]);
    }
    if (g_ngpus > 1) {
      fprintf(stderr, "[sbg] %d devices, %llu sharded search phases\n", g_ngpus,
          (unsigned long long)g_sharded_calls);
    }
  }
  for (int i = 0; i < g_ngpus; i++) {
    sbg_destroy(g_handles[i]);
    g_handles[i] = NULL;
  }
}

static sbg_handle *handle(void) {
  if (g_handle == NULL) {
    const double t_init = now();
    const char *dev = getenv("SBG_DEVICE");
    const char *gpus = getenv("SBG_GPUS");
    const int first = dev != NULL ? atoi(dev) : 0;
    int want = gpus != NULL ? atoi(gpus) : 1;
    if (want < 1) want = 1;
    if (want > SBG_SHIM_MAX_GPUS) {
      fprintf(stderr, "sboxgates_b200: SBG_GPUS=%d clamped to %d\n", want, SBG_SHIM_MAX_GPUS);
      want = SBG_SHIM_MAX_GPUS;
    }
    g_stats = getenv("SBG_SHIM_STATS") != NULL;
    g_lut_chain = getenv("SBG_LUT_CHAIN") != NULL && atoi(getenv("SBG_LUT_CHAIN")) != 0;
    g_lut_shared = getenv("SBG_LUT_SHARED") != NULL && atoi(getenv("SBG_LUT_SHARED")) != 0;
    for (int i = 0; i < want; i++) {
      int rc = sbg_create(&g_handles[i], first + i);
      if (rc != SBG_OK) {
        fprintf(stderr, "sboxgates_b200: sbg_create(device %d)\n", first + i);
        die("sbg_create", rc, g_handles[i]);
      }
      g_ngpus = i + 1;
    }
    for (int i = 1; i < g_ngpus; i++) {
      if (pthread_create(&g_threads[i], NULL, shard_thread, (void *)(intptr_t)i) != 0) abort();
    }
    if (getenv("SBG_SHARD_MIN5") != NULL) g_shard_min5 = atof(getenv("SBG_SHARD_MIN5"));
    if (getenv("SBG_SHARD_MIN7") != NULL) g_shard_min7 = atof(getenv("SBG_SHARD_MIN7"));
    if (getenv("SBG_SHARD_MIN_LIST") != NULL) g_shard_min_list = atoi(getenv("SBG_SHARD_MIN_LIST"));
    atexit(shim_exit);
    g_init_seconds = now() - t_init;
  }
  return g_handle;
}

/* SBG_SHIM_TRACE=file (diagnostics): one line per search_5lut / search_7lut the reference would have
   made -- width, n, a hash of the inputs, found, ret[] -- so that runs of the two shim variants (and
   recorded reference runs) can be compared call by call. */
static FILE *g_trace = NULL;
static void trace_call(int which, const sbg_state *st, const sbg_ttable target,
    const sbg_ttable mask, bool found, const uint16_t *ret) {
  static int init = 0;
  if (!init) {
    init = 1;
    const char *path = getenv("SBG_SHIM_TRACE");
    if (path != NULL) g_trace = fopen(path, "w");
  }
  if (g_trace == NULL) return;
  uint64_t hsh = 1469598103934665603ull;
  const unsigned char *p = (const unsigned char *)&st->gates[0];
  for (int g = 0; g < st->num_gates; g++) {
    for (int b = 0; b < 32; b++) hsh = (hsh ^ p[(size_t)g * sizeof(sbg_gate) + b]) * 1099511628211ull;
  }
  p = (const unsigned char *)&target;
  for (int b = 0; b < 32; b++) hsh = (hsh ^ p[b]) * 1099511628211ull;
  p = (const unsigned char *)&mask;
  for (int b = 0; b < 32; b++) hsh = (hsh ^ p[b]) * 1099511628211ull;
  fprintf(g_trace, "%d %d %016llx %d", which, st->num_gates, (unsigned long long)hsh, found ? 1 : 0);
  for (int i = 0; i < 10; i++) fprintf(g_trace, " %d", found ? ret[i] : 0);
  fprintf(g_trace, "\n");
  fflush(g_trace);
}

static double n_choose(int n, int k) {
  double r = 1.0;
  for (int i = 1; i <= k; i++) r = r * (double)(n - i + 1) / (double)i;
  return r;
}

static uint64_t g_flat[SBG_SHIM_MAX_GATES * 4];
static uint64_t g_t[4], g_m[4];

static void load(sbg_handle *h, const sbg_state *st, const sbg_ttable target, const sbg_ttable mask,
    const int8_t *inbits) {
  uint64_t *flat = g_flat, *t = g_t, *m = g_m;
  const int n = st->num_gates;
  for (int i = 0; i < n; i++) {
    memcpy(flat + 4 * i, &st->gates[i].table, 32);
  }
  memcpy(t, &target, 32);
  memcpy(m, &mask, 32);
  int rc = sbg_load_problem(h, flat, n, t, m, inbits);
  if (rc != SBG_OK) die("sbg_load_problem", rc, h);
}

static void add_kernel_times(sbg_handle *h) {
  for (int i = 0; i < 4; i++) g_kernel_ms[i] += sbg_last_kernel_ms(h, i);
}

/* The two shuffles (lut.c:125-135, 362-378) from a source of random values. */
static void shuffle5(uint64_t (*draw)(void *), void *ctx, uint8_t *func_order) {
  for (int i = 0; i < 256; i++) func_order[i] = (uint8_t)i;
  for (int i = 0; i < 256; i++) {
    const uint64_t j = draw(ctx) % (uint64_t)(i + 1);
    const uint8_t t = func_order[i];
    func_order[i] = func_order[j];
    func_order[j] = t;
  }
}

static void shuffle7(uint64_t (*draw)(void *), void *ctx, uint8_t *outer_order,
    uint8_t *middle_order) {
  for (int i = 0; i < 256; i++) outer_order[i] = middle_order[i] = (uint8_t)i;
  for (int i = 0; i < 256; i++) {
    const uint64_t oj = draw(ctx) % (uint64_t)(i + 1);
    const uint64_t mj = draw(ctx) % (uint64_t)(i + 1);
    const uint8_t ot = outer_order[i];
    const uint8_t mt = middle_order[i];
    outer_order[i] = outer_order[oj];
    middle_order[i] = middle_order[mj];
    outer_order[oj] = ot;
    middle_order[mj] = mt;
  }
}

static uint64_t draw_now(void *ctx) {
  (void)ctx;
  return xorshift1024();
}

/* search_5lut / search_7lut of the loaded state over all devices (the searches large enough to
   shard), result in *res. */
static void sharded_search5(sbg_handle *h, const sbg_state *st, const int8_t *inbits,
    const uint8_t *func_order, sbg_result *res) {
  shard_job jobs[SBG_SHIM_MAX_GPUS];
  uint64_t key = SBG_KEY_NONE;
  for (int i = 0; i < g_ngpus; i++) {
    jobs[i] = (shard_job){.part = i, .phase = 5, .flat = g_flat, .n = st->num_gates,
        .target = g_t, .mask = g_m, .inbits = inbits, .order_a = func_order};
  }
  run_shards(jobs);
  for (int i = 0; i < g_ngpus; i++) key = jobs[i].key < key ? jobs[i].key : key;
  int rc = sbg_finish5(h, key, func_order, res);
  if (rc != SBG_OK) die("sbg_finish5", rc, h);
}

static void sharded_search7(sbg_handle *h, const sbg_state *st, const int8_t *inbits,
    const uint8_t *outer_order, const uint8_t *middle_order, sbg_result *res) {
  /* phase 1 sharded: per-device ordered lists -> gathered and merged on every device, cut at
     SBG_LIST_CAP (lut.c:329-349 at size 1) */
  shard_job jobs[SBG_SHIM_MAX_GPUS];
  for (int i = 0; i < g_ngpus; i++) {
    jobs[i] = (shard_job){.part = i, .phase = 71, .flat = g_flat, .n = st->num_gates,
        .target = g_t, .mask = g_m, .inbits = inbits};
  }
  run_shards(jobs);
  int total = 0;
  int rc = sbg_allgather_merge7(g_handles, g_ngpus, &total);
  if (rc != SBG_OK) die("sbg_allgather_merge7", rc, h);
  uint64_t key = SBG_KEY_NONE;
  if (total >= g_shard_min_list) {
    for (int i = 0; i < g_ngpus; i++) {
      jobs[i] = (shard_job){.part = i, .phase = 72, .order_a = outer_order,
          .order_b = middle_order};
    }
    run_shards(jobs);
    for (int i = 0; i < g_ngpus; i++) key = jobs[i].key < key ? jobs[i].key : key;
  } else {
    rc = sbg_decomp7_part(h, 0, 1, outer_order, middle_order, &key);
    if (rc != SBG_OK) die("sbg_decomp7_part", rc, h);
  }
  rc = sbg_finish7(h, key, outer_order, middle_order, res);
  if (rc != SBG_OK) die("sbg_finish7", rc, h);
}

static void print_found5(const uint16_t *ret) { /* lut.c:219-222 */
  printf("[% 4d] Found 5LUT: %02x %02x    %3d %3d %3d %3d %3d\n", 0, ret[0], ret[1], ret[2],
      ret[3], ret[4], ret[5], ret[6]);
}

static void print_found7(const uint16_t *ret) { /* lut.c:470-473 */
  printf("[% 4d] Found 7LUT: %02x %02x %02x %3d %3d %3d %3d %3d %3d %3d\n", 0, ret[0], ret[1],
      ret[2], ret[3], ret[4], ret[5], ret[6], ret[7], ret[8], ret[9]);
}

/* get_lut_function's random fill of never-constrained LUT bits (lut.c:104-106): one draw iff some
   inner cell was not seen under the mask. */
static uint8_t fill_dont_cares(uint8_t func, uint8_t seen) {
  if (seen != 0xff) func |= (uint8_t)(~seen & (uint8_t)xorshift1024());
  return func;
}

bool search_5lut(const sbg_state st, const sbg_ttable target, const sbg_ttable mask,
    const int8_t *inbits, uint16_t *ret, int verbosity) {
  if (ret == NULL || st.num_gates < 5) abort(); /* lut.c:118-119 */
  const double t0 = now();
  sbg_handle *h = handle();

  uint8_t func_order[256]; /* lut.c:125-135: 256 draws, always */
  shuffle5(draw_now, NULL, func_order);
  memset(ret, 0, sizeof(uint16_t) * 10); /* lut.c:171 */

  load(h, &st, target, mask, inbits);
  sbg_result res;
  if (g_ngpus > 1 && n_choose(st.num_gates, 5) >= g_shard_min5) {
    sharded_search5(h, &st, inbits, func_order, &res);
  } else {
    int rc = sbg_search5(h, func_order, &res);
    if (rc != SBG_OK) die("sbg_search5", rc, h);
  }
  if (res.found) {
    ret[0] = res.func_outer;
    ret[1] = fill_dont_cares(res.func_inner, res.inner_seen);
    for (int i = 0; i < 5; i++) ret[2 + i] = res.gates[i];
    if (verbosity >= 1) print_found5(ret);
  }
  trace_call(5, &st, target, mask, res.found != 0, ret);
  g_calls[0]++;
  g_seconds[0] += now() - t0;
  add_kernel_times(h);
  return res.found != 0;
}

bool search_7lut(const sbg_state st, const sbg_ttable target, const sbg_ttable mask,
    const int8_t *inbits, uint16_t *ret, int verbosity) {
  if (ret == NULL || st.num_gates < 7) abort(); /* lut.c:258-259 */
  const double t0 = now();
  sbg_handle *h = handle();

  /* lut.c:362-378 draws these after phase 1; phase 1 draws nothing, so the stream is the same. */
  uint8_t outer_order[256], middle_order[256];
  shuffle7(draw_now, NULL, outer_order, middle_order);
  memset(ret, 0, sizeof(uint16_t) * 10); /* lut.c:383 */

  load(h, &st, target, mask, inbits);
  sbg_result res;
  if (g_ngpus > 1 && n_choose(st.num_gates, 7) >= g_shard_min7) {
    sharded_search7(h, &st, inbits, outer_order, middle_order, &res);
  } else {
    int rc = sbg_search7(h, outer_order, middle_order, &res);
    if (rc != SBG_OK) die("sbg_search7", rc, h);
  }
  if (res.found) {
    ret[0] = res.func_outer;
    ret[1] = res.func_middle;
    ret[2] = fill_dont_cares(res.func_inner, res.inner_seen);
    for (int i = 0; i < 7; i++) ret[3 + i] = res.gates[i];
    if (verbosity >= 1) print_found7(ret);
  }
  trace_call(7, &st, target, mask, res.found != 0, ret);
  g_calls[1]++;
  g_seconds[1] += now() - t0;
  add_kernel_times(h);
  return res.found != 0;
}

void sbg_shim_stats(uint64_t *calls5, uint64_t *calls7, double *seconds5, double *seconds7) {
  if (calls5 != NULL) *calls5 = g_calls[0];
  if (calls7 != NULL) *calls7 = g_calls[1];
  if (seconds5 != NULL) *seconds5 = g_seconds[0];
  if (seconds7 != NULL) *seconds7 = g_seconds[1];
}

#ifdef SBG_SHIM_NODE
/* ---- lut_search as one device call (lut.c:489-631) ------------------------------------------- */

/* Host functions the reference's lut_search calls (sboxgates.h:78-112, state.h:104-108). */
uint16_t add_lut(sbg_state *st, uint8_t func, sbg_ttable table, uint16_t gid1, uint16_t gid2,
    uint16_t gid3);
bool check_num_gates_possible(const sbg_state *st, int add, int add_sat, const sbg_options *opt);
bool ttable_equals_mask(const sbg_ttable in1, const sbg_ttable in2, const sbg_ttable mask);
sbg_ttable generate_lut_ttable(const uint8_t function, const sbg_ttable in1, const sbg_ttable in2,
    const sbg_ttable in3);
int get_num_inputs(const sbg_state *st);

/* Look-ahead in front of the host's generator.  Everyone -- the host's own code and this file --
   draws through xorshift1024() below, so the sequence of values is the host generator's, in order;
   peeking only makes values that WILL be drawn next known early. */
#define LA_SIZE 1024
static uint64_t la_buf[LA_SIZE];
static unsigned la_head = 0, la_count = 0;

uint64_t xorshift1024(void) {
  if (la_count != 0) {
    const uint64_t v = la_buf[la_head];
    la_head = (la_head + 1) % LA_SIZE;
    la_count--;
    return v;
  }
  return sbg_host_xorshift1024();
}

typedef struct { unsigned next; } peek_ctx;

static uint64_t draw_peek(void *ctx) {
  peek_ctx *p = (peek_ctx *)ctx;
  while (la_count <= p->next) {
    la_buf[(la_head + la_count) % LA_SIZE] = sbg_host_xorshift1024();
    la_count++;
  }
  return la_buf[(la_head + p->next++) % LA_SIZE];
}

static void consume(unsigned k) {
  for (unsigned i = 0; i < k; i++) (void)xorshift1024();
}

/* The reference re-verifies every gate it returns (sboxgates.h:31-44). */
static uint16_t checked(uint16_t gate, const sbg_state *st, const sbg_ttable target,
    const sbg_ttable mask, int line) {
  if (gate == SBG_SHIM_NO_GATE || ttable_equals_mask(target, st->gates[gate].table, mask)) {
    return gate;
  }
  fprintf(stderr, "Return assertion in lut_search failed: %s:%d.\n", __FILE__, line);
  abort();
}

static void require(bool ok, int line) {
  if (!ok) {
    fprintf(stderr, "sboxgates_b200: assertion failed (%s:%d)\n", __FILE__, line);
    abort();
  }
}

uint16_t lut_search(sbg_state *st, const sbg_ttable target, const sbg_ttable mask,
    const int8_t *inbits, const uint16_t *gate_order, const sbg_options *opt) {
  require(st != NULL && inbits != NULL && gate_order != NULL && opt != NULL && opt->lut_graph,
      __LINE__); /* lut.c:491-495 */
  const double t0 = now();
  sbg_handle *h = handle();
  const int n = st->num_gates;
  /* which stages the reference would run if the earlier ones fail (lut.c:525-527, 553, 582-593):
     the state is not modified on those paths, so the gate-budget checks can be made up front */
  const bool do5 = check_num_gates_possible(st, 2, 0, opt);
  const bool do7 = do5 && check_num_gates_possible(st, 3, 0, opt);
  const bool big5 = g_ngpus > 1 && n_choose(n, 5) >= g_shard_min5;
  const bool big7 = g_ngpus > 1 && n_choose(n, 7) >= g_shard_min7;

  /* The shuffles search_5lut / search_7lut would make, from values the host generator will yield
     next (looked at, not consumed): 256 for the first (lut.c:125-135), then 512 for the second
     (lut.c:362-378); a stage's draws are consumed below once it is known to have run. */
  uint8_t order5[256], outer[256], middle[256];
  peek_ctx pk = {0};
  if (do5 && n >= 5) shuffle5(draw_peek, &pk, order5);
  if (do7 && n >= 7) shuffle7(draw_peek, &pk, outer, middle);

  load(h, st, target, mask, inbits);
  sbg_job job;
  memset(&job, 0, sizeof(job));
  job.slot = 0;
  job.gate_order = gate_order;
  job.flags = SBG_DO_SCAN3;
  /* SBG_NODE_SPLIT=1 (diagnostics): every stage as a device call of its own */
  static int split = -1;
  if (split < 0) split = getenv("SBG_NODE_SPLIT") != NULL && atoi(getenv("SBG_NODE_SPLIT")) != 0;
  const bool chain5 = do5 && n >= 5 && !big5 && !split;
  /* with SBG_LUT_SHARED the shared-input stage sits between search_5lut and search_7lut, so the
     device call stops after search_5lut */
  const bool chain7 = chain5 && do7 && n >= 7 && !big7 && !g_lut_shared;
  if (chain5) {
    job.flags |= SBG_DO_SEARCH5;
    job.order5 = order5;
  }
  if (chain7) {
    job.flags |= SBG_DO_SEARCH7;
    job.outer7 = outer;
    job.middle7 = middle;
  }
  sbg_node_result nr;
  int rc = sbg_search_node(h, &job, &nr);
  if (rc != SBG_OK) die("sbg_search_node", rc, h);
  add_kernel_times(h);
  g_calls[2]++;

  uint16_t out = SBG_SHIM_NO_GATE;
  int stage = 0;
  bool chained = false;   /* the node took the 7-LUT chain (SBG_LUT_CHAIN) */
  bool shared = false;    /* the node took the shared-input pair (SBG_LUT_SHARED) */
  if (nr.found_stage == 3) { /* lut.c:501-523 */
    const uint16_t gi = nr.gates3[0], gk = nr.gates3[1], gm = nr.gates3[2];
    uint8_t func = nr.func3;
    if (opt->randomize) func = fill_dont_cares(func, nr.seen3);
    const sbg_ttable nt = generate_lut_ttable(func, st->gates[gi].table, st->gates[gk].table,
        st->gates[gm].table);
    require(ttable_equals_mask(target, nt, mask), __LINE__);
    out = checked(add_lut(st, func, nt, gi, gk, gm), st, target, mask, __LINE__);
    stage = 3;
    goto done;
  }
  if (!do5) goto done; /* lut.c:525-527 */

  if (opt->verbosity >= 2) printf("[   0] Search 5.\n"); /* lut.c:549-551 */
  if (n >= 5) {
    consume(256);
    sbg_result r5 = nr.r5;
    if (big5) {
      sharded_search5(h, st, inbits, order5, &r5);
    } else if (!chain5) {
      rc = sbg_search5(h, order5, &r5);
      if (rc != SBG_OK) die("sbg_search5", rc, h);
    }
    if (r5.found) { /* lut.c:555-580 */
      uint16_t ret[10] = {0};
      ret[0] = r5.func_outer;
      ret[1] = fill_dont_cares(r5.func_inner, r5.inner_seen);
      for (int i = 0; i < 5; i++) ret[2 + i] = r5.gates[i];
      trace_call(5, st, target, mask, true, ret);
      if (opt->verbosity >= 1) {
        print_found5(ret);
        printf("[   0]   Selected: %02x %02x    %3d %3d %3d %3d %3d\n", ret[0], ret[1], ret[2],
            ret[3], ret[4], ret[5], ret[6]);
      }
      const sbg_ttable t_outer = generate_lut_ttable((uint8_t)ret[0], st->gates[ret[2]].table,
          st->gates[ret[3]].table, st->gates[ret[4]].table);
      const sbg_ttable t_inner = generate_lut_ttable((uint8_t)ret[1], t_outer,
          st->gates[ret[5]].table, st->gates[ret[6]].table);
      require(ttable_equals_mask(target, t_inner, mask), __LINE__);
      const uint16_t g_outer = add_lut(st, (uint8_t)ret[0], t_outer, ret[2], ret[3], ret[4]);
      out = checked(add_lut(st, (uint8_t)ret[1], t_inner, g_outer, ret[5], ret[6]), st, target,
          mask, __LINE__);
      stage = 5;
      goto done;
    }
    trace_call(5, st, target, mask, false, NULL);
    if (g_lut_shared) {
      /* not in the reference: the first two-LUT circuit whose L2 reads one of L1's inputs again,
         under search_5lut's function order, before search_7lut runs */
      const double ts = now();
      sbg_result rs;
      rc = sbg_search4_shared(h, order5, &rs);
      if (rc != SBG_OK) die("sbg_search4_shared", rc, h);
      g_shared_calls++;
      g_shared_seconds += now() - ts;
      if (rs.found) {
        const uint16_t *g = rs.gates;
        const uint8_t l1 = rs.func_outer;
        const uint8_t l2 = fill_dont_cares(rs.func_inner, rs.inner_seen);
        if (opt->verbosity >= 1) {
          printf("[   0]   Selected shared: %02x %02x    %3d %3d %3d %3d %3d\n", l1, l2, g[0], g[1],
              g[2], g[3], g[4]);
        }
        const sbg_ttable t1 = generate_lut_ttable(l1, st->gates[g[0]].table,
            st->gates[g[1]].table, st->gates[g[2]].table);
        const sbg_ttable t2 = generate_lut_ttable(l2, t1, st->gates[g[3]].table,
            st->gates[g[4]].table);
        require(ttable_equals_mask(target, t2, mask), __LINE__);
        const uint16_t g1 = add_lut(st, l1, t1, g[0], g[1], g[2]);
        out = checked(add_lut(st, l2, t2, g1, g[3], g[4]), st, target, mask, __LINE__);
        stage = 5;
        shared = true;
        goto done;
      }
    }
  }
  if (!do7) goto done; /* lut.c:582-586 */

  if (opt->verbosity >= 2) printf("[   0] Search 7.\n"); /* lut.c:590-592 */
  if (n >= 7) {
    consume(512);
    sbg_result r7 = nr.r7;
    if (!chain7) {
      /* the chain did not include this stage: run it now, over all devices when it is large */
      if (big7) {
        sharded_search7(h, st, inbits, outer, middle, &r7);
      } else {
        rc = sbg_search7(h, outer, middle, &r7);
        if (rc != SBG_OK) die("sbg_search7", rc, h);
      }
    }
    if (r7.found) { /* lut.c:595-625 */
      uint16_t ret[10];
      ret[0] = r7.func_outer;
      ret[1] = r7.func_middle;
      ret[2] = fill_dont_cares(r7.func_inner, r7.inner_seen);
      for (int i = 0; i < 7; i++) ret[3 + i] = r7.gates[i];
      trace_call(7, st, target, mask, true, ret);
      if (opt->verbosity >= 1) {
        print_found7(ret);
        printf("[   0]   Selected: %02x %02x %02x %3d %3d %3d %3d %3d %3d %3d\n", ret[0], ret[1],
            ret[2], ret[3], ret[4], ret[5], ret[6], ret[7], ret[8], ret[9]);
      }
      const sbg_ttable t_outer = generate_lut_ttable((uint8_t)ret[0], st->gates[ret[3]].table,
          st->gates[ret[4]].table, st->gates[ret[5]].table);
      const sbg_ttable t_middle = generate_lut_ttable((uint8_t)ret[1], st->gates[ret[6]].table,
          st->gates[ret[7]].table, st->gates[ret[8]].table);
      const sbg_ttable t_inner = generate_lut_ttable((uint8_t)ret[2], t_outer, t_middle,
          st->gates[ret[9]].table);
      require(ttable_equals_mask(target, t_inner, mask), __LINE__);
      /* lut.c:622-624 nests the two add_lut calls as arguments of the third; C leaves their order
         unspecified and gcc (the reference's compiler, CMakeLists.txt) evaluates arguments right to
         left on x86-64: the MIDDLE LUT gets the lower gate number.  Mirrored here, since gate numbers
         are part of the graph (and of its fingerprint). */
      const uint16_t g_middle = add_lut(st, (uint8_t)ret[1], t_middle, ret[6], ret[7], ret[8]);
      const uint16_t g_outer = add_lut(st, (uint8_t)ret[0], t_outer, ret[3], ret[4], ret[5]);
      out = checked(add_lut(st, (uint8_t)ret[2], t_inner, g_outer, g_middle, ret[9]), st, target,
          mask, __LINE__);
      stage = 7;
      goto done;
    }
    trace_call(7, st, target, mask, false, NULL);
    if (g_lut_chain) {
      /* not in the reference: the first 7-LUT chain over the list search_7lut just tried, which the
         handle still holds (sbg_search_node / sbg_search7 installed it, or the merge of a sharded
         phase 1 did on every device) */
      const double tc = now();
      sbg_result rc7;
      rc = sbg_search7_chain(h, outer, middle, &rc7);
      if (rc != SBG_OK) die("sbg_search7_chain", rc, h);
      g_chain_calls++;
      g_chain_seconds += now() - tc;
      if (rc7.found) {
        const uint16_t *g = rc7.gates;
        const uint8_t l1 = rc7.func_outer, l2 = rc7.func_middle;
        const uint8_t l3 = fill_dont_cares(rc7.func_inner, rc7.inner_seen);
        if (opt->verbosity >= 1) {
          printf("[   0]   Selected chain: %02x %02x %02x %3d %3d %3d %3d %3d %3d %3d\n", l1, l2,
              l3, g[0], g[1], g[2], g[3], g[4], g[5], g[6]);
        }
        const sbg_ttable t1 = generate_lut_ttable(l1, st->gates[g[0]].table,
            st->gates[g[1]].table, st->gates[g[2]].table);
        const sbg_ttable t2 = generate_lut_ttable(l2, t1, st->gates[g[3]].table,
            st->gates[g[4]].table);
        const sbg_ttable t3 = generate_lut_ttable(l3, t2, st->gates[g[5]].table,
            st->gates[g[6]].table);
        require(ttable_equals_mask(target, t3, mask), __LINE__);
        const uint16_t g1 = add_lut(st, l1, t1, g[0], g[1], g[2]);
        const uint16_t g2 = add_lut(st, l2, t2, g1, g[3], g[4]);
        out = checked(add_lut(st, l3, t3, g2, g[5], g[6]), st, target, mask, __LINE__);
        stage = 7;
        chained = true;
        goto done;
      }
    }
  }
  if (opt->verbosity >= 2) { /* lut.c:627-629 */
    printf("[   0] No LUTs found. Num gates: %d\n", st->num_gates - get_num_inputs(st));
  }
done:
  g_node_stage[shared ? 5 : chained ? 4 : stage == 0 ? 0 : (stage - 1) / 2]++;
  g_seconds[2] += now() - t0;
  return out;
}
#endif /* SBG_SHIM_NODE */
