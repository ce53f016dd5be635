/* tests/enum_oracle.c -- TEST INFRASTRUCTURE, not product code.
 *
 * CPU enumeration of every match of search_5lut / search_7lut / lut_search's 3-LUT scan, the
 * checker of sbg_enum5 / sbg_enum7 / sbg_enum3.  The loops are those of orc_search5_key /
 * orc_decomp7_key (oracle/sbg_oracle.c) and orc_scan3_key (below)
 * without the early exit: every candidate is decided, the matches are counted, and the first
 * max_keys keys (the loops run in ascending key order) are written out.  The 7-LUT candidates are
 * decided on the true gate tables (no stale outer cache).  Built together with oracle/sbg_oracle.c
 * by tests/_enum_support.py.
 *
 * The *_range forms walk one range [lo, hi) of lexicographic combination ranks, so that a large
 * space can be cut into pieces and checked on several threads: the phase-1 list of search_7lut,
 * search_5lut's first-match key, its enumeration, and the 3-LUT scan of lut_search and its
 * enumeration.
 */
#include <stdlib.h>
#include <string.h>

#include "sbg_oracle.h"

static int rejected(const uint16_t *comb, int t, const int8_t *inbits) {
  for (int k = 0; k < 8 && inbits[k] != -1; k++) { /* lut.c:177-185 */
    for (int m = 0; m < t; m++) {
      if (comb[m] == (uint16_t)inbits[k]) return 1;
    }
  }
  return 0;
}

static void note(uint64_t key, uint64_t *total, uint64_t *keys, uint64_t max_keys) {
  if (*total < max_keys) keys[*total] = key;
  (*total)++;
}

/* The combinations of ranks [lo, hi) as lexicographic t-subsets of {0..n-1}, hi clipped to C(n,t).
   Starts at orc_nth_combination(lo) and steps with orc_next_combination, so that a partition of
   the ranks visits every combination exactly once. */
static int64_t range_start(int n, int t, int64_t lo, int64_t *hi, uint16_t *comb) {
  const int64_t all = orc_n_choose_k(n, t);
  if (*hi > all) *hi = all;
  if (lo < *hi) orc_nth_combination(lo, n, t, comb);
  return lo;
}

/* lut.c:174-230 over the 5-combinations of ranks [lo, hi): returns the number of matches (after
   the first one if stop_at_first); *feasible = feasible combinations met. */
static uint64_t enum5_range(const uint64_t *tables, int n, const uint64_t *target,
    const uint64_t *mask, const int8_t *inbits, const uint8_t *func_order, int64_t lo, int64_t hi,
    uint64_t max_keys, uint64_t *keys, uint64_t *feasible, int stop_at_first) {
  int rows[10][5];
  for (int k = 0; k < 10; k++) orc_order5_row(k, rows[k]);
  uint16_t nums[5];
  uint64_t total = 0;
  *feasible = 0;
  for (int64_t r = range_start(n, 5, lo, &hi, nums); r < hi; r++, orc_next_combination(nums, 5, n)) {
    if (rejected(nums, 5, inbits)) continue;
    uint64_t tt[5 * 4];
    for (int m = 0; m < 5; m++) memcpy(tt + 4 * m, tables + 4 * nums[m], 32);
    if (!orc_check_n_lut_possible(5, target, mask, tt)) continue;
    (*feasible)++;
    for (int k = 0; k < 10; k++) {
      const int *o = rows[k];
      for (int pos = 0; pos < 256; pos++) {
        uint64_t t_outer[4];
        uint8_t fi, seen;
        orc_lut_ttable(func_order[pos], tt + 4 * o[0], tt + 4 * o[1], tt + 4 * o[2], t_outer);
        if (orc_solve_inner(t_outer, tt + 4 * o[3], tt + 4 * o[4], target, mask, &fi, &seen)) {
          note((uint64_t)r << 12 | (uint64_t)k << 8 | (uint64_t)pos, &total, keys, max_keys);
          if (stop_at_first) return total;
        }
      }
    }
  }
  return total;
}

/* enum5 over ranks [lo, hi): the count, the feasible count and the first max_keys keys. */
uint64_t orc_enum5_range(const uint64_t *tables, int n, const uint64_t *target,
    const uint64_t *mask, const int8_t *inbits, const uint8_t *func_order, int64_t lo, int64_t hi,
    uint64_t max_keys, uint64_t *keys, uint64_t *feasible) {
  return enum5_range(tables, n, target, mask, inbits, func_order, lo, hi, max_keys, keys, feasible,
      0);
}

/* The whole space: returns the number of matches; *feasible = feasible combinations. */
uint64_t orc_enum5(const uint64_t *tables, int n, const uint64_t *target, const uint64_t *mask,
    const int8_t *inbits, const uint8_t *func_order, uint64_t max_keys, uint64_t *keys,
    uint64_t *feasible) {
  return orc_enum5_range(tables, n, target, mask, inbits, func_order, 0, orc_n_choose_k(n, 5),
      max_keys, keys, feasible);
}

/* orc_search5_key's first-match key restricted to ranks [lo, hi); UINT64_MAX if none. */
uint64_t orc_search5_range(const uint64_t *tables, int n, const uint64_t *target,
    const uint64_t *mask, const int8_t *inbits, const uint8_t *func_order, int64_t lo, int64_t hi) {
  uint64_t key = UINT64_MAX, feasible;
  enum5_range(tables, n, target, mask, inbits, func_order, lo, hi, 1, &key, &feasible, 1);
  return key;
}

/* The feasible 5-combinations (inbits applied) of ranks [lo, hi): what enum5_range counts in
   *feasible, without deciding any of them. */
uint64_t orc_feasible5_range(const uint64_t *tables, int n, const uint64_t *target,
    const uint64_t *mask, const int8_t *inbits, int64_t lo, int64_t hi) {
  uint16_t nums[5];
  uint64_t feasible = 0;
  for (int64_t r = range_start(n, 5, lo, &hi, nums); r < hi; r++, orc_next_combination(nums, 5, n)) {
    if (rejected(nums, 5, inbits)) continue;
    uint64_t tt[5 * 4];
    for (int m = 0; m < 5; m++) memcpy(tt + 4 * m, tables + 4 * nums[m], 32);
    feasible += orc_check_n_lut_possible(5, target, mask, tt) ? 1 : 0;
  }
  return feasible;
}

/* lut.c:290-327 over the 7-combinations of ranks [lo, hi): writes the first `cap` feasible ones
   (7 x uint16 each, inbits applied) in order; returns how many there are in the range. */
int64_t orc_filter7_range(const uint64_t *tables, int n, const uint64_t *target,
    const uint64_t *mask, const int8_t *inbits, int64_t lo, int64_t hi, uint16_t *list,
    int64_t cap) {
  uint16_t nums[7];
  int64_t count = 0;
  for (int64_t r = range_start(n, 7, lo, &hi, nums); r < hi; r++, orc_next_combination(nums, 7, n)) {
    if (rejected(nums, 7, inbits)) continue;
    uint64_t tt[7 * 4];
    for (int m = 0; m < 7; m++) memcpy(tt + 4 * m, tables + 4 * nums[m], 32);
    if (!orc_check_n_lut_possible(7, target, mask, tt)) continue;
    if (count < cap) memcpy(list + 7 * count, nums, 7 * sizeof(uint16_t));
    count++;
  }
  return count;
}

/* The entries of a 7-LUT list (count x 7 gates) that orc_check_n_lut_possible(7) rejects: returns
   how many, and the index of the first in *first (-1 if none). */
int64_t orc_check7_list(const uint64_t *tables, const uint64_t *target, const uint64_t *mask,
    const uint16_t *list, int64_t count, int64_t *first) {
  int64_t bad = 0;
  *first = -1;
  for (int64_t i = 0; i < count; i++) {
    uint64_t tt[7 * 4];
    for (int m = 0; m < 7; m++) memcpy(tt + 4 * m, tables + 4 * list[7 * i + m], 32);
    if (orc_check_n_lut_possible(7, target, mask, tt)) continue;
    if (bad++ == 0) *first = i;
  }
  return bad;
}

/* lut.c:501-523: the first triple of lut_search's 3-LUT scan over the gate order `order`, among
   the position triples i < k < m of ranks [lo, hi) (lexicographic 3-subsets of {0..n-1}).  Returns
   i<<18 | k<<9 | m, or UINT64_MAX if no triple of the range realises the target under the mask. */
uint64_t orc_scan3_key(const uint64_t *tables, int n, const uint64_t *target, const uint64_t *mask,
    const uint16_t *order, int64_t lo, int64_t hi) {
  uint16_t pos[3];
  for (int64_t r = range_start(n, 3, lo, &hi, pos); r < hi; r++, orc_next_combination(pos, 3, n)) {
    uint64_t tt[3 * 4];
    for (int m = 0; m < 3; m++) memcpy(tt + 4 * m, tables + 4 * order[pos[m]], 32);
    if (orc_check_n_lut_possible(3, target, mask, tt)) {
      return (uint64_t)pos[0] << 18 | (uint64_t)pos[1] << 9 | pos[2];
    }
  }
  return UINT64_MAX;
}

/* orc_scan3_key without the early exit, the checker of sbg_enum3: every position triple of ranks
   [lo, hi) whose gates pass check_n_lut_possible(3, ...) under the mask is a match
   (get_lut_function cannot fail then).  Returns the number of matches and writes the first
   max_keys keys i<<18 | k<<9 | m. */
uint64_t orc_enum3_range(const uint64_t *tables, int n, const uint64_t *target,
    const uint64_t *mask, const uint16_t *order, int64_t lo, int64_t hi, uint64_t max_keys,
    uint64_t *keys) {
  uint16_t pos[3];
  uint64_t total = 0;
  for (int64_t r = range_start(n, 3, lo, &hi, pos); r < hi; r++, orc_next_combination(pos, 3, n)) {
    uint64_t tt[3 * 4];
    for (int m = 0; m < 3; m++) memcpy(tt + 4 * m, tables + 4 * order[pos[m]], 32);
    if (orc_check_n_lut_possible(3, target, mask, tt)) {
      note((uint64_t)pos[0] << 18 | (uint64_t)pos[1] << 9 | pos[2], &total, keys, max_keys);
    }
  }
  return total;
}

/* lut.c:416-484 over the list (count entries of 7 gates each): returns the number of matches. */
uint64_t orc_enum7(const uint64_t *tables, const uint64_t *target, const uint64_t *mask,
    const uint16_t *list, int count, const uint8_t *outer_order, const uint8_t *middle_order,
    uint64_t max_keys, uint64_t *keys) {
  int rows[70][7];
  for (int k = 0; k < 70; k++) orc_order7_row(k, rows[k]);
  uint64_t (*t_outer)[4] = malloc(256 * 32);
  uint64_t (*t_middle)[4] = malloc(256 * 32);
  if (t_outer == NULL || t_middle == NULL) abort();
  uint64_t total = 0;
  for (int i = 0; i < count; i++) {
    const uint16_t *tuple = list + 7 * i;
    for (int k = 0; k < 70; k++) {
      uint16_t g[7];
      for (int m = 0; m < 7; m++) g[m] = tuple[rows[k][m]];
      for (int f = 0; f < 256; f++) {
        orc_lut_ttable((uint8_t)f, tables + 4 * g[0], tables + 4 * g[1], tables + 4 * g[2],
            t_outer[f]);
        orc_lut_ttable((uint8_t)f, tables + 4 * g[3], tables + 4 * g[4], tables + 4 * g[5],
            t_middle[f]);
      }
      for (int po = 0; po < 256; po++) {
        for (int pm = 0; pm < 256; pm++) {
          uint8_t fi, seen;
          if (orc_solve_inner(t_outer[outer_order[po]], t_middle[middle_order[pm]],
              tables + 4 * g[6], target, mask, &fi, &seen)) {
            note((uint64_t)i << 23 | (uint64_t)k << 16 | (uint64_t)po << 8 | (uint64_t)pm, &total,
                keys, max_keys);
          }
        }
      }
    }
  }
  free(t_outer);
  free(t_middle);
  return total;
}
