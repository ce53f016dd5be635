/* tests/enum_oracle.c -- TEST INFRASTRUCTURE, not product code.
 *
 * CPU enumeration of every match of search_5lut / search_7lut, the checker of sbg_enum5 /
 * sbg_enum7.  The loops are those of orc_search5_key / orc_decomp7_key (oracle/sbg_oracle.c)
 * without the early exit: every candidate is decided, the matches are counted, and the first
 * max_keys keys (the loops run in ascending key order) are written out.  The 7-LUT candidates are
 * decided on the true gate tables (no stale outer cache).  Built together with oracle/sbg_oracle.c
 * by tests/test_enum_cpu.py.
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

/* lut.c:174-230 over all of C(n,5): returns the number of matches; *feasible = feasible
   combinations. */
uint64_t orc_enum5(const uint64_t *tables, int n, const uint64_t *target, const uint64_t *mask,
    const int8_t *inbits, const uint8_t *func_order, uint64_t max_keys, uint64_t *keys,
    uint64_t *feasible) {
  int rows[10][5];
  for (int k = 0; k < 10; k++) orc_order5_row(k, rows[k]);
  const int64_t combos = orc_n_choose_k(n, 5);
  uint16_t nums[5] = {0, 1, 2, 3, 4};
  uint64_t total = 0;
  *feasible = 0;
  for (int64_t r = 0; r < combos; r++, orc_next_combination(nums, 5, n)) {
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
        }
      }
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
