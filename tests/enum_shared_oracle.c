/* tests/enum_shared_oracle.c -- TEST INFRASTRUCTURE, not product code.
 *
 * CPU enumeration of every realisation of a target by two LUTs whose second reads one of the
 * first's inputs again, L2(L1(a,b,c), u, v) with {u, v} = {s, d}, s one of a, b, c: the checker of
 * sbg_enum4_shared.  Every 4-combination of the state is visited in lexicographic order; one with a
 * gate listed in inbits, or that fails orc_check_n_lut_possible(4), is skipped.  Every candidate
 * (combination, row, po) is then decided by direct evaluation: L1's table from its three gate
 * tables, then orc_solve_inner on (L1, u, v) under the mask -- no summaries, no cell tables.
 * Built with oracle/sbg_oracle.c by tests/_enum_shared_reference.py.
 */
#include <string.h>

#include "sbg_oracle.h"

/* Row k = 3 j + q: d at position j of the combination, L1 over the other three positions
   (ascending), s = the q-th of them; record order a, b, c (L1's), then u < v = {s, j}. */
void orc_shared_row(int k, int *row) {
  const int j = k / 3, q = k % 3;
  int r = 0;
  for (int i = 0; i < 4; i++) {
    if (i != j) row[r++] = i;
  }
  const int s = row[q];
  row[3] = s < j ? s : j;
  row[4] = s < j ? j : s;
}

/* Every shared-input match of the state, in ascending key order rank<<12 | k<<8 | po (rank = the
   combination's lexicographic rank among C(n,4)).  The first max_keys keys go to keys[], with L2's
   solved bits and seen cells to inner[] / seen[]; *feasible = the combinations that pass inbits
   and check_n_lut_possible(4); returns the number of matches. */
uint64_t orc_enum4_shared(const uint64_t *tables, int n, const uint64_t *target,
    const uint64_t *mask, const int8_t *inbits, const uint8_t *func_order, uint64_t max_keys,
    uint64_t *keys, uint8_t *inner, uint8_t *seen, uint64_t *feasible) {
  int rows[12][5];
  for (int k = 0; k < 12; k++) orc_shared_row(k, rows[k]);
  int excluded[512] = {0};
  for (int i = 0; i < 8 && inbits[i] != -1; i++) excluded[inbits[i]] = 1;
  uint64_t total = 0, feas = 0, rank = 0;
  uint16_t g[4] = {0, 1, 2, 3};
  for (; n >= 4; rank++, orc_next_combination(g, 4, n)) {
    if (excluded[g[0]] || excluded[g[1]] || excluded[g[2]] || excluded[g[3]]) goto next;
    {
      uint64_t packed[16];
      for (int i = 0; i < 4; i++) memcpy(packed + 4 * i, tables + 4 * g[i], 32);
      if (!orc_check_n_lut_possible(4, target, mask, packed)) goto next;
    }
    feas++;
    for (int k = 0; k < 12; k++) {
      const uint64_t *G[5];
      for (int i = 0; i < 5; i++) G[i] = tables + 4 * g[rows[k][i]];
      for (int po = 0; po < 256; po++) {
        uint64_t x1[4];
        uint8_t f, s;
        orc_lut_ttable(func_order[po], G[0], G[1], G[2], x1);
        if (!orc_solve_inner(x1, G[3], G[4], target, mask, &f, &s)) continue;
        if (total < max_keys) {
          keys[total] = rank << 12 | (uint64_t)k << 8 | (uint64_t)po;
          inner[total] = f;
          seen[total] = s;
        }
        total++;
      }
    }
  next:
    if (g[0] == n - 4) break;   /* the last combination */
  }
  *feasible = feas;
  return total;
}
