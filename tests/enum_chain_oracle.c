/* tests/enum_chain_oracle.c -- TEST INFRASTRUCTURE, not product code.
 *
 * CPU enumeration of every realisation of a target by the 7-LUT chain L3(L2(L1(a,b,c), d, e), f, g),
 * the checker of sbg_enum7_chain.  Every candidate (combination, row, po, pm) is decided by direct
 * evaluation: L1's table from the three gate tables, L2's from L1's and d, e, and then
 * orc_solve_inner on (L2, f, g) under the mask -- no cubes, no classes.  The one shortcut is exact:
 * an L1 whose 5-input remainder (L1, d, e, f, g) already puts a masked 1 and a masked 0 in one cell
 * has no L2 (the two positions agree on L2, f and g as well), so its 256 L2 are not tried.
 * Built with oracle/sbg_oracle.c by tests/_enum_chain_reference.py.
 */
#include <string.h>

#include "sbg_oracle.h"

/* Row k = 6 j + q: j = the lexicographic index of L1's position triple among the 3-subsets of
   0..6, q = that of {d, e} among the 2-subsets of the four other positions; f, g the other two. */
void orc_chain_row(int k, int *row) {
  int idx = 0;
  for (int a = 0; a < 7; a++) for (int b = a + 1; b < 7; b++) for (int c = b + 1; c < 7; c++) {
    int rest[4], r = 0;
    for (int i = 0; i < 7; i++) {
      if (i != a && i != b && i != c) rest[r++] = i;
    }
    for (int d = 0; d < 4; d++) for (int e = d + 1; e < 4; e++, idx++) {
      if (idx != k) continue;
      row[0] = a; row[1] = b; row[2] = c; row[3] = rest[d]; row[4] = rest[e];
      int w = 5;
      for (int i = 0; i < 4; i++) {
        if (i != d && i != e) row[w++] = rest[i];
      }
    }
  }
}

/* Whether some masked cell of the 5 tables t[0..4] holds a masked 1 and a masked 0. */
static int conflict5(const uint64_t *const *t, const uint64_t *target, const uint64_t *mask) {
  for (int cell = 0; cell < 32; cell++) {
    uint64_t one = 0, zero = 0;
    for (int w = 0; w < 4; w++) {
      uint64_t in = mask[w];
      for (int i = 0; i < 5; i++) in &= ((cell >> (4 - i)) & 1) ? t[i][w] : ~t[i][w];
      one |= in & target[w];
      zero |= in & ~target[w];
    }
    if (one && zero) return 1;
  }
  return 0;
}

/* Every chain match of the combinations tuples[0..ntuples-1] (7 gate numbers each, ascending), in
   ascending key order idx<<24 | k<<16 | po<<8 | pm (idx = the tuple's index here).  The first
   max_keys keys go to keys[], with L3's solved bits and seen cells to inner[] / seen[]; returns the
   number of matches. */
uint64_t orc_enum7_chain(const uint64_t *tables, const uint64_t *target, const uint64_t *mask,
    const uint16_t *tuples, int64_t ntuples, const uint8_t *outer_order,
    const uint8_t *middle_order, uint64_t max_keys, uint64_t *keys, uint8_t *inner, uint8_t *seen) {
  int rows[210][7];
  for (int k = 0; k < 210; k++) orc_chain_row(k, rows[k]);
  uint64_t total = 0;
  for (int64_t t = 0; t < ntuples; t++) {
    const uint16_t *g = tuples + 7 * t;
    for (int k = 0; k < 210; k++) {
      const uint64_t *G[7];
      for (int i = 0; i < 7; i++) G[i] = tables + 4 * g[rows[k][i]];
      for (int po = 0; po < 256; po++) {
        uint64_t x1[4], x2[4];
        orc_lut_ttable(outer_order[po], G[0], G[1], G[2], x1);
        const uint64_t *rem[5] = {x1, G[3], G[4], G[5], G[6]};
        if (conflict5(rem, target, mask)) continue;
        for (int pm = 0; pm < 256; pm++) {
          orc_lut_ttable(middle_order[pm], x1, G[3], G[4], x2);
          uint8_t f, s;
          if (!orc_solve_inner(x2, G[5], G[6], target, mask, &f, &s)) continue;
          if (total < max_keys) {
            keys[total] = (uint64_t)t << 24 | (uint64_t)k << 16 | (uint64_t)po << 8 | (uint64_t)pm;
            inner[total] = f;
            seen[total] = s;
          }
          total++;
        }
      }
    }
  }
  return total;
}
