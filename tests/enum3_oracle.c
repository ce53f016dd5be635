/* tests/enum3_oracle.c -- TEST INFRASTRUCTURE, not product code.
 *
 * CPU enumeration of every match of lut_search's 3-LUT scan (lut.c:501-523), the checker of
 * sbg_enum3.  The loop is orc_scan3_key's (tests/enum_oracle.c) without the early exit: every
 * position triple i < k < m of the gate order whose gates pass check_n_lut_possible(3, ...) under
 * the mask is a match (get_lut_function cannot fail then).  Built together with oracle/sbg_oracle.c
 * by tests/_enum3_support.py.
 */
#include <string.h>

#include "sbg_oracle.h"

/* Over the position triples of ranks [lo, hi) (lexicographic 3-subsets of {0..n-1}, hi clipped to
   C(n,3)): returns the number of matches and writes the first max_keys keys i<<18 | k<<9 | m.  A
   partition of the ranks visits every triple exactly once, so pieces can run on several threads. */
uint64_t orc_enum3_range(const uint64_t *tables, int n, const uint64_t *target,
    const uint64_t *mask, const uint16_t *order, int64_t lo, int64_t hi, uint64_t max_keys,
    uint64_t *keys) {
  const int64_t all = orc_n_choose_k(n, 3);
  if (hi > all) hi = all;
  uint16_t pos[3];
  if (lo < hi) orc_nth_combination(lo, n, 3, pos);
  uint64_t total = 0;
  for (int64_t r = lo; r < hi; r++, orc_next_combination(pos, 3, n)) {
    uint64_t tt[3 * 4];
    for (int m = 0; m < 3; m++) memcpy(tt + 4 * m, tables + 4 * order[pos[m]], 32);
    if (!orc_check_n_lut_possible(3, target, mask, tt)) continue;
    if (total < max_keys) keys[total] = (uint64_t)pos[0] << 18 | (uint64_t)pos[1] << 9 | pos[2];
    total++;
  }
  return total;
}
