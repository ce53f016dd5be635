"""CPU: the seeded call sequences of test_handle_calls_gpu.py still reach what that test was written
to reach -- each seed's sequence holds every defect pattern of _handle_support.patterns at least
once (a list consumer after a batch or after restaging the current slot, waves that repeat a slot
with a change or rows pending, two waves, a batch on a side stream)."""
import pytest

import _handle_support as H


@pytest.mark.parametrize("seed", H.SEEDS)
def test_sequence_reaches_every_pattern(seed):
    pool = H.make_pool(seed)
    ops = H.generate(seed, pool)
    assert len(ops) == H.STEPS
    missing = H.PATTERNS - H.patterns(pool, ops)
    assert not missing, (seed, sorted(missing))


@pytest.mark.parametrize("seed", H.SEEDS)
def test_sequence_is_reproducible_and_stays_in_range(seed):
    pool = H.make_pool(seed)
    ops = H.generate(seed, pool)
    assert ops == H.generate(seed, H.make_pool(seed))
    sizes = sorted(s.n for s in pool)
    assert sizes[-2:] == list(H.BIG) and 7 <= sizes[0] and sizes[-3] <= 48
    for op in ops:
        if op[0] == "batch":
            assert all(0 <= slot < 64 and flags for slot, flags, _ in op[1])
        if op[0] in ("stage", "use"):
            assert 0 <= op[1] < 64
