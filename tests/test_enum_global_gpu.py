"""GPU: global ranks across shares (sbg_enum_block_sums / sbg_enum_set_global).  P shares are P
LutEngine(0) handles, each counting part q of P; their block sums are gathered once through host
numpy arrays and once through CUDA torch tensors.  Every global fetch and pick, summed word-wise
over the shares, must equal what one whole-share handle (part 0 of 1) returns.  Also: large totals
against the closed forms of tests/_fetch_support.py (5-LUT at n = 40 and 64, the latter and the
7-LUT past 2^32; 3-LUT at n = 500, the largest state, C(500, 3) < 2^32), the error codes and cursor
rules, and DistributedLutSearch's enumeration over gloo (and NCCL when there are two GPUs)."""
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch

import _enum_reference as R
import _enum_support as E
import _fetch_support as F
import _support as S
import sboxgates_b200 as sb
from sboxgates_b200 import native
from test_enum_fetch_gpu import CASES, _case_state, _run

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_STATE = -1, -4
PMAX = 8


@pytest.fixture(scope="module")
def shares():
    engs = [sb.LutEngine(0) for _ in range(PMAX)]
    yield engs
    for e in engs:
        e.close()


def _gather(engs, via):
    counts = [e.enum_block_count() for e in engs]
    stride = max(max(counts), 1)
    if via == "numpy":
        sums = np.zeros((len(engs), stride), dtype=np.uint64)
        for q, e in enumerate(engs):
            sums[q, :counts[q]] = e.enum_block_sums()
    else:
        sums = torch.zeros((len(engs), stride), dtype=torch.int64, device="cuda")
        for q, e in enumerate(engs):
            e.enum_block_sums(out=sums[q])
    return sums, counts


def _count_global(engs, width, orders, via="numpy"):
    """Counts part q of P on engs[q] and makes every cursor global; returns the whole's total."""
    P = len(engs)
    for q, e in enumerate(engs):
        _run(e, width, orders, 0, True, q, P)
    sums, counts = _gather(engs, via)
    totals = {e.enum_set_global(sums, counts) for e in engs}
    assert len(totals) == 1
    return totals.pop()


def _summed(outs):
    """The shares' records summed as 64-bit words; checks that each slot has exactly one owner."""
    words = np.stack([o.view(np.uint64) for o in outs])
    owners = (np.stack([o["width"] for o in outs]) != 0).sum(axis=0)
    assert np.all(owners == 1), np.nonzero(owners != 1)[0][:10]
    for o in outs:   # the non-owners hold all-zero records
        z = o["width"] == 0
        assert not np.any(o[z].view(np.uint64)), "a non-owner wrote a non-zero record"
    return words.sum(axis=0, dtype=np.uint64).view(sb.MATCH_DTYPE)


def _fetch(engs, first, count):
    outs = [e.fetch_matches(first, count) for e in engs]
    assert len({len(o) for o in outs}) == 1
    return _summed(outs) if len(outs[0]) else outs[0]


def _pick(engs, ranks):
    return _summed([e.pick_matches(ranks) for e in engs])


@pytest.mark.parametrize("P", [1, 2, 3, 7])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_global_fetch_and_pick_equal_the_whole(engine, shares, case, P):
    width, (tabs, tgt, mask, inb), orders = _case_state(case)
    engine.load(tabs, tgt, mask, inb)
    total = _run(engine, width, orders, 0).total
    whole = engine.fetch_matches(0, total)
    assert len(whole) == total
    engs = shares[:P]
    for e in engs:
        e.load(tabs, tgt, mask, inb)
    for via in ("numpy", "torch"):
        assert _count_global(engs, width, orders, via) == total
        rs = np.random.RandomState(100 * case + P)
        # every rank once: its owner, and the block seams where the owner changes
        full = [e.fetch_matches(0, total) for e in engs]
        assert np.array_equal(_summed(full), whole)
        assert R.check_realises(_summed(full), tabs, tgt, mask) == total
        owner = np.argmax(np.stack([f["width"] for f in full]) != 0, axis=0)
        seams = [int(r) for r in np.nonzero(np.diff(owner))[0] + 1]
        for s in seams[:5] + seams[-3:]:
            for a, b in ((s, s + 1), (s - 1, s + 1), (max(0, s - 7), s), (s, s + 9)):
                assert np.array_equal(_fetch(engs, a, b - a), whole[a:b]), (s, a, b)
        for _ in range(8):
            first = int(rs.randint(0, total))
            count = int(rs.randint(1, max(2, total // 3)))
            assert np.array_equal(_fetch(engs, first, count), whole[first:first + count])
        tail = _fetch(engs, max(0, total - 3), 100)
        assert np.array_equal(tail, whole[max(0, total - 3):])
        for first, count in ((total, 5), (total + 1000, 5), (0, 0), (total // 2, 0)):
            assert all(len(e.fetch_matches(first, count)) == 0 for e in engs)
        ranks = np.concatenate([[total - 1, 0], rs.randint(0, total, 200), [0, total - 1],
                                rs.randint(0, total, 5).repeat(3)]).astype(np.int64)
        rs.shuffle(ranks)
        assert np.array_equal(_pick(engs, ranks), whole[ranks])
        # sample_matches on the shares, summed, is the whole handle's sample with the same seed
        k = min(total, 50)
        e_whole = _run(engine, width, orders, 0)
        r_whole, m_whole = sb.sample_matches(engine, e_whole, k, seed=case)
        got = [sb.sample_matches(e, sb.Enumeration(total, 0, whole[:0]), k, seed=case)
               for e in engs]
        assert all(np.array_equal(r, r_whole) for r, _ in got)
        assert np.array_equal(_summed([m for _, m in got]), m_whole)


def _check_closed(engs, total, record, rs, picks, state):
    """Pages and picks of the summed shares against the closed form; every record realises the
    target of `state` (tables, target, mask)."""
    for first in (0, total // 2 - 300, total // 2, total - 4096):
        got = _fetch(engs, first, 600 if first else 4096)
        assert len(got) == min(600 if first else 4096, total - first)
        assert R.check_realises(got, *state, what=first) == len(got)
        for j in sorted({0, len(got) - 1} | {int(x) for x in rs.randint(0, len(got), 30)}):
            assert F.as_tuple(got[j]) == record(first + j), (first, j)
    ranks = np.random.default_rng(int(rs.randint(1 << 30))).choice(total, picks, replace=False)
    got = _pick(engs, ranks)
    assert R.check_realises(got, *state, what="picks") == len(got)
    for r, rec in zip(ranks, got):
        assert F.as_tuple(rec) == record(int(r)), int(r)


@pytest.mark.parametrize("n,want", [(40, 1_684_500_480), (64, 19_518_750_720)])
def test_5lut_empty_mask_closed_form(shares, n, want):
    tabs = S.synthetic_state(n, seed=5100 + n)
    tgt = S.sbox_target(S.rijndael_sbox(), 6)
    mask = np.zeros(4, dtype=np.uint64)
    order = E.orders(n)[0]
    for e in shares:
        e.load(tabs, tgt, mask, [])
    total = _count_global(shares, 5, [None, order], "torch")
    assert total == F.total5(n, []) == want   # n = 64: past 2^32
    rows5 = S.order5_rows()
    _check_closed(shares, total, lambda r: F.record5(r, tabs, tgt, mask, [], order, rows5),
                  np.random.RandomState(5), 1000, (tabs, tgt, mask))


def test_7lut_n40_past_2_32(shares):
    n = 40
    tabs = S.synthetic_state(n, seed=5200)
    tgt = S.sbox_target(S.rijndael_sbox(), 4)
    mask = np.zeros(4, dtype=np.uint64)
    _, outer, middle = E.orders(77)
    engs = shares[:3]
    for e in engs:
        e.load(tabs, tgt, mask, [])
    total = _count_global(engs, 7, [None, None, outer, middle])
    assert total == F.total7(n, 100_000) == 458_752_000_000
    rows7 = S.order7_rows()
    _check_closed(engs, total,
                  lambda r: F.record7(r, tabs, tgt, mask, outer, middle, rows7, 100_000),
                  np.random.RandomState(7), 1000, (tabs, tgt, mask))


def test_3lut_n500(shares):
    n = 500
    tabs = S.synthetic_state(n, seed=5000)
    tgt = S.sbox_target(S.rijndael_sbox(), 3)
    mask = np.zeros(4, dtype=np.uint64)
    order = [int(x) for x in np.random.RandomState(5001).permutation(n)]
    for e in shares:
        e.load(tabs, tgt, mask, [])
    total = _count_global(shares, 3, [order])
    assert total == F.total3(n)
    _check_closed(shares, total, lambda r: F.record3(r, tabs, tgt, mask, order),
                  np.random.RandomState(3), 1000, (tabs, tgt, mask))


def _raw_set_global(eng, sums, stride, counts, nparts=None):
    sums = np.ascontiguousarray(sums, dtype=np.uint64)
    cnt = np.ascontiguousarray(counts, dtype=np.uint64)
    total = C.c_uint64()
    return eng.lib.sbg_enum_set_global(eng._h, sums.ctypes.data_as(C.c_void_p), stride,
                                       cnt.ctypes.data_as(native.u64p),
                                       len(counts) if nparts is None else nparts, C.byref(total))


def test_errors_and_cursor_rules():
    width, (tabs, tgt, mask, inb), orders = _case_state(5)
    engs = [sb.LutEngine(0) for _ in range(3)]
    try:
        e0 = engs[0]
        nb = C.c_uint64()
        assert e0.lib.sbg_enum_block_sums(e0._h, None, C.byref(nb)) == ERR_STATE
        assert _raw_set_global(e0, np.zeros((1, 1)), 1, [0]) == ERR_STATE
        for e in engs:
            e.load(tabs, tgt, mask, inb)
        # a count-free call leaves no cursor
        _run(e0, width, orders, 5, count=False, part=0, nparts=3)
        assert _raw_set_global(e0, np.zeros((3, 1)), 1, [0, 0, 0]) == ERR_STATE
        locals_ = []
        for q, e in enumerate(engs):
            t = _run(e, width, orders, 0, True, q, 3).total
            locals_.append((t, e.fetch_matches(0, t)))
        sums, counts = _gather(engs, "numpy")
        stride = sums.shape[1]
        assert not np.array_equal(sums[0], sums[1])   # so that swapping them is detectable
        swapped = sums[[1, 0, 2]]
        bad = [(sums, stride, counts, 2), (sums, stride, [counts[0] + 1] + counts[1:], 3),
               (sums, max(counts) - 1, counts, 3), (swapped, stride, counts, 3)]
        for s, st, cn, np_ in bad:
            for q in (0, 1):
                assert _raw_set_global(engs[q], s, st, cn, np_) == ERR_ARG, (st, cn, np_, q)
                t, m = locals_[q]
                assert np.array_equal(engs[q].fetch_matches(0, t), m)   # still local and usable
        total = {e.enum_set_global(sums, counts) for e in engs}.pop()
        assert total == sum(t for t, _ in locals_)
        assert _raw_set_global(e0, sums, stride, counts) == ERR_STATE   # already global
        # block sums, fetch and pick keep it
        whole = _summed([e.fetch_matches(0, total) for e in engs])
        for e in engs:
            assert np.array_equal(e.enum_block_sums(), sums[engs.index(e), :counts[engs.index(e)]])
        assert np.array_equal(_pick(engs, [total - 1, 0, 0]), whole[[total - 1, 0, 0]])
        assert np.array_equal(_fetch(engs, 0, total), whole)
        # a call that ends cursors ends a global one
        e0.load(tabs, tgt, mask, inb)
        assert e0.lib.sbg_enum_block_sums(e0._h, None, C.byref(nb)) == ERR_STATE
        with pytest.raises(RuntimeError):
            e0.fetch_matches(0, 1)
        # nparts == 1 changes nothing observable
        t = _run(e0, width, orders, 0).total
        ref = e0.fetch_matches(0, t)
        assert e0.enum_set_global(e0.enum_block_sums()[None, :], [e0.enum_block_count()]) == t
        assert np.array_equal(e0.fetch_matches(0, t), ref)
    finally:
        for e in engs:
            e.close()


# -- DistributedLutSearch on one GPU ---------------------------------------------------------------

DIST_CASES = [0, 5, 9]   # widths 3, 5, 7 from CASES


def _dist_worker(rank, world, port, backend, q):
    import torch.distributed as dist
    from sboxgates_b200.distributed import DistributedLutSearch
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = rank if backend == "nccl" else 0
    if backend == "nccl":
        torch.cuda.set_device(dev)
    dist.init_process_group(backend, rank=rank, world_size=world)
    eng = sb.LutEngine(dev)
    try:
        drv = DistributedLutSearch(eng)
        out = []
        for case in DIST_CASES:
            width, (tabs, tgt, mask, inb), orders = _case_state(case)
            eng.load(tabs, tgt, mask, inb)
            if width == 3:
                e = drv.enumerate3(orders[0], 7)
            elif width == 5:
                e = drv.enumerate5(orders[1], 7)
            else:
                e = drv.enumerate7(orders[2], orders[3], 7)
            t = e.total
            page = drv.fetch_matches(t // 3, 40)
            ranks = np.random.RandomState(case).randint(0, t, 60)
            pick = drv.pick_matches(ranks)
            sample = drv.sample_matches(e, min(t, 25), seed=case)
            out.append((e.total, e.feasible, e.matches.tobytes(), page.tobytes(), pick.tobytes(),
                        sample[0].tolist(), sample[1].tobytes()))
        q.put((rank, out, drv.collectives))
    finally:
        eng.close()
        dist.destroy_process_group()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _spawn(world, backend, worker=_dist_worker):
    """Runs worker(rank, world, port, backend, queue) in `world` processes; returns what each put
    on the queue."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=worker, args=(r, world, port, backend, q))
             for r in range(world)]
    for p in procs:
        p.start()
    try:
        got = [q.get(timeout=600) for _ in range(world)]
    finally:
        for p in procs:
            p.join(timeout=120)
            if p.is_alive():
                p.kill()
                p.join()
    assert all(p.exitcode == 0 for p in procs)
    return got


def _single(engine):
    out = []
    for case in DIST_CASES:
        width, (tabs, tgt, mask, inb), orders = _case_state(case)
        engine.load(tabs, tgt, mask, inb)
        e = _run(engine, width, orders, 7)
        t = e.total
        page = engine.fetch_matches(t // 3, 40)
        pick = engine.pick_matches(np.random.RandomState(case).randint(0, t, 60))
        sample = sb.sample_matches(engine, e, min(t, 25), seed=case)
        out.append((e.total, e.feasible, e.matches.tobytes(), page.tobytes(), pick.tobytes(),
                    sample[0].tolist(), sample[1].tobytes()))
    return out


@pytest.mark.parametrize("world", [2, 3])
def test_distributed_enumeration_gloo(engine, world):
    want = _single(engine)
    for rank, out, collectives in _spawn(world, "gloo"):
        assert out == want, rank
        # per enumeration: 2 gathers + 1 all-reduce (first K); then page, pick, sample: 1 each
        assert collectives == len(DIST_CASES) * 6, rank


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_distributed_enumeration_nccl(engine):
    want = _single(engine)
    for rank, out, _ in _spawn(2, "nccl"):
        assert out == want, rank
