"""CPU: DistributedLutSearch's enumeration over gloo, world 2 and 3, with an oracle-backed stand-in
engine that deals shares, block sums, global cursors and zero-record fetch and pick the way the
library does (include/sboxgates_b200.h, "global ranks across shares").  Also: the header declares
sbg_enum_block_sums / sbg_enum_set_global and native.SIGNATURES binds them as declared."""
import ctypes as C
import math
import os
import re
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import _enum_support as E
import _support as S
import sboxgates_b200 as sb
from sboxgates_b200 import native
from sboxgates_b200.distributed import DistributedLutSearch
from test_distributed_cpu import OracleEngine
from test_enum_fetch_gpu import _planted

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEAL = 16


def _pair_rank(n, i, k):
    return i * (2 * n - i - 1) // 2 + (k - i - 1)


class GlobalOracleEngine(OracleEngine):
    """The enumeration part of LutEngine on the CPU oracle's whole match list.  A record holds the
    key and the width only.  feasible: the whole's on part 0, 0 on the others (what matters here
    is that the driver sums them)."""

    def _enum(self, width, keys, feasible, k, part, nparts):
        keys = np.asarray(keys, dtype=np.uint64)
        n = self.n
        if width == 3:
            blk = np.array([_pair_rank(n, int(x) >> 18, (int(x) >> 9) & 0x1FF) // DEAL
                            for x in keys], dtype=np.int64)
            blocks = -(-math.comb(n, 2) // DEAL)
        elif width == 5:
            blk = np.array([E.comb_rank(n - 2, 3, E.nth_comb(n, 5, int(x) >> 12)[:3]) // DEAL
                            for x in keys], dtype=np.int64)
            blocks = -(-math.comb(n - 2, 3) // DEAL)
        else:
            blk = (keys >> np.uint64(23)).astype(np.int64)
            blocks = len(self.list)
        self.whole = np.zeros(len(keys), dtype=sb.MATCH_DTYPE)
        self.whole["key"] = keys
        self.whole["width"] = width
        self.blk, self.blocks, self.part, self.nparts = blk, blocks, part, nparts
        self.mine = blk % nparts == part
        self.share = self.whole[self.mine]
        self.glob = False
        return sb.Enumeration(len(self.share), feasible if part == 0 else 0, self.share[:k].copy())

    def enumerate3(self, order, k, count=True, part=0, nparts=1):
        _, keys = E.enum3_range(self.tables, self.target, self.mask, order, 1 << 20)
        return self._enum(3, keys, len(keys), k, part, nparts)

    def enumerate5(self, order, k, count=True, part=0, nparts=1):
        _, keys, feas = E.oracle_enum5(self.tables, self.target, self.mask, self.inbits, order,
                                       1 << 20)
        return self._enum(5, keys, feas, k, part, nparts)

    def enumerate7(self, outer, middle, k, count=True, part=0, nparts=1):
        _, keys = E.oracle_enum7(self.tables, self.target, self.mask, E.unpack_list(self.list),
                                 outer, middle, 1 << 20)
        return self._enum(7, keys, len(self.list), k, part, nparts)

    def _share_blocks(self, q):
        return -(-(self.blocks - q) // self.nparts) if self.blocks > q else 0

    def enum_block_count(self):
        return self._share_blocks(self.part)

    def enum_block_sums(self, out=None):
        nb = self.enum_block_count()
        sums = np.bincount(self.blk[self.mine] // self.nparts, minlength=nb).astype(np.uint64)
        if out is None:
            return sums
        out[:nb] = torch.from_numpy(sums.view(np.int64))
        return out

    def enum_set_global(self, sums, counts):
        sums = np.asarray(sums).view(np.uint64)
        if len(counts) != self.nparts or \
                any(int(c) != self._share_blocks(q) for q, c in enumerate(counts)):
            raise RuntimeError("bad counts")
        if not np.array_equal(sums[self.part, :counts[self.part]], self.enum_block_sums()):
            raise RuntimeError("own row differs")
        self.glob = True
        return int(sum(int(sums[q, :c].sum()) for q, c in enumerate(counts)))

    def _owned(self, ranks):
        recs = self.whole[ranks].copy()
        recs[~self.mine[ranks]] = np.zeros(1, dtype=sb.MATCH_DTYPE)
        return recs

    def fetch_matches(self, first, count):
        src = self.whole if self.glob else self.share
        hi = min(first + count, len(src))
        if first >= hi:
            return np.zeros(0, dtype=sb.MATCH_DTYPE)
        return self._owned(np.arange(first, hi)) if self.glob else self.share[first:hi].copy()

    def pick_matches(self, ranks):
        ranks = np.asarray(ranks, dtype=np.int64)
        return self._owned(ranks) if self.glob else self.share[ranks].copy()


def _state(width, seed):
    """A planted state (a circuit of `width` gates realises the target) with matches to deal."""
    n, spec = {3: (12, 2), 5: (10, 1), 7: (10, 0)}[width]
    return _planted(n, spec, [], seed, width)


def _orders(seed, n):
    o5, outer, middle = E.orders(seed)
    return [int(x) for x in np.random.RandomState(seed).permutation(n)], o5, outer, middle


def _calls(drv_or_eng, width, orders, k):
    if width == 3:
        return drv_or_eng.enumerate3(orders[0], k)
    if width == 5:
        return drv_or_eng.enumerate5(orders[1], k)
    return drv_or_eng.enumerate7(orders[2], orders[3], k)


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        drv = DistributedLutSearch(GlobalOracleEngine())
        out = []
        for width in (3, 5, 7):
            tabs, tgt, mask, inb = _state(width, 30 + width)
            drv.engine.load(tabs, tgt, mask, inb)
            e = _calls(drv, width, _orders(40 + width, len(tabs)), 5)
            t = e.total
            page = drv.fetch_matches(t // 3, 20)
            pick = drv.pick_matches(np.random.RandomState(width).randint(0, t, 30))
            ranks, sample = drv.sample_matches(e, min(t, 10), seed=width)
            out.append((t, e.feasible, e.matches["key"].tolist(), page["key"].tolist(),
                        pick["key"].tolist(), ranks.tolist(), sample["key"].tolist()))
        q.put((rank, out, drv.collectives))
    finally:
        dist.destroy_process_group()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _expected():
    want = []
    for width in (3, 5, 7):
        tabs, tgt, mask, inb = _state(width, 30 + width)
        orders = _orders(40 + width, len(tabs))
        if width == 3:
            _, keys = E.enum3_range(tabs, tgt, mask, orders[0], 1 << 20)
            feas = len(keys)
        elif width == 5:
            _, keys, feas = E.oracle_enum5(tabs, tgt, mask, inb, orders[1], 1 << 20)
        else:
            lst, _ = S.oracle_filter7(tabs, tgt, mask, inb)
            _, keys = E.oracle_enum7(tabs, tgt, mask, np.asarray(lst, dtype=np.uint16).reshape(-1, 7),
                                     orders[2], orders[3], 1 << 20)
            feas = len(lst)
        keys = [int(x) for x in keys]
        t = len(keys)
        assert t > 0, width
        pick = np.random.RandomState(width).randint(0, t, 30)
        ranks = np.sort(np.random.default_rng(width).choice(t, min(t, 10), replace=False))
        want.append((t, feas, keys[:5], keys[t // 3:t // 3 + 20], [keys[r] for r in pick],
                     ranks.tolist(), [keys[r] for r in ranks]))
    return want


@pytest.mark.parametrize("world", [2, 3])
def test_distributed_enumeration_equals_the_oracle(world):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        got = [q.get(timeout=300) for _ in range(world)]
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
                p.join()
    assert all(p.exitcode == 0 for p in procs)
    want = _expected()
    for rank, out, collectives in got:
        assert out == want, rank
        # per enumeration: (blocks, feasible) gather, block-sum gather, first-K all-reduce; then
        # one all-reduce each for the page, the pick and the sample
        assert collectives == 3 * 6, rank


def test_header_declares_block_sums_and_set_global():
    with open(os.path.join(ROOT, "include", "sboxgates_b200.h")) as f:
        text = re.sub(r"\s+", " ", f.read())
    assert "int sbg_enum_block_sums(sbg_handle *h, uint64_t *out, uint64_t *nblocks);" in text
    assert ("int sbg_enum_set_global(sbg_handle *h, const uint64_t *sums, uint64_t stride, "
            "const uint64_t *counts, int nparts, uint64_t *total);") in text


def test_bindings_match_the_declarations():
    u64p = C.POINTER(C.c_uint64)
    assert native.SIGNATURES["sbg_enum_block_sums"] == (C.c_int, [C.c_void_p, C.c_void_p, u64p])
    assert native.SIGNATURES["sbg_enum_set_global"] == (
        C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, u64p, C.c_int, u64p])
    lib = native.load_library()
    assert lib.sbg_enum_block_sums.restype is C.c_int
    assert lib.sbg_enum_set_global.argtypes[2] is C.c_uint64
