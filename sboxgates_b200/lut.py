"""Host-side mirror of the reference's LUT-search interface (lut.h:28-58) on top of the CUDA
library.

`search_5lut` / `search_7lut` take what the reference functions take -- the gate truth tables of
the state, target, mask, the used input bits -- plus the RNG the reference keeps as a static
(sboxgates.c:246-268), and return `(found, ret)` with `ret` the 10-entry array the reference fills
(lut.c:202-211, 453-462).  RNG consumption matches the reference call for call.
"""
import ctypes as C
from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

from . import native
from .native import (SbgResult, SbgJob, SbgNodeResult, NativeLibraryError, SBG_KEY_NONE,
                     SBG_LIST_CAP, SBG_DO_SCAN3, SBG_DO_SEARCH5, SBG_DO_SEARCH7, MATCH_DTYPE,
                     SBG_ENUM_MAX_MATCHES, SBG_MAX_GATES, SBG_MAX_DEPTH, SBG_DEPTH_BINS,
                     SBG_ENUM7_ALL_MAX_GATES, SBG_SHAPE_TREE, SBG_SHAPE_CHAIN, SBG_SHAPE_SHARED)

NO_GATE = 0xFFFF  # state.h:30


@dataclass
class SearchResult:
    found: bool
    ret: List[int]                 # the reference's ret[10]
    ordering: int = -1
    key: int = SBG_KEY_NONE
    index: int = 0
    tuples_feasible: int = 0
    tuples_swept: int = 0
    stale_outer: bool = False
    gates: List[int] = field(default_factory=list)
    pos_outer: int = 0             # position of func_outer / func_middle in the shuffled orders
    pos_middle: int = 0


@dataclass
class Enumeration:
    """The matches of one search state (sbg_enum3 / sbg_enum5 / sbg_enum7): `total` = how many there
    are in the share (None if the count was skipped), `feasible` = feasible triples met (= the
    matches counted) / feasible 5-combinations met / length of the 7-LUT list, `matches` = the
    first min(max_matches, total) of them in ascending key order (the
    reference's enumeration order), a structured array of dtype MATCH_DTYPE."""
    total: Optional[int]
    feasible: int
    matches: np.ndarray


def shuffled_order(rng):
    """lut.c:125-135: Fisher-Yates over 0..255, one draw per element (256 draws)."""
    order = list(range(256))
    for i in range(256):
        j = rng.next() % (i + 1)
        order[i], order[j] = order[j], order[i]
    return bytes(order)


def shuffled_orders7(rng):
    """lut.c:362-378: outer and middle orders, draws interleaved (512 draws)."""
    outer = list(range(256))
    middle = list(range(256))
    for i in range(256):
        oj = rng.next() % (i + 1)
        mj = rng.next() % (i + 1)
        outer[i], outer[oj] = outer[oj], outer[i]
        middle[i], middle[mj] = middle[mj], middle[i]
    return bytes(outer), bytes(middle)


def _u64(a):
    a = np.ascontiguousarray(a, dtype=np.uint64)
    return a, a.ctypes.data_as(native.u64p)


def _rank_array(ranks):
    """The ranks of a pick or group-sizes call, checked: a contiguous 1-D uint64 array of at most
    SBG_ENUM_MAX_MATCHES non-negative integers."""
    r = np.asarray(ranks)
    if r.ndim != 1 or (r.size > 0 and r.dtype.kind not in "iu"):
        raise ValueError("ranks must be a 1-D integer array")
    if r.shape[0] > SBG_ENUM_MAX_MATCHES:
        raise ValueError("at most %d ranks per call" % SBG_ENUM_MAX_MATCHES)
    if r.size > 0 and r.dtype.kind == "i" and int(r.min()) < 0:
        raise ValueError("ranks must not be negative")
    return np.ascontiguousarray(r, dtype=np.uint64)


def _order_ptr(order):
    buf = (C.c_uint8 * 256).from_buffer_copy(bytes(order))
    return buf


def ordering_row(width, k):
    lib = native.load_library()
    row = (C.c_int * width)()
    if lib.sbg_ordering_row(width, k, row) != 0:
        raise ValueError("bad ordering (%d, %d)" % (width, k))
    return [int(x) for x in row]


def chain_row(k):
    """Row k (0..209) of the 7-LUT chain L3(L2(L1(a,b,c), d, e), f, g) (sbg_chain_row): the
    combination's positions in record order a..g.  k = 6 j + q: j = L1's position triple, q = the
    pair {d, e} among the other four, both in lexicographic order."""
    lib = native.load_library()
    row = (C.c_int * 7)()
    if lib.sbg_chain_row(int(k), row) != 0:
        raise ValueError("bad chain row %r" % (k,))
    return [int(x) for x in row]


def shared_row(k):
    """Row k (0..11) of the shared-input two-LUT circuit L2(L1(a,b,c), u, v) (sbg_shared_row): the
    4-combination's positions in record order a, b, c, u, v.  k = 3 j + q: j = the position of d,
    the gate L1 does not read; q = the index of the shared gate s among L1's three positions;
    (u, v) = {s, d} ascending."""
    lib = native.load_library()
    row = (C.c_int * 5)()
    if lib.sbg_shared_row(int(k), row) != 0:
        raise ValueError("bad shared-input row %r" % (k,))
    return [int(x) for x in row]


def lut_table(func, in1, in2, in3):
    """generate_lut_ttable (state.c:202-230)."""
    lib = native.load_library()
    _, p1 = _u64(in1)
    _, p2 = _u64(in2)
    _, p3 = _u64(in3)
    out = np.zeros(4, dtype=np.uint64)
    lib.sbg_lut_table(func, p1, p2, p3, out.ctypes.data_as(native.u64p))
    return out


def solve_inner(in1, in2, in3, target, mask):
    """get_lut_function without the random fill (lut.c:79-103): (ok, func, seen)."""
    lib = native.load_library()
    arrs = [_u64(x) for x in (in1, in2, in3, target, mask)]
    f = C.c_uint8()
    s = C.c_uint8()
    ok = lib.sbg_solve_inner(*[a[1] for a in arrs], C.byref(f), C.byref(s))
    return bool(ok), f.value, s.value


class LutEngine:
    """One CUDA device's search engine (an `sbg_handle`)."""

    def __init__(self, device=0, stream=None):
        self.lib = native.load_library()
        self._h = C.c_void_p()
        rc = self.lib.sbg_create(C.byref(self._h), int(device))
        if rc != 0:
            msg = self.lib.sbg_last_error(self._h).decode() if self._h else "sbg_create failed"
            if self._h:
                self.lib.sbg_destroy(self._h)
                self._h = C.c_void_p()
            raise NativeLibraryError("sbg_create(device=%d): %s" % (device, msg))
        self.device = device
        self.n = 0              # gates of the current problem (the current slot's)
        self._cur = 0
        self._slot_n = {}
        if stream is not None:
            self.set_stream(stream)

    def close(self):
        if getattr(self, "_h", None):
            self.lib.sbg_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError("sboxgates_b200: %s (code %d)"
                               % (self.lib.sbg_last_error(self._h).decode(), rc))

    def set_stream(self, cuda_stream_ptr):
        self._check(self.lib.sbg_set_stream(self._h, C.c_void_p(cuda_stream_ptr)))

    @property
    def launches(self):
        return int(self.lib.sbg_launch_count(self._h))

    def kernel_ms(self, which):
        return float(self.lib.sbg_last_kernel_ms(self._h, which))

    def set_timing(self, on):
        """Kernel-family timing (CUDA events inside the chains; off by default)."""
        self._check(self.lib.sbg_set_timing(self._h, 1 if on else 0))

    def transfer_stats(self):
        """(h2d bytes, d2h bytes, bulk uploads, incremental uploads, unchanged states) so far."""
        out = (C.c_uint64 * 5)()
        self._check(self.lib.sbg_transfer_stats(self._h, out))
        return [int(x) for x in out]

    def alu_peak(self):
        """Measured LOP3 issue rate of the device, warp instructions per second."""
        v = C.c_double()
        self._check(self.lib.sbg_alu_peak(self._h, C.byref(v)))
        return float(v.value)

    # -- problem -------------------------------------------------------------------------------
    def load(self, tables, target, mask, inbits):
        tables, tp = _u64(tables)
        if tables.ndim != 2 or tables.shape[1] != 4:
            raise ValueError("tables must have shape (n, 4)")
        target, gp = _u64(target)
        mask, mp = _u64(mask)
        ib = np.full(8, -1, dtype=np.int8)
        ib[:len(inbits)] = inbits
        self.n = tables.shape[0]
        self._slot_n[0] = self.n
        self._cur = 0
        self._check(self.lib.sbg_load_problem(self._h, tp, self.n, gp, mp,
                                              ib.ctypes.data_as(native.i8p)))

    def stage(self, slot, tables, target, mask, inbits):
        """Uploads a search state into device-resident slot `slot` without selecting it."""
        tables, tp = _u64(tables)
        target, gp = _u64(target)
        mask, mp = _u64(mask)
        ib = np.full(8, -1, dtype=np.int8)
        ib[:len(inbits)] = inbits
        self._check(self.lib.sbg_stage_problem(self._h, slot, tp, tables.shape[0], gp, mp,
                                               ib.ctypes.data_as(native.i8p)))
        self._staged(slot, tables.shape[0])

    def _staged(self, slot, n):
        self._slot_n[slot] = n
        if slot == self._cur:   # restaging the current slot changes the current problem
            self.n = n

    def prepare_state(self, tables, target, mask, inbits):
        """Marshals a state's host buffers once (numpy -> pointers) for stage_prepared: a caller that
        stages the same host arrays repeatedly, or wants the marshalling out of a timed region."""
        tables, tp = _u64(tables)
        target, gp = _u64(target)
        mask, mp = _u64(mask)
        ib = np.full(8, -1, dtype=np.int8)
        ib[:len(inbits)] = inbits
        return (tables, tp, target, gp, mask, mp, ib, ib.ctypes.data_as(native.i8p),
                int(tables.shape[0]))

    def stage_prepared(self, slot, prep):
        """stage() on the result of prepare_state (which keeps the host buffers alive)."""
        self._check(self.lib.sbg_stage_problem(self._h, slot, prep[1], prep[8], prep[3], prep[5],
                                               prep[7]))
        self._staged(slot, prep[8])

    def use(self, slot):
        self._check(self.lib.sbg_use_problem(self._h, slot))
        self.n = self._slot_n[slot]
        self._cur = slot

    # -- whole searches ------------------------------------------------------------------------
    def search5(self, func_order):
        res = SbgResult()
        self._check(self.lib.sbg_search5(self._h, _order_ptr(func_order), C.byref(res)))
        return res

    def search7(self, outer_order, middle_order):
        res = SbgResult()
        self._check(self.lib.sbg_search7(self._h, _order_ptr(outer_order),
                                         _order_ptr(middle_order), C.byref(res)))
        return res

    def search7_chain(self, outer_order, middle_order):
        """The first 7-LUT chain L3(L2(L1(a,b,c), d, e), f, g) over the 7-LUT list search7 tries
        (sbg_search7_chain; the installed list of the current problem, else phase 1 runs and
        installs it): an SbgResult with key idx << 24 | k << 16 | po << 8 | pm, ordering = the chain
        row k, gates a..g in chain-row order and L3's solved bits (see chain_result_luts)."""
        res = SbgResult()
        self._check(self.lib.sbg_search7_chain(self._h, _order_ptr(outer_order),
                                               _order_ptr(middle_order), C.byref(res)))
        return res

    def search4_shared(self, func_order):
        """The first shared-input two-LUT circuit L2(L1(a,b,c), u, v), {u, v} = {s, d} with s one
        of a, b, c, over every 4-combination (sbg_search4_shared): an SbgResult laid out as a
        search5 result (gates a, b, c, u, v; key rank << 12 | k << 8 | po, ordering = the
        shared_row k), so result5_to_ret applies L2's fill to it."""
        res = SbgResult()
        self._check(self.lib.sbg_search4_shared(self._h, _order_ptr(func_order), C.byref(res)))
        return res

    # -- one call per node / batches of nodes --------------------------------------------------
    @staticmethod
    def _job(slot, order5=None, outer=None, middle=None, gate_order=None):
        """Builds an SbgJob; returns (job, keepalive buffers)."""
        job = SbgJob()
        keep = []
        job.slot = slot
        flags = 0
        if gate_order is not None:
            go = (C.c_uint16 * len(gate_order))(*[int(g) for g in gate_order])
            keep.append(go)
            job.gate_order = C.cast(go, C.POINTER(C.c_uint16))
            flags |= SBG_DO_SCAN3
        if order5 is not None:
            b = _order_ptr(order5)
            keep.append(b)
            job.order5 = C.cast(b, C.POINTER(C.c_uint8))
            flags |= SBG_DO_SEARCH5
        if outer is not None:
            bo, bm = _order_ptr(outer), _order_ptr(middle)
            keep += [bo, bm]
            job.outer7 = C.cast(bo, C.POINTER(C.c_uint8))
            job.middle7 = C.cast(bm, C.POINTER(C.c_uint8))
            flags |= SBG_DO_SEARCH7
        job.flags = flags
        return job, keep

    def search_node(self, slot=0, order5=None, outer=None, middle=None, gate_order=None):
        """scan3 -> search_5lut -> search_7lut of one staged state as one device call chain."""
        job, keep = self._job(slot, order5, outer, middle, gate_order)
        res = SbgNodeResult()
        self._check(self.lib.sbg_search_node(self._h, C.byref(job), C.byref(res)))
        self.n = self._slot_n.get(slot, self.n)   # the node's slot is now the current problem
        self._cur = slot
        return res

    def search_batch(self, jobs):
        """jobs: list of dicts with keys slot, order5, outer, middle, gate_order (any may be absent).
        Returns the list of SbgNodeResult, one per job."""
        arr = (SbgJob * len(jobs))()
        keep = []
        for i, j in enumerate(jobs):
            job, k = self._job(j.get("slot", 0), j.get("order5"), j.get("outer"), j.get("middle"),
                               j.get("gate_order"))
            arr[i] = job
            keep.append(k)
        res = (SbgNodeResult * len(jobs))()
        self._check(self.lib.sbg_search_batch(self._h, len(jobs), arr, res))
        return list(res)

    def prepare_jobs(self, jobs):
        """The job array of search_batch, built once: (array, keep-alive buffers, count)."""
        arr = (SbgJob * len(jobs))()
        keep = []
        for i, j in enumerate(jobs):
            job, k = self._job(j.get("slot", 0), j.get("order5"), j.get("outer"), j.get("middle"),
                               j.get("gate_order"))
            arr[i] = job
            keep.append(k)
        return arr, keep, len(jobs)

    def search_batch_prepared(self, prepared):
        """search_batch on the result of prepare_jobs."""
        arr, _, count = prepared
        res = (SbgNodeResult * count)()
        self._check(self.lib.sbg_search_batch(self._h, count, arr, res))
        return list(res)

    def list7_device(self):
        """(device pointer, count) of this device's ordered phase-1 list."""
        ptr = C.c_void_p()
        cnt = C.c_int()
        self._check(self.lib.sbg_list7_device(self._h, C.byref(ptr), C.byref(cnt)))
        return ptr.value, cnt.value

    def set_list7_device(self, dev_ptr, stride, counts):
        """Merges ascending runs already in device memory (run r at dev_ptr + 8 * r * stride)."""
        arr = (C.c_int * len(counts))(*[int(c) for c in counts])
        self._check(self.lib.sbg_set_list7_device(self._h, C.c_void_p(dev_ptr), int(stride), arr,
                                                  len(counts)))

    # -- sharded building blocks ---------------------------------------------------------------
    def search5_part(self, part, nparts, func_order):
        key = C.c_uint64()
        self._check(self.lib.sbg_search5_part(self._h, part, nparts, _order_ptr(func_order),
                                              C.byref(key)))
        return key.value

    def finish5(self, key, func_order):
        res = SbgResult()
        self._check(self.lib.sbg_finish5(self._h, key, _order_ptr(func_order), C.byref(res)))
        return res

    def filter7_part(self, part, nparts):
        out = np.zeros(SBG_LIST_CAP, dtype=np.uint64)
        cnt = C.c_int()
        self._check(self.lib.sbg_filter7_part(self._h, part, nparts,
                                              out.ctypes.data_as(native.u64p), C.byref(cnt)))
        return out[:cnt.value].copy()

    def filter7_part_device(self, part, nparts):
        """Phase 1 of this part; the ordered list stays on the device.  Returns its length."""
        cnt = C.c_int()
        self._check(self.lib.sbg_filter7_part(self._h, part, nparts, None, C.byref(cnt)))
        return cnt.value

    def filter7_keep_local(self):
        """Phase 1 over the whole space on this device; the sorted, capped list stays in HBM as the
        installed list.  Returns its length."""
        cnt = C.c_int()
        self._check(self.lib.sbg_filter7_part(self._h, 0, 1, None, C.byref(cnt)))
        return cnt.value

    def set_list7(self, packed):
        packed, pp = _u64(packed)
        self._check(self.lib.sbg_set_list7(self._h, pp, int(packed.shape[0])))

    def decomp7_part(self, part, nparts, outer_order, middle_order):
        key = C.c_uint64()
        self._check(self.lib.sbg_decomp7_part(self._h, part, nparts, _order_ptr(outer_order),
                                              _order_ptr(middle_order), C.byref(key)))
        return key.value

    def finish7(self, key, outer_order, middle_order):
        res = SbgResult()
        self._check(self.lib.sbg_finish7(self._h, key, _order_ptr(outer_order),
                                         _order_ptr(middle_order), C.byref(res)))
        return res

    # -- enumeration ---------------------------------------------------------------------------
    def _enumerate(self, fn, orders, max_matches, count, part, nparts):
        max_matches = int(max_matches)
        if not 0 <= max_matches <= SBG_ENUM_MAX_MATCHES:
            raise ValueError("max_matches must lie in 0..%d" % SBG_ENUM_MAX_MATCHES)
        out = np.zeros(max(max_matches, 1), dtype=MATCH_DTYPE)
        n_out, total, feasible = C.c_uint64(), C.c_uint64(), C.c_uint64()
        # function orders as 256 bytes; a ctypes array (the gate order) as it is
        bufs = [o if isinstance(o, C.Array) else _order_ptr(o) for o in orders]
        self._check(fn(self._h, part, nparts, *bufs, max_matches, out.ctypes.data_as(C.c_void_p),
                       C.byref(n_out), C.byref(total) if count else None, C.byref(feasible)))
        return Enumeration(int(total.value) if count else None, int(feasible.value),
                           out[:n_out.value].copy())

    def enumerate5(self, func_order, max_matches, count=True, part=0, nparts=1):
        """Every match of search_5lut on the current problem: the total (count=True) and the first
        max_matches in key order.  count=False may stop as soon as those are known."""
        return self._enumerate(self.lib.sbg_enum5, [func_order], max_matches, count, part, nparts)

    def enumerate7(self, outer_order, middle_order, max_matches, count=True, part=0, nparts=1):
        """The same for search_7lut, over the installed phase-1 list (run here if there is none)."""
        return self._enumerate(self.lib.sbg_enum7, [outer_order, middle_order], max_matches, count,
                               part, nparts)

    def enumerate7_all(self, outer_order, middle_order, max_matches, count=True, part=0,
                       nparts=1):
        """The same over every 7-combination of the problem instead of the phase-1 list
        (sbg_enum7_all, 7 <= n <= SBG_ENUM7_ALL_MAX_GATES): keys rank << 23 | k << 16 | po << 8 | pm
        with the combination's rank among all C(n, 7), records as enumerate7's, and `feasible` =
        the feasible combinations, which the list's cap hides.  The installed list stays."""
        return self._enumerate(self.lib.sbg_enum7_all, [outer_order, middle_order], max_matches,
                               count, part, nparts)

    def enumerate7_chain(self, outer_order, middle_order, max_matches, count=True, part=0,
                         nparts=1):
        """The 7-LUT realisations wired as a chain L3(L2(L1(a,b,c), d, e), f, g), which search_7lut
        never tries (sbg_enum7_chain), over the combinations enumerate7_all takes: keys rank << 24 |
        k << 16 | po << 8 | pm with k a chain_row, L1 = outer_order[po], L2 = middle_order[pm], and
        records of shape SBG_SHAPE_CHAIN (see chain_luts).  The installed list stays."""
        return self._enumerate(self.lib.sbg_enum7_chain, [outer_order, middle_order], max_matches,
                               count, part, nparts)

    def enumerate4_shared(self, func_order, max_matches, count=True, part=0, nparts=1):
        """The two-LUT realisations search_5lut never tries, L2(L1(a,b,c), u, v) with {u, v} =
        {s, d} and s one of a, b, c (sbg_enum4_shared), over every 4-combination: keys rank << 12 |
        k << 8 | po with k a shared_row and L1 = func_order[po], records of width 4 and shape
        SBG_SHAPE_SHARED laid out as 5-LUT records (match_to_ret reads them).  The installed 7-LUT
        list stays."""
        return self._enumerate(self.lib.sbg_enum4_shared, [func_order], max_matches, count, part,
                               nparts)

    def enumerate3(self, gate_order, max_matches, count=True, part=0, nparts=1):
        """Every match of lut_search's 3-LUT scan over `gate_order` (a permutation of the current
        problem's gates): the feasible position triples, keys i << 18 | k << 9 | m."""
        go = np.ascontiguousarray(gate_order, dtype=np.uint16)
        if go.ndim != 1 or go.shape[0] != self.n:
            raise ValueError("gate_order must list the problem's %d gates" % self.n)
        buf = (C.c_uint16 * go.shape[0]).from_buffer_copy(go.tobytes())
        return self._enumerate(self.lib.sbg_enum3, [buf], max_matches, count, part, nparts)

    # -- matches at any rank of the last counted enumeration (the cursor) -----------------------
    def fetch_matches(self, first, count):
        """The matches at ranks first .. min(first + count, total) - 1 of the last counted
        enumeration on this engine (ranks within its share, ascending key order), as a MATCH_DTYPE
        array: the same records that enumeration emits at those ranks.  Nothing is counted again.
        Raises RuntimeError if something other than a fetch, a pick or a query ran on the engine
        since that enumeration (the cursor is gone).

        On a global cursor (enum_set_global) the ranks are ranks of the whole and the length is
        the same on every share: this share's records at the ranks it owns, all-zero records
        (width 0) at every other rank.  Summing the shares' outputs as 64-bit words gives the
        whole's records."""
        first, count = int(first), int(count)
        if not 0 <= first < 2**64:
            raise ValueError("first must lie in 0..2**64-1")
        if not 0 <= count <= SBG_ENUM_MAX_MATCHES:
            raise ValueError("count must lie in 0..%d" % SBG_ENUM_MAX_MATCHES)
        out = np.zeros(max(count, 1), dtype=MATCH_DTYPE)
        n_out = C.c_uint64()
        self._check(self.lib.sbg_enum_fetch(self._h, first, count, out.ctypes.data_as(C.c_void_p),
                                            C.byref(n_out)))
        return out[:n_out.value].copy()

    def pick_matches(self, ranks):
        """The matches at the given ranks of the last counted enumeration, in the order of `ranks`
        (a 1-D integer array; any order, repeats allowed, each below the total).

        On a global cursor (enum_set_global) the ranks are ranks of the whole, below the whole's
        total: this share's records at the ranks it owns, all-zero records (width 0) at every other
        slot.  Summing the shares' outputs as 64-bit words gives the whole's records."""
        r = _rank_array(ranks)
        out = np.zeros(max(r.shape[0], 1), dtype=MATCH_DTYPE)
        self._check(self.lib.sbg_enum_pick(self._h, r.ctypes.data_as(native.u64p), r.shape[0],
                                           out.ctypes.data_as(C.c_void_p)))
        return out[:r.shape[0]].copy()

    def group_sizes(self, ranks):
        """The number of matches in the group at each of the given ranks of the last counted
        enumeration, as a numpy uint64 array in the order of `ranks` (checked as pick_matches
        checks them): the matches the ungrouped enumeration, under the same depth and function
        filters, counts with that group's match_group id.  All ones on an ungrouped cursor and for
        enumerate3.  Nothing is counted again but the wanted groups' own matches.

        On a global cursor (enum_set_global): this share's sizes at the ranks it owns, 0 at every
        other slot.  Summing the shares' outputs gives the whole's sizes."""
        r = _rank_array(ranks)
        out = np.zeros(max(r.shape[0], 1), dtype=np.uint64)
        self._check(self.lib.sbg_enum_group_sizes(self._h, r.ctypes.data_as(native.u64p),
                                                  r.shape[0], out.ctypes.data_as(native.u64p)))
        return out[:r.shape[0]].copy()

    # -- global ranks across shares (the cursor of a sharded count) -----------------------------
    def enum_block_count(self):
        """The number of deal blocks of the cursor's share (the length enum_block_sums fills)."""
        nb = C.c_uint64()
        self._check(self.lib.sbg_enum_block_sums(self._h, None, C.byref(nb)))
        return int(nb.value)

    def enum_block_sums(self, out=None):
        """The match count of each deal block of the cursor's share, in local block order.  out=None:
        returns a numpy uint64 array; else out (a contiguous 64-bit torch tensor, CPU or CUDA, with
        at least that many elements) is filled through its data pointer and returned."""
        nb = C.c_uint64()
        n = self.enum_block_count()
        if out is None:
            arr = np.zeros(max(n, 1), dtype=np.uint64)
            if n > 0:
                self._check(self.lib.sbg_enum_block_sums(self._h, arr.ctypes.data_as(C.c_void_p),
                                                         C.byref(nb)))
            return arr[:n]
        if out.element_size() != 8 or not out.is_contiguous() or out.numel() < n:
            raise ValueError("out must be a contiguous 64-bit tensor of at least %d elements" % n)
        if n > 0:
            _torch_stream_done(out)
            self._check(self.lib.sbg_enum_block_sums(self._h, C.c_void_p(out.data_ptr()),
                                                     C.byref(nb)))
        return out

    def enum_set_global(self, sums, counts):
        """Makes the cursor global: `sums` is (nparts, stride) -- row q holds part q's block sums
        in its first counts[q] entries -- as a numpy array or a torch tensor (CPU or CUDA) of
        64-bit integers.  Returns the whole's total; fetch_matches and pick_matches then take
        ranks of the whole."""
        counts = np.ascontiguousarray([int(c) for c in counts], dtype=np.uint64)
        if isinstance(sums, np.ndarray):
            sums = np.ascontiguousarray(sums)
            if sums.ndim != 2 or sums.dtype.itemsize != 8 or sums.dtype.kind not in "iu":
                raise ValueError("sums must be a 2-D array of 64-bit integers")
            ptr, stride = sums.ctypes.data, sums.shape[1]
        else:
            if sums.dim() != 2 or sums.element_size() != 8 or not sums.is_contiguous():
                raise ValueError("sums must be a contiguous 2-D tensor of 64-bit integers")
            ptr, stride = sums.data_ptr(), sums.shape[1]
            _torch_stream_done(sums)
        if sums.shape[0] != counts.shape[0]:
            raise ValueError("sums has %d rows for %d parts" % (sums.shape[0], counts.shape[0]))
        total = C.c_uint64()
        self._check(self.lib.sbg_enum_set_global(self._h, C.c_void_p(ptr), int(stride),
                                                 counts.ctypes.data_as(native.u64p),
                                                 int(counts.shape[0]), C.byref(total)))
        return int(total.value)

    # -- depth filter: the realisations at or below a circuit depth -----------------------------
    def set_depth_filter(self, depth, max_depth):
        """Later enumerate3/5/7 calls keep only the matches of depth <= max_depth, `depth` giving
        the depth of each of the problem's gates (see match_depth).  Ends the cursor.  The
        searches never read the filter."""
        d, max_depth = _depth_args(depth, max_depth)
        buf = (C.c_uint16 * d.shape[0]).from_buffer_copy(d.tobytes())
        self._check(self.lib.sbg_enum_set_depth(self._h, buf, d.shape[0], max_depth))

    def clear_depth_filter(self):
        """Removes the depth filter.  Ends the cursor."""
        self._check(self.lib.sbg_enum_set_depth(self._h, None, 0, 0))

    def depth_counts(self):
        """The cursor's matches per depth (index = depth) as a numpy uint64 array, cut after the
        last non-empty bin.  The cursor must have been counted under a depth filter."""
        out = np.zeros(SBG_DEPTH_BINS, dtype=np.uint64)
        self._check(self.lib.sbg_enum_depth_counts(self._h, out.ctypes.data_as(native.u64p),
                                                   SBG_DEPTH_BINS))
        return _trim(out)

    # -- function filter: the realisations whose LUTs lie in given sets of functions -------------
    def set_function_filter(self, outer=None, middle=None, inner=None):
        """Later enumerate3/5/7 calls keep only the matches whose LUTs lie in the given sets of
        3-input functions (iterables of function numbers 0..255, None = all 256; see
        match_functions_allowed): the outer LUT in `outer` (5- and 7-LUT), the middle LUT in
        `middle` (7-LUT), and the inner LUT completable inside `inner`.  Combines with the depth
        filter.  Ends the cursor.  The searches never read the filter."""
        sets = [_function_set(s, r) for s, r in ((outer, "outer"), (middle, "middle"),
                                                  (inner, "inner"))]
        if all(s is None for s in sets):
            # all three given as None: a filter that keeps everything, i.e. none
            self.clear_function_filter()
            return
        ptrs = [None if s is None else s.ctypes.data_as(native.u64p) for s in sets]
        self._check(self.lib.sbg_enum_set_functions(self._h, *ptrs))

    def clear_function_filter(self):
        """Removes the function filter.  Ends the cursor."""
        self._check(self.lib.sbg_enum_set_functions(self._h, None, None, None))

    # -- grouping: the distinct gate sets and wirings that realise a state -----------------------
    def set_grouping(self, grouping):
        """Later enumerate5/7 calls enumerate groups of matches (see match_group): None = every
        match, "shape" = one per gate set and ordering row (the wiring), "tuple" = one per gate set.
        A group counts if one of its matches passes the depth and function filters, and its record
        is its first match, the ungrouped record of that key; ranks count groups.  enumerate3 is
        unchanged (a 3-LUT key is its own group).  Ends the cursor.  The searches never read it."""
        if grouping not in _GROUPINGS:
            raise ValueError("grouping must be None, 'shape' or 'tuple', not %r" % (grouping,))
        self._check(self.lib.sbg_enum_set_grouping(self._h, _GROUPINGS[grouping]))


def inner_table(inner=None):
    """sbg_inner_table: a uint8 array of 6,561 entries, entry p3(seen) + p3(ones) = 1 iff some
    function of `inner` (None: all 256) has (f & seen) == ones."""
    lib = native.load_library()
    s = _function_set(inner, "inner")
    out = np.zeros(6561, dtype=np.uint8)
    ptr = None if s is None else s.ctypes.data_as(native.u64p)
    if lib.sbg_inner_table(ptr, out.ctypes.data_as(C.POINTER(C.c_uint8))) != 0:
        raise NativeLibraryError("sbg_inner_table failed")
    return out


# -- grouping: the distinct gate sets and wirings that realise a state ---------------------------
_GROUPINGS = {None: native.SBG_GROUP_NONE, "shape": native.SBG_GROUP_SHAPE,
              "tuple": native.SBG_GROUP_TUPLE}
# the key bits below a group's id, per (grouping, width, wiring): positions (shape), then the row
_GROUP_SHIFT = {("shape", 5, "tree"): 8, ("shape", 7, "tree"): 16, ("tuple", 5, "tree"): 12,
                ("tuple", 7, "tree"): 23, ("shape", 7, "chain"): 16, ("tuple", 7, "chain"): 24,
                ("shape", 4, "shared"): 8, ("tuple", 4, "shared"): 12}
# the wiring each width's records may have
_SHAPES = {3: ("tree",), 4: ("shared",), 5: ("tree",), 7: ("tree", "chain")}


def match_group(key, width, grouping, shape="tree"):
    """The id of the group an enumerated match's key belongs to under a grouping (see
    LutEngine.set_grouping): the key itself for None and for width 3, else key >> 8 / key >> 16
    (shape, 5- / 7-LUT) or key >> 12 / key >> 23 (tuple).  shape="chain" reads a key of
    enumerate7_chain (width 7): key >> 16 (shape) or key >> 24 (tuple); shape="shared" a key of
    enumerate4_shared (width 4, the only width with that wiring): key >> 8 (shape) or key >> 12
    (tuple), as a 5-LUT key.  Matches of one group have equal ids; groups come in ascending id
    order."""
    if grouping not in _GROUPINGS:
        raise ValueError("grouping must be None, 'shape' or 'tuple', not %r" % (grouping,))
    if width not in _SHAPES:
        raise ValueError("width must be 3, 4, 5 or 7")
    if shape not in ("tree", "chain", "shared"):
        raise ValueError("shape must be 'tree', 'chain' or 'shared', not %r" % (shape,))
    if shape not in _SHAPES[width]:
        raise ValueError("width %d has no %r wiring" % (width, shape))
    key = int(key)
    if not 0 <= key < 2**64:
        raise ValueError("key must lie in 0..2**64-1")
    if grouping is None or width == 3:
        return key
    return key >> _GROUP_SHIFT[(grouping, width, shape)]


def _depth_args(depth, max_depth):
    """A depth filter's arguments, checked: (uint16 array of the gate depths, bound)."""
    d = np.asarray(depth)
    if d.ndim != 1 or not 1 <= d.shape[0] <= SBG_MAX_GATES:
        raise ValueError("depth must be a 1-D array of 1..%d gate depths" % SBG_MAX_GATES)
    if d.dtype.kind not in "iu":
        raise ValueError("depth must hold integers")
    if int(d.min()) < 0 or int(d.max()) > SBG_MAX_DEPTH:
        raise ValueError("gate depths must lie in 0..%d" % SBG_MAX_DEPTH)
    max_depth = int(max_depth)
    if not 0 <= max_depth < 2**32:
        raise ValueError("max_depth must lie in 0..2**32-1")
    return np.ascontiguousarray(d, dtype=np.uint16), max_depth


def _trim(hist):
    """A histogram without its trailing empty bins."""
    nz = np.flatnonzero(hist)
    return hist[:int(nz[-1]) + 1].copy() if nz.size else hist[:0].copy()


def _is_shared(record):
    """Whether a MATCH_DTYPE record is a shared-input pair (enumerate4_shared)."""
    return int(record["width"]) == 4 and int(record["shape"]) == SBG_SHAPE_SHARED


def match_depth(record, depth):
    """The depth of the gate an enumerated match (a MATCH_DTYPE record) would add, given the depth
    of every gate of the problem: 1 + max(Da, Db, Dc) for a 3-LUT; 1 + max(1 + max(Da, Db, Dc),
    Dd, De) for a 5-LUT (outer LUT over a, b, c); 1 + max(1 + max(Da, Db, Dc), 1 + max(Dd, De, Df),
    Dg) for a 7-LUT (outer over a, b, c, middle over d, e, f); 1 + max(1 + max(1 + max(Da, Db, Dc),
    Dd, De), Df, Dg) for a 7-LUT chain (the record's shape); 1 + max(1 + max(Da, Db, Dc), Du, Dv)
    for a shared-input pair (width 4; gates a, b, c, u, v, one repeated).  Gates in the record's
    order."""
    width = int(record["width"])
    shared = _is_shared(record)
    d = [int(depth[int(g)]) for g in record["gates"][:5 if shared else width]]
    if width == 3:
        return 1 + max(d)
    if width == 5 or shared:
        return 1 + max(1 + max(d[:3]), d[3], d[4])
    if width == 7 and int(record["shape"]) == SBG_SHAPE_CHAIN:
        return 1 + max(1 + max(1 + max(d[:3]), d[3], d[4]), d[5], d[6])
    if width == 7:
        return 1 + max(1 + max(d[:3]), 1 + max(d[3:6]), d[6])
    raise ValueError("not a match record (width %d)" % width)


def shallowest_matches(engine, width, orders, depth, max_matches, whole=False, shape="tree"):
    """The shallowest realisations of the current problem by the width-3, 5 or 7 enumeration:
    one count with the loosest bound gives the depth histogram, a second counts at its first
    non-empty depth.  `orders` are the enumerate call's order arguments: (gate_order,),
    (func_order,) or (outer, middle).  Returns (minimum depth or None, the number of matches at
    it, the first max_matches of them in key order).  The filter stays installed at the minimum
    depth, so the engine's cursor serves the shallowest set (fetch_matches, pick_matches).
    `engine` is a LutEngine or a DistributedLutSearch.  Use it with no grouping or with "shape"
    grouping: under "tuple" grouping a gate set is binned at the depth of its first match, which
    need not be its shallowest.  whole=True (width 7 only) searches every 7-combination
    (enumerate7_all) instead of the phase-1 list, so the result is the state's shallowest 7-LUT
    realisation, not the list's.  shape="chain" (width 7 only) takes the chain realisations of
    enumerate7_chain, which always cover every 7-combination; shape="shared" (width 4, orders
    (func_order,)) the shared-input pairs of enumerate4_shared."""
    if width not in _SHAPES:
        raise ValueError("width must be 3, 4, 5 or 7")
    if whole and width != 7:
        raise ValueError("whole=True applies to width 7 only")
    if shape not in ("tree", "chain", "shared"):
        raise ValueError("shape must be 'tree', 'chain' or 'shared', not %r" % (shape,))
    if shape not in _SHAPES[width]:
        raise ValueError("width %d has no %r wiring" % (width, shape))
    name = ("enumerate7_chain" if shape == "chain" else "enumerate4_shared" if shape == "shared"
            else "enumerate7_all" if whole else "enumerate%d" % width)
    run = getattr(engine, name)
    engine.set_depth_filter(depth, SBG_DEPTH_BINS - 1)
    run(*orders, 0)
    hist = engine.depth_counts()
    if hist.size == 0:
        return None, 0, np.zeros(0, dtype=MATCH_DTYPE)
    dmin = int(np.flatnonzero(hist)[0])
    engine.set_depth_filter(depth, dmin)
    e = run(*orders, max_matches)
    return dmin, int(e.total), e.matches


# -- function filter: the realisations whose LUTs lie in given sets of functions -----------------
# 3-input functions are numbered as for lut_table: bit in1 << 2 | in2 << 1 | in3 of the number is
# the output.  The truth tables of the three inputs in that numbering:
_IN3 = (0xF0, 0xCC, 0xAA)


def _affine_functions():
    out = set()
    for c in range(2):
        for sel in range(8):
            f = 0xFF if c else 0
            for i in range(3):
                if (sel >> i) & 1:
                    f ^= _IN3[i]
            out.add(f)
    return frozenset(out)


AFFINE_FUNCTIONS = _affine_functions()
"""The 16 3-input functions of algebraic degree <= 1: constants, inputs and their XORs, and their
complements (cheap under masking, MPC and FHE)."""


def gate_functions(available_gates):
    """The 3-input functions one two-input gate computes: graph.gate2_table(t, x, y) for a gate
    type t whose bit is set in `available_gates` (the reference's --available-gates bitfield over
    the 16 types of graph.GATE_NAMES) and x, y any of the LUT's three inputs, equal ones included
    (so a gate that passes or inverts an input, or gives a constant, counts as itself).  194 is
    AND, OR and XOR."""
    from .graph import gate2_table
    available_gates = int(available_gates)
    if not 0 <= available_gates < 1 << 16:
        raise ValueError("available_gates must be a 16-bit gate-type bitfield")
    out = set()
    for t in range(16):
        if (available_gates >> t) & 1:
            for x in _IN3:
                for y in _IN3:
                    out.add(gate2_table(t, x, y) & 0xFF)
    return frozenset(out)


def _function_set(funcs, role):
    """A function filter role, checked: None (all 256) or the 4-word uint64 bitmap of a set."""
    if funcs is None:
        return None
    if isinstance(funcs, (str, bytes)):
        raise ValueError("%s must be an iterable of function numbers" % role)
    words = np.zeros(4, dtype=np.uint64)
    for f in funcs:
        if isinstance(f, (bool, np.bool_)) or not isinstance(f, (int, np.integer)):
            raise ValueError("%s: function numbers must be integers, not %r" % (role, f))
        f = int(f)
        if not 0 <= f < 256:
            raise ValueError("%s: function %d outside 0..255" % (role, f))
        words[f >> 6] |= np.uint64(1 << (f & 63))
    return words


def inner_completes(func_inner, inner_seen, f):
    """Whether function f agrees with an inner LUT's solved bits: (f & inner_seen) == func_inner."""
    return (int(f) & int(inner_seen)) == int(func_inner)


def allowed_fill(func_inner, inner_seen, inner=None):
    """The smallest function of `inner` (None: all 256) that completes an inner LUT's solved bits
    (func_inner over the cells inner_seen), or None if none does.  With it a caller builds a circuit
    whose LUTs all lie in the filter's sets; match_to_ret's random fill may leave `inner`."""
    cands = range(256) if inner is None else sorted(int(f) for f in inner)
    for f in cands:
        if inner_completes(func_inner, inner_seen, f):
            return f
    return None


def match_functions_allowed(record, outer=None, middle=None, inner=None):
    """The function filter's test on one enumerated match (a MATCH_DTYPE record), sets as for
    LutEngine.set_function_filter (None: all 256): func_outer in outer (5- and 7-LUT), func_middle
    in middle (7-LUT), and allowed_fill finds an inner function.  A shared-input record (width 4)
    is tested as a 5-LUT one: outer = L1, inner = L2."""
    width = int(record["width"])
    if width not in (3, 5, 7) and not _is_shared(record):
        raise ValueError("not a match record (width %d)" % width)
    if width > 3 and outer is not None and int(record["func_outer"]) not in set(outer):
        return False
    if width == 7 and middle is not None and int(record["func_middle"]) not in set(middle):
        return False
    return allowed_fill(record["func_inner"], record["inner_seen"], inner) is not None


def _torch_stream_done(t):
    """Waits for the work torch has queued on a CUDA tensor's device.  The engine reads or writes
    the tensor on its own stream, which is not ordered after torch's (a zero fill, a collective);
    the engine's calls wait for their own stream before returning."""
    if t.is_cuda:
        import torch
        torch.cuda.current_stream(t.device).synchronize()


def sample_matches(engine, enumeration, k, seed=None):
    """k distinct matches drawn uniformly from the whole match set of `enumeration`, which must be
    the last counted enumeration on `engine` (its cursor): returns (ranks, matches) with the ranks
    ascending and matches[i] the match at ranks[i].  The ranks come from
    numpy.random.default_rng(seed).choice(total, k, replace=False); the reference has no sampling,
    so no xorshift1024 stream is involved and the caller's RNG stays untouched.

    On a global cursor pass the whole's total (enumeration.total): every share draws the same
    ranks from the same seed, and its matches are zero records at the ranks other shares own;
    summed over the shares they are the whole's sample."""
    if enumeration.total is None:
        raise ValueError("the enumeration was not counted (count=False): it has no cursor")
    k, total = int(k), int(enumeration.total)
    if not 0 <= k <= total:
        raise ValueError("k must lie in 0..%d (the enumeration's total)" % total)
    if k > SBG_ENUM_MAX_MATCHES:
        raise ValueError("at most %d matches per sample" % SBG_ENUM_MAX_MATCHES)
    ranks = np.sort(np.random.default_rng(seed).choice(total, k, replace=False)).astype(np.uint64)
    return ranks, engine.pick_matches(ranks)


def unpack_tuple7(packed):
    """63-bit packed 7-combination -> list of gate numbers."""
    p = int(packed)
    return [(p >> (9 * (6 - i))) & 0x1FF for i in range(7)]


def pack_tuple7(gates):
    p = 0
    for g in gates:
        p = (p << 9) | int(g)
    return p


def _fill(func_inner, inner_seen, rng):
    """The random don't-care fill of get_lut_function (lut.c:104-106): one draw iff a cell is
    unseen."""
    fi = int(func_inner)
    if inner_seen != 0xFF:
        fi |= (~int(inner_seen) & 0xFF) & (rng.next() & 0xFF)
    return fi


def result5_to_ret(res, rng):
    """sbg_result -> the reference's ret[10] for search_5lut (lut.c:202-211), applying the random
    don't-care fill of get_lut_function (lut.c:104-106)."""
    if not res.found:
        return SearchResult(False, [0] * 10, key=int(res.key), tuples_feasible=int(res.tuples_feasible),
                            tuples_swept=int(res.tuples_swept))
    fi = _fill(res.func_inner, res.inner_seen, rng)
    gates = [int(g) for g in res.gates[:5]]
    ret = [res.func_outer, fi] + gates + [0, 0, 0]
    return SearchResult(True, ret, ordering=res.ordering, key=int(res.key), index=int(res.index),
                        tuples_feasible=int(res.tuples_feasible),
                        tuples_swept=int(res.tuples_swept), gates=gates, pos_outer=int(res.pos_outer))


def result7_to_ret(res, rng):
    """sbg_result -> ret[10] for search_7lut (lut.c:453-462)."""
    if not res.found:
        return SearchResult(False, [0] * 10, key=int(res.key), tuples_feasible=int(res.tuples_feasible),
                            tuples_swept=int(res.tuples_swept))
    fi = _fill(res.func_inner, res.inner_seen, rng)
    gates = [int(g) for g in res.gates[:7]]
    ret = [res.func_outer, res.func_middle, fi] + gates
    return SearchResult(True, ret, ordering=res.ordering, key=int(res.key), index=int(res.index),
                        tuples_feasible=int(res.tuples_feasible),
                        tuples_swept=int(res.tuples_swept), stale_outer=bool(res.stale_outer),
                        gates=gates, pos_outer=int(res.pos_outer), pos_middle=int(res.pos_middle))


def search_5lut(engine, tables, target, mask, inbits, rng):
    """lut.h:46-47.  Returns a SearchResult; `.found`, `.ret` are the reference's outputs."""
    if len(tables) < 5:
        raise ValueError("search_5lut needs at least 5 gates (lut.c:119)")
    order = shuffled_order(rng)
    engine.load(tables, target, mask, inbits)
    return result5_to_ret(engine.search5(order), rng)


def search_7lut(engine, tables, target, mask, inbits, rng):
    """lut.h:54-55."""
    if len(tables) < 7:
        raise ValueError("search_7lut needs at least 7 gates (lut.c:259)")
    # The reference draws its 512 shuffle values after phase 1 (lut.c:362-378); phase 1 itself
    # draws nothing, so drawing them first leaves the RNG stream unchanged.
    outer, middle = shuffled_orders7(rng)
    engine.load(tables, target, mask, inbits)
    return result7_to_ret(engine.search7(outer, middle), rng)


def match_to_ret(match, rng):
    """One enumerated match (a record of Enumeration.matches) -> the reference's ret[10]
    (lut.c:202-211 / 453-462), the don't-care bits of the inner function filled from `rng` as
    get_lut_function would fill them.  A 3-LUT match has no ret[10]: see match_to_lut3.  A
    shared-input match (enumerate4_shared, width 4) has search_5lut's layout [L1, L2, a, b, c, u,
    v, 0, 0, 0], one of u, v repeating one of a, b, c: its LUTs are added as a 5-LUT result's are,
    L1 over (a, b, c), then L2 over (L1, u, v)."""
    if int(match["width"]) == 3:
        raise ValueError("a 3-LUT match has no ret[10]; use match_to_lut3")
    if int(match["shape"]) == SBG_SHAPE_CHAIN:
        raise ValueError("a chain match has no ret[10] (search_7lut's wiring); use chain_luts")
    fi = _fill(match["func_inner"], match["inner_seen"], rng)
    gates = [int(g) for g in match["gates"]]
    if int(match["width"]) == 5 or _is_shared(match):
        return [int(match["func_outer"]), fi] + gates[:5] + [0, 0, 0]
    return [int(match["func_outer"]), int(match["func_middle"]), fi] + gates


def match_to_lut3(match, rng):
    """One enumerated 3-LUT match -> the add_lut call lut_search would make for it (lut.c:510-518):
    (function, gi, gk, gm), the don't-care bits filled from `rng` as get_lut_function fills them
    (one draw iff a cell is unseen)."""
    if int(match["width"]) != 3:
        raise ValueError("not a 3-LUT match (width %d)" % int(match["width"]))
    fi = _fill(match["func_inner"], match["inner_seen"], rng)
    return (fi, int(match["gates"][0]), int(match["gates"][1]), int(match["gates"][2]))


def chain_luts(match, rng_or_fill):
    """One enumerated chain match (enumerate7_chain) -> its three LUTs in the order a circuit
    builder appends them: [(L1, (a, b, c)), (L2, (("new", 0), d, e)), (L3, (("new", 1), f, g))],
    ("new", k) being the k-th LUT of the list (LutSearchResult's convention).  L3 is filled:
    rng_or_fill is either an int, a complete function that agrees with the solved bits (see
    allowed_fill), or an rng whose draw fills the don't-care bits as get_lut_function would (one
    draw iff a cell is unseen)."""
    if int(match["width"]) != 7 or int(match["shape"]) != SBG_SHAPE_CHAIN:
        raise ValueError("not a chain match (width %d, shape %d)"
                         % (int(match["width"]), int(match["shape"])))
    return _chain_luts(match["func_outer"], match["func_middle"], match["func_inner"],
                       match["inner_seen"], match["gates"], rng_or_fill)


def chain_result_luts(res, rng_or_fill):
    """A found chain result (LutEngine.search7_chain, an SbgResult) -> its three LUTs, as
    chain_luts gives them for a match: [(L1, (a, b, c)), (L2, (("new", 0), d, e)),
    (L3, (("new", 1), f, g))], L3 filled from rng_or_fill (an int or an rng, as there)."""
    if not res.found:
        raise ValueError("the chain search found nothing")
    return _chain_luts(res.func_outer, res.func_middle, res.func_inner, res.inner_seen,
                       res.gates, rng_or_fill)


def _chain_luts(func_outer, func_middle, func_inner, inner_seen, gates, rng_or_fill):
    """The three LUTs of a chain L3(L2(L1(a,b,c), d, e), f, g), gates a..g, with L3 filled."""
    if isinstance(rng_or_fill, (int, np.integer)):
        f3 = int(rng_or_fill)
        if not 0 <= f3 < 256 or not inner_completes(func_inner, inner_seen, f3):
            raise ValueError("function %d does not complete the inner LUT" % f3)
    else:
        f3 = _fill(func_inner, inner_seen, rng_or_fill)
    g = [int(x) for x in gates]
    return [(int(func_outer), (g[0], g[1], g[2])),
            (int(func_middle), (("new", 0), g[3], g[4])),
            (f3, (("new", 1), g[5], g[6]))]


def decode_key3(key):
    """3-LUT key -> (i, k, m), the positions of the triple in the gate order."""
    key = int(key)
    return key >> 18, (key >> 9) & 0x1FF, key & 0x1FF


def decode_key5(key):
    """5-LUT key -> (rank of the combination, ordering k, position in the function order)."""
    key = int(key)
    return key >> 12, (key >> 8) & 0xF, key & 0xFF


def decode_key7(key):
    """7-LUT key -> (list index, or the combination's rank for enumerate7_all, ordering k, outer
    position, middle position)."""
    key = int(key)
    return key >> 23, (key >> 16) & 0x7F, (key >> 8) & 0xFF, key & 0xFF


def decode_key7_chain(key):
    """7-LUT chain key (enumerate7_chain) -> (the combination's rank, chain row k, outer position,
    middle position)."""
    key = int(key)
    return key >> 24, (key >> 16) & 0xFF, (key >> 8) & 0xFF, key & 0xFF


def enumerate_5lut(engine, tables, target, mask, inbits, order, max_matches, count=True, part=0,
                   nparts=1):
    """Every realisation of the state by search_5lut's decomposition under the function order
    `order` (an Enumeration).  Consumes no RNG; match_to_ret applies the fill per match."""
    if len(tables) < 5:
        raise ValueError("search_5lut needs at least 5 gates (lut.c:119)")
    engine.load(tables, target, mask, inbits)
    return engine.enumerate5(order, max_matches, count, part, nparts)


def enumerate_7lut(engine, tables, target, mask, inbits, outer, middle, max_matches, count=True,
                   part=0, nparts=1):
    """The same for search_7lut, over the state's phase-1 list (the first SBG_LIST_CAP feasible
    7-combinations), decided on the true gate tables."""
    if len(tables) < 7:
        raise ValueError("search_7lut needs at least 7 gates (lut.c:259)")
    engine.load(tables, target, mask, inbits)
    return engine.enumerate7(outer, middle, max_matches, count, part, nparts)


def enumerate_7lut_all(engine, tables, target, mask, inbits, outer, middle, max_matches,
                       count=True, part=0, nparts=1):
    """The same over every feasible 7-combination of the state, not only the phase-1 list
    (LutEngine.enumerate7_all; at most SBG_ENUM7_ALL_MAX_GATES gates)."""
    if not 7 <= len(tables) <= SBG_ENUM7_ALL_MAX_GATES:
        raise ValueError("the whole-space 7-LUT enumeration takes 7..%d gates"
                         % SBG_ENUM7_ALL_MAX_GATES)
    engine.load(tables, target, mask, inbits)
    return engine.enumerate7_all(outer, middle, max_matches, count, part, nparts)


def enumerate_7lut_chain(engine, tables, target, mask, inbits, outer, middle, max_matches,
                         count=True, part=0, nparts=1):
    """The realisations by the 7-LUT chain L3(L2(L1(a,b,c), d, e), f, g), which search_7lut never
    tries, over every feasible 7-combination (LutEngine.enumerate7_chain; at most
    SBG_ENUM7_ALL_MAX_GATES gates).  Consumes no RNG; chain_luts applies the fill per match."""
    if not 7 <= len(tables) <= SBG_ENUM7_ALL_MAX_GATES:
        raise ValueError("the 7-LUT chain enumeration takes 7..%d gates" % SBG_ENUM7_ALL_MAX_GATES)
    engine.load(tables, target, mask, inbits)
    return engine.enumerate7_chain(outer, middle, max_matches, count, part, nparts)


def enumerate_4lut_shared(engine, tables, target, mask, inbits, order, max_matches, count=True,
                          part=0, nparts=1):
    """The realisations by two LUTs whose L2 reads one of L1's inputs again, L2(L1(a,b,c), u, v)
    with {u, v} = {s, d} and s one of a, b, c, which search_5lut never tries, over every feasible
    4-combination under search_5lut's function order `order` (LutEngine.enumerate4_shared).
    Consumes no RNG; match_to_ret applies the fill per match."""
    if len(tables) < 4:
        raise ValueError("the shared-input two-LUT circuits need at least 4 gates")
    engine.load(tables, target, mask, inbits)
    return engine.enumerate4_shared(order, max_matches, count, part, nparts)


def enumerate_3lut(engine, tables, target, mask, inbits, gate_order, max_matches, count=True,
                   part=0, nparts=1):
    """Every realisation of the state by lut_search's 3-LUT scan over `gate_order` (an
    Enumeration; inbits plays no part, as in the scan).  Consumes no RNG; match_to_lut3 applies
    the fill per match."""
    if len(tables) < 3:
        raise ValueError("the 3-LUT scan needs at least 3 gates")
    engine.load(tables, target, mask, inbits)
    return engine.enumerate3(gate_order, max_matches, count, part, nparts)


def enumerate_lut_search(engine, tables, target, mask, inbits, gate_order, rng, max_matches,
                         count=True, allow5=True, allow7=True):
    """Every realisation of a node by each stage of lut_search (lut.c:489-631):
    {3: Enumeration, 5: Enumeration or None, 7: Enumeration or None}.  Stage 5 and stage 7 get the
    function orders lut_search would use, drawn from a COPY of `rng` in lut_search's sequence
    (order5, then outer / middle); `rng` itself is not advanced.  A stage lut_search would not run
    (allow5 / allow7 = check_num_gates_possible(st, 2 / 3), lut.c:525, 582; too few gates) is None.
    Stage 3 needs n >= 3 (None otherwise); stage 7 runs over the state's phase-1 list."""
    n = len(tables)
    ahead = rng.copy()
    order5 = shuffled_order(ahead) if (allow5 and n >= 5) else None
    outer = middle = None
    if allow5 and allow7 and n >= 7:
        outer, middle = shuffled_orders7(ahead)
    engine.load(tables, target, mask, inbits)
    out = {3: None, 5: None, 7: None}
    if n >= 3:
        out[3] = engine.enumerate3(gate_order, max_matches, count)
    if order5 is not None:
        out[5] = engine.enumerate5(order5, max_matches, count)
    if outer is not None:
        out[7] = engine.enumerate7(outer, middle, max_matches, count)
    return out


@dataclass
class LutSearchResult:
    """What lut_search() would add to the graph (lut.c:489-631): `luts` = the add_lut calls in
    order, each (function, in1, in2, in3) with inputs either gate numbers or ("new", k) = the k-th
    LUT added by this call; `stage` = 3, 5, 7 or 0 (NO_GATE); `shape` = how a stage-7 result wires
    its three LUTs: "tree" (search_7lut's) or "chain" (lut_search(..., chain=True)); a stage-5
    result is "tree" (search_5lut's) or "shared" (lut_search(..., shared=True))."""
    stage: int
    luts: List[tuple] = field(default_factory=list)
    node: object = None
    shape: str = "tree"


def lut_search(engine, tables, target, mask, inbits, gate_order, rng, allow5=True, allow7=True, *,
               shared=False, chain=False):
    """lut.c:489-631 as ONE device call: the 3-LUT scan over the caller's shuffled gate order
    (lut.c:501-523), search_5lut (lut.c:553) and search_7lut (lut.c:593), each only if the earlier
    ones found nothing.  allow5 / allow7 = check_num_gates_possible(st, 2 / 3) (lut.c:525, 582).

    chain=True adds a stage the reference does not have: when search_7lut ran and found nothing,
    the first 7-LUT chain L3(L2(L1(a,b,c), d, e), f, g) over the same list and orders
    (LutEngine.search7_chain), returned as stage 7 with shape "chain" and luts [(L1, a, b, c),
    (L2, ("new", 0), d, e), (L3, ("new", 1), f, g)].  A node without a chain gets exactly the result
    and RNG state of chain=False.

    shared=True adds a stage the reference does not have between search_5lut and search_7lut: when
    search_5lut ran and found nothing, the first two-LUT circuit whose L2 reads one of L1's inputs
    again (LutEngine.search4_shared, under search_5lut's order), returned as stage 5 with shape
    "shared" and luts [(L1, a, b, c), (L2, ("new", 0), u, v)].  search_7lut then does not run, so its
    512 draws do not happen; the device call of the node stops after search_5lut, and search_7lut
    is a call of its own (LutEngine.search7) when the stage finds nothing.  A node without a match
    gets exactly the result and RNG state of shared=False, with or without chain.  Both switches
    are keyword-only, so that a call cannot set one where it meant the other.

    RNG: the reference draws 256 values on entry to search_5lut and 512 before phase 2 of
    search_7lut, plus one per solved LUT with unseen cells (lut.c:104-106; the chain's L3 likewise).
    Which of those happen depends on the stages' outcomes, so the shuffles are computed from a COPY
    of the generator (looking ahead) and the real one is advanced afterwards by exactly what the
    reference would have consumed."""
    n = len(tables)
    ahead = rng.copy()
    order5 = shuffled_order(ahead) if (allow5 and n >= 5) else None
    outer = middle = None
    if allow5 and allow7 and n >= 7:
        outer, middle = shuffled_orders7(ahead)
    engine.load(tables, target, mask, inbits)
    staged = shared and order5 is not None   # search_7lut waits for the shared-input stage
    node = engine.search_node(0, order5, None if staged else outer, None if staged else middle,
                              gate_order)
    if node.found_stage == 3:
        fi = node.func3
        if node.seen3 != 0xFF:
            fi |= (~node.seen3 & 0xFF) & (rng.next() & 0xFF)
        return LutSearchResult(3, [(fi, int(node.gates3[0]), int(node.gates3[1]),
                                    int(node.gates3[2]))], node)
    if order5 is None:
        return LutSearchResult(0, [], node)
    for _ in range(256):
        rng.next()
    if node.found_stage == 5:
        r = result5_to_ret(node.r5, rng).ret
        return LutSearchResult(5, [(r[0], r[2], r[3], r[4]), (r[1], ("new", 0), r[5], r[6])], node)
    if staged:
        res = engine.search4_shared(order5)
        if res.found:
            r = result5_to_ret(res, rng).ret
            return LutSearchResult(5, [(r[0], r[2], r[3], r[4]), (r[1], ("new", 0), r[5], r[6])],
                                   node, shape="shared")
    if outer is None:
        return LutSearchResult(0, [], node)
    for _ in range(512):
        rng.next()
    r7 = engine.search7(outer, middle) if staged else node.r7
    if r7.found:
        r = result7_to_ret(r7, rng).ret
        # lut.c:622-624 nests the outer and middle add_lut calls as arguments of the third; gcc
        # evaluates them right to left, so the MIDDLE LUT is added first (lower gate number)
        return LutSearchResult(7, [(r[1], r[6], r[7], r[8]), (r[0], r[3], r[4], r[5]),
                                   (r[2], ("new", 1), ("new", 0), r[9])], node)
    if chain:
        # the engine still holds this node's list (search_node or search7 installed it)
        res = engine.search7_chain(outer, middle)
        if res.found:
            luts = [(f,) + ins for f, ins in chain_result_luts(res, rng)]
            return LutSearchResult(7, luts, node, shape="chain")
    return LutSearchResult(0, [], node)
