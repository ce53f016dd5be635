"""Multi-GPU search: one process per GPU, `torch.distributed` for the plumbing.

The reference parallelises search_5lut / search_7lut over MPI ranks with a master/worker protocol
(lut.c:137-159, 212-238, 329-360, 463-482, 664-740; sboxgates.c:619-642): contiguous slices of the
combination space, first finder wins.  Here every rank runs the same host program with the same
RNG state, takes an interleaved share of the work items, and the ranks agree on the answer with
  * search_5lut: one all-reduce(MIN) of the 64-bit key (rank of combination, ordering, position);
  * search_7lut: one all-gather of the per-rank hit lists (phase 1, lut.c:329-349), then one
    all-reduce(MIN) of the key (list index, ordering, outer position, middle position).
Because the key orders candidates exactly as the reference's single-rank loop visits them, the
result is the reference's size == 1 result for any number of GPUs.

Enumeration (enumerate3/5/7, fetch_matches, pick_matches, sample_matches) always shards when
world > 1: every rank counts its share, one all-gather of (blocks, feasible) and one of the block
sums make every rank's cursor global (sbg_enum_set_global), and each fetch or pick is the engine
call plus one all-reduce(SUM) of the records, where every rank holds the ranks it owns and zero
records elsewhere.

The engine is any object with the `LutEngine` part-methods; the CPU tests drive this module over
`gloo` with an oracle-backed stand-in engine, the product uses `LutEngine` (CUDA) over `nccl`.
"""
import math
import time

import numpy as np
import torch
import torch.distributed as dist

from .lut import (MATCH_DTYPE, SBG_DEPTH_BINS, SBG_KEY_NONE, SBG_LIST_CAP, Enumeration,
                  _trim, result5_to_ret, result7_to_ret, sample_matches, shuffled_order,
                  shuffled_orders7)

_I64_MAX = (1 << 63) - 1


def _key_to_i64(key):
    # Keys use < 2^63 except the "none" sentinel, which maps to int64 max (still the maximum).
    return _I64_MAX if key == SBG_KEY_NONE else int(key)


def _i64_to_key(v):
    return SBG_KEY_NONE if v == _I64_MAX else int(v)


class _DeviceArray:
    """A raw device pointer as something torch can wrap without a copy."""

    def __init__(self, ptr, count):
        self.__cuda_array_interface__ = {"shape": (count,), "typestr": "<i8", "data": (ptr, False),
                                         "version": 2}


class DistributedLutSearch:
    """Sharding pays only when a search is large: below the thresholds every rank simply runs the
    whole (sub)search itself -- same inputs, same deterministic result, no collective at all."""

    def __init__(self, engine, group=None, device=None, shard_min_tuples5=5e7,
                 shard_min_tuples7=2e8, shard_min_list=8192):
        self.engine = engine
        self.shard_min_tuples5 = shard_min_tuples5
        self.shard_min_tuples7 = shard_min_tuples7
        self.shard_min_list = shard_min_list
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        backend = dist.get_backend(group)
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device()) if backend == "nccl" \
                else torch.device("cpu")
        self.device = device
        self.collectives = 0
        self.collective_ms = 0.0      # host time spent inside collectives (incl. waiting for peers)
        self.last_phase1_sharded = False

    # -- collectives ---------------------------------------------------------------------------
    def _allreduce_min_key(self, key):
        t0 = time.perf_counter()
        t = torch.tensor([_key_to_i64(key)], dtype=torch.int64, device=self.device)
        dist.all_reduce(t, op=dist.ReduceOp.MIN, group=self.group)
        self.collectives += 1
        out = _i64_to_key(int(t.item()))
        self.collective_ms += 1e3 * (time.perf_counter() - t0)
        return out

    def _allgather_lists(self, local):
        """local: sorted uint64 array (<= SBG_LIST_CAP).  Returns the concatenation over ranks.
        Host path (gloo / engines without a device-side list)."""
        cnt = torch.tensor([local.shape[0]], dtype=torch.int64, device=self.device)
        counts = [torch.zeros_like(cnt) for _ in range(self.world)]
        dist.all_gather(counts, cnt, group=self.group)
        counts = [int(c.item()) for c in counts]
        width = max(counts)
        self.collectives += 1
        if width == 0:
            return np.zeros(0, dtype=np.uint64)
        buf = torch.zeros(width, dtype=torch.int64)
        buf[:local.shape[0]] = torch.from_numpy(local.view(np.int64))
        buf = buf.to(self.device)
        parts = [torch.empty_like(buf) for _ in range(self.world)]
        dist.all_gather(parts, buf, group=self.group)
        self.collectives += 1
        out = [p[:c].cpu().numpy().view(np.uint64) for p, c in zip(parts, counts)]
        return np.concatenate(out)

    def _allgather_merge_on_device(self, count):
        """NCCL path: every rank's ordered list goes straight from its engine's device buffer into
        one gathered device buffer (all_gather_into_tensor over NVLink) and is merged there
        (sbg_set_list7_device); no list ever visits the host.  Returns the merged length."""
        t0 = time.perf_counter()
        cnt = torch.tensor([count], dtype=torch.int64, device=self.device)
        counts = torch.empty(self.world, dtype=torch.int64, device=self.device)
        dist.all_gather_into_tensor(counts, cnt, group=self.group)
        counts = counts.tolist()          # `world` integers: grid sizes are chosen on the host
        self.collectives += 1
        width = max(max(counts), 1)
        mine = torch.zeros(width, dtype=torch.int64, device=self.device)
        if count > 0:
            ptr, n = self.engine.list7_device()
            mine[:count] = torch.as_tensor(_DeviceArray(ptr, n), device=self.device)[:count]
        gathered = torch.empty(self.world * width, dtype=torch.int64, device=self.device)
        dist.all_gather_into_tensor(gathered, mine, group=self.group)
        self.collectives += 1
        # the merge kernel runs on the engine's stream, the collective on torch's: order them
        torch.cuda.current_stream().synchronize()
        self.collective_ms += 1e3 * (time.perf_counter() - t0)
        self.engine.set_list7_device(gathered.data_ptr(), width, counts)
        self._keepalive = gathered
        return min(sum(counts), SBG_LIST_CAP)

    # -- searches ------------------------------------------------------------------------------
    def search5_sharded(self, order):
        """The current problem's 5-LUT search with a given function order -> raw sbg_result."""
        n = self.engine.n
        if self.world == 1 or math.comb(n, 5) < self.shard_min_tuples5:
            return self.engine.finish5(self.engine.search5_part(0, 1, order), order)
        key = self.engine.search5_part(self.rank, self.world, order)
        key = self._allreduce_min_key(key)
        return self.engine.finish5(key, order)

    def _install_list7(self):
        """search_7lut phase 1: every rank installs the same list, built sharded (and merged) when
        the space is large, else by each rank alone.  Returns its length."""
        n = self.engine.n
        self.last_phase1_sharded = not (self.world == 1 or math.comb(n, 7) < self.shard_min_tuples7)
        if not self.last_phase1_sharded:
            # phase 1 replicated: every rank builds (and keeps on its device) the same full list
            return self.engine.filter7_keep_local()
        if self.device.type == "cuda" and hasattr(self.engine, "filter7_part_device"):
            return self._allgather_merge_on_device(
                self.engine.filter7_part_device(self.rank, self.world))
        local = self.engine.filter7_part(self.rank, self.world)
        merged = self._allgather_lists(local)
        # Every rank installs the same merged list: the runs are merged and cut at
        # SBG_LIST_CAP entries (lut.c:316-318 at size == 1).
        self.engine.set_list7(merged)
        return min(len(merged), SBG_LIST_CAP)

    def search7_sharded(self, outer, middle):
        count = self._install_list7()
        if self.world == 1 or count < self.shard_min_list:
            key = self.engine.decomp7_part(0, 1, outer, middle)
        else:
            key = self.engine.decomp7_part(self.rank, self.world, outer, middle)
            key = self._allreduce_min_key(key)
        return self.engine.finish7(key, outer, middle)

    def search_5lut(self, tables, target, mask, inbits, rng):
        order = shuffled_order(rng)
        self.engine.load(tables, target, mask, inbits)
        return result5_to_ret(self.search5_sharded(order), rng)

    def search_7lut(self, tables, target, mask, inbits, rng):
        outer, middle = shuffled_orders7(rng)
        self.engine.load(tables, target, mask, inbits)
        return result7_to_ret(self.search7_sharded(outer, middle), rng)

    # -- enumeration: ranks of the whole across the ranks' shares ------------------------------
    def _globalize(self, feasible):
        """All-gathers every rank's (deal blocks, feasible) and block sums, and makes the engine's
        cursor global.  Returns (the whole's total, feasible summed over the ranks)."""
        t0 = time.perf_counter()
        nb = self.engine.enum_block_count()
        mine = torch.tensor([nb, feasible], dtype=torch.int64, device=self.device)
        meta = torch.empty(2 * self.world, dtype=torch.int64, device=self.device)
        dist.all_gather_into_tensor(meta, mine, group=self.group)
        meta = meta.view(self.world, 2).tolist()
        self.collectives += 1
        counts = [int(m[0]) for m in meta]
        width = max(max(counts), 1)
        if self.device.type == "cuda":
            # the sums go from the engine's device straight into the gathered device buffer;
            # set_global reads only the first counts[q] entries of each row.  enum_block_sums waits
            # for torch's stream before the engine writes the row on its own.
            row = torch.empty(width, dtype=torch.int64, device=self.device)
            self.engine.enum_block_sums(out=row)
            sums = torch.empty(self.world * width, dtype=torch.int64, device=self.device)
            dist.all_gather_into_tensor(sums, row, group=self.group)
            # set_global reads them on the engine's stream, the collective ran on torch's
            torch.cuda.current_stream().synchronize()
            sums = sums.view(self.world, width)
        else:
            row = torch.zeros(width, dtype=torch.int64)
            row[:nb] = torch.from_numpy(self.engine.enum_block_sums().view(np.int64))
            parts = [torch.empty_like(row) for _ in range(self.world)]
            dist.all_gather(parts, row, group=self.group)
            sums = torch.stack(parts).numpy()
        self.collectives += 1
        total = self.engine.enum_set_global(sums, counts)
        self.collective_ms += 1e3 * (time.perf_counter() - t0)
        return total, sum(int(m[1]) for m in meta)

    def _sum_records(self, recs):
        """One all-reduce(SUM) of every rank's records (the ranks it owns, zero records elsewhere)."""
        t0 = time.perf_counter()
        t = torch.from_numpy(recs.view(np.int64).copy()).to(self.device)
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)
        self.collectives += 1
        out = t.cpu().numpy().view(MATCH_DTYPE).copy()
        self.collective_ms += 1e3 * (time.perf_counter() - t0)
        assert not np.any(out["width"] == 0), "a rank of the whole is owned by no share"
        return out

    def _enumerate(self, run, max_matches, list_length=None):
        if self.world == 1:
            return run(int(max_matches), 0, 1)
        local = run(0, self.rank, self.world)
        total, feasible = self._globalize(local.feasible)
        first = self.fetch_matches(0, max_matches)
        return Enumeration(total, feasible if list_length is None else list_length, first)

    def enumerate3(self, gate_order, max_matches):
        """Every match of lut_search's 3-LUT scan of the current problem over `gate_order`: the
        whole's total and feasible count and its first max_matches records, with this engine's
        cursor made global for fetch_matches / pick_matches / sample_matches."""
        return self._enumerate(
            lambda k, part, nparts: self.engine.enumerate3(gate_order, k, True, part, nparts),
            max_matches)

    def enumerate5(self, order, max_matches):
        """The same for search_5lut with a given function order."""
        return self._enumerate(
            lambda k, part, nparts: self.engine.enumerate5(order, k, True, part, nparts),
            max_matches)

    def enumerate7(self, outer, middle, max_matches):
        """The same for search_7lut; the list is installed as search7_sharded installs it, and
        `feasible` is its length."""
        count = self._install_list7()
        return self._enumerate(
            lambda k, part, nparts: self.engine.enumerate7(outer, middle, k, True, part, nparts),
            max_matches, list_length=count)

    def enumerate7_all(self, outer, middle, max_matches):
        """The same over every 7-combination (LutEngine.enumerate7_all): no list is installed, and
        `feasible` is the whole's feasible combinations, summed over the ranks."""
        return self._enumerate(
            lambda k, part, nparts: self.engine.enumerate7_all(outer, middle, k, True, part, nparts),
            max_matches)

    def enumerate7_chain(self, outer, middle, max_matches):
        """The 7-LUT chain realisations (LutEngine.enumerate7_chain), over every 7-combination as
        enumerate7_all: no list is installed, and `feasible` is summed over the ranks."""
        return self._enumerate(
            lambda k, part, nparts: self.engine.enumerate7_chain(outer, middle, k, True, part,
                                                                 nparts),
            max_matches)

    def enumerate4_shared(self, order, max_matches):
        """The shared-input two-LUT realisations (LutEngine.enumerate4_shared), over every
        4-combination: no list is installed, and `feasible` is summed over the ranks."""
        return self._enumerate(
            lambda k, part, nparts: self.engine.enumerate4_shared(order, k, True, part, nparts),
            max_matches)

    def fetch_matches(self, first, count):
        """The whole's matches at ranks first .. min(first + count, total) - 1 (the last
        enumerate* call's), the same on every rank."""
        recs = self.engine.fetch_matches(first, count)
        if self.world == 1 or recs.shape[0] == 0:
            return recs
        return self._sum_records(recs)

    def pick_matches(self, ranks):
        """The whole's matches at the given ranks, in their order, the same on every rank."""
        recs = self.engine.pick_matches(ranks)
        if self.world == 1 or recs.shape[0] == 0:
            return recs
        return self._sum_records(recs)

    def group_sizes(self, ranks):
        """The whole's group sizes at the given ranks (LutEngine.group_sizes), in their order, the
        same on every rank: one all-reduce(SUM) of the shares' arrays (each share's sizes at the
        ranks it owns, 0 elsewhere)."""
        local = self.engine.group_sizes(ranks)
        if self.world == 1 or local.shape[0] == 0:
            return local
        t0 = time.perf_counter()
        t = torch.from_numpy(local.view(np.int64).copy()).to(self.device)
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)
        self.collectives += 1
        out = t.cpu().numpy().view(np.uint64).copy()
        self.collective_ms += 1e3 * (time.perf_counter() - t0)
        assert not np.any(out == 0), "a rank of the whole is owned by no share"
        return out

    def sample_matches(self, enumeration, k, seed=None):
        """k distinct matches drawn uniformly from the whole (lut.sample_matches); every rank draws
        the same ranks from the same seed."""
        return sample_matches(self, enumeration, k, seed)

    # -- depth filter ----------------------------------------------------------------------------
    def set_depth_filter(self, depth, max_depth):
        """The engine's depth filter (LutEngine.set_depth_filter), on every rank: later
        enumerations count, rank and fetch within the matches of depth <= max_depth."""
        self.engine.set_depth_filter(depth, max_depth)

    def clear_depth_filter(self):
        self.engine.clear_depth_filter()

    # -- function filter -------------------------------------------------------------------------
    def set_function_filter(self, outer=None, middle=None, inner=None):
        """The engine's function filter (LutEngine.set_function_filter), on every rank: later
        enumerations count, rank and fetch within the matches whose LUTs lie in the sets."""
        self.engine.set_function_filter(outer, middle, inner)

    def clear_function_filter(self):
        self.engine.clear_function_filter()

    # -- grouping --------------------------------------------------------------------------------
    def set_grouping(self, grouping):
        """The engine's grouping (LutEngine.set_grouping), on every rank: later enumerations count,
        rank and fetch groups of matches (None, "shape" or "tuple")."""
        self.engine.set_grouping(grouping)

    def depth_counts(self):
        """The whole's matches per depth of the last enumerate* call (counted under a filter):
        one all-reduce(SUM) of the ranks' histograms.  Trimmed after the last non-empty bin."""
        local = self.engine.depth_counts()
        if self.world == 1:
            return local
        t0 = time.perf_counter()
        full = np.zeros(SBG_DEPTH_BINS, dtype=np.uint64)
        full[:local.shape[0]] = local
        t = torch.from_numpy(full.view(np.int64).copy()).to(self.device)
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group)
        self.collectives += 1
        out = t.cpu().numpy().view(np.uint64)
        self.collective_ms += 1e3 * (time.perf_counter() - t0)
        return _trim(out)
