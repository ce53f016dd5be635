"""Seeded call sequences over one sbg_handle, and a model of the handle state they go through.

The sequences mix what a graph build, bench.py and DistributedLutSearch do on one handle: staged
slots, single node calls and batches (slots repeated, more jobs than lanes), the sharded phase-1 /
phase-2 steps, enumerations with fetch and pick, a torch side stream and the depth filter.  The
model says, for every step, which state each slot holds, which slot is current, and which (slot,
state) the installed 7-LUT list belongs to -- so a test can ask a fresh reference handle for what
the step must return.  Nothing here needs a device: the CPU test checks that each seed still
reaches the call patterns the GPU test was written for."""
import numpy as np

import _support as S

SEEDS = (11, 23)
STEPS = 300
LANES = 8
SCAN3, SEARCH5, SEARCH7 = 1, 2, 4
BIG = (130, 500)          # more changed gates than travel as kernel arguments: the bulk copy
NO7 = 500                 # search_7lut's phase 1 at this size sweeps C(500, 7): left out


class State:
    """One search state of the pool: gate tables, target, mask, the used input bits."""

    def __init__(self, idx, tabs, tgt, mask, inb):
        self.idx, self.tabs, self.tgt, self.mask, self.inb = idx, tabs, tgt, mask, inb
        self.n = len(tabs)

    def args(self):
        return self.tabs, self.tgt, self.mask, self.inb


def random_mask(rs, size):
    mask = np.zeros(4, dtype=np.uint64)
    for p in rs.choice(256, size, replace=False):
        mask[p >> 6] |= np.uint64(1) << np.uint64(int(p) & 63)
    return mask


def make_pool(seed, count=12):
    """`count` states: n from 7 to 48 under mux masks of depth 0-3 or random masks, with sbox
    targets and targets some 3-, 5- or 7-gate circuit realises; the last two are large (n = 130
    and n = 500, all 256 positions) with a planted 5-LUT, so that their searches end early."""
    rs = np.random.RandomState(seed)
    sbox = S.rijndael_sbox()
    pool = []
    for i in range(count - 2):
        n = int(rs.randint(7, 49))
        tabs = S.synthetic_state(n, seed=int(rs.randint(1 << 30)), num_inputs=min(8, n))
        if i % 3 == 2:
            mask, inb = random_mask(rs, int(rs.choice([9, 33, 70, 140]))), []
        else:
            fixed = [(int(b), int(rs.randint(0, 2)))
                     for b in rs.choice(8, int(rs.randint(0, 4)), replace=False)]
            mask, inb = S.mux_mask(fixed), [b for b, _ in fixed if b < n]
        kind = i % 4
        g = [int(x) for x in rs.choice(n, 7, replace=False)]
        f = [int(x) for x in rs.randint(1, 255, 3)]
        if kind == 0:
            tgt = S.sbox_target(sbox, int(rs.randint(0, 8)))
        elif kind == 1:
            tgt = S.lut_table(f[0], tabs[g[0]], tabs[g[1]], tabs[g[2]])
        elif kind == 2:
            tgt = S.lut_table(f[0], S.lut_table(f[1], tabs[g[0]], tabs[g[1]], tabs[g[2]]),
                              tabs[g[3]], tabs[g[4]])
        else:
            tgt = S.lut_table(f[0], S.lut_table(f[1], tabs[g[0]], tabs[g[1]], tabs[g[2]]),
                              S.lut_table(f[2], tabs[g[3]], tabs[g[4]], tabs[g[5]]), tabs[g[6]])
        pool.append(State(i, tabs, tgt, mask, inb))
    full = np.full(4, np.uint64(2**64 - 1), dtype=np.uint64)
    for j, n in enumerate(BIG):
        tabs = S.synthetic_state(n, seed=int(rs.randint(1 << 30)))
        tgt = S.lut_table(0xCA, S.lut_table(0x96, tabs[9], tabs[12], tabs[17]), tabs[20], tabs[23])
        pool.append(State(count - 2 + j, tabs, tgt, full, []))
    return pool


def job_orders(seed, n):
    """The orders of one job: search_5lut's, search_7lut's two, create_circuit's gate order."""
    rs = np.random.RandomState(seed)
    return dict(order5=bytes(rs.permutation(256).astype(np.uint8)),
                outer=bytes(rs.permutation(256).astype(np.uint8)),
                middle=bytes(rs.permutation(256).astype(np.uint8)),
                gate_order=[int(x) for x in rs.permutation(n)])


def job_kwargs(flags, seed, n):
    """search_node / search_batch keyword arguments of a job with the given SBG_DO_* flags."""
    o = job_orders(seed, n)
    kw = {}
    if flags & SCAN3:
        kw["gate_order"] = o["gate_order"]
    if flags & SEARCH5:
        kw["order5"] = o["order5"]
    if flags & SEARCH7:
        kw["outer"], kw["middle"] = o["outer"], o["middle"]
    return kw


def batch_waves(jobs):
    return [jobs[b:b + LANES] for b in range(0, len(jobs), LANES)]


class Model:
    """What the handle holds between calls.

    slots: slot -> pool index of the staged state; version: slot -> changes staged so far (an
    identical restage is no change); cur: the current slot (None: no problem); lst: (slot, version,
    what) of lane 0's list, what = ("whole",) for the phase-1 list or ("part", p, k) for a part's
    list of sbg_filter7_part(p, k > 1), or None.  lst_parts: the parts of the phase 1 behind the
    whole list (1, or k for sbg_filter7_part(p, k) of every part merged by sbg_set_list7*, whose
    sweep is part k-1's).  changed / rows: a slot's change not yet applied on the device (a lazy
    load) / its position-major rows built."""

    def __init__(self, pool):
        self.pool = pool
        self.slots, self.version = {}, {}
        self.cur, self.lst = None, None
        self.lst_parts = 1
        self.changed, self.rows = {}, {}
        self.filter_n = None

    def state(self, slot=None):
        s = self.cur if slot is None else slot
        return None if s is None else self.pool[self.slots[s]]

    def list_of_current(self):
        """The part of lane 0's list that belongs to the current problem as staged now: what, or
        None."""
        if self.lst is None or self.cur is None:
            return None
        slot, ver, what = self.lst
        return what if (slot, ver) == (self.cur, self.version[self.cur]) else None

    def _stage(self, slot, idx, lazy):
        if self.slots.get(slot) == idx:
            return
        self.slots[slot] = idx
        self.version[slot] = self.version.get(slot, 0) + 1
        self.changed[slot] = lazy
        self.rows[slot] = False

    def _begin(self, slot, rows):
        self.changed[slot] = False
        if rows:
            self.rows[slot] = True

    def _whole(self, slot, parts=1):
        self.lst = (slot, self.version[slot], ("whole",))
        self.lst_parts = parts

    def apply(self, op, stages=None):
        """Advances the model by one operation that succeeded.  stages: the found_stage of each job
        of a node call or batch (a 7-LUT stage installs its list unless an earlier stage matched)."""
        kind = op[0]
        if kind == "load":
            self._stage(0, op[1], True)
            self.cur, self.lst = 0, None
        elif kind == "stage":
            self._stage(op[1], op[2], False)
        elif kind == "use":
            self.cur, self.lst = op[1], None
        elif kind == "search5":
            self._begin(self.cur, False)
        elif kind == "search7":
            self._begin(self.cur, True)
            self._whole(self.cur)
        elif kind == "node":
            slot, flags = op[1], op[2]
            self.cur, self.lst = slot, None
            seven = bool(flags & SEARCH7) and self.state(slot).n >= 7
            self._begin(slot, seven)
            if seven and stages[0] not in (3, 5):
                self._whole(slot)
        elif kind == "batch":
            jobs = op[1]
            for base, wave in zip(range(0, len(jobs), LANES), batch_waves(jobs)):
                for slot, flags, _ in wave:
                    self._begin(slot, bool(flags & SEARCH7))
                slot, flags, _ = wave[0]
                self.lst = None
                if flags & SEARCH7 and stages[base] not in (3, 5):
                    self._whole(slot)
        elif kind == "filter":
            self._begin(self.cur, True)
            self._whole(self.cur, op[1])
        elif kind == "enum" and op[1] == 7:
            if self.list_of_current() != ("whole",):
                self._begin(self.cur, True)
                self._whole(self.cur)
            self._begin(self.cur, False)
        elif kind == "enum":
            self._begin(self.cur, False)
        elif kind == "consume" and op[1] == "enum7":
            self.apply(("enum", 7))
        elif kind == "depth":
            self.filter_n = op[2] if op[1] else None


# ------------------------------------------------------------------------------------------------
# The generator

def generate(seed, pool, steps=STEPS):
    """A seeded sequence of `steps` operations (tuples, see Model.apply and the GPU test's
    runner).  Consumers of the installed list (enumerate7, decomp7_part + finish7, list7_device)
    are drawn more often right after the calls that leave lane 0's list with another slot or state:
    a batch, a restage of the current slot."""
    rs = np.random.RandomState(seed)
    model = Model(pool)
    ops = []
    side = False
    last = None

    def fits7(idx):
        return pool[idx].n != NO7

    def emit(op):
        nonlocal last
        ops.append(op)
        last = op[0]
        # the generator's model does not know which stage a search ends at: it assumes none matched
        model.apply(op, stages=[0] * (len(op[1]) if op[0] == "batch" else 1))

    emit(("load", int(rs.randint(len(pool) - 2))))
    while len(ops) < steps:
        staged = sorted(model.slots)
        cur_state = model.state()
        can7 = cur_state is not None and fits7(cur_state.idx)
        r = rs.randint(100)
        if last in ("batch", "stage") and rs.randint(2):
            # a list consumer right after what may have moved the list
            what = ["enum7", "decomp", "list7"][rs.randint(3)]
            if can7:
                emit(("consume", what, int(rs.randint(1 << 30))))
                continue
        if r < 6:
            emit(("load", int(rs.randint(len(pool)))))
        elif r < 18:
            slot = int(rs.choice([model.cur, model.cur, 1, 2, 3, 5, 9])) if model.cur is not None \
                else int(rs.randint(6))
            if model.list_of_current() is not None and rs.randint(2):
                slot = model.cur
            # restaging the current slot: half the time the state it already holds
            idx = model.slots.get(slot) if slot in model.slots and rs.randint(3) == 0 \
                else int(rs.randint(len(pool)))
            emit(("stage", slot, idx))
        elif r < 23 and staged:
            emit(("use", int(rs.choice(staged))))
        elif r < 28:
            emit(("search5", int(rs.randint(1 << 30))))
        elif r < 33 and can7:
            emit(("search7", int(rs.randint(1 << 30))))
        elif r < 41 and staged:
            slot = int(rs.choice(staged))
            flags = int(rs.randint(1, 8))
            if not fits7(model.slots[slot]):
                flags &= ~SEARCH7
                flags |= SCAN3
            emit(("node", slot, flags, int(rs.randint(1 << 30))))
        elif r < 58 and staged:
            # a batch: slots drawn with repeats; sometimes a second wave; sometimes the current slot
            # restaged (or loaded) just before, so that the batch meets a pending change
            if rs.randint(3) == 0:
                emit(("load", int(rs.randint(len(pool)))) if rs.randint(2) else
                     ("stage", int(rs.choice(staged)), int(rs.randint(len(pool)))))
                staged = sorted(model.slots)
            njobs = int(rs.choice([1, 2, 3, 4, 6, 8, 9, 12]))
            hot = int(rs.choice(staged))
            jobs = []
            for _ in range(njobs):
                slot = hot if rs.randint(2) else int(rs.choice(staged))
                flags = int(rs.choice([SCAN3, SEARCH5, SEARCH7, SCAN3 | SEARCH7, SEARCH5 | SEARCH7,
                                       SCAN3 | SEARCH5 | SEARCH7]))
                if not fits7(model.slots[slot]):
                    flags = (flags & ~SEARCH7) | SCAN3
                jobs.append((slot, flags, int(rs.randint(1 << 30))))
            emit(("batch", tuple(jobs)))
        elif r < 66 and can7:
            emit(("filter", int(rs.choice([1, 2, 3])), bool(rs.randint(2)),
                  int(rs.randint(1 << 30))))
        elif r < 86 and cur_state is not None:
            width = int(rs.choice([3, 5, 7] if can7 else [3, 5]))
            emit(("enum", width, bool(rs.randint(2)), int(rs.choice([0, 1, 5, 40])),
                  int(rs.randint(1 << 30))))
        elif r < 90 and can7:
            emit(("consume", ["enum7", "decomp", "list7"][rs.randint(3)], int(rs.randint(1 << 30))))
        elif r < 95:
            side = not side
            emit(("stream", side))
        elif cur_state is not None:
            on = model.filter_n is None or rs.randint(3) == 0
            emit(("depth", on, cur_state.n, int(rs.randint(1 << 30))) if on else
                 ("depth", False, 0, 0))
    return ops


# ------------------------------------------------------------------------------------------------
# The call patterns each seed must contain

def patterns(pool, ops):
    """The set of defect patterns the sequence reaches:
    batch_list_other: a batch whose last wave's lane 0 ran search_7lut on a slot other than the
        current one, then a list consumer with nothing in between that installs or drops a list;
    restage_current: a real change staged into the current slot while lane 0 held its list, then
        a list consumer;
    wave_repeat_changed: a wave that puts one slot on two lanes while the slot has a change
        pending (a lazy load);
    wave_repeat_rows: a wave that puts one slot on two lanes, one of them with search_7lut, while
        the slot's rows are not built;
    two_waves: a batch of more than LANES jobs;
    stream_batch: a batch on a torch side stream."""
    model = Model(pool)
    found = set()
    moved = None      # "batch" / "restage" while lane 0's list is stale for the current problem
    side = False
    for op in ops:
        kind = op[0]
        if kind == "consume" and moved is not None:
            found.add({"batch": "batch_list_other", "restage": "restage_current"}[moved])
        if kind == "batch":
            jobs = op[1]
            if len(jobs) > LANES:
                found.add("two_waves")
            if side:
                found.add("stream_batch")
            for wave in batch_waves(jobs):
                slots = [j[0] for j in wave]
                for s in set(slots):
                    if slots.count(s) < 2:
                        continue
                    if model.changed.get(s):
                        found.add("wave_repeat_changed")
                    if not model.rows.get(s) and any(f & SEARCH7 for sl, f, _ in wave if sl == s):
                        found.add("wave_repeat_rows")
            last0 = batch_waves(jobs)[-1][0]
            moved = "batch" if last0[1] & SEARCH7 and last0[0] != model.cur else None
        elif kind == "stage" and op[1] == model.cur and model.slots.get(op[1]) != op[2] \
                and model.list_of_current() is not None:
            moved = "restage"
        elif kind in ("load", "use", "search7", "node", "filter", "enum", "consume"):
            if not (kind == "enum" and op[1] != 7):
                moved = None
        if kind == "stream":
            side = op[1]
        model.apply(op, stages=[0] * (len(op[1]) if kind == "batch" else 1))
    return found


PATTERNS = {"batch_list_other", "restage_current", "wave_repeat_changed", "wave_repeat_rows",
            "two_waves", "stream_batch"}
