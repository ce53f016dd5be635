"""GPU: a handle gives back all the device memory it took.  Every cycle creates a LutEngine, grows
each kind of device buffer it has (a node search and a batch on all lanes, phase 1 with a list
install, counts, fetches, picks, block sums and global ranks at widths 3, 5 and 7) and closes it.
The process's device memory, read from NVML per process so that other users of the GPU do not
disturb it, must be back where it stood after one warm-up cycle."""
import pytest
import torch

import _handle_support as H
import _support as S
import sboxgates_b200 as sb

pytestmark = pytest.mark.gpu

CYCLES = 20
GRANULE = 2 << 20   # the driver's allocation granule: NVML cannot see less
PROBE = 64 << 20


def _usage(nvml):
    """NVML's device memory per process: {(device index, pid): bytes}."""
    out = {}
    for i in range(nvml.nvmlDeviceGetCount()):
        dev = nvml.nvmlDeviceGetHandleByIndex(i)
        for p in nvml.nvmlDeviceGetComputeRunningProcesses(dev):
            if p.usedGpuMemory is not None:
                out[(i, p.pid)] = p.usedGpuMemory
    return out


def _own_entry(nvml):
    """This process's key in _usage, and the probe that found it (keep it alive).  NVML reports PIDs
    of its own namespace, which inside a container are not os.getpid(), so the entry is the one that
    grows by a PROBE-byte allocation; None if not exactly one does."""
    before = _usage(nvml)
    probe = torch.empty(PROBE, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    after = _usage(nvml)
    grown = [k for k, v in after.items() if 0 <= v - before.get(k, 0) - PROBE <= GRANULE]
    return (grown[0] if len(grown) == 1 else None), probe


def _cycle(state, orders):
    eng = sb.LutEngine(0)
    try:
        for slot in range(H.LANES):
            eng.stage(slot, *state)
        eng.search_node(0, **orders)
        eng.search_batch([dict(slot=s, **orders) for s in range(H.LANES)])
        eng.use(0)
        eng.set_list7(eng.filter7_part(0, 1))
        for width in (3, 5, 7):
            if width == 3:
                e = eng.enumerate3(orders["gate_order"], 64)
            elif width == 5:
                e = eng.enumerate5(orders["order5"], 64)
            else:
                e = eng.enumerate7(orders["outer"], orders["middle"], 64)
            assert e.total > 0, width
            eng.fetch_matches(0, 16)
            eng.pick_matches([0, e.total - 1, e.total // 2])
            sums = eng.enum_block_sums()
            assert eng.enum_set_global(sums.reshape(1, -1), [len(sums)]) == e.total
            eng.fetch_matches(e.total // 2, 16)
            eng.pick_matches([e.total - 1, 0])
    finally:
        eng.close()


def test_handle_returns_device_memory():
    nvml = pytest.importorskip("pynvml")
    try:
        nvml.nvmlInit()
    except nvml.NVMLError as err:
        pytest.skip("NVML unavailable: %s" % err)
    try:
        n = 24
        tabs = S.synthetic_state(n, seed=5)
        # 8 positions: matches at every width (47 3-LUT, 1,205,340 5-LUT, a 17,810-entry list)
        fixed = [(0, 1), (5, 0), (6, 1), (2, 0), (7, 1)]
        state = (tabs, S.sbox_target(S.rijndael_sbox(), 3), S.mux_mask(fixed), [b for b, _ in fixed])
        orders = H.job_orders(77, n)
        _cycle(state, orders)
        own, _probe = _own_entry(nvml)
        if own is None:
            pytest.skip("NVML does not show this process's allocations")
        base = _usage(nvml)[own]
        for _ in range(CYCLES):
            _cycle(state, orders)
        after = _usage(nvml).get(own)
        assert after is not None and abs(after - base) <= GRANULE, (base, after)
    finally:
        nvml.nvmlShutdown()
