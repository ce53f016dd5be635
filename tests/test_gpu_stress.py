"""GPU: randomised differential test (scripts/stress_gpu.py): all phase-1 kernel forms,
sharded and unsharded paths, fused and two-kernel search_5lut, one-call and step-by-step
search_7lut must agree with each other, and with the CPU oracle wherever it is affordable."""
import os
import subprocess
import sys

import pytest

import _support as S

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("seed", [11, 12])
def test_randomised_cross_check(seed):
    res = subprocess.run([sys.executable, os.path.join(S.ROOT, "scripts", "stress_gpu.py"), "120",
                          str(seed)], capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    assert "stress ok" in res.stdout
