"""CPU: the host side of group sizes -- the header's declaration and cursor-lifetime entry, the
ctypes signature, and group_sizes' argument checks that need no device."""
import ctypes as C
import os

import numpy as np
import pytest

import _support as S
import sboxgates_b200 as sb
from sboxgates_b200 import native


def _header():
    with open(os.path.join(S.ROOT, "include", "sboxgates_b200.h")) as f:
        return f.read()


def test_header_declares_group_sizes():
    header = _header()
    assert ("int sbg_enum_group_sizes(sbg_handle *h, const uint64_t *ranks, uint64_t nranks, "
            "uint64_t *sizes);") in header
    u64p = C.POINTER(C.c_uint64)
    assert native.SIGNATURES["sbg_enum_group_sizes"] == (C.c_int, [C.c_void_p, u64p, C.c_uint64,
                                                                   u64p])
    # the grouping section points at the call instead of saying sizes are not reported
    grouping = header[header.index("---- grouping:"):header.index("---- helpers shared")]
    assert "not reported" not in grouping and "sbg_enum_group_sizes" in grouping


def test_lifetime_lists_group_sizes_among_the_keepers():
    header = _header()
    lifetime = header[header.index("Cursor lifetime:"):header.index("Without a cursor")]
    keepers = [line for line in lifetime.split(";") if line.strip().endswith("keep it")]
    assert len(keepers) == 1 and "sbg_enum_group_sizes" in keepers[0]
    assert "sbg_enum_pick" in keepers[0] and "sbg_enum_depth_counts" in keepers[0]


def test_group_sizes_argument_checks():
    eng = sb.LutEngine.__new__(sb.LutEngine)   # no device: the checks run before the library
    for bad in ([-1], np.array([3, -2]), [[0, 1]], np.zeros((2, 2), dtype=np.uint64), [0.5],
                np.zeros(native.SBG_ENUM_MAX_MATCHES + 1, dtype=np.uint64)):
        with pytest.raises(ValueError):
            eng.group_sizes(bad)
