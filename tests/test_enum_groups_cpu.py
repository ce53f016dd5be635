"""CPU: the host side of grouped enumeration -- match_group by hand for every width and grouping,
its argument checks, set_grouping's checks that need no device, and the header's declarations."""
import ctypes as C
import os

import pytest

import _support as S
import sboxgates_b200 as sb
from sboxgates_b200 import native


def test_match_group_by_hand():
    k3 = 5 << 18 | 9 << 9 | 30
    for g in (None, "shape", "tuple"):
        assert sb.match_group(k3, 3, g) == k3                       # a 3-LUT key is its own group
    # 5-LUT: tuple rank << 12 | ordering row << 8 | position
    k5 = 123_456 << 12 | 7 << 8 | 201
    assert sb.match_group(k5, 5, None) == k5
    assert sb.match_group(k5, 5, "shape") == 123_456 << 4 | 7
    assert sb.match_group(k5, 5, "tuple") == 123_456
    # 7-LUT: list index << 23 | ordering row << 16 | outer position << 8 | middle position
    k7 = 99_999 << 23 | 69 << 16 | 255 << 8 | 3
    assert sb.match_group(k7, 7, None) == k7
    assert sb.match_group(k7, 7, "shape") == 99_999 * 128 + 69
    assert sb.match_group(k7, 7, "tuple") == 99_999
    # keys differing only in functions share a shape; in the row too, a gate set
    assert sb.match_group(k5 ^ 0xFF, 5, "shape") == sb.match_group(k5, 5, "shape")
    assert sb.match_group(k5 ^ (1 << 8), 5, "shape") != sb.match_group(k5, 5, "shape")
    assert sb.match_group(k5 ^ (1 << 8), 5, "tuple") == sb.match_group(k5, 5, "tuple")
    assert sb.match_group(k7 ^ 0xFFFF, 7, "shape") == sb.match_group(k7, 7, "shape")
    assert sb.match_group(k7 ^ (1 << 16), 7, "tuple") == sb.match_group(k7, 7, "tuple")
    assert sb.match_group(2**64 - 1, 7, "tuple") == (2**64 - 1) >> 23


def test_match_group_argument_checks():
    for bad in ("wiring", 1, "SHAPE"):
        with pytest.raises(ValueError):
            sb.match_group(0, 5, bad)
    for width in (2, 4, 6, 8):
        with pytest.raises(ValueError):
            sb.match_group(0, width, "shape")
    for key in (-1, 2**64):
        with pytest.raises(ValueError):
            sb.match_group(key, 7, "tuple")


def test_set_grouping_argument_checks():
    eng = sb.LutEngine.__new__(sb.LutEngine)   # no device: the check runs before the library
    for bad in ("wiring", 1, 0, "Tuple", True):
        with pytest.raises(ValueError):
            eng.set_grouping(bad)


def test_header_declares_the_grouping():
    with open(os.path.join(S.ROOT, "include", "sboxgates_b200.h")) as f:
        header = f.read()
    assert "int sbg_enum_set_grouping(sbg_handle *h, int grouping);" in header
    for name, value in (("SBG_GROUP_NONE", 0), ("SBG_GROUP_SHAPE", 1), ("SBG_GROUP_TUPLE", 2)):
        assert "#define %s %d " % (name, value) in header
        assert getattr(native, name) == value
    assert native.SIGNATURES["sbg_enum_set_grouping"] == (C.c_int, [C.c_void_p, C.c_int])
    lifetime = header[header.index("Cursor lifetime:"):header.index("Without a cursor")]
    assert "sbg_enum_set_grouping ends it, whatever the call returns." in lifetime
    assert "match_group" in sb.__all__
