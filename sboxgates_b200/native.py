"""ctypes binding of libsboxgates_b200.so (include/sboxgates_b200.h).

The library is built in-tree by `__graft_entry__.build()` / `make -C sboxgates_b200/csrc`.  If it is
missing, loading fails loudly -- there is deliberately no fallback implementation.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# SBG_LIB: another build of the same library (A/B measurements of kernel variants)
LIB_PATH = os.environ.get("SBG_LIB") or os.path.join(_HERE, "libsboxgates_b200.so")

SBG_OK = 0
SBG_LIST_CAP = 100000
SBG_KEY_NONE = (1 << 64) - 1


class NativeLibraryError(RuntimeError):
    pass


class SbgResult(C.Structure):
    _fields_ = [
        ("found", C.c_int32), ("ordering", C.c_int32), ("pos_outer", C.c_int32),
        ("pos_middle", C.c_int32), ("func_outer", C.c_uint8), ("func_middle", C.c_uint8),
        ("func_inner", C.c_uint8), ("inner_seen", C.c_uint8), ("gates", C.c_uint16 * 7),
        ("stale_outer", C.c_uint16), ("index", C.c_uint64), ("key", C.c_uint64),
        ("tuples_feasible", C.c_uint64), ("tuples_swept", C.c_uint64),
    ]


class SbgJob(C.Structure):
    _fields_ = [("slot", C.c_int32), ("flags", C.c_int32), ("order5", C.POINTER(C.c_uint8)),
                ("outer7", C.POINTER(C.c_uint8)), ("middle7", C.POINTER(C.c_uint8)),
                ("gate_order", C.POINTER(C.c_uint16))]


class SbgNodeResult(C.Structure):
    _fields_ = [("found_stage", C.c_int32), ("gates3", C.c_uint16 * 3), ("func3", C.c_uint8),
                ("seen3", C.c_uint8), ("key3", C.c_uint64), ("r5", SbgResult), ("r7", SbgResult)]


class SbgMatch(C.Structure):
    """One enumerated match (sbg_match, 32 bytes)."""
    _fields_ = [("key", C.c_uint64), ("gates", C.c_uint16 * 7), ("func_outer", C.c_uint8),
                ("func_middle", C.c_uint8), ("func_inner", C.c_uint8), ("inner_seen", C.c_uint8),
                ("width", C.c_uint8), ("shape", C.c_uint8), ("pad", C.c_uint8 * 4)]


# The same layout as a numpy structured dtype: enumeration results arrive as one array.
MATCH_DTYPE = np.dtype([("key", "<u8"), ("gates", "<u2", (7,)), ("func_outer", "u1"),
                        ("func_middle", "u1"), ("func_inner", "u1"), ("inner_seen", "u1"),
                        ("width", "u1"), ("shape", "u1"), ("pad", "u1", (4,))])
SBG_ENUM_MAX_MATCHES = 1 << 24
SBG_ENUM7_ALL_MAX_GATES = 64   # largest n of the whole-space 7-LUT enumeration (sbg_enum7_all)
SBG_MAX_GATES = 500
SBG_MAX_DEPTH = 1020      # largest gate depth of a depth filter
SBG_DEPTH_BINS = 1024     # bins of the depth histogram
SBG_GROUP_NONE = 0        # enumeration groupings (sbg_enum_set_grouping): every match,
SBG_GROUP_SHAPE = 1       #   one per (gates, ordering row),
SBG_GROUP_TUPLE = 2       #   one per gate set
SBG_SHAPE_TREE = 0        # a 7-LUT record's wiring (sbg_match::shape): L3(L1(a,b,c), L2(d,e,f), g),
SBG_SHAPE_CHAIN = 1       #   or L3(L2(L1(a,b,c), d, e), f, g) (sbg_enum7_chain);
SBG_SHAPE_SHARED = 2      # a width-4 record: L2(L1(a,b,c), u, v), u or v one of a, b, c (sbg_enum4_shared)

SBG_DO_SCAN3, SBG_DO_SEARCH5, SBG_DO_SEARCH7 = 1, 2, 4
SBG_LANES = 8

u64p = C.POINTER(C.c_uint64)
u8p = C.POINTER(C.c_uint8)
i8p = C.POINTER(C.c_int8)

# name -> (restype, argtypes): every symbol include/sboxgates_b200.h declares.
SIGNATURES = {
    "sbg_create": (C.c_int, [C.POINTER(C.c_void_p), C.c_int]),
    "sbg_destroy": (None, [C.c_void_p]),
    "sbg_last_error": (C.c_char_p, [C.c_void_p]),
    "sbg_set_stream": (C.c_int, [C.c_void_p, C.c_void_p]),
    "sbg_launch_count": (C.c_uint64, [C.c_void_p]),
    "sbg_plan_tickets": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_uint32, C.c_int, C.c_uint64,
                                   C.POINTER(C.c_uint64)]),
    "sbg_weighted_tickets": (C.c_int, [C.c_int, C.c_uint32, C.POINTER(C.c_uint32)]),
    "sbg_last_kernel_ms": (C.c_float, [C.c_void_p, C.c_int]),
    "sbg_set_timing": (C.c_int, [C.c_void_p, C.c_int]),
    "sbg_transfer_stats": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64)]),
    "sbg_host_seconds": (C.c_int, [C.c_void_p, C.POINTER(C.c_double)]),
    "sbg_alu_peak": (C.c_int, [C.c_void_p, C.POINTER(C.c_double)]),
    "sbg_search_node": (C.c_int, [C.c_void_p, C.POINTER(SbgJob), C.POINTER(SbgNodeResult)]),
    "sbg_search_batch": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(SbgJob),
                                   C.POINTER(SbgNodeResult)]),
    "sbg_list7_device": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int)]),
    "sbg_allgather_merge7": (C.c_int, [C.POINTER(C.c_void_p), C.c_int, C.POINTER(C.c_int)]),
    "sbg_set_list7_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_int),
                                       C.c_int]),
    "sbg_load_problem": (C.c_int, [C.c_void_p, u64p, C.c_int, u64p, u64p, i8p]),
    "sbg_stage_problem": (C.c_int, [C.c_void_p, C.c_int, u64p, C.c_int, u64p, u64p, i8p]),
    "sbg_use_problem": (C.c_int, [C.c_void_p, C.c_int]),
    "sbg_search5": (C.c_int, [C.c_void_p, u8p, C.POINTER(SbgResult)]),
    "sbg_search7": (C.c_int, [C.c_void_p, u8p, u8p, C.POINTER(SbgResult)]),
    "sbg_search7_chain": (C.c_int, [C.c_void_p, u8p, u8p, C.POINTER(SbgResult)]),
    "sbg_search4_shared": (C.c_int, [C.c_void_p, u8p, C.POINTER(SbgResult)]),
    "sbg_search5_part": (C.c_int, [C.c_void_p, C.c_int, C.c_int, u8p, u64p]),
    "sbg_finish5": (C.c_int, [C.c_void_p, C.c_uint64, u8p, C.POINTER(SbgResult)]),
    "sbg_filter7_part": (C.c_int, [C.c_void_p, C.c_int, C.c_int, u64p, C.POINTER(C.c_int)]),
    "sbg_set_list7": (C.c_int, [C.c_void_p, u64p, C.c_int]),
    "sbg_decomp7_part": (C.c_int, [C.c_void_p, C.c_int, C.c_int, u8p, u8p, u64p]),
    "sbg_finish7": (C.c_int, [C.c_void_p, C.c_uint64, u8p, u8p, C.POINTER(SbgResult)]),
    "sbg_ordering_row": (C.c_int, [C.c_int, C.c_int, C.POINTER(C.c_int)]),
    "sbg_chain_row": (C.c_int, [C.c_int, C.POINTER(C.c_int)]),
    "sbg_shared_row": (C.c_int, [C.c_int, C.POINTER(C.c_int)]),
    "sbg_solve_inner": (C.c_int, [u64p, u64p, u64p, u64p, u64p, u8p, u8p]),
    "sbg_lut_table": (None, [C.c_uint8, u64p, u64p, u64p, u64p]),
    "sbg_enum5": (C.c_int, [C.c_void_p, C.c_int, C.c_int, u8p, C.c_uint64, C.c_void_p, u64p, u64p,
                            u64p]),
    "sbg_enum7": (C.c_int, [C.c_void_p, C.c_int, C.c_int, u8p, u8p, C.c_uint64, C.c_void_p, u64p,
                            u64p, u64p]),
    "sbg_enum7_all": (C.c_int, [C.c_void_p, C.c_int, C.c_int, u8p, u8p, C.c_uint64, C.c_void_p,
                                u64p, u64p, u64p]),
    "sbg_enum7_chain": (C.c_int, [C.c_void_p, C.c_int, C.c_int, u8p, u8p, C.c_uint64, C.c_void_p,
                                  u64p, u64p, u64p]),
    "sbg_enum4_shared": (C.c_int, [C.c_void_p, C.c_int, C.c_int, u8p, C.c_uint64, C.c_void_p, u64p,
                                   u64p, u64p]),
    "sbg_enum3": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_uint16), C.c_uint64,
                            C.c_void_p, u64p, u64p, u64p]),
    "sbg_enum_fetch": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, u64p]),
    "sbg_enum_pick": (C.c_int, [C.c_void_p, u64p, C.c_uint64, C.c_void_p]),
    "sbg_enum_block_sums": (C.c_int, [C.c_void_p, C.c_void_p, u64p]),
    "sbg_enum_set_global": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, u64p, C.c_int, u64p]),
    "sbg_enum_set_depth": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint16), C.c_int, C.c_uint32]),
    "sbg_enum_depth_counts": (C.c_int, [C.c_void_p, u64p, C.c_uint32]),
    "sbg_enum_set_functions": (C.c_int, [C.c_void_p, u64p, u64p, u64p]),
    "sbg_inner_table": (C.c_int, [u64p, C.POINTER(C.c_uint8)]),
    "sbg_enum_set_grouping": (C.c_int, [C.c_void_p, C.c_int]),
    "sbg_enum_group_sizes": (C.c_int, [C.c_void_p, u64p, C.c_uint64, u64p]),
}

_lib = None


def load_library(path=None):
    """Loads the shared library and binds every declared symbol; raises NativeLibraryError if the
    library or a symbol is missing."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or LIB_PATH
    if not os.path.exists(p):
        raise NativeLibraryError(
            "%s not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` or "
            "`make -C sboxgates_b200/csrc`; sboxgates_b200 has no fallback implementation" % p)
    try:
        lib = C.CDLL(p)
    except OSError as exc:
        raise NativeLibraryError("cannot load %s: %s" % (p, exc)) from exc
    for name, (restype, argtypes) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as exc:
            raise NativeLibraryError("%s lacks symbol %s" % (p, name)) from exc
        fn.restype = restype
        fn.argtypes = argtypes
    if path is None:
        _lib = lib
    return lib
