"""sboxgates_b200 -- H100-native 3-LUT exhaustive search (the `--lut` path of dansarie/sboxgates).

The product is `libsboxgates_b200.so` (hand-written sm_90a CUDA kernels behind the C ABI in
include/sboxgates_b200.h) plus `csrc/lut_shim.c`, which gives it the reference's own
`search_5lut` / `search_7lut` signatures (lut.h:46-55).  This package is the Python host-side mirror
of that interface, used by the tests, bench.py and the multi-GPU (one process per GPU) driver.
There is no CPU implementation in here: importing works without a GPU, constructing an engine
does not.
"""
from .rng import Xorshift1024
from .lut import LutEngine, SearchResult, NO_GATE, search_5lut, search_7lut, shuffled_order, \
    shuffled_orders7, ordering_row, solve_inner, lut_table, lut_search, LutSearchResult, \
    Enumeration, enumerate_3lut, enumerate_5lut, enumerate_7lut, enumerate_7lut_all, \
    enumerate_7lut_chain, enumerate_4lut_shared, enumerate_lut_search, chain_row, chain_luts, \
    chain_result_luts, decode_key7_chain, shared_row, \
    match_to_ret, match_to_lut3, decode_key3, decode_key5, decode_key7, sample_matches, \
    match_depth, shallowest_matches, AFFINE_FUNCTIONS, gate_functions, match_functions_allowed, \
    allowed_fill, inner_table, match_group
from .native import load_library, NativeLibraryError, MATCH_DTYPE, SBG_MAX_DEPTH, SBG_DEPTH_BINS, \
    SBG_SHAPE_TREE, SBG_SHAPE_CHAIN, SBG_SHAPE_SHARED

__all__ = [
    "Xorshift1024", "LutEngine", "SearchResult", "NO_GATE", "search_5lut", "search_7lut",
    "shuffled_order", "shuffled_orders7", "ordering_row", "solve_inner", "lut_table",
    "lut_search", "LutSearchResult", "Enumeration", "enumerate_3lut", "enumerate_5lut",
    "enumerate_7lut", "enumerate_7lut_all", "enumerate_7lut_chain", "enumerate_4lut_shared",
    "enumerate_lut_search", "chain_row", "chain_luts", "chain_result_luts", "decode_key7_chain",
    "shared_row", "match_to_ret",
    "match_to_lut3", "decode_key3",
    "decode_key5", "decode_key7", "sample_matches", "match_depth", "shallowest_matches",
    "AFFINE_FUNCTIONS", "gate_functions", "match_functions_allowed", "allowed_fill", "inner_table",
    "match_group",
    "MATCH_DTYPE", "SBG_MAX_DEPTH", "SBG_DEPTH_BINS", "SBG_SHAPE_TREE", "SBG_SHAPE_CHAIN",
    "SBG_SHAPE_SHARED", "load_library", "NativeLibraryError",
]
