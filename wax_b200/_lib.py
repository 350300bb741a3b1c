"""ctypes loader for libwaxvs_cuda.so (the C-ABI in include/wax_vs_cuda.h).

The library is the product: there is no Python/CPU fallback.  If the shared object is missing this module
raises at import of the symbol table; if no CUDA device is present every engine call returns
WAX_VS_ERR_CUDA, surfaced as WaxError.invalidToc by engine.py (as MetalVectorEngine does for a missing
Metal device, MetalVectorEngine.swift:167-169).
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

PKG = Path(__file__).resolve().parent
LIB_PATH = PKG / "libwaxvs_cuda.so"

# return codes (include/wax_vs_cuda.h)
OK, ERR_NULL, ERR_DIMENSION, ERR_CAPACITY, ERR_CUDA, ERR_FORMAT, ERR_ARGUMENT, ERR_BUFFER, ERR_UNSUPPORTED = (
    0, -1, -2, -3, -4, -5, -6, -7, -8)
MAX_RESULTS = 10_000
NO_FILTER = 0xFFFFFFFF          # WAX_VS_NO_FILTER: a query of wax_vs_search_batch_multi_filtered without a filter
MAX_DIMENSIONS = 1_000_000
MAX_PER_GROUP = 128             # WAX_VS_MAX_PER_GROUP: rows per group of wax_vs_search_grouped
SHARD_HANDLE_BYTES, SHARD_MAX_RANKS, SHARD_MAX_K = 128, 16, 128
SHARD_MAX_GROUPS = 256          # WAX_VS_SHARD_MAX_GROUPS: clamp(top_groups) of the sharded grouped search
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1   # wax_vs_where bounds meaning "no bound"
NO_LOCATION = -(1 << 31)        # WAX_VS_NO_LOCATION: the lat_bin of a row without a location
# WAX_VS_COLUMN_*: the side columns an engine holds (wax_vs_export_columns / wax_vs_absorb_rows)
COLUMN_GROUPS, COLUMN_ATTRIBUTES, COLUMN_LOCATIONS, COLUMN_TERMS = 1, 2, 4, 8


class Candidate(C.Structure):
    """wax_vs_candidate (24 bytes)."""
    _fields_ = [("distance", C.c_float), ("valid", C.c_uint32), ("row", C.c_uint64), ("frame_id", C.c_uint64)]


class Where(C.Structure):
    """wax_vs_where (32 bytes)."""
    _fields_ = [("after", C.c_int64), ("before", C.c_int64), ("all_tags", C.c_uint64), ("no_tags", C.c_uint64)]


class WhereNear(C.Structure):
    """wax_vs_where_near (56 bytes)."""
    _fields_ = [("where", Where), ("latitude", C.c_double), ("longitude", C.c_double), ("radius_m", C.c_double)]


class RootClause(C.Structure):
    """wax_vs_root_clause (16 bytes)."""
    _fields_ = [("all_tags", C.c_uint64), ("no_tags", C.c_uint64)]


# Every symbol include/wax_vs_cuda.h declares, with its signature.  tests/test_abi.py checks this table
# against the header and against the built library.
_f32p, _u64p, _u32p, _u8p = C.POINTER(C.c_float), C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.POINTER(C.c_uint8)
_f64p = C.POINTER(C.c_double)
_eng = C.c_void_p
SIGNATURES = {
    "wax_vs_device_count": (C.c_int32, [C.POINTER(C.c_int32)]),
    "wax_vs_create": (C.c_int32, [C.c_uint32, C.c_uint8, C.POINTER(C.c_int32), C.c_int32, C.POINTER(_eng)]),
    "wax_vs_destroy": (None, [_eng]),
    "wax_vs_dimensions": (C.c_int32, [_eng, _u32p]),
    "wax_vs_similarity": (C.c_int32, [_eng, _u8p]),
    "wax_vs_count": (C.c_int32, [_eng, _u64p]),
    "wax_vs_reserve": (C.c_int32, [_eng, C.c_uint64]),
    "wax_vs_add": (C.c_int32, [_eng, C.c_uint64, _f32p, C.c_uint32]),
    "wax_vs_add_batch": (C.c_int32, [_eng, _u64p, _f32p, C.c_uint64, C.c_uint32]),
    "wax_vs_remove": (C.c_int32, [_eng, C.c_uint64]),
    "wax_vs_remove_batch": (C.c_int32, [_eng, _u64p, C.c_uint64, _u64p]),
    "wax_vs_rebalance": (C.c_int32, [_eng, _u64p]),
    "wax_vs_add_batch_keyed": (C.c_int32, [_eng, _u64p, _f32p, C.c_uint64, C.c_uint32, C.c_uint64, _u64p]),
    "wax_vs_contains": (C.c_int32, [_eng, _u64p, C.c_uint64, _u8p]),
    "wax_vs_deserialize_rows": (C.c_int32, [_eng, _u8p, C.c_uint64, C.c_uint64, C.c_uint64]),
    "wax_vs_export_rows": (C.c_int32, [_eng, C.c_uint64, C.c_uint64, _u64p, _f32p, _u64p]),
    "wax_vs_export_rows_device": (C.c_int32, [_eng, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p]),
    "wax_vs_export_columns": (C.c_int32, [_eng, C.c_uint64, C.c_uint64, C.c_void_p, _u64p, _u64p, C.c_uint64, _u64p, _u32p]),
    "wax_vs_absorb_rows": (C.c_int32, [_eng, _u64p, _u64p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, _u64p, _u64p]),
    "wax_vs_search": (C.c_int32, [_eng, _f32p, C.c_uint32, C.c_int64, _u64p, _f32p, C.c_uint32, _u32p]),
    "wax_vs_search_filtered": (C.c_int32, [_eng, _f32p, C.c_uint32, C.c_int64, _u64p, C.c_uint64, C.c_int32, _u64p, _f32p,
                                           C.c_uint32, _u32p]),
    "wax_vs_search_batch_filtered": (C.c_int32, [_eng, _f32p, C.c_uint32, C.c_uint32, C.c_int64, _u64p, C.c_uint64, C.c_int32,
                                                 _u64p, _f32p, C.c_uint32, _u32p]),
    "wax_vs_shard_search_filtered": (C.c_int32, [_eng, _f32p, C.c_uint32, C.c_int64, _u64p, C.c_uint64, C.c_int32, _u64p,
                                                 _f32p, C.c_uint32, _u32p]),
    "wax_vs_search_batch_multi_filtered": (C.c_int32, [_eng, _f32p, C.c_uint32, C.c_uint32, C.c_int64, _u64p, _u64p,
                                                       C.POINTER(C.c_int32), C.c_uint32, _u32p, _u64p, _f32p, C.c_uint32,
                                                       _u32p]),
    "wax_vs_set_groups": (C.c_int32, [_eng, _u64p, _u64p, C.c_uint64, _u64p]),
    "wax_vs_search_grouped": (C.c_int32, [_eng, _f32p, C.c_uint32, C.c_int64, C.c_uint32, _u64p, C.c_uint64, C.c_int32,
                                          _u64p, _f32p, _u64p, C.c_uint32, _u32p]),
    "wax_vs_search_batch_grouped": (C.c_int32, [_eng, _f32p, C.c_uint32, C.c_uint32, C.c_int64, C.c_uint32, _u64p,
                                                C.c_uint64, C.c_int32, _u64p, _f32p, _u64p, C.c_uint32, _u32p]),
    "wax_vs_set_attributes": (C.c_int32, [_eng, _u64p, C.POINTER(C.c_int64), _u64p, C.c_uint64, _u64p]),
    "wax_vs_search_batch_where": (C.c_int32, [_eng, _f32p, C.c_uint32, C.c_uint32, C.c_int64, _u64p, _u64p,
                                              C.POINTER(C.c_int32), C.c_uint32, _u32p, C.c_void_p, C.c_uint32, _u32p,
                                              _u64p, _f32p, C.c_uint32, _u32p]),
    "wax_vs_search_batch_grouped_where": (C.c_int32, [_eng, _f32p, C.c_uint32, C.c_uint32, C.c_int64, C.c_uint32, _u64p,
                                                      C.c_uint64, C.c_int32, C.c_void_p, _u64p, _f32p, _u64p, C.c_uint32,
                                                      _u32p]),
    "wax_vs_set_locations": (C.c_int32, [_eng, _u64p, _f64p, _f64p, C.c_uint64, _u64p]),
    "wax_vs_location_box": (C.c_int32, [C.c_double, C.c_double, C.c_double, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "wax_vs_location_bin": (C.c_int32, [C.c_double, C.c_double, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "wax_vs_search_batch_where_near": (C.c_int32, [_eng, _f32p, C.c_uint32, C.c_uint32, C.c_int64, _u64p, _u64p,
                                                   C.POINTER(C.c_int32), C.c_uint32, _u32p, C.c_void_p, C.c_uint32,
                                                   _u32p, _u64p, _f32p, C.c_uint32, _u32p]),
    "wax_vs_search_batch_grouped_where_near": (C.c_int32, [_eng, _f32p, C.c_uint32, C.c_uint32, C.c_int64, C.c_uint32,
                                                           _u64p, C.c_uint64, C.c_int32, C.c_void_p, _u64p, _f32p, _u64p,
                                                           C.c_uint32, _u32p]),
    "wax_vs_search_batch_grouped_multi_where": (C.c_int32, [_eng, _f32p, C.c_uint32, C.c_uint32, C.c_int64, C.c_uint32,
                                                            _u64p, _u64p, C.POINTER(C.c_int32), C.c_uint32, _u32p,
                                                            C.c_void_p, C.c_uint32, _u32p, _u64p, _f32p, _u64p,
                                                            C.c_uint32, _u32p]),
    "wax_vs_set_terms": (C.c_int32, [_eng, _u64p, _u64p, _u64p, C.c_uint64, _u64p]),
    "wax_vs_search_batch_where_terms": (C.c_int32, [_eng, _f32p, C.c_uint32, C.c_uint32, C.c_int64, _u64p, _u64p,
                                                    C.POINTER(C.c_int32), C.c_uint32, _u32p, C.c_void_p, C.c_uint32,
                                                    _u32p, _u64p, _u64p, _u64p, _f32p, C.c_uint32, _u32p]),
    "wax_vs_search_batch_where_groups": (C.c_int32, [_eng, _f32p, C.c_uint32, C.c_uint32, C.c_int64, _u64p, _u64p,
                                                     C.POINTER(C.c_int32), C.c_uint32, _u32p, C.c_void_p, C.c_uint32,
                                                     _u32p, _u64p, _u64p, _u64p, _u64p, _u64p, _f32p, C.c_uint32, _u32p]),
    "wax_vs_search_batch_grouped_multi_where_groups": (C.c_int32, [_eng, _f32p, C.c_uint32, C.c_uint32, C.c_int64,
                                                                   C.c_uint32, _u64p, _u64p, C.POINTER(C.c_int32),
                                                                   C.c_uint32, _u32p, C.c_void_p, C.c_uint32, _u32p,
                                                                   _u64p, _u64p, _u64p, _f32p, _u64p, C.c_uint32, _u32p]),
    "wax_vs_set_root_tags": (C.c_int32, [_eng, _u64p, _u64p, C.c_uint64, _u64p]),
    "wax_vs_search_batch_where_roots": (C.c_int32, [_eng, _f32p, C.c_uint32, C.c_uint32, C.c_int64, _u64p, _u64p,
                                                    C.POINTER(C.c_int32), C.c_uint32, _u32p, C.c_void_p, C.c_uint32,
                                                    _u32p, _u64p, _u64p, _u64p, _u64p, C.c_void_p, _u64p, _f32p,
                                                    C.c_uint32, _u32p]),
    "wax_vs_search_batch_grouped_multi_where_roots": (C.c_int32, [_eng, _f32p, C.c_uint32, C.c_uint32, C.c_int64,
                                                                  C.c_uint32, _u64p, _u64p, C.POINTER(C.c_int32),
                                                                  C.c_uint32, _u32p, C.c_void_p, C.c_uint32, _u32p,
                                                                  _u64p, _u64p, C.c_void_p, _u64p, _f32p, _u64p,
                                                                  C.c_uint32, _u32p]),
    "wax_vs_shard_search_where": (C.c_int32, [_eng, _f32p, C.c_uint32, C.c_int64, _u64p, C.c_uint64, C.c_int32, C.c_void_p,
                                              _u64p, C.c_uint32, _u64p, _f32p, C.c_uint32, _u32p]),
    "wax_vs_search_batch_where_device": (C.c_int32, [_eng, C.c_void_p, C.c_uint32, C.c_int64, _u64p, _u64p,
                                                     C.POINTER(C.c_int32), C.c_uint32, _u32p, C.c_void_p, C.c_uint32, _u32p,
                                                     _u64p, _u64p, C.c_uint64, C.c_void_p, C.c_void_p]),
    "wax_vs_shard_grouped_heads_device": (C.c_int32, [_eng, C.c_void_p, C.c_uint32, C.c_int64, C.c_uint32, _u64p, _u64p,
                                                      C.POINTER(C.c_int32), C.c_uint32, _u32p, C.c_void_p, C.c_uint32,
                                                      _u32p, C.c_uint64, C.c_void_p, C.c_void_p]),
    "wax_vs_merge_group_heads_device": (C.c_int32, [_eng, C.c_void_p, C.c_uint32, C.c_uint32, C.c_int64, C.c_uint32,
                                                    C.c_void_p, C.c_void_p]),
    "wax_vs_shard_grouped_expand_device": (C.c_int32, [_eng, C.c_void_p, C.c_uint32, C.c_int64, C.c_uint32, _u64p, _u64p,
                                                       C.POINTER(C.c_int32), C.c_uint32, _u32p, C.c_void_p, C.c_uint32,
                                                       _u32p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p,
                                                       C.c_void_p]),
    "wax_vs_search_batch": (C.c_int32, [_eng, _f32p, C.c_uint32, C.c_uint32, C.c_int64, _u64p, _f32p,
                                        C.c_uint32, _u32p]),
    "wax_vs_search_device": (C.c_int32, [_eng, C.c_void_p, C.c_uint32, C.c_int64, C.c_uint64, C.c_void_p,
                                         C.c_void_p]),
    "wax_vs_search_batch_device": (C.c_int32, [_eng, C.c_void_p, C.c_uint32, C.c_int64, C.c_uint64, C.c_void_p,
                                               C.c_void_p]),
    "wax_vs_merge_candidates_device": (C.c_int32, [_eng, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                                   C.c_void_p, C.c_void_p]),
    "wax_vs_shard_open": (C.c_int32, [_eng, C.c_int32, C.c_int32, C.c_uint64, _u8p]),
    "wax_vs_shard_connect": (C.c_int32, [_eng, _u8p, C.c_int32]),
    "wax_vs_shard_close": (C.c_int32, [_eng]),
    "wax_vs_shard_search": (C.c_int32, [_eng, _f32p, C.c_uint32, C.c_int64, _u64p, _f32p, C.c_uint32, _u32p]),
    "wax_vs_shard_search_device": (C.c_int32, [_eng, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "wax_vs_serialized_length": (C.c_int32, [_eng, _u64p]),
    "wax_vs_serialize": (C.c_int32, [_eng, _u8p, C.c_uint64, _u64p]),
    "wax_vs_deserialize": (C.c_int32, [_eng, _u8p, C.c_uint64]),
    "wax_vs_last_error": (C.c_char_p, []),
    "wax_vs_debug_pool_stats": (C.c_int32, [_eng, _u64p, _u64p]),
    "wax_vs_debug_fill_synthetic": (C.c_int32, [_eng, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, C.c_int32]),
    "wax_vs_debug_read_rows": (C.c_int32, [_eng, C.c_uint64, C.c_uint64, _f32p]),
    "wax_vs_debug_time_search": (C.c_int32, [_eng, C.c_uint32, C.c_int64, C.c_uint64, C.c_uint32, C.c_uint32,
                                             _f32p, _u64p]),
    "wax_vs_debug_time_shard_search": (C.c_int32, [_eng, C.c_uint32, C.c_int64, C.c_uint64, C.c_uint32, C.c_uint32,
                                                   _f32p, _u64p]),
    "wax_vs_debug_transfer_probe": (C.c_int32, [_eng, C.c_uint64, _f32p]),
    "wax_vs_debug_phase_trace": (C.c_int32, [_eng, C.c_int64, C.c_uint32, _f32p]),
    "wax_vs_debug_batch_stats": (C.c_int32, [_eng, _u64p, _u64p]),
    "wax_vs_debug_counter": (C.c_int32, [_eng, C.c_char_p, _u64p]),
    "wax_vs_debug_last_scan": (C.c_int32, [_eng, _u32p]),
    "wax_vs_debug_time_search_batch": (C.c_int32, [_eng, C.c_uint32, C.c_int64, C.c_uint64, C.c_uint32, C.c_uint32,
                                                   _f32p, _u64p, _u32p]),
    "wax_vs_debug_batch_nominations": (C.c_int32, [_eng, _f32p, C.c_uint32, C.c_int64, _u32p, _f32p, _u32p, _u64p,
                                                   C.c_uint64, _u32p]),
    "wax_vs_debug_shadow_nominations": (C.c_int32, [_eng, _f32p, C.c_int64, _u32p, _u64p, _u32p, C.POINTER(Candidate),
                                                    _u32p]),
    "wax_vs_debug_read_shadow": (C.c_int32, [_eng, C.c_uint64, C.c_uint64, C.POINTER(C.c_uint16)]),
    "wax_vs_debug_int8_nominations": (C.c_int32, [_eng, _f32p, C.c_int64, _u32p, _u64p, _u32p, C.POINTER(Candidate),
                                                  _u32p]),
    "wax_vs_debug_read_int8_shadow": (C.c_int32, [_eng, C.c_uint64, C.c_uint64, _u8p, _f32p, _f32p]),
    "wax_vs_debug_u4_nominations": (C.c_int32, [_eng, _f32p, C.c_int64, _u32p, _u64p, C.c_uint64, _u32p,
                                                C.POINTER(Candidate), _u32p, _f32p]),
    "wax_vs_debug_read_u4_shadow": (C.c_int32, [_eng, C.c_uint64, C.c_uint64, _u8p, _f32p, _f32p]),
    "wax_vs_debug_stream_read": (C.c_int32, [_eng, C.c_uint32, _f32p, _u64p]),
    "wax_vs_debug_set_option": (C.c_int32, [_eng, C.c_char_p, C.c_int64]),
    "wax_vs_version": (C.c_char_p, []),
}

_lib = None


def lib() -> C.CDLL:
    """Load libwaxvs_cuda.so; raise loudly when it has not been built (no fallback exists)."""
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise ImportError(
                f"{LIB_PATH} is missing: the CUDA extension is the only implementation of the vector scan. "
                "Build it with `python -m wax_b200.build` (or __graft_entry__.build()).")
        handle = C.CDLL(str(LIB_PATH))
        for name, (restype, argtypes) in SIGNATURES.items():
            fn = getattr(handle, name)  # AttributeError if a declared symbol is not exported
            fn.restype = restype
            fn.argtypes = argtypes
        _lib = handle
    return _lib


def last_error() -> str:
    return lib().wax_vs_last_error().decode("utf-8", "replace")
