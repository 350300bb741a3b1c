"""wax_b200 -- H100-native (sm_90a) brute-force vector scan + top-k behind Wax's `VectorSearchEngine` surface.

Scope: the hot path named by BASELINE.json (SURVEY.md section 8) and nothing else.  The numeric work lives in
libwaxvs_cuda.so (wax_b200/csrc, C-ABI in include/wax_vs_cuda.h); this package is the host-side mirror of
the reference interface plus the row-sharded multi-GPU wrapper.
"""
from .engine import (CUDAVectorEngine, CapacityExceeded, EncodingError, InvalidToc, TermDictionary,
                     VectorEnginePreference, VectorMetric, VectorSearchSession, WaxError, Where, is_normalized_l2,
                     location_bin, location_box, normalize_l2)

__all__ = [
    "CUDAVectorEngine", "VectorSearchSession", "VectorMetric", "VectorEnginePreference", "WaxError",
    "EncodingError", "CapacityExceeded", "InvalidToc", "Where", "normalize_l2", "is_normalized_l2",
    "location_box", "location_bin", "TermDictionary",
]
