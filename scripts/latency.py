"""Kernel time and end-to-end latency across corpus sizes (single GPU), incl. BASELINE configs[0] (10K x 384)."""
import json
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import ctypes as C  # noqa: E402

from wax_b200 import CUDAVectorEngine, VectorMetric, _lib as L  # noqa: E402

out = []
rng = np.random.default_rng(0)
for rows in (10_000, 100_000, 174_000, 1_250_000, 2_500_000, 5_000_000, 10_000_000):
    eng = CUDAVectorEngine(VectorMetric.cosine, 384)
    eng.fill_synthetic(2, rows)
    q = rng.standard_normal(384).astype(np.float32)
    for _ in range(5):
        eng.search(q, 10)
    n = 200 if rows <= 2_500_000 else 50
    t0 = time.perf_counter()
    for _ in range(n):
        eng.search(q, 10)
    e2e_us = (time.perf_counter() - t0) / n * 1e6
    # the same call at the C-ABI with preallocated buffers (what a compiled host pays; the mirror adds numpy/tuple work)
    ids, scores, cnt = np.empty(10, np.uint64), np.empty(10, np.float32), C.c_uint32(0)
    args = (eng.handle, q.ctypes.data_as(C.POINTER(C.c_float)), 384, 10, ids.ctypes.data_as(C.POINTER(C.c_uint64)),
            scores.ctypes.data_as(C.POINTER(C.c_float)), 10, C.byref(cnt))
    fn = L.lib().wax_vs_search
    for _ in range(5):
        fn(*args)
    t0 = time.perf_counter()
    for _ in range(n):
        fn(*args)
    abi_us = (time.perf_counter() - t0) / n * 1e6
    ms, _ = eng.time_search(10, n, warmup=5, n_queries=8)
    ms72, _ = eng.time_search(72, n, warmup=5, n_queries=8)
    rec = {"rows": rows, "kernel_us_back_to_back": round(ms / n * 1e3, 2), "e2e_us_sync_call": round(e2e_us, 2), "e2e_us_c_abi_call": round(abi_us, 2),
           "gbs_kernel": round(rows * 384 * 4 / (ms / n) / 1e6, 1), "kernel_us_k72": round(ms72 / n * 1e3, 2)}
    out.append(rec); print(json.dumps(rec), flush=True)
    eng.close()
if len(sys.argv) > 1:                                   # optional: the records as one JSON file
    Path(sys.argv[1]).write_text(json.dumps(out, indent=1))
