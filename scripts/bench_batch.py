#!/usr/bin/env python
"""Batched-query benchmark (BASELINE configs 3 and 5) -- companion of bench.py, same conventions:
`value` = device-only (queries resident in HBM, CUDA events on the launching stream inside the library),
`e2e` = through the public call (wax_vs_search_batch via the mirror) with HOST query/result buffers.
Prints one JSON line per config."""
import json
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from wax_b200 import CUDAVectorEngine, VectorMetric  # noqa: E402

TF32_NOMINAL_TFLOPS = 495.0    # dense TF32, H100 SXM data sheet (used when no measured peak is present)
BF16_NOMINAL_TFLOPS = 989.0    # dense BF16, H100 SXM data sheet
try:
    _peaks = json.loads((ROOT / "MEASURED_PEAKS.json").read_text())
except Exception:  # noqa: BLE001
    _peaks = {}
BF16_BURST = float(_peaks.get("bf16_tflops", BF16_NOMINAL_TFLOPS))            # cuBLAS bf16 8192^3, best of 10
BF16_SUSTAINED = float(_peaks.get("bf16_tflops_sustained", BF16_BURST))        # back to back for 4 s
CONFIGS = [
    dict(name="configs[2]: 10M x 384 fp32, batch 1024, top-10 cosine", metric=VectorMetric.cosine, rows=10_000_000,
         dims=384, batch=1024, k=10, normalize=True, seed=2),
    dict(name="configs[4]: 10M x 768 fp32 (rows not normalised), batch 256, top-100 dot", metric=VectorMetric.dot,
         rows=10_000_000, dims=768, batch=256, k=100, normalize=False, seed=5),
    # l2 on the tensor-core levels is opt-in (batch_l2) for now: the shapes of configs[2] and configs[4]
    dict(name="10M x 384 fp32, batch 1024, top-10 l2", metric=VectorMetric.l2, rows=10_000_000, dims=384, batch=1024,
         k=10, normalize=True, seed=2, options=dict(batch_l2=1)),
    dict(name="10M x 768 fp32 (rows not normalised), batch 256, top-100 l2", metric=VectorMetric.l2, rows=10_000_000,
         dims=768, batch=256, k=100, normalize=False, seed=5, options=dict(batch_l2=1)),
]
steps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
# nominations: "bf16" (default: bf16 wgmmas over the bf16 shadow of the corpus) or "tf32" (from the fp32 corpus)
nominate = sys.argv[2] if len(sys.argv) > 2 else "bf16"
options = [kv.split("=") for kv in sys.argv[3:]]          # engine tuning options, e.g. batch_pair=1 batch_ares=0
only = [int(v) for k, v in options if k == "only"]        # only=0 .. only=3: run just that config (repeatable)
options = [(k, v) for k, v in options if k != "only"]
for ci, cfg in enumerate(CONFIGS):
    if only and ci not in only:
        continue
    eng = CUDAVectorEngine(cfg["metric"], cfg["dims"])
    eng.fill_synthetic(cfg["seed"], cfg["rows"], normalize=cfg["normalize"])
    eng.set_option("batch_bf16", 1 if nominate == "bf16" else 0)
    cfg_options = list(cfg.get("options", {}).items()) + options
    for k, v in cfg_options:
        eng.set_option(k, int(v))
    ms, launches, bad = eng.time_search_batch(cfg["batch"], cfg["k"], steps, warmup=2)
    per = ms / steps
    flops = 2.0 * cfg["batch"] * cfg["rows"] * cfg["dims"]
    rng = np.random.default_rng(1)
    qs = rng.uniform(-1, 1, size=(cfg["batch"], cfg["dims"])).astype(np.float32)
    qs /= np.linalg.norm(qs, axis=1, keepdims=True)
    eng.search_batch_arrays(qs, cfg["k"])
    t0, f0 = eng.batch_stats()
    t = time.perf_counter()
    for _ in range(steps):
        ids, scores, ns = eng.search_batch_arrays(qs, cfg["k"])
    e2e_s = (time.perf_counter() - t) / steps
    res = [[(int(ids[0, 0]), float(scores[0, 0]))]]
    t1, f1 = eng.batch_stats()
    bf16 = eng.counter("batch_bf16_queries") > 0
    peak = BF16_BURST if bf16 else TF32_NOMINAL_TFLOPS
    single_ms, _ = eng.time_search(cfg["k"], 5, warmup=2, n_queries=2)
    line = {
        "metric": "queries/sec (batched)", "config": {"workload": cfg["name"]}, "value": cfg["batch"] / per * 1e3,
        "unit": "queries/s", "ms_per_batch": per, "steps": steps,
        "dtype": ("bf16" if bf16 else "tf32") + " nominate + f32 exact re-score",
        "roofline": {"bound": "tensor", "achieved": flops / (per * 1e-3) / 1e12, "peak": peak,
                     "unit": "TFLOP/s", "frac": flops / (per * 1e-3) / 1e12 / peak,
                     "peak_source": ("measured cuBLAS bf16 burst (MEASURED_PEAKS.json bf16_tflops)" if bf16 else
                                     "nominal dense TF32 (no measured TF32 figure in MEASURED_PEAKS.json)"),
                     "frac_of_sustained_cublas_bf16": flops / (per * 1e-3) / 1e12 / BF16_SUSTAINED if bf16 else None,
                     "frac_of_nominal": flops / (per * 1e-3) / 1e12 / (BF16_NOMINAL_TFLOPS if bf16 else TF32_NOMINAL_TFLOPS),
                     "useful_flops_per_launch": flops,
                     "hbm_floor_ms": cfg["rows"] * cfg["dims"] * (2 if bf16 else 4) / 7.5e12 * 1e3},
        "shadow_gb": eng.counter("shadow_bytes") / 1e9, "tf32_retry_queries": eng.counter("batch_retry_queries"),
        "filter_bf16_queries": eng.counter("batch_filter_bf16_queries"),
        "e2e": {"value": cfg["batch"] / e2e_s, "unit": "queries/s", "ms_per_batch": e2e_s * 1e3,
                "h2d_bytes_per_step": int(qs.nbytes), "d2h_bytes_per_step": cfg["batch"] * cfg["k"] * 24,
                "api": "wax_vs_search_batch (host queries -> host ids/scores arrays)"},
        "gpu_launches_per_batch": launches / steps, "unproven_queries_last_step": bad,
        "tensor_path_queries": t1 - t0, "exact_fallback_queries": f1 - f0,
        "single_query_path_ms": single_ms / 5, "speedup_vs_single_query_loop": (single_ms / 5) * cfg["batch"] / per,
        "check_top1": res[0][0], "options": dict(cfg_options),
    }
    print(json.dumps(line), flush=True)
    eng.close()
