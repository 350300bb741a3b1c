"""Grouped search (wax_vs_search_grouped) against the over-fetching plain searches Wax's PhotoRAG / VideoRAG issue today.

Corpus: 10 M x 384 cosine rows from fill_synthetic.  Every figure is the wall time of the public C call from host buffers
(median of --iters calls after warm-up, queries rotated).  Workloads:
  (a) groups of 8 consecutive rows, 12 groups x 1 row
  (b) groups of 360 consecutive rows, 12 groups x 3 rows
  (c) as (b) with hashed groups (not contiguous)
  (d) as (b) under an allow-list of 1 M frames
each beside wax_vs_search (wax_vs_search_filtered for (d)) at k = 12, 200 and 400.  For (b) and (c) it also counts how many
of the exact 12 groups / 36 rows a k = 400 over-fetch grouped on the host recovers.  Further: set_groups for 10 M frames, the
first grouped search after a mutation (index build) and the group-reduce / expansion kernel times (torch.profiler, in a
run of their own).  Prints one JSON line (also written to the file --out names, if given).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from wax_b200 import CUDAVectorEngine, VectorMetric  # noqa: E402
from wax_b200 import _lib as L  # noqa: E402

ROWS, DIMS = 10_000_000, 384


def _u64(a):
    return a.ctypes.data_as(C.POINTER(C.c_uint64))


def _f32(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


class Caller:
    """The public C calls with preallocated host buffers (no Python list building inside the timed region)."""

    def __init__(self, eng):
        self.h = eng.handle
        self.ids = np.zeros(L.MAX_RESULTS, np.uint64)
        self.scores = np.zeros(L.MAX_RESULTS, np.float32)
        self.groups = np.zeros(L.MAX_RESULTS, np.uint64)
        self.n = C.c_uint32(0)

    def grouped(self, q, top, per, allow=None):
        fp, nf, mode = (_u64(allow), allow.size, 0) if allow is not None else (None, 0, 1)
        rc = L.lib().wax_vs_search_grouped(self.h, _f32(q), q.size, top, per, fp, nf, mode, _u64(self.ids),
                                           _f32(self.scores), _u64(self.groups), L.MAX_RESULTS, C.byref(self.n))
        assert rc == L.OK, L.last_error()
        return self.n.value

    def plain(self, q, k, allow=None):
        if allow is None:
            rc = L.lib().wax_vs_search(self.h, _f32(q), q.size, k, _u64(self.ids), _f32(self.scores), L.MAX_RESULTS,
                                       C.byref(self.n))
        else:
            rc = L.lib().wax_vs_search_filtered(self.h, _f32(q), q.size, k, _u64(allow), allow.size, 0, _u64(self.ids),
                                                _f32(self.scores), L.MAX_RESULTS, C.byref(self.n))
        assert rc == L.OK, L.last_error()
        return self.n.value


def timed(fn, queries, iters, warmup):
    for i in range(warmup):
        fn(queries[i % len(queries)])
    ts = []
    for i in range(iters):
        t0 = time.perf_counter()
        fn(queries[i % len(queries)])
        ts.append((time.perf_counter() - t0) * 1e3)
    return round(statistics.median(ts), 3)


def recovery(caller, eng, q, group_of, top, per, allow=None):
    """How much of the exact answer a k = 400 over-fetch grouped on the host (parentId ?? id, best rows first) finds."""
    exact = eng.search_grouped(q, top, per, allow=allow)
    n = caller.plain(q, 400, allow)
    picked = {}
    for f in caller.ids[:n].tolist():
        g = int(group_of(f))
        if g not in picked and len(picked) == top:
            continue
        picked.setdefault(g, [])
        if len(picked[g]) < per:
            picked[g].append(f)
    exact_groups = [g for g, _ in exact]
    exact_rows = {f for _, hits in exact for f, _ in hits}
    got_rows = {f for hits in picked.values() for f in hits}
    return {"groups": sum(g in picked for g in exact_groups), "of_groups": len(exact_groups),
            "rows": len(exact_rows & got_rows), "of_rows": len(exact_rows)}


def kernel_times(eng, q, workloads):
    """Device time of the grouped-search kernels per call, from torch.profiler (CUPTI) in a run of its own."""
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
    except Exception as exc:          # pragma: no cover - reported, not hidden
        return {"error": f"torch.profiler unavailable: {exc}"}
    out = {}
    for name, (setup, top, per, allow) in workloads.items():
        setup()
        eng.search_grouped(q, top, per, allow=allow)                   # build the index outside the trace
        reps = 5
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                eng.search_grouped(q, top, per, allow=allow)
            torch.cuda.synchronize()
        acc = {}
        for ev in prof.events():
            if ev.device_type is not None and "CUDA" in str(ev.device_type):
                key = ev.name.split("<")[0].split("(")[0].replace("void ", "").replace("waxvs::", "").strip()
                acc[key] = acc.get(key, 0.0) + ev.device_time / reps / 1e3
        out[name] = {k: round(v, 4) for k, v in sorted(acc.items(), key=lambda kv: -kv[1])[:12]}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=ROWS)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    rows = args.rows
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    eng = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    eng.fill_synthetic(1, rows)
    call = Caller(eng)
    rng = np.random.default_rng(0)
    queries = [np.ascontiguousarray(q) for q in rng.standard_normal((8, DIMS)).astype(np.float32)]
    queries = [q / np.linalg.norm(q) for q in queries]
    frames = np.arange(rows, dtype=np.uint64)
    n_hashed = rows // 360
    layouts = {
        "blocks8": lambda f: f // 8 * 8,
        "blocks360": lambda f: f // 360 * 360,
        "hashed360": lambda f: (f * 2654435761) % n_hashed + 10**12,
    }
    allow = np.sort(rng.choice(rows, min(1_000_000, rows), replace=False)).astype(np.uint64)
    res = {"gpu": smi, "rows": rows, "dims": DIMS, "metric": "cosine", "iters": args.iters, "unit": "ms (median wall time)"}

    t0 = time.perf_counter()
    eng.set_groups(frames, layouts["blocks8"](frames))
    res["set_groups_10m_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
    t0 = time.perf_counter()
    call.grouped(queries[0], 12, 1)
    res["first_grouped_after_mutation_ms"] = round((time.perf_counter() - t0) * 1e3, 2)

    base = {k: timed(lambda q, k=k: call.plain(q, k), queries, args.iters, args.warmup) for k in (12, 200, 400)}
    base_f = {k: timed(lambda q, k=k: call.plain(q, k, allow), queries, args.iters, args.warmup) for k in (12, 200, 400)}
    work = {}
    work["a_blocks8_12x1"] = timed(lambda q: call.grouped(q, 12, 1), queries, args.iters, args.warmup)
    eng.set_groups(frames, layouts["blocks360"](frames))
    call.grouped(queries[0], 12, 3)
    work["b_blocks360_12x3"] = timed(lambda q: call.grouped(q, 12, 3), queries, args.iters, args.warmup)
    work["d_blocks360_12x3_allow1m"] = timed(lambda q: call.grouped(q, 12, 3, allow), queries, args.iters, args.warmup)
    rec = {"b": recovery(call, eng, queries[0], layouts["blocks360"], 12, 3)}
    eng.set_groups(frames, layouts["hashed360"](frames))
    call.grouped(queries[0], 12, 3)
    work["c_hashed360_12x3"] = timed(lambda q: call.grouped(q, 12, 3), queries, args.iters, args.warmup)
    rec["c"] = recovery(call, eng, queries[0], layouts["hashed360"], 12, 3)
    res.update(search_k=base, search_filtered_allow1m_k=base_f, grouped=work, overfetch400_recovers=rec)
    res["grouped_over_search400"] = {k: round(v / (base_f[400] if k.startswith("d") else base[400]), 3)
                                     for k, v in work.items()}
    res["kernels_ms_per_call"] = kernel_times(eng, queries[0], {
        "a": (lambda: eng.set_groups(frames, layouts["blocks8"](frames)), 12, 1, None),
        "b": (lambda: eng.set_groups(frames, layouts["blocks360"](frames)), 12, 3, None),
        "c": (lambda: eng.set_groups(frames, layouts["hashed360"](frames)), 12, 3, None),
    })
    eng.close()
    line = json.dumps(res)
    print(line, flush=True)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
