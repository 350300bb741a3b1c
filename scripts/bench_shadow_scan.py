#!/usr/bin/env python
"""Single-query bf16-shadow route against the fp32 scan (DESIGN 4.1) -- companion of bench.py, same conventions:
device-only times (queries resident in HBM, CUDA events on the launching stream inside the library), one query in
flight.  In one process and one engine the fp32 scan (option shadow_scan = 0) and the default route alternate, round by
round, so that both see the same clocks and the same HBM.

    python scripts/bench_shadow_scan.py [--rounds 5] [--steps 50] [--out FILE] [--sweep] [--tune]

Reports ms per query of both routes, their ratio and the spread over the rounds, the fallbacks counted, GB/s over the
SHADOW bytes (what the route reads: rows * dims * 2 per query, plus the re-scored nominees) against the same run's plain
read of the fp32 corpus (stream_read_gbs), the cost of the first search after fill_synthetic and after a remove (the
shadow builds then), k = 1 / 10 / 32, 10 M x 768 dot, and with --sweep the corpus sizes 10 K .. 10 M that set the
route's size threshold.  --tune alternates shapes of the SHADOW form (rows per step, warps, ring depth) on 10 M x 384.
Prints one JSON line (and writes it to --out)."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from wax_b200 import CUDAVectorEngine, VectorMetric  # noqa: E402

N_DISTINCT, SEED = 64, 1002


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except Exception as ex:  # noqa: BLE001
        return repr(ex)


def per_query_ms(eng, k, steps, warmup=3):
    ms, launches = eng.time_search(k, steps, warmup=warmup, n_queries=N_DISTINCT, seed=SEED)
    return ms / steps, launches / steps


def counts(eng):
    return eng.counter("single_shadow_queries"), eng.counter("single_shadow_fallbacks")


def alternate(eng, k, rounds, steps):
    """rounds x (fp32 scan, default route), steps device-timed queries each."""
    fp32, route, launches = [], [], None
    q0, f0 = counts(eng)
    for _ in range(rounds):
        eng.set_option("shadow_scan", 0)
        fp32.append(per_query_ms(eng, k, steps)[0])
        eng.set_option("shadow_scan", 1)
        ms, launches = per_query_ms(eng, k, steps)
        route.append(ms)
    q1, f1 = counts(eng)
    m_fp32, m_route = float(np.median(fp32)), float(np.median(route))
    return {"k": k, "fp32_ms": m_fp32, "route_ms": m_route, "speedup": m_fp32 / m_route,
            "fp32_ms_rounds": fp32, "route_ms_rounds": route,
            "route_spread_pct": (max(route) - min(route)) / m_route * 100, "fp32_spread_pct": (max(fp32) - min(fp32)) / m_fp32 * 100,
            "route_launches_per_query": launches, "route_queries": q1 - q0, "fallbacks": f1 - f0}


def first_search_ms(eng, dims, seed):
    """Wall time of one synchronous search (host query in, host result out)."""
    q = np.random.default_rng(seed).standard_normal(dims).astype(np.float32)
    t = time.perf_counter()
    eng.search(q, 10)
    return (time.perf_counter() - t) * 1e3


def headline(args):
    rows, dims = 10_000_000, 384
    eng = CUDAVectorEngine(VectorMetric.cosine, dims)
    eng.fill_synthetic(2, rows)
    out = {"workload": f"{rows} x {dims} fp32 cosine, one query in flight, {N_DISTINCT} distinct queries"}
    out["first_search_after_fill_ms"] = first_search_ms(eng, dims, 1)          # norms + shadow build
    out["steady_search_ms"] = float(np.median([first_search_ms(eng, dims, 2 + i) for i in range(5)]))
    eng.time_search(10, 20, warmup=0, n_queries=N_DISTINCT, seed=SEED)           # settle
    out["k"] = [alternate(eng, k, args.rounds, args.steps) for k in (10, 1, 32)]
    read = eng.stream_read_gbs(5)
    r10 = out["k"][0]
    shadow_bytes = rows * dims * 2
    out["stream_read_gbs"] = read
    out["route_gbs_on_shadow_bytes"] = shadow_bytes / (r10["route_ms"] * 1e-3) / 1e9
    out["fp32_gbs_on_corpus_bytes"] = rows * dims * 4 / (r10["fp32_ms"] * 1e-3) / 1e9
    eng.remove(123)
    out["first_search_after_remove_ms"] = first_search_ms(eng, dims, 3)        # shadow rebuild
    out["steady_search_after_remove_ms"] = float(np.median([first_search_ms(eng, dims, 4 + i) for i in range(5)]))
    if args.tune:
        out["tune"] = tune(eng, args)
    eng.close()
    return out


def tune(eng, args):
    """Shapes of the SHADOW form (its own options: the guarded fp32 scan keeps its shape), alternated round by round;
    0 = the engine's default."""
    shapes = [(0, 0, 0), (8, 8, 3), (8, 12, 2), (8, 16, 2), (4, 16, 2), (4, 16, 3), (16, 8, 2), (4, 12, 3)]
    cands = [dict(shadow_rows_per_step=r, shadow_warps=w, shadow_stages=s) for r, w, s in shapes]
    times, proven, failed = [[] for _ in cands], [0] * len(cands), [0] * len(cands)
    for _ in range(args.rounds):
        for i, c in enumerate(cands):
            for key, v in c.items():
                eng.set_option(key, v)
            q0, f0 = counts(eng)
            times[i].append(per_query_ms(eng, 10, args.steps)[0])
            q1, f1 = counts(eng)
            proven[i] += q1 - q0
            failed[i] += f1 - f0
    for key in cands[0]:
        eng.set_option(key, 0)
    return [dict(c, ms=float(np.median(t)), ms_rounds=t, route_queries=p, fallbacks=f)
            for c, t, p, f in zip(cands, times, proven, failed)]


def dot768(args):
    rows, dims = 10_000_000, 768
    eng = CUDAVectorEngine(VectorMetric.dot, dims)
    eng.fill_synthetic(5, rows, normalize=False)
    eng.time_search(10, 10, warmup=0, n_queries=N_DISTINCT, seed=SEED)
    out = alternate(eng, 10, args.rounds, args.steps)
    out["workload"] = f"{rows} x {dims} fp32 dot (rows not normalised)"
    eng.close()
    return out


def sweep(args):
    res = []
    for rows in (10_000, 30_000, 100_000, 300_000, 500_000, 1_000_000, 3_000_000, 10_000_000):
        eng = CUDAVectorEngine(VectorMetric.cosine, 384)
        eng.fill_synthetic(2, rows)
        eng.set_option("shadow_scan_min_bytes", 0)
        eng.time_search(10, 10, warmup=0, n_queries=N_DISTINCT, seed=SEED)
        r = alternate(eng, 10, args.rounds, args.steps)
        res.append({"rows": rows, "fp32_mb": rows * 384 * 4 / 2**20, "fp32_ms": r["fp32_ms"], "route_ms": r["route_ms"],
                    "speedup": r["speedup"], "fallbacks": r["fallbacks"]})
        eng.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--out", default=None)
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--tune", action="store_true")
    ap.add_argument("--no-dot", action="store_true")
    args = ap.parse_args()
    line = {"gpu": gpu_info(), "rounds": args.rounds, "steps_per_round": args.steps, "headline": headline(args)}
    if not args.no_dot:
        line["dot_768"] = dot768(args)
    if args.sweep:
        line["sweep"] = sweep(args)
    text = json.dumps(line)
    print(text, flush=True)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(line, indent=1) + "\n")


if __name__ == "__main__":
    main()
