#!/usr/bin/env python
"""Single-query shadow route against the fp32 scan (DESIGN 4.1) -- companion of bench.py, same conventions:
device-only times (queries resident in HBM, CUDA events on the launching stream inside the library), one query in
flight.  In one process and one engine the fp32 scan (option shadow_scan = 0), the route on the bf16 shadow
(int8_scan_min_bytes out of reach), the route on the int8 shadow (u4_scan_min_bytes out of reach) and the route on the
4-bit shadow alternate, round by round, so that all four see the same clocks and the same HBM.

    python scripts/bench_shadow_scan.py [--rounds 5] [--steps 50] [--out FILE] [--sweep] [--tune]

Reports ms per query of the three arms, their ratios and the spread over the rounds, the fallbacks counted, GB/s over
the shadow bytes (what a route reads: rows * dims * 2 per query for bf16, rows * (dims + 4) for int8 codes and scales,
rows * (dims / 2 + 4) for 4-bit codes and half steps)
against the same run's plain read of the fp32 corpus (stream_read_gbs), the cost of the first search after
fill_synthetic and after a remove (the shadow builds then), k = 1 / 10 / 32, 10 M x 768 dot, and with --sweep the corpus
sizes 10 K .. 10 M that set the size thresholds.  --tune alternates shapes of the U4 form (rows per step, warps, ring
depth) on 10 M x 384.
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
DEFAULT_INT8_MIN = 512 << 20     # the engine's default int8_scan_min_bytes (waxvs_engine.cu Tuning)


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


NO_INT8 = 1 << 62          # int8_scan_min_bytes that keeps every corpus on the bf16 shadow


def alternate(eng, k, rounds, steps, int8_min=0):
    """rounds x (fp32 scan, bf16 route, int8 route, 4-bit route), steps device-timed queries each; int8_min: the engine's
    int8_scan_min_bytes / u4_scan_min_bytes for the int8 and u4 arms (the default threshold, or 0 below it)."""
    arms = {"fp32": [], "bf16": [], "int8": [], "u4": []}
    seen = {a: [0, 0, 0] for a in arms}           # route queries, fallbacks, nominations of the arm's own form
    launches = {}
    for _ in range(rounds):
        for arm in arms:
            eng.set_option("shadow_scan", 0 if arm == "fp32" else 1)
            eng.set_option("int8_scan_min_bytes", NO_INT8 if arm == "bf16" else int8_min)
            eng.set_option("u4_scan_min_bytes", int8_min if arm == "u4" else NO_INT8)
            own = "single_u4_queries" if arm == "u4" else "single_int8_queries"
            (q0, f0), i0 = counts(eng), eng.counter(own)
            ms, launches[arm] = per_query_ms(eng, k, steps)
            (q1, f1), i1 = counts(eng), eng.counter(own)
            arms[arm].append(ms)
            seen[arm] = [seen[arm][0] + q1 - q0, seen[arm][1] + f1 - f0, seen[arm][2] + i1 - i0]
    eng.set_option("shadow_scan", 1)
    eng.set_option("int8_scan_min_bytes", int8_min)
    eng.set_option("u4_scan_min_bytes", int8_min)
    med = {a: float(np.median(t)) for a, t in arms.items()}
    out = {"k": k, "fp32_ms": med["fp32"], "bf16_ms": med["bf16"], "int8_ms": med["int8"],
           "u4_ms": med["u4"], "int8_vs_bf16": med["bf16"] / med["int8"], "int8_vs_fp32": med["fp32"] / med["int8"],
           "u4_vs_int8": med["int8"] / med["u4"]}
    for a, t in arms.items():
        out[f"{a}_ms_rounds"] = t
        out[f"{a}_spread_pct"] = (max(t) - min(t)) / med[a] * 100
        out[f"{a}_launches_per_query"] = launches[a]
    for a in ("bf16", "int8", "u4"):
        out[f"{a}_route_queries"], out[f"{a}_fallbacks"], out[f"{a}_{'u4' if a == 'u4' else 'int8'}_nominations"] = seen[a]
    return out


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
    out["k"] = [alternate(eng, k, args.rounds, args.steps, int8_min=DEFAULT_INT8_MIN) for k in (10, 1, 32)]
    read = eng.stream_read_gbs(5)
    r10 = out["k"][0]
    out["stream_read_gbs"] = read
    out["bf16_gbs_on_shadow_bytes"] = rows * dims * 2 / (r10["bf16_ms"] * 1e-3) / 1e9
    out["int8_gbs_on_shadow_bytes"] = rows * (dims + 4) / (r10["int8_ms"] * 1e-3) / 1e9     # codes + scales
    out["int8_frac_of_stream_read"] = out["int8_gbs_on_shadow_bytes"] / read
    out["u4_gbs_on_shadow_bytes"] = rows * (dims // 2 + 4) / (r10["u4_ms"] * 1e-3) / 1e9    # codes + half steps
    out["u4_frac_of_stream_read"] = out["u4_gbs_on_shadow_bytes"] / read
    out["fp32_gbs_on_corpus_bytes"] = rows * dims * 4 / (r10["fp32_ms"] * 1e-3) / 1e9
    eng.remove(123)
    out["first_search_after_remove_ms"] = first_search_ms(eng, dims, 3)        # shadow rebuild
    out["steady_search_after_remove_ms"] = float(np.median([first_search_ms(eng, dims, 4 + i) for i in range(5)]))
    if args.tune:
        out["tune"] = tune(eng, args)
    eng.close()
    return out


def tune(eng, args):
    """Shapes of the U4 form (its own options: the guarded fp32 scan keeps its shape), alternated round by round;
    0 = the engine's default."""
    shapes = [(0, 0, 0), (16, 16, 2), (16, 16, 4), (16, 12, 4), (16, 8, 6), (8, 16, 3), (8, 16, 4), (8, 16, 6)]
    cands = [dict(u4_rows_per_step=r, u4_warps=w, u4_stages=s) for r, w, s in shapes]
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
    out = alternate(eng, 10, args.rounds, args.steps, int8_min=DEFAULT_INT8_MIN)
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
        r = alternate(eng, 10, args.rounds, args.steps, int8_min=0)
        res.append({"rows": rows, "fp32_mb": rows * 384 * 4 / 2**20, "fp32_ms": r["fp32_ms"], "bf16_ms": r["bf16_ms"],
                    "int8_ms": r["int8_ms"], "int8_vs_bf16": r["int8_vs_bf16"], "int8_vs_fp32": r["int8_vs_fp32"],
                    "int8_fallbacks": r["int8_fallbacks"], "int8_nominations": r["int8_int8_nominations"],
                    "u4_ms": r["u4_ms"], "u4_vs_int8": r["u4_vs_int8"], "u4_fallbacks": r["u4_fallbacks"],
                    "u4_nominations": r["u4_u4_nominations"]})
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
