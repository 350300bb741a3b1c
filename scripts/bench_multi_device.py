"""Multi-device handle overhead: `CUDAVectorEngine(devices=[0] * R)` against one engine on the same corpus.

    python scripts/bench_multi_device.py [record] [--rows N] [--dims D] [--reps K]

Cosine, 10 M x 384 by default.  One phase per R in (2, 4): the single engine and a handle of R shards hold the same
corpus (the two with their shadows take about 60 GB of an 80 GB H100; a third engine would not fit, so the handles take
turns), and every timed call alternates between them.  Workloads, median wall times:
  - one `search` at k = 10;
  - a batch of 1 024 queries at top-10;
  - where: the batch under per-query 20 % time windows (`search_batch_where`);
  - grouped: the batch in groups of 360 rows, 12 groups x 3 frames (`search_batch_grouped`).
Every answer of the handle is compared with the single engine's.  On one GPU the shards share it, so these figures are
the handle's overhead, not multi-GPU scaling.  The card's name and power limit are read in the same run.  `record`
writes the JSON to scripts/records/bench_multi_device_h100.json.
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from wax_b200 import CUDAVectorEngine, VectorMetric, Where  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def fill(engines, rows, dims, seed):
    """The same corpus into every engine, 1 M rows at a time (the host never holds all of it); timestamps = row."""
    rng = np.random.default_rng(seed)
    chunk = 1_000_000
    for lo in range(0, rows, chunk):
        n = min(chunk, rows - lo)
        vec = rng.standard_normal((n, dims), dtype=np.float32)
        ids = np.arange(lo, lo + n, dtype=np.uint64)
        for e in engines:
            e.add_batch(ids, vec)
    ids = np.arange(rows, dtype=np.uint64)
    for e in engines:
        e.set_attributes(ids, ids.astype(np.int64))
        e.set_groups(ids, ids // 360)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("record", nargs="?")
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--dims", type=int, default=384)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    rng = np.random.default_rng(1)
    singles = rng.standard_normal((a.reps, a.dims), dtype=np.float32)
    batch = rng.standard_normal((1024, a.dims), dtype=np.float32)
    starts = rng.integers(0, int(a.rows * 0.8), 1024)
    wheres = [Where(after=int(s), before=int(s + a.rows // 5)) for s in starts[:64]]
    query_where = [i % len(wheres) for i in range(1024)]
    work = {
        "search_k10_ms": lambda e, rep: e.search(singles[rep], 10),
        "batch1024_top10_ms": lambda e, rep: [x.tobytes() for x in e.search_batch_arrays(batch, 10)],
        "where_20pct_batch1024_top10_ms": lambda e, rep: e.search_batch_where(batch, 10, wheres, query_where),
        "grouped_360_12x3_batch1024_ms": lambda e, rep: e.search_batch_grouped(batch, 12, 3),
    }
    one = CUDAVectorEngine(VectorMetric.cosine, a.dims)
    result = {"card": card(), "corpus": f"{a.rows} x {a.dims} cosine", "reps": a.reps, "median_ms": {}}
    for r in (2, 4):
        multi = CUDAVectorEngine(VectorMetric.cosine, a.dims, devices=[0] * r)
        fill([multi] + ([one] if r == 2 else []), a.rows, a.dims, seed=0)
        times = {"single": {m: [] for m in work}, f"R={r}": {m: [] for m in work}}
        for rep in range(a.reps + 1):                           # round 0 warms every shape up
            for m, fn in work.items():
                got = {}
                for name, e in (("single", one), (f"R={r}", multi)):   # alternating: the same noise for both
                    t0 = time.perf_counter()
                    got[name] = fn(e, rep % a.reps)
                    if rep:
                        times[name][m].append((time.perf_counter() - t0) * 1e3)
                assert got["single"] == got[f"R={r}"], (r, m, rep)
        for name, t in times.items():
            result["median_ms"].setdefault(name, {}).update({m: float(np.median(v)) for m, v in t.items()}
                                                           if name != "single" or r == 2 else {})
            if name == "single" and r == 4:
                result["median_ms"]["single (R=4 phase)"] = {m: float(np.median(v)) for m, v in t.items()}
        multi.close()
    result["answers_equal"] = True
    one.close()
    print(json.dumps(result, indent=2))
    if a.record:
        path = Path(__file__).resolve().parent / "records" / "bench_multi_device_h100.json"
        path.write_text(json.dumps(result, indent=2) + "\n")


if __name__ == "__main__":
    main()
