"""Multi-device rebalance: what `CUDAVectorEngine.rebalance()` costs after a skewing bulk delete.

    python scripts/bench_multi_rebalance.py [record] [--rows N] [--dims D] [--reps K]

Cosine, 10 M x 384 by default, filled as bench_multi_device.py fills it (timestamps and groups set, so every moved row
takes its attributes and group along).  One phase per R in (2, 4) with devices [0] * R: the same 30 % of the rows are
removed, the rows of the lower half of the shards, which leaves the shards skewed; then one `rebalance`.  The single
engine is filled once and the handles take turns beside it, as in bench_multi_device.py.  Reported per phase:
  - rows and bytes moved, the wall seconds of `rebalance` and the effective GB/s (bytes moved / seconds);
  - the first single query and the first batch of 1 024 after it (they rebuild the receivers' shadows and norms),
    against the steady-state medians of the same calls before and after it;
  - that every sampled answer equals one engine's with the same history.
On one GPU the shards share it: these figures are the cost of the move, not the latency a balanced handle gains on
several GPUs, which is not measured here.  The card's name and power limit are read in the same run.  `record` writes
the JSON to scripts/records/bench_multi_rebalance_h100.json.
"""
import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from bench_multi_device import card, fill  # noqa: E402
from wax_b200 import CUDAVectorEngine, VectorMetric  # noqa: E402


def skew_ids(rows, fraction, chunk=1_000_000):
    """The ids a removal of `fraction` of the rows takes: the first half of each 1 M chunk, chunk by chunk.  fill() adds
    each chunk to shards of equal size, so each chunk splits in R contiguous parts in shard order and the removed rows
    are those of the lower half of the shards (shard 0 of 2; shards 0 and 1 of 4)."""
    ids = np.arange(rows, dtype=np.uint64)
    return ids[ids % chunk < chunk // 2][:int(rows * fraction)]


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

    def one_query(e, rep):
        return e.search(singles[rep % a.reps], 10)

    def one_batch(e, rep):
        return [x.tobytes() for x in e.search_batch_arrays(batch, 10)]

    def timed(fn, e, rep):
        t0 = time.perf_counter()
        out = fn(e, rep)
        return (time.perf_counter() - t0) * 1e3, out

    def steady(multi, one):
        """Median ms of the handle's calls; every answer checked against one engine's."""
        ms = {"search_k10_ms": [], "batch1024_top10_ms": []}
        for rep in range(a.reps + 1):                           # round 0 warms every shape up
            for name, fn in (("search_k10_ms", one_query), ("batch1024_top10_ms", one_batch)):
                t, got = timed(fn, multi, rep)
                assert got == fn(one, rep), (name, rep)
                if rep:
                    ms[name].append(t)
        return {m: float(np.median(v)) for m, v in ms.items()}

    one = CUDAVectorEngine(VectorMetric.cosine, a.dims)
    result = {"card": card(), "corpus": f"{a.rows} x {a.dims} cosine", "removed_fraction": 0.3, "reps": a.reps,
              "phases": {}}
    gone = skew_ids(a.rows, 0.3)
    for r in (2, 4):
        multi = CUDAVectorEngine(VectorMetric.cosine, a.dims, devices=[0] * r)
        fill([multi] + ([one] if r == 2 else []), a.rows, a.dims, seed=0)
        assert multi.remove_batch(gone) == gone.size
        if r == 2:
            assert one.remove_batch(gone) == gone.size
        phase = {"shard_rows_before": [multi.counter(f"shard_rows.{s}") for s in range(r)],
                 "steady_before": steady(multi, one)}
        t0 = time.perf_counter()
        moved = multi.rebalance()
        seconds = time.perf_counter() - t0
        phase["shard_rows_after"] = [multi.counter(f"shard_rows.{s}") for s in range(r)]
        t, got = timed(one_query, multi, 0)
        assert got == one_query(one, 0)
        phase["first_search_k10_after_ms"] = t
        t, got = timed(one_batch, multi, 0)
        assert got == one_batch(one, 0)
        phase["first_batch1024_top10_after_ms"] = t
        phase["steady_after"] = steady(multi, one)
        phase.update({"rows_moved": moved, "bytes_moved": moved * a.dims * 4, "rebalance_s": seconds,
                      "effective_GBps": moved * a.dims * 4 / seconds / 1e9 if seconds > 0 else None,
                      "second_rebalance_moved": multi.rebalance()})
        assert multi.count == one.count
        result["phases"][f"R={r}"] = phase
        multi.close()
    result["answers_equal"] = True
    one.close()
    print(json.dumps(result, indent=2))
    if a.record:
        path = Path(__file__).resolve().parent / "records" / "bench_multi_rebalance_h100.json"
        path.write_text(json.dumps(result, indent=2) + "\n")


if __name__ == "__main__":
    main()
