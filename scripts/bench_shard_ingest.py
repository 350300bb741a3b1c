#!/usr/bin/env python
"""Corpus methods of the row-sharded engine at world 1 (ShardedVectorEngine without a process group, DESIGN.md section
4.15) against the same calls on one CUDAVectorEngine: 10 M x 384 cosine rows.
  add_batch   10 batches of 1 M new rows (appends), then 1 M rows of upserts spread over the corpus;
  remove_batch  1 M ids, every tenth frame;
  serialize   the whole corpus to MV2V bytes (the sharded form gathers keys and rows in chunks and places them by key);
  deserialize   those bytes back.
Each line reports wall seconds and rows per second of one call sequence (the host buffers are pageable numpy arrays),
the card's name and power limit, and whether the sharded bytes equal the single engine's.

usage: scripts/bench_shard_ingest.py [record.json]"""
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from wax_b200 import CUDAVectorEngine, VectorMetric, sharded  # noqa: E402

N, DIMS, BATCH = 10_000_000, 384, 1_000_000
record = Path(sys.argv[1]) if len(sys.argv) > 1 else None


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as ex:  # noqa: BLE001
        return {"gpu": "unknown", "power_limit": "unknown", "error": repr(ex)}


def timed(fn):
    t = time.perf_counter()
    out = fn()
    return time.perf_counter() - t, out


def run(eng, rows, upserts):
    """The call sequence; returns ({step: seconds}, MV2V bytes)."""
    sec = {}
    sec["add_batch"], _ = timed(lambda: [eng.add_batch(np.arange(i, i + BATCH, dtype=np.uint64) * 3, rows)
                                         for i in range(0, N, BATCH)])
    sec["add_batch_upsert"], _ = timed(lambda: eng.add_batch(upserts, rows))
    sec["remove_batch"], _ = timed(lambda: eng.remove_batch(np.arange(0, N, 10, dtype=np.uint64) * 3))
    sec["serialize"], blob = timed(eng.serialize)
    sec["deserialize"], _ = timed(lambda: eng.deserialize(blob))
    return sec, blob


def main():
    info = card()
    rng = np.random.default_rng(3)
    rows = rng.standard_normal((BATCH, DIMS), dtype=np.float32)
    rows /= np.linalg.norm(rows, axis=1, keepdims=True)
    upserts = np.sort(rng.choice(N, BATCH, replace=False)).astype(np.uint64) * 3
    counts = {"add_batch": N, "add_batch_upsert": BATCH, "remove_batch": N // 10, "serialize": N - N // 10,
              "deserialize": N - N // 10}
    lines = []
    single = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    single_sec, single_blob = run(single, rows, upserts)
    single.close()
    sh = sharded.ShardedVectorEngine(VectorMetric.cosine, DIMS)
    try:
        sh_sec, sh_blob = run(sh, rows, upserts)
        same = sh_blob == single_blob                      # bytearrays: compared in place
        count = sh.count()
    finally:
        sh.close()
    del single_blob, sh_blob
    for step, n in counts.items():
        lines.append({"step": step, "rows": n, "sharded_world1_s": sh_sec[step], "single_engine_s": single_sec[step],
                      "sharded_rows_per_s": n / sh_sec[step], "single_rows_per_s": n / single_sec[step],
                      "corpus": f"{N} x {DIMS} cosine", "bytes_equal": same, "final_count": count, **info})
        print(json.dumps(lines[-1]), flush=True)
    if record:
        record.parent.mkdir(parents=True, exist_ok=True)
        record.write_text(json.dumps({"note": "world 1 on one GPU: the host-side cost of the sharded corpus methods",
                                      "workloads": lines}, indent=1) + "\n")


if __name__ == "__main__":
    main()
