"""Multi-process rebalance: what `ShardedVectorEngine.rebalance()` costs after a skewing bulk delete.

    python scripts/bench_shard_rebalance.py [record] [--rows N] [--dims D] [--reps K]

Two ranks under gloo, both engines on device 0.  Cosine, 10 M x 384 by default, filled through the collective add_batch in
chunks of 1 M rows with timestamps and groups set (so every moved row takes its attributes and group along); then 30 % of
the rows, all held by rank 0, are removed and `rebalance()` evens the ranks out.  Reported:
  - rows and bytes moved and the wall seconds of `rebalance()` (every rank waits at a barrier before and after it);
  - each rank's own engine, timed before and after: one query at k = 10 and a batch of 1 024 at k = 10, the first call
    after the rebalance (the receiver rebuilds its shadows and norms) and the steady-state median.  A sharded search waits
    for the slowest rank;
  - whether the sharded serialize() bytes equal those of one engine with the same history (SHA-256 of each).
Two ranks sharing one GPU over gloo measure the protocol's cost: the rows cross the host twice.  Neither NVLink
transfer nor the multi-GPU latency a balanced corpus gains is measured here.  The card's name and power limit are read
in the same run.  `record` writes the JSON to scripts/records/bench_shard_rebalance_h100.json.
"""
import argparse
import hashlib
import json
import os
import socket
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from bench_multi_device import card  # noqa: E402


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def rank_main(rank, world, port, a, out_dir):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from wax_b200 import CUDAVectorEngine, VectorMetric, sharded
    try:
        eng = sharded.ShardedVectorEngine(VectorMetric.cosine, a.dims, device=0)
        one = CUDAVectorEngine(VectorMetric.cosine, a.dims, device=0) if rank == 0 else None
        rng = np.random.default_rng(0)
        chunk = 1_000_000
        for lo in range(0, a.rows, chunk):
            n = min(chunk, a.rows - lo)
            vec = rng.standard_normal((n, a.dims), dtype=np.float32)
            ids = np.arange(lo, lo + n, dtype=np.uint64)
            eng.add_batch(ids, vec)
            if one is not None:
                one.add_batch(ids, vec)
        ids = np.arange(a.rows, dtype=np.uint64)
        for e in (eng, one):
            if e is not None:
                e.set_attributes(ids, ids.astype(np.int64))
                e.set_groups(ids, ids // 360)
        gone = [eng.engine.export_rows(0, int(a.rows * 0.3), vectors=False)[0] if rank == 0 else None]
        dist.broadcast_object_list(gone, src=0)
        assert eng.remove_batch(gone[0]) == gone[0].size
        if one is not None:
            one.remove_batch(gone[0])

        q_rng = np.random.default_rng(1)
        singles = q_rng.standard_normal((a.reps, a.dims), dtype=np.float32)
        batch = q_rng.standard_normal((1024, a.dims), dtype=np.float32)
        own = eng.engine

        def timed(fn):
            t0 = time.perf_counter()
            fn()
            return (time.perf_counter() - t0) * 1e3

        calls = {"search_k10_ms": lambda rep: own.search(singles[rep % a.reps], 10),
                 "batch1024_top10_ms": lambda rep: own.search_batch_arrays(batch, 10)}

        def steady():
            ms = {name: [] for name in calls}
            for rep in range(a.reps + 1):                       # round 0 warms every shape up
                for name, fn in calls.items():
                    t = timed(lambda: fn(rep))
                    if rep:
                        ms[name].append(t)
            return {m: float(np.median(v)) for m, v in ms.items()}

        mine = {"rows_before": own.count, "steady_before": steady()}
        dist.barrier()
        t0 = time.perf_counter()
        moved = eng.rebalance()
        dist.barrier()
        seconds = time.perf_counter() - t0
        mine["rows_after"] = own.count
        mine["first_search_k10_after_ms"] = timed(lambda: calls["search_k10_ms"](0))
        mine["first_batch1024_top10_after_ms"] = timed(lambda: calls["batch1024_top10_ms"](0))
        mine["steady_after"] = steady()
        mine["second_rebalance_moved"] = eng.rebalance()
        blob = eng.serialize()
        result = None
        if rank == 0:
            sharded_sha = hashlib.sha256(blob).hexdigest()
            del blob
            one_sha = hashlib.sha256(one.serialize()).hexdigest()
            result = {"rows_moved": moved, "bytes_moved": moved * a.dims * 4, "rebalance_s": seconds,
                      "serialize_equals_one_engine": sharded_sha == one_sha}
        every = [None] * world
        dist.all_gather_object(every, mine)
        if rank == 0:
            result["ranks"] = every
            Path(out_dir, "result.json").write_text(json.dumps(result))
            one.close()
        eng.close()
    finally:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("record", nargs="?")
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--dims", type=int, default=384)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    import torch.multiprocessing as mp
    with tempfile.TemporaryDirectory() as tmp:
        mp.spawn(rank_main, args=(2, _free_port(), a, tmp), nprocs=2, join=True)
        res = json.loads(Path(tmp, "result.json").read_text())
    out = {"card": card(), "corpus": f"{a.rows} x {a.dims} cosine, timestamps and groups set",
           "ranks": "2 processes under gloo, both on device 0", "removed": "30 % of the rows, all from rank 0",
           "reps": a.reps, **res}
    print(json.dumps(out, indent=2))
    assert out["serialize_equals_one_engine"]
    if a.record:
        path = Path(__file__).resolve().parent / "records" / "bench_shard_rebalance_h100.json"
        path.write_text(json.dumps(out, indent=2) + "\n")


if __name__ == "__main__":
    main()
