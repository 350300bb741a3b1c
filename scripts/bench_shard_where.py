#!/usr/bin/env python
"""Sharded where search against the single-engine where search on the same corpus: 10 M x 384 cosine rows
(fill_synthetic), timestamps increasing with the row plus seeded jitter, 1 % of the rows tagged deleted, top-10.  The
ranks are engines on ONE H100 (world 1, 2 and 4), so the numbers measure the sharded form's overhead on one device,
not multi-GPU scaling.  Workloads (those of scripts/bench_where.py):
  (a) 1 024 distinct random windows of 20 % of the rows;
  (b) no window, no_tags excluding the rows tagged deleted;
  (c) 1 024 windows of about 5 000 rows (the gather class);
  (e) a single query with a 20 % window, through the fused collective (wax_vs_shard_search_where, one thread per rank).
(a)-(c) run the batched device form: every rank's wax_vs_search_batch_where_device into its slice of one buffer (the
layout an all-gather leaves), one wax_vs_merge_candidates_device and one copy to the host; no all-gather is needed
on one device.  Each line reports the wall time of the sharded call and of CUDAVectorEngine.search_batch_where /
search_where on one engine, the card's name and power limit, and the answers that differ from the single engine's.

usage: scripts/bench_shard_where.py [record.json] [steps]"""
import ctypes as C
import json
import subprocess
import sys
import threading
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from wax_b200 import CUDAVectorEngine, VectorMetric, Where, sharded  # noqa: E402
from wax_b200 import _lib as L  # noqa: E402
from wax_b200.engine import _WhereArgs  # noqa: E402

N, DIMS, B, K = 10_000_000, 384, 1024, 10
DELETED = 1
record = Path(sys.argv[1]) if len(sys.argv) > 1 else None
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 3


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as ex:  # noqa: BLE001
        return {"gpu": "unknown", "power_limit": "unknown", "error": repr(ex)}


def timed(fn, n):
    out = fn()                                  # warm-up: every shape the timed window uses
    t = time.perf_counter()
    for _ in range(n):
        fn()
    return (time.perf_counter() - t) / n, out


def bits(hits):
    return [(i, np.float32(s).view(np.uint32).item()) for i, s in hits]


class Ranks:
    """`world` engines on this device holding contiguous shards of the synthetic corpus, connected as a shard group."""

    def __init__(self, world, ts, tags):
        self.world = world
        self.engines, self.ranges = [], []
        for r in range(world):
            lo, hi = sharded.shard_range(N, world, r)
            eng = CUDAVectorEngine(VectorMetric.cosine, DIMS)
            eng.fill_synthetic(2, hi - lo, first_row=lo, id_base=lo)
            eng.set_attributes(np.arange(lo, hi, dtype=np.uint64), ts[lo:hi], tags[lo:hi])
            self.engines.append(eng)
            self.ranges.append((lo, hi))
        blobs = [e.shard_open(r, world, self.ranges[r][0]) for r, e in enumerate(self.engines)]
        for e in self.engines:
            e.shard_connect(blobs)

    def batch_where(self, d_qs, wheres, query_where):
        import torch
        b = int(d_qs.shape[0])
        a = _WhereArgs(wheres, query_where, None, None, b)
        gathered = torch.empty(self.world * b * K * 24, dtype=torch.uint8, device="cuda")
        for r, eng in enumerate(self.engines):
            rc = L.lib().wax_vs_search_batch_where_device(eng.handle, C.c_void_p(d_qs.data_ptr()), b, K, *a.filter_args(),
                                                          *a.where_args(near=True), *a.term_args(), self.ranges[r][0],
                                                          C.c_void_p(gathered.data_ptr() + r * b * K * 24), None)
            assert rc == L.OK, L.last_error()
        merged = torch.empty(b * K * 24, dtype=torch.uint8, device="cuda")
        assert L.lib().wax_vs_merge_candidates_device(self.engines[0].handle, C.c_void_p(gathered.data_ptr()), self.world,
                                                      b, K, K, C.c_void_p(merged.data_ptr()), None) == L.OK
        best = merged.cpu().numpy().view(sharded.CAND_DTYPE).reshape(b, K)
        scores = sharded.score_from_distance(0, best["distance"])
        return [[(int(best["frame_id"][i, j]), float(scores[i, j])) for j in range(int(best["valid"][i].sum()))]
                for i in range(b)]

    def fused_where(self, q, where, iters):
        """iters collective calls back to back on one thread per rank; returns (seconds per call, rank 0's answer)."""
        out, errors = [None] * self.world, []
        start = threading.Barrier(self.world + 1)

        def work(r):
            try:
                start.wait()
                for _ in range(iters):
                    out[r] = self.engines[r].shard_search_where(q, K, where)
            except Exception as ex:  # noqa: BLE001
                errors.append(ex)
        threads = [threading.Thread(target=work, args=(r,)) for r in range(self.world)]
        [t.start() for t in threads]
        start.wait()
        t0 = time.perf_counter()
        [t.join() for t in threads]
        assert not errors, errors[:1]
        assert all(x == out[0] for x in out)
        return (time.perf_counter() - t0) / iters, out[0]

    def close(self):
        for e in self.engines:
            e.close()


def main():
    import torch
    info = card()
    rng = np.random.default_rng(11)
    ts = np.arange(N, dtype=np.int64) * 16 + rng.integers(0, 16, N)
    tags = np.zeros(N, np.uint64)
    tags[rng.choice(N, N // 100, replace=False)] = DELETED
    single = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    single.fill_synthetic(2, N, normalize=True)
    single.set_attributes(np.arange(N, dtype=np.uint64), ts, tags)
    qs = rng.uniform(-1, 1, size=(B, DIMS)).astype(np.float32)
    qs /= np.linalg.norm(qs, axis=1, keepdims=True)
    d_qs = torch.from_numpy(qs).cuda()

    def windows(rows, count):
        starts = rng.integers(0, N - rows, count)
        return [Where(after=int(ts[s]), before=int(ts[s + rows])) for s in starts]

    work = {
        "(a) 1024 windows of 20 %": (windows(N // 5, B), list(range(B))),
        "(b) no window, no_tags = deleted (1 %)": ([Where(no_tags=DELETED)], [0] * B),
        "(c) 1024 windows of 5 000 rows (gather)": (windows(5000, B), list(range(B))),
    }
    single_ms, single_ans = {}, {}
    for name, (wheres, qw) in work.items():
        s, single_ans[name] = timed(lambda: single.search_batch_where(qs, K, wheres, qw), steps)
        single_ms[name] = s * 1e3
    w_e = windows(N // 5, 1)[0]
    s, single_e = timed(lambda: single.search_where(qs[0], K, w_e), 20)
    single_ms["(e)"] = s * 1e3
    lines = []
    for world in (1, 2, 4):
        ranks = Ranks(world, ts, tags)
        try:
            for name, (wheres, qw) in work.items():
                s, got = timed(lambda: ranks.batch_where(d_qs, wheres, qw), steps)
                mism = sum(bits(got[i]) != bits(single_ans[name][i]) for i in range(B))
                lines.append({"workload": name, "world": world, "corpus": f"{N} x {DIMS} cosine, fill_synthetic",
                              "batch": B, "top_k": K, "steps": steps, "sharded_device_form_ms": s * 1e3,
                              "single_engine_ms": single_ms[name], "ratio": s * 1e3 / single_ms[name],
                              "mismatches": int(mism), **info})
                print(json.dumps(lines[-1]), flush=True)
            ranks.fused_where(qs[0], w_e, 3)                       # warm-up
            s, got = ranks.fused_where(qs[0], w_e, 20)
            lines.append({"workload": "(e) single query, 20 % window, fused collective", "world": world,
                          "corpus": f"{N} x {DIMS} cosine", "top_k": K, "sharded_fused_ms": s * 1e3,
                          "single_engine_ms": single_ms["(e)"], "ratio": s * 1e3 / single_ms["(e)"],
                          "mismatches": 0 if bits(got) == bits(single_e) else 1, **info})
            print(json.dumps(lines[-1]), flush=True)
        finally:
            ranks.close()
    single.close()
    if record:
        record.parent.mkdir(parents=True, exist_ok=True)
        record.write_text(json.dumps({"note": "ranks share one GPU: the sharded form's overhead, not multi-GPU scaling",
                                      "workloads": lines}, indent=1) + "\n")


if __name__ == "__main__":
    main()
