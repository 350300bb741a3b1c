#!/usr/bin/env python
"""Sharded grouped search against the single engine's search_batch_grouped_multi_where on the same corpus: 10 M x 384
cosine rows (fill_synthetic), batch 1 024.  The ranks are engines on ONE H100 (world 1, 2 and 4), so the numbers measure
the protocol's overhead on one device, not multi-GPU scaling.  Workloads:
  (a) groups of 8 consecutive rows, 12 groups x 1 row;
  (b) groups of 360 consecutive rows, 12 groups x 3 rows;
  (c) as (b) with hashed groups (each group's 360 rows spread over the corpus, so over every shard);
  (d) as (b) with a where of each query's own: a window of 20 % of the rows and a deleted skip (1 % of the rows).
The whole flow is timed: every rank's wax_vs_shard_grouped_heads_device into its slice of one buffer (the layout an
all-gather leaves), wax_vs_merge_group_heads_device, and for per_group > 1 every rank's wax_vs_shard_grouped_expand_device,
wax_vs_merge_candidates_device and one copy to the host; no all-gather is needed on one device.  Each line reports the
wall time of the flow and of the single engine's call, the ranks' round-2 expansions (counter
"shard_grouped_expanded_groups" per flow), the card's name and power limit, and the answers that differ from the single
engine's.

usage: scripts/bench_shard_grouped.py [record.json] [steps]"""
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from wax_b200 import CUDAVectorEngine, VectorMetric, Where, sharded  # noqa: E402
from wax_b200 import _lib as L  # noqa: E402
from wax_b200.engine import _WhereArgs  # noqa: E402

N, DIMS, B = 10_000_000, 384, 1024
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
    out = fn()                                  # warm-up: the group index, mirrors and every shape the timed window uses
    t = time.perf_counter()
    for _ in range(n):
        fn()
    return (time.perf_counter() - t) / n, out


def bits(answer):
    return [(g, [(f, np.float32(s).view(np.uint32).item()) for f, s in hits]) for g, hits in answer]


class Ranks:
    """`world` engines on this device holding contiguous shards of the synthetic corpus."""

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

    def set_groups(self, groups):
        for (lo, hi), eng in zip(self.ranges, self.engines):
            eng.set_groups(np.arange(lo, hi, dtype=np.uint64), groups[lo:hi])

    def expanded(self):
        return sum(e.counter("shard_grouped_expanded_groups") for e in self.engines)

    def grouped(self, d_qs, top_groups, per_group, wheres, query_where):
        import torch
        b, g, p, world = int(d_qs.shape[0]), top_groups, per_group, self.world
        a = _WhereArgs(wheres, query_where, None, None, b)
        q = C.c_void_p(d_qs.data_ptr())
        hb = b * g * p * 32
        heads = torch.empty(world * hb, dtype=torch.uint8, device="cuda")
        for r, eng in enumerate(self.engines):
            rc = L.lib().wax_vs_shard_grouped_heads_device(eng.handle, q, b, g, p, *a.filter_args(), *a.where_args(near=True),
                                                           self.ranges[r][0], C.c_void_p(heads.data_ptr() + r * hb), None)
            assert rc == L.OK, L.last_error()
        chosen = torch.empty(b * g * 32, dtype=torch.uint8, device="cuda")
        assert L.lib().wax_vs_merge_group_heads_device(self.engines[0].handle, C.c_void_p(heads.data_ptr()), world, b, g, p,
                                                       C.c_void_p(chosen.data_ptr()), None) == L.OK, L.last_error()
        if p == 1:
            host = chosen.cpu().numpy()
            merged = None
        else:
            rb = b * g * p * 24
            rows = torch.empty(world * rb, dtype=torch.uint8, device="cuda")
            for r, eng in enumerate(self.engines):
                rc = L.lib().wax_vs_shard_grouped_expand_device(eng.handle, q, b, g, p, *a.filter_args(),
                                                                *a.where_args(near=True), C.c_void_p(chosen.data_ptr()),
                                                                C.c_void_p(heads.data_ptr() + r * hb), self.ranges[r][0],
                                                                C.c_void_p(rows.data_ptr() + r * rb), None)
                assert rc == L.OK, L.last_error()
            merged = torch.empty(rb, dtype=torch.uint8, device="cuda")
            assert L.lib().wax_vs_merge_candidates_device(self.engines[0].handle, C.c_void_p(rows.data_ptr()), world, b * g,
                                                          p, p, C.c_void_p(merged.data_ptr()), None) == L.OK
            host = torch.cat([chosen, merged]).cpu().numpy()
        groups = host[:b * g * 32].view(sharded.GROUP_CAND_DTYPE).reshape(b, g)
        if merged is None:
            best = groups.reshape(b, g, 1)
        else:
            best = host[b * g * 32:].view(sharded.CAND_DTYPE).reshape(b, g, p)
        scores = sharded.score_from_distance(0, best["distance"])
        return [[(int(groups["group_id"][i, j]), [(int(best["frame_id"][i, j, m]), float(scores[i, j, m]))
                                                   for m in range(best.shape[2]) if best["valid"][i, j, m]])
                 for j in range(g) if groups["valid"][i, j]] for i in range(b)]

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
    rows = np.arange(N, dtype=np.uint64)
    shapes = {"8 consecutive": rows // 8, "360 consecutive": rows // 360,
              "360 hashed": (rows * np.uint64(0x9E3779B97F4A7C15) >> np.uint64(32)) % np.uint64(N // 360)}
    single = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    single.fill_synthetic(2, N, normalize=True)
    single.set_attributes(rows, ts, tags)
    qs = rng.uniform(-1, 1, size=(B, DIMS)).astype(np.float32)
    qs /= np.linalg.norm(qs, axis=1, keepdims=True)
    d_qs = torch.from_numpy(qs).cuda()
    starts = rng.integers(0, N - N // 5, B)
    windows = [Where(after=int(ts[s]), before=int(ts[s + N // 5]), no_tags=DELETED) for s in starts]
    work = {                                    # name: (grouping, top_groups, per_group, wheres, query_where)
        "(a) groups of 8 consecutive rows, 12 x 1": ("8 consecutive", 12, 1, [], [None] * B),
        "(b) groups of 360 consecutive rows, 12 x 3": ("360 consecutive", 12, 3, [], [None] * B),
        "(c) hashed groups of 360 rows, 12 x 3": ("360 hashed", 12, 3, [], [None] * B),
        "(d) as (b), per-query 20 % window + deleted skip": ("360 consecutive", 12, 3, windows, list(range(B))),
    }
    single_ms, single_ans = {}, {}
    for name, (shape, g, p, wheres, qw) in work.items():
        single.set_groups(rows, shapes[shape])
        s, single_ans[name] = timed(lambda: single.search_batch_grouped_multi_where(qs, g, p, wheres, qw), steps)
        single_ms[name] = s * 1e3
        print(json.dumps({"workload": name, "single_engine_ms": single_ms[name]}), flush=True)
    single.close()
    lines = []
    for world in (1, 2, 4):
        ranks = Ranks(world, ts, tags)
        try:
            for name, (shape, g, p, wheres, qw) in work.items():
                ranks.set_groups(shapes[shape])
                ranks.grouped(d_qs, g, p, wheres, qw)               # warm-up outside the expansion count
                e0 = ranks.expanded()
                s, got = timed(lambda: ranks.grouped(d_qs, g, p, wheres, qw), steps)
                mism = sum(bits(got[i]) != bits(single_ans[name][i]) for i in range(B))
                lines.append({"workload": name, "world": world, "corpus": f"{N} x {DIMS} cosine, fill_synthetic",
                              "batch": B, "top_groups": g, "per_group": p, "steps": steps, "sharded_flow_ms": s * 1e3,
                              "single_engine_ms": single_ms[name], "ratio": s * 1e3 / single_ms[name],
                              "expanded_groups_per_flow": (ranks.expanded() - e0) / (steps + 1),
                              "mismatches": int(mism), **info})
                print(json.dumps(lines[-1]), flush=True)
        finally:
            ranks.close()
    if record:
        record.parent.mkdir(parents=True, exist_ok=True)
        record.write_text(json.dumps({"note": "ranks share one GPU: the protocol's overhead, not multi-GPU scaling",
                                      "workloads": lines}, indent=1) + "\n")


if __name__ == "__main__":
    main()
