#!/usr/bin/env python
"""VideoRAG's video filter below the top-k (wax_vs_search_batch_where_groups, _grouped_multi_where_groups) on 10 M x 384
cosine rows (fill_synthetic).  Rows form groups of 360 consecutive frames (a video's segments), each group's id being
its first frame's (the root); 1 % are tagged deleted; timestamps are seeded uniform in [0, 1000).  Batch 1 024, top-10.
Workloads:
  (a) plain: each query its own 8 groups AND a 20 % time window AND not deleted;
  (b) grouped 12 x 3: each query its own 16 groups AND a 20 % time window (VideoRAG's request);
  (c) plain: each query one of 32 sets of 2 000 groups (720 K rows: the bitset class);
  (d) one query, 100 groups.
Each reports the wall time of the public C call, alternating in the same run with two baselines: the same filter as
host-built id allow-lists passed with the same where (no groups) to the same entry's allow-list form (its host build
time is reported apart), and the unfiltered batch.  Every answer of the two filtered forms must be identical.  Prints
one JSON line per workload with the card's name and power limit, and writes them all to the record file given as the
first argument.

usage: scripts/bench_where_groups.py [record.json] [steps]"""
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from wax_b200 import CUDAVectorEngine, VectorMetric, Where  # noqa: E402

N, DIMS, B, K = 10_000_000, 384, 1024, 10
GROUP, DELETED = 360, 1
N_GROUPS = (N + GROUP - 1) // GROUP
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


def alternate(fns, n):
    """Mean wall time of each callable, run in turn n times after one warm-up round."""
    for f in fns:
        f()
    total = [0.0] * len(fns)
    for _ in range(n):
        for i, f in enumerate(fns):
            t = time.perf_counter()
            f()
            total[i] += time.perf_counter() - t
    return [t / n for t in total]


def main():
    info = card()
    eng = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    eng.fill_synthetic(2, N, normalize=True)
    rng = np.random.default_rng(29)
    frames = np.arange(N, dtype=np.uint64)
    ts = rng.integers(0, 1000, N).astype(np.int64)
    tags = np.where(rng.random(N) < 0.01, DELETED, 0).astype(np.uint64)
    eng.set_attributes(frames, ts, tags)
    eng.set_groups(frames, frames // GROUP * GROUP)
    qs = rng.uniform(-1, 1, size=(B, DIMS)).astype(np.float32)
    qs /= np.linalg.norm(qs, axis=1, keepdims=True)

    def window(w):
        a = int(rng.integers(0, 800))
        return dict(after=a, before=a + 200, **w)

    def host_lists(ws):
        """The frames of each where's groups, as the caller builds them today (VideoRAGOrchestrator.swift:239-247)."""
        t = time.perf_counter()
        lists = [("allow", np.concatenate([np.arange(g, min(g + GROUP, N), dtype=np.uint64) for g in w.groups]))
                 for w in ws]
        return lists, time.perf_counter() - t

    def plain(ws):
        return [Where(after=w.after, before=w.before, no_tags=w.no_tags) for w in ws]

    sets = [tuple(int(g) * GROUP for g in rng.choice(N_GROUPS, 2000, replace=False)) for _ in range(32)]
    workloads = [
        ("(a) 1024 x (own 8 groups AND 20 % window AND not deleted)", False,
         [Where(**window(dict(no_tags=DELETED, groups=tuple(int(g) * GROUP for g in rng.choice(N_GROUPS, 8, replace=False)))))
          for _ in range(B)]),
        ("(b) grouped 12 x 3, 1024 x (own 16 groups AND 20 % window)", True,
         [Where(**window(dict(groups=tuple(int(g) * GROUP for g in rng.choice(N_GROUPS, 16, replace=False)))))
          for _ in range(B)]),
        ("(c) 1024 x (one of 32 sets of 2000 groups)", False, [Where(groups=sets[i % 32]) for i in range(B)]),
    ]
    lines = []
    units0, walked0 = eng.counter("where_group_units"), eng.counter("where_group_rows_walked")
    for name, grouped, ws in workloads:
        qw = list(range(B))
        if name.startswith("(c)"):             # 32 distinct lists: queries name theirs
            lists, build = host_lists(ws[:32])
            pw, qf = plain(ws[:32]), [i % 32 for i in range(B)]
            pqw = qf
        else:
            lists, build = host_lists(ws)
            pw, qf, pqw = plain(ws), qw, qw
        if grouped:
            group_call = lambda: eng.search_batch_grouped_multi_where(qs, 12, 3, ws, qw)                 # noqa: E731
            id_call = lambda: eng.search_batch_grouped_multi_where(qs, 12, 3, pw, pqw, lists, qf)        # noqa: E731
            unfiltered = lambda: eng.search_batch_grouped(qs, 12, per_group=3)                          # noqa: E731
        else:
            group_call = lambda: eng.search_batch_where(qs, K, ws, qw)                                   # noqa: E731
            id_call = lambda: eng.search_batch_where(qs, K, pw, pqw, lists, qf)                          # noqa: E731
            unfiltered = lambda: eng.search_batch_arrays(qs, K)                                         # noqa: E731
        group_s, id_s, plain_s = alternate([group_call, id_call, unfiltered], steps)
        got, want = group_call(), id_call()
        mismatches = sum(g != w for g, w in zip(got, want))
        line = {"workload": name, "corpus": f"{N} x {DIMS} cosine, fill_synthetic, groups of {GROUP}", "batch": B,
                "top_k": "12 groups x 3" if grouped else K, "steps": steps, "where_groups_ms": group_s * 1e3,
                "host_allow_list_form_ms": id_s * 1e3, "host_allow_list_build_ms": build * 1e3,
                "unfiltered_ms": plain_s * 1e3, "allow_list_ids": int(sum(x.size for _, x in lists)), "checked": B,
                "mismatches": int(mismatches), **info}
        lines.append(line)
        print(json.dumps(line), flush=True)
    # (d) one query, 100 groups
    w = Where(groups=tuple(int(g) * GROUP for g in rng.choice(N_GROUPS, 100, replace=False)))
    lists, build = host_lists([w])
    q = qs[0]
    group_call = lambda: eng.search_where(q, K, w)                                                      # noqa: E731
    id_call = lambda: eng.search_filtered(q, K, allow=lists[0][1])                                      # noqa: E731
    plain_call = lambda: eng.search(q, K)                                                               # noqa: E731
    group_s, id_s, plain_s = alternate([group_call, id_call, plain_call], max(steps, 20))
    line = {"workload": "(d) one query, 100 groups", "corpus": f"{N} x {DIMS}", "top_k": K,
            "where_groups_ms": group_s * 1e3, "host_allow_list_form_ms": id_s * 1e3,
            "host_allow_list_build_ms": build * 1e3, "unfiltered_ms": plain_s * 1e3,
            "mismatches": 0 if group_call() == id_call() else 1, **info}
    lines.append(line)
    print(json.dumps(line), flush=True)
    setup = {"where_group_units": eng.counter("where_group_units") - units0,
             "where_group_rows_walked": eng.counter("where_group_rows_walked") - walked0,
             "group_index_builds": eng.counter("group_index_builds"), **info}
    try:                                       # device time of the group kernels: one call of (a) and (c), own run
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.init()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.search_batch_where(qs, K, workloads[0][2], list(range(B)))
            eng.search_batch_where(qs, K, workloads[2][2], list(range(B)))
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            if "where_group" in ev.key or "filter_bits" in ev.key or "gather_" in ev.key:
                kern[ev.key.split("(")[0]] = {"calls": ev.count, "device_ms_total": ev.device_time_total / 1e3}
        setup["kernels_a_c_one_call_each"] = kern
    except Exception as ex:  # noqa: BLE001
        setup["kernels_error"] = repr(ex)
    print(json.dumps(setup), flush=True)
    if record:
        record.parent.mkdir(parents=True, exist_ok=True)
        record.write_text(json.dumps({"workloads": lines, "setup": setup}, indent=1) + "\n")
    eng.close()


if __name__ == "__main__":
    main()
