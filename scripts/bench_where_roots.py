#!/usr/bin/env python
"""PhotoRAG's and VideoRAG's root test below the top-k (wax_vs_search_batch_where_roots,
_grouped_multi_where_roots) on 10 M x 384 cosine rows (fill_synthetic).  Rows form groups of 360 consecutive frames,
each group's id being its first frame's (the root); each group's root-tag word is IS_ROOT, except 2 % of the groups
also SUPERSEDED, 1 % also DELETED and 0.5 % without IS_ROOT (a root without meta); timestamps are seeded uniform in
[0, 1000).  The root clause is PhotoRAG's: all IS_ROOT, none of DELETED | SUPERSEDED.  Batch 1 024.
Workloads:
  (a) plain top-10 under the root clause, against the same filter as a host-built deny-list of the failing groups' frames
      (its build time reported apart) and against the unfiltered batch;
  (b) grouped 12 x 3, each query its own 20 % window AND the root clause, against PhotoRAG's form: grouped search over
      the window alone fetching twice the groups, the failing roots dropped on the host -- with the number of queries
      that come back with fewer than 12 groups that way;
  (c) one grouped query, the same two forms.
Each reports the wall time of the public call, alternating in the same run with the other forms.  Every answer of the
root clause must equal the deny-list form's, and PhotoRAG's form's wherever that one is not short.  Prints one JSON
line per workload with the card's name and power limit, and writes them all to the record file given as the first
argument.

usage: scripts/bench_where_roots.py [record.json] [steps]"""
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
GROUP = 360
IS_ROOT, DELETED, SUPERSEDED = 1, 2, 4
PHOTO = dict(root_all_tags=IS_ROOT, root_no_tags=DELETED | SUPERSEDED)
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
    rng = np.random.default_rng(31)
    frames = np.arange(N, dtype=np.uint64)
    ts = rng.integers(0, 1000, N).astype(np.int64)
    eng.set_attributes(frames, ts, None)
    eng.set_groups(frames, frames // GROUP * GROUP)
    roots = np.arange(0, N, GROUP, dtype=np.uint64)
    u = rng.random(roots.size)
    words = np.where(u < 0.02, IS_ROOT | SUPERSEDED, np.where(u < 0.03, IS_ROOT | DELETED,
                                                              np.where(u < 0.035, 0, IS_ROOT))).astype(np.uint64)
    eng.set_root_tags(roots, words)
    live = {int(g) for g, w in zip(roots, words) if w == IS_ROOT}
    qs = rng.uniform(-1, 1, size=(B, DIMS)).astype(np.float32)
    qs /= np.linalg.norm(qs, axis=1, keepdims=True)
    lines = []

    # (a) plain top-10 under the root clause
    def deny_list():
        """The frames of every group whose root fails, as a caller would list them from its frame metadata."""
        t = time.perf_counter()
        failing = roots[words != IS_ROOT]
        ids = (failing[:, None] + np.arange(GROUP, dtype=np.uint64)[None, :]).reshape(-1)
        return ids[ids < N], time.perf_counter() - t
    deny, build = deny_list()
    root_call = lambda: eng.search_batch_where(qs, K, [Where(**PHOTO)], [0] * B)                        # noqa: E731
    deny_call = lambda: eng.search_batch_multi_filtered(qs, K, [("deny", deny)], [0] * B)              # noqa: E731
    unfiltered = lambda: eng.search_batch_arrays(qs, K)                                                 # noqa: E731
    root_s, deny_s, plain_s = alternate([root_call, deny_call, unfiltered], steps)
    got, want = root_call(), deny_call()
    line = {"workload": "(a) 1024 x top-10 under the root clause", "corpus": f"{N} x {DIMS} cosine, fill_synthetic, "
            f"groups of {GROUP}", "batch": B, "top_k": K, "steps": steps, "where_roots_ms": root_s * 1e3,
            "host_deny_list_form_ms": deny_s * 1e3, "host_deny_list_build_ms": build * 1e3,
            "unfiltered_ms": plain_s * 1e3, "deny_list_ids": int(deny.size), "checked": B,
            "mismatches": int(sum(g != w for g, w in zip(got, want))), **info}
    lines.append(line)
    print(json.dumps(line), flush=True)

    # (b) grouped 12 x 3, own 20 % window AND the root clause, against PhotoRAG's over-fetch and drop
    def photo_form(q, ws):
        """Grouped search over the window alone for twice the groups, the failing roots dropped on the host."""
        over = eng.search_batch_grouped_multi_where(q, 24, 3, ws, list(range(len(ws))))
        return [[grp for grp in ans if grp[0] in live][:12] for ans in over]
    starts = rng.integers(0, 800, B)
    win = [Where(after=int(a), before=int(a) + 200) for a in starts]
    rooted = [Where(after=int(a), before=int(a) + 200, **PHOTO) for a in starts]
    root_call = lambda: eng.search_batch_grouped_multi_where(qs, 12, 3, rooted, list(range(B)))        # noqa: E731
    photo_call = lambda: photo_form(qs, win)                                                            # noqa: E731
    unfiltered = lambda: eng.search_batch_grouped(qs, 12, per_group=3)                                  # noqa: E731
    root_s, photo_s, plain_s = alternate([root_call, photo_call, unfiltered], steps)
    got, want = root_call(), photo_call()
    short = [i for i in range(B) if len(want[i]) < 12]
    line = {"workload": "(b) grouped 12 x 3, 1024 x (own 20 % window AND the root clause)", "batch": B,
            "top_k": "12 groups x 3", "steps": steps, "where_roots_ms": root_s * 1e3,
            "photorag_overfetch_2x_ms": photo_s * 1e3, "unfiltered_ms": plain_s * 1e3,
            "photorag_short_queries": len(short), "where_roots_short_queries": sum(len(g) < 12 for g in got),
            "checked": B - len(short),
            "mismatches": int(sum(got[i] != want[i] for i in range(B) if i not in set(short))), **info}
    lines.append(line)
    print(json.dumps(line), flush=True)

    # (c) one grouped query
    q = qs[:1]
    root_call = lambda: eng.search_batch_grouped_multi_where(q, 12, 3, rooted[:1], [0])                # noqa: E731
    photo_call = lambda: photo_form(q, win[:1])                                                         # noqa: E731
    plain_call = lambda: eng.search_grouped(q[0], 12, per_group=3)                                      # noqa: E731
    root_s, photo_s, plain_s = alternate([root_call, photo_call, plain_call], max(steps, 20))
    got, want = root_call(), photo_call()
    line = {"workload": "(c) one grouped query, 12 x 3, 20 % window AND the root clause", "top_k": "12 groups x 3",
            "where_roots_ms": root_s * 1e3, "photorag_overfetch_2x_ms": photo_s * 1e3, "unfiltered_ms": plain_s * 1e3,
            "photorag_short": len(want[0]) < 12, "mismatches": 0 if len(want[0]) < 12 or got == want else 1, **info}
    lines.append(line)
    print(json.dumps(line), flush=True)

    setup = {"root_column_builds": eng.counter("root_column_builds"),
             "group_index_builds": eng.counter("group_index_builds"), **info}
    try:                                       # device time of the rooted where kernels: one call of (a), own run
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.init()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.search_batch_where(qs, K, [Where(**PHOTO)], [0] * B)
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            if "where_" in ev.key or "filter_bits" in ev.key or "root_column" in ev.key:
                kern[ev.key.split("(")[0]] = {"calls": ev.count, "device_ms_total": ev.device_time_total / 1e3}
        setup["kernels_a_one_call"] = kern
    except Exception as ex:  # noqa: BLE001
        setup["kernels_error"] = repr(ex)
    print(json.dumps(setup), flush=True)
    if record:
        record.parent.mkdir(parents=True, exist_ok=True)
        record.write_text(json.dumps({"workloads": lines, "setup": setup}, indent=1) + "\n")
    eng.close()
    bad = sum(line_["mismatches"] for line_ in lines)
    if bad:
        sys.exit(f"{bad} answers differ between the forms")


if __name__ == "__main__":
    main()
