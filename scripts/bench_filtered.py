#!/usr/bin/env python
"""Batched search with one filter per query (wax_vs_search_batch_multi_filtered) on 10 M x 384 cosine rows
(fill_synthetic, implicit frame ids), batch 1 024, top-10.  Workloads:
  (a) 1 024 distinct deny-lists of 10 000 rows, one per query;
  (b) 16 allow-lists of 2 M rows, assigned round-robin;
  (c) 1 024 allow-lists of 5 000 rows, one per query (the gather class);
  (d) 256 queries of each of (a) to (c) plus 256 unfiltered queries.
Each workload reports the wall time of the public C call (host queries in, host ids / scores out; it ends in a
stream synchronise) and queries per second.  Baselines in the same run: the unfiltered wax_vs_search_batch of the same
queries, one wax_vs_search_batch_filtered call per distinct filter, and 32 single wax_vs_search_filtered calls
(extrapolated to the batch).  A sample of answers is checked against wax_vs_search_filtered.  Prints one JSON line
per workload, with the card's name and power limit.

usage: scripts/bench_filtered.py [steps]"""
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from wax_b200 import CUDAVectorEngine, VectorMetric  # noqa: E402
from wax_b200 import _lib as L  # noqa: E402

N, DIMS, B, K = 10_000_000, 384, 1024, 10
steps = int(sys.argv[1]) if len(sys.argv) > 1 else 5


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as ex:  # noqa: BLE001
        return {"gpu": "unknown", "power_limit": "unknown", "error": repr(ex)}


class Call:
    """Prebuilt arguments of one wax_vs_search_batch_multi_filtered call (the timing covers the C call only)."""

    def __init__(self, eng, qs, filters, query_filter):
        self.eng, self.qs = eng, np.ascontiguousarray(qs, np.float32)
        self.filters = filters
        self.fids = np.concatenate([f for _, f in filters]).astype(np.uint64) if filters else np.zeros(0, np.uint64)
        self.off = np.zeros(len(filters) + 1, np.uint64)
        self.off[1:] = np.cumsum([f.size for _, f in filters])
        self.modes = np.asarray([0 if m == "allow" else 1 for m, _ in filters], np.int32)
        self.qf = np.asarray([L.NO_FILTER if f is None else f for f in query_filter], np.uint32)
        self.query_filter = query_filter
        self.ids = np.zeros((len(qs), K), np.uint64)
        self.scores = np.zeros((len(qs), K), np.float32)
        self.ns = np.zeros(len(qs), np.uint32)

    def __call__(self):
        P = C.POINTER
        rc = L.lib().wax_vs_search_batch_multi_filtered(
            self.eng._h, self.qs.ctypes.data_as(P(C.c_float)), len(self.qs), DIMS, K,
            self.fids.ctypes.data_as(P(C.c_uint64)), self.off.ctypes.data_as(P(C.c_uint64)),
            self.modes.ctypes.data_as(P(C.c_int32)), len(self.modes), self.qf.ctypes.data_as(P(C.c_uint32)),
            self.ids.ctypes.data_as(P(C.c_uint64)), self.scores.ctypes.data_as(P(C.c_float)), K,
            self.ns.ctypes.data_as(P(C.c_uint32)))
        assert rc == L.OK, L.last_error()

    def hits(self, qi):
        return [(int(self.ids[qi, j]), float(self.scores[qi, j])) for j in range(int(self.ns[qi]))]


def timed(fn, n):
    fn()                                        # warm-up: every shape the timed window uses
    t = time.perf_counter()
    for _ in range(n):
        fn()
    return (time.perf_counter() - t) / n


def main():
    info = card()
    eng = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    eng.fill_synthetic(2, N, normalize=True)
    rng = np.random.default_rng(7)
    qs = rng.uniform(-1, 1, size=(B, DIMS)).astype(np.float32)
    qs /= np.linalg.norm(qs, axis=1, keepdims=True)
    perm = rng.permutation(N).astype(np.uint64)
    deny = [("deny", rng.integers(0, N, 10_000).astype(np.uint64)) for _ in range(B)]
    big = [("allow", np.take(perm, np.arange(i * 625_000, i * 625_000 + 2_000_000) % N)) for i in range(16)]
    small = [("allow", rng.integers(0, N, 5_000).astype(np.uint64)) for _ in range(B)]
    q4 = B // 4
    workloads = {
        "(a) 1024 deny-lists of 10 000 rows": (deny, list(range(B))),
        "(b) 16 allow-lists of 2 M rows, round-robin": (big, [i % 16 for i in range(B)]),
        "(c) 1024 allow-lists of 5 000 rows (gather)": (small, list(range(B))),
        "(d) 256 each of (a), (b), (c) and unfiltered": (
            deny[:q4] + big + small[:q4],
            list(range(q4)) + [q4 + i % 16 for i in range(q4)] + [q4 + 16 + i for i in range(q4)] + [None] * q4),
    }

    eng.search_batch_arrays(qs, K)
    unfiltered_s = timed(lambda: eng.search_batch_arrays(qs, K), steps)
    for name, (filters, query_filter) in workloads.items():
        call = Call(eng, qs, filters, query_filter)
        t0, f0 = eng.batch_stats()
        p0 = eng.counter("filter_bitset_passes")
        wall = timed(call, steps)
        t1, f1 = eng.batch_stats()
        p1 = eng.counter("filter_bitset_passes")
        # baseline 1: one wax_vs_search_batch_filtered call per distinct filter (its queries grouped), one round
        groups = {}
        for qi, f in enumerate(query_filter):
            groups.setdefault(f, []).append(qi)

        def per_filter():
            for f, members in groups.items():
                if f is None:
                    eng.search_batch_arrays(qs[members], K)
                else:
                    mode, fids = filters[f]
                    eng.search_batch_filtered(qs[members], K, **{mode: fids})
        per_filter_s = timed(per_filter, 1)
        # baseline 2: 32 single filtered searches, extrapolated to the batch
        sample = list(range(0, B, B // 32))[:32]

        def singles():
            for qi in sample:
                f = query_filter[qi]
                if f is None:
                    eng.search(qs[qi], K)
                else:
                    mode, fids = filters[f]
                    eng.search_filtered(qs[qi], K, **{mode: fids})
        single_s = timed(singles, 1) / len(sample)
        # correctness sample: ids and score bits against the single-query filtered search
        call()
        mismatches = 0
        for qi in sample[:8] + [B - 1]:
            f = query_filter[qi]
            want = eng.search(qs[qi], K) if f is None else eng.search_filtered(qs[qi], K, **{filters[f][0]: filters[f][1]})
            got = call.hits(qi)
            same = [i for i, _ in got] == [i for i, _ in want] and \
                np.array_equal(np.float32([s for _, s in got]).view(np.uint32), np.float32([s for _, s in want]).view(np.uint32))
            mismatches += 0 if same else 1
        line = {
            "workload": name, "corpus": f"{N} x {DIMS} cosine, fill_synthetic", "batch": B, "top_k": K, "steps": steps,
            "wall_ms": wall * 1e3, "queries_per_s": B / wall,
            "unfiltered_search_batch_ms": unfiltered_s * 1e3, "vs_unfiltered": wall / unfiltered_s,
            "per_filter_search_batch_filtered_ms": per_filter_s * 1e3, "distinct_filters": len(groups),
            "single_search_filtered_ms_each": single_s * 1e3, "single_loop_ms_extrapolated": single_s * B * 1e3,
            "tensor_queries_per_call": (t1 - t0) / (steps + 1), "fallback_queries_per_call": (f1 - f0) / (steps + 1),
            "filter_bitset_passes_per_call": (p1 - p0) / (steps + 1),
            "checked": len(sample[:8]) + 1, "mismatches": mismatches, **info,
        }
        print(json.dumps(line), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
