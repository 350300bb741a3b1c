#!/usr/bin/env python
"""Frame-attribute predicates below the top-k (wax_vs_search_batch_where) on 10 M x 384 cosine rows (fill_synthetic),
timestamps increasing with the row plus seeded jitter, 1 % of the rows tagged deleted; batch 1 024, top-10.  Workloads:
  (a) 1 024 distinct random windows of 20 % of the rows;
  (b) no window, no_tags excluding the rows tagged deleted;
  (c) 1 024 windows of about 5 000 rows (the gather class);
  (d) (a) ANDed with one 1 M-frame id allow-list;
  (e) a single search_where with a 20 % window.
Each reports the wall time of the public C call, against the same filter expressed as id lists (multi_filtered /
search_filtered; where that form would resolve more than about 100 M ids a sample of queries is timed and extrapolated,
and the line says so) and the unfiltered search_batch / search of the same queries.  A separate run under torch.profiler
reports the device time of the where kernels.  Prints one JSON line per workload with the card's name and power limit,
and writes them all to the record file given as the first argument.

usage: scripts/bench_where.py [record.json] [steps]"""
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from wax_b200 import CUDAVectorEngine, VectorMetric, Where  # noqa: E402
from wax_b200 import _lib as L  # noqa: E402

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


class WhereCall:
    """Prebuilt arguments of one wax_vs_search_batch_where call (the timing covers the C call only)."""

    def __init__(self, eng, qs, wheres, query_where, filters=(), query_filter=None):
        P = C.POINTER
        self.eng, self.qs = eng, np.ascontiguousarray(qs, np.float32)
        b = len(self.qs)
        self.fids = np.concatenate([f for _, f in filters]).astype(np.uint64) if filters else np.zeros(1, np.uint64)
        self.off = np.zeros(len(filters) + 1, np.uint64)
        self.off[1:] = np.cumsum([f.size for _, f in filters])
        self.modes = np.asarray([0 if m == "allow" else 1 for m, _ in filters] or [0], np.int32)
        self.nf = len(filters)
        qf = query_filter if query_filter is not None else [None] * b
        self.qf = np.asarray([L.NO_FILTER if f is None else f for f in qf], np.uint32)
        self.qw = np.asarray([L.NO_FILTER if w is None else w for w in query_where], np.uint32)
        self.w = (L.Where * len(wheres))(*[w.to_c() for w in wheres])
        self.nw = len(wheres)
        self.ids = np.zeros((b, K), np.uint64)
        self.scores = np.zeros((b, K), np.float32)
        self.ns = np.zeros(b, np.uint32)
        self.args = (self.qs.ctypes.data_as(P(C.c_float)), b, DIMS, K, self.fids.ctypes.data_as(P(C.c_uint64)),
                     self.off.ctypes.data_as(P(C.c_uint64)), self.modes.ctypes.data_as(P(C.c_int32)), self.nf,
                     self.qf.ctypes.data_as(P(C.c_uint32)), C.cast(self.w, C.c_void_p), self.nw,
                     self.qw.ctypes.data_as(P(C.c_uint32)), self.ids.ctypes.data_as(P(C.c_uint64)),
                     self.scores.ctypes.data_as(P(C.c_float)), K, self.ns.ctypes.data_as(P(C.c_uint32)))

    def __call__(self):
        rc = L.lib().wax_vs_search_batch_where(self.eng._h, *self.args)
        assert rc == L.OK, L.last_error()

    def hits(self, qi):
        return [(int(self.ids[qi, j]), float(self.scores[qi, j])) for j in range(int(self.ns[qi]))]


def timed(fn, n):
    fn()                                        # warm-up: every shape the timed window uses
    t = time.perf_counter()
    for _ in range(n):
        fn()
    return (time.perf_counter() - t) / n


def bits(hits):
    return [(i, np.float32(s).view(np.uint32).item()) for i, s in hits]


def main():
    info = card()
    eng = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    eng.fill_synthetic(2, N, normalize=True)
    rng = np.random.default_rng(11)
    frames = np.arange(N, dtype=np.uint64)
    ts = np.arange(N, dtype=np.int64) * 16 + rng.integers(0, 16, N)
    tags = np.zeros(N, np.uint64)
    deleted = rng.choice(N, N // 100, replace=False)
    tags[deleted] = DELETED
    t = time.perf_counter()
    eng.set_attributes(frames, ts, tags)
    set_ms = (time.perf_counter() - t) * 1e3
    qs = rng.uniform(-1, 1, size=(B, DIMS)).astype(np.float32)
    qs /= np.linalg.norm(qs, axis=1, keepdims=True)

    def windows(rows, count):
        starts = rng.integers(0, N - rows, count)
        return [Where(after=int(ts[s]), before=int(ts[s + rows])) for s in starts], starts

    wide, wide_starts = windows(N // 5, B)
    narrow, narrow_starts = windows(5000, B)
    allow_1m = np.sort(rng.choice(N, 1_000_000, replace=False)).astype(np.uint64)
    unfiltered_s = timed(lambda: eng.search_batch_arrays(qs, K), steps)

    def window_rows(w):                        # timestamps increase with the row: a window is a row range
        return np.arange(np.searchsorted(ts, w.after), np.searchsorted(ts, w.before), dtype=np.uint64)

    def id_form(filters_of, sample):
        """The same answers through multi_filtered with the passing frames as allow-lists: `sample` queries."""
        lists = [("allow", filters_of(qi)) for qi in sample]
        call = lambda: eng.search_batch_multi_filtered(qs[sample], K, lists, list(range(len(sample))))
        return timed(call, 1), call()

    lines = []
    uploads0 = eng.counter("attribute_uploads")
    work = {
        "(a) 1024 windows of 20 %": (WhereCall(eng, qs, wide, list(range(B))), lambda qi: window_rows(wide[qi]), 16),
        "(b) no window, no_tags = deleted (1 %)": (WhereCall(eng, qs, [Where(no_tags=DELETED)], [0] * B), None, B),
        "(c) 1024 windows of 5 000 rows (gather)": (WhereCall(eng, qs, narrow, list(range(B))),
                                                    lambda qi: window_rows(narrow[qi]), B),
        "(d) (a) AND a 1 M-frame allow-list": (WhereCall(eng, qs, wide, list(range(B)), [("allow", allow_1m)], [0] * B),
                                               lambda qi: np.intersect1d(window_rows(wide[qi]), allow_1m), 64),
    }
    for name, (call, rows_of, sample_n) in work.items():
        passes0 = eng.counter("filter_bitset_passes")
        wall = timed(call, steps)
        passes = (eng.counter("filter_bitset_passes") - passes0) / (steps + 1)
        if rows_of is None:                    # (b) as an id list: one deny-list of the deleted frames for every query
            id_call = lambda: eng.search_batch_filtered(qs, K, deny=frames[deleted])
            id_s, want_all = timed(id_call, 1), id_call()
            sample = list(range(B))
            ids_resolved = deleted.size
        else:
            sample = list(range(0, B, B // sample_n))[:sample_n]
            id_s, want_all = id_form(rows_of, sample)
            ids_resolved = sum(rows_of(qi).size for qi in sample) * (B // len(sample))
        extrapolated = len(sample) < B
        mismatches = sum(bits(call.hits(qi)) != bits(want_all[j]) for j, qi in enumerate(sample))
        line = {"workload": name, "corpus": f"{N} x {DIMS} cosine, fill_synthetic", "batch": B, "top_k": K,
                "steps": steps, "wall_ms": wall * 1e3, "queries_per_s": B / wall,
                "unfiltered_search_batch_ms": unfiltered_s * 1e3, "vs_unfiltered": wall / unfiltered_s,
                "id_list_form_ms": id_s * 1e3 * (B / len(sample)), "id_list_form_extrapolated_from_queries":
                    len(sample) if extrapolated else None, "id_list_ids_resolved": int(ids_resolved),
                "filter_bitset_passes_per_call": passes, "checked": len(sample), "mismatches": int(mismatches), **info}
        lines.append(line)
        print(json.dumps(line), flush=True)
    # (e) one query, a 20 % window
    w = wide[0]
    q = qs[0]
    single = timed(lambda: eng.search_where(q, K, w), 20)
    allow = window_rows(w)
    single_ids = timed(lambda: eng.search_filtered(q, K, allow=allow), 3)
    plain = timed(lambda: eng.search(q, K), 20)
    same = bits(eng.search_where(q, K, w)) == bits(eng.search_filtered(q, K, allow=allow))
    line = {"workload": "(e) single search_where, 20 % window", "corpus": f"{N} x {DIMS} cosine", "top_k": K,
            "wall_ms": single * 1e3, "search_filtered_2M_allow_list_ms": single_ids * 1e3, "unfiltered_search_ms": plain * 1e3,
            "single_shadow_queries": eng.counter("single_shadow_queries"), "mismatches": 0 if same else 1, **info}
    lines.append(line)
    print(json.dumps(line), flush=True)
    setup = {"set_attributes_10M_ms": set_ms, "attribute_uploads": eng.counter("attribute_uploads") - uploads0, **info}
    # device time of the where kernels: one call of (a), (b), (c) under torch.profiler, in a run of its own
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.init()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for call, _, _ in list(work.values())[:3]:
                call()
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            if "where_" in ev.key or "filter_bits" in ev.key or "gather_" in ev.key:
                kern[ev.key.split("(")[0]] = {"calls": ev.count, "device_ms_total": ev.device_time_total / 1e3}
        setup["kernels_a_b_c_one_call_each"] = kern
    except Exception as ex:  # noqa: BLE001
        setup["kernels_error"] = repr(ex)
    print(json.dumps(setup), flush=True)
    if record:
        record.parent.mkdir(parents=True, exist_ok=True)
        record.write_text(json.dumps({"workloads": lines, "setup": setup}, indent=1) + "\n")
    eng.close()


if __name__ == "__main__":
    main()
