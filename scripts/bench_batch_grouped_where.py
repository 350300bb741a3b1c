#!/usr/bin/env python
"""Batched grouped search with a where and an id filter of each query's own (wax_vs_search_batch_grouped_multi_where)
on 10 M x 384 cosine rows (fill_synthetic) in groups of 360 consecutive rows.  Attributes and locations as
bench_where_near.py: 70 % of the rows carry a location, clustered around 300 seeded centres, 1 % are tagged deleted,
timestamps increase with the row.  Batch 1 024.  Workloads:
  (a) each query its own 20 % time window AND not deleted; 12 groups x 1 frame;
  (b) each query its own 25 km box AND 20 % window AND not deleted; 12 x 1 (PhotoRAG);
  (c) each query its own allow-list of 5 000 frames (the gather class); 12 x 3 (VideoRAG);
  (d) 16 distinct wheres of (b)'s form spread over the 1 024 queries; 12 x 1.
Each reports the wall time of the public C call, alternating in the same run with the unfiltered search_batch_grouped
and, for (d), with one search_batch_grouped_where call per distinct where.  The other baseline, one search_grouped call
per query under the allow-list of the frames passing its where and filter (built on the host, as PhotoRAG builds its
location allow-list), is timed over 32 queries and extrapolated to the batch; those 32 answers must equal the batch's,
bit for bit.  Prints one JSON line per workload with the card's name and power limit, and writes them all to the
record file given as the first argument.

usage: scripts/bench_batch_grouped_where.py [record.json] [steps]"""
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from wax_b200 import CUDAVectorEngine, VectorMetric, Where, location_box  # noqa: E402

N, DIMS, B, GROUP, SAMPLE = 10_000_000, 384, 1024, 360, 32
DELETED = 1
COUNTERS = ("grouped_batch_covered_queries", "grouped_batch_expanded_groups", "grouped_batch_fallback_queries",
            "grouped_batch_expansion_passes", "filter_bitset_passes")
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


def flat(res):
    return [(g, f, int(np.float32(s).view(np.uint32))) for g, hits in res for f, s in hits]


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
    rng = np.random.default_rng(17)
    frames = np.arange(N, dtype=np.uint64)
    eng.set_groups(frames, frames // GROUP)
    ts = np.arange(N, dtype=np.int64)
    tags = np.where(rng.random(N) < 0.01, DELETED, 0).astype(np.uint64)
    eng.set_attributes(frames, ts, tags)
    n_c = 300
    lat_c, lon_c = rng.uniform(-60, 60, n_c), rng.uniform(-170, 170, n_c)
    c = rng.integers(0, n_c, N)
    lat = lat_c[c] + 0.18 * rng.standard_normal(N)                 # about 20 km
    lon = lon_c[c] + 0.18 * rng.standard_normal(N) / np.cos(np.radians(lat_c[c]))
    none = rng.random(N) >= 0.7
    lat[none] = np.nan
    lon[none] = np.nan
    eng.set_locations(frames, lat, lon)
    lat_bin, lon_bin = np.floor(lat * 100.0), np.floor(lon * 100.0)
    qs = rng.uniform(-1, 1, size=(B, DIMS)).astype(np.float32)
    qs /= np.linalg.norm(qs, axis=1, keepdims=True)

    def window():
        a = int(rng.integers(0, N - N // 5))
        return a, a + N // 5

    def passing(w, flt):
        """The frames query (w, flt) may return, on the host: PhotoRAG's allow-list (box bins) ANDed with the window,
        the tag clause and the id filter."""
        ok = np.ones(N, bool)
        if w is not None:
            ok &= (ts >= w.after) & (ts < w.before) & ((tags & np.uint64(w.no_tags)) == 0)
            if w.near is not None:
                la, lb, lo, hi = location_box(*w.near)
                ok &= (lat_bin >= la) & (lat_bin <= lb) & (lon_bin >= lo) & (lon_bin <= hi)
        if flt is not None:
            ok &= np.isin(frames, flt[1], assume_unique=True)
        return frames[ok]

    def boxed():
        a, b = window()
        ci = int(rng.integers(0, n_c))
        return Where(after=a, before=b, no_tags=DELETED, near=(float(lat_c[ci]), float(lon_c[ci]), 25_000.0))

    workloads = []
    ws = [Where(after=a, before=b, no_tags=DELETED) for a, b in (window() for _ in range(B))]
    workloads.append(("(a) 1024 x (own 20 % window AND not deleted), 12 x 1", 12, 1, ws, list(range(B)), [], [None] * B))
    ws = [boxed() for _ in range(B)]
    workloads.append(("(b) 1024 x (own 25 km box AND 20 % window AND not deleted), 12 x 1", 12, 1, ws, list(range(B)),
                      [], [None] * B))
    fl = [("allow", np.sort(rng.choice(N, 5000, replace=False)).astype(np.uint64)) for _ in range(B)]
    workloads.append(("(c) 1024 x (own allow-list of 5 000 frames), 12 x 3", 12, 3, [], [None] * B, fl, list(range(B))))
    ws = [boxed() for _ in range(16)]
    workloads.append(("(d) 16 distinct (25 km box AND 20 % window AND not deleted) over 1024 queries, 12 x 1", 12, 1, ws,
                      [i % 16 for i in range(B)], [], [None] * B))

    lines = []
    for name, top, per, ws, qw, fl, qf in workloads:
        call = lambda: eng.search_batch_grouped_multi_where(qs, top, per, ws, qw, fl, qf)
        plain = lambda: eng.search_batch_grouped(qs, top, per)
        fns = [call, plain]
        if name.startswith("(d)"):
            members = [np.flatnonzero(np.asarray(qw) == w) for w in range(len(ws))]
            fns.append(lambda: [eng.search_batch_grouped_where(qs[m], top, per, ws[w]) for w, m in enumerate(members)])
        times = alternate(fns, steps)
        before = {k: eng.counter(k) for k in COUNTERS}
        got = call()
        counts = {k: eng.counter(k) - v for k, v in before.items()}
        sample = rng.choice(B, SAMPLE, replace=False)
        lists, build, loop = [], 0.0, 0.0
        for qi in sample:
            t = time.perf_counter()
            allow = passing(None if qw[qi] is None else ws[qw[qi]], None if qf[qi] is None else fl[qf[qi]])
            build += time.perf_counter() - t
            lists.append(allow)
        want = []
        for qi, allow in zip(sample, lists):
            t = time.perf_counter()
            want.append(eng.search_grouped(qs[qi], top, per, allow=allow) if allow.size else [])
            loop += time.perf_counter() - t
        mismatches = sum(flat(got[qi]) != flat(w) for qi, w in zip(sample, want))
        line = {"workload": name, "corpus": f"{N} x {DIMS} cosine, fill_synthetic, groups of {GROUP}", "batch": B,
                "top_groups": top, "per_group": per, "steps": steps, "multi_where_ms": times[0] * 1e3,
                "unfiltered_grouped_batch_ms": times[1] * 1e3,
                "single_call_loop_ms_extrapolated_from_32": loop / SAMPLE * B * 1e3,
                "single_call_allow_list_host_build_ms_extrapolated_from_32": build / SAMPLE * B * 1e3,
                "mean_allow_list_frames": float(np.mean([x.size for x in lists])),
                "checked": SAMPLE, "mismatches": int(mismatches), "counters_one_call": counts, **info}
        if len(times) > 2:
            line["one_grouped_where_call_per_distinct_where_ms"] = times[2] * 1e3
        lines.append(line)
        print(json.dumps(line), flush=True)
    if record:
        record.parent.mkdir(parents=True, exist_ok=True)
        record.write_text(json.dumps({"workloads": lines}, indent=1) + "\n")
    eng.close()


if __name__ == "__main__":
    main()
