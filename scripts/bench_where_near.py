#!/usr/bin/env python
"""PhotoRAG's location query below the top-k (wax_vs_search_batch_where_near) on 10 M x 384 cosine rows
(fill_synthetic): 70 % of the rows carry a location, clustered around 300 seeded centres with a spread of about 20 km,
1 % are tagged deleted, timestamps increase with the row; batch 1 024, top-10.  Workloads:
  (a) 1 024 queries, each a 25 km radius AND a 20 % time window AND not deleted;
  (b) the same with 1 km radii (the gather class);
  (c) grouped in PhotoRAG's shape: groups of 8 rows, 12 groups x 1 frame, one box (25 km) and window for the batch;
  (d) one query, a 25 km radius AND a 20 % window.
Each reports the wall time of the public C call, measured alternating in the same run against two baselines: today's
PhotoRAG form (the allow-list of every frame in the box's bins, built on the host and passed with the same where to
search_batch_where / search_batch_grouped_where; its host build time is reported apart) and the unfiltered batch.
Sampled answers of the two forms must be identical.  A separate run under torch.profiler reports the device time of the
where kernels.  Prints one JSON line per workload with the card's name and power limit, and writes them all to the
record file given as the first argument.

usage: scripts/bench_where_near.py [record.json] [steps]"""
import json
import math
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from wax_b200 import CUDAVectorEngine, VectorMetric, Where, location_box  # noqa: E402

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


def bits(hits):
    return [(i, np.float32(s).view(np.uint32).item()) for i, s in hits]


class Bins:
    """index.locationBins as one sorted array: the located rows ordered by (latBin, lonBin).  A box's allow-list is the
    union of its bins' rows, one searchsorted pair per lat bin (bins are disjoint, so the union is a concatenation)."""

    def __init__(self, lat, lon):
        located = np.flatnonzero(~np.isnan(lat))
        lat_bin = np.floor(lat[located] * 100.0).astype(np.int64)
        lon_bin = np.floor(lon[located] * 100.0).astype(np.int64)
        key = (lat_bin << 32) + (lon_bin + (1 << 31))
        order = np.argsort(key, kind="stable")
        self.key, self.rows = key[order], located[order].astype(np.uint64)

    def allowlist(self, near):
        box = location_box(*near)
        assert box is not None
        lat_lo, lat_hi, lon_lo, lon_hi = box
        assert lon_lo <= lon_hi                    # the antimeridian branch needs a negative lonDelta
        parts = []
        for lb in range(lat_lo, lat_hi + 1):
            a = np.searchsorted(self.key, (lb << 32) + (lon_lo + (1 << 31)), "left")
            b = np.searchsorted(self.key, (lb << 32) + (lon_hi + (1 << 31)), "right")
            parts.append(self.rows[a:b])
        return np.concatenate(parts) if parts else np.zeros(0, np.uint64)


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
    t = time.perf_counter()
    eng.set_locations(frames, lat, lon)
    set_ms = (time.perf_counter() - t) * 1e3
    index = Bins(lat, lon)
    qs = rng.uniform(-1, 1, size=(B, DIMS)).astype(np.float32)
    qs /= np.linalg.norm(qs, axis=1, keepdims=True)

    def wheres(radius, count):
        out = []
        for _ in range(count):
            a = int(rng.integers(0, N - N // 5))
            ci = int(rng.integers(0, n_c))
            out.append(Where(after=a, before=a + N // 5, no_tags=DELETED,
                             near=(float(lat_c[ci]), float(lon_c[ci]), radius)))
        return out

    def photorag_form(ws):
        """Today's PhotoRAG request: the box's frames as an allow-list beside the same where (no near)."""
        t = time.perf_counter()
        lists = [("allow", index.allowlist(w.near)) for w in ws]
        build = time.perf_counter() - t
        plain = [Where(after=w.after, before=w.before, no_tags=w.no_tags) for w in ws]
        return lists, plain, build

    lines = []
    uploads0 = eng.counter("location_uploads")
    unfiltered = lambda: eng.search_batch_arrays(qs, K)
    for name, radius in (("(a) 1024 x (25 km AND 20 % window AND not deleted)", 25_000.0),
                         ("(b) 1024 x (1 km AND 20 % window AND not deleted)", 1_000.0)):
        ws = wheres(radius, B)
        lists, plain, build = photorag_form(ws)
        near_call = lambda: eng.search_batch_where(qs, K, ws, list(range(B)))
        id_call = lambda: eng.search_batch_where(qs, K, plain, list(range(B)), lists, list(range(B)))
        near_s, id_s, plain_s = alternate([near_call, id_call, unfiltered], steps)
        got, want = near_call(), id_call()
        mismatches = sum(bits(g) != bits(w) for g, w in zip(got, want))
        line = {"workload": name, "corpus": f"{N} x {DIMS} cosine, fill_synthetic", "batch": B, "top_k": K,
                "steps": steps, "where_near_ms": near_s * 1e3, "photorag_allow_list_form_ms": id_s * 1e3,
                "photorag_allow_list_host_build_ms": build * 1e3, "unfiltered_search_batch_ms": plain_s * 1e3,
                "allow_list_ids": int(sum(x.size for _, x in lists)), "checked": B, "mismatches": int(mismatches),
                **info}
        lines.append(line)
        print(json.dumps(line), flush=True)
    # (c) grouped, one box and window for the batch
    eng.set_groups(frames, frames // 8)
    w = wheres(25_000.0, 1)[0]
    lists, plain, build = photorag_form([w])
    near_call = lambda: eng.search_batch_grouped_where(qs, 12, 1, w)
    id_call = lambda: eng.search_batch_grouped_where(qs, 12, 1, plain[0], allow=lists[0][1])
    plain_call = lambda: eng.search_batch_grouped(qs, 12, 1)
    near_s, id_s, plain_s = alternate([near_call, id_call, plain_call], steps)
    got, want = near_call(), id_call()
    line = {"workload": "(c) grouped: groups of 8, 12 x 1, one 25 km box AND 20 % window", "corpus": f"{N} x {DIMS}",
            "batch": B, "where_near_ms": near_s * 1e3, "photorag_allow_list_form_ms": id_s * 1e3,
            "photorag_allow_list_host_build_ms": build * 1e3, "unfiltered_grouped_batch_ms": plain_s * 1e3,
            "allow_list_ids": int(lists[0][1].size), "checked": B,
            "mismatches": int(sum(g != x for g, x in zip(got, want))), **info}
    lines.append(line)
    print(json.dumps(line), flush=True)
    # (d) one query
    w = wheres(25_000.0, 1)[0]
    lists, plain, build = photorag_form([w])
    q = qs[0]
    near_call = lambda: eng.search_where(q, K, w)
    id_call = lambda: eng.search_where(q, K, plain[0], allow=lists[0][1])
    plain_call = lambda: eng.search(q, K)
    near_s, id_s, plain_s = alternate([near_call, id_call, plain_call], max(steps, 20))
    line = {"workload": "(d) one query, 25 km AND 20 % window", "corpus": f"{N} x {DIMS}", "top_k": K,
            "where_near_ms": near_s * 1e3, "photorag_allow_list_form_ms": id_s * 1e3,
            "photorag_allow_list_host_build_ms": build * 1e3, "unfiltered_search_ms": plain_s * 1e3,
            "mismatches": 0 if bits(near_call()) == bits(id_call()) else 1, **info}
    lines.append(line)
    print(json.dumps(line), flush=True)
    setup = {"set_locations_10M_ms": set_ms, "location_uploads": eng.counter("location_uploads") - uploads0, **info}
    # device time of the where kernels: one call of (a) and (b) under torch.profiler, in a run of its own
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.init()
        wa, wb = wheres(25_000.0, B), wheres(1_000.0, B)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.search_batch_where(qs, K, wa, list(range(B)))
            eng.search_batch_where(qs, K, wb, list(range(B)))
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            if "where_" in ev.key or "filter_bits" in ev.key or "gather_" in ev.key:
                kern[ev.key.split("(")[0]] = {"calls": ev.count, "device_ms_total": ev.device_time_total / 1e3}
        setup["kernels_a_b_one_call_each"] = kern
    except Exception as ex:  # noqa: BLE001
        setup["kernels_error"] = repr(ex)
    print(json.dumps(setup), flush=True)
    if record:
        record.parent.mkdir(parents=True, exist_ok=True)
        record.write_text(json.dumps({"workloads": lines, "setup": setup}, indent=1) + "\n")
    eng.close()


if __name__ == "__main__":
    main()
