"""Batched grouped search (wax_vs_search_batch_grouped) against a loop of wax_vs_search_grouped over the same queries.

Corpus: 10 M x 384 cosine rows from fill_synthetic, batches of 1 024 and 64 queries.  Workloads:
  (a) groups of 8 consecutive rows, 12 groups x 1 row
  (b) groups of 360 consecutive rows, 12 x 3
  (c) hashed groups (not contiguous, 360 rows on average), 12 x 3
  (d) as (b) under an allow-list of 1 M frames
  (e) one group holding half the rows, 12 x 3 (expansions of a 5 M-row group when its listed rows fall short)
  (f) one group holding 99 % of the rows, 12 x 3: the top rows name too few groups, every query falls back
Per workload and batch size: the batch call (median of --iters after a warm-up), one timed loop of the single call over the
same queries, search_batch at k = k_c (the coverage level's floor; search_batch_filtered for (d)), queries per second,
the three grouped_batch_* counters of one batch call, and whether every query's answer equals its single call (ids, group
ids, order, score bits).  The card name and power limit are read in the same run.  Prints one JSON line (also written to
the file --out names, if given).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from wax_b200 import CUDAVectorEngine, VectorMetric  # noqa: E402
from wax_b200 import _lib as L  # noqa: E402

ROWS, DIMS = 10_000_000, 384
COUNTERS = ("grouped_batch_covered_queries", "grouped_batch_expanded_groups", "grouped_batch_fallback_queries")


def _u64(a):
    return a.ctypes.data_as(C.POINTER(C.c_uint64))


def _f32(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _u32(a):
    return a.ctypes.data_as(C.POINTER(C.c_uint32))


def _filter(allow):
    return (_u64(allow), allow.size, 0) if allow is not None else (None, 0, 1)


def batch_grouped(h, qs, top, per, allow):
    b, cap = qs.shape[0], top * per
    ids, groups = np.zeros((b, cap), np.uint64), np.zeros((b, cap), np.uint64)
    scores, ns = np.zeros((b, cap), np.float32), np.zeros(b, np.uint32)
    fp, nf, mode = _filter(allow)
    rc = L.lib().wax_vs_search_batch_grouped(h, _f32(qs), b, DIMS, top, per, fp, nf, mode, _u64(ids), _f32(scores),
                                             _u64(groups), cap, _u32(ns))
    assert rc == L.OK, L.last_error()
    return ids, scores, groups, ns


def loop_grouped(h, qs, top, per, allow):
    b, cap = qs.shape[0], top * per
    ids, groups = np.zeros((b, cap), np.uint64), np.zeros((b, cap), np.uint64)
    scores, ns = np.zeros((b, cap), np.float32), np.zeros(b, np.uint32)
    fp, nf, mode = _filter(allow)
    n = C.c_uint32(0)
    for i in range(b):
        rc = L.lib().wax_vs_search_grouped(h, _f32(qs[i]), DIMS, top, per, fp, nf, mode, _u64(ids[i]), _f32(scores[i]),
                                           _u64(groups[i]), cap, C.byref(n))
        assert rc == L.OK, L.last_error()
        ns[i] = n.value
    return ids, scores, groups, ns


def plain_batch(h, qs, k, allow):
    b = qs.shape[0]
    ids, scores, ns = np.zeros((b, k), np.uint64), np.zeros((b, k), np.float32), np.zeros(b, np.uint32)
    if allow is None:
        rc = L.lib().wax_vs_search_batch(h, _f32(qs), b, DIMS, k, _u64(ids), _f32(scores), k, _u32(ns))
    else:
        rc = L.lib().wax_vs_search_batch_filtered(h, _f32(qs), b, DIMS, k, _u64(allow), allow.size, 0, _u64(ids),
                                                  _f32(scores), k, _u32(ns))
    assert rc == L.OK, L.last_error()


def same(a, b):
    ids, scores, groups, ns = a
    ids2, scores2, groups2, ns2 = b
    if not np.array_equal(ns, ns2):
        return False
    for i in range(ns.size):
        m = int(ns[i])
        if not (np.array_equal(ids[i, :m], ids2[i, :m]) and np.array_equal(groups[i, :m], groups2[i, :m]) and
                np.array_equal(scores[i, :m].view(np.uint32), scores2[i, :m].view(np.uint32))):
            return False
    return True


def timed(fn, iters):
    out, ts = None, []
    for _ in range(iters):
        t0 = time.perf_counter()
        out = fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return out, statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=ROWS)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--batches", default="1024,64")
    ap.add_argument("--workloads", default="abcdef")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    rows = args.rows
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    eng = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    eng.fill_synthetic(1, rows)
    h = eng.handle
    rng = np.random.default_rng(0)
    batches = [int(x) for x in args.batches.split(",")]
    qs_all = rng.standard_normal((max(batches), DIMS)).astype(np.float32)
    qs_all /= np.linalg.norm(qs_all, axis=1, keepdims=True)
    frames = np.arange(rows, dtype=np.uint64)
    half = frames.copy()
    half[rng.permutation(rows)[: rows // 2]] = 10**15
    most = frames.copy()
    most[rng.permutation(rows)[: rows * 99 // 100]] = 10**15
    allow = np.sort(rng.choice(rows, min(1_000_000, rows), replace=False)).astype(np.uint64)
    workloads = {
        "a": ("blocks8, 12 x 1", frames // 8 * 8, 12, 1, None),
        "b": ("blocks360, 12 x 3", frames // 360 * 360, 12, 3, None),
        "c": ("hashed360, 12 x 3", (frames * 2654435761) % (rows // 360) + 10**12, 12, 3, None),
        "d": ("blocks360 under a 1 M-frame allow-list, 12 x 3", frames // 360 * 360, 12, 3, allow),
        "e": ("one group of half the rows, 12 x 3", half, 12, 3, None),
        "f": ("one group of 99 % of the rows, 12 x 3 (crowded)", most, 12, 3, None),
    }
    res = {"gpu": smi, "rows": rows, "dims": DIMS, "metric": "cosine", "iters": args.iters,
           "unit": "ms per batch (wall time of the C call)", "workloads": {}}
    for key in args.workloads:
        name, groups, top, per, flt = workloads[key]
        eng.set_groups(frames, groups)
        k_c = min(1024, max(128, 4 * top))
        entry = {"name": name, "k_c": k_c}
        for b in batches:
            qs = np.ascontiguousarray(qs_all[:b])
            batch_grouped(h, qs, top, per, flt)                       # warm-up (index build, scratch)
            c0 = np.array([eng.counter(c) for c in COUNTERS])
            batch_grouped(h, qs, top, per, flt)
            c1 = np.array([eng.counter(c) for c in COUNTERS])
            got, t_batch = timed(lambda: batch_grouped(h, qs, top, per, flt), args.iters)
            want, t_loop = timed(lambda: loop_grouped(h, qs, top, per, flt), 1)
            plain_batch(h, qs, k_c, flt)
            _, t_floor = timed(lambda: plain_batch(h, qs, k_c, flt), args.iters)
            entry[f"batch{b}"] = {
                "batch_ms": round(t_batch, 2), "loop_ms": round(t_loop, 2), "search_batch_kc_ms": round(t_floor, 2),
                "batch_qps": round(b / t_batch * 1e3, 1), "loop_qps": round(b / t_loop * 1e3, 1),
                "speedup_vs_loop": round(t_loop / t_batch, 2),
                "counters": dict(zip(COUNTERS, (c1 - c0).tolist())),
                "equal_to_single": bool(same(got, want)),
            }
        res["workloads"][key] = entry
    eng.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
