#!/usr/bin/env python
"""Wax's metadataFilter below the top-k (wax_vs_search_batch_where_terms) on 10 M x 384 cosine rows (fill_synthetic).
Every row holds one session_id term (sessions of seeded, log-uniform sizes between 100 and 600 K frames, one of exactly
5 000) and one of four kind terms; 1 % are tagged deleted; timestamps increase with the row.  Batch 1 024, top-10.
Workloads:
  (a) 1 024 queries, each its own small session (<= 20 000 frames) AND not deleted;
  (b) 1 024 queries over the 16 largest sessions AND not deleted;
  (c) 1 024 queries, each a session AND a kind AND a 20 % time window;
  (d) one query in the session of 5 000 frames AND not deleted.
Each reports the wall time of the public C call, alternating in the same run with two baselines: the same filter as a
host-built id allow-list passed with the same where (no terms) to search_batch_where (its host build time is reported
apart), and the unfiltered batch.  Sampled answers of the two filtered forms must be identical.  Also reports the wall
time of set_terms for every row and of the first search, which builds the term index, and the index's device bytes.
Prints one JSON line per workload with the card's name and power limit, and writes them all to the record file given as
the first argument.

usage: scripts/bench_where_terms.py [record.json] [steps]"""
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
SESSION, KIND = 1 << 32, 16                # term ids: SESSION + s, KIND + k
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
    rng = np.random.default_rng(23)
    frames = np.arange(N, dtype=np.uint64)
    tags = np.where(rng.random(N) < 0.01, DELETED, 0).astype(np.uint64)
    eng.set_attributes(frames, np.arange(N, dtype=np.int64), tags)
    sizes = [5000]
    while sum(sizes) < N:
        sizes.append(int(np.exp(rng.uniform(np.log(100), np.log(600_000)))))
    sizes[-1] -= sum(sizes) - N
    sizes = np.asarray(sizes)
    session = np.repeat(np.arange(sizes.size), sizes)[rng.permutation(N)]
    kind = rng.integers(0, 4, N)
    terms = np.stack([SESSION + session.astype(np.uint64), KIND + kind.astype(np.uint64)], 1).reshape(-1)
    offsets = np.arange(N + 1, dtype=np.uint64) * 2
    p = lambda a: a.ctypes.data_as(C.POINTER(C.c_uint64))
    t = time.perf_counter()
    assigned = C.c_uint64(0)
    assert L.lib().wax_vs_set_terms(eng._h, p(frames), p(offsets), p(terms), N, C.byref(assigned)) == L.OK
    set_ms = (time.perf_counter() - t) * 1e3
    order = np.argsort(session, kind="stable")                # the host form: each session's frames, once
    starts = np.concatenate([[0], np.cumsum(sizes)])
    members = lambda s: frames[order[starts[s]:starts[s + 1]]]
    qs = rng.uniform(-1, 1, size=(B, DIMS)).astype(np.float32)
    qs /= np.linalg.norm(qs, axis=1, keepdims=True)

    t = time.perf_counter()
    eng.search_where(qs[0], K, Where(terms=(SESSION + 0,)))
    first_ms = (time.perf_counter() - t) * 1e3

    small = np.flatnonzero(sizes <= 20_000)
    large = np.argsort(sizes)[-16:]
    workloads = []
    ws = [Where(terms=(SESSION + int(s),), no_tags=DELETED) for s in rng.choice(small, B)]
    workloads.append(("(a) 1024 x (own small session AND not deleted)", ws, None))
    ws = [Where(terms=(SESSION + int(s),), no_tags=DELETED) for s in rng.choice(large, B)]
    workloads.append(("(b) 1024 x (one of 16 large sessions AND not deleted)", ws, None))
    ws = []
    for s in rng.integers(0, sizes.size, B):
        a = int(rng.integers(0, N - N // 5))
        ws.append(Where(terms=(SESSION + int(s), KIND + int(rng.integers(0, 4))), after=a, before=a + N // 5))
    workloads.append(("(c) 1024 x (session AND kind AND 20 % window)", ws, None))

    def host_form(ws):
        t = time.perf_counter()
        lists = []
        for w in ws:
            rows = members(int(w.terms[0] - SESSION))
            if len(w.terms) > 1:
                rows = rows[kind[rows.astype(np.int64)] == w.terms[1] - KIND]
            lists.append(("allow", rows))
        build = time.perf_counter() - t
        plain = [Where(after=w.after, before=w.before, no_tags=w.no_tags) for w in ws]
        return lists, plain, build

    lines = []
    builds0 = eng.counter("term_index_builds")
    unfiltered = lambda: eng.search_batch_arrays(qs, K)
    for name, ws, _ in workloads:
        lists, plain, build = host_form(ws)
        terms_call = lambda: eng.search_batch_where(qs, K, ws, list(range(B)))
        id_call = lambda: eng.search_batch_where(qs, K, plain, list(range(B)), lists, list(range(B)))
        terms_s, id_s, plain_s = alternate([terms_call, id_call, unfiltered], steps)
        got, want = terms_call(), id_call()
        mismatches = sum(bits(g) != bits(w) for g, w in zip(got, want))
        line = {"workload": name, "corpus": f"{N} x {DIMS} cosine, fill_synthetic", "batch": B, "top_k": K,
                "steps": steps, "where_terms_ms": terms_s * 1e3, "host_allow_list_form_ms": id_s * 1e3,
                "host_allow_list_build_ms": build * 1e3, "unfiltered_search_batch_ms": plain_s * 1e3,
                "allow_list_ids": int(sum(x.size for _, x in lists)), "checked": B, "mismatches": int(mismatches),
                **info}
        lines.append(line)
        print(json.dumps(line), flush=True)
    # (d) one query in the session of 5 000 frames
    w = Where(terms=(SESSION + 0,), no_tags=DELETED)
    lists, plain, build = host_form([w])
    q = qs[0]
    terms_call = lambda: eng.search_where(q, K, w)
    id_call = lambda: eng.search_where(q, K, plain[0], allow=lists[0][1])
    plain_call = lambda: eng.search(q, K)
    terms_s, id_s, plain_s = alternate([terms_call, id_call, plain_call], max(steps, 20))
    line = {"workload": "(d) one query, a session of 5000 frames AND not deleted", "corpus": f"{N} x {DIMS}",
            "top_k": K, "where_terms_ms": terms_s * 1e3, "host_allow_list_form_ms": id_s * 1e3,
            "host_allow_list_build_ms": build * 1e3, "unfiltered_search_ms": plain_s * 1e3,
            "mismatches": 0 if bits(terms_call()) == bits(id_call()) else 1, **info}
    lines.append(line)
    print(json.dumps(line), flush=True)
    setup = {"set_terms_10M_ms": set_ms, "first_search_with_index_build_ms": first_ms, "sessions": int(sizes.size),
             "term_index_bytes": eng.counter("term_index_bytes"),
             "term_index_builds_during_workloads": eng.counter("term_index_builds") - builds0, **info}
    try:                                       # device time of the term kernels: one call of (a) and (b), own run
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.init()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.search_batch_where(qs, K, workloads[0][1], list(range(B)))
            eng.search_batch_where(qs, K, workloads[1][1], list(range(B)))
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            if "term_" in ev.key or "filter_bits" in ev.key or "gather_" in ev.key:
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
