"""GPU: the argument checks of the filtered, where and grouped entry points, malformed call by malformed call.

Every host entry point must fail alike on a multi-device handle (two shards on device 0) and on one engine, empty and
after an add_batch: the same code, the same wax_vs_last_error() text and the same out_n.  Several calls carry more than
one fault, so the order of the checks is pinned too.  The one known difference is the sharded grouped form's refusal of
clamp(top_groups) > 256, asserted on its own.  The device and shard forms refuse a multi-device handle, so each of their
calls is pinned to the code and reason one engine gives."""
import ctypes as C

import numpy as np
import pytest
import torch

from wax_b200 import CUDAVectorEngine, VectorMetric
from wax_b200 import _lib as L

pytestmark = pytest.mark.gpu

DIMS, NQ, CAP, ROWS = 16, 3, 512, 40
SENTINEL = 0xDEAD
NF = L.NO_FILTER
BAD_BOX = (40.0, -73.9, 1e300)                  # a radius whose box is not representable
BOX_REASON = "location box of (40, -73.9, 1e+300 m) is not representable"

# the valid arguments every call starts from; a fault replaces some of them
BASE = dict(nq=NQ, qlen=DIMS, top_k=10, per_group=2, ids=[1, 2, 3], n_ids=3, mode=0, offsets=[0, 2, 3], modes=[0, 1],
            n_filters=2, qf=[0, 1, NF], where=(100, 900, 0, 0), near=(40.0, -73.9, 5000.0), qw=[0, NF, 1], n_wheres=2,
            term_offsets=[0, 1, 2], terms=[5, 6], stride=CAP, out_ids=True, out_scores=True, out_groups=True, out_n=True,
            queries=True)


def _u64(v):
    return None if v is None else (C.c_uint64 * max(len(v), 1))(*v)


def _u32(v):
    return None if v is None else (C.c_uint32 * max(len(v), 1))(*v)


def _i32(v):
    return None if v is None else (C.c_int32 * max(len(v), 1))(*v)


def _where(w):
    return L.Where(w[0], w[1], w[2], w[3])


def _wheres(a, near):
    """n_wheres wheres, the second one carrying a["near"] (a location box, or None)."""
    if a["where"] is None:
        return None
    n = max(a["n_wheres"], 1)
    if not near:
        return C.cast((L.Where * n)(*[_where(a["where"])] * n), C.c_void_p)
    arr = (L.WhereNear * n)(*[L.WhereNear(_where(a["where"]), 40.0, -73.9, 5000.0)] * n)
    if n > 1 and a["near"] is not None:
        arr[1] = L.WhereNear(_where(a["where"]), *a["near"])
    return C.cast(arr, C.c_void_p)


def _one_where(a, near):
    if a["where"] is None:
        return None
    w = L.WhereNear(_where(a["where"]), *a["near"]) if near else _where(a["where"])
    return C.cast(C.pointer(w), C.c_void_p)


def _host_call(name, h, fault):
    """One call of a host entry point: (rc, reason when it failed, out_n or None)."""
    a = dict(BASE, **fault)
    rng = np.random.default_rng(1)
    q = rng.standard_normal((max(a["nq"], 1), DIMS)).astype(np.float32)
    qp = q.ctypes.data_as(C.POINTER(C.c_float)) if a["queries"] else None
    ids = np.zeros((max(a["nq"], 1), CAP), np.uint64)
    scores = np.zeros((max(a["nq"], 1), CAP), np.float32)
    groups = np.zeros((max(a["nq"], 1), CAP), np.uint64)
    out_n = np.full(max(a["nq"], 1), SENTINEL, np.uint32)
    oi = ids.ctypes.data_as(C.POINTER(C.c_uint64)) if a["out_ids"] else None
    os_ = scores.ctypes.data_as(C.POINTER(C.c_float)) if a["out_scores"] else None
    og = groups.ctypes.data_as(C.POINTER(C.c_uint64)) if a["out_groups"] else None
    on = out_n.ctypes.data_as(C.POINTER(C.c_uint32)) if a["out_n"] else None
    filters = (_u64(a["ids"]), _u64(a["offsets"]), _i32(a["modes"]), a["n_filters"], _u32(a["qf"]))
    one = (_u64(a["ids"]), a["n_ids"], a["mode"])
    lib = L.lib()
    if name == "search_filtered":
        rc = lib.wax_vs_search_filtered(h, qp, a["qlen"], a["top_k"], *one, oi, os_, a["stride"], on)
    elif name == "search_batch_filtered":
        rc = lib.wax_vs_search_batch_filtered(h, qp, a["nq"], a["qlen"], a["top_k"], *one, oi, os_, a["stride"], on)
    elif name == "search_batch_multi_filtered":
        rc = lib.wax_vs_search_batch_multi_filtered(h, qp, a["nq"], a["qlen"], a["top_k"], *filters, oi, os_, a["stride"],
                                                    on)
    elif name in ("search_batch_where", "search_batch_where_near"):
        fn = getattr(lib, "wax_vs_" + name)
        rc = fn(h, qp, a["nq"], a["qlen"], a["top_k"], *filters, _wheres(a, name.endswith("near")), a["n_wheres"],
                _u32(a["qw"]), oi, os_, a["stride"], on)
    elif name == "search_batch_where_terms":
        rc = lib.wax_vs_search_batch_where_terms(h, qp, a["nq"], a["qlen"], a["top_k"], *filters, _wheres(a, True),
                                                 a["n_wheres"], _u32(a["qw"]), _u64(a["term_offsets"]), _u64(a["terms"]),
                                                 oi, os_, a["stride"], on)
    elif name == "search_grouped":
        rc = lib.wax_vs_search_grouped(h, qp, a["qlen"], a["top_k"], a["per_group"], *one, oi, os_, og, a["stride"], on)
    elif name == "search_batch_grouped":
        rc = lib.wax_vs_search_batch_grouped(h, qp, a["nq"], a["qlen"], a["top_k"], a["per_group"], *one, oi, os_, og,
                                             a["stride"], on)
    elif name in ("search_batch_grouped_where", "search_batch_grouped_where_near"):
        fn = getattr(lib, "wax_vs_" + name)
        rc = fn(h, qp, a["nq"], a["qlen"], a["top_k"], a["per_group"], *one, _one_where(a, name.endswith("near")), oi, os_,
                og, a["stride"], on)
    elif name == "search_batch_grouped_multi_where":
        rc = lib.wax_vs_search_batch_grouped_multi_where(h, qp, a["nq"], a["qlen"], a["top_k"], a["per_group"], *filters,
                                                         _wheres(a, True), a["n_wheres"], _u32(a["qw"]), oi, os_, og,
                                                         a["stride"], on)
    else:
        raise KeyError(name)
    n = 1 if name in ("search_filtered", "search_grouped") else a["nq"]
    return rc, L.last_error() if rc else "", out_n[:n].tolist() if a["out_n"] else None


FILTERED = ["search_filtered", "search_batch_filtered"]
MULTI_FILTERED = ["search_batch_multi_filtered"]
WHERE = ["search_batch_where", "search_batch_where_near", "search_batch_where_terms"]
GROUPED = ["search_grouped", "search_batch_grouped"]
GROUPED_WHERE = ["search_batch_grouped_where", "search_batch_grouped_where_near"]
GROUPED_MULTI = ["search_batch_grouped_multi_where"]
ALL = FILTERED + MULTI_FILTERED + WHERE + GROUPED + GROUPED_WHERE + GROUPED_MULTI
PER_QUERY = MULTI_FILTERED + WHERE + GROUPED_MULTI
ONE_FILTER = FILTERED + GROUPED + GROUPED_WHERE

# (entry points, fault): every call of the table runs on the multi-device handle and on one engine, empty and not
FAULTS = [
    (ALL, {}),                                                           # valid
    (ALL, {"out_n": False}),
    (ALL, {"out_ids": False}),
    (ALL, {"out_scores": False}),
    (ALL, {"queries": False}),
    (ALL, {"qlen": DIMS + 1}),
    (ALL, {"qlen": DIMS + 1, "stride": 1}),                              # the query before the buffer size
    (ALL, {"stride": 1}),
    (ALL, {"nq": 0, "qlen": DIMS + 1}),
    (ALL, {"top_k": 0}),
    (ALL, {"top_k": -5, "per_group": 1}),
    (GROUPED + GROUPED_WHERE + GROUPED_MULTI, {"out_groups": False}),
    (GROUPED + GROUPED_WHERE + GROUPED_MULTI, {"per_group": 0}),
    (GROUPED + GROUPED_WHERE + GROUPED_MULTI, {"per_group": L.MAX_PER_GROUP + 1}),
    (GROUPED + GROUPED_WHERE + GROUPED_MULTI, {"top_k": 100, "per_group": 128}),
    (GROUPED + GROUPED_WHERE + GROUPED_MULTI, {"per_group": 0, "out_ids": False}),   # the outputs first
    (GROUPED + GROUPED_WHERE + GROUPED_MULTI, {"per_group": 0, "mode": 2, "modes": [0, 5]}),
    (GROUPED + GROUPED_WHERE + GROUPED_MULTI, {"top_k": 300, "per_group": 0}),
    (GROUPED + GROUPED_WHERE + GROUPED_MULTI, {"top_k": 300, "per_group": 1}),
    (GROUPED + GROUPED_WHERE + GROUPED_MULTI, {"top_k": 300, "per_group": 1, "qlen": DIMS + 1}),
    (GROUPED + GROUPED_WHERE + GROUPED_MULTI, {"top_k": 300, "per_group": 1, "queries": False}),
    (GROUPED + GROUPED_WHERE + GROUPED_MULTI, {"top_k": 300, "per_group": 1, "stride": 1}),
    (GROUPED + GROUPED_WHERE + GROUPED_MULTI, {"top_k": 300, "per_group": 1, "mode": 2, "qf": [0, 7, NF]}),
    (ONE_FILTER, {"mode": 2}),
    (ONE_FILTER, {"mode": -1, "ids": None}),                             # the mode before the ids
    (ONE_FILTER, {"ids": None}),
    (ONE_FILTER, {"ids": None, "n_ids": 0}),
    (ONE_FILTER, {"ids": [], "n_ids": 0, "mode": 1}),                    # an empty deny-list
    (ONE_FILTER, {"ids": [], "n_ids": 0, "mode": 0}),                    # an empty allow-list
    (ONE_FILTER, {"mode": 2, "out_n": False}),
    (PER_QUERY, {"offsets": None}),
    (PER_QUERY, {"modes": None}),
    (PER_QUERY, {"qf": None}),
    (PER_QUERY, {"qf": None, "nq": 0}),
    (PER_QUERY, {"ids": None}),
    (PER_QUERY, {"modes": [0, 5]}),
    (PER_QUERY, {"offsets": [1, 2, 3]}),
    (PER_QUERY, {"offsets": [0, 3, 2]}),
    (PER_QUERY, {"qf": [0, 7, NF]}),
    (PER_QUERY, {"modes": [0, 5], "offsets": [1, 2, 3]}),                # the modes before the offsets
    (PER_QUERY, {"offsets": [0, 3, 2], "ids": None}),                    # the offsets before the ids
    (PER_QUERY, {"ids": None, "qf": [0, 7, NF]}),                        # the ids before the queries' filters
    (PER_QUERY, {"offsets": None, "modes": [0, 5]}),
    (PER_QUERY, {"n_filters": 0, "offsets": [0], "modes": None, "qf": [NF, NF, NF]}),
    (PER_QUERY, {"out_n": False, "offsets": None}),
    (WHERE + GROUPED_MULTI, {"where": None}),
    (WHERE + GROUPED_MULTI, {"qw": None}),
    (WHERE + GROUPED_MULTI, {"qw": [0, 9, NF]}),
    (WHERE + GROUPED_MULTI, {"qw": [0, 9, NF], "qf": [0, 7, NF]}),       # the filters before the wheres
    (WHERE + GROUPED_MULTI, {"where": None, "n_wheres": 0, "qw": [NF, NF, NF]}),
    (WHERE + GROUPED_MULTI, {"where": (0, 10, 0, 0), "qw": [0, 0, 0]}),
    (WHERE + GROUPED_MULTI, {"near": BAD_BOX}),
    (WHERE + GROUPED_MULTI, {"near": (float("nan"), -73.9, 1000.0)}),
    (WHERE + GROUPED_MULTI, {"near": (40.0, float("nan"), 1e9)}),
    (WHERE + GROUPED_MULTI, {"near": (40.0, -73.9, float("inf"))}),
    (WHERE + GROUPED_MULTI, {"near": (40.0, -73.9, float("nan"))}),
    (WHERE + GROUPED_MULTI, {"near": BAD_BOX, "qw": [0, 9, NF]}),        # the where list before the boxes
    (WHERE + GROUPED_MULTI, {"near": BAD_BOX, "qlen": DIMS + 1}),        # the boxes before the query
    (WHERE + GROUPED_MULTI, {"near": BAD_BOX, "stride": 1}),
    (GROUPED_MULTI, {"near": BAD_BOX, "per_group": 0}),                  # the grouped arguments first
    (GROUPED_MULTI, {"near": BAD_BOX, "top_k": 300, "per_group": 1}),
    (["search_batch_where_terms"], {"term_offsets": None}),
    (["search_batch_where_terms"], {"term_offsets": None, "near": BAD_BOX}),
    (["search_batch_where_terms"], {"term_offsets": None, "qw": [0, 9, NF]}),
    (["search_batch_where_terms"], {"term_offsets": [1, 1, 2]}),
    (["search_batch_where_terms"], {"term_offsets": [0, 2, 1]}),
    (["search_batch_where_terms"], {"terms": None}),
    (["search_batch_where_terms"], {"term_offsets": [0, 33, 34], "terms": list(range(34))}),   # too many terms
    (["search_batch_where_terms"], {"term_offsets": [0, 32, 33], "terms": list(range(33))}),
    (["search_batch_where_terms"], {"term_offsets": [0, 33, 34], "terms": list(range(34)), "near": BAD_BOX}),
    (["search_batch_where_terms"], {"terms": None, "near": BAD_BOX}),   # the term lists before the boxes
    (["search_batch_where_terms"], {"term_offsets": [0, 0, 0], "terms": None}),
    (["search_batch_where_terms"], {"terms": [5, 5], "qw": [0, 1, 1]}),  # equal term wheres
    (GROUPED_WHERE, {"where": None}),
    (GROUPED_WHERE, {"where": None, "out_n": False}),                   # the where first
    (GROUPED_WHERE, {"where": None, "per_group": 0}),
    (["search_batch_grouped_where_near"], {"near": BAD_BOX}),
    (["search_batch_grouped_where_near"], {"near": BAD_BOX, "out_ids": False}),   # the box before the grouped arguments
    (["search_batch_grouped_where_near"], {"near": BAD_BOX, "per_group": 0}),
    (["search_batch_grouped_where_near"], {"near": BAD_BOX, "mode": 2}),
    (["search_batch_grouped_where_near"], {"near": (float("nan"), -73.9, 1000.0)}),
    (["search_batch_grouped_where_near"], {"near": (40.0, -73.9, float("inf")), "top_k": 300, "per_group": 1}),
]

CALLS = [(name, fault) for names, fault in FAULTS for name in names]


@pytest.fixture(scope="module")
def handles():
    multi = CUDAVectorEngine(VectorMetric.cosine, DIMS, devices=[0, 0])
    one = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    yield multi, one
    multi.close()
    one.close()


def _compare(multi, one):
    """Every call alike on both handles; returns how many the multi-device handle refused for clamp(top_groups)."""
    refused = 0
    for name, fault in CALLS:
        got, want = _host_call(name, multi.handle, fault), _host_call(name, one.handle, fault)
        a = dict(BASE, **fault)
        clamp = min(max(a["top_k"], 1), L.MAX_RESULTS)
        after_common_checks = want[0] in (L.OK, L.ERR_DIMENSION, L.ERR_BUFFER) or want[1] == "query is NULL"
        if "grouped" in name and clamp > L.SHARD_MAX_GROUPS and after_common_checks:
            # the one known difference: once the common checks pass, the handle refuses what the sharded grouped form
            # refuses, empty or not, with out_n zeroed
            assert got == (L.ERR_UNSUPPORTED, f"sharded grouped search takes clamp(top_groups) <= "
                           f"{L.SHARD_MAX_GROUPS} (got {clamp})", [0] * len(want[2])), (name, fault)
            refused += 1
            continue
        assert got == want, (name, fault)
    return refused


def test_host_entries_fail_alike_on_a_multi_device_handle(handles):
    multi, one = handles
    assert multi.count == 0 and one.count == 0
    assert _compare(multi, one) == 4 * len(GROUPED + GROUPED_WHERE + GROUPED_MULTI)
    rng = np.random.default_rng(7)
    ids = np.arange(1, ROWS + 1, dtype=np.uint64)
    vecs = rng.standard_normal((ROWS, DIMS)).astype(np.float32)
    multi.add_batch(ids, vecs)
    one.add_batch(ids, vecs)
    assert _compare(multi, one) == 4 * len(GROUPED + GROUPED_WHERE + GROUPED_MULTI)
    # the table reaches every code one engine gives
    codes = {_host_call(name, one.handle, fault)[0] for name, fault in CALLS}
    assert codes == {L.OK, L.ERR_NULL, L.ERR_DIMENSION, L.ERR_ARGUMENT, L.ERR_BUFFER}, codes


# ---- the device and shard forms on one engine: each call pinned to its (code, reason) ---------------------------------
WHERE_DEVICE = [
    ({"engine": None}, (L.ERR_NULL, "NULL argument")),
    ({"offsets": None}, (L.ERR_NULL, "NULL argument")),
    ({"modes": [0, 5]}, (L.ERR_ARGUMENT, "filter mode must be 0 (allow-list) or 1 (deny-list)")),
    ({"offsets": [1, 2, 3]}, (L.ERR_ARGUMENT, "filter_offsets[0] must be 0")),
    ({"offsets": [0, 3, 2]}, (L.ERR_ARGUMENT, "filter_offsets decrease at filter 1")),
    ({"ids": None}, (L.ERR_NULL, "frame_ids is NULL")),
    ({"qf": [0, 7, NF]}, (L.ERR_ARGUMENT, "query 1 names filter 7 of 2")),
    ({"where": None}, (L.ERR_NULL, "NULL argument")),
    ({"qw": None}, (L.ERR_NULL, "NULL argument")),
    ({"qw": [0, 9, NF]}, (L.ERR_ARGUMENT, "query 1 names where 9 of 2")),
    ({"qw": [0, 9, NF], "modes": [0, 5]}, (L.ERR_ARGUMENT, "filter mode must be 0 (allow-list) or 1 (deny-list)")),
    ({"d_queries": None}, (L.ERR_NULL, "NULL argument")),
    ({"d_out": None}, (L.ERR_NULL, "NULL argument")),
    ({"d_queries": None, "qw": [0, 9, NF]}, (L.ERR_ARGUMENT, "query 1 names where 9 of 2")),   # device pointers after
    ({"near": BAD_BOX, "terms_list": False}, (L.ERR_ARGUMENT, BOX_REASON)),
    ({"near": BAD_BOX, "d_out": None}, (L.ERR_NULL, "NULL argument")),                          # ... before the clauses
    ({"near": BAD_BOX}, (L.ERR_ARGUMENT, BOX_REASON)),
    ({"near": (40.0, -73.9, float("inf")), "terms_list": False},
     (L.ERR_ARGUMENT, "location box of (40, -73.9, inf m) is not representable")),
    ({"term_offsets": [1, 1, 2]}, (L.ERR_ARGUMENT, "where_term_offsets[0] must be 0")),
    ({"term_offsets": [0, 2, 1]}, (L.ERR_ARGUMENT, "where_term_offsets decrease at list 1")),
    ({"terms": None}, (L.ERR_NULL, "term list is NULL")),
    ({"term_offsets": [0, 33, 34], "terms": list(range(34))},
     (L.ERR_ARGUMENT, "where_term_offsets: list 0 has 33 terms, at most 32 are allowed")),
    ({"term_offsets": [0, 33, 34], "terms": list(range(34)), "near": BAD_BOX},
     (L.ERR_ARGUMENT, "where_term_offsets: list 0 has 33 terms, at most 32 are allowed")),
]

GROUPED_DEVICE = [
    ({"engine": None}, (L.ERR_NULL, "NULL argument")),
    ({"per_group": 0}, (L.ERR_ARGUMENT, "per_group must be in [1, 128] (got 0)")),
    ({"per_group": 129}, (L.ERR_ARGUMENT, "per_group must be in [1, 128] (got 129)")),
    ({"top_k": 100, "per_group": 128}, (L.ERR_ARGUMENT, "clamp(top_groups) x per_group = 12800 exceeds 10000")),
    ({"per_group": 0, "offsets": None}, (L.ERR_ARGUMENT, "per_group must be in [1, 128] (got 0)")),
    ({"top_k": 300, "per_group": 1},
     (L.ERR_UNSUPPORTED, "sharded grouped search takes clamp(top_groups) <= 256 (got 300)")),
    ({"top_k": 300, "per_group": 1, "qf": [0, 7, NF]}, (L.ERR_ARGUMENT, "query 1 names filter 7 of 2")),
    ({"top_k": 300, "per_group": 1, "qw": [0, 9, NF]}, (L.ERR_ARGUMENT, "query 1 names where 9 of 2")),
    ({"top_k": 300, "per_group": 1, "d_queries": None},
     (L.ERR_UNSUPPORTED, "sharded grouped search takes clamp(top_groups) <= 256 (got 300)")),
    ({"offsets": None}, (L.ERR_NULL, "NULL argument")),
    ({"modes": [0, 5]}, (L.ERR_ARGUMENT, "filter mode must be 0 (allow-list) or 1 (deny-list)")),
    ({"offsets": [0, 3, 2]}, (L.ERR_ARGUMENT, "filter_offsets decrease at filter 1")),
    ({"ids": None}, (L.ERR_NULL, "frame_ids is NULL")),
    ({"where": None}, (L.ERR_NULL, "NULL argument")),
    ({"qw": [0, 9, NF]}, (L.ERR_ARGUMENT, "query 1 names where 9 of 2")),
    ({"d_queries": None}, (L.ERR_NULL, "NULL argument")),
    ({"d_out": None}, (L.ERR_NULL, "NULL argument")),
    ({"near": BAD_BOX}, (L.ERR_ARGUMENT, BOX_REASON)),
    ({"near": BAD_BOX, "d_out": None}, (L.ERR_NULL, "NULL argument")),
    ({"near": BAD_BOX, "qw": [0, 9, NF]}, (L.ERR_ARGUMENT, "query 1 names where 9 of 2")),
]

EXPAND_ONLY = [
    ({"d_chosen": None}, (L.ERR_NULL, "NULL argument")),
    ({"d_own_heads": None}, (L.ERR_NULL, "NULL argument")),
    ({"d_chosen": None, "near": BAD_BOX}, (L.ERR_ARGUMENT, BOX_REASON)),           # the clauses first
    ({"d_chosen": None, "top_k": 300, "per_group": 1},
     (L.ERR_UNSUPPORTED, "sharded grouped search takes clamp(top_groups) <= 256 (got 300)")),
]


def _device_call(name, h, fault, dev):
    """One call of a device form, with real device buffers wherever a pointer is valid, so no call can touch memory it
    does not own even if a check were missing."""
    a = {**BASE, "engine": True, "d_queries": True, "d_out": True, "d_chosen": True, "d_own_heads": True, "terms_list": True,
         **fault}
    eng = h if a["engine"] else None
    dq = C.c_void_p(dev["queries"].data_ptr()) if a["d_queries"] else None
    filters = (_u64(a["ids"]), _u64(a["offsets"]), _i32(a["modes"]), a["n_filters"], _u32(a["qf"]))
    wheres = (_wheres(a, True), a["n_wheres"], _u32(a["qw"]))
    lib = L.lib()
    if name == "where_device":
        out = C.c_void_p(dev["cands"].data_ptr()) if a["d_out"] else None
        terms = (_u64(a["term_offsets"]), _u64(a["terms"])) if a["terms_list"] else (None, None)
        rc = lib.wax_vs_search_batch_where_device(eng, dq, NQ, a["top_k"], *filters, *wheres, *terms, 0, out, None)
    elif name == "heads":
        out = C.c_void_p(dev["heads"].data_ptr()) if a["d_out"] else None
        rc = lib.wax_vs_shard_grouped_heads_device(eng, dq, NQ, a["top_k"], a["per_group"], *filters, *wheres, 0, out, None)
    else:
        out = C.c_void_p(dev["cands"].data_ptr()) if a["d_out"] else None
        chosen = C.c_void_p(dev["chosen"].data_ptr()) if a["d_chosen"] else None
        own = C.c_void_p(dev["heads"].data_ptr()) if a["d_own_heads"] else None
        rc = lib.wax_vs_shard_grouped_expand_device(eng, dq, NQ, a["top_k"], a["per_group"], *filters, *wheres, chosen,
                                                    own, 0, out, None)
    return rc, L.last_error() if rc else ""


def test_device_forms_pin_their_checks():
    eng = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    slots = NQ * L.MAX_RESULTS
    dev = {"queries": torch.zeros(NQ * DIMS, dtype=torch.float32, device="cuda:0"),
           "cands": torch.zeros(slots * C.sizeof(L.Candidate), dtype=torch.uint8, device="cuda:0"),
           "heads": torch.zeros(slots * 40, dtype=torch.uint8, device="cuda:0"),
           "chosen": torch.zeros(slots * 40, dtype=torch.uint8, device="cuda:0")}
    try:
        for filled in (False, True):
            if filled:
                rng = np.random.default_rng(3)
                eng.add_batch(np.arange(1, ROWS + 1, dtype=np.uint64), rng.standard_normal((ROWS, DIMS)).astype(np.float32))
            for name, table in (("where_device", WHERE_DEVICE), ("heads", GROUPED_DEVICE),
                                ("expand", GROUPED_DEVICE + EXPAND_ONLY)):
                for fault, want in table:
                    assert _device_call(name, eng.handle, fault, dev) == want, (name, filled, fault)
        torch.cuda.synchronize()
    finally:
        eng.close()
