"""GPU: batched grouped search (wax_vs_search_batch_grouped).  Every query's answer must equal wax_vs_search_grouped for
that query alone -- ids, group ids, order and score bits -- and some are checked against the grouped oracle as well.
The routing (coverage level, expansions, single-query fall-back) is checked through its counters."""
import ctypes as C
import threading

import numpy as np
import pytest

from oracle import grouped as og
from wax_b200 import CUDAVectorEngine, VectorMetric
from wax_b200 import _lib as L

pytestmark = pytest.mark.gpu

COUNTERS = ("grouped_batch_covered_queries", "grouped_batch_expanded_groups", "grouped_batch_fallback_queries")


def flat(res):
    """[(group, [(id, score), ...]), ...] -> [(group, id, score bits), ...]"""
    return [(g, f, int(np.float32(s).view(np.uint32))) for g, hits in res for f, s in hits]


def expect(o, metric, corpus, ids, groups, q, top, per, allowed_rows=None):
    allowed = None
    if allowed_rows is not None:
        allowed = np.zeros(corpus.shape[0], bool)
        allowed[np.asarray(allowed_rows, np.int64)] = True
    r, _, s, g = og.search_grouped(metric.value, corpus, q, groups, top, per, allowed=allowed, mode=o.ACC_F32_TREE,
                                   threads=8)
    return [(int(gg), int(ids[int(rr)]), int(ss)) for rr, ss, gg in zip(r, s.view(np.uint32), g)]


def make_engine(o, metric, n, dims, seed):
    corpus = o.synth_rows(seed, 0, n, dims, normalize=(metric is not VectorMetric.dot))
    ids = np.arange(n, dtype=np.uint64) * 3 + 17
    eng = CUDAVectorEngine(metric, dims)
    eng.add_batch(ids, corpus)
    return eng, corpus, ids


def layouts(n, ids, rng):
    half = ids.copy()
    half[rng.permutation(n)[: n // 2]] = 999_999_999
    return {
        "blocks8": ids[(np.arange(n) // 8) * 8],
        "blocks360": ids[(np.arange(n) // 360) * 360],
        "hashed": (np.arange(n, dtype=np.uint64) * 2654435761) % max(n // 8, 1) + 10**12,
        "half": half,
    }


def counters(eng):
    return np.array([eng.counter(c) for c in COUNTERS], np.int64)


def check_batch(eng, qs, top, per, **flt):
    """The batch against one single call per query; returns the batch's answers."""
    got = eng.search_batch_grouped(qs, top, per_group=per, **flt)
    assert len(got) == len(qs)
    for i, q in enumerate(qs):
        assert flat(got[i]) == flat(eng.search_grouped(q, top, per_group=per, **flt)), (i, top, per, list(flt))
    return got


@pytest.mark.parametrize("metric,batch_l2", [(VectorMetric.cosine, 0), (VectorMetric.dot, 0), (VectorMetric.l2, 0),
                                             (VectorMetric.l2, 1)])
@pytest.mark.parametrize("dims", [384, 768, 100])                  # 100: dims % 32 != 0, the per-query route
def test_batch_grouped_matches_single(oracle, metric, batch_l2, dims):
    n = 70_001                                                        # >= 64 k_c for k_c up to 1 024
    rng = np.random.default_rng(dims + metric.value)
    eng, corpus, ids = make_engine(oracle, metric, n, dims, 4100 + dims)
    eng.set_option("batch_l2", batch_l2)
    qs = oracle.synth_rows(4200 + dims, 0, 64, dims, True)
    tensor_route = dims % 32 == 0 and (metric is not VectorMetric.l2 or batch_l2)
    for name, groups in layouts(n, ids, rng).items():
        eng.set_groups(ids, groups)
        for top, per in ((12, 1), (12, 3), (5, 128), (400, 8), (80, 125)):
            before = counters(eng)
            got = check_batch(eng, qs, top, per)
            d = counters(eng) - before
            assert d[0] + d[2] == len(qs)
            if not tensor_route or top > 256:
                assert d[0] == 0 and d[2] == len(qs), (name, top, per)
            elif name != "blocks360" and top <= 12:
                assert d[0] == len(qs), (name, top, per)             # random queries: the coverage level answers
            if name == "half" and (top, per) == (5, 128) and tensor_route:
                assert d[1] > 0, "the half group is expanded"
        assert flat(got[0]) == expect(oracle, metric, corpus, ids, groups, qs[0], 80, 125), name
    eng.close()


@pytest.mark.parametrize("batch", [1, 3, 64, 1024])
def test_batch_sizes_and_large_kc(oracle, batch):
    n, dims = 80_000, 384
    eng, corpus, ids = make_engine(oracle, VectorMetric.cosine, n, dims, 4300)
    groups = layouts(n, ids, np.random.default_rng(1))["blocks8"]
    eng.set_groups(ids, groups)
    qs = oracle.synth_rows(4301, 0, batch, dims, True)
    for top, per in ((12, 3), (40, 2), (256, 1), (100, 4)):          # k_c = 128, 160, 1 024, 400
        before = counters(eng)
        got = eng.search_batch_grouped(qs, top, per_group=per)
        d = counters(eng) - before
        sample = range(batch) if batch <= 64 else range(0, batch, 37)
        for i in sample:
            assert flat(got[i]) == flat(eng.search_grouped(qs[i], top, per_group=per)), (i, top, per)
        if batch < 4:
            assert d[2] == batch                                      # small batches: the single-query pipeline
        else:
            assert d[0] == batch
    assert flat(got[0]) == expect(oracle, VectorMetric.cosine, corpus, ids, groups, qs[0], 100, 4)
    assert eng.search_batch_grouped(np.zeros((0, dims), np.float32), 5) == []
    eng.close()


def test_crowded_and_uncrowded_mixed(oracle):
    """Two videos of 360 segments each sit next to some queries: their top-128 rows name only 2 groups, so those queries
    run the single-query pipeline; the others are answered by the coverage level."""
    n, dims = 80_000, 384
    corpus = oracle.synth_rows(4400, 0, n, dims, normalize=True)
    q = oracle.synth_row(4401, 0, dims, True)
    rng = np.random.default_rng(17)
    crowd = rng.choice(n, 720, replace=False)
    rows = q[None, :] + rng.standard_normal((720, dims)).astype(np.float32) * 0.01
    corpus[crowd] = rows / np.linalg.norm(rows, axis=1, keepdims=True)
    ids = np.arange(n, dtype=np.uint64) + 1
    groups = ids // 360 * 360 + 10**9
    groups[crowd[:360]] = 1
    groups[crowd[360:]] = 2
    eng = CUDAVectorEngine(VectorMetric.cosine, dims)
    eng.add_batch(ids, corpus)
    eng.set_groups(ids, groups)
    others = oracle.synth_rows(4402, 0, 40, dims, True)
    near = np.stack([q + rng.standard_normal(dims).astype(np.float32) * 1e-4 for _ in range(24)])
    qs = np.concatenate([others[:20], near, others[20:]])
    before = counters(eng)
    got = check_batch(eng, qs, 12, 3)
    d = counters(eng) - before
    assert d[2] == 24 and d[0] == 40
    assert {1, 2} <= {g for g, _ in got[20]} and len(got[20]) == 12
    assert flat(got[20]) == expect(oracle, VectorMetric.cosine, corpus, ids, groups, qs[20], 12, 3)
    eng.close()


def test_half_group_expansion(oracle):
    # one group of half the rows: its best rows beyond the coverage list come from a multi-level expansion
    n, dims = 200_003, 128
    eng, corpus, ids = make_engine(oracle, VectorMetric.cosine, n, dims, 4500)
    groups = layouts(n, ids, np.random.default_rng(9))["half"]
    eng.set_groups(ids, groups)
    qs = oracle.synth_rows(4501, 0, 16, dims, True)
    for top, per in ((5, 128), (78, 128), (3, 100)):
        before = counters(eng)
        got = check_batch(eng, qs, top, per)
        d = counters(eng) - before
        assert d[0] == 16, (top, per)
        if top <= 32:         # k_c = 128 lists about 64 rows of the half group: expanded wherever it is selected
            assert d[1] == sum(any(g == 999_999_999 for g, _ in got[i]) for i in range(16)) > 0, (top, per)
        assert flat(got[3]) == expect(oracle, VectorMetric.cosine, corpus, ids, groups, qs[3], top, per)
    eng.close()


def test_batch_grouped_filters(oracle):
    n, dims = 80_000, 384
    rng = np.random.default_rng(13)
    eng, corpus, ids = make_engine(oracle, VectorMetric.cosine, n, dims, 4600)
    groups = layouts(n, ids, rng)["blocks8"]
    eng.set_groups(ids, groups)
    qs = oracle.synth_rows(4601, 0, 32, dims, True)
    small = np.sort(rng.choice(n, 3_000, replace=False))             # gather class
    large = np.sort(rng.choice(n, 30_000, replace=False))            # tensor class under a bitset
    deny = np.sort(rng.choice(n, 20_000, replace=False))
    few = np.sort(rng.choice(n, 50, replace=False))                  # fewer than k_c rows allowed
    for top, per in ((12, 1), (12, 3), (30, 20)):
        check_batch(eng, qs, top, per, allow=np.concatenate([ids[small], np.uint64([1, 2**62])]))
        got = check_batch(eng, qs, top, per, allow=ids[large])
        assert flat(got[1]) == expect(oracle, VectorMetric.cosine, corpus, ids, groups, qs[1], top, per, large)
        check_batch(eng, qs, top, per, deny=ids[deny])
        got = check_batch(eng, qs, top, per, allow=ids[few])
        assert flat(got[2]) == expect(oracle, VectorMetric.cosine, corpus, ids, groups, qs[2], top, per, few)
        before = counters(eng)
        check_batch(eng, qs, top, per, deny=ids[: n - 40])           # a deny-list leaving fewer than k_c rows
        assert (counters(eng) - before)[2] == len(qs)
        check_batch(eng, qs, top, per, deny=[])
    assert eng.search_batch_grouped(qs, 5, 2, allow=[]) == [[]] * len(qs)
    assert eng.search_batch_grouped(qs, 5, 2, deny=ids) == [[]] * len(qs)
    eng.close()


def test_ties_and_non_finite_rows(oracle):
    n, dims = 60_000, 384
    corpus = oracle.synth_rows(4700, 0, n, dims, normalize=True)
    qs = oracle.synth_rows(4701, 0, 16, dims, True)
    rng = np.random.default_rng(21)
    dup = rng.choice(n, 4_000, replace=False)
    corpus[dup[2_000:]] = corpus[dup[:2_000]]                         # exact ties between rows of different groups
    for i in range(4):                                                # rows tied with each query's best rows
        corpus[dup[2 * i + 10]] = qs[i]
        corpus[dup[2 * i + 11]] = qs[i]
    bad = rng.choice(np.setdiff1d(np.arange(n), dup), 300, replace=False)
    corpus[bad[:100]] = np.nan
    corpus[bad[100:200]] = np.inf
    corpus[bad[200:]] = -np.inf
    ids = np.arange(n, dtype=np.uint64) + 5
    groups = (np.arange(n, dtype=np.uint64) * 2654435761) % 7_000
    eng = CUDAVectorEngine(VectorMetric.cosine, dims)
    eng.add_batch(ids, corpus)
    eng.set_groups(ids, groups)
    for top, per in ((12, 1), (12, 3), (40, 8)):
        got = check_batch(eng, qs, top, per)
        for i in (0, 3):
            assert flat(got[i]) == expect(oracle, VectorMetric.cosine, corpus, ids, groups, qs[i], top, per), (i, top)
    eng.close()


def test_one_index_build_and_concurrent_calls(oracle):
    n, dims = 100_000, 384
    eng, corpus, ids = make_engine(oracle, VectorMetric.cosine, n, dims, 4800)
    eng.set_groups(ids, ids // 24)
    qs = oracle.synth_rows(4801, 0, 32, dims, True)
    before = eng.counter("group_index_builds")
    results, errors = {}, []

    def run(i):
        try:
            if i % 2:
                results[i] = [flat(r) for r in eng.search_batch_grouped(qs, 20, per_group=4)]
            else:
                results[i] = [flat(eng.search_grouped(q, 20, per_group=4)) for q in qs[:4]]
        except Exception as exc:   # surfaced below
            errors.append(exc)

    threads = [threading.Thread(target=run, args=(i,)) for i in range(6)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors
    assert eng.counter("group_index_builds") == before + 1            # batch and single calls share one build
    for i in (1, 3, 5):
        assert results[i] == results[1]
    for i in (0, 2, 4):
        assert results[i] == results[1][:4]
    eng.close()


def test_batch_grouped_argument_checks(oracle):
    dims = 64
    eng = CUDAVectorEngine(VectorMetric.cosine, dims)
    lib, h = L.lib(), eng.handle
    qs = np.ones((2, dims), np.float32)
    ids = np.zeros(64, np.uint64); scores = np.zeros(64, np.float32); grp = np.zeros(64, np.uint64)
    ns = np.full(2, 7, np.uint32)
    f32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    u64 = lambda a: a.ctypes.data_as(C.POINTER(C.c_uint64))
    u32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_uint32))

    def call(top=4, per=2, fids=None, nids=0, mode=1, out_ids=ids, out_scores=scores, out_groups=grp, stride=16,
             qlen=dims, out_n=True, nq=2):
        return lib.wax_vs_search_batch_grouped(h, f32(qs), nq, qlen, top, per, fids, nids, mode,
                                               None if out_ids is None else u64(out_ids),
                                               None if out_scores is None else f32(out_scores),
                                               None if out_groups is None else u64(out_groups), stride,
                                               u32(ns) if out_n else None)

    for engine_state in ("empty", "filled"):                         # checked before the empty-engine return
        assert call(per=0) == L.ERR_ARGUMENT
        assert call(per=129) == L.ERR_ARGUMENT
        assert call(top=5001, per=2) == L.ERR_ARGUMENT
        assert call(top=10**9, per=2) == L.ERR_ARGUMENT
        assert call(mode=2) == L.ERR_ARGUMENT
        assert call(mode=-1) == L.ERR_ARGUMENT
        assert call(out_ids=None) == L.ERR_NULL
        assert call(out_scores=None) == L.ERR_NULL
        assert call(out_groups=None) == L.ERR_NULL
        assert call(out_n=False) == L.ERR_NULL
        assert call(nids=3) == L.ERR_NULL
        if engine_state == "empty":
            assert call(qlen=dims + 1) == L.OK and ns.tolist() == [0, 0]
            ns[:] = 7
            assert call(nq=0) == L.OK
            eng.fill_synthetic(3000, 1000)
    assert call(nq=0) == L.OK
    assert call(qlen=dims + 1) == L.ERR_DIMENSION
    assert call(top=4, per=5, stride=19) == L.ERR_BUFFER
    assert call(top=4, per=4, stride=16) == L.OK and ns.tolist() == [4, 4]
    assert call(top=10_000, per=1, stride=999, nq=1) == L.ERR_BUFFER  # min(10 000, N = 1 000) entries
    eng.close()


@pytest.mark.parametrize("layout", ["blocks8", "hashed"])
def test_batch_grouped_fullsize_10m(oracle, layout):
    rows, dims = 10_000_000, 384
    eng = CUDAVectorEngine(VectorMetric.cosine, dims)
    eng.fill_synthetic(1, rows)
    r = np.arange(rows, dtype=np.uint64)
    groups = r // 8 * 8 if layout == "blocks8" else (r * 2654435761) % (rows // 8)
    eng.set_groups(r, groups)
    qs = oracle.synth_rows(5100, 0, 1024, dims, normalize=True)
    before = counters(eng)
    got = eng.search_batch_grouped(qs, 12, per_group=3)
    assert (counters(eng) - before)[0] == 1024
    for i in range(0, 1024, 8):
        assert flat(got[i]) == flat(eng.search_grouped(qs[i], 12, per_group=3)), i
    eng.close()
