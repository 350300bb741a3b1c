"""GPU: batched search with one filter per query (wax_vs_search_batch_multi_filtered).  Every answer must equal the
single-query filtered search under that query's filter (the plain search when unfiltered): same ids, same order, same
score bits; some answers are checked against the oracle run on the allowed subset directly."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_filtered import _expect
from wax_b200 import CUDAVectorEngine, InvalidToc, VectorMetric
from wax_b200 import _lib as L

pytestmark = pytest.mark.gpu

N, DIMS = 80_000, 384


def _engine(oracle, metric, seed, batch_l2=0):
    corpus = oracle.synth_rows(seed, 0, N, DIMS, normalize=(metric is not VectorMetric.dot))
    ids = np.arange(N, dtype=np.uint64) * 3 + 77                        # frameIds distinct from rows
    eng = CUDAVectorEngine(metric, DIMS)
    eng.add_batch(ids, corpus)
    if batch_l2:
        eng.set_option("batch_l2", 1)
    return eng, corpus, ids


def _single(eng, q, k, flt):
    if flt is None:
        return eng.search(q, k)
    kind, fids = flt
    return eng.search_filtered(q, k, **{kind: fids})


def _bits(hits):
    return [(i, np.float32(s).view(np.uint32).item()) for i, s in hits]


def _same(got, want):
    assert _bits(got) == _bits(want)


def _filters(rng, ids):
    """The filter kinds of the issue: gather, two tensor-class, per-query scan, empty, unknown ids only."""
    small = rng.choice(N, 700, replace=False)
    large = rng.choice(N, 40_000, replace=False)
    deny = rng.choice(N, 50_000, replace=False)
    keep3 = rng.choice(N, 3, replace=False)
    deny_all_but_3 = np.setdiff1d(np.arange(N), keep3)
    filters = [("allow", np.concatenate([ids[small], ids[small[:25]], np.array([5, 2**60], np.uint64)])),   # gather
               ("allow", ids[large]),                                                                      # tensor
               ("deny", ids[deny]),                                                                        # tensor
               ("deny", ids[deny_all_but_3]),                                                              # scan
               ("allow", np.zeros(0, np.uint64)),                                                          # empty
               ("allow", np.array([1, 2, 2**62], np.uint64))]                                              # unknown only
    allowed = [set(small.tolist()), set(large.tolist()), set(range(N)) - set(deny.tolist()), set(keep3.tolist()), set(), set()]
    return filters, allowed


@pytest.mark.parametrize("metric,batch_l2", [(VectorMetric.cosine, 0), (VectorMetric.dot, 0), (VectorMetric.l2, 1),
                                             (VectorMetric.l2, 0)])
def test_each_query_equals_the_single_query_filtered_search(oracle, metric, batch_l2):
    eng, corpus, ids = _engine(oracle, metric, 2100 + metric.value, batch_l2)
    rng = np.random.default_rng(2101 + metric.value + batch_l2)
    filters, allowed = _filters(rng, ids)
    b = 300                                                                # 3 query groups
    qs = oracle.synth_rows(2102 + metric.value, 0, b, DIMS, normalize=True)
    choice = rng.integers(-1, len(filters), b)
    choice[:len(filters) + 1] = np.arange(-1, len(filters))               # every kind at least once
    query_filter = [None if c < 0 else int(c) for c in choice]
    n_tensor = sum(1 for f in query_filter if f in (1, 2) or f is None)
    for k in (10, 72, 200):
        t0, f0 = eng.batch_stats()
        got = eng.search_batch_multi_filtered(qs, k, filters, query_filter)
        t1, f1 = eng.batch_stats()
        assert len(got) == b
        for qi, f in enumerate(query_filter):
            _same(got[qi], _single(eng, qs[qi], k, None if f is None else filters[f]))
        for f in range(len(filters)):                                      # the first query of each filter vs the oracle
            qi = query_filter.index(f)
            assert got[qi] == _expect(oracle, metric, corpus, ids, allowed[f], qs[qi], k), (f, k)
        assert all(got[qi] == [] for qi, f in enumerate(query_filter) if f in (4, 5))
        assert all(len(got[qi]) == 3 for qi, f in enumerate(query_filter) if f == 3)
        if metric is not VectorMetric.l2 or batch_l2:
            assert (t1 - t0) + (f1 - f0) == n_tensor, "the tensor-class queries must take the tensor-core levels"
            assert f1 - f0 <= 5, f"{f1 - f0} of {n_tensor} tensor-class queries fell back to the exact scan"


def test_filters_are_not_mixed_between_queries(oracle):
    """256 identical queries, each under its own filter allowing a disjoint set of rows: half as allow-lists (gather
    class), half as deny-lists of everything else (tensor class).  A wrong index into the bitsets or the spans returns
    rows of another query's set."""
    eng, corpus, ids = _engine(oracle, VectorMetric.cosine, 2200)
    rng = np.random.default_rng(2201)
    b = 256
    sets = np.array_split(rng.permutation(N), b)                           # 312 or 313 rows each
    everything = np.arange(N)
    filters = []
    for i, rows in enumerate(sets):
        if i % 2 == 0:
            filters.append(("allow", ids[rows]))
        else:
            filters.append(("deny", ids[np.setdiff1d(everything, rows)]))
    q = oracle.synth_row(2202, 0, DIMS, True)
    qs = np.repeat(q[None, :], b, axis=0)
    t0, f0 = eng.batch_stats()
    got = eng.search_batch_multi_filtered(qs, 10, filters, list(range(b)))
    t1, f1 = eng.batch_stats()
    assert (t1 - t0) + (f1 - f0) == b // 2
    for i, rows in enumerate(sets):
        own = set(ids[rows].tolist())
        assert len(got[i]) == 10 and all(fid in own for fid, _ in got[i]), i
    for i in range(0, b, 17):
        _same(got[i], _single(eng, q, 10, filters[i]))
    assert got[1] == _expect(oracle, VectorMetric.cosine, corpus, ids, set(sets[1].tolist()), q, 10)


def test_large_k_over_several_launches(oracle):
    """k = 1000: a launch holds fewer queries than the batch, so the per-launch filter indices and the filter-level
    compaction of the unproven queries run over several chunks."""
    eng, corpus, ids = _engine(oracle, VectorMetric.cosine, 2300)
    rng = np.random.default_rng(2301)
    filters = [("deny", ids[rng.choice(N, 20_000, replace=False)]), ("allow", ids[rng.choice(N, 30_000, replace=False)]),
               ("deny", ids[rng.choice(N, 5_000, replace=False)]), ("allow", ids[rng.choice(N, 60_000, replace=False)])]
    b = 1100
    qs = oracle.synth_rows(2302, 0, b, DIMS, normalize=True)
    query_filter = [None if c == len(filters) else int(c) for c in rng.integers(0, len(filters) + 1, b)]
    t0, f0 = eng.batch_stats()
    got = eng.search_batch_multi_filtered(qs, 1000, filters, query_filter)
    t1, f1 = eng.batch_stats()
    assert (t1 - t0) + (f1 - f0) == b
    for qi in list(range(0, b, 9)) + list(range(b - 40, b)):
        f = query_filter[qi]
        _same(got[qi], _single(eng, qs[qi], 1000, None if f is None else filters[f]))


def test_bitset_budget_splits_the_tensor_class(oracle):
    eng, corpus, ids = _engine(oracle, VectorMetric.dot, 2400)
    rng = np.random.default_rng(2401)
    filters = [("deny" if i % 2 else "allow", ids[rng.choice(N, 30_000, replace=False)]) for i in range(7)]
    b = 200
    qs = oracle.synth_rows(2402, 0, b, DIMS, normalize=True)
    query_filter = [None if c == 7 else int(c) for c in rng.integers(0, 8, b)]
    p0 = eng.counter("filter_bitset_passes")
    whole = eng.search_batch_multi_filtered(qs, 24, filters, query_filter)
    p1 = eng.counter("filter_bitset_passes")
    words = (N + 31) // 32
    eng.set_option("filter_bitset_bytes", 3 * words * 4)                   # three bitsets per pass
    split = eng.search_batch_multi_filtered(qs, 24, filters, query_filter)
    p2 = eng.counter("filter_bitset_passes")
    assert p1 - p0 == 1 and p2 - p1 == 3
    assert [_bits(h) for h in split] == [_bits(h) for h in whole]
    for qi in range(0, b, 11):
        f = query_filter[qi]
        _same(split[qi], _single(eng, qs[qi], 24, None if f is None else filters[f]))


def test_equivalences_and_argument_checks(oracle):
    eng, corpus, ids = _engine(oracle, VectorMetric.cosine, 2500)
    rng = np.random.default_rng(2501)
    qs = oracle.synth_rows(2502, 0, 40, DIMS, normalize=True)
    for kind, n in (("allow", 700), ("allow", 40_000), ("deny", 50_000)):
        fids = ids[rng.choice(N, n, replace=False)]
        got = eng.search_batch_multi_filtered(qs, 10, [(kind, fids)], [0] * len(qs))
        assert [_bits(h) for h in got] == [_bits(h) for h in eng.search_batch_filtered(qs, 10, **{kind: fids})]
    got = eng.search_batch_multi_filtered(qs, 10, [], [None] * len(qs))
    assert [_bits(h) for h in got] == [_bits(h) for h in eng.search_batch(qs, 10)]
    assert eng.search_batch_multi_filtered([], 10, [("allow", ids[:3])], []) == []
    with pytest.raises(InvalidToc):
        eng.search_batch_multi_filtered(qs[:2], 10, [(2, ids[:3])], [0, 0])                # mode other than 0 / 1
    with pytest.raises(InvalidToc):
        eng.search_batch_multi_filtered(qs[:2], 10, [("allow", ids[:3])], [0, 1])          # index out of range
    with pytest.raises(ValueError):
        eng.search_batch_multi_filtered(qs[:2], 10, [("allow", ids[:3])], [0])             # one index per query

    def raw(engine, offsets, modes, query_filter, fids=ids[:4], n_filters=None, out_stride=10):
        b = len(query_filter)
        q = np.ascontiguousarray(qs[:b])
        off = np.asarray(offsets, np.uint64)
        md = np.asarray(modes, np.int32)
        qf = np.asarray(query_filter, np.uint32)
        out_ids = np.zeros((b, out_stride), np.uint64)
        out_sc = np.zeros((b, out_stride), np.float32)
        ns = np.zeros(b, np.uint32)
        return L.lib().wax_vs_search_batch_multi_filtered(
            engine._h, q.ctypes.data_as(C.POINTER(C.c_float)), b, DIMS, 10,
            None if fids is None else fids.ctypes.data_as(C.POINTER(C.c_uint64)), off.ctypes.data_as(C.POINTER(C.c_uint64)),
            md.ctypes.data_as(C.POINTER(C.c_int32)), len(md) if n_filters is None else n_filters,
            qf.ctypes.data_as(C.POINTER(C.c_uint32)), out_ids.ctypes.data_as(C.POINTER(C.c_uint64)),
            out_sc.ctypes.data_as(C.POINTER(C.c_float)), out_stride, ns.ctypes.data_as(C.POINTER(C.c_uint32)))

    fids = np.ascontiguousarray(ids[:4])
    assert raw(eng, [0, 2, 4], [0, 1], [0, 1], fids) == L.OK
    assert raw(eng, [1, 2, 4], [0, 1], [0, 1], fids) == L.ERR_ARGUMENT               # offsets[0] != 0
    assert raw(eng, [0, 3, 2], [0, 1], [0, 1], fids) == L.ERR_ARGUMENT               # decreasing offsets
    assert raw(eng, [0, 2, 4], [0, 1], [0, 2], fids) == L.ERR_ARGUMENT               # filter index out of range
    assert raw(eng, [0, 2, 4], [0, 1], [0, L.NO_FILTER], fids) == L.OK
    assert raw(eng, [0, 2, 4], [0, 1], [0, 1], None) == L.ERR_NULL                   # ids named but NULL
    assert raw(eng, [0, 0, 0], [0, 1], [0, 1], None) == L.OK                         # no ids: NULL allowed
    assert raw(eng, [0, 2, 4], [0, 1], [1, 1], fids, out_stride=9) == L.ERR_BUFFER    # deny-list allows >= 10 rows
    assert raw(eng, [0, 2, 4], [0, 1], [0, 0], fids, out_stride=2) == L.OK            # two allowed rows: stride 2 will do
    # validation runs before the empty-engine early return
    empty = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    assert raw(empty, [0, 2, 4], [0, 7], [0, 1], fids) == L.ERR_ARGUMENT
    assert raw(empty, [0, 2, 4], [0, 1], [0, 5], fids) == L.ERR_ARGUMENT
    assert raw(empty, [0, 2, 4], [0, 1], [0, 1], fids) == L.OK
