"""GPU: frame-attribute predicates below the top-k (wax_vs_search_batch_where, wax_vs_search_batch_grouped_where).
Every answer must be identical -- ids, order, score bits -- to the id-filtered search under an allow-list of exactly the
frames that pass, computed here with numpy; some answers are also checked against the oracle on the passing subset."""
import threading

import numpy as np
import pytest

from test_gpu_filtered import _expect
from wax_b200 import CUDAVectorEngine, VectorMetric, Where

pytestmark = pytest.mark.gpu

N, DIMS = 80_000, 384
DELETED, SUPERSEDED, LABEL = 1 << 0, 1 << 1, 1 << 5


def _bits(hits):
    return [(i, np.float32(s).view(np.uint32).item()) for i, s in hits]


def _attributes(rng, n):
    ts = np.arange(n, dtype=np.int64) * 10 + rng.integers(0, 10, n)          # increasing with the row, seeded jitter
    tags = np.zeros(n, np.uint64)
    tags[rng.choice(n, n // 100, replace=False)] |= DELETED
    tags[rng.choice(n, n // 20, replace=False)] |= SUPERSEDED
    tags[rng.random(n) < 0.5] |= LABEL
    return ts, tags


def _engine(oracle, metric, seed, batch_l2=0):
    corpus = oracle.synth_rows(seed, 0, N, DIMS, normalize=(metric is not VectorMetric.dot))
    ids = np.arange(N, dtype=np.uint64) * 3 + 77
    eng = CUDAVectorEngine(metric, DIMS)
    eng.add_batch(ids, corpus)
    if batch_l2:
        eng.set_option("batch_l2", 1)
    rng = np.random.default_rng(seed + 1)
    ts, tags = _attributes(rng, N)
    assert eng.set_attributes(ids, ts, tags) == N
    return eng, corpus, ids, ts, tags


def _passing(where, ts, tags):
    ok = (ts >= where.after) & ((ts < where.before) | (where.before == np.iinfo(np.int64).max))
    ok &= (tags & np.uint64(where.all_tags)) == np.uint64(where.all_tags)
    ok &= (tags & np.uint64(where.no_tags)) == 0
    return ok


def _allowed_rows(where, flt, ids, ts, tags):
    ok = np.ones(ids.size, bool) if where is None else _passing(where, ts, tags)
    if flt is not None:
        kind, fids = flt
        listed = np.isin(ids, np.asarray(fids, np.uint64))
        ok &= listed if kind == "allow" else ~listed
    return np.flatnonzero(ok)


def _expected(eng, qs, k, wheres, query_where, filters, query_filter, ids, ts, tags):
    """multi_filtered with an allow-list of exactly the passing frames (the plain filter / none when no where)."""
    lists, qf = [], []
    for qi in range(len(qs)):
        w, f = query_where[qi], query_filter[qi]
        if w is None:
            if f is None:
                qf.append(None)
                continue
            lists.append(filters[f])
        else:
            rows = _allowed_rows(wheres[w], None if f is None else filters[f], ids, ts, tags)
            lists.append(("allow", ids[rows]))
        qf.append(len(lists) - 1)
    return eng.search_batch_multi_filtered(qs, k, lists, qf)


def _windows(ts, rng, frac, count):
    """`count` random time windows covering about `frac` of the rows."""
    out = []
    n = ts.size
    for _ in range(count):
        a = int(rng.integers(0, n - int(frac * n)))
        b = a + max(int(frac * n), 1)
        out.append(Where(after=int(ts[a]), before=int(ts[min(b, n - 1)])))
    return out


def _wheres(ts):
    return [Where(after=int(ts[N // 10]), before=int(ts[N // 10 + N // 5])),            # 0 wide window: tensor class
            Where(after=int(ts[5000]), before=int(ts[5600])),                           # 1 narrow window: gather
            Where(after=int(ts[777]), before=int(ts[780])),                             # 2 three rows: scan class
            Where(after=100, before=100),                                               # 3 empty
            Where(no_tags=DELETED | SUPERSEDED),                                        # 4 no window, status flags
            Where(after=int(ts[N // 4]), before=int(ts[3 * N // 4]), all_tags=LABEL),   # 5 label + window
            Where(all_tags=DELETED, no_tags=DELETED)]                                   # 6 overlapping masks: nothing


@pytest.mark.parametrize("metric,batch_l2", [(VectorMetric.cosine, 0), (VectorMetric.dot, 0), (VectorMetric.l2, 1),
                                             (VectorMetric.l2, 0)])
def test_each_answer_equals_multi_filtered_with_the_passing_allow_list(oracle, metric, batch_l2):
    eng, corpus, ids, ts, tags = _engine(oracle, metric, 4100 + metric.value, batch_l2)
    rng = np.random.default_rng(4101 + metric.value + batch_l2)
    wheres = _wheres(ts)
    filters = [("allow", ids[rng.choice(N, 30_000, replace=False)]),                   # allow-list AND where
               ("deny", ids[rng.choice(N, 20_000, replace=False)]),                    # deny-list AND where
               ("allow", ids[rng.choice(N, 700, replace=False)]),                      # small allow-list
               ("deny", ids[5000:5100])]                                               # deny inside the narrow window
    combos = [(w, f) for w in [None] + list(range(len(wheres))) for f in [None] + list(range(len(filters)))]
    for b in (1, 3, 64):
        order = rng.permutation(len(combos))
        picks = [combos[i] for i in order[:b]] if b < len(combos) else \
            combos + [combos[i] for i in rng.integers(0, len(combos), b - len(combos))]
        qs = oracle.synth_rows(4102 + metric.value + b, 0, b, DIMS, normalize=True)
        query_where = [w for w, _ in picks]
        query_filter = [f for _, f in picks]
        for k in (1, 10, 72, 200):
            got = eng.search_batch_where(qs, k, wheres, query_where, filters, query_filter)
            want = _expected(eng, qs, k, wheres, query_where, filters, query_filter, ids, ts, tags)
            assert len(got) == b
            for qi in range(b):
                assert _bits(got[qi]) == _bits(want[qi]), (b, k, picks[qi])
    # every combination in one batch, and the oracle on the passing subset for a few
    qs = oracle.synth_rows(4199 + metric.value, 0, len(combos), DIMS, normalize=True)
    got = eng.search_batch_where(qs, 10, wheres, [w for w, _ in combos], filters, [f for _, f in combos])
    want = _expected(eng, qs, 10, wheres, [w for w, _ in combos], filters, [f for _, f in combos], ids, ts, tags)
    for qi, (w, f) in enumerate(combos):
        assert _bits(got[qi]) == _bits(want[qi]), (w, f)
        if f is None and w in (0, 1, 2, 3, 4):
            rows = _allowed_rows(wheres[w], None, ids, ts, tags)
            assert got[qi] == _expect(oracle, metric, corpus, ids, list(rows), qs[qi], 10)


def test_batch_of_1024_and_many_pairs_over_three_bitsets():
    rng = np.random.default_rng(4300)
    eng = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    eng.fill_synthetic(4301, N, id_base=1000)
    ids = np.arange(N, dtype=np.uint64) + 1000
    ts, tags = _attributes(rng, N)
    eng.set_attributes(ids, ts, tags)
    words = (N + 31) // 32
    eng.set_option("filter_bitset_bytes", 3 * words * 4)
    wheres = _windows(ts, rng, 0.2, 10) + _windows(ts, rng, 0.005, 6) + [Where(no_tags=DELETED)]
    filters = [("deny", ids[rng.choice(N, 5000, replace=False)])]
    b = 1024
    qs = np.asarray(rng.standard_normal((b, DIMS)), np.float32)
    query_where = [None if c < 0 else int(c) for c in rng.integers(-1, len(wheres), b)]
    query_filter = [None if c < 0 else int(c) for c in rng.integers(-1, len(filters), b)]
    passes0 = eng.counter("filter_bitset_passes")
    got = eng.search_batch_where(qs, 10, wheres, query_where, filters, query_filter)
    assert eng.counter("filter_bitset_passes") - passes0 >= 4                      # > 3 wide pairs: several sub-batches
    want = _expected(eng, qs, 10, wheres, query_where, filters, query_filter, ids, ts, tags)
    for qi in range(b):
        assert _bits(got[qi]) == _bits(want[qi]), qi
    single = eng.search_where(qs[0], 10, wheres[0], deny=filters[0][1])          # the batch of one
    assert _bits(single) == _bits(_expected(eng, qs[:1], 10, wheres, [0], filters, [0], ids, ts, tags)[0])


def test_single_query_takes_the_shadow_route_under_the_where_bitset(oracle):
    n = 200_000                                          # large enough for the unrolled TMA shape the route needs
    eng = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    eng.fill_synthetic(4400, n, id_base=3)
    ids = np.arange(n, dtype=np.uint64) + 3
    ts, tags = _attributes(np.random.default_rng(4402), n)
    eng.set_attributes(ids, ts, tags)
    eng.set_option("shadow_scan_min_bytes", 0)                                      # this corpus takes the route
    wheres = [Where(after=int(ts[n // 10]), before=int(ts[n // 10 + n // 5])), Where(no_tags=DELETED | SUPERSEDED),
              Where(after=int(ts[n // 4]), before=int(ts[3 * n // 4]), all_tags=LABEL)]
    q = oracle.synth_rows(4401, 0, 1, DIMS, normalize=True)
    routed = lambda: (eng.counter("single_shadow_queries"), eng.counter("single_shadow_fallbacks"))
    for w in range(len(wheres)):
        before = routed()
        got = eng.search_where(q[0], 10, wheres[w])
        after = routed()
        assert after == (before[0] + 1, before[1]), (w, before, after)             # the route answered, proof held
        eng.set_option("shadow_scan", 0)
        fp32 = eng.search_where(q[0], 10, wheres[w])
        eng.set_option("shadow_scan", 1)
        assert _bits(got) == _bits(fp32)
        assert _bits(got) == _bits(_expected(eng, q, 10, wheres, [w], [], [None], ids, ts, tags)[0])


def _grouped_engine(oracle, seed):
    rng = np.random.default_rng(seed)
    corpus = oracle.synth_rows(seed, 0, N, DIMS, normalize=True)
    base = corpus[0].copy()
    crowd = base + 0.02 * rng.standard_normal((4000, DIMS)).astype(np.float32)   # rows 0..3999: one crowded group
    corpus[:4000] = crowd / np.linalg.norm(crowd, axis=1, keepdims=True)
    ids = np.arange(N, dtype=np.uint64) * 2 + 9
    eng = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    eng.add_batch(ids, corpus)
    groups = np.where(np.arange(N) < 4000, 1, 1000 + np.arange(N) // 5).astype(np.uint64)
    eng.set_groups(ids, groups)
    ts, tags = _attributes(rng, N)
    eng.set_attributes(ids, ts, tags)
    return eng, corpus, ids, ts, tags


def test_grouped_where_equals_grouped_search_under_the_passing_allow_list(oracle):
    eng, corpus, ids, ts, tags = _grouped_engine(oracle, 4500)
    rng = np.random.default_rng(4501)
    wheres = [Where(no_tags=DELETED), Where(after=int(ts[0]), before=int(ts[N // 2]), no_tags=SUPERSEDED),
              Where(after=int(ts[3000]), before=int(ts[3300])), Where(after=5, before=5)]
    deny = ids[rng.choice(N, 3000, replace=False)]
    allow = ids[rng.choice(N, 40_000, replace=False)]
    for n in (1, 64, 1024):
        qs = np.asarray(rng.standard_normal((n, DIMS)), np.float32)
        qs[0] = corpus[1]                                                        # a crowded query
        for w, flt in ((0, None), (1, ("deny", deny)), (1, ("allow", allow)), (2, None), (3, None)):
            kw = {} if flt is None else {flt[0]: flt[1]}
            got = eng.search_batch_grouped_where(qs, 5, 3, wheres[w], **kw)
            rows = _allowed_rows(wheres[w], flt, ids, ts, tags)
            check = range(n) if n <= 64 else rng.choice(n, 32, replace=False)
            for qi in check:
                want = eng.search_grouped(qs[qi], 5, 3, allow=ids[rows]) if rows.size else []
                assert got[qi] == want, (n, w, flt and flt[0], qi)
    assert eng.counter("grouped_batch_expanded_groups") > 0
    assert eng.counter("grouped_batch_fallback_queries") > 0


def test_attributes_follow_their_rows():
    rng = np.random.default_rng(4600)
    dims = 64
    eng = CUDAVectorEngine(VectorMetric.cosine, dims)
    model = {}                                                                     # frame id -> (ts, tags)
    vec = lambda m: np.asarray(rng.standard_normal((m, dims)), np.float32)
    ids = np.arange(100, 2100, dtype=np.uint64)
    eng.add_batch(ids, vec(ids.size))
    for i in ids:
        model[int(i)] = (0, 0)

    def check():
        for w in (Where(after=1, before=500), Where(all_tags=2), Where(no_tags=2), Where(before=1)):
            want = sorted(f for f, (t, g) in model.items() if w.passes(t, g))
            got = eng.search_where(rng.standard_normal(dims), 10_000, w)
            assert sorted(i for i, _ in got) == want, w

    uploads = eng.counter("attribute_uploads")
    check()
    assert eng.counter("attribute_uploads") == uploads + 1
    check()
    assert eng.counter("attribute_uploads") == uploads + 1                        # once per invalidation, not per search
    ts = rng.integers(0, 1000, ids.size)
    tg = rng.integers(0, 4, ids.size).astype(np.uint64)
    assert eng.set_attributes(np.concatenate([ids, [1, 2]]), np.concatenate([ts, [5, 5]]),
                              np.concatenate([tg, [1, 1]])) == ids.size           # unknown ids ignored
    for i, t, g in zip(ids, ts, tg):
        model[int(i)] = (int(t), int(g))
    check()
    assert eng.counter("attribute_uploads") == uploads + 2
    eng.set_attributes(ids[:10], tags=np.full(10, 2, np.uint64))                  # NULL timestamps: kept
    eng.set_attributes(ids[10:20], timestamps=np.full(10, 7))                     # NULL tags: kept
    eng.set_attributes(ids[20:22].repeat(2), np.array([1, 2, 3, 4]))              # a later entry wins
    for i in ids[:10]:
        model[int(i)] = (model[int(i)][0], 2)
    for i in ids[10:20]:
        model[int(i)] = (7, model[int(i)][1])
    model[int(ids[20])] = (2, model[int(ids[20])][1])
    model[int(ids[21])] = (4, model[int(ids[21])][1])
    check()
    eng.add(int(ids[5]), vec(1)[0])                                                # upsert keeps the attributes
    new = np.arange(5000, 5050, dtype=np.uint64)
    eng.add_batch(new, vec(new.size))                                              # appended frames get the defaults
    for i in new:
        model[int(i)] = (0, 0)
    eng.add_batch(np.array([7000, 150, 6000], np.uint64), vec(3))                  # out of order: upsert + appends
    model[7000] = model[6000] = (0, 0)
    check()
    eng.remove(int(ids[3]))
    del model[int(ids[3])]
    gone = ids[rng.choice(ids.size, 300, replace=False)]
    eng.remove_batch(gone)
    for i in gone:
        model.pop(int(i), None)
    check()
    blob = eng.serialize()
    eng.deserialize(blob)                                                          # MV2V carries no attributes: reset
    model = {f: (0, 0) for f in model}
    check()
    eng.set_attributes(np.array(sorted(model), np.uint64), np.full(len(model), 3))
    eng.fill_synthetic(4601, 500, id_base=10)                                      # reset too
    model = {10 + r: (0, 0) for r in range(500)}
    check()


def test_a_search_concurrent_with_set_attributes_sees_old_or_new():
    rng = np.random.default_rng(4700)
    eng = CUDAVectorEngine(VectorMetric.cosine, 128)
    n = 20_000
    eng.fill_synthetic(4701, n)
    ids = np.arange(n, dtype=np.uint64)
    ts_a = np.where(ids % 2 == 0, 1, 0).astype(np.int64)                           # A: even frames pass
    ts_b = np.where(ids % 3 == 0, 1, 0).astype(np.int64)                           # B: multiples of three pass
    eng.set_attributes(ids, ts_a)
    w = Where(after=1)
    sets = [set(ids[ts_a == 1].tolist()), set(ids[ts_b == 1].tolist())]
    stop = threading.Event()
    seen, errors = [], []

    def reader():
        q = np.asarray(rng.standard_normal(128), np.float32)
        while not stop.is_set():
            try:
                got = {i for i, _ in eng.search_where(q, 10_000, w)}
                seen.append(got)
            except Exception as exc:                                               # surfaced below
                errors.append(exc)
                return

    t = threading.Thread(target=reader)
    t.start()
    for i in range(20):
        eng.set_attributes(ids, ts_b if i % 2 == 0 else ts_a)
    stop.set()
    t.join()
    assert not errors
    assert seen
    for got in seen:                                    # k = 10 000 returns every passing frame: 10 000 or 6 667 of them
        assert got == sets[0] or got == sets[1]


def test_ties_and_non_finite_rows(oracle):
    rng = np.random.default_rng(4800)
    n, dims = 20_000, 128
    corpus = oracle.synth_rows(4801, 0, n, dims, normalize=True)
    corpus[100:140] = corpus[99]                                                   # exact ties
    corpus[200] = np.nan
    corpus[201] = np.inf
    ids = np.arange(n, dtype=np.uint64) + 5
    eng = CUDAVectorEngine(VectorMetric.cosine, dims)
    eng.add_batch(ids, corpus)
    ts, tags = _attributes(rng, n)
    eng.set_attributes(ids, ts, tags)
    wheres = [Where(after=int(ts[90]), before=int(ts[300])), Where(before=int(ts[5000])), Where(no_tags=DELETED)]
    qs = np.stack([corpus[99], corpus[150], corpus[0]])
    for k in (1, 10, 72):
        for wi in range(len(wheres)):
            got = eng.search_batch_where(qs, k, wheres, [wi] * 3)
            want = _expected(eng, qs, k, wheres, [wi] * 3, [], [None] * 3, ids, ts, tags)
            for qi in range(3):
                assert _bits(got[qi]) == _bits(want[qi])


def test_full_size_mixed_wheres():
    rng = np.random.default_rng(4900)
    n, dims = 10_000_000, 384
    eng = CUDAVectorEngine(VectorMetric.cosine, dims)
    eng.fill_synthetic(4901, n)
    ids = np.arange(n, dtype=np.uint64)
    ts, tags = _attributes(rng, n)
    eng.set_attributes(ids, ts, tags)
    wheres = _windows(ts, rng, 0.2, 8) + _windows(ts, rng, 0.0005, 4) + [Where(no_tags=DELETED)]
    b = 1024
    qs = np.asarray(rng.standard_normal((b, dims)), np.float32)
    query_where = [int(w) for w in rng.integers(0, len(wheres), b)]
    got = eng.search_batch_where(qs, 10, wheres, query_where)
    for qi in rng.choice(b, 16, replace=False):
        w = wheres[query_where[qi]]
        rows = _allowed_rows(w, None, ids, ts, tags)
        want = eng.search_batch_multi_filtered(qs[qi:qi + 1], 10, [("allow", ids[rows])], [0])[0]
        assert _bits(got[qi]) == _bits(want), qi
