"""GPU: term clauses below the top-k (wax_vs_search_batch_where_terms), Wax's metadataFilter as required term ids.  The
reference allow-list is computed here in numpy -- the frames whose term set holds every required id AND pass the time,
tag and location clauses AND the id filter -- and every answer must be identical (ids, order, score bits) to the
id-filtered search under it."""
import threading

import numpy as np
import pytest

from test_gpu_filtered import _expect
from test_gpu_where import DELETED, SUPERSEDED, _attributes, _bits
from test_gpu_where_near import REGION, PhotoIndex, _allowed, _locations
from wax_b200 import CUDAVectorEngine, TermDictionary, VectorMetric, Where

pytestmark = pytest.mark.gpu

N, DIMS = 80_000, 384
COMMON, RARE, NOBODY = 1, 2, 3            # held by ~80 % of rows, ~2 %, none
KIND = 10                                 # KIND + k, k < 4
SESSION = 1000                            # SESSION + s


def _terms(rng, n, n_sessions=40):
    """Seeded term sets: a session (sizes skewed), a kind, COMMON on 80 %, RARE on 2 %; 5 % of rows get no terms."""
    p = rng.pareto(1.2, n_sessions) + 0.05
    session = rng.choice(n_sessions, n, p=p / p.sum())
    kind = rng.integers(0, 4, n)
    common = rng.random(n) < 0.8
    rare = rng.random(n) < 0.02
    bare = rng.random(n) < 0.05
    lists = []
    for r in range(n):
        if bare[r]:
            lists.append([])
            continue
        t = [SESSION + int(session[r]), KIND + int(kind[r])]
        if common[r]:
            t.append(COMMON)
        if rare[r]:
            t += [RARE, RARE]                                                      # duplicates are kept once
        lists.append(t)
    return lists


def _has(lists, terms):
    """Rows whose set holds every id of `terms`."""
    req = set(terms)
    return np.fromiter((req <= set(t) for t in lists), bool, len(lists))


def _allowed_terms(where, flt, ids, ts, tags, index, lists):
    rows = _allowed(where, flt, ids, ts, tags, index)
    if where is not None and where.terms:
        rows = rows[_has(lists, where.terms)[rows]]
    return rows


def _expected(eng, qs, k, wheres, query_where, filters, query_filter, ids, ts, tags, index, lists):
    out, qf = [], []
    for qi in range(len(qs)):
        w, f = query_where[qi], query_filter[qi]
        if w is None:
            if f is None:
                qf.append(None)
                continue
            out.append(filters[f])
        else:
            out.append(("allow", ids[_allowed_terms(wheres[w], None if f is None else filters[f], ids, ts, tags, index,
                                                    lists)]))
        qf.append(len(out) - 1)
    return eng.search_batch_multi_filtered(qs, k, out, qf)


def _engine(oracle, metric, seed, batch_l2=0):
    corpus = oracle.synth_rows(seed, 0, N, DIMS, normalize=(metric is not VectorMetric.dot))
    ids = np.arange(N, dtype=np.uint64) * 3 + 77
    eng = CUDAVectorEngine(metric, DIMS)
    eng.add_batch(ids, corpus)
    if batch_l2:
        eng.set_option("batch_l2", 1)
    rng = np.random.default_rng(seed + 1)
    ts, tags = _attributes(rng, N)
    eng.set_attributes(ids, ts, tags)
    lat, lon, _ = _locations(rng, N)
    eng.set_locations(ids, lat, lon)
    lists = _terms(rng, N)
    assert eng.set_terms(ids, lists) == N
    return eng, corpus, ids, ts, tags, PhotoIndex(ids, lat, lon), lists


def _wheres(ts, lists):
    counts = {}
    for t in lists:
        for x in t:
            counts[x] = counts.get(x, 0) + 1
    big = max((x for x in counts if x >= SESSION), key=counts.get)             # the largest session
    mid = ((REGION[0] + REGION[1]) / 2, (REGION[2] + REGION[3]) / 2)
    window = dict(after=int(ts[N // 10]), before=int(ts[N // 10 + N // 5]))
    return [Where(terms=(COMMON, RARE)),                                          # 0 common first, rare second: gather
            Where(terms=(COMMON,)),                                               # 1 > 16 384 rows: tensor
            Where(terms=(NOBODY,)),                                               # 2 a term nobody holds: empty
            Where(terms=(KIND, KIND, COMMON), no_tags=DELETED, **window),         # 3 duplicates AND window AND tags
            Where(terms=(big,), near=(mid[0], mid[1], 100_000.0)),        # 4 a session AND a box
            Where(terms=(COMMON, KIND + 1, RARE, big)),                       # 5 four terms
            Where(terms=(COMMON, KIND + 2), near=(mid[0], mid[1], 100_000.0),
                  no_tags=SUPERSEDED),                                            # 6 terms AND box AND tags
            Where(terms=(RARE, NOBODY)),                                          # 7 a held term and a missing one
            Where(no_tags=DELETED)]                                               # 8 no term clause


@pytest.mark.parametrize("metric,batch_l2", [(VectorMetric.cosine, 0), (VectorMetric.dot, 0), (VectorMetric.l2, 1),
                                             (VectorMetric.l2, 0)])
def test_each_answer_equals_multi_filtered_with_the_numpy_allow_list(oracle, metric, batch_l2):
    eng, corpus, ids, ts, tags, index, lists = _engine(oracle, metric, 6100 + metric.value, batch_l2)
    rng = np.random.default_rng(6101 + metric.value + batch_l2)
    wheres = _wheres(ts, lists)
    sizes = [_allowed_terms(w, None, ids, ts, tags, index, lists).size for w in wheres]
    assert 0 < sizes[0] <= 16384 and sizes[1] > 16384 and sizes[2] == 0 and sizes[3] > 0 and sizes[4] > 0
    assert sizes[5] > 0 and sizes[6] > 0 and sizes[7] == 0
    filters = [("allow", ids[rng.choice(N, 30_000, replace=False)]),                   # allow-list AND terms: host
               ("deny", ids[rng.choice(N, 20_000, replace=False)]),                    # deny-list AND terms: device
               ("allow", ids[rng.choice(N, 700, replace=False)])]
    combos = [(w, f) for w in [None] + list(range(len(wheres))) for f in [None] + list(range(len(filters)))]
    builds = eng.counter("term_index_builds")
    for b in (1, 3, 64):
        order = rng.permutation(len(combos))
        picks = [combos[i] for i in order[:b]] if b < len(combos) else \
            combos + [combos[i] for i in rng.integers(0, len(combos), b - len(combos))]
        qs = oracle.synth_rows(6102 + metric.value + b, 0, b, DIMS, normalize=True)
        query_where = [w for w, _ in picks]
        query_filter = [f for _, f in picks]
        for k in (1, 10, 72, 200):
            got = eng.search_batch_where(qs, k, wheres, query_where, filters, query_filter)
            want = _expected(eng, qs, k, wheres, query_where, filters, query_filter, ids, ts, tags, index, lists)
            assert len(got) == b
            for qi in range(b):
                assert _bits(got[qi]) == _bits(want[qi]), (b, k, picks[qi])
    assert eng.counter("term_index_builds") == builds + 1                          # built once, reused
    assert eng.counter("term_index_bytes") > 0
    qs = oracle.synth_rows(6199 + metric.value, 0, len(combos), DIMS, normalize=True)
    got = eng.search_batch_where(qs, 10, wheres, [w for w, _ in combos], filters, [f for _, f in combos])
    want = _expected(eng, qs, 10, wheres, [w for w, _ in combos], filters, [f for _, f in combos], ids, ts, tags, index,
                     lists)
    for qi, (w, f) in enumerate(combos):
        assert _bits(got[qi]) == _bits(want[qi]), (w, f)
        if f is None and w in (0, 3, 5, 6):                                          # and the oracle, for a few
            rows = _allowed_terms(wheres[w], None, ids, ts, tags, index, lists)
            assert got[qi] == _expect(oracle, metric, corpus, ids, list(rows), qs[qi], 10)


def test_batch_of_1024_and_many_units_over_three_bitsets():
    rng = np.random.default_rng(6300)
    eng = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    eng.fill_synthetic(6301, N, id_base=1000)
    ids = np.arange(N, dtype=np.uint64) + 1000
    ts, tags = _attributes(rng, N)
    eng.set_attributes(ids, ts, tags)
    lists = _terms(rng, N)
    eng.set_terms(ids, lists)
    index = PhotoIndex(ids, np.full(N, np.nan), np.full(N, np.nan))
    words = (N + 31) // 32
    eng.set_option("filter_bitset_bytes", 3 * words * 4)
    wheres = [Where(terms=(COMMON, KIND + k), no_tags=DELETED) for k in range(4)]             # wide units
    wheres += [Where(terms=(SESSION + s,)) for s in range(40)]                                  # sessions of all sizes
    wheres += [Where(terms=(COMMON,)), Where(terms=(RARE, COMMON)), Where(no_tags=DELETED)]
    filters = [("deny", ids[rng.choice(N, 500 * (j + 1), replace=False)]) for j in range(5)]    # five deny-lists
    filters.append(("allow", ids[rng.choice(N, 20_000, replace=False)]))
    b = 1024
    qs = np.asarray(rng.standard_normal((b, DIMS)), np.float32)
    query_where = [None if c < 0 else int(c) for c in rng.integers(-1, len(wheres), b)]
    query_filter = [None if c < 0 else int(c) for c in rng.integers(-1, len(filters), b)]
    passes0 = eng.counter("filter_bitset_passes")
    got = eng.search_batch_where(qs, 10, wheres, query_where, filters, query_filter)
    assert eng.counter("filter_bitset_passes") - passes0 >= 4                      # > 3 wide units: several sub-batches
    want = _expected(eng, qs, 10, wheres, query_where, filters, query_filter, ids, ts, tags, index, lists)
    for qi in range(b):
        assert _bits(got[qi]) == _bits(want[qi]), qi


def test_single_query_takes_the_shadow_route_under_the_term_bitset(oracle):
    n = 200_000
    rng = np.random.default_rng(6402)
    eng = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    eng.fill_synthetic(6400, n, id_base=3)
    ids = np.arange(n, dtype=np.uint64) + 3
    ts, tags = _attributes(rng, n)
    eng.set_attributes(ids, ts, tags)
    lists = _terms(rng, n)
    eng.set_terms(ids, lists)
    index = PhotoIndex(ids, np.full(n, np.nan), np.full(n, np.nan))
    eng.set_option("shadow_scan_min_bytes", 0)
    wheres = [Where(terms=(COMMON,)), Where(terms=(COMMON, KIND), after=int(ts[n // 10]), no_tags=DELETED)]
    q = oracle.synth_rows(6401, 0, 1, DIMS, normalize=True)
    routed = lambda: (eng.counter("single_shadow_queries"), eng.counter("single_shadow_fallbacks"))
    for w in range(len(wheres)):
        assert _allowed_terms(wheres[w], None, ids, ts, tags, index, lists).size > 16384   # a bitset, not a gather
        before = routed()
        got = eng.search_where(q[0], 10, wheres[w])
        assert routed() == (before[0] + 1, before[1])
        eng.set_option("shadow_scan", 0)
        fp32 = eng.search_where(q[0], 10, wheres[w])
        eng.set_option("shadow_scan", 1)
        assert _bits(got) == _bits(fp32)
        assert _bits(got) == _bits(_expected(eng, q, 10, wheres, [w], [], [None], ids, ts, tags, index, lists)[0])


def test_terms_follow_their_rows():
    rng = np.random.default_rng(6600)
    dims = 64
    eng = CUDAVectorEngine(VectorMetric.cosine, dims)
    model = {}                                                                     # frame id -> term set
    vec = lambda m: np.asarray(rng.standard_normal((m, dims)), np.float32)
    ids = np.arange(100, 2100, dtype=np.uint64)
    eng.add_batch(ids, vec(ids.size))
    for i in ids:
        model[int(i)] = set()
    clauses = [Where(terms=(5,)), Where(terms=(5, 6)), Where(terms=(7,), no_tags=2), Where(terms=(99,))]
    tag_of = {}

    def check():
        for w in clauses:
            want = sorted(f for f, t in model.items() if w.passes(0, tag_of.get(f, 0), None, t))
            got = eng.search_where(rng.standard_normal(dims), 10_000, w)
            assert sorted(i for i, _ in got) == want, w

    builds = eng.counter("term_index_builds")
    check()                                                                        # no terms: nothing passes
    assert eng.counter("term_index_builds") == builds + 1
    check()
    assert eng.counter("term_index_builds") == builds + 1                         # once per invalidation
    lists = [list(rng.choice([5, 6, 7, 8], rng.integers(0, 4))) for _ in ids]
    assert eng.set_terms(np.concatenate([ids, [1, 2]]), lists + [[5], [6]]) == ids.size   # unknown ids ignored
    for i, t in zip(ids, lists):
        model[int(i)] = set(int(x) for x in t)
    check()
    assert eng.counter("term_index_builds") == builds + 2
    eng.set_terms(ids[10:12].repeat(2), [[5], [7], [5, 6], [6]])                   # a later entry wins
    model[int(ids[10])], model[int(ids[11])] = {5, 6}, {6}
    eng.set_terms(ids[20:30], [[]] * 10)                                           # an empty list clears
    for i in ids[20:30]:
        model[int(i)] = set()
    for _ in range(6):                                                             # rewrites: the pool is compacted
        eng.set_terms(ids[:500], [[5, 6, 7]] * 500)
    for i in ids[:500]:
        model[int(i)] = {5, 6, 7}
    check()
    eng.add(int(ids[40]), vec(1)[0])                                               # upsert keeps the set
    new = np.arange(5000, 5050, dtype=np.uint64)
    eng.add_batch(new, vec(new.size))                                              # appended frames have none
    for i in new:
        model[int(i)] = set()
    eng.add_batch(np.array([7000, 150, 6000], np.uint64), vec(3))                  # out of order: upsert + appends
    model[7000] = model[6000] = set()
    check()
    eng.set_attributes(ids[:300], tags=np.full(300, 2, np.uint64))                 # the tag clause beside the terms
    tag_of = {int(i): 2 for i in ids[:300]}
    check()
    b0 = eng.counter("term_index_builds")
    eng.remove(int(ids[3]))
    del model[int(ids[3])]
    check()
    gone = ids[rng.choice(ids.size, 300, replace=False)]
    eng.remove_batch(gone)
    for i in gone:
        model.pop(int(i), None)
    check()
    assert eng.counter("term_index_builds") == b0 + 2                          # one build per invalidation
    eng.deserialize(eng.serialize())                                               # MV2V carries no terms: reset
    model = {f: set() for f in model}
    tag_of = {}
    check()
    eng.set_terms(np.array(sorted(model), np.uint64), [[5, 6]] * len(model))
    eng.fill_synthetic(6601, 500, id_base=10)                                      # reset too
    model = {10 + r: set() for r in range(500)}
    check()
    eng.set_terms(np.arange(10, 510, dtype=np.uint64), [[5]] * 250 + [[6, 5]] * 250)
    model = {10 + r: ({5} if r < 250 else {5, 6}) for r in range(500)}
    check()


def test_a_search_concurrent_with_set_terms_sees_old_or_new():
    rng = np.random.default_rng(6700)
    eng = CUDAVectorEngine(VectorMetric.cosine, 128)
    n = 20_000
    eng.fill_synthetic(6701, n)
    ids = np.arange(n, dtype=np.uint64)
    lists_a = [[5] if i % 2 == 0 else [] for i in range(n)]
    lists_b = [[5, 6] if i % 3 == 0 else [6] for i in range(n)]
    eng.set_terms(ids, lists_a)
    w = Where(terms=(5,))
    sets = [set(ids[::2].tolist()), set(ids[::3].tolist())]
    stop = threading.Event()
    seen, errors = [], []

    def reader():
        q = np.asarray(rng.standard_normal(128), np.float32)
        while not stop.is_set():
            try:
                seen.append({i for i, _ in eng.search_where(q, 10_000, w)})
            except Exception as exc:                                               # surfaced below
                errors.append(exc)
                return

    t = threading.Thread(target=reader)
    t.start()
    for i in range(20):
        eng.set_terms(ids, lists_b if i % 2 == 0 else lists_a)
    stop.set()
    t.join()
    assert not errors
    assert seen
    for got in seen:
        assert got == sets[0] or got == sets[1]


def test_ties_and_non_finite_rows(oracle):
    rng = np.random.default_rng(6800)
    n, dims = 20_000, 128
    corpus = oracle.synth_rows(6801, 0, n, dims, normalize=True)
    corpus[100:140] = corpus[99]                                                   # exact ties
    corpus[200] = np.nan
    corpus[201] = np.inf
    ids = np.arange(n, dtype=np.uint64) + 5
    eng = CUDAVectorEngine(VectorMetric.cosine, dims)
    eng.add_batch(ids, corpus)
    ts, tags = _attributes(rng, n)
    eng.set_attributes(ids, ts, tags)
    lists = [[5, 6] if r < 1000 else ([6] if r % 7 else []) for r in range(n)]
    eng.set_terms(ids, lists)
    index = PhotoIndex(ids, np.full(n, np.nan), np.full(n, np.nan))
    wheres = [Where(terms=(5,)), Where(terms=(6, 5), before=int(ts[5000])), Where(terms=(6,), no_tags=DELETED)]
    qs = np.stack([corpus[99], corpus[150], corpus[0]])
    for k in (1, 10, 72):
        for wi in range(len(wheres)):
            got = eng.search_batch_where(qs, k, wheres, [wi] * 3)
            want = _expected(eng, qs, k, wheres, [wi] * 3, [], [None] * 3, ids, ts, tags, index, lists)
            for qi in range(3):
                assert _bits(got[qi]) == _bits(want[qi])


def test_metadata_filter_through_the_dictionary(oracle):
    rng = np.random.default_rng(6850)
    n, dims = 5000, 64
    eng = CUDAVectorEngine(VectorMetric.cosine, dims)
    eng.fill_synthetic(6851, n)
    ids = np.arange(n, dtype=np.uint64)
    d = TermDictionary()
    sessions = [f"s{int(x)}" for x in rng.integers(0, 20, n)]
    metas = [None if r % 11 == 0 else {"session_id": sessions[r]} for r in range(n)]
    labels = [["pinned"] if r % 5 == 0 else [] for r in range(n)]
    eng.set_terms(ids, [d.frame_terms(metas[r], [("kind", "note")], labels[r]) for r in range(n)])
    q = np.asarray(rng.standard_normal(dims), np.float32)
    for flt, keep in [(({"session_id": "s3"},), lambda r: metas[r] is not None and metas[r]["session_id"] == "s3"),
                      (({"session_id": "s3"}, [("kind", "note")], ["pinned"]),
                       lambda r: metas[r] is not None and metas[r]["session_id"] == "s3" and r % 5 == 0),
                      (({}, [("kind", "other")]), lambda r: False),
                      (({},), lambda r: True)]:
        got = eng.search_where(q, 10_000, Where(terms=d.filter_terms(*flt)))
        assert sorted(i for i, _ in got) == [r for r in range(n) if keep(r)], flt


def test_full_size_session_workload():
    rng = np.random.default_rng(6900)
    n, dims = 10_000_000, 384
    eng = CUDAVectorEngine(VectorMetric.cosine, dims)
    eng.fill_synthetic(6901, n)
    ids = np.arange(n, dtype=np.uint64)
    tags = np.where(rng.random(n) < 0.01, DELETED, 0).astype(np.uint64)
    eng.set_attributes(ids, tags=tags)
    sizes = rng.integers(100, 20_000, 1500)
    session = np.repeat(np.arange(sizes.size), sizes)[:n]
    session = np.concatenate([session, np.full(n - session.size, sizes.size)])     # the rest: one big session
    session = session[rng.permutation(n)]
    eng.set_terms(ids, [[SESSION + int(s)] for s in session])
    b = 1024
    qs = np.asarray(rng.standard_normal((b, dims)), np.float32)
    pick = rng.integers(0, sizes.size, b)
    wheres = [Where(terms=(SESSION + int(s),), no_tags=DELETED) for s in pick]
    got = eng.search_batch_where(qs, 10, wheres, list(range(b)))
    for qi in rng.choice(b, 12, replace=False):
        ok = (session == pick[qi]) & ((tags & np.uint64(DELETED)) == 0)
        want = eng.search_batch_multi_filtered(qs[qi:qi + 1], 10, [("allow", ids[ok])], [0])[0]
        assert _bits(got[qi]) == _bits(want), qi


def test_many_wide_units_under_a_reduced_budget():
    """Hundreds of distinct wide units, with and without deny-lists, under a budget of three bitsets: each wide unit gets
    its bits set inside the sub-batch split, nothing lists its rows."""
    rng = np.random.default_rng(6950)
    eng = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    eng.fill_synthetic(6951, N, id_base=500)
    ids = np.arange(N, dtype=np.uint64) + 500
    ts, tags = _attributes(rng, N)
    eng.set_attributes(ids, ts, tags)
    lists = _terms(rng, N)
    eng.set_terms(ids, lists)
    index = PhotoIndex(ids, np.full(N, np.nan), np.full(N, np.nan))
    eng.set_option("filter_bitset_bytes", 3 * ((N + 31) // 32) * 4)
    wheres = []
    for j in range(200):                                   # half the corpus's timestamps: > 16 384 rows each
        a = int(rng.integers(0, N // 2))
        wheres.append(Where(terms=(COMMON,), after=int(ts[a]), before=int(ts[a + N // 2 - 1]) + j % 2))
    filters = [("deny", ids[rng.choice(N, 2000 * (j + 1), replace=False)]) for j in range(4)]
    b = 1024
    qs = np.asarray(rng.standard_normal((b, DIMS)), np.float32)
    query_where = [int(x) for x in rng.integers(0, len(wheres), b)]
    query_filter = [None if c < 0 else int(c) for c in rng.integers(-1, len(filters), b)]
    sizes = {_allowed_terms(wheres[w], None, ids, ts, tags, index, lists).size for w in set(query_where)}
    assert min(sizes) > 16384
    passes0 = eng.counter("filter_bitset_passes")
    got = eng.search_batch_where(qs, 10, wheres, query_where, filters, query_filter)
    assert eng.counter("filter_bitset_passes") - passes0 >= 200 // 3
    want = _expected(eng, qs, 10, wheres, query_where, filters, query_filter, ids, ts, tags, index, lists)
    for qi in range(b):
        assert _bits(got[qi]) == _bits(want[qi]), qi


def test_equal_wheres_are_one_unit():
    """1 024 where objects naming 16 sessions plan 16 units: the same sub-batches and answers as the 16 wheres."""
    rng = np.random.default_rng(6960)
    eng = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    eng.fill_synthetic(6961, N)
    ids = np.arange(N, dtype=np.uint64)
    ts, tags = _attributes(rng, N)
    eng.set_attributes(ids, ts, tags)
    lists = _terms(rng, N, n_sessions=16)
    eng.set_terms(ids, lists)
    index = PhotoIndex(ids, np.full(N, np.nan), np.full(N, np.nan))
    distinct = [Where(terms=(SESSION + s, COMMON), no_tags=DELETED) for s in range(16)]
    b = 1024
    pick = [int(x) for x in rng.integers(0, 16, b)]
    each = [Where(terms=(COMMON, SESSION + s, COMMON), no_tags=DELETED) for s in pick]   # equal after sort and dedup
    qs = np.asarray(rng.standard_normal((b, DIMS)), np.float32)
    p0 = eng.counter("filter_bitset_passes")
    got16 = eng.search_batch_where(qs, 10, distinct, pick)
    p1 = eng.counter("filter_bitset_passes")
    got = eng.search_batch_where(qs, 10, each, list(range(b)))
    p2 = eng.counter("filter_bitset_passes")
    assert p2 - p1 == p1 - p0
    want = _expected(eng, qs, 10, distinct, pick, [], [None] * b, ids, ts, tags, index, lists)
    for qi in range(b):
        assert _bits(got[qi]) == _bits(want[qi]) == _bits(got16[qi]), qi


def test_a_reset_releases_the_index():
    eng = CUDAVectorEngine(VectorMetric.cosine, 64)
    eng.fill_synthetic(6970, 10_000)
    eng.set_terms(np.arange(10_000, dtype=np.uint64), [[5, 6]] * 10_000)
    eng.search_where(np.ones(64, np.float32), 10, Where(terms=(5,)))
    assert eng.counter("term_index_bytes") >= 20_000 * 4
    eng.fill_synthetic(6971, 10_000)
    assert eng.counter("term_index_bytes") == 0
    eng.set_terms(np.arange(10_000, dtype=np.uint64), [[5]] * 10_000)
    eng.search_where(np.ones(64, np.float32), 10, Where(terms=(5,)))
    eng.deserialize(eng.serialize())
    assert eng.counter("term_index_bytes") == 0
    assert eng.search_where(np.ones(64, np.float32), 10, Where(terms=(5,))) == []
