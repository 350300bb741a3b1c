"""GPU: batched grouped search with a where and an id filter of each query's own
(wax_vs_search_batch_grouped_multi_where).  Every answer must equal wax_vs_search_grouped for that query alone under an
allow-list of exactly the frames passing its where (time, tag and location clauses, PhotoRAG's bins rebuilt here) and
its id filter: frame ids, group ids, order and score bits.  A subset is checked against the grouped oracle as well, and
the routing (coverage level, expansion passes, crowded queries) through the counters."""
import ctypes as C

import numpy as np
import pytest

from oracle import grouped as og
from test_gpu_where import DELETED, LABEL, SUPERSEDED, _attributes
from test_gpu_where_near import REGION, PhotoIndex, _allowed, _locations
from wax_b200 import CUDAVectorEngine, VectorMetric, Where, location_box
from wax_b200 import _lib as L

pytestmark = pytest.mark.gpu

N = 80_000
COUNTERS = ("grouped_batch_covered_queries", "grouped_batch_expanded_groups", "grouped_batch_fallback_queries",
            "grouped_batch_expansion_passes", "filter_bitset_passes")


def flat(res):
    """[(group, [(id, score), ...]), ...] -> [(group, id, score bits), ...]"""
    return [(g, f, int(np.float32(s).view(np.uint32))) for g, hits in res for f, s in hits]


def counters(eng):
    return {c: eng.counter(c) for c in COUNTERS}


def delta(eng, before):
    return {c: eng.counter(c) - v for c, v in before.items()}


class Corpus:
    """80 000 rows in groups of 8, with attributes and clustered locations, and the reference allow-lists."""

    def __init__(self, oracle, metric, dims, seed, batch_l2=0):
        self.metric = metric
        self.corpus = oracle.synth_rows(seed, 0, N, dims, normalize=(metric is not VectorMetric.dot))
        self.ids = np.arange(N, dtype=np.uint64) * 3 + 41
        self.eng = CUDAVectorEngine(metric, dims)
        self.eng.add_batch(self.ids, self.corpus)
        self.eng.set_option("batch_l2", batch_l2)
        self.groups = self.ids[(np.arange(N) // 8) * 8]
        self.eng.set_groups(self.ids, self.groups)
        rng = np.random.default_rng(seed + 1)
        self.ts, self.tags = _attributes(rng, N)
        self.eng.set_attributes(self.ids, self.ts, self.tags)
        self.lat, self.lon, self.centres = _locations(rng, N)
        self.eng.set_locations(self.ids, self.lat, self.lon)
        self.index = PhotoIndex(self.ids, self.lat, self.lon)
        self._rows = {}

    def rows(self, wheres, filters, w, f):
        """The rows query (w, f) may return."""
        key = (id(wheres), id(filters), w, f)
        if key not in self._rows:
            self._rows[key] = _allowed(None if w is None else wheres[w], None if f is None else filters[f], self.ids,
                                       self.ts, self.tags, self.index)
        return self._rows[key]

    def single(self, q, top, per, wheres, filters, w, f):
        """wax_vs_search_grouped under the allow-list of the passing frames."""
        if w is None and f is None:
            return self.eng.search_grouped(q, top, per)
        rows = self.rows(wheres, filters, w, f)
        return self.eng.search_grouped(q, top, per, allow=self.ids[rows]) if rows.size else []


def wheres_of(c):
    ts = c.ts
    mid = ((REGION[0] + REGION[1]) / 2, (REGION[2] + REGION[3]) / 2)
    k = c.centres[5]
    return [Where(after=int(ts[N // 10]), before=int(ts[N // 10 + N // 2]), no_tags=DELETED),     # 0 wide window
            Where(after=int(ts[1000]), before=int(ts[4000])),                                      # 1 narrow: listed
            Where(near=(mid[0], mid[1], 100_000.0)),                                               # 2 wide box
            Where(near=(k[0], k[1], 1000.0)),                                                      # 3 narrow box
            Where(near=(0.5, 179.995, 20_000.0), all_tags=LABEL),                                  # 4 the antimeridian
            Where(after=int(ts[N // 10]), before=int(ts[N // 10 + N // 2]), no_tags=DELETED | SUPERSEDED,
                  near=(k[0], k[1], 25_000.0)),                                                    # 5 box AND window
            Where(after=10, before=5),                                                             # 6 admits nothing
            Where(near=(-60.0, -60.0, 25_000.0)),                                                  # 7 an empty box
            Where(no_tags=DELETED, near=(0.0, 0.0, 0.0))]                                          # 8 no location clause


def filters_of(c, wheres, rng):
    deny = set(c.ids[rng.choice(N, 3000, replace=False)].tolist())
    for w in wheres:                                   # some denied rows inside every where: a bitset, not a listing
        rows = _allowed(w, None, c.ids, c.ts, c.tags, c.index)
        deny |= set(c.ids[rows[:5]].tolist())
    return [("allow", c.ids[rng.choice(N, 5000, replace=False)]),          # 0 small: the gather class
            ("allow", c.ids[rng.choice(N, 30_000, replace=False)]),        # 1 large
            ("deny", np.fromiter(deny, np.uint64, len(deny))),              # 2
            ("deny", c.ids[np.arange(N) >= 100])]                           # 3 leaves 100 rows, fewer than k_c


# (where, filter) pairs by the class of the batched filtered search they fall in
TENSOR = [(None, None), (0, None), (2, None), (8, None), (None, 1), (None, 2), (5, 2), (4, 2), (0, 2), (8, 1)]
GATHER = [(None, 0), (1, None), (3, None), (5, None), (4, None), (3, 0), (0, 0), (6, None), (7, None), (6, 1)]
MIXED = TENSOR + GATHER + [(None, 3), (1, 3), (6, 2)]


def run(c, qs, top, per, wheres, filters, pairs, rng):
    qw = [pairs[i % len(pairs)][0] for i in range(len(qs))]
    qf = [pairs[i % len(pairs)][1] for i in range(len(qs))]
    perm = rng.permutation(len(qs))
    qw, qf = [qw[i] for i in perm], [qf[i] for i in perm]
    got = c.eng.search_batch_grouped_multi_where(qs, top, per, wheres, qw, filters, qf)
    assert len(got) == len(qs)
    return got, qw, qf


def check_single(c, qs, top, per, wheres, filters, got, qw, qf, which=None):
    for i in (range(len(qs)) if which is None else which):
        want = c.single(qs[i], top, per, wheres, filters, qw[i], qf[i])
        assert flat(got[i]) == flat(want), (i, qw[i], qf[i], top, per)


@pytest.mark.parametrize("metric,batch_l2", [(VectorMetric.cosine, 0), (VectorMetric.dot, 0), (VectorMetric.l2, 0),
                                             (VectorMetric.l2, 1)])
@pytest.mark.parametrize("dims", [384, 100])                      # 100: dims % 32 != 0, tensor batches go crowded
def test_each_answer_equals_its_single_grouped_search(oracle, metric, batch_l2, dims):
    c = Corpus(oracle, metric, dims, 7100 + dims + metric.value, batch_l2)
    rng = np.random.default_rng(7101 + dims + 10 * metric.value + batch_l2)
    wheres = wheres_of(c)
    filters = filters_of(c, wheres, rng)
    sizes = [c.rows(wheres, filters, w, None).size for w in range(len(wheres))]
    assert sizes[0] > 16384 and 128 < sizes[1] <= 16384 and sizes[2] > 16384 and 0 < sizes[3] <= 16384
    assert 0 < sizes[4] <= 16384 and 128 < sizes[5] <= 16384 and sizes[6] == 0 and sizes[7] == 0
    assert c.rows(wheres, filters, None, 3).size == 100
    qs = oracle.synth_rows(7200 + dims, 0, 64, dims, True)
    tensor_route = dims % 32 == 0 and (metric is not VectorMetric.l2 or batch_l2)
    for per in (1, 3):
        for name, pairs in (("tensor", TENSOR), ("gather", GATHER), ("mixed", MIXED)):
            before = counters(c.eng)
            got, qw, qf = run(c, qs, 12, per, wheres, filters, pairs, rng)
            check_single(c, qs, 12, per, wheres, filters, got, qw, qf)
            d = delta(c.eng, before)
            staged = sum(c.rows(wheres, filters, w, f).size > 0 for w, f in zip(qw, qf))
            assert d["grouped_batch_covered_queries"] + d["grouped_batch_fallback_queries"] == staged
            if name == "mixed" or (name == "tensor" and not tensor_route):
                assert d["grouped_batch_covered_queries"] == 0, name
            else:
                assert d["grouped_batch_covered_queries"] > 0, name
    c.eng.close()


def test_a_subset_against_the_grouped_oracle(oracle):
    c = Corpus(oracle, VectorMetric.cosine, 384, 7300)
    rng = np.random.default_rng(7301)
    wheres = wheres_of(c)
    filters = filters_of(c, wheres, rng)
    qs = oracle.synth_rows(7302, 0, 48, 384, True)
    for pairs in (TENSOR, GATHER):
        got, qw, qf = run(c, qs, 7, 3, wheres, filters, pairs, rng)
        for i in rng.choice(len(qs), 10, replace=False):
            allowed = np.zeros(N, bool)
            allowed[c.rows(wheres, filters, qw[i], qf[i])] = True
            r, _, s, g = og.search_grouped(VectorMetric.cosine.value, c.corpus, qs[i], c.groups, 7, 3, allowed=allowed,
                                           mode=oracle.ACC_F32_TREE, threads=8)
            want = [(int(gg), int(c.ids[int(rr)]), int(ss)) for rr, ss, gg in zip(r, s.view(np.uint32), g)]
            assert flat(got[i]) == want, (i, qw[i], qf[i])
    c.eng.close()


def test_expansions_split_over_the_bitset_budget(oracle):
    c = Corpus(oracle, VectorMetric.cosine, 384, 7400)
    rng = np.random.default_rng(7401)
    starts = rng.integers(0, N // 2, 40)
    wheres = [Where(after=int(c.ts[s]), before=int(c.ts[s + N // 3]), no_tags=DELETED) for s in starts]
    deny = [("deny", c.ids[rng.choice(N, 2000, replace=False)])]
    qs = oracle.synth_rows(7402, 0, 80, 384, True)
    qw = [i % 40 for i in range(80)]
    qf = [None if i % 3 else 0 for i in range(80)]                  # 40 wheres x (none, deny): more than 40 pairs
    want = c.eng.search_batch_grouped_multi_where(qs, 12, 3, wheres, qw, deny, qf)
    words = (N + 31) // 32
    c.eng.set_option("filter_bitset_bytes", 2 * words * 4)          # two bitsets per pass
    before = counters(c.eng)
    got = c.eng.search_batch_grouped_multi_where(qs, 12, 3, wheres, qw, deny, qf)
    d = delta(c.eng, before)
    assert d["filter_bitset_passes"] > 1 and d["grouped_batch_expansion_passes"] > 1, d
    assert d["grouped_batch_covered_queries"] > 0 and d["grouped_batch_expanded_groups"] > 0, d
    assert [flat(x) for x in got] == [flat(x) for x in want]
    check_single(c, qs, 12, 3, wheres, deny, got, qw, qf, rng.choice(80, 24, replace=False))
    c.eng.close()


def test_crowded_queries_take_the_single_query_pipeline(oracle):
    c = Corpus(oracle, VectorMetric.cosine, 384, 7500)
    rng = np.random.default_rng(7501)
    groups = c.groups.copy()
    groups[: 19_800] = 1                                           # 99 % of the rows of window 0 in one group
    c.eng.set_groups(c.ids, groups)
    wheres = [Where(after=int(c.ts[0]), before=int(c.ts[20_000])),
              Where(after=int(c.ts[30_000]), before=int(c.ts[70_000]), no_tags=DELETED)]
    filters = [("deny", c.ids[rng.choice(N, 1000, replace=False)])]
    qs = oracle.synth_rows(7502, 0, 64, 384, True)
    qw = [i % 2 for i in range(64)]
    qf = [None if i % 4 < 2 else 0 for i in range(64)]
    before = counters(c.eng)
    got = c.eng.search_batch_grouped_multi_where(qs, 12, 2, wheres, qw, filters, qf)
    d = delta(c.eng, before)
    assert d["grouped_batch_fallback_queries"] > 0 and d["grouped_batch_covered_queries"] > 0, d
    check_single(c, qs, 12, 2, wheres, filters, got, qw, qf)
    c.eng.close()


def test_one_pair_for_every_query_is_the_one_where_search(oracle):
    c = Corpus(oracle, VectorMetric.cosine, 384, 7600)
    rng = np.random.default_rng(7601)
    wheres = wheres_of(c)
    filters = filters_of(c, wheres, rng)
    qs = oracle.synth_rows(7602, 0, 48, 384, True)
    for w in (0, 1, 2, 3, 5, 8):
        for f in (None, 0, 1, 2):
            kw = {} if f is None else {filters[f][0]: filters[f][1]}
            got = c.eng.search_batch_grouped_multi_where(qs, 12, 3, [wheres[w]], [0] * 48, filters,
                                                         [f] * 48)
            want = c.eng.search_batch_grouped_where(qs, 12, 3, wheres[w], **kw)
            assert [flat(x) for x in got] == [flat(x) for x in want], (w, f)
            if wheres[w].near is None:                             # ... and the where_near entry point
                near = Where(after=wheres[w].after, before=wheres[w].before, all_tags=wheres[w].all_tags,
                             no_tags=wheres[w].no_tags, near=(0.0, 0.0, 0.0))
                want = c.eng.search_batch_grouped_where(qs, 12, 3, near, **kw)
                assert [flat(x) for x in got] == [flat(x) for x in want], (w, f, "near")
    c.eng.close()


def _raw(eng, qs, top=5, per=2, fids=None, offsets=None, modes=None, n_filters=None, qf=None, wheres=None,
         n_wheres=None, qw=None, ids=True, scores=True, groups=True, stride=None, ns=True):
    """One direct C call with valid defaults (no filter, one where named by every query); an argument given as
    "null" is passed as NULL."""
    b = qs.shape[0]
    cap = max(1, min(L.MAX_RESULTS, top * per)) if stride is None else stride
    a = {}
    a["fids"] = np.zeros(1, np.uint64) if fids is None else fids
    a["offsets"] = np.zeros(1, np.uint64) if offsets is None else offsets
    a["modes"] = np.zeros(1, np.int32) if modes is None else modes
    a["qf"] = np.full(b, L.NO_FILTER, np.uint32) if qf is None else qf
    a["qw"] = np.zeros(b, np.uint32) if qw is None else qw
    w = (L.WhereNear * 1)(Where().to_c_near()) if wheres is None else wheres
    outs = (np.empty((max(b, 1), cap), np.uint64), np.empty((max(b, 1), cap), np.float32),
            np.empty((max(b, 1), cap), np.uint64), np.zeros(max(b, 1), np.uint32))
    ptr = lambda x, t: None if isinstance(x, str) else x.ctypes.data_as(C.POINTER(t))
    return L.lib().wax_vs_search_batch_grouped_multi_where(
        eng.handle, qs.ctypes.data_as(C.POINTER(C.c_float)), b, qs.shape[1], top, per, ptr(a["fids"], C.c_uint64),
        ptr(a["offsets"], C.c_uint64), ptr(a["modes"], C.c_int32), 0 if n_filters is None else n_filters,
        ptr(a["qf"], C.c_uint32), None if isinstance(w, str) else C.cast(w, C.c_void_p),
        1 if n_wheres is None else n_wheres, ptr(a["qw"], C.c_uint32),
        ptr(outs[0], C.c_uint64) if ids is True else None, ptr(outs[1], C.c_float) if scores is True else None,
        ptr(outs[2], C.c_uint64) if groups is True else None, cap, ptr(outs[3], C.c_uint32) if ns is True else None)


def test_edge_cases_and_argument_checks(oracle):
    dims = 64
    empty = CUDAVectorEngine(VectorMetric.cosine, dims)
    qs = np.asarray(np.random.default_rng(7700).standard_normal((3, dims)), np.float32)
    assert empty.search_batch_grouped_multi_where(qs, 5, 2, [Where()], [0, None, 0]) == [[], [], []]
    assert empty.search_batch_grouped_multi_where(qs[:0], 5, 2, [Where()], []) == []
    # every check runs before the empty-engine early return
    assert _raw(empty, qs) == L.OK
    assert _raw(empty, qs, per=0) == L.ERR_ARGUMENT
    assert _raw(empty, qs, per=129) == L.ERR_ARGUMENT
    assert _raw(empty, qs, top=200, per=128) == L.ERR_ARGUMENT               # 200 x 128 > 10 000
    assert _raw(empty, qs, groups=None) == L.ERR_NULL
    assert _raw(empty, qs, ns=None) == L.ERR_NULL
    assert _raw(empty, qs, qw=np.array([0, 1, 0], np.uint32)) == L.ERR_ARGUMENT   # where 1 of 1
    assert _raw(empty, qs, qf=np.array([0, L.NO_FILTER, 0], np.uint32)) == L.ERR_ARGUMENT   # filter 0 of 0
    assert _raw(empty, qs, offsets=np.array([0, 2], np.uint64), modes=np.array([2], np.int32),
                n_filters=1, qf=np.zeros(3, np.uint32)) == L.ERR_ARGUMENT    # mode 2
    assert _raw(empty, qs, offsets=np.array([1, 2], np.uint64), modes=np.zeros(1, np.int32),
                n_filters=1) == L.ERR_ARGUMENT                                # offsets start at 1
    assert _raw(empty, qs, offsets=np.array([0, 2], np.uint64), modes=np.zeros(1, np.int32), n_filters=1,
                fids="null") == L.ERR_NULL
    assert _raw(empty, qs, wheres="null") == L.ERR_NULL
    assert _raw(empty, qs, qw="null") == L.ERR_NULL
    assert _raw(empty, qs, offsets="null") == L.ERR_NULL
    bad_box = (L.WhereNear * 1)(Where(near=(0.0, 0.0, float("inf"))).to_c_near())
    assert _raw(empty, qs, wheres=bad_box) == L.ERR_ARGUMENT
    with pytest.raises(ValueError):
        empty.search_batch_grouped_multi_where(qs, 5, 2, [Where(terms=(1,))], [0, 0, 0])
    empty.close()

    rng = np.random.default_rng(7701)
    n = 4000
    eng = CUDAVectorEngine(VectorMetric.cosine, dims)
    corpus = np.asarray(rng.standard_normal((n, dims)), np.float32)
    ids = np.arange(n, dtype=np.uint64) + 100
    eng.add_batch(ids, corpus)
    eng.set_groups(ids, ids // 4)
    assert _raw(eng, qs, stride=9) == L.ERR_BUFFER                          # 5 x 2 entries
    assert _raw(eng, qs[:0]) == L.OK
    ts = np.arange(n, dtype=np.int64)
    eng.set_attributes(ids, ts, np.zeros(n, np.uint64))
    w = [Where(after=100, before=2100), Where(after=0, before=4000, near=(41.0, 11.0, 5000.0))]

    def check(wheres, qw):
        got = eng.search_batch_grouped_multi_where(qs, 5, 2, wheres, qw)
        for i in range(len(qs)):
            rows = [r for r in range(n) if wheres[qw[i]].passes(int(ts[r]), int(tags[r]), loc[r])]
            want = eng.search_grouped(qs[i], 5, 2, allow=ids[rows]) if rows else []
            assert got[i] == want, i
        single = eng.search_batch_grouped_multi_where(qs[:1], 5, 2, wheres, qw[:1])   # a batch of one
        assert single[0] == got[0]

    tags = np.zeros(n, np.uint64)
    loc = [None] * n
    check(w, [0, 1, 0])
    ts = ts[::-1].copy()                                                   # the next call sees new attributes
    tags[::3] = DELETED
    eng.set_attributes(ids, ts, tags)
    w[0] = Where(after=100, before=2100, no_tags=DELETED)
    check(w, [0, 1, 1])
    lat = 41.0 + 0.02 * rng.standard_normal(n)                             # ... new locations
    lon = 11.0 + 0.02 * rng.standard_normal(n)
    lat[n // 2:] = 10.0
    eng.set_locations(ids, lat, lon)
    loc = [(int(np.floor(a * 100.0)), int(np.floor(b * 100.0))) for a, b in zip(lat, lon)]
    check(w, [1, 0, 1])
    gone = rng.choice(n, 1000, replace=False)                              # ... and rows removed
    eng.remove_batch(ids[gone])
    keep = np.setdiff1d(np.arange(n), gone)
    ids, ts, tags, corpus = ids[keep], ts[keep], tags[keep], corpus[keep]
    loc = [loc[r] for r in keep]
    n = keep.size
    check(w, [1, 0, 1])
    eng.close()


def test_full_size_photo_batch():
    rng = np.random.default_rng(7800)
    n, dims, b = 10_000_000, 384, 1024
    eng = CUDAVectorEngine(VectorMetric.cosine, dims)
    eng.fill_synthetic(7801, n)
    ids = np.arange(n, dtype=np.uint64)
    eng.set_groups(ids, ids // 360)
    ts = np.arange(n, dtype=np.int64)
    tags = np.where(rng.random(n) < 0.01, DELETED, 0).astype(np.uint64)
    eng.set_attributes(ids, ts, tags)
    n_c = 300
    lat_c, lon_c = rng.uniform(-60, 60, n_c), rng.uniform(-170, 170, n_c)
    c = rng.integers(0, n_c, n)
    lat = lat_c[c] + 0.18 * rng.standard_normal(n)
    lon = lon_c[c] + 0.18 * rng.standard_normal(n) / np.cos(np.radians(lat_c[c]))
    none = rng.random(n) >= 0.7
    lat[none] = lon[none] = np.nan
    eng.set_locations(ids, lat, lon)
    lat_bin, lon_bin = np.floor(lat * 100.0), np.floor(lon * 100.0)
    qs = np.asarray(rng.standard_normal((b, dims)), np.float32)
    wheres = []
    for _ in range(b):
        a = int(rng.integers(0, n - n // 5))
        ci = int(rng.integers(0, n_c))
        wheres.append(Where(after=a, before=a + n // 5, no_tags=DELETED, near=(float(lat_c[ci]), float(lon_c[ci]), 25_000.0)))
    got = eng.search_batch_grouped_multi_where(qs, 12, 1, wheres, list(range(b)))
    for qi in rng.choice(b, 32, replace=False):
        w = wheres[qi]
        la, lb, lo, hi = location_box(*w.near)
        assert lo <= hi
        ok = (lat_bin >= la) & (lat_bin <= lb) & (lon_bin >= lo) & (lon_bin <= hi)
        ok &= (ts >= w.after) & (ts < w.before) & ((tags & np.uint64(DELETED)) == 0)
        want = eng.search_grouped(qs[qi], 12, 1, allow=ids[ok])
        assert flat(got[qi]) == flat(want), qi
    eng.close()
