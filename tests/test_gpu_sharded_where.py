"""GPU: where search over the row-sharded engine -- the fused collective (wax_vs_shard_search_where) and the rank-local
device form (wax_vs_search_batch_where_device) merged by wax_vs_merge_candidates_device.  The ranks are engines on one
device driven by one thread each (test_gpu_sharded.Group).  Every sharded answer must be identical (ids, order, score
bits) on every rank to CUDAVectorEngine.search_batch_where on one engine holding the whole corpus."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_sharded import Group
from wax_b200 import CUDAVectorEngine, InvalidToc, VectorMetric, Where, sharded
from wax_b200 import _lib as L

DELETED, SUPERSEDED = 1 << 0, 1 << 1
SESSION, KIND = 1000, 10


def _bits(hits):
    return [(i, np.float32(s).view(np.uint32).item()) for i, s in hits]


def _attributes(rng, n):
    ts = np.arange(n, dtype=np.int64) * 10 + rng.integers(0, 10, n)
    tags = np.zeros(n, np.uint64)
    tags[rng.choice(n, n // 100, replace=False)] |= DELETED
    tags[rng.choice(n, n // 20, replace=False)] |= SUPERSEDED
    return ts, tags


def _locations(rng, n):
    """Clusters around a few centres, 30 % of the rows without a location (NaN)."""
    lat_c, lon_c = rng.uniform(40.0, 42.0, 8), rng.uniform(10.0, 12.5, 8)
    c = rng.integers(0, 8, n)
    lat = lat_c[c] + 0.05 * rng.standard_normal(n)
    lon = lon_c[c] + 0.05 * rng.standard_normal(n)
    none = rng.random(n) >= 0.7
    lat[none] = np.nan
    lon[none] = np.nan
    return lat, lon, (float(lat_c[0]), float(lon_c[0]))


def _terms(rng, n, n_sessions=12):
    session = rng.integers(0, n_sessions, n)
    kind = rng.integers(0, 4, n)
    return [[] if rng.random() < 0.05 else [SESSION + int(session[r]), KIND + int(kind[r])] for r in range(n)]


class World:
    """One corpus with attributes, locations and terms: a single engine and a shard group over it."""

    def __init__(self, oracle, metric, world, n, dims=128, seed=4100, corpus=None):
        rng = np.random.default_rng(seed)
        self.n = n
        self.corpus = corpus if corpus is not None else oracle.synth_rows(seed, 0, n, dims,
                                                                          normalize=(metric is not VectorMetric.dot))
        self.ids = np.arange(n, dtype=np.uint64) * 3 + 77
        self.ts, self.tags = _attributes(rng, n)
        self.lat, self.lon, self.centre = _locations(rng, n)
        self.terms = _terms(rng, n)
        self.single = CUDAVectorEngine(metric, self.corpus.shape[1])
        self.single.add_batch(self.ids, self.corpus)
        self.grp = Group(metric, self.corpus.shape[1], corpus=self.corpus, ids=self.ids, world=world)
        for eng in [self.single] + self.grp.engines:
            self.describe(eng)

    def describe(self, eng):
        """The full lists on every engine: each rank ignores the ids it does not hold."""
        eng.set_attributes(self.ids, self.ts, self.tags)
        eng.set_locations(self.ids, self.lat, self.lon)
        eng.set_terms(self.ids, self.terms)

    def window(self, lo, hi, **kw):
        return Where(after=int(self.ts[lo]), before=int(self.ts[min(hi, self.n - 1)]), **kw)

    def check(self, q, k, where, allow=None, deny=None):
        res = self.grp.collective(lambda r, e: e.shard_search_where(q, k, where, allow=allow, deny=deny))
        assert all(x == res[0] for x in res), "ranks disagree on the merged result"
        flt = [("allow", allow)] if allow is not None else ([("deny", deny)] if deny is not None else [])
        want = self.single.search_batch_where([q], k, [where], [0], flt, [0 if flt else None])[0]
        assert _bits(res[0]) == _bits(want), (where, k)
        return res[0]

    def close(self):
        self.grp.close()
        self.single.close()


def _wheres(w):
    n = w.n
    lo1, hi1 = w.grp.ranges[1]
    edge = w.grp.ranges[0][1]
    return {
        "20%": w.window(n // 3, n // 3 + n // 5, no_tags=DELETED),
        "narrow": w.window(edge - 1500, edge + 1500, no_tags=DELETED | SUPERSEDED),
        "box": Where(near=(w.centre[0], w.centre[1], 25_000.0)),
        "terms": Where(terms=(SESSION + 3, KIND + 1)),
        "nothing": Where(after=10**15),
        "one rank": w.window(lo1 + 10, lo1 + (hi1 - lo1) // 2),
    }


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [VectorMetric.cosine, VectorMetric.dot, VectorMetric.l2])
@pytest.mark.parametrize("world", [2, 3, 8])
def test_fused_sharded_where_equals_the_single_engine(oracle, metric, world):
    w = World(oracle, metric, world, 40_003)
    rng = np.random.default_rng(world)
    try:
        q = oracle.synth_row(4200 + world, 0, w.corpus.shape[1], True)
        allow = w.ids[rng.choice(w.n, w.n // 3, replace=False)]
        for k in (1, 10, 128):
            deny = [i for i, _ in w.single.search(q, 40)] + w.ids[rng.choice(w.n, 500, replace=False)].tolist()
            for name, where in _wheres(w).items():
                got = w.check(q, k, where)
                if name == "nothing":
                    assert got == []
                else:
                    assert len(got) == k
                w.check(q, k, where, allow=allow)
                w.check(q, k, where, deny=deny)
                w.check(q, k, where, deny=[])                                  # a deny-list of nothing: no filter
            assert w.check(q, k, Where(), allow=[]) == []                      # an allow-list of nothing
    finally:
        w.close()


@pytest.mark.gpu
def test_ties_across_shards_and_short_shards(oracle):
    """Period-256 duplicates under a where, so equal distances sit on every shard and the merge breaks them by global
    row; then 8 ranks over 7 rows (one empty shard, the others below k)."""
    dims, n = 64, 3000
    base = oracle.synth_rows(50, 0, 256, dims)
    corpus = np.ascontiguousarray(base[np.arange(n) % 256])
    w = World(oracle, VectorMetric.cosine, 4, n, corpus=corpus)
    try:
        for k in (10, 40, 100):
            for where in (w.window(100, 2900, no_tags=DELETED), Where(terms=(SESSION + 2,)), w.window(0, 1200)):
                w.check(base[7], k, where)
                w.check(base[7], k, where, deny=w.ids[:50])
    finally:
        w.close()
    corpus = oracle.synth_rows(51, 0, 7, 128)
    w = World(oracle, VectorMetric.cosine, 8, 7, corpus=corpus)
    try:
        q = oracle.synth_row(52, 0, 128, True)
        for where in (Where(), w.window(1, 5), Where(no_tags=DELETED), Where(after=10**15)):
            for k in (3, 10):
                w.check(q, k, where)
                w.check(q, k, where, allow=w.ids[[0, 2, 6]])
    finally:
        w.close()


def _device_form(w, qs, k, wheres, query_where, filters, query_filter):
    """Every rank's wax_vs_search_batch_where_device into its slice of one all-gather-shaped buffer, then the merge."""
    import torch
    from wax_b200.engine import _WhereArgs
    b, world = len(qs), w.grp.world
    a = _WhereArgs(wheres, query_where, filters, query_filter, b)
    d_qs = torch.from_numpy(np.ascontiguousarray(qs, np.float32)).cuda()
    gathered = torch.full((world * b * k * 24,), 0xAB, dtype=torch.uint8, device="cuda")   # no slot left unwritten
    for r, eng in enumerate(w.grp.engines):
        rc = L.lib().wax_vs_search_batch_where_device(eng.handle, C.c_void_p(d_qs.data_ptr()), b, k, *a.filter_args(),
                                                      *a.where_args(near=True), *a.term_args(), w.grp.ranges[r][0],
                                                      C.c_void_p(gathered.data_ptr() + r * b * k * 24), None)
        assert rc == 0, L.last_error()
    torch.cuda.synchronize()
    local = gathered.cpu().numpy().view(sharded.CAND_DTYPE).reshape(world, b, k)
    for r in range(world):                  # each list sorted by (distance, global row), padding last and zeroed
        for qi in range(b):
            lst = local[r, qi]
            m = int(lst["valid"].sum())
            assert lst["valid"][:m].all() and not lst[m:].view(np.uint8).any()
            assert np.all((lst["row"][:m] >= w.grp.ranges[r][0]) & (lst["row"][:m] < w.grp.ranges[r][1]))
    out = torch.zeros(b * k * 24, dtype=torch.uint8, device="cuda")
    assert L.lib().wax_vs_merge_candidates_device(w.single.handle, C.c_void_p(gathered.data_ptr()), world, b, k, k,
                                                  C.c_void_p(out.data_ptr()), None) == 0, L.last_error()
    torch.cuda.synchronize()
    best = out.cpu().numpy().view(sharded.CAND_DTYPE).reshape(b, k)
    scores = sharded.score_from_distance(w.single.metric.to_vec_similarity(), best["distance"])
    return [[(int(best["frame_id"][i, j]), float(scores[i, j])) for j in range(int(best["valid"][i].sum()))]
            for i in range(b)]


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [VectorMetric.cosine, VectorMetric.l2])
def test_device_form_merged_equals_the_single_engine(oracle, metric):
    w = World(oracle, metric, 3, 60_001)
    rng = np.random.default_rng(9)
    try:
        if metric is VectorMetric.l2:
            for eng in [w.single] + w.grp.engines:
                eng.set_option("batch_l2", 1)
        ws = list(_wheres(w).values())
        filters = [("allow", w.ids[rng.choice(w.n, 3000, replace=False)]),          # gather class
                   ("allow", w.ids[rng.choice(w.n, w.n // 2, replace=False)]),      # tensor class
                   ("deny", w.ids[rng.choice(w.n, w.n - 100, replace=False)])]      # scan class: fewer rows than k
        b = 300
        qs = oracle.synth_rows(4300, 0, b, w.corpus.shape[1], normalize=True)
        qw = [None if i % 7 == 0 else int(rng.integers(0, len(ws))) for i in range(b)]
        qf = [None if i % 3 == 0 else int(rng.integers(0, len(filters))) for i in range(b)]
        for k in (10, 200):
            got = _device_form(w, qs, k, ws, qw, filters, qf)
            want = w.single.search_batch_where(qs, k, ws, qw, filters, qf)
            for i in range(b):
                assert _bits(got[i]) == _bits(want[i]), (k, i, qw[i], qf[i])
        # the fused form refuses k = 200 before it joins any exchange
        q = qs[0]
        with pytest.raises(InvalidToc, match="top_k <= 128"):
            w.grp.engines[0].shard_search_where(q, 200, ws[0])
    finally:
        w.close()


@pytest.mark.gpu
def test_mirrors_built_inside_the_collective_and_many_calls(oracle):
    """The first sharded where call after set_attributes / set_locations / set_terms builds every rank's mirrors and term
    index inside the collective; then 50 calls with changing wheres and filters grow the scratch while the group is
    connected."""
    w = World(oracle, VectorMetric.cosine, 3, 50_000)
    rng = np.random.default_rng(11)
    try:
        q = oracle.synth_row(4400, 0, w.corpus.shape[1], True)
        w.check(q, 10, Where(near=(w.centre[0], w.centre[1], 25_000.0), terms=(SESSION + 1,), no_tags=DELETED))
        w.ts = w.ts[::-1].copy()                                            # new attributes, locations and terms
        w.terms = w.terms[::-1]
        for eng in [w.single] + w.grp.engines:
            w.describe(eng)
        w.check(q, 10, Where(near=(w.centre[0], w.centre[1], 25_000.0), terms=(SESSION + 5, KIND + 2)))
        for i in range(50):
            lo = int(rng.integers(0, w.n - 2000))
            width = int(rng.choice([200, 5000, 20_000]))
            where = [w.window(lo, lo + width), Where(terms=(SESSION + i % 12,) + ((KIND + i % 4,) if i % 2 else ())),
                     Where(near=(w.centre[0] + 0.01 * (i % 5), w.centre[1], 5_000.0 * (1 + i % 6))),
                     w.window(lo, lo + width, terms=(SESSION + i % 12,))][i % 4]
            flt = [dict(), dict(allow=w.ids[rng.choice(w.n, int(rng.integers(1, 30_000)), replace=False)]),
                   dict(deny=w.ids[rng.choice(w.n, int(rng.integers(1, 30_000)), replace=False)])][i % 3]
            w.check(oracle.synth_row(4500 + i, 0, w.corpus.shape[1], True), int(rng.choice([1, 10, 64, 128])), where, **flt)
    finally:
        w.close()


def test_shard_search_where_argument_checks():
    """They return before the engine is locked or any CUDA call is made (a placeholder handle stands in for an engine),
    so every rank fails alike before any rank joins an exchange."""
    eng = C.cast((C.c_uint8 * (1 << 16))(), C.c_void_p)
    q = np.zeros(8, np.float32)
    ids, sc, n = np.zeros(16, np.uint64), np.zeros(16, np.float32), C.c_uint32(0)
    terms = np.arange(40, dtype=np.uint64)

    def call(where=Where(), mode=0, n_terms=0, n_ids=0):
        w = C.byref(where.to_c_near()) if where is not None else None
        return L.lib().wax_vs_shard_search_where(eng, q.ctypes.data_as(C.POINTER(C.c_float)), 8, 10,
                                                 ids.ctypes.data_as(C.POINTER(C.c_uint64)), n_ids, mode, w,
                                                 terms.ctypes.data_as(C.POINTER(C.c_uint64)) if n_terms else None, n_terms,
                                                 ids.ctypes.data_as(C.POINTER(C.c_uint64)),
                                                 sc.ctypes.data_as(C.POINTER(C.c_float)), 16, C.byref(n))
    assert call(where=None) == L.ERR_NULL
    assert call(n_terms=33) == L.ERR_ARGUMENT and "at most 32" in L.last_error()
    assert call(mode=2) == L.ERR_ARGUMENT
    assert call(where=Where(near=(0.0, 0.0, float("inf")))) == L.ERR_ARGUMENT
    assert L.lib().wax_vs_shard_search_where(eng, None, 8, 10, None, 3, 0, C.byref(Where().to_c_near()), None, 0, None,
                                             None, 0, C.byref(n)) == L.ERR_NULL          # ids NULL with n_ids > 0
    assert L.lib().wax_vs_search_batch_where_device(eng, None, 1, 10, None, None, None, 0, None, None, 0, None, None, None,
                                                    0, None, None) == L.ERR_NULL
