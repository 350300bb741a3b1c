"""GPU: PhotoRAG's location clause below the top-k (wax_vs_search_batch_where_near,
wax_vs_search_batch_grouped_where_near).  The reference allow-list is built here exactly as PhotoRAG builds it -- a dict
from (latBin, lonBin) to frame ids, unioned over the box buildLocationAllowlist walks -- and every answer must be
identical (ids, order, score bits) to the id-filtered search under that allow-list ANDed with the time and tag clauses
and the id filter."""
import math
import threading

import numpy as np
import pytest

from test_gpu_filtered import _expect
from test_gpu_where import DELETED, LABEL, SUPERSEDED, _attributes, _bits, _passing
from test_location_semantics import build_location_allowlist_box
from wax_b200 import CUDAVectorEngine, VectorMetric, Where

pytestmark = pytest.mark.gpu

N, DIMS = 80_000, 384
REGION = (40.0, 42.0, 10.0, 12.5)          # most cluster centres: dense enough for a box of > 16 384 rows


def _locations(rng, n, n_centres=48, spread=0.05, located=0.7):
    """Seeded clusters: `located` of the rows near one of the centres (most in REGION, two at the antimeridian and one
    by the north pole), the rest without a location (NaN pairs)."""
    lat_c = rng.uniform(REGION[0], REGION[1], n_centres)
    lon_c = rng.uniform(REGION[2], REGION[3], n_centres)
    lat_c[:3] = [0.5, -0.5, 89.99]
    lon_c[:3] = [179.995, -179.995, 0.0]
    c = rng.integers(0, n_centres, n)
    lat = lat_c[c] + spread * rng.standard_normal(n)
    lon = lon_c[c] + spread * rng.standard_normal(n)
    none = rng.random(n) >= located
    lat[none] = np.nan
    lon[none] = np.nan
    return lat, lon, np.stack([lat_c, lon_c], 1)


class PhotoIndex:
    """PhotoRAG's index.locationBins (PhotoRAGOrchestrator.swift:766-771) and buildLocationAllowlist's union
    (:843-852), over the engine's frame ids."""

    def __init__(self, ids, lat, lon):
        self.bins = {}
        for fid, a, b in zip(ids.tolist(), lat.tolist(), lon.tolist()):
            if math.isnan(a):
                continue
            self.bins.setdefault((math.floor(a * 100.0), math.floor(b * 100.0)), set()).add(fid)

    def allowlist(self, near):
        """The frame-id set, or None for "no location clause"."""
        got = build_location_allowlist_box(*near)
        if got is None:
            return None
        (lat_lo, lat_hi), ranges = got
        out = set()
        for lat_bin in range(lat_lo, lat_hi + 1):
            for lo, hi in ranges:
                for lon_bin in range(lo, hi + 1):
                    out |= self.bins.get((lat_bin, lon_bin), set())
        return out


def _allowed(where, flt, ids, ts, tags, index):
    ok = np.ones(ids.size, bool) if where is None else _passing(where, ts, tags)
    if where is not None and where.near is not None:
        allow = index.allowlist(where.near)
        if allow is not None:
            ok &= np.isin(ids, np.fromiter(allow, np.uint64, len(allow)))
    if flt is not None:
        listed = np.isin(ids, np.asarray(flt[1], np.uint64))
        ok &= listed if flt[0] == "allow" else ~listed
    return np.flatnonzero(ok)


def _expected(eng, qs, k, wheres, query_where, filters, query_filter, ids, ts, tags, index):
    lists, qf = [], []
    for qi in range(len(qs)):
        w, f = query_where[qi], query_filter[qi]
        if w is None:
            if f is None:
                qf.append(None)
                continue
            lists.append(filters[f])
        else:
            lists.append(("allow", ids[_allowed(wheres[w], None if f is None else filters[f], ids, ts, tags, index)]))
        qf.append(len(lists) - 1)
    return eng.search_batch_multi_filtered(qs, k, lists, qf)


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
    lat, lon, centres = _locations(rng, N)
    assert eng.set_locations(ids, lat, lon) == N
    return eng, corpus, ids, ts, tags, PhotoIndex(ids, lat, lon), centres


def _wheres(ts, centres):
    mid = ((REGION[0] + REGION[1]) / 2, (REGION[2] + REGION[3]) / 2)
    c = centres[5]
    return [Where(near=(mid[0], mid[1], 100_000.0)),                                         # 0 > 16 384 rows: tensor
            Where(near=(c[0], c[1], 1000.0)),                                                # 1 one cluster's core: gather
            Where(near=(c[0], c[1], 3.0), no_tags=DELETED),                                  # 2 a bin or two: few rows
            Where(near=(-60.0, -60.0, 25_000.0)),                                            # 3 an empty box
            Where(near=(mid[0], mid[1], 1e7)),                                               # 4 the 100 000-bin guard
            Where(after=int(ts[N // 10]), before=int(ts[N // 10 + N // 2]), no_tags=DELETED | SUPERSEDED,
                  near=(c[0], c[1], 25_000.0)),                                              # 5 box AND window AND tags
            Where(near=(0.5, 179.995, 20_000.0), all_tags=LABEL),                            # 6 at the antimeridian
            Where(near=(89.995, 0.0, 100.0)),                                                # 7 by the pole: +-10 degrees
            Where(no_tags=DELETED)]                                                          # 8 no location clause


@pytest.mark.parametrize("metric,batch_l2", [(VectorMetric.cosine, 0), (VectorMetric.dot, 0), (VectorMetric.l2, 1),
                                             (VectorMetric.l2, 0)])
def test_each_answer_equals_multi_filtered_with_photorags_allow_list(oracle, metric, batch_l2):
    eng, corpus, ids, ts, tags, index, centres = _engine(oracle, metric, 5100 + metric.value, batch_l2)
    rng = np.random.default_rng(5101 + metric.value + batch_l2)
    wheres = _wheres(ts, centres)
    sizes = [_allowed(w, None, ids, ts, tags, index).size for w in wheres]
    assert sizes[0] > 16384 and 0 < sizes[1] <= 16384 and sizes[2] < 200 and sizes[3] == 0 and sizes[4] == N
    assert sizes[6] > 0 and sizes[7] > 0
    filters = [("allow", ids[rng.choice(N, 30_000, replace=False)]),                   # allow-list AND where
               ("deny", ids[rng.choice(N, 20_000, replace=False)]),                    # deny-list AND where
               ("allow", ids[rng.choice(N, 700, replace=False)])]                      # small allow-list
    combos = [(w, f) for w in [None] + list(range(len(wheres))) for f in [None] + list(range(len(filters)))]
    for b in (1, 3, 64):
        order = rng.permutation(len(combos))
        picks = [combos[i] for i in order[:b]] if b < len(combos) else \
            combos + [combos[i] for i in rng.integers(0, len(combos), b - len(combos))]
        qs = oracle.synth_rows(5102 + metric.value + b, 0, b, DIMS, normalize=True)
        query_where = [w for w, _ in picks]
        query_filter = [f for _, f in picks]
        for k in (1, 10, 72, 200):
            got = eng.search_batch_where(qs, k, wheres, query_where, filters, query_filter)
            want = _expected(eng, qs, k, wheres, query_where, filters, query_filter, ids, ts, tags, index)
            assert len(got) == b
            for qi in range(b):
                assert _bits(got[qi]) == _bits(want[qi]), (b, k, picks[qi])
    qs = oracle.synth_rows(5199 + metric.value, 0, len(combos), DIMS, normalize=True)
    got = eng.search_batch_where(qs, 10, wheres, [w for w, _ in combos], filters, [f for _, f in combos])
    want = _expected(eng, qs, 10, wheres, [w for w, _ in combos], filters, [f for _, f in combos], ids, ts, tags, index)
    for qi, (w, f) in enumerate(combos):
        assert _bits(got[qi]) == _bits(want[qi]), (w, f)
        if f is None and w in (0, 1, 2, 5):                                          # and the oracle, for a few
            rows = _allowed(wheres[w], None, ids, ts, tags, index)
            assert got[qi] == _expect(oracle, metric, corpus, ids, list(rows), qs[qi], 10)


def test_no_location_clause_is_the_where_search():
    rng = np.random.default_rng(5200)
    eng = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    eng.fill_synthetic(5201, N, id_base=11)
    ids = np.arange(N, dtype=np.uint64) + 11
    ts, tags = _attributes(rng, N)
    eng.set_attributes(ids, ts, tags)
    lat, lon, _ = _locations(rng, N)
    eng.set_locations(ids, lat, lon)
    qs = np.asarray(rng.standard_normal((8, DIMS)), np.float32)
    uploads = eng.counter("location_uploads")
    for near in ((41.0, 11.0, 0.0), (41.0, 11.0, -5.0), (41.0, 11.0, float("nan")), (41.0, 11.0, 1e7)):
        w = Where(no_tags=DELETED, after=int(ts[100]), near=near)
        plain = Where(no_tags=DELETED, after=int(ts[100]))
        assert [_bits(h) for h in eng.search_batch_where(qs, 10, [w], [0] * 8)] == \
            [_bits(h) for h in eng.search_batch_where(qs, 10, [plain], [0] * 8)]
    assert eng.counter("location_uploads") == uploads                             # no box: the mirror is not needed
    with pytest.raises(Exception, match="not representable"):
        eng.search_batch_where(qs, 10, [Where(near=(0.0, 0.0, float("inf")))], [0] * 8)


def test_batch_of_1024_and_many_pairs_over_three_bitsets():
    rng = np.random.default_rng(5300)
    eng = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    eng.fill_synthetic(5301, N, id_base=1000)
    ids = np.arange(N, dtype=np.uint64) + 1000
    ts, tags = _attributes(rng, N)
    eng.set_attributes(ids, ts, tags)
    lat, lon, centres = _locations(rng, N, spread=0.3)
    eng.set_locations(ids, lat, lon)
    index = PhotoIndex(ids, lat, lon)
    words = (N + 31) // 32
    eng.set_option("filter_bitset_bytes", 3 * words * 4)
    wide = [Where(near=(float(c[0]), float(c[1]), 60_000.0), no_tags=DELETED) for c in centres[3:13]]
    narrow = [Where(near=(float(c[0]), float(c[1]), 2_000.0)) for c in centres[13:19]]
    wheres = wide + narrow + [Where(no_tags=DELETED)]
    filters = [("deny", ids[rng.choice(N, 5000, replace=False)]), ("allow", ids[rng.choice(N, 20_000, replace=False)])]
    b = 1024
    qs = np.asarray(rng.standard_normal((b, DIMS)), np.float32)
    query_where = [None if c < 0 else int(c) for c in rng.integers(-1, len(wheres), b)]
    query_filter = [None if c < 0 else int(c) for c in rng.integers(-1, len(filters), b)]
    passes0 = eng.counter("filter_bitset_passes")
    got = eng.search_batch_where(qs, 10, wheres, query_where, filters, query_filter)
    assert eng.counter("filter_bitset_passes") - passes0 >= 4                      # > 3 wide pairs: several sub-batches
    want = _expected(eng, qs, 10, wheres, query_where, filters, query_filter, ids, ts, tags, index)
    for qi in range(b):
        assert _bits(got[qi]) == _bits(want[qi]), qi


def test_count_pass_chunks_with_and_without_a_box():
    rng = np.random.default_rng(5350)
    eng = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    eng.fill_synthetic(5351, N, id_base=40)
    ids = np.arange(N, dtype=np.uint64) + 40
    ts, tags = _attributes(rng, N)
    eng.set_attributes(ids, ts, tags)
    lat, lon, centres = _locations(rng, N)
    eng.set_locations(ids, lat, lon)
    index = PhotoIndex(ids, lat, lon)
    # 300 wheres without an id filter, one count-pass predicate each: the first chunk of 256 has no box, the second
    # has a box in each where; narrow and wide ones on both sides, so the listing and bitset passes see both too
    plain = []
    for _ in range(256):
        a = int(rng.integers(0, N - 30_000))
        span = int(rng.choice([2_000, 30_000]))
        plain.append(Where(after=int(ts[a]), before=int(ts[a + span]), no_tags=DELETED))
    boxed = [Where(near=(float(c[0]), float(c[1]), float(rng.choice([2_000.0, 120_000.0]))), no_tags=SUPERSEDED)
             for c in centres[3:47]]
    wheres = plain + boxed
    b = len(wheres)
    assert b > 256
    sizes = [_allowed(w, None, ids, ts, tags, index).size for w in wheres]
    for part in (sizes[:256], sizes[256:]):
        assert min(part) <= 16384 < max(part)                                      # gather and bitset on each side
    qs = np.asarray(rng.standard_normal((b, DIMS)), np.float32)
    uploads = eng.counter("location_uploads")
    got = eng.search_batch_where(qs, 10, wheres, list(range(b)))
    assert eng.counter("location_uploads") == uploads + 1
    want = _expected(eng, qs, 10, wheres, list(range(b)), [], [None] * b, ids, ts, tags, index)
    for qi in range(b):
        assert _bits(got[qi]) == _bits(want[qi]), qi


def test_single_query_takes_the_shadow_route_under_the_near_bitset(oracle):
    n = 200_000
    rng = np.random.default_rng(5402)
    eng = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    eng.fill_synthetic(5400, n, id_base=3)
    ids = np.arange(n, dtype=np.uint64) + 3
    ts, tags = _attributes(rng, n)
    eng.set_attributes(ids, ts, tags)
    lat, lon, _ = _locations(rng, n)
    eng.set_locations(ids, lat, lon)
    index = PhotoIndex(ids, lat, lon)
    eng.set_option("shadow_scan_min_bytes", 0)
    mid = ((REGION[0] + REGION[1]) / 2, (REGION[2] + REGION[3]) / 2)
    wheres = [Where(near=(mid[0], mid[1], 100_000.0)),
              Where(near=(mid[0], mid[1], 80_000.0), after=int(ts[n // 10]), before=int(ts[n // 10 + n // 2]),
                    no_tags=DELETED)]
    q = oracle.synth_rows(5401, 0, 1, DIMS, normalize=True)
    routed = lambda: (eng.counter("single_shadow_queries"), eng.counter("single_shadow_fallbacks"))
    for w in range(len(wheres)):
        assert _allowed(wheres[w], None, ids, ts, tags, index).size > 16384       # a bitset, not a gather
        before = routed()
        got = eng.search_where(q[0], 10, wheres[w])
        assert routed() == (before[0] + 1, before[1])
        eng.set_option("shadow_scan", 0)
        fp32 = eng.search_where(q[0], 10, wheres[w])
        eng.set_option("shadow_scan", 1)
        assert _bits(got) == _bits(fp32)
        assert _bits(got) == _bits(_expected(eng, q, 10, wheres, [w], [], [None], ids, ts, tags, index)[0])


def test_grouped_where_near_equals_grouped_search_under_the_allow_list(oracle):
    rng = np.random.default_rng(5500)
    corpus = oracle.synth_rows(5500, 0, N, DIMS, normalize=True)
    crowd = corpus[0] + 0.02 * rng.standard_normal((4000, DIMS)).astype(np.float32)
    corpus[:4000] = crowd / np.linalg.norm(crowd, axis=1, keepdims=True)         # rows 0..3999: one crowded group
    ids = np.arange(N, dtype=np.uint64) * 2 + 9
    eng = CUDAVectorEngine(VectorMetric.cosine, DIMS)
    eng.add_batch(ids, corpus)
    eng.set_groups(ids, np.where(np.arange(N) < 4000, 1, 1000 + np.arange(N) // 8).astype(np.uint64))
    ts, tags = _attributes(rng, N)
    eng.set_attributes(ids, ts, tags)
    lat, lon, centres = _locations(rng, N)
    lat[:4000] = 41.0 + 0.01 * rng.standard_normal(4000)                           # the crowd sits in the wide box
    lon[:4000] = 11.25 + 0.01 * rng.standard_normal(4000)
    eng.set_locations(ids, lat, lon)
    index = PhotoIndex(ids, lat, lon)
    c = centres[5]
    wheres = [Where(near=(41.0, 11.25, 100_000.0), no_tags=DELETED),
              Where(near=(41.0, 11.25, 25_000.0), after=int(ts[0]), before=int(ts[N // 2]), no_tags=SUPERSEDED),
              Where(near=(float(c[0]), float(c[1]), 1000.0)),
              Where(near=(-60.0, -60.0, 25_000.0))]
    deny = ids[rng.choice(N, 3000, replace=False)]
    allow = ids[rng.choice(N, 40_000, replace=False)]
    for n in (1, 64, 1024):
        qs = np.asarray(rng.standard_normal((n, DIMS)), np.float32)
        qs[0] = corpus[1]                                                          # a crowded query
        for w, flt in ((0, None), (1, ("deny", deny)), (1, ("allow", allow)), (2, None), (3, None)):
            kw = {} if flt is None else {flt[0]: flt[1]}
            got = eng.search_batch_grouped_where(qs, 5, 3, wheres[w], **kw)
            rows = _allowed(wheres[w], flt, ids, ts, tags, index)
            check = range(n) if n <= 64 else rng.choice(n, 32, replace=False)
            for qi in check:
                want = eng.search_grouped(qs[qi], 5, 3, allow=ids[rows]) if rows.size else []
                assert got[qi] == want, (n, w, flt and flt[0], qi)
    assert eng.counter("grouped_batch_expanded_groups") > 0
    assert eng.counter("grouped_batch_fallback_queries") > 0


def test_locations_follow_their_rows():
    rng = np.random.default_rng(5600)
    dims = 64
    eng = CUDAVectorEngine(VectorMetric.cosine, dims)
    model = {}                                                                     # frame id -> (latBin, lonBin) or None
    vec = lambda m: np.asarray(rng.standard_normal((m, dims)), np.float32)
    ids = np.arange(100, 2100, dtype=np.uint64)
    eng.add_batch(ids, vec(ids.size))
    for i in ids:
        model[int(i)] = None
    boxes = [Where(near=(41.0, 11.0, 30_000.0)), Where(near=(41.2, 11.2, 3_000.0), no_tags=2),
             Where(near=(0.0, 0.0, 1.0))]

    tag_of = {}                                                                    # frame id -> tags, when set

    def check():
        for w in boxes:
            want = sorted(f for f, loc in model.items() if w.passes(0, tag_of.get(f, 0), loc))
            got = eng.search_where(rng.standard_normal(dims), 10_000, w)
            assert sorted(i for i, _ in got) == want, w

    uploads = eng.counter("location_uploads")
    check()                                                                        # no locations: nothing passes
    assert eng.counter("location_uploads") == uploads + 1
    check()
    assert eng.counter("location_uploads") == uploads + 1                         # once per invalidation
    lat = 41.0 + 0.2 * rng.standard_normal(ids.size)
    lon = 11.0 + 0.2 * rng.standard_normal(ids.size)
    lat[:5], lon[:5] = [0.0, -0.0, 0.001, -0.001, 0.0], [0.0, 0.0, -0.001, 0.001, 0.005]
    assert eng.set_locations(np.concatenate([ids, [1, 2]]), np.concatenate([lat, [0, 0]]),
                             np.concatenate([lon, [0, 0]])) == ids.size            # unknown ids ignored
    for i, a, b in zip(ids, lat, lon):
        model[int(i)] = (math.floor(a * 100.0), math.floor(b * 100.0))
    check()
    assert eng.counter("location_uploads") == uploads + 2
    eng.set_locations(ids[10:12].repeat(2), [41.0, 0.0, 41.0, 0.0], [11.0, 0.0, 11.0, 0.0])   # a later entry wins
    model[int(ids[10])] = model[int(ids[11])] = (0, 0)
    eng.set_locations(ids[20:30], np.full(10, np.nan), np.full(10, np.nan))       # a NaN pair clears
    for i in ids[20:30]:
        model[int(i)] = None
    with pytest.raises(Exception):
        eng.set_locations(ids[30:32], [41.0, np.inf], [11.0, 11.0])               # nothing written
    check()
    eng.add(int(ids[40]), vec(1)[0])                                               # upsert keeps the location
    new = np.arange(5000, 5050, dtype=np.uint64)
    eng.add_batch(new, vec(new.size))                                              # appended frames have none
    for i in new:
        model[int(i)] = None
    eng.add_batch(np.array([7000, 150, 6000], np.uint64), vec(3))                  # out of order: upsert + appends
    model[7000] = model[6000] = None
    check()
    eng.set_attributes(ids[:300], tags=np.full(300, 2, np.uint64))                 # the tag clause beside the box
    tag_of = {int(i): 2 for i in ids[:300]}
    check()
    eng.remove(int(ids[3]))
    del model[int(ids[3])]
    gone = ids[rng.choice(ids.size, 300, replace=False)]
    eng.remove_batch(gone)
    for i in gone:
        model.pop(int(i), None)
    check()
    eng.deserialize(eng.serialize())                                               # MV2V carries no locations: reset
    model = {f: None for f in model}
    tag_of = {}
    check()
    eng.set_locations(np.array(sorted(model), np.uint64), np.full(len(model), 41.0), np.full(len(model), 11.0))
    eng.fill_synthetic(5601, 500, id_base=10)                                      # reset too
    model = {10 + r: None for r in range(500)}
    check()


def test_a_search_concurrent_with_set_locations_sees_old_or_new():
    rng = np.random.default_rng(5700)
    eng = CUDAVectorEngine(VectorMetric.cosine, 128)
    n = 20_000
    eng.fill_synthetic(5701, n)
    ids = np.arange(n, dtype=np.uint64)
    inside = lambda m: np.where(m, 41.0, -41.0)
    lat_a, lat_b = inside(ids % 2 == 0), inside(ids % 3 == 0)                      # A: even frames inside, B: thirds
    lon = np.full(n, 11.0)
    eng.set_locations(ids, lat_a, lon)
    w = Where(near=(41.0, 11.0, 5000.0))
    sets = [set(ids[lat_a > 0].tolist()), set(ids[lat_b > 0].tolist())]
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
        eng.set_locations(ids, lat_b if i % 2 == 0 else lat_a, lon)
    stop.set()
    t.join()
    assert not errors
    assert seen
    for got in seen:
        assert got == sets[0] or got == sets[1]


def test_ties_and_non_finite_rows(oracle):
    rng = np.random.default_rng(5800)
    n, dims = 20_000, 128
    corpus = oracle.synth_rows(5801, 0, n, dims, normalize=True)
    corpus[100:140] = corpus[99]                                                   # exact ties
    corpus[200] = np.nan
    corpus[201] = np.inf
    ids = np.arange(n, dtype=np.uint64) + 5
    eng = CUDAVectorEngine(VectorMetric.cosine, dims)
    eng.add_batch(ids, corpus)
    ts, tags = _attributes(rng, n)
    eng.set_attributes(ids, ts, tags)
    lat = np.where(np.arange(n) < 1000, 41.0, 50.0) + 0.001 * rng.standard_normal(n)
    lon = np.full(n, 11.0)
    eng.set_locations(ids, lat, lon)
    index = PhotoIndex(ids, lat, lon)
    wheres = [Where(near=(41.0, 11.0, 2000.0)), Where(near=(41.0, 11.0, 2000.0), before=int(ts[5000])),
              Where(near=(50.0, 11.0, 2000.0), no_tags=DELETED)]
    qs = np.stack([corpus[99], corpus[150], corpus[0]])
    for k in (1, 10, 72):
        for wi in range(len(wheres)):
            got = eng.search_batch_where(qs, k, wheres, [wi] * 3)
            want = _expected(eng, qs, k, wheres, [wi] * 3, [], [None] * 3, ids, ts, tags, index)
            for qi in range(3):
                assert _bits(got[qi]) == _bits(want[qi])


def test_full_size_photo_workload():
    rng = np.random.default_rng(5900)
    n, dims = 10_000_000, 384
    eng = CUDAVectorEngine(VectorMetric.cosine, dims)
    eng.fill_synthetic(5901, n)
    ids = np.arange(n, dtype=np.uint64)
    ts = np.arange(n, dtype=np.int64)
    tags = np.where(rng.random(n) < 0.01, DELETED, 0).astype(np.uint64)
    eng.set_attributes(ids, ts, tags)
    n_c = 300
    lat_c, lon_c = rng.uniform(-60, 60, n_c), rng.uniform(-170, 170, n_c)
    c = rng.integers(0, n_c, n)
    lat = lat_c[c] + 0.18 * rng.standard_normal(n)
    lon = lon_c[c] + 0.18 * rng.standard_normal(n)
    none = rng.random(n) >= 0.7
    lat[none] = lon[none] = np.nan
    eng.set_locations(ids, lat, lon)
    lat_bin, lon_bin = np.floor(lat * 100.0), np.floor(lon * 100.0)
    b = 1024
    qs = np.asarray(rng.standard_normal((b, dims)), np.float32)
    wheres = []
    for i in range(b):
        a = int(rng.integers(0, n - n // 5))
        ci = int(rng.integers(0, n_c))
        r = 25_000.0 if i % 2 == 0 else 1_000.0
        wheres.append(Where(after=a, before=a + n // 5, no_tags=DELETED, near=(float(lat_c[ci]), float(lon_c[ci]), r)))
    got = eng.search_batch_where(qs, 10, wheres, list(range(b)))
    for qi in rng.choice(b, 12, replace=False):
        w = wheres[qi]
        (la, lb), ranges = build_location_allowlist_box(*w.near)
        ok = (lat_bin >= la) & (lat_bin <= lb) & (lon_bin >= ranges[0][0]) & (lon_bin <= ranges[0][1])
        ok &= (ts >= w.after) & (ts < w.before) & ((tags & np.uint64(DELETED)) == 0)
        want = eng.search_batch_multi_filtered(qs[qi:qi + 1], 10, [("allow", ids[ok])], [0])[0]
        assert _bits(got[qi]) == _bits(want), qi
