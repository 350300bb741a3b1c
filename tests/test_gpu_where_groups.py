"""GPU: group clauses below the top-k (wax_vs_search_batch_where_groups, wax_vs_search_batch_grouped_multi_where_groups),
VideoRAG's videoIDs as "the row's group is one of these".  The reference allow-list is computed here in numpy -- the
frames whose group is named AND pass the time, tag, location and term clauses AND the id filter -- and every answer must
be identical (ids, order, score bits) to the id-filtered search (grouped: search_grouped) under it."""
import ctypes as C
import threading

import numpy as np
import pytest
import torch

from wax_b200 import CUDAVectorEngine, VectorMetric, Where
from wax_b200 import _lib as L

pytestmark = pytest.mark.gpu

N = 40_000
DELETED = 1
GROUP = 360                                   # consecutive rows per group, as VideoRAG's segments of one video


class Corpus:
    """An engine and the host model of its frames: ids, timestamps, tags, groups (None: implicit), terms."""

    def __init__(self, metric, dims, n=N, seed=0, layout="consecutive", batch_l2=0, devices=None):
        rng = np.random.default_rng(seed)
        self.rng = rng
        self.vecs = rng.standard_normal((n, dims), dtype=np.float32)
        if metric is not VectorMetric.dot:
            self.vecs /= np.linalg.norm(self.vecs, axis=1, keepdims=True)
        self.ids = np.arange(n, dtype=np.uint64) * 3 + 77
        self.eng = CUDAVectorEngine(metric, dims, devices=devices) if devices else CUDAVectorEngine(metric, dims)
        self.eng.add_batch(self.ids, self.vecs)
        if batch_l2:
            self.eng.set_option("batch_l2", 1)
        self.ts = rng.integers(0, 1000, n).astype(np.int64)
        self.tags = (rng.random(n) < 0.01).astype(np.uint64) * DELETED | rng.integers(0, 4, n).astype(np.uint64) << 1
        self.eng.set_attributes(self.ids, self.ts, self.tags)
        rows = np.arange(n)
        if layout == "consecutive":
            self.groups = self.ids[rows // GROUP * GROUP]                    # the root is the group's first frame
        elif layout == "hashed":
            self.groups = ((rows * 2654435761) % 997).astype(np.uint64) + 5_000_000
        elif layout == "half":
            self.groups = np.where(rows % 2 == 0, 9_000_000, rows // 50 + 9_000_001).astype(np.uint64)
        else:                                                                # implicit: each frame is its own group
            self.groups = None
        if self.groups is not None:
            self.eng.set_groups(self.ids, self.groups)
        self.terms = None

    def group_of(self):
        return self.ids if self.groups is None else self.groups

    def set_terms(self, lists):
        self.terms = lists
        self.eng.set_terms(self.ids, lists)

    def passing(self, where, flt=None):
        """Frame ids passing `where` AND the id filter (mode, ids)."""
        ok = np.ones(self.ids.size, bool)
        if where is not None:
            ok &= (self.ts >= where.after) & ((self.ts < where.before) | (where.before == np.iinfo(np.int64).max))
            ok &= (self.tags & np.uint64(where.all_tags)) == np.uint64(where.all_tags)
            ok &= (self.tags & np.uint64(where.no_tags)) == 0
            if where.groups:
                ok &= np.isin(self.group_of(), np.asarray(where.groups, np.uint64))
            if where.terms:
                req = set(where.terms)
                ok &= np.fromiter((req <= set(t) for t in self.terms), bool, ok.size) if self.terms else False
        if flt is not None:
            listed = np.isin(self.ids, np.asarray(flt[1], np.uint64))
            ok &= listed if flt[0] in ("allow", 0) else ~listed
        return self.ids[ok]

    def expected(self, qs, k, wheres, qw, filters=(), qf=None):
        qf = qf or [None] * len(qs)
        allow = [("allow", self.passing(None if w is None else wheres[w], None if f is None else filters[f]))
                 if (w is not None or f is not None) else None for w, f in zip(qw, qf)]
        lists = [a for a in allow if a is not None]
        index, j = [], 0
        for a in allow:
            index.append(None if a is None else j)
            j += a is not None
        return self.eng.search_batch_multi_filtered(qs, k, lists, index)

    def check(self, qs, k, wheres, qw, filters=(), qf=None):
        got = self.eng.search_batch_where(qs, k, wheres, qw, list(filters), qf)
        want = self.expected(qs, k, wheres, qw, filters, qf)
        for i, (g, w) in enumerate(zip(got, want)):
            assert g == w, ("query", i)
        return got

    def queries(self, b):
        return self.rng.standard_normal((b, self.vecs.shape[1]), dtype=np.float32)


def _roots(c, idx):
    """The group ids of consecutive groups idx (the root frames' ids)."""
    return tuple(int(c.ids[i * GROUP]) for i in idx)


def _mixed_wheres(c):
    g = c.group_of()
    some = tuple(int(x) for x in np.unique(g)[:: max(1, np.unique(g).size // 9)][:9])
    return [
        Where(groups=some),                                                   # groups alone
        Where(after=200, before=400, no_tags=DELETED, groups=some),           # AND a 20 % window AND not deleted
        Where(groups=some[:2] + some[:2] + ((1 << 64) - 1, 12345)),           # duplicates and unknown ids
        Where(groups=((1 << 64) - 1,)),                                       # only unknown ids: nothing passes
        Where(after=100, before=900, all_tags=2),                             # an empty group list is no clause
        Where(groups=tuple(int(x) for x in np.unique(g)[:3000])),             # a wide unit
    ]


@pytest.mark.parametrize("metric,dims,batch_l2", [(VectorMetric.cosine, 384, 0), (VectorMetric.dot, 384, 0),
                                                  (VectorMetric.l2, 384, 0), (VectorMetric.l2, 384, 1),
                                                  (VectorMetric.cosine, 768, 0), (VectorMetric.cosine, 100, 0),
                                                  (VectorMetric.dot, 100, 0)])
def test_answers_equal_the_allow_list_form(metric, dims, batch_l2):
    c = Corpus(metric, dims, seed=dims + metric.value, batch_l2=batch_l2)
    wheres = _mixed_wheres(c)
    qs = c.queries(96)
    qw = [i % (len(wheres) + 1) if i % (len(wheres) + 1) < len(wheres) else None for i in range(96)]
    filters = [("allow", c.ids[::5]), ("deny", c.ids[::3])]
    qf = [None if i % 3 == 0 else (i % 2) for i in range(96)]
    for k in (1, 10, 100):
        c.check(qs, k, wheres, qw)
        c.check(qs, k, wheres, qw, filters, qf)
    c.eng.close()


@pytest.mark.parametrize("layout", ["consecutive", "hashed", "implicit", "half"])
def test_group_layouts(layout):
    c = Corpus(VectorMetric.cosine, 384, seed=3, layout=layout)
    wheres = _mixed_wheres(c)
    if layout == "half":
        wheres.append(Where(groups=(9_000_000,), no_tags=DELETED))          # one group holding half the rows
        wheres.append(Where(groups=(9_000_000, 9_000_003), after=500))
    qs = c.queries(64)
    qw = [i % len(wheres) for i in range(64)]
    for k in (10, 72):
        c.check(qs, k, wheres, qw)
    c.check(qs[:1], 10, wheres, [len(wheres) - 1])
    c.eng.close()


def test_terms_and_locations_with_groups():
    c = Corpus(VectorMetric.cosine, 384, seed=5)
    rare = c.rng.random(N) < 0.01
    c.set_terms([[1, 2] if r else [1] for r in rare])                       # term 1 on every row, term 2 on 1 %
    lat = np.where(np.arange(N) % 4 == 0, 48.85, 10.0)
    c.eng.set_locations(c.ids, lat, np.full(N, 2.35))
    many = _roots(c, range(0, 100, 2))                                       # 50 groups: 18 000 rows
    few = _roots(c, range(3))                                                # 3 groups: 1 080 rows
    wheres = [Where(terms=(2,), groups=many),                                # rarest posting (~400) < group union
              Where(terms=(1,), groups=few),                                 # group union < the posting (every row)
              Where(terms=(1, 2), groups=few, no_tags=DELETED),
              Where(near=(48.85, 2.35, 5000.0), groups=many),                 # a box and groups
              Where(terms=(3,), groups=many)]                                # a term no row holds
    qs = c.queries(40)
    qw = [i % len(wheres) for i in range(40)]
    got = c.eng.search_batch_where(qs, 10, wheres, qw)
    lat_ok = np.isin(c.ids, c.ids[np.arange(N) % 4 == 0])
    for i, w in enumerate(qw):
        where = wheres[w]
        keep = np.isin(c.ids, c.passing(Where(after=where.after, before=where.before, all_tags=where.all_tags,
                                                   no_tags=where.no_tags, terms=where.terms, groups=where.groups)))
        if where.near is not None:
            keep &= lat_ok
        want = c.eng.search_batch_multi_filtered(qs[i:i + 1], 10, [("allow", c.ids[keep])], [0])[0]
        assert got[i] == want, ("query", i)
    # which source each unit walks: the rarest posting of where 0, the group union of where 1
    before = c.eng.counter("where_group_rows_walked")
    c.eng.search_batch_where(qs[:2], 10, wheres[:2], [0, 1])
    assert c.eng.counter("where_group_rows_walked") - before == int(rare.sum()) + 3 * GROUP
    c.eng.close()


def test_classes_units_and_rows_walked():
    c = Corpus(VectorMetric.cosine, 384, seed=7)
    narrow = [Where(groups=_roots(c, (i, i + 7)), no_tags=DELETED) for i in range(20)]             # 720 rows each
    wide = [Where(groups=_roots(c, range(i, 100, 3)), after=100) for i in range(3)]                 # ~12 000 rows
    wide += [Where(groups=_roots(c, range(j % 2, 110, 2)), after=j) for j in range(6)]              # > 16 384 rows
    wheres = narrow + wide + [Where(groups=_roots(c, (0, 7)), no_tags=DELETED)]                     # equal to narrow[0]
    qs = c.queries(200)
    qw = [i % len(wheres) for i in range(200)]
    units, walked = c.eng.counter("where_group_units"), c.eng.counter("where_group_rows_walked")
    c.check(qs, 10, wheres, qw)
    assert c.eng.counter("where_group_units") - units == len(wheres) - 1                           # equal wheres are one
    sizes = sum(len(set(w.groups)) * GROUP for w in wheres[:-1])
    assert c.eng.counter("where_group_rows_walked") - walked == sizes                              # no corpus pass
    c.eng.set_option("filter_bitset_bytes", 3 * ((N + 31) // 32) * 4)                             # 3 bitsets per pass
    passes = c.eng.counter("filter_bitset_passes")
    c.check(qs, 10, wheres, qw)
    assert c.eng.counter("filter_bitset_passes") - passes >= 2
    c.eng.close()


def test_a_batch_of_one_takes_the_shadow_route_under_a_wide_bitset():
    c = Corpus(VectorMetric.cosine, 384, seed=9)
    c.eng.set_option("batch_bf16", 1)
    c.eng.set_option("shadow_scan_min_bytes", 0)
    w = [Where(groups=_roots(c, range(0, 110, 2)), no_tags=DELETED)]      # ~19 600 rows: wider than a gather
    q = c.queries(1)
    before = c.eng.counter("single_shadow_queries")
    got = c.eng.search_batch_where(q, 10, w, [0])
    assert c.eng.counter("single_shadow_queries") - before == 1
    assert got == c.expected(q, 10, w, [0])
    c.eng.close()


def _grouped_expected(c, q, g, p, where, flt=None):
    return c.eng.search_grouped(q, g, per_group=p, allow=c.passing(where, flt))


@pytest.mark.parametrize("layout", ["consecutive", "hashed"])
def test_grouped_answers_equal_search_grouped(layout):
    c = Corpus(VectorMetric.cosine, 384, seed=11, layout=layout)
    gs = np.unique(c.group_of())
    own = [Where(groups=tuple(int(x) for x in gs[i * 16:(i + 1) * 16]), after=200, before=400) for i in range(8)]
    wheres = own + [Where(groups=tuple(int(x) for x in gs[::2]), no_tags=DELETED),   # a wide unit
                    Where(groups=(int(gs[0]),)),                                       # one group: a crowded query
                    Where(groups=((1 << 64) - 1,))]
    qs = c.queries(48)
    qw = [i % len(wheres) for i in range(48)]
    filters = [("deny", c.ids[::4]), ("allow", c.ids[::2])]
    qf = [None if i % 3 else (i // 3) % 2 for i in range(48)]
    for g, p in ((12, 3), (5, 1), (3, 40)):
        got = c.eng.search_batch_grouped_multi_where(qs, g, p, wheres, qw, filters, qf)
        for i in range(48):
            flt = None if qf[i] is None else filters[qf[i]]
            assert got[i] == _grouped_expected(c, qs[i], g, p, wheres[qw[i]], flt), (g, p, i)
    # expansions under the bitsets of many wide units, three per pass
    c.eng.set_option("filter_bitset_bytes", 3 * ((N + 31) // 32) * 4)
    wide = [Where(groups=tuple(int(x) for x in gs[i::5])) for i in range(5)]
    got = c.eng.search_batch_grouped_multi_where(qs[:20], 12, 3, wide, [i % 5 for i in range(20)])
    for i in range(20):
        assert got[i] == _grouped_expected(c, qs[i], 12, 3, wide[i % 5]), ("wide", i)
    one = c.eng.search_batch_grouped_where(qs[:2], 12, 3, wheres[0])
    assert one == [_grouped_expected(c, qs[i], 12, 3, wheres[0]) for i in range(2)]
    c.eng.close()


def test_lifecycle_follows_the_frames():
    c = Corpus(VectorMetric.cosine, 384, n=8_000, seed=13)
    w = [Where(groups=_roots(c, (0, 3))), Where(groups=(4242,))]
    qs = c.queries(8)
    c.check(qs, 10, w, [0, 1] * 4)
    moved = c.ids[5 * GROUP:5 * GROUP + 100]                                 # set_groups re-assigns
    c.eng.set_groups(moved, np.full(moved.size, 4242, np.uint64))
    c.groups[5 * GROUP:5 * GROUP + 100] = 4242
    c.check(qs, 10, w, [0, 1] * 4)
    c.eng.add(int(c.ids[10]), c.vecs[11])                                     # upsert keeps the group
    c.vecs[10] = c.vecs[11]
    c.check(qs, 10, w, [0, 1] * 4)
    gone = c.ids[::7]                                                         # removes
    c.eng.remove_batch(gone)
    keep = ~np.isin(c.ids, gone)
    c.ids, c.vecs, c.ts, c.tags, c.groups = c.ids[keep], c.vecs[keep], c.ts[keep], c.tags[keep], c.groups[keep]
    c.check(qs, 10, w, [0, 1] * 4)
    new = np.arange(1_000_000, 1_000_050, dtype=np.uint64)                    # an appended frame is its own group
    vec = c.rng.standard_normal((50, 384), dtype=np.float32)
    vec /= np.linalg.norm(vec, axis=1, keepdims=True)
    c.eng.add_batch(new, vec)
    c.ids, c.vecs = np.concatenate([c.ids, new]), np.concatenate([c.vecs, vec])
    c.ts, c.tags = np.concatenate([c.ts, np.zeros(50, np.int64)]), np.concatenate([c.tags, np.zeros(50, np.uint64)])
    c.groups = np.concatenate([c.groups, new])
    w2 = w + [Where(groups=(int(new[3]), int(new[7])))]
    c.check(qs, 10, w2, [0, 1, 2] * 2 + [2, 2])
    blob = c.eng.serialize()                                                  # deserialize: every frame its own group
    c.eng.deserialize(blob)
    c.groups = None
    c.ts, c.tags = np.zeros_like(c.ts), np.zeros_like(c.tags)
    c.check(qs, 10, [Where(groups=tuple(int(x) for x in c.ids[:40])), w[0]], [0, 1] * 4)
    c.eng.close()


def test_a_search_concurrent_with_set_groups_sees_old_or_new():
    c = Corpus(VectorMetric.cosine, 384, n=20_000, seed=17)
    w = [Where(groups=(777,))]
    qs = c.queries(4)
    rows = c.ids[:3 * GROUP]
    old = c.eng.search_batch_where(qs, 10, w, [0] * 4)
    assert old == [[]] * 4
    new_groups = c.groups.copy()
    new_groups[:3 * GROUP] = 777
    c.groups = new_groups
    new = c.expected(qs, 10, w, [0] * 4)
    seen = []

    def search():
        for _ in range(20):
            seen.append(c.eng.search_batch_where(qs, 10, w, [0] * 4))
    t = threading.Thread(target=search)
    t.start()
    c.eng.set_groups(rows, np.full(rows.size, 777, np.uint64))
    t.join()
    assert all(s == old or s == new for s in seen)
    assert c.eng.search_batch_where(qs, 10, w, [0] * 4) == new
    c.eng.close()


def test_multi_device_handle_equals_one_engine():
    devices = [i % torch.cuda.device_count() for i in range(2)]
    one = Corpus(VectorMetric.cosine, 384, seed=19)
    multi = Corpus(VectorMetric.cosine, 384, seed=19, devices=devices)
    wheres = _mixed_wheres(one)
    qs = one.queries(64)
    qw = [i % len(wheres) for i in range(64)]
    filters = [("deny", one.ids[::3])]
    qf = [None if i % 2 else 0 for i in range(64)]
    assert multi.eng.search_batch_where(qs, 10, wheres, qw, filters, qf) == one.check(qs, 10, wheres, qw, filters, qf)
    gw = [Where(groups=_roots(one, range(i, 100, 9)), after=200) for i in range(4)]
    assert (multi.eng.search_batch_grouped_multi_where(qs[:16], 12, 3, gw, [i % 4 for i in range(16)]) ==
            one.eng.search_batch_grouped_multi_where(qs[:16], 12, 3, gw, [i % 4 for i in range(16)]))
    gone = one.ids[: N // 3]
    for c in (one, multi):
        c.eng.remove_batch(gone)
    multi.eng.rebalance()
    assert (multi.eng.search_batch_where(qs, 10, wheres, qw) == one.eng.search_batch_where(qs, 10, wheres, qw))
    assert (multi.eng.search_batch_grouped_multi_where(qs[:16], 12, 3, gw, [i % 4 for i in range(16)]) ==
            one.eng.search_batch_grouped_multi_where(qs[:16], 12, 3, gw, [i % 4 for i in range(16)]))
    one.eng.close()
    multi.eng.close()


def _raw(eng, qs, offsets, groups, n_wheres=1, grouped=False, term_offsets=None):
    b = qs.shape[0]
    cap = 30
    ids = np.zeros(b * cap, np.uint64)
    sc = np.zeros(b * cap, np.float32)
    gr = np.zeros(b * cap, np.uint64)
    ns = np.zeros(b, np.uint32)
    wh = (L.WhereNear * n_wheres)(*[Where().to_c_near() for _ in range(n_wheres)])
    qw = np.zeros(b, np.uint32)
    qf = np.full(b, L.NO_FILTER, np.uint32)
    fo = np.zeros(1, np.uint64)
    u64 = C.POINTER(C.c_uint64)
    p = lambda a: None if a is None else a.ctypes.data_as(u64)                # noqa: E731
    head = (eng.handle, qs.ctypes.data_as(C.POINTER(C.c_float)), b, qs.shape[1])
    filt = (None, fo.ctypes.data_as(u64), None, 0, qf.ctypes.data_as(C.POINTER(C.c_uint32)), C.cast(wh, C.c_void_p),
            n_wheres, qw.ctypes.data_as(C.POINTER(C.c_uint32)))
    if grouped:
        return L.lib().wax_vs_search_batch_grouped_multi_where_groups(
            *head, 10, 3, *filt, p(offsets), p(groups), ids.ctypes.data_as(u64), sc.ctypes.data_as(C.POINTER(C.c_float)),
            gr.ctypes.data_as(u64), cap, ns.ctypes.data_as(C.POINTER(C.c_uint32)))
    return L.lib().wax_vs_search_batch_where_groups(
        *head, 10, *filt, p(term_offsets), None, p(offsets), p(groups), ids.ctypes.data_as(u64),
        sc.ctypes.data_as(C.POINTER(C.c_float)), cap, ns.ctypes.data_as(C.POINTER(C.c_uint32)))


@pytest.mark.parametrize("grouped", [False, True])
def test_argument_checks(grouped):
    eng = CUDAVectorEngine(VectorMetric.cosine, 16)                          # empty: the checks come first
    qs = np.ones((2, 16), np.float32)
    g = np.array([5, 6], np.uint64)
    assert _raw(eng, qs, None, g, grouped=grouped) == L.ERR_NULL
    assert _raw(eng, qs, np.array([0, 2], np.uint64), None, grouped=grouped) == L.ERR_NULL
    assert _raw(eng, qs, np.array([1, 2], np.uint64), g, grouped=grouped) == L.ERR_ARGUMENT
    assert _raw(eng, qs, np.array([0, 2, 1], np.uint64), g, n_wheres=2, grouped=grouped) == L.ERR_ARGUMENT
    big = np.arange(65_537, dtype=np.uint64)
    assert _raw(eng, qs, np.array([0, 65_537], np.uint64), big, grouped=grouped) == L.ERR_ARGUMENT
    assert _raw(eng, qs, np.array([0, 65_536], np.uint64), big, grouped=grouped) == L.OK
    assert _raw(eng, qs, np.array([0, 0], np.uint64), None, grouped=grouped) == L.OK   # no group: the plain entry
    if not grouped:
        assert _raw(eng, qs, np.array([0, 2], np.uint64), g, term_offsets=np.array([1, 1], np.uint64)) == L.ERR_ARGUMENT
    eng.close()


def test_full_size_against_the_allow_list_form():
    n, dims, b = 10_000_000, 384, 1024
    eng = CUDAVectorEngine(VectorMetric.cosine, dims)
    eng.fill_synthetic(1, n)
    frames = np.arange(n, dtype=np.uint64)
    roots = frames // GROUP * GROUP
    eng.set_groups(frames, roots)
    rng = np.random.default_rng(23)
    ts = rng.integers(0, 1000, n).astype(np.int64)
    tags = (rng.random(n) < 0.01).astype(np.uint64)
    eng.set_attributes(frames, ts, tags)
    qs = rng.standard_normal((b, dims), dtype=np.float32)
    n_groups = (n + GROUP - 1) // GROUP
    chosen = [rng.choice(n_groups, 8, replace=False) for _ in range(b)]
    wheres = [Where(after=400, before=600, no_tags=DELETED, groups=tuple(int(g) * GROUP for g in ch)) for ch in chosen]
    got = eng.search_batch_where(qs, 10, wheres, list(range(b)))
    allow = []
    for w, ch in zip(wheres, chosen):
        rows = np.concatenate([np.arange(g * GROUP, min((g + 1) * GROUP, n)) for g in ch])
        rows = rows[(ts[rows] >= 400) & (ts[rows] < 600) & (tags[rows] == 0)]
        allow.append(("allow", frames[rows]))
    want = eng.search_batch_multi_filtered(qs, 10, allow, list(range(b)))
    assert got == want
    eng.close()
