"""GPU: root clauses below the top-k (wax_vs_search_batch_where_roots, wax_vs_search_batch_grouped_multi_where_roots),
PhotoRAG's and VideoRAG's test on each hit's root frame as a predicate on the root-tag word of the row's group.  The
reference allow-list is computed here in numpy -- the frames whose group's word passes the root clause AND pass the
time, tag, location, term and group clauses AND the id filter -- and every answer must be identical (ids, order, score
bits) to the id-filtered search (grouped: search_grouped) under it."""
import ctypes as C
import threading

import numpy as np
import pytest
import torch

from wax_b200 import CUDAVectorEngine, VectorMetric, Where
from wax_b200 import _lib as L

pytestmark = pytest.mark.gpu

N = 40_000
DELETED = 1                                   # a frame's own tag
GROUP = 360                                   # consecutive rows per group, as one video's segments or a photo's regions
IS_ROOT, GONE, SUPERSEDED = 1, 2, 4           # root-tag bits, as the bindings set them from the root's FrameMeta
PHOTO = dict(root_all_tags=IS_ROOT, root_no_tags=GONE | SUPERSEDED)


class Corpus:
    """An engine and the host model of its frames: ids, timestamps, tags, groups (None: implicit), terms, root tags."""

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
        else:                                                                # implicit: each frame is its own group
            self.groups = None
        if self.groups is not None:
            self.eng.set_groups(self.ids, self.groups)
        self.terms = None
        self.words = {}
        gs = np.unique(self.group_of())
        pick = rng.random(gs.size)                                           # 5 % without a word (no meta): IS_ROOT unset
        word = np.where(pick < 0.1, IS_ROOT | SUPERSEDED, np.where(pick < 0.2, IS_ROOT | GONE, IS_ROOT | 8))
        keep = pick >= 0.05
        self.set_root_tags(gs[keep], word[keep].astype(np.uint64))

    def group_of(self):
        return self.ids if self.groups is None else self.groups

    def set_root_tags(self, gids, words):
        got = self.eng.set_root_tags(gids, words)
        for g, w in zip(gids, words):
            self.words[int(g)] = int(w)
        return got

    def word_of(self):
        return np.fromiter((self.words.get(int(g), 0) for g in self.group_of()), np.uint64, self.ids.size)

    def set_terms(self, lists):
        self.terms = lists
        self.eng.set_terms(self.ids, lists)

    def passing(self, where, flt=None, locs=None):
        """Frame ids passing `where` AND the id filter (mode, ids); `locs` the rows inside the where's box."""
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
            if where.near is not None:
                ok &= locs
            if where.has_root_clause:
                w = self.word_of()
                ok &= (w & np.uint64(where.root_all_tags)) == np.uint64(where.root_all_tags)
                ok &= (w & np.uint64(where.root_no_tags)) == 0
        if flt is not None:
            listed = np.isin(self.ids, np.asarray(flt[1], np.uint64))
            ok &= listed if flt[0] in ("allow", 0) else ~listed
        return self.ids[ok]

    def expected(self, qs, k, wheres, qw, filters=(), qf=None, locs=None):
        qf = qf or [None] * len(qs)
        allow = [("allow", self.passing(None if w is None else wheres[w], None if f is None else filters[f], locs))
                 if (w is not None or f is not None) else None for w, f in zip(qw, qf)]
        lists = [a for a in allow if a is not None]
        index, j = [], 0
        for a in allow:
            index.append(None if a is None else j)
            j += a is not None
        return self.eng.search_batch_multi_filtered(qs, k, lists, index)

    def check(self, qs, k, wheres, qw, filters=(), qf=None, locs=None):
        got = self.eng.search_batch_where(qs, k, wheres, qw, list(filters), qf)
        want = self.expected(qs, k, wheres, qw, filters, qf, locs)
        for i, (g, w) in enumerate(zip(got, want)):
            assert g == w, ("query", i)
        return got

    def queries(self, b):
        return self.rng.standard_normal((b, self.vecs.shape[1]), dtype=np.float32)


def _roots(c, idx):
    """The group ids of consecutive groups idx (the root frames' ids)."""
    return tuple(int(c.ids[i * GROUP]) for i in idx)


def _mixed_wheres(c):
    gs = np.unique(c.group_of())
    some = tuple(int(x) for x in gs[:: max(1, gs.size // 9)][:9])
    return [
        Where(**PHOTO),                                                       # the root clause alone
        Where(after=200, before=400, no_tags=DELETED, **PHOTO),               # AND a 20 % window AND not deleted
        Where(root_no_tags=SUPERSEDED),                                       # "no" bits only
        Where(root_all_tags=GONE, root_no_tags=GONE),                         # admits nothing
        Where(root_all_tags=IS_ROOT | SUPERSEDED, after=500),                 # a narrow root set
        Where(groups=some, **PHOTO),                                          # AND a group clause
        Where(after=100, before=900, all_tags=2),                             # no root clause
    ]


@pytest.mark.parametrize("metric,dims,batch_l2", [(VectorMetric.cosine, 384, 0), (VectorMetric.dot, 384, 0),
                                                  (VectorMetric.l2, 384, 0), (VectorMetric.l2, 384, 1),
                                                  (VectorMetric.cosine, 100, 0)])
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


@pytest.mark.parametrize("layout", ["consecutive", "hashed", "implicit"])
def test_group_layouts(layout):
    c = Corpus(VectorMetric.cosine, 384, seed=3, layout=layout)
    wheres = _mixed_wheres(c)
    qs = c.queries(64)
    qw = [i % len(wheres) for i in range(64)]
    for k in (10, 72):
        c.check(qs, k, wheres, qw)
    c.check(qs[:1], 10, wheres, [0])
    c.eng.close()


def test_every_clause_combined_with_the_root_clause():
    c = Corpus(VectorMetric.cosine, 384, seed=5)
    rare = c.rng.random(N) < 0.02
    c.set_terms([[1, 2] if r else [1] for r in rare])                       # term 1 on every row, term 2 on 2 %
    inside = np.arange(N) % 4 == 0
    c.eng.set_locations(c.ids, np.where(inside, 48.85, 10.0), np.full(N, 2.35))
    many = _roots(c, range(0, 100, 2))
    wheres = [Where(terms=(2,), **PHOTO),                                    # a narrow term unit
              Where(terms=(1,), after=100, **PHOTO),                         # a wide term unit
              Where(near=(48.85, 2.35, 5000.0), **PHOTO),                    # a box
              Where(near=(48.85, 2.35, 5000.0), terms=(2,), groups=many, no_tags=DELETED, **PHOTO),
              Where(groups=_roots(c, (0, 3, 5)), **PHOTO),                   # a narrow group unit
              Where(groups=many, after=300, **PHOTO),                        # a wide group unit
              Where(all_tags=4, root_no_tags=SUPERSEDED)]
    qs = c.queries(56)
    qw = [i % len(wheres) for i in range(56)]
    filters = [("allow", c.ids[::2]), ("deny", c.ids[::7])]
    qf = [None if i % 3 == 0 else (i % 2) for i in range(56)]
    for k in (10, 50):
        c.check(qs, k, wheres, qw, locs=inside)
        c.check(qs, k, wheres, qw, filters, qf, locs=inside)
    c.eng.close()


def test_classes_and_the_lazy_column():
    c = Corpus(VectorMetric.cosine, 384, seed=7)
    assert c.eng.counter("root_column_builds") == 0
    c.check(c.queries(4), 10, [Where(after=10)], [0] * 4)                   # no root clause: nothing built
    assert c.eng.counter("root_column_builds") == 0
    narrow = [Where(after=i * 10, before=i * 10 + 30, **PHOTO) for i in range(20)]          # ~1 000 rows: gathered
    wide = [Where(after=i * 10, root_no_tags=SUPERSEDED) for i in range(6)]                 # > 16 384 rows: bitsets
    units = [Where(groups=_roots(c, (i, i + 7)), **PHOTO) for i in range(4)]               # narrow group units
    units += [Where(groups=_roots(c, range(i, 110, 2)), **PHOTO) for i in range(2)]        # wide group units
    wheres = narrow + wide + units
    qs = c.queries(192)
    qw = [i % len(wheres) for i in range(192)]
    passes = c.eng.counter("filter_bitset_passes")                                          # tensor-class sub-batches
    gunits = c.eng.counter("where_group_units")
    c.check(qs, 10, wheres, qw)
    assert c.eng.counter("root_column_builds") == 1
    assert c.eng.counter("where_group_units") - gunits == len(units)
    assert c.eng.counter("filter_bitset_passes") - passes >= 1
    c.eng.set_option("filter_bitset_bytes", 3 * ((N + 31) // 32) * 4)                       # 3 bitsets per pass
    passes = c.eng.counter("filter_bitset_passes")
    c.check(qs, 10, wheres, qw)
    assert c.eng.counter("filter_bitset_passes") - passes >= 2
    assert c.eng.counter("root_column_builds") == 1                                          # kept while nothing changed
    c.eng.close()


def test_a_batch_of_one_takes_the_shadow_route():
    c = Corpus(VectorMetric.cosine, 384, seed=9)
    c.eng.set_option("batch_bf16", 1)
    c.eng.set_option("shadow_scan_min_bytes", 0)
    w = [Where(no_tags=DELETED, **PHOTO)]
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
    own = [Where(after=i * 100, before=i * 100 + 200, **PHOTO) for i in range(8)]
    wheres = own + [Where(groups=tuple(int(x) for x in gs[:16]), **PHOTO),
                    Where(root_all_tags=GONE, root_no_tags=GONE),                           # admits nothing
                    Where(groups=(int(gs[0]),), root_no_tags=SUPERSEDED)]                   # a crowded query
    qs = c.queries(48)
    qw = [i % len(wheres) for i in range(48)]
    filters = [("deny", c.ids[::4]), ("allow", c.ids[::2])]
    qf = [None if i % 3 else (i // 3) % 2 for i in range(48)]
    live = {int(g) for g in gs if (c.words.get(int(g), 0) & (GONE | SUPERSEDED | IS_ROOT)) == IS_ROOT}
    for g, p in ((12, 3), (5, 1), (3, 40)):
        got = c.eng.search_batch_grouped_multi_where(qs, g, p, wheres, qw, filters, qf)
        for i in range(48):
            flt = None if qf[i] is None else filters[qf[i]]
            want = _grouped_expected(c, qs[i], g, p, wheres[qw[i]], flt)
            assert got[i] == want, (g, p, i)
            if qw[i] < 8 and qf[i] is None:                                 # PhotoRAG's case: never short, never stale
                assert len(got[i]) == g and all(grp in live for grp, _ in got[i])
    one = c.eng.search_batch_grouped_where(qs[:1], 12, 3, wheres[0])
    assert one == [_grouped_expected(c, qs[0], 12, 3, wheres[0])]
    two = c.eng.search_batch_grouped_where(qs[:2], 12, 3, wheres[1], deny=c.ids[::4])
    assert two == [_grouped_expected(c, qs[i], 12, 3, wheres[1], ("deny", c.ids[::4])) for i in range(2)]
    c.eng.close()


def test_lifecycle_keeps_the_tags_by_group():
    c = Corpus(VectorMetric.cosine, 384, n=8_000, seed=13)
    w = [Where(**PHOTO), Where(groups=(4242, 4343), root_no_tags=GONE), Where(root_all_tags=16)]
    qs = c.queries(8)
    qw = [0, 1, 2, 0, 1, 2, 0, 0]
    c.check(qs, 10, w, qw)
    assert c.set_root_tags([4242, 4242, 16, 4343], np.array([GONE, 16, 16, 16], np.uint64)) == 3   # tags before rows
    c.check(qs, 10, w, qw)                                                    # a later entry for the same id wins
    moved = c.ids[5 * GROUP:5 * GROUP + 100]                                  # set_groups moves rows into 4242
    c.eng.set_groups(moved, np.full(moved.size, 4242, np.uint64))
    c.groups[5 * GROUP:5 * GROUP + 100] = 4242
    c.check(qs, 10, w, qw)
    first = _roots(c, (0, 1, 2))                                              # upserts of the words
    c.set_root_tags(first, np.array([IS_ROOT | SUPERSEDED, IS_ROOT, 0], np.uint64))
    c.check(qs, 10, w, qw)
    c.eng.add(int(c.ids[10]), c.vecs[11])                                     # an upserted row keeps its group's word
    c.vecs[10] = c.vecs[11]
    c.check(qs, 10, w, qw)
    gone = c.ids[::7]                                                         # removes
    c.eng.remove_batch(gone)
    keep = ~np.isin(c.ids, gone)
    c.ids, c.vecs, c.ts, c.tags, c.groups = c.ids[keep], c.vecs[keep], c.ts[keep], c.tags[keep], c.groups[keep]
    c.check(qs, 10, w, qw)
    new = np.arange(1_000_000, 1_000_050, dtype=np.uint64)                    # appended frames: their own groups
    vec = c.rng.standard_normal((50, 384), dtype=np.float32)
    vec /= np.linalg.norm(vec, axis=1, keepdims=True)
    c.set_root_tags(new[:10], np.full(10, IS_ROOT, np.uint64))                # given before the frames arrive
    c.eng.add_batch(new, vec)
    c.ids, c.vecs = np.concatenate([c.ids, new]), np.concatenate([c.vecs, vec])
    c.ts, c.tags = np.concatenate([c.ts, np.zeros(50, np.int64)]), np.concatenate([c.tags, np.zeros(50, np.uint64)])
    c.groups = np.concatenate([c.groups, new])
    c.check(qs, 10, w, qw)
    blob = c.eng.serialize()                                                  # deserialize clears the words
    c.eng.deserialize(blob)
    c.groups = None
    c.ts, c.tags = np.zeros_like(c.ts), np.zeros_like(c.tags)
    c.words = {}
    c.check(qs, 10, w + [Where(root_no_tags=IS_ROOT)], qw[:7] + [3])
    assert c.eng.search_batch_where(qs, 10, [Where(**PHOTO)], [0] * 8) == [[]] * 8
    c.eng.close()


def test_a_search_concurrent_with_set_root_tags_sees_old_or_new():
    c = Corpus(VectorMetric.cosine, 384, n=20_000, seed=17)
    w = [Where(**PHOTO)]
    qs = c.queries(4)
    old = c.check(qs, 10, w, [0] * 4)
    flip = np.unique(c.group_of())[::2]
    before = dict(c.words)
    for g in flip:
        c.words[int(g)] = IS_ROOT | SUPERSEDED
    new = c.expected(qs, 10, w, [0] * 4)
    c.words = before
    assert new != old
    seen = []

    def search():
        for _ in range(20):
            seen.append(c.eng.search_batch_where(qs, 10, w, [0] * 4))
    t = threading.Thread(target=search)
    t.start()
    c.set_root_tags(flip, np.full(flip.size, IS_ROOT | SUPERSEDED, np.uint64))
    t.join()
    assert all(s == old or s == new for s in seen)
    assert c.eng.search_batch_where(qs, 10, w, [0] * 4) == new
    c.eng.close()


def test_multi_device_handle_equals_one_engine():
    devices = [i % torch.cuda.device_count() for i in range(2)]
    one = Corpus(VectorMetric.cosine, 384, seed=19)
    multi = Corpus(VectorMetric.cosine, 384, seed=19, devices=devices)
    gs = np.unique(one.group_of())
    assert multi.eng.set_root_tags(gs[:5], np.full(5, IS_ROOT, np.uint64)) == \
        one.eng.set_root_tags(gs[:5], np.full(5, IS_ROOT, np.uint64)) == 5                 # one engine's count
    wheres = _mixed_wheres(one)
    qs = one.queries(64)
    qw = [i % len(wheres) for i in range(64)]
    filters = [("deny", one.ids[::3])]
    qf = [None if i % 2 else 0 for i in range(64)]
    assert multi.eng.search_batch_where(qs, 10, wheres, qw, filters, qf) == one.eng.search_batch_where(
        qs, 10, wheres, qw, filters, qf)
    gw = [Where(after=i * 200, before=i * 200 + 300, **PHOTO) for i in range(4)]
    assert (multi.eng.search_batch_grouped_multi_where(qs[:16], 12, 3, gw, [i % 4 for i in range(16)]) ==
            one.eng.search_batch_grouped_multi_where(qs[:16], 12, 3, gw, [i % 4 for i in range(16)]))
    gone = one.ids[: N // 3]
    for c in (one, multi):
        c.eng.remove_batch(gone)
    multi.eng.rebalance()
    assert multi.eng.search_batch_where(qs, 10, wheres, qw) == one.eng.search_batch_where(qs, 10, wheres, qw)
    assert (multi.eng.search_batch_grouped_multi_where(qs[:16], 12, 3, gw, [i % 4 for i in range(16)]) ==
            one.eng.search_batch_grouped_multi_where(qs[:16], 12, 3, gw, [i % 4 for i in range(16)]))
    for c in (one, multi):
        c.eng.set_root_tags(gs[::3], np.full(gs[::3].size, IS_ROOT | GONE, np.uint64))
    assert multi.eng.search_batch_where(qs, 10, wheres, qw) == one.eng.search_batch_where(qs, 10, wheres, qw)
    one.eng.close()
    multi.eng.close()


def _raw(eng, qs, roots, offsets=np.zeros(2, np.uint64), grouped=False, term_offsets=None):
    b = qs.shape[0]
    cap = 30
    ids = np.zeros(b * cap, np.uint64)
    sc = np.zeros(b * cap, np.float32)
    gr = np.zeros(b * cap, np.uint64)
    ns = np.zeros(b, np.uint32)
    wh = (L.WhereNear * 1)(Where().to_c_near())
    qw = np.zeros(b, np.uint32)
    qf = np.full(b, L.NO_FILTER, np.uint32)
    fo = np.zeros(1, np.uint64)
    u64 = C.POINTER(C.c_uint64)
    p = lambda a: None if a is None else a.ctypes.data_as(u64)                # noqa: E731
    rc = None if roots is None else C.cast((L.RootClause * 1)(L.RootClause(*roots)), C.c_void_p)
    head = (eng.handle, qs.ctypes.data_as(C.POINTER(C.c_float)), b, qs.shape[1])
    filt = (None, fo.ctypes.data_as(u64), None, 0, qf.ctypes.data_as(C.POINTER(C.c_uint32)), C.cast(wh, C.c_void_p), 1,
            qw.ctypes.data_as(C.POINTER(C.c_uint32)))
    if grouped:
        return L.lib().wax_vs_search_batch_grouped_multi_where_roots(
            *head, 10, 3, *filt, p(offsets), None, rc, ids.ctypes.data_as(u64), sc.ctypes.data_as(C.POINTER(C.c_float)),
            gr.ctypes.data_as(u64), cap, ns.ctypes.data_as(C.POINTER(C.c_uint32)))
    return L.lib().wax_vs_search_batch_where_roots(
        *head, 10, *filt, p(term_offsets), None, p(offsets), None, rc, ids.ctypes.data_as(u64),
        sc.ctypes.data_as(C.POINTER(C.c_float)), cap, ns.ctypes.data_as(C.POINTER(C.c_uint32)))


@pytest.mark.parametrize("grouped", [False, True])
def test_argument_checks(grouped):
    eng = CUDAVectorEngine(VectorMetric.cosine, 16)                          # empty: the checks come first
    qs = np.ones((2, 16), np.float32)
    assert _raw(eng, qs, (1, 2), offsets=None, grouped=grouped) == L.ERR_NULL
    assert _raw(eng, qs, (1, 2), offsets=np.array([1, 1], np.uint64), grouped=grouped) == L.ERR_ARGUMENT
    assert _raw(eng, qs, (1, 2), offsets=np.array([0, 2], np.uint64), grouped=grouped) == L.ERR_NULL   # ids NULL
    assert _raw(eng, qs, (1, 2), grouped=grouped) == L.OK
    assert _raw(eng, qs, (0, 0), grouped=grouped) == L.OK                   # no root clause: the _groups entry
    assert _raw(eng, qs, None, grouped=grouped) == L.OK
    if not grouped:
        assert _raw(eng, qs, (1, 2), term_offsets=np.array([1, 1], np.uint64)) == L.ERR_ARGUMENT
    with pytest.raises(ValueError):
        eng.set_root_tags([1, 2], [3])
    assert eng.set_root_tags([], []) == 0
    g = (C.c_uint64 * 1)(5)
    assert L.lib().wax_vs_set_root_tags(eng.handle, None, g, 1, None) == L.ERR_NULL
    assert L.lib().wax_vs_set_root_tags(eng.handle, g, None, 1, None) == L.ERR_NULL
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
    eng.set_attributes(frames, ts, None)
    gs = np.arange(0, n, GROUP, dtype=np.uint64)
    u = rng.random(gs.size)
    words = np.where(u < 0.02, IS_ROOT | SUPERSEDED, np.where(u < 0.03, IS_ROOT | GONE,
                                                              np.where(u < 0.035, 0, IS_ROOT))).astype(np.uint64)
    eng.set_root_tags(gs, words)
    qs = rng.standard_normal((b, dims), dtype=np.float32)
    wheres = [Where(after=i % 800, before=i % 800 + 200, **PHOTO) for i in range(b)]
    got = eng.search_batch_where(qs, 10, wheres, list(range(b)))
    live_row = words[frames // GROUP] == IS_ROOT
    allow = [("allow", frames[live_row & (ts >= w.after) & (ts < w.before)]) for w in wheres[:8]]
    want = eng.search_batch_multi_filtered(qs[:8], 10, allow, list(range(8)))
    assert got[:8] == want
    got = eng.search_batch_where(qs, 10, [Where(**PHOTO)], [0] * b)
    want = eng.search_batch_multi_filtered(qs, 10, [("allow", frames[live_row])], [0] * b)
    assert got == want
    eng.close()
