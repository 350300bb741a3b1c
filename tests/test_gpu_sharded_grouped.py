"""GPU: grouped search over the row-sharded engine (DESIGN.md section 4.14) -- round 1 (wax_vs_shard_grouped_heads_device),
merge 1 (wax_vs_merge_group_heads_device), round 2 (wax_vs_shard_grouped_expand_device) and merge 2
(wax_vs_merge_candidates_device).  The ranks are engines on one device; each writes its slice of one all-gather-shaped
buffer pre-filled with a poison byte, so an unwritten slot cannot pass.  Every answer must equal
search_batch_grouped_multi_where on one engine holding the whole corpus: frame ids, group ids, group-major order and
score bits."""
import ctypes as C

import numpy as np
import pytest

from wax_b200 import CUDAVectorEngine, VectorMetric, Where, sharded
from wax_b200 import _lib as L

DELETED = 1 << 0
POISON = 0xAB


def _bits(answer):
    return [(g, [(f, np.float32(s).view(np.uint32).item()) for f, s in hits]) for g, hits in answer]


class Corpus:
    """One corpus with groups, attributes and locations: a single engine and `world` rank engines over its contiguous
    shards, every engine given the full lists (a rank ignores the frames it does not hold)."""

    def __init__(self, oracle, metric, world, n, groups, dims=128, seed=7100, corpus=None):
        rng = np.random.default_rng(seed)
        self.n, self.world, self.metric = n, world, metric
        self.corpus = corpus if corpus is not None else oracle.synth_rows(seed, 0, n, dims,
                                                                          normalize=(metric is not VectorMetric.dot))
        self.ids = np.arange(n, dtype=np.uint64) * 5 + 11
        self.groups = groups
        self.row_groups = groups if groups is not None else self.ids            # unset: every frame its own group
        self.ts = np.arange(n, dtype=np.int64) * 10
        self.tags = np.where(rng.random(n) < 0.05, DELETED, 0).astype(np.uint64)
        lat_c, lon_c = 41.0, 11.0
        self.lat = lat_c + 0.05 * rng.standard_normal(n)
        self.lon = lon_c + 0.05 * rng.standard_normal(n)
        self.centre = (lat_c, lon_c)
        self.single = CUDAVectorEngine(metric, self.corpus.shape[1])
        self.single.add_batch(self.ids, self.corpus)
        self.engines, self.ranges = [], []
        for r in range(world):
            lo, hi = sharded.shard_range(n, world, r)
            eng = CUDAVectorEngine(metric, self.corpus.shape[1])
            if hi > lo:
                eng.add_batch(self.ids[lo:hi], self.corpus[lo:hi])
            self.engines.append(eng)
            self.ranges.append((lo, hi))
        for eng in [self.single] + self.engines:
            if groups is not None:
                eng.set_groups(self.ids, groups)
            eng.set_attributes(self.ids, self.ts, self.tags)
            eng.set_locations(self.ids, self.lat, self.lon)
            if metric is VectorMetric.l2:
                eng.set_option("batch_l2", 1)

    def group_of(self, fid):
        return int(self.row_groups[(int(fid) - 11) // 5])

    def window(self, lo, hi, **kw):
        return Where(after=int(self.ts[lo]), before=int(self.ts[min(hi, self.n - 1)]), **kw)

    def expanded(self):
        return sum(e.counter("shard_grouped_expanded_groups") for e in self.engines)

    def close(self):
        for e in [self.single] + self.engines:
            e.close()


def _answer_of_records(rec, sim):
    """[G][P] records (group-major, padding valid = 0) -> [(group id, [(frame id, score), ...]), ...]."""
    out = []
    for slot in rec:
        hits = [(int(x["frame_id"]), float(s)) for x, s in zip(slot, sharded.score_from_distance(sim, slot["distance"]))
                if x["valid"]]
        if hits:
            out.append((int(slot[0]["group_id"]), hits))
    return out


def _run(c, qs, top_groups, per_group, wheres, qw, filters, qf, check_rounds=True):
    """The whole protocol over the rank engines; checks each rank's round-1 list and, on a few queries, its round-2
    slots; returns the merged answers."""
    import torch
    from wax_b200.engine import _WhereArgs
    b, world, sim = len(qs), c.world, c.metric.to_vec_similarity()
    g, p = min(max(int(top_groups), 1), 10_000), per_group
    a = _WhereArgs(wheres, qw, filters, qf, b)
    d_qs = torch.from_numpy(np.ascontiguousarray(qs, np.float32)).cuda()
    hb = b * g * p * 32
    heads = torch.full((world * hb,), POISON, dtype=torch.uint8, device="cuda")
    for r, eng in enumerate(c.engines):
        rc = L.lib().wax_vs_shard_grouped_heads_device(eng.handle, C.c_void_p(d_qs.data_ptr()), b, top_groups, p,
                                                       *a.filter_args(), *a.where_args(near=True), c.ranges[r][0],
                                                       C.c_void_p(heads.data_ptr() + r * hb), None)
        assert rc == 0, L.last_error()
    torch.cuda.synchronize()
    local = heads.cpu().numpy().view(sharded.GROUP_CAND_DTYPE).reshape(world, b, g, p)
    if check_rounds:
        for r, eng in enumerate(c.engines):
            own = eng.search_batch_grouped_multi_where(qs, top_groups, p, wheres, qw, filters, qf)
            for i in range(b):
                assert _bits(_answer_of_records(local[r, i], sim)) == _bits(own[i]), (r, i)
                lst = local[r, i].reshape(-1)
                assert not lst[lst["valid"] == 0].view(np.uint8).any()            # padding is zeroed
                v = lst[lst["valid"] != 0]
                assert np.all((v["row"] >= c.ranges[r][0]) & (v["row"] < c.ranges[r][1]))
                assert [c.group_of(f) for f in v["frame_id"]] == v["group_id"].tolist()
    chosen = torch.full((b * g * 32,), POISON, dtype=torch.uint8, device="cuda")
    assert L.lib().wax_vs_merge_group_heads_device(c.single.handle, C.c_void_p(heads.data_ptr()), world, b, top_groups, p,
                                                   C.c_void_p(chosen.data_ptr()), None) == 0, L.last_error()
    torch.cuda.synchronize()
    ch = chosen.cpu().numpy().view(sharded.GROUP_CAND_DTYPE).reshape(b, g)
    assert not ch[ch["valid"] == 0].view(np.uint8).any()
    if p == 1:
        return [_answer_of_records(ch[i].reshape(g, 1), sim) for i in range(b)]
    rb = b * g * p * 24
    rows = torch.full((world * rb,), POISON, dtype=torch.uint8, device="cuda")
    for r, eng in enumerate(c.engines):
        rc = L.lib().wax_vs_shard_grouped_expand_device(eng.handle, C.c_void_p(d_qs.data_ptr()), b, top_groups, p,
                                                        *a.filter_args(), *a.where_args(near=True),
                                                        C.c_void_p(chosen.data_ptr()), C.c_void_p(heads.data_ptr() + r * hb),
                                                        c.ranges[r][0], C.c_void_p(rows.data_ptr() + r * rb), None)
        assert rc == 0, L.last_error()
    torch.cuda.synchronize()
    slots = rows.cpu().numpy().view(sharded.CAND_DTYPE).reshape(world, b, g, p)
    if check_rounds:       # a slot = the rank's grouped answer for the query under an allow-list of the group's frames
        for r, eng in enumerate(c.engines):
            for i in range(min(b, 3)):
                for s in range(g):
                    lst = slots[r, i, s]
                    m = int(lst["valid"].sum())
                    assert lst["valid"][:m].all() and not lst[m:].view(np.uint8).any()
                    if not ch[i, s]["valid"]:
                        assert m == 0
                        continue
                    gid = int(ch[i, s]["group_id"])
                    frames = c.ids[c.row_groups == gid]
                    if qf[i] is not None:
                        listed = np.isin(frames, np.asarray(filters[qf[i]][1], np.uint64))
                        frames = frames[listed if filters[qf[i]][0] == "allow" else ~listed]
                    want = eng.search_batch_grouped_multi_where(qs[i:i + 1], 1, p, wheres, qw[i:i + 1],
                                                                [("allow", frames)], [0])[0] if eng.count else []
                    scores = sharded.score_from_distance(sim, lst["distance"][:m])
                    got = [(gid, [(int(f), float(x)) for f, x in zip(lst["frame_id"][:m], scores)])] if m else []
                    assert _bits(got) == _bits(want), (r, i, s)
    merged = torch.zeros(b * g * p * 24, dtype=torch.uint8, device="cuda")
    assert L.lib().wax_vs_merge_candidates_device(c.single.handle, C.c_void_p(rows.data_ptr()), world, b * g, p, p,
                                                  C.c_void_p(merged.data_ptr()), None) == 0, L.last_error()
    torch.cuda.synchronize()
    best = merged.cpu().numpy().view(sharded.CAND_DTYPE).reshape(b, g, p)
    out = []
    for i in range(b):
        ans = []
        for s in range(g):
            if ch[i, s]["valid"]:
                sc = sharded.score_from_distance(sim, best[i, s]["distance"])
                ans.append((int(ch[i, s]["group_id"]), [(int(x["frame_id"]), float(v)) for x, v in zip(best[i, s], sc)
                                                        if x["valid"]]))
        out.append(ans)
    return out


def _shapes(n, world):
    rows = np.arange(n, dtype=np.uint64)
    return {
        "consecutive8": rows // 8,
        "consecutive360": rows // 360 + 1_000_000,
        "hashed": (rows * 2654435761) % 4093 % 500,
        "giant": np.zeros(n, np.uint64),
        "unset": None,
    }


def _filters_and_wheres(c, rng):
    n = c.n
    wheres = [c.window(n // 3, n // 3 + n // 5), Where(no_tags=DELETED),
              Where(near=(c.centre[0], c.centre[1], 3_000.0)), Where(after=10**15)]
    filters = [("allow", c.ids[rng.choice(n, 3000, replace=False)]),           # gather class
               ("allow", c.ids[rng.choice(n, n // 2, replace=False)]),         # tensor class
               ("deny", c.ids[rng.choice(n, n - 100, replace=False)])]         # fewer rows than k_c
    return wheres, filters


def _check(c, oracle, b, top_groups, per_group, seed, check_rounds=True):
    rng = np.random.default_rng(seed)
    qs = oracle.synth_rows(seed, 0, b, c.corpus.shape[1], normalize=True)
    wheres, filters = _filters_and_wheres(c, rng)
    qw = [None if i % 5 == 0 else int(rng.integers(0, len(wheres))) for i in range(b)]
    qf = [None if i % 3 == 0 else int(rng.integers(0, len(filters))) for i in range(b)]
    got = _run(c, qs, top_groups, per_group, wheres, qw, filters, qf, check_rounds)
    want = c.single.search_batch_grouped_multi_where(qs, top_groups, per_group, wheres, qw, filters, qf)
    for i in range(b):
        assert _bits(got[i]) == _bits(want[i]), (i, qw[i], qf[i])
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("metric", [VectorMetric.cosine, VectorMetric.dot, VectorMetric.l2])
@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_sharded_grouped_equals_the_single_engine(oracle, metric, world):
    n = 20_003
    for name, groups in _shapes(n, world).items():
        c = Corpus(oracle, metric, world, n, groups)
        try:
            for top_groups, per_group in ((12, 1), (12, 3)):
                _check(c, oracle, 24, top_groups, per_group, seed=world * 100 + len(name),
                       check_rounds=(name in ("consecutive360", "hashed") and metric is VectorMetric.cosine))
            _check(c, oracle, 1, 5, 4, seed=world, check_rounds=False)                # one query: the single pipeline
        finally:
            c.close()


@pytest.mark.gpu
def test_ties_across_shards_and_short_shards(oracle):
    """Period-256 duplicates, so equal distances sit on every shard; then 8 ranks over 7 rows."""
    dims, n = 64, 3000
    base = oracle.synth_rows(50, 0, 256, dims)
    corpus = np.ascontiguousarray(base[np.arange(n) % 256])
    for groups in (np.arange(n, dtype=np.uint64) // 10, (np.arange(n, dtype=np.uint64) * 7) % 61, None):
        c = Corpus(oracle, VectorMetric.cosine, 4, n, groups, corpus=corpus)
        try:
            for per_group in (1, 3, 20):
                _check(c, oracle, 16, 12, per_group, seed=51 + per_group)
        finally:
            c.close()
    corpus = oracle.synth_rows(51, 0, 7, 128)
    c = Corpus(oracle, VectorMetric.cosine, 8, 7, np.array([0, 0, 1, 1, 1, 2, 0], np.uint64), corpus=corpus)
    try:
        qs = oracle.synth_rows(52, 0, 3, 128, normalize=True)
        for top_groups, per_group in ((1, 1), (3, 2), (10, 4)):
            got = _run(c, qs, top_groups, per_group, [Where()], [None, 0, None], [("allow", c.ids[[0, 2, 6]])],
                       [None, None, 0])
            want = c.single.search_batch_grouped_multi_where(qs, top_groups, per_group, [Where()], [None, 0, None],
                                                             [("allow", c.ids[[0, 2, 6]])], [None, None, 0])
            assert [_bits(x) for x in got] == [_bits(x) for x in want]
    finally:
        c.close()


@pytest.mark.gpu
def test_round_two_scores_only_groups_across_a_boundary(oracle):
    """Consecutive groups cut at the shard boundaries are always listed by the one rank that holds them: round 2 only
    copies.  Groups across a boundary, and hashed groups, are scored on the ranks that did not list them."""
    world, n = 4, 4 * 8 * 700
    aligned = np.arange(n, dtype=np.uint64) // 8
    c = Corpus(oracle, VectorMetric.cosine, world, n, aligned)
    try:
        _check(c, oracle, 40, 12, 3, seed=61, check_rounds=False)
        assert c.expanded() == 0
    finally:
        c.close()
    n = 20_003
    for groups in (np.arange(n, dtype=np.uint64) // 360, (np.arange(n, dtype=np.uint64) * 2654435761) % 4093 % 500):
        c = Corpus(oracle, VectorMetric.cosine, 3, n, groups)
        try:
            _check(c, oracle, 40, 12, 3, seed=62, check_rounds=False)
            assert c.expanded() > 0
        finally:
            c.close()


@pytest.mark.gpu
def test_sharded_engine_world_one_matches_the_single_engine(oracle):
    dims, n = 384, 30_000
    single = CUDAVectorEngine(VectorMetric.cosine, dims)
    single.fill_synthetic(5, n)
    eng = sharded.ShardedVectorEngine(VectorMetric.cosine, dims, total_rows=n)
    try:
        eng.fill_synthetic(5)
        frames = np.arange(n, dtype=np.uint64)
        for e in (single, eng):
            e.set_groups(frames, frames // 6)
            e.set_attributes(frames, frames.astype(np.int64), frames % 4)
        qs = oracle.synth_rows(70, 0, 20, dims, normalize=True)
        wheres = [Where(after=1000, before=15000, no_tags=1), Where(after=5000)]
        filters = [("allow", frames[::7]), ("deny", frames[::3])]
        qw, qf = [i % 3 if i % 3 < 2 else None for i in range(20)], [None if i % 4 == 0 else i % 2 for i in range(20)]
        for per_group in (1, 3):
            got = eng.search_batch_grouped(qs, 12, per_group, wheres, qw, filters, qf)
            assert got == single.search_batch_grouped_multi_where(qs, 12, per_group, wheres, qw, filters, qf)
        assert eng.search_grouped(qs[0], 5, 3) == single.search_grouped(qs[0], 5, 3)
        assert eng.search_grouped(qs[1], 5, 2, where=wheres[0], deny=frames[::3]) == \
            single.search_batch_grouped_multi_where(qs[1:2], 5, 2, wheres, [0], [("deny", frames[::3])], [0])[0]
    finally:
        eng.close()
        single.close()


def test_sharded_grouped_argument_checks():
    """They return before the engine is locked or any CUDA call is made (a placeholder handle stands in for an engine),
    so every rank fails alike before any exchange."""
    eng = C.cast((C.c_uint8 * (1 << 16))(), C.c_void_p)
    off = np.zeros(1, np.uint64)
    qf = np.full(2, L.NO_FILTER, np.uint32)
    buf = C.c_void_p(16)           # never dereferenced: the checks fail first

    def heads(top_groups=12, per_group=3, d_queries=buf, d_out=buf):
        return L.lib().wax_vs_shard_grouped_heads_device(eng, d_queries, 2, top_groups, per_group, None,
                                                         off.ctypes.data_as(C.POINTER(C.c_uint64)), None, 0,
                                                         qf.ctypes.data_as(C.POINTER(C.c_uint32)), None, 0,
                                                         qf.ctypes.data_as(C.POINTER(C.c_uint32)), 0, d_out, None)

    def expand(top_groups=12, per_group=3, chosen=buf):
        return L.lib().wax_vs_shard_grouped_expand_device(eng, buf, 2, top_groups, per_group, None,
                                                          off.ctypes.data_as(C.POINTER(C.c_uint64)), None, 0,
                                                          qf.ctypes.data_as(C.POINTER(C.c_uint32)), None, 0,
                                                          qf.ctypes.data_as(C.POINTER(C.c_uint32)), chosen, buf, 0, buf,
                                                          None)

    def merge(world=2, top_groups=12, per_group=3, gathered=buf):
        return L.lib().wax_vs_merge_group_heads_device(eng, gathered, world, 2, top_groups, per_group, buf, None)

    assert heads(top_groups=257) == L.ERR_UNSUPPORTED and "<= 256" in L.last_error()
    assert expand(top_groups=257) == L.ERR_UNSUPPORTED
    assert merge(top_groups=257) == L.ERR_UNSUPPORTED
    assert heads(per_group=0) == L.ERR_ARGUMENT and expand(per_group=129) == L.ERR_ARGUMENT
    assert merge(per_group=0) == L.ERR_ARGUMENT
    assert heads(d_queries=None) == L.ERR_NULL and heads(d_out=None) == L.ERR_NULL and expand(chosen=None) == L.ERR_NULL
    assert merge(world=0) == L.ERR_ARGUMENT and merge(world=17) == L.ERR_ARGUMENT and merge(gathered=None) == L.ERR_NULL
    bad = np.array([0, 5], np.uint32)          # a query naming a where that does not exist
    assert L.lib().wax_vs_shard_grouped_heads_device(eng, buf, 2, 12, 3, None, off.ctypes.data_as(C.POINTER(C.c_uint64)),
                                                     None, 0, qf.ctypes.data_as(C.POINTER(C.c_uint32)), None, 0,
                                                     bad.ctypes.data_as(C.POINTER(C.c_uint32)), 0, buf, None) \
        == L.ERR_ARGUMENT
