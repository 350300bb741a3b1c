"""GPU: grouped search (wax_vs_search_grouped) against the grouped oracle in ACC_F32_TREE mode -- identical ids, group ids,
order and score bits -- plus its equivalences, the group index's life cycle and the argument checks."""
import ctypes as C
import threading

import numpy as np
import pytest

from oracle import grouped as og
from wax_b200 import CUDAVectorEngine, VectorMetric
from wax_b200 import _lib as L

pytestmark = pytest.mark.gpu


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


def make_engine(o, metric, n, dims, seed, groups=None):
    corpus = o.synth_rows(seed, 0, n, dims, normalize=(metric is not VectorMetric.dot))
    ids = np.arange(n, dtype=np.uint64) * 3 + 17                      # frame ids distinct from rows
    eng = CUDAVectorEngine(metric, dims)
    eng.add_batch(ids, corpus)
    if groups is not None:
        assert eng.set_groups(ids, groups) == n
    return eng, corpus, ids


def layouts(n, ids, rng):
    half = ids.copy()
    half[rng.permutation(n)[: n // 2]] = 999_999_999
    return {
        "blocks8": ids[(np.arange(n) // 8) * 8],                      # root = first frame of each block of 8
        "blocks360": ids[(np.arange(n) // 360) * 360],
        "hashed": (np.arange(n, dtype=np.uint64) * 2654435761) % max(n // 8, 1) + 10**12,   # not contiguous
        "half": half,                                                 # skew: one group holds half the rows
    }


@pytest.mark.parametrize("metric", list(VectorMetric))
@pytest.mark.parametrize("dims", [384, 768, 100, 102])          # 102: rows too ragged for TMA, scan_ldg_kernel
def test_grouped_matches_oracle(oracle, metric, dims):
    n = 20_011                                                        # ragged
    rng = np.random.default_rng(dims + metric.value)
    eng, corpus, ids = make_engine(oracle, metric, n, dims, 2100 + dims)
    q = oracle.synth_row(2200 + dims, 0, dims, True)
    for name, groups in layouts(n, ids, rng).items():
        eng.set_groups(ids, groups)
        for top, per in ((12, 1), (12, 3), (5, 128), (1, 1), (400, 8)):
            got = flat(eng.search_grouped(q, top, per_group=per))
            assert got == expect(oracle, metric, corpus, ids, groups, q, top, per), (name, top, per)
    eng.close()


def test_grouped_top_groups_sweep(oracle):
    n, dims = 30_000, 384
    rng = np.random.default_rng(5)
    eng, corpus, ids = make_engine(oracle, VectorMetric.cosine, n, dims, 2300)
    groups = layouts(n, ids, rng)["blocks8"]
    eng.set_groups(ids, groups)
    q = oracle.synth_row(2301, 0, dims, True)
    for top in list(range(1, 33)) + [100, 129, 1000, 3750, 10_000]:   # 3 750 groups exist: more asked than exist
        got = flat(eng.search_grouped(q, top))
        assert got == expect(oracle, VectorMetric.cosine, corpus, ids, groups, q, top, 1), top
    for top, per in ((80, 125), (10_000, 1), (100, 100)):               # products of exactly 10 000
        got = flat(eng.search_grouped(q, top, per_group=per))
        assert got == expect(oracle, VectorMetric.cosine, corpus, ids, groups, q, top, per), (top, per)
    eng.close()


def test_grouped_skew_multi_level_expansion(oracle):
    # one group of 100 000 rows: the expansion needs three levels of tile lists
    n, dims = 200_003, 128
    rng = np.random.default_rng(9)
    eng, corpus, ids = make_engine(oracle, VectorMetric.l2, n, dims, 2400)
    groups = layouts(n, ids, rng)["half"]
    eng.set_groups(ids, groups)
    q = oracle.synth_row(2401, 0, dims, True)
    for top, per in ((5, 128), (78, 128), (3, 2)):
        got = flat(eng.search_grouped(q, top, per_group=per))
        assert got == expect(oracle, VectorMetric.l2, corpus, ids, groups, q, top, per), (top, per)
    eng.close()


def test_grouped_without_groups_equals_search(oracle):
    for metric in VectorMetric:
        n, dims = 25_000, 384
        eng, corpus, ids = make_engine(oracle, metric, n, dims, 2500 + metric.value)
        q = oracle.synth_row(2510, 0, dims, True)
        for k in list(range(1, 33)) + [72, 128, 129, 200, 1000, 10_000]:
            plain = eng.search(q, k)
            got = eng.search_grouped(q, k)
            assert [(f, f) for f, _ in plain] == [(g, hits[0][0]) for g, hits in got], k
            assert all(len(h) == 1 for _, h in got)
            assert np.array_equal(np.float32([s for _, s in plain]).view(np.uint32),
                                  np.float32([h[0][1] for _, h in got]).view(np.uint32)), k
        eng.close()


def test_grouped_filters(oracle):
    n, dims = 40_000, 384
    rng = np.random.default_rng(13)
    eng, corpus, ids = make_engine(oracle, VectorMetric.cosine, n, dims, 2600)
    groups = layouts(n, ids, rng)["blocks8"]
    eng.set_groups(ids, groups)
    q = oracle.synth_row(2601, 0, dims, True)
    allow_rows = np.sort(rng.choice(n, 9_000, replace=False))
    deny_rows = np.sort(rng.choice(n, 20_000, replace=False))
    sub_allow = CUDAVectorEngine(VectorMetric.cosine, dims)             # a corpus of only the allowed rows
    sub_allow.add_batch(ids[allow_rows], corpus[allow_rows])
    sub_allow.set_groups(ids[allow_rows], groups[allow_rows])
    keep = np.setdiff1d(np.arange(n), deny_rows)
    sub_deny = CUDAVectorEngine(VectorMetric.cosine, dims)
    sub_deny.add_batch(ids[keep], corpus[keep])
    sub_deny.set_groups(ids[keep], groups[keep])
    for top, per in ((12, 1), (12, 3), (300, 30)):
        a = eng.search_grouped(q, top, per, allow=np.concatenate([ids[allow_rows], np.uint64([1, 2**62])]))
        assert flat(a) == flat(sub_allow.search_grouped(q, top, per))
        assert flat(a) == expect(oracle, VectorMetric.cosine, corpus, ids, groups, q, top, per, allow_rows)
        d = eng.search_grouped(q, top, per, deny=ids[deny_rows])
        assert flat(d) == flat(sub_deny.search_grouped(q, top, per))
        assert flat(eng.search_grouped(q, top, per, deny=[])) == flat(eng.search_grouped(q, top, per))
    assert eng.search_grouped(q, 5, 2, allow=[]) == []
    assert eng.search_grouped(q, 5, 2, deny=ids) == []
    for e in (eng, sub_allow, sub_deny):
        e.close()


def test_crowding_fixture(oracle):
    """Two videos of 360 segments each sit right next to the query: the 400 best frames hold only those two groups,
    the grouped search still returns 12 distinct groups (VideoRAGOrchestrator.swift:252's over-fetch would not)."""
    n, dims = 50_000, 384
    corpus = oracle.synth_rows(2700, 0, n, dims, normalize=True)
    q = oracle.synth_row(2701, 0, dims, True)
    rng = np.random.default_rng(17)
    crowd = rng.choice(n, 720, replace=False)
    noise = rng.standard_normal((720, dims)).astype(np.float32) * 0.01
    crowd_rows = q[None, :] + noise
    corpus[crowd] = crowd_rows / np.linalg.norm(crowd_rows, axis=1, keepdims=True)
    ids = np.arange(n, dtype=np.uint64) + 1
    groups = ids // 360 * 360 + 10**9                                 # ordinary videos of 360 consecutive frames
    groups[crowd[:360]] = 1
    groups[crowd[360:]] = 2
    eng = CUDAVectorEngine(VectorMetric.cosine, dims)
    eng.add_batch(ids, corpus)
    eng.set_groups(ids, groups)
    over = eng.search(q, 400)
    assert len({int(groups[f - 1]) for f, _ in over}) == 2
    got = eng.search_grouped(q, 12, per_group=3)
    assert len({g for g, _ in got}) == 12 and {1, 2} <= {g for g, _ in got}
    assert flat(got) == expect(oracle, VectorMetric.cosine, corpus, ids, groups, q, 12, 3)
    eng.close()


def test_groups_follow_mutations_and_index_builds(oracle):
    n, dims = 5_000, 128
    eng, corpus, ids = make_engine(oracle, VectorMetric.cosine, n, dims, 2800)
    model_ids, model_rows = list(ids), list(corpus)
    model_groups = dict(zip(ids.tolist(), (ids // 10 * 10).tolist()))
    eng.set_groups(ids, ids // 10 * 10)
    q = oracle.synth_row(2801, 0, dims, True)
    builds = [eng.counter("group_index_builds")]

    def check():
        c = np.stack(model_rows)
        i = np.asarray(model_ids, np.uint64)
        g = np.asarray([model_groups.get(int(x), int(x)) for x in model_ids], np.uint64)
        for top, per in ((7, 1), (7, 4)):
            assert flat(eng.search_grouped(q, top, per)) == expect(oracle, VectorMetric.cosine, c, i, g, q, top, per)
        after = eng.counter("group_index_builds")
        assert after == builds[-1] + 1, "one index build per mutation"
        eng.search_grouped(q, 3, 2)
        assert eng.counter("group_index_builds") == after, "the index is reused between searches"
        builds.append(after)

    check()
    v = oracle.synth_row(2802, 0, dims, True)                         # add: a new frame is its own group
    eng.add(10**6, v); model_ids.append(10**6); model_rows.append(v)
    check()
    w = q + 0.001                                                     # upsert: the frame keeps its group
    eng.add(int(ids[42]), w); model_rows[42] = w.astype(np.float32)
    check()
    eng.remove(int(ids[7])); del model_rows[7]; del model_ids[7]      # remove
    check()
    gone = [int(x) for x in ids[100:400:3]]
    eng.remove_batch(gone)
    keep = [j for j, f in enumerate(model_ids) if f not in set(gone)]
    model_ids = [model_ids[j] for j in keep]; model_rows = [model_rows[j] for j in keep]
    check()
    eng.set_groups(model_ids[:50], [5] * 50)                          # set_groups after the mutations
    model_groups.update({f: 5 for f in model_ids[:50]})
    check()
    blob = eng.serialize()                                            # deserialize: every row its own group again
    eng.deserialize(blob)
    model_groups = {}
    check()
    eng.set_groups(model_ids, [f // 100 for f in model_ids])
    model_groups = {f: f // 100 for f in model_ids}
    check()
    eng.fill_synthetic(2800, n, id_base=17)                           # fill_synthetic: implicit ids, own groups
    model_ids = list(range(17, 17 + n)); model_rows = list(oracle.synth_rows(2800, 0, n, dims, normalize=True))
    model_groups = {}
    check()
    eng.set_groups(model_ids[::2], [7] * len(model_ids[::2]))
    model_groups = {f: 7 for f in model_ids[::2]}
    check()
    eng.close()


def test_concurrent_grouped_searches_share_one_build(oracle):
    n, dims = 100_000, 384
    eng, corpus, ids = make_engine(oracle, VectorMetric.cosine, n, dims, 2900, groups=None)
    eng.set_groups(ids, ids // 24)
    q = oracle.synth_row(2901, 0, dims, True)
    before = eng.counter("group_index_builds")
    results, errors = [None] * 8, []

    def run(i):
        try:
            results[i] = flat(eng.search_grouped(q, 20, per_group=4))
        except Exception as exc:   # surfaced below
            errors.append(exc)

    threads = [threading.Thread(target=run, args=(i,)) for i in range(8)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors
    assert all(r == results[0] for r in results)
    assert eng.counter("group_index_builds") == before + 1
    eng.close()


def test_grouped_argument_checks(oracle):
    dims = 64
    eng = CUDAVectorEngine(VectorMetric.cosine, dims)
    lib, h = L.lib(), eng.handle
    q = np.ones(dims, np.float32)
    ids = np.zeros(16, np.uint64); scores = np.zeros(16, np.float32); grp = np.zeros(16, np.uint64)
    n = C.c_uint32(7)
    f32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    u64 = lambda a: a.ctypes.data_as(C.POINTER(C.c_uint64))

    def call(top=4, per=2, fids=None, nids=0, mode=1, out_ids=ids, out_scores=scores, out_groups=grp, cap=16,
             qlen=dims, out_n=True):
        return lib.wax_vs_search_grouped(h, f32(q), qlen, top, per, fids, nids, mode,
                                         None if out_ids is None else u64(out_ids),
                                         None if out_scores is None else f32(out_scores),
                                         None if out_groups is None else u64(out_groups), cap,
                                         C.byref(n) if out_n else None)

    for engine_state in ("empty", "filled"):                         # checked before the empty-engine return
        assert call(per=0) == L.ERR_ARGUMENT
        assert call(per=129) == L.ERR_ARGUMENT
        assert call(top=5001, per=2) == L.ERR_ARGUMENT
        assert call(top=10**9, per=2) == L.ERR_ARGUMENT               # clamps to 10 000 x 2
        assert call(mode=2) == L.ERR_ARGUMENT
        assert call(mode=-1) == L.ERR_ARGUMENT
        assert call(out_ids=None) == L.ERR_NULL
        assert call(out_scores=None) == L.ERR_NULL
        assert call(out_groups=None) == L.ERR_NULL
        assert call(out_n=False) == L.ERR_NULL
        assert call(nids=3) == L.ERR_NULL
        if engine_state == "empty":
            assert call(qlen=dims + 1) == L.OK and n.value == 0       # as wax_vs_search: empty first
            assert eng.search_grouped(q, 5, 3) == []
            eng.fill_synthetic(3000, 1000)
    assert call(qlen=dims + 1) == L.ERR_DIMENSION
    assert call(top=4, per=5, cap=19) == L.ERR_BUFFER
    assert call(top=4, per=4, cap=16) == L.OK and n.value == 4       # every row is its own group: one row each
    assert call(top=10_000, per=1, cap=999) == L.ERR_BUFFER           # min(10 000, N = 1 000) entries
    big = np.zeros(1000, np.uint64); bs = np.zeros(1000, np.float32); bg = np.zeros(1000, np.uint64)
    assert call(top=10_000, per=1, out_ids=big, out_scores=bs, out_groups=bg, cap=1000) == L.OK and n.value == 1000
    assert lib.wax_vs_set_groups(h, None, None, 0, None) == L.OK
    assert lib.wax_vs_set_groups(h, None, u64(grp), 1, None) == L.ERR_NULL
    assigned = C.c_uint64(9)
    fr = np.array([5, 6, 5, 10**9], np.uint64)                       # repeated and unknown frames
    gr = np.array([1, 2, 3, 4], np.uint64)
    assert lib.wax_vs_set_groups(h, u64(fr), u64(gr), 4, C.byref(assigned)) == L.OK and assigned.value == 2
    res = {f: g for g, hits in eng.search_grouped(q, 10_000) for f, _ in hits}
    assert res[5] == 3 and res[6] == 2 and res[7] == 7               # a later entry wins; unset = own id
    eng.close()


@pytest.mark.parametrize("layout", ["blocks8", "hashed"])
def test_grouped_fullsize_10m(oracle, layout):
    rows, dims = 10_000_000, 384
    eng = CUDAVectorEngine(VectorMetric.cosine, dims)
    eng.fill_synthetic(1, rows)
    r = np.arange(rows, dtype=np.uint64)
    groups = r // 8 * 8 if layout == "blocks8" else (r * 2654435761) % (rows // 8)
    eng.set_groups(r, groups)
    qs = oracle.synth_rows(3100, 0, 4, dims, normalize=True)
    want = og.search_grouped_synth(oracle.COSINE, 1, 0, rows, dims, True, qs, groups, 12, 3, mode=oracle.ACC_F32_TREE,
                                   threads=oracle.host_threads())
    for qi in range(4):
        got = flat(eng.search_grouped(qs[qi], 12, per_group=3))
        wr, _, ws, wg = want[qi]
        assert got == [(int(g), int(f), int(s)) for f, s, g in zip(wr, ws.view(np.uint32), wg)], qi
    eng.close()
