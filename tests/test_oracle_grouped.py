"""The grouped-search oracle (oracle/wax_oracle_grouped.c) against a direct Python restatement of the semantics:
sort every row that takes part by (distance, row), walk the list, keep the first clamp(top_groups) groups met and at
most per_group rows of each."""
import zlib

import numpy as np
import pytest

from oracle import grouped as og
from oracle import oracle as o

N, DIMS = 600, 24


def restated(metric, corpus, query, row_group, top_groups, per_group, allowed_rows=None):
    rows = np.arange(corpus.shape[0]) if allowed_rows is None else np.asarray(sorted(set(allowed_rows)), np.int64)
    if rows.size == 0:
        return [], [], []
    # o.search returns every finite row of the sub-corpus, best first, ties by row (the subset keeps row order)
    r, d, s = o.search(metric, corpus[rows], query, min(rows.size, o.MAX_RESULTS), mode=o.ACC_F32_TREE)
    order, rank = [], {}
    picked = {}
    for sub, score in zip(r.tolist(), s.tolist()):
        row = int(rows[sub])
        g = int(row_group[row])
        if g not in rank:
            if len(order) == o.clamp_topk(top_groups):
                rank[g] = None
                continue
            rank[g] = len(order)
            order.append(g)
            picked[g] = []
        if rank[g] is not None and len(picked[g]) < per_group:
            picked[g].append((row, np.float32(score)))
    out_rows = [row for g in order for row, _ in picked[g]]
    out_scores = [sc for g in order for _, sc in picked[g]]
    out_groups = [g for g in order for _ in picked[g]]
    return out_rows, out_scores, out_groups


def corpus_for(kind, rng):
    c = rng.standard_normal((N, DIMS)).astype(np.float32)
    if kind == "ties":
        c = np.ones((N, DIMS), np.float32)      # every row at the same distance: ranks go by row
    elif kind == "nonfinite":
        c[5] = np.nan
        c[17, 3] = np.inf
        c[40, 0] = -np.inf
    return c


def layout(kind, rng):
    if kind == "singletons":
        return np.arange(N, dtype=np.uint64) + 1000
    if kind == "one":
        return np.full(N, 7, np.uint64)
    if kind == "half":
        g = np.arange(N, dtype=np.uint64) + 5000
        g[rng.permutation(N)[: N // 2]] = 42
        return g
    if kind == "blocks":
        return (np.arange(N, dtype=np.uint64) // 8) * 8
    return rng.integers(0, 37, N).astype(np.uint64) * 1_000_003     # hashed: groups are not contiguous


def check(metric, corpus, query, groups, top_groups, per_group, allowed=None):
    r, d, s, g = og.search_grouped(metric, corpus, query, groups, top_groups, per_group, allowed=allowed,
                                   mode=o.ACC_F32_TREE)
    rows = None if allowed is None else np.flatnonzero(np.asarray(allowed, bool))
    er, es, eg = restated(metric, corpus, query, groups, top_groups, per_group, rows)
    assert r.tolist() == er
    assert g.tolist() == eg
    assert np.array_equal(s.view(np.uint32), np.float32(es).view(np.uint32))
    return r, g


@pytest.mark.parametrize("metric", [o.COSINE, o.DOT, o.L2])
@pytest.mark.parametrize("per_group", [1, 3, 128])
@pytest.mark.parametrize("groups_kind", ["singletons", "one", "half", "blocks", "hashed"])
@pytest.mark.parametrize("top_groups", [4, 10_000])
def test_grouped_oracle_matches_restatement(metric, per_group, groups_kind, top_groups):
    rng = np.random.default_rng(zlib.crc32(repr((metric, per_group, groups_kind, top_groups)).encode()))
    corpus = corpus_for("plain", rng)
    q = rng.standard_normal(DIMS).astype(np.float32)
    groups = layout(groups_kind, rng)
    r, g = check(metric, corpus, q, groups, top_groups, per_group)
    n_groups = len(set(groups.tolist()))
    assert len(dict.fromkeys(g.tolist())) == min(o.clamp_topk(top_groups), n_groups)


@pytest.mark.parametrize("metric", [o.COSINE, o.DOT, o.L2])
@pytest.mark.parametrize("kind", ["ties", "nonfinite"])
@pytest.mark.parametrize("per_group", [1, 3])
def test_grouped_oracle_ties_and_nonfinite(metric, kind, per_group):
    rng = np.random.default_rng(11)
    corpus = corpus_for(kind, rng)
    q = np.ones(DIMS, np.float32) if kind == "ties" else rng.standard_normal(DIMS).astype(np.float32)
    groups = layout("hashed", rng)
    r, _ = check(metric, corpus, q, groups, 9, per_group)
    if kind == "nonfinite":
        assert not {5, 17, 40} & set(r.tolist())
    else:   # exact ties across groups: groups rank by their lowest row, rows ascend within a group
        firsts = {}
        for row in range(N):
            firsts.setdefault(int(groups[row]), row)
        want = sorted(firsts.values())[:9]
        seen = list(dict.fromkeys(int(groups[x]) for x in r.tolist()))
        assert [firsts[gid] for gid in seen] == want


@pytest.mark.parametrize("metric", [o.COSINE, o.L2])
@pytest.mark.parametrize("mode", ["allow", "deny"])
@pytest.mark.parametrize("per_group", [1, 3, 128])
def test_grouped_oracle_filters(metric, mode, per_group):
    rng = np.random.default_rng(3)
    corpus = corpus_for("plain", rng)
    q = rng.standard_normal(DIMS).astype(np.float32)
    groups = layout("blocks", rng)
    listed = rng.permutation(N)[: N // 3]
    allowed = listed if mode == "allow" else np.setdiff1d(np.arange(N), listed)
    mask = np.zeros(N, bool)
    mask[allowed] = True
    r, _ = check(metric, corpus, q, groups, 12, per_group, allowed=mask)
    assert set(r.tolist()) <= set(allowed.tolist())
    # a filtered grouped search equals the unfiltered one over a corpus of only the allowed rows
    keep = np.sort(allowed)
    r2, _, s2, g2 = og.search_grouped(metric, corpus[keep], q, groups[keep], 12, per_group, mode=o.ACC_F32_TREE)
    assert keep[r2.astype(np.int64)].tolist() == r.tolist()


def test_grouped_oracle_singletons_equal_plain_search():
    rng = np.random.default_rng(5)
    corpus = corpus_for("plain", rng)
    q = rng.standard_normal(DIMS).astype(np.float32)
    for k in (1, 7, 32, 200):
        r, d, s, _ = og.search_grouped(o.COSINE, corpus, q, np.arange(N, dtype=np.uint64), k, 1, mode=o.ACC_F32_TREE)
        er, ed, es = o.search(o.COSINE, corpus, q, k, mode=o.ACC_F32_TREE)
        assert r.tolist() == er.tolist() and np.array_equal(s.view(np.uint32), es.view(np.uint32))


def test_grouped_oracle_synth_matches_dense():
    dims, n = 32, 3000
    corpus = o.synth_rows(9, 0, n, dims, normalize=True)
    qs = o.synth_rows(10, 0, 3, dims, normalize=True)
    groups = (np.arange(n, dtype=np.uint64) * 2654435761) % 97
    allowed = np.arange(0, n, 3)
    res = og.search_grouped_synth(o.COSINE, 9, 0, n, dims, True, qs, groups, 10, 3, allowed=allowed,
                                  mode=o.ACC_F32_TREE, threads=3)
    for q in range(3):
        r, d, s, g = og.search_grouped(o.COSINE, corpus, qs[q], groups, 10, 3, allowed=allowed, mode=o.ACC_F32_TREE)
        assert res[q][0].tolist() == r.tolist() and res[q][3].tolist() == g.tolist()
        assert np.array_equal(res[q][2].view(np.uint32), s.view(np.uint32))
