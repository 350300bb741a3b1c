"""GPU: l2 batches on the tensor-core levels (option `batch_l2` = 1).  The nomination score is score' = q.v - |v|^2 / 2
(|q - v|^2 = |q|^2 - 2 score', so the heaps and thresholds work unchanged); the exact re-score and the l2 proof
(`l2_proof` in waxvs_batch.cuh) must make every answer identical to the single-query path -- same ids, same score bits."""
import ctypes as C
import zlib

import numpy as np
import pytest

from test_gpu_nomination import BF16_EPS, FORMS, TF32_EPS, _check_heaps, _data, _hidden_winner, _unit
from wax_b200 import CUDAVectorEngine, VectorMetric, sharded

pytestmark = pytest.mark.gpu

L2 = VectorMetric.l2


def _engine(corpus, **opts):
    eng = CUDAVectorEngine(L2, corpus.shape[1])
    eng.add_batch(list(range(corpus.shape[0])), corpus)
    eng.set_option("batch_l2", 1)
    for key, value in opts.items():
        eng.set_option(key, value)
    return eng


def _loop(eng, qs, k):
    eng.set_option("batch_tensor", 0)
    out = [eng.search(q, k) for q in qs]
    eng.set_option("batch_tensor", 1)
    return out


def _corpus(oracle, kind, n, dims, seed):
    if kind == "unit":
        return oracle.synth_rows(seed, 0, n, dims, normalize=True)
    if kind == "unnormalised":
        return oracle.synth_rows(seed, 0, n, dims, normalize=False)
    assert kind == "mixed"          # norms spread over 1e-3 .. 1e3
    c = oracle.synth_rows(seed, 0, n, dims, normalize=True)
    return c * np.float32(10.0) ** np.random.default_rng(seed).uniform(-3, 3, (n, 1)).astype(np.float32)


@pytest.mark.parametrize("dims,n,b,k", [(384, 100_003, 5, 10), (384, 100_003, 129, 10), (384, 50_000, 300, 72),
                                        (768, 30_001, 64, 100), (128, 70_000, 17, 32), (32, 9_999, 8, 1),
                                        (384, 255, 6, 10), (384, 257, 6, 10), (384, 1, 4, 10), (1024, 20_000, 33, 10)])
@pytest.mark.parametrize("kind", ["unit", "unnormalised", "mixed"])
@pytest.mark.parametrize("bf16", [1, 0])
def test_l2_batch_equals_single_query_path(oracle, kind, dims, n, b, k, bf16):
    corpus = _corpus(oracle, kind, n, dims, seed=1900 + dims)
    eng = _engine(corpus, batch_bf16=bf16)
    qs = oracle.synth_rows(1901 + b, 0, b, dims, normalize=True)
    t0, f0 = eng.batch_stats()
    got = eng.search_batch(qs, k)
    t1, f1 = eng.batch_stats()
    assert (t1 - t0) + (f1 - f0) == b, "the batch did not go through the tensor path"
    assert got == _loop(eng, qs, k)
    # unit rows: |q| max|v| = 1, the bound is as tight as for cosine and (nearly) every query is proven or filtered.
    # Elsewhere a large max|v| can make E_M exceed the distance gaps, and the exact scan answers: equality is the claim.
    if kind == "unit" and n >= 1000:
        assert f1 - f0 <= max(1, b // 50), f"{f1 - f0} of {b} queries fell back to the exact path"
    r, _, s = oracle.search(oracle.L2, corpus, qs[0], k, mode=oracle.ACC_F32_TREE, threads=4)
    assert [g[0] for g in got[0]] == r.tolist()
    assert np.array_equal(np.float32([g[1] for g in got[0]]).view(np.uint32), s.view(np.uint32))


@pytest.mark.parametrize("pair,ares", [(0, 1), (0, 0), (1, 1), (1, 0)])
@pytest.mark.parametrize("dims,n,b,k", [(384, 100_003, 300, 10), (384, 150_000, 130, 200), (768, 70_000, 9, 1000)])
def test_l2_kernel_forms_and_large_k_equal_single_query_path(oracle, dims, n, b, k, pair, ares):
    """Resident or streamed queries, single CTA or CTA pair (bf16), and the TF32 pair form; k = 200 and 1 000 take the
    large-k shape (64-entry heaps, 1 024 nominees re-scored).  On these unit rows level 1 still proves k = 200; k = 1 000
    needs the filter level."""
    corpus = _corpus(oracle, "unit", n, dims, seed=2000 + dims)
    eng = _engine(corpus, batch_pair=pair, batch_ares=ares)
    qs = oracle.synth_rows(2001 + b, 0, b, dims, normalize=True)
    for bf16 in (1, 0):
        eng.set_option("batch_bf16", bf16)
        t0, f0 = eng.batch_stats()
        filt0 = eng.counter("batch_retry_queries") + eng.counter("batch_filter_bf16_queries")
        got = eng.search_batch(qs, k)
        t1, f1 = eng.batch_stats()
        assert (t1 - t0) + (f1 - f0) == b, "the batch did not take the tensor-core levels"
        assert f1 - f0 <= max(1, b // 20), f"{f1 - f0} of {b} queries fell back to the exact scan"
        if k >= 1000:
            assert eng.counter("batch_retry_queries") + eng.counter("batch_filter_bf16_queries") > filt0
        sample = sorted(set(range(0, b, max(1, b // 12))) | {b - 1})
        want = _loop(eng, qs[sample], k)
        assert [got[i] for i in sample] == want


def _l2_bound(eps, qn, vn, dims):
    """E(|v|) of the l2 proof: the nomination error of score' against q.v - |v|^2 / 2."""
    return (1.01 * eps + (dims + 1) * 2.0 ** -23) * qn * vn + (dims + 2) * 2.0 ** -24 * vn * vn


def _measure(eng, corpus, qs, k=10, allowed=None):
    n, dims = corpus.shape
    d = eng.batch_nominations(qs, k, allow_rows=None if allowed is None else np.flatnonzero(allowed))
    scores = d["scores"]
    assert not np.any(scores.view(np.uint32) == 0xFFFFFFFF), "some (query, row) score' was never written"
    c64, q64 = corpus.astype(np.float64), qs.astype(np.float64)
    vn, qn = np.linalg.norm(c64, axis=1), np.linalg.norm(q64, axis=1)
    ref = q64 @ c64.T - 0.5 * (vn * vn)[None, :]
    eps = BF16_EPS if d["bf16"] else TF32_EPS
    err = np.abs(scores.astype(np.float64) - ref)
    bound = _l2_bound(eps, qn[:, None], vn[None, :], dims)
    bad = ~(err <= bound)
    assert not bad.any(), (f"score' outside the l2 bound for {bad.sum()} entries; worst error / bound "
                           f"{np.max(err / bound):.3f} at {np.unravel_index(np.argmax(err / bound), err.shape)}")
    _check_heaps(d, n, qs.shape[0], allowed)
    return d, float(np.max(err / bound))


L2_COMBOS = [("unit", 0, 1, 4), ("mixed", 1, 127, 129), ("dot", 0, 128, 127), ("worst", 1, 129, 300),
             ("worst", 0, 3077, 300), ("dot", 0, 20_077, 129)]


@pytest.mark.parametrize("name,opts,dims", FORMS, ids=[f[0] for f in FORMS])
def test_l2_nomination_scores_stay_within_the_proof_bound(name, opts, dims):
    """Every form's l2 score' against fp64 q.v - |v|^2 / 2 at every (query, row), within E(|v|); heaps against the
    scores.  "dot" data are un-normalised rows and queries, "worst" the all-one-sign rounding corpus."""
    rng = np.random.default_rng(zlib.crc32(("l2" + name).encode()))
    ratios = {}
    for kind, di, n, b in L2_COMBOS:
        corpus, qs = _data(kind, rng, n, b, dims[di])
        eng = _engine(corpus, **opts)
        d, ratio = _measure(eng, corpus, qs)
        eng.close()
        assert d["bf16"] == opts["batch_bf16"] and d["kprime"] == opts["batch_heap"]
        ratios[(kind, dims[di], n, b)] = ratio
    print(f"\n[l2 nomination bound] {name}: largest error / E(|v|) = {max(ratios.values()):.4f} "
          f"(worst-case corpus {max(v for key, v in ratios.items() if key[0] == 'worst'):.4f})")


def test_l2_near_duplicates_and_offset_cluster_stay_exact(oracle):
    """Thousands of rows within 1e-6 of the best match (no bound separates them), and a cluster far from the origin
    (|c| = 50, noise ~ 1: E_M ~ eps |q| M dwarfs the gaps, the read-out's proof flags are all 0): exact answers."""
    dims, n = 384, 20_000
    rng = np.random.default_rng(3)
    base = oracle.synth_row(77, 0, dims, True)
    corpus = oracle.synth_rows(78, 0, n, dims)
    corpus[:3000] = base + rng.standard_normal((3000, dims)).astype(np.float32) * np.float32(1e-6)
    eng = _engine(corpus)
    qs = np.stack([base, oracle.synth_row(79, 0, dims, True), base * np.float32(2.5), corpus[5000]])
    got = eng.search_batch(qs, 10)
    assert got == _loop(eng, qs, 10)
    r, _, s = oracle.search(oracle.L2, corpus, qs[0], 10, mode=oracle.ACC_F32_TREE, threads=4)
    assert [g[0] for g in got[0]] == r.tolist()
    eng.close()
    c = rng.standard_normal(dims)
    offset = (50.0 * c / np.linalg.norm(c) + rng.standard_normal((n, dims)) / np.sqrt(dims)).astype(np.float32)
    qs = (offset[rng.integers(0, n, 40)] + 0.3 * rng.standard_normal((40, dims)) / np.sqrt(dims)).astype(np.float32)
    for bf16 in (1, 0):
        eng = _engine(offset, batch_bf16=bf16)
        assert eng.batch_nominations(qs, 10)["ok"].sum() == 0
        got = eng.search_batch(qs, 10)
        assert got == _loop(eng, qs, 10)
        r, _, s = oracle.search(oracle.L2, offset, qs[0], 10, mode=oracle.ACC_F32_TREE, threads=4)
        assert [g[0] for g in got[0]] == r.tolist()
        eng.close()


@pytest.mark.parametrize("bf16", [1, 0])
def test_l2_proof_refuses_a_hidden_winner(bf16):
    """The dot hidden-winner rows with the query scaled by 2^6 (exact): the l2 order is then the dot order (the decoys'
    q.v deficit outweighs their |v|^2 / 2 differences), row 0 is the nearest row, and its score' rounds below 24
    decoys of its slice.  Level 1 must not prove that query; the batch still answers exactly."""
    rng = np.random.default_rng(31 + bf16)
    dims, n = 256, 6_000
    q, corpus = _hidden_winner(rng, dims, n, bf16, n_decoys=24)
    q = q * np.float32(64.0)
    qs = np.concatenate([q, _unit(rng, 5, dims)])
    eng = _engine(corpus, batch_bf16=bf16, batch_heap=16, batch_ares=0)
    d, _ = _measure(eng, corpus, qs, k=1)
    sc = d["scores"][0]
    dist = np.sum((corpus.astype(np.float64) - q[0].astype(np.float64)) ** 2, axis=1)
    assert np.argmin(dist) == 0 and np.sum(sc[1:25] > sc[0]) == 24, "the construction did not hide the winner"
    assert not _check_heaps(d, n, qs.shape[0])[0, 0], "the hidden winner was nominated after all"
    assert d["ok"][0] == 0, "level 1 claimed a proof for a query whose best row it never nominated"
    got = eng.search_batch(qs, 1)
    assert got == _loop(eng, qs, 1) and got[0][0][0] == 0
    eng.close()


@pytest.mark.parametrize("bf16", [1, 0])
def test_l2_edge_rows_and_a_row_whose_norm_overflows(oracle, bf16):
    """Zero, NaN and +-inf rows, and a finite row with |v| ~ 1e20 (its fp32 sum v^2 overflows: w = inf, score' = -inf)
    queried by itself: it must come back first, and max|v| makes every proof of the batch refuse."""
    dims, n = 384, 20_000
    corpus = oracle.synth_rows(90, 0, n, dims)
    corpus[7] = 0.0
    corpus[8, 5] = np.nan
    corpus[9, 6] = np.inf
    corpus[10, 3] = -np.inf
    corpus[11] = corpus[11] * np.float32(1e20)
    with np.errstate(over="ignore"):
        assert np.isinf(np.sum(corpus[11] ** 2, dtype=np.float32)) and np.isfinite(corpus[11]).all()
    qs = np.concatenate([corpus[11:12], oracle.synth_rows(91, 0, 7, dims), corpus[7:8]])
    eng = _engine(corpus, batch_bf16=bf16)
    assert eng.batch_nominations(qs, 10)["ok"].sum() == 0
    got = eng.search_batch(qs, 10)
    assert got == _loop(eng, qs, 10)
    assert got[0][0][0] == 11 and got[-1][0][0] == 7
    assert all(i not in (8, 9, 10) for hits in got for i, _ in hits)
    eng.close()


def test_l2_caches_follow_appends_and_mutations(oracle):
    """|v|^2 / 2 is cached with the norms: an append extends the cache (norms_rows follows the row count), overwriting
    a row with a larger norm and removing rows rebuild it; every answer equals the loop."""
    dims, n = 384, 6_000
    corpus = oracle.synth_rows(95, 0, n, dims)
    eng = _engine(corpus)
    qs = oracle.synth_rows(96, 0, 8, dims)
    assert eng.search_batch(qs, 10) == _loop(eng, qs, 10)
    assert eng.counter("norms_rows") == n
    eng.add_batch([7000, 7001], np.stack([qs[0], qs[1]]))                         # append
    got = eng.search_batch(qs, 10)
    assert eng.counter("norms_rows") == n + 2
    assert got == _loop(eng, qs, 10) and got[0][0][0] == 7000
    eng.add(11, corpus[11] * np.float32(1000.0))                                  # overwrite: larger norm
    assert eng.batch_nominations(qs, 10)["ok"].sum() == 0                        # max|v| = 1000 now
    assert eng.search_batch(qs, 10) == _loop(eng, qs, 10)
    eng.remove(3)
    eng.remove(11)
    got = eng.search_batch(qs, 10)
    assert got == _loop(eng, qs, 10)
    assert eng.counter("norms_rows") == n + 2 - 2                                 # rebuilt from the removed row on
    eng.close()


def test_l2_batched_filtered_search_equals_the_per_query_filtered_search(oracle):
    """One filter, a batch: small allow-lists take the gather, large allow- and deny-lists the tensor-core levels with
    the row filter below the top-k; every answer equals the per-query filtered search."""
    n, dims, b = 80_000, 384, 130
    rng = np.random.default_rng(23)
    corpus = oracle.synth_rows(1500, 0, n, dims, normalize=True)
    ids = (np.arange(n, dtype=np.uint64) * 3 + 77)
    eng = CUDAVectorEngine(L2, dims)
    eng.add_batch(ids, corpus)
    eng.set_option("batch_l2", 1)
    qs = oracle.synth_rows(1501, 0, b, dims, normalize=True)
    cases = [("allow", rng.choice(n, 700, replace=False)), ("allow", rng.choice(n, 40_000, replace=False)),
             ("deny", rng.choice(n, 50_000, replace=False))]
    for kind, rows in cases:
        for k in (10, 72):
            kw = {kind: ids[rows]}
            t0, f0 = eng.batch_stats()
            got = eng.search_batch_filtered(qs, k, **kw)
            t1, f1 = eng.batch_stats()
            eng.set_option("batch_tensor", 0)
            assert all(got[qi] == eng.search_filtered(qs[qi], k, **kw) for qi in range(0, b, 9)), (kind, len(rows), k)
            eng.set_option("batch_tensor", 1)
            if len(rows) > 16_384:
                assert (t1 - t0) + (f1 - f0) == b, "a large filtered batch must take the tensor-core levels"
                assert f1 - f0 <= 3, f"{f1 - f0} of {b} filtered queries fell back to the exact scan"
    eng.close()


def test_l2_device_batch_with_a_row_offset_returns_the_loop_candidates(oracle):
    """wax_vs_search_batch_device (the sharded engine's search_batch) with row_offset != 0: the tensor-core levels
    return the candidates the single-query loop returns."""
    import torch
    from wax_b200 import _lib as L
    dims, n, b, k, offset = 384, 50_000, 140, 10, 1_000_000
    eng = _engine(oracle.synth_rows(97, 0, n, dims))
    d_qs = torch.from_numpy(oracle.synth_rows(98, 0, b, dims)).cuda()

    def run():
        buf = torch.zeros(b * k * 24, dtype=torch.uint8, device="cuda")
        rc = L.lib().wax_vs_search_batch_device(eng.handle, C.c_void_p(d_qs.data_ptr()), b, k, offset,
                                                C.c_void_p(buf.data_ptr()), C.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == 0, L.last_error()
        torch.cuda.synchronize()
        return buf.cpu().numpy().view(sharded.CAND_DTYPE).copy()

    t0, f0 = eng.batch_stats()
    got = run()
    t1, f1 = eng.batch_stats()
    assert (t1 - t0) + (f1 - f0) == b and f1 - f0 <= 2
    eng.set_option("batch_tensor", 0)
    want = run()
    for f in ("valid", "row", "frame_id"):
        assert np.array_equal(got[f], want[f]), f
    assert np.array_equal(got["distance"].view(np.uint32), want["distance"].view(np.uint32))
    assert got["valid"].all() and got["row"].min() >= offset
    eng.close()


def test_l2_full_size_batch(oracle):
    """10 M x 384 unit rows, batch 1024, top-10 l2 (the shape of BASELINE configs[2]): 16 sampled queries equal the
    loop, and the whole batch is proven or filtered without the exact scan."""
    n, dims, b = 10_000_000, 384, 1024
    eng = CUDAVectorEngine(L2, dims)
    eng.fill_synthetic(2, n)
    eng.set_option("batch_l2", 1)
    qs = oracle.synth_rows(1010, 0, b, dims, normalize=True)
    t0, f0 = eng.batch_stats()
    got = eng.search_batch(qs, 10)
    t1, f1 = eng.batch_stats()
    assert t1 - t0 == b and f1 - f0 == 0, (t1 - t0, f1 - f0)
    sample = list(range(0, b, b // 16))
    assert [got[i] for i in sample] == _loop(eng, qs[sample], 10)
    eng.close()
