"""GPU: seeded randomised differential testing -- random shapes, metrics, k, duplicates, zero / NaN / Inf rows,
mutations and filters, every result compared bit-for-bit (ids and score bits) with the oracle in the kernels'
accumulation order."""
import numpy as np
import pytest

from wax_b200 import CUDAVectorEngine, VectorMetric

pytestmark = pytest.mark.gpu

DIMS = [1, 3, 4, 5, 8, 31, 32, 33, 64, 96, 100, 127, 128, 129, 160, 256, 300, 384, 400, 512, 640, 768, 1000, 1024,
        1536, 2048, 2052]


def _bits(scores):
    return np.float32(scores).view(np.uint32).tolist()


def _corpus(rng, n, dims, style):
    c = rng.standard_normal((n, dims)).astype(np.float32)
    if style == "unit":
        c /= np.maximum(np.linalg.norm(c, axis=1, keepdims=True), 1e-12)
    elif style == "scaled":
        c *= rng.uniform(1e-3, 1e3, size=(n, 1)).astype(np.float32)
    elif style == "quantised":                        # few distinct values -> many exact ties
        c = np.round(c * 2).astype(np.float32) / 2
    if n > 4:
        dup = rng.integers(0, n, size=max(1, n // 10))
        c[dup] = c[rng.integers(0, n, size=dup.size)]                  # exact duplicates
        special = rng.integers(0, n, size=min(6, n))
        c[special[0]] = 0.0
        if special.size > 2:
            c[special[1], rng.integers(0, dims)] = np.nan
            c[special[2], rng.integers(0, dims)] = np.inf
    return np.ascontiguousarray(c.astype(np.float32))


@pytest.mark.parametrize("seed", range(40))
def test_random_search_cases(oracle, seed):
    rng = np.random.default_rng(10_000 + seed)
    dims = int(rng.choice(DIMS))
    n = int(rng.choice([1, 2, 7, 33, 257, 1000, 4097, 20_000])) if dims <= 1024 else int(rng.choice([1, 33, 1500]))
    metric = VectorMetric(int(rng.integers(0, 3)))
    style = str(rng.choice(["unit", "plain", "scaled", "quantised"]))
    corpus = _corpus(rng, n, dims, style)
    ids = rng.permutation(np.arange(n, dtype=np.uint64) * 3 + 17)
    eng = CUDAVectorEngine(metric, dims)
    eng.add_batch(ids, corpus)
    for _ in range(3):
        q = rng.standard_normal(dims).astype(np.float32) * np.float32(rng.choice([1.0, 0.01, 50.0]))
        if rng.random() < 0.15:
            q = corpus[rng.integers(0, n)].copy()
            q[~np.isfinite(q)] = 0.0
        k = int(rng.choice([1, 2, 10, 31, 32, 33, 72, 128, 129, 500, 10_000, 50_000]))
        got = eng.search(q, k)
        r, d, s = oracle.search(metric.value, corpus, q, k, mode=oracle.ACC_F32_TREE, threads=2)
        assert [g[0] for g in got] == [int(ids[int(i)]) for i in r], (seed, dims, n, metric, style, k)
        assert _bits([g[1] for g in got]) == s.view(np.uint32).tolist(), (seed, dims, n, metric, style, k)


@pytest.mark.parametrize("seed", range(12))
def test_random_batch_and_filter_cases(oracle, seed):
    rng = np.random.default_rng(20_000 + seed)
    dims = int(rng.choice([32, 64, 128, 256, 384, 768]))
    n = int(rng.choice([300, 5000, 40_000]))
    metric = VectorMetric(int(rng.integers(0, 2)))
    corpus = _corpus(rng, n, dims, str(rng.choice(["unit", "plain", "quantised"])))
    eng = CUDAVectorEngine(metric, dims)
    eng.add_batch(np.arange(n, dtype=np.uint64), corpus)
    eng.set_option("batch_pair", int(rng.integers(0, 2)))
    _ = rng.integers(0, 2)          # former batch_ts draw: kept so each seed's cases stay the same
    b = int(rng.choice([4, 9, 130, 257]))
    # drawn AFTER the shapes above so the earlier draws (and cases) of each seed stay what they were
    for opt in ("batch_bf16", "batch_ares"):
        eng.set_option(opt, int(np.random.default_rng(30_000 + seed).integers(0, 2)) if opt == "batch_bf16"
                       else int(np.random.default_rng(31_000 + seed).integers(0, 2)))
    k = int(rng.choice([1, 10, 72, 100]))
    qs = rng.standard_normal((b, dims)).astype(np.float32)
    got = eng.search_batch(qs, k)
    for qi in rng.choice(b, size=min(b, 6), replace=False):
        r, d, s = oracle.search(metric.value, corpus, qs[qi], k, mode=oracle.ACC_F32_TREE, threads=2)
        assert [g[0] for g in got[qi]] == r.tolist(), (seed, dims, n, b, k, int(qi))
        assert _bits([g[1] for g in got[qi]]) == s.view(np.uint32).tolist()
    # filter
    allow_rows = np.sort(rng.choice(n, size=int(rng.choice([1, 50, n // 3])), replace=False))
    got = eng.search_filtered(qs[0], k, allow=allow_rows.astype(np.uint64))
    r, d, s = oracle.search(metric.value, corpus[allow_rows], qs[0], k, mode=oracle.ACC_F32_TREE, threads=2)
    assert [g[0] for g in got] == [int(allow_rows[int(i)]) for i in r]
    assert _bits([g[1] for g in got]) == s.view(np.uint32).tolist()
