"""CPU model of the single-query route's proof under the int8 shadow's measured bound (DESIGN 4.1).

The int8 shadow stores each row v^ (cosine: v / |v|, dot: v) as codes c_i = rne(v^_i / s) with s = max|v^_i| / 127, and
measures rho = ||v^ - s c||_2 from what it stored (shadow_int8_kernel).  Then |q.v^ - s (q.c)| <= |q| rho for every
query (Cauchy-Schwarz), and the finish proves with eps_rel = rho_max / M (M = 1 cosine, max|v| dot).  This checks, on
random, clustered and adversarial rows (outlier dimensions, components on rounding midpoints, zero and subnormal rows),
that the measured bound holds row by row and that a proven flag is never wrong: whenever the exact k-th score of the
re-scored nominees clears the 128th nominee's score' by eps, the nominees hold the true top-k.  A model of the math, not
of the CUDA code: tests/test_gpu_int8_shadow.py checks the code."""
import numpy as np
import pytest

BF16_EPS = 1.03 * 2.0 ** -7
K_PRIME, RESCORE = 128, 256


def int8_shadow(vhat):
    """(codes, scales, rho per row) as shadow_int8_kernel stores and measures them."""
    vhat = np.ascontiguousarray(vhat, np.float32)
    m = np.abs(vhat).max(axis=1)
    s = (m / np.float32(127.0)).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        c = np.where(s[:, None] > 0, np.rint(vhat / s[:, None]), 0.0)
    c = np.clip(c, -127, 127).astype(np.float64)
    r = vhat.astype(np.float64) - s.astype(np.float64)[:, None] * c
    rho = np.sqrt(np.einsum("ij,ij->i", r, r)) * (1.0 + 2.0 ** -40)
    return c, s, rho


def scores(q, v, metric):
    """(score' = s (q.c), exact score in the same units, vhat, rho per row, eps_rel * scale of the finish)."""
    norms = np.linalg.norm(v.astype(np.float64), axis=1)
    if metric == "cosine":
        # the cached 1/|v| is 0 when fl(sum v^2) is (rows of tiny components): such a row scores 0, as in the fp32 scan
        live = np.einsum("ij,ij->i", v, v, dtype=np.float32) > 0
        inv = np.where(live, 1.0 / np.where(live, norms, 1.0), 0.0).astype(np.float32)
        vhat = (v * inv[:, None]).astype(np.float32)
        exact = np.where(live, (v.astype(np.float64) @ q.astype(np.float64)) / np.where(live, norms, 1.0), 0.0)
        m = 1.0
    else:
        vhat = v.astype(np.float32)
        exact = v.astype(np.float64) @ q.astype(np.float64)
        m = float(norms.max())
    c, s, rho = int8_shadow(vhat)
    sprime = s.astype(np.float64) * (c @ q.astype(np.float64))
    qn = float(np.linalg.norm(q.astype(np.float64)))
    eps_rel = float(rho.max()) / m
    return sprime, exact, vhat, rho, eps_rel, qn * m


def proof(sprime, exact, scale, k, eps_rel):
    """The finish on one slice of 128 nominees: (proven, exact k-th score of the re-scored nominees)."""
    order = np.argsort(-sprime, kind="stable")
    nominees = order[:K_PRIME]
    tau = sprime[order[K_PRIME - 1]] if sprime.size > K_PRIME else -np.inf
    sk = np.sort(exact[nominees[:RESCORE]])[::-1][k - 1]
    return bool(sk > tau + eps_rel * scale * 1.01) or not np.isfinite(tau), sk


def corpus(rng, kind, n, dims):
    if kind == "uniform":                       # the benchmark's distribution
        return rng.uniform(-1.0, 1.0, (n, dims)).astype(np.float32)
    if kind == "clustered":                     # near neighbours: proofs fail sometimes
        c = rng.standard_normal((4, dims)).astype(np.float32)
        return (c[rng.integers(0, 4, n)] + np.float32(0.05) * rng.standard_normal((n, dims)).astype(np.float32))
    if kind == "outlier":                       # one large dimension coarsens every row's scale
        v = rng.uniform(-1.0, 1.0, (n, dims)).astype(np.float32)
        v[:, 7] *= np.float32(40.0)
        return v
    if kind == "midpoints":                     # components on code rounding midpoints: the largest residual per row
        codes = rng.integers(-126, 126, (n, dims)).astype(np.float32)
        v = (codes + np.float32(0.5)) * np.float32(2.0 ** -7)
        v[:, 0] = np.float32(127 * 2.0 ** -7)   # s = 2^-7 exactly
        return v
    v = rng.uniform(-1.0, 1.0, (n, dims)).astype(np.float32)      # "special": zero, subnormal and tiny rows mixed in
    v[::97] = 0.0
    v[1::89] *= np.float32(2.0 ** -140)
    v[2::83] = np.float32(2.0 ** -149) * rng.integers(-3, 4, (v[2::83].shape[0], dims)).astype(np.float32)
    return v


@pytest.mark.parametrize("metric", ["cosine", "dot"])
def test_the_measured_bound_holds_and_a_proven_flag_is_never_wrong(metric):
    rng = np.random.default_rng(88)
    proven_cases = unproven_cases = 0
    for case in range(48):
        kind = ["uniform", "clustered", "outlier", "midpoints", "special"][case % 5]
        dims = int(rng.choice([128, 384]))
        n = int(rng.choice([300, 2000]))
        v = corpus(rng, kind, n, dims)
        q = v[rng.integers(0, n)] + np.float32(0.3 / np.sqrt(dims)) * rng.standard_normal(dims).astype(np.float32)
        q = (q * np.float32(rng.uniform(0.3, 3.0))).astype(np.float32)
        k = int(rng.choice([1, 10, 32]))
        sprime, exact, vhat, rho, eps_rel, scale = scores(q, v, metric)
        # row by row: |s (q.c) - q.v^| <= |q| rho_r (up to the fp64 evaluation here)
        qn = float(np.linalg.norm(q.astype(np.float64)))
        approx = vhat.astype(np.float64) @ q.astype(np.float64)
        assert np.all(np.abs(sprime - approx) <= qn * rho * (1 + 1e-9) + 1e-300), (metric, kind, case)
        # the whole bound: |score' - exact| <= eps_rel * scale, plus the pre-scale's fp32 rounding (cosine)
        assert np.all(np.abs(sprime - exact) <= eps_rel * scale * 1.01 + dims * 2.0 ** -23 * scale), (metric, kind, case)
        proven, sk = proof(sprime, exact, scale, k, eps_rel)
        true_kth = np.sort(exact)[::-1][k - 1]
        if proven:
            proven_cases += 1
            assert sk == true_kth, (metric, kind, case, "a proven result missed a true top-k row")
        else:
            unproven_cases += 1
    assert proven_cases >= 10 and unproven_cases >= 3, (proven_cases, unproven_cases)


def test_the_int8_bound_is_no_coarser_than_bf16_on_the_benchmark_distribution_and_coarser_with_outliers():
    """The selection rule: unit rows of the benchmark's distribution measure rho_max well under kBf16Eps (the route takes
    the int8 shadow); a corpus with one dimension 40x larger measures it above (the route keeps the bf16 shadow)."""
    rng = np.random.default_rng(5)
    for kind, below in (("uniform", True), ("outlier", False)):
        v = corpus(rng, kind, 20_000, 384)
        vhat = (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(np.float32)
        rho_max = float(int8_shadow(vhat)[2].max())
        assert (rho_max <= BF16_EPS) == below, (kind, rho_max)
    assert rho_max > BF16_EPS
