"""CPU: numpy model of the 4-bit form of the single-query shadow route (DESIGN 4.1).

Row coding (16 mid-rise levels, half step h = max|v^| / 16, the row decodes to h (2u - 15), rho measured from the codes),
query coding (int8, s_q = max|q| / 127, rho_q measured), the integer score and the proof inequality

    |q.v^ - score'| <= |q| rho + rho_q (|v^| + rho) + roundings

on random and adversarial rows: whenever the model's proof holds, the nominees hold the exact top-k.  Plus the per-CTA
nominee budget: with every CTA keeping its best 256 of ~1/132 of the rows, the cut stays below what the proof needs.
"""
import numpy as np
import pytest

F32 = np.float32


def code_rows(vhat):
    """(u [n, d] in 0..15, h [n] fp32, rho [n] fp64) as shadow_u4_kernel stores them."""
    vhat = vhat.astype(F32)
    with np.errstate(all="ignore"):
        m = np.abs(vhat).max(axis=1)
        h = (m / F32(16.0)).astype(F32)
        step = (F32(2.0) * h).astype(F32)
        bad = ~np.isfinite(vhat).all(axis=1) | ~np.isfinite(h)
        u = np.floor((vhat / step[:, None]).astype(F32)) + 8
        u = np.where((h[:, None] > 0) & ~bad[:, None], np.clip(np.nan_to_num(u), 0, 15), 8).astype(np.int64)
        r = vhat.astype(np.float64) - h.astype(np.float64)[:, None] * (2 * u - 15)
        rho = np.sqrt(np.einsum("ij,ij->i", r, r))
    rho[bad] = np.inf
    return u, h, rho


def code_query(q):
    """(c_q int [d], s_q fp32, rho_q fp64) as the U4 form of the scan codes the query."""
    q = q.astype(F32)
    with np.errstate(all="ignore"):
        s_q = F32(np.abs(q).max() / F32(127.0))
        ok = np.isfinite(q).all() and np.isfinite(s_q) and s_q > 0
        c = np.clip(np.rint((q / s_q).astype(F32)), -127, 127).astype(np.int64) if ok else np.zeros(q.size, np.int64)
        e = q.astype(np.float64) - np.float64(s_q) * c
        rho_q = np.sqrt(e @ e) if np.isfinite(q).all() and np.isfinite(s_q) else np.inf
    return c, s_q, rho_q


def scores_u4(u, h, c, s_q):
    """score' = fl(fl(s_q h) (2 sum c u - 15 sum c)): the integer is exact, two fp32 roundings."""
    i = 2 * (u @ c) - 15 * c.sum()
    assert np.abs(i).max(initial=0) < 2 ** 24
    with np.errstate(all="ignore"):
        return ((F32(s_q) * h).astype(F32) * i.astype(F32)).astype(F32)


def proof(vhat, q, k, n_keep):
    """Nominate the n_keep best rows by score', re-score them exactly, prove as shadow_rescore_kernel does (fp64 model of
    its fp32 inequality, slacks included).  Returns (proven, nominated rows)."""
    u, h, rho = code_rows(vhat)
    c, s_q, rho_q = code_query(q)
    sp = scores_u4(u, h, c, s_q).astype(np.float64)
    sp = np.where(np.isfinite(sp), sp, np.inf)
    order = np.argsort(-sp, kind="stable")
    nominated, left = order[:n_keep], order[n_keep:]
    exact = vhat.astype(np.float64) @ q.astype(np.float64)
    if left.size == 0:
        return True, nominated
    tau = sp[left].max()
    qn = np.sqrt(q.astype(np.float64) @ q.astype(np.float64))
    vmax = np.sqrt(np.einsum("ij,ij->i", vhat.astype(np.float64), vhat.astype(np.float64))).max()
    rho_max = rho.max()
    eps = 1.01 * (qn * rho_max + rho_q * (vmax + rho_max)) + vhat.shape[1] * 2.0 ** -23 * qn * vmax + 1e-30
    kth = np.sort(exact[nominated])[::-1][k - 1] if nominated.size >= k else -np.inf
    proven = bool(np.isfinite(eps) and kth > tau + eps and qn * qn >= 2.0 ** -126 and np.isfinite(qn))
    return proven, nominated


def unit(x):
    return (x / np.linalg.norm(x, axis=-1, keepdims=True)).astype(F32)


def corpora(rng, n, d):
    yield "uniform", unit(rng.uniform(-1, 1, (n, d)))
    base = unit(rng.standard_normal(d))
    yield "clustered", unit(base + 0.02 * rng.standard_normal((n, d)))
    v = rng.uniform(-1, 1, (n, d)); v[:, 7] *= 40.0
    yield "outlier_dimension", unit(v)
    lv = (rng.integers(0, 16, (n, d)) * 2 - 15).astype(F32)          # values on the level boundaries / centres
    lv[:, 0] = 15
    yield "on_levels", (lv * F32(2.0 ** -6)).astype(F32)
    z = unit(rng.uniform(-1, 1, (n, d))); z[3] = 0; z[4] = F32(2.0 ** -149) * rng.integers(-3, 4, d); z[5] *= F32(2.0 ** -120)
    yield "zero_and_subnormal_rows", z.astype(F32)


@pytest.mark.parametrize("d", [128, 384])
def test_bound_holds_and_a_proven_flag_is_never_wrong(d):
    rng = np.random.default_rng(d)
    n, k = 4000, 10
    for name, vhat in corpora(rng, n, d):
        u, h, rho = code_rows(vhat)
        vn = np.sqrt(np.einsum("ij,ij->i", vhat.astype(np.float64), vhat.astype(np.float64)))
        for scale in (1.0, 2.0 ** -60, 2.0 ** 60, 1e-3):
            q = (unit(rng.standard_normal(d)) * F32(scale)).astype(F32)
            c, s_q, rho_q = code_query(q)
            sp = scores_u4(u, h, c, s_q).astype(np.float64)
            exact = vhat.astype(np.float64) @ q.astype(np.float64)
            qn = np.linalg.norm(q.astype(np.float64))
            bound = qn * rho + rho_q * (vn + rho) + 2.0 ** -22 * np.abs(sp) + 1e-30
            assert (np.abs(sp - exact) <= bound).all(), (name, scale)
            truth = set(np.argsort(-exact, kind="stable")[:k].tolist())
            kth = np.sort(exact)[::-1][k - 1]
            for keep in (k, 64, 256, 2048):
                proven, nominated = proof(vhat, q, k, keep)
                if proven:
                    best = set(nominated[np.argsort(-exact[nominated], kind="stable")[:k]].tolist())
                    assert best == truth or np.sort(exact[list(best)])[0] == kth, (name, scale, keep)


def test_refused_when_the_query_or_a_row_is_not_finite():
    rng = np.random.default_rng(1)
    vhat = unit(rng.uniform(-1, 1, (600, 128)))
    q = unit(rng.standard_normal(128))
    q[5] = np.inf
    assert not proof(vhat, q, 10, 256)[0]
    vhat[9, 3] = np.nan
    assert not proof(vhat, unit(rng.standard_normal(128)), 10, 256)[0]


def test_per_cta_budget_of_256_on_the_benchmark_distribution():
    """10 M x 384 uniform[-1, 1] normalised rows over 132 CTAs: score' of a unit query is close to N(0, 1/d), so a CTA's
    256th of ~75.8 K rows and a warp's 128th of ~4.7 K sit at normal quantiles; with the bound measured on a sample, both
    cuts stay below (10th best of 10 M) - eps, which is what the proof needs."""
    from scipy.stats import norm
    rng = np.random.default_rng(7)
    d, rows, ctas, warps = 384, 10_000_000, 132, 16
    vhat = unit(rng.uniform(-1, 1, (20000, d)))
    u, h, rho = code_rows(vhat)
    q = unit(rng.standard_normal(d))
    c, s_q, rho_q = code_query(q)
    sigma = scores_u4(u, h, c, s_q).astype(np.float64).std()
    assert abs(sigma * np.sqrt(d) - 1.0) < 0.05
    eps = 1.01 * (1.03 * rho.max() + rho_q * (1.0001 + 1.03 * rho.max())) + d * 2.0 ** -23     # 3 % for the 10 M rows' maximum
    t10 = norm.isf(10 / rows) * sigma
    cta_cut = norm.isf(256 / (rows / ctas)) * sigma
    warp_cut = norm.isf(128 / (rows / ctas / warps)) * sigma
    assert t10 - eps > 1.1 * cta_cut > warp_cut
