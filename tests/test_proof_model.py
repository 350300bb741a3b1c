"""CPU model of the batched path's completeness arguments (DESIGN 4.5 / 4.5.1) with REAL operand rounding:
bf16 round-to-nearest (torch) and TF32 truncation of the operands, products accumulated in float64.  On an H100 (80 GB
HBM3, 400 W limit) tests/test_gpu_nomination.py measured the whole nomination error, operand rounding plus the tensor
core's fp32 accumulation, at up to 0.955 of the bf16 bound and 0.786 of the TF32 bound on a worst-case rounding corpus
(TF32 operands are truncated there, as modelled here); the finish kernel adds dims * 2^-23 on top.

It checks the two claims the kernels rely on, on adversarial clustered data where the proofs sometimes hold and
sometimes do not:
  level 1  -- IF `exact k-th score of the re-scored nominees > max(tau_excl, (R+1)-th nominee) + eps` THEN the
              re-scored nominees contain the true top-k (so a "proven" flag is never wrong);
  level 2  -- the filter threshold tau* = (exact k-th score of the nominees) - eps_tf32 never excludes a true top-k
              row, whether or not level 1 proved anything (the filter level is complete by construction).
The constants are the kernels' (`kBf16Eps`, `kTf32Eps` in wax_b200/csrc/waxvs_batch.cuh).  This is a model of the
math, not of the CUDA code: the GPU tests check the code."""
import numpy as np
import pytest
import torch

BF16_EPS = 1.03 * 2.0 ** -7
TF32_EPS = 1.25 * 2.0 ** -9


def to_bf16(x):
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(torch.bfloat16).to(torch.float32).numpy()


def to_tf32(x):      # the tensor core reads the top 19 bits of an fp32 operand (10 mantissa bits): truncation
    return (np.ascontiguousarray(x, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def clustered(rng, n, dims, centres, sigma):
    c = rng.standard_normal((centres, dims)).astype(np.float32)
    c /= np.linalg.norm(c, axis=1, keepdims=True)
    v = c[rng.integers(0, centres, n)] + np.float32(sigma / np.sqrt(dims)) * rng.standard_normal((n, dims)).astype(np.float32)
    scale = rng.uniform(0.25, 4.0, size=(n, 1)).astype(np.float32)        # cosine must not care; dot does
    return (v * scale).astype(np.float32)


def nomination_scores(q, v, metric, rounder, prescale):
    """score' as the tensor-core pass produces it, and the exact score in the same units (cosine: q.v/|v|)."""
    norms = np.linalg.norm(v.astype(np.float64), axis=1)
    if metric == "cosine":
        if prescale:      # bf16 shadow rows are pre-scaled by 1/|v| (fp32), then rounded
            b = rounder((v / norms[:, None].astype(np.float32)).astype(np.float32)).astype(np.float64)
            sprime = b @ rounder(q).astype(np.float64)
        else:             # TF32: raw rows, the epilogue multiplies by the cached 1/|v|
            sprime = (rounder(v).astype(np.float64) @ rounder(q).astype(np.float64)) / norms
        exact = (v.astype(np.float64) @ q.astype(np.float64)) / norms
        scale = float(np.linalg.norm(q.astype(np.float64)))
    else:
        sprime = rounder(v).astype(np.float64) @ rounder(q).astype(np.float64)
        exact = v.astype(np.float64) @ q.astype(np.float64)
        scale = float(np.linalg.norm(q.astype(np.float64))) * float(norms.max())
    return sprime, exact, scale


def level1(sprime, exact, scale, k, kprime, slices, rescore, eps_rel):
    n = sprime.size
    bounds = [n * s // slices for s in range(slices + 1)]
    nominees, tau_excl = [], -np.inf
    for s in range(slices):
        idx = np.arange(bounds[s], bounds[s + 1])
        if idx.size == 0:
            continue
        order = idx[np.argsort(-sprime[idx], kind="stable")]
        nominees.extend(order[:kprime].tolist())
        if order.size > kprime:                          # the heap filled up and excluded rows: its root bounds them
            tau_excl = max(tau_excl, sprime[order[kprime - 1]])
    nominees = np.array(nominees)
    nominees = nominees[np.argsort(-sprime[nominees], kind="stable")]
    rescored = nominees[:rescore]
    tau = tau_excl
    if nominees.size > rescore:
        tau = max(tau, sprime[nominees[rescore]])
    if rescored.size < k:
        return False, rescored, None
    sk = np.sort(exact[rescored])[::-1][k - 1]
    proven = bool(sk > tau + eps_rel * scale * 1.01) or not np.isfinite(tau)
    return proven, rescored, sk


@pytest.mark.parametrize("metric", ["cosine", "dot"])
@pytest.mark.parametrize("level", ["bf16", "tf32"])
def test_a_proven_flag_is_never_wrong_and_the_filter_threshold_never_cuts_a_true_result(metric, level):
    rng = np.random.default_rng(2024)
    rounder, eps_rel, prescale = (to_bf16, BF16_EPS, True) if level == "bf16" else (to_tf32, TF32_EPS, False)
    proven_cases = unproven_cases = 0
    for case in range(60):
        dims = int(rng.choice([64, 128, 384]))
        n = int(rng.choice([600, 3000]))
        centres = int(rng.choice([2, 8, 60, n]))
        sigma = float(rng.choice([0.02, 0.1, 0.35, 1.0]))
        v = clustered(rng, n, dims, centres, sigma)
        if metric == "cosine":
            pass
        else:
            v /= np.linalg.norm(v, axis=1, keepdims=True)           # dot on unit rows: the bound uses max |v| = 1
        q = (v[rng.integers(0, n)] + np.float32(0.2 / np.sqrt(dims)) * rng.standard_normal(dims).astype(np.float32)) \
            * np.float32(rng.uniform(0.3, 3.0))
        k = int(rng.choice([1, 10, 40]))
        kprime, slices = (16, int(rng.choice([4, 18, 37]))) if k <= 10 else (64, int(rng.choice([2, 9])))
        rescore = 256 if k <= 16 else 512
        sprime, exact, scale = nomination_scores(q, v, metric, rounder, prescale)
        # the rounding bound itself (what eps stands for)
        assert np.all(np.abs(sprime - exact) <= eps_rel * scale), (metric, level, case)
        proven, rescored, sk = level1(sprime, exact, scale, k, kprime, slices, rescore, eps_rel)
        true_kth = np.sort(exact)[::-1][k - 1]
        if proven:
            proven_cases += 1
            assert sk == true_kth, (metric, level, case, "a proven result missed a true top-k row")
        else:
            unproven_cases += 1
        # level 2: threshold from the nominees' exact k-th score, filter pass in TF32 on the raw rows
        if sk is not None:
            s_tf32, _, scale_f = nomination_scores(q, v, metric, to_tf32, False)
            tau_star = sk - TF32_EPS * scale_f * 1.01
            candidates = s_tf32 > tau_star - abs(tau_star) * 2.0 ** -20
            top = np.argsort(-exact, kind="stable")[:k]
            assert candidates[top].all(), (metric, level, case, "the filter threshold cut a true top-k row")
            assert exact[candidates].max() == exact.max()
    assert proven_cases >= 10 and unproven_cases >= 5, (proven_cases, unproven_cases)   # both outcomes were exercised
