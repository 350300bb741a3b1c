"""CPU model of the l2 batched path's completeness arguments (DESIGN 4.5, `l2_proof` in waxvs_batch.cuh) with REAL
operand rounding: bf16 round-to-nearest (torch) and TF32 truncation of the operands, products accumulated in float64,
and the cached w = 0.5 * sum v^2 in fp32.

The l2 nomination score is score' = q~.v~ - w, an approximation of h = q.v - |v|^2 / 2, and |q - v|^2 = |q|^2 - 2 h.
On clustered, mixed-norm and offset data (where the proofs sometimes hold and sometimes do not) it checks:
  bound    -- |score' - h| <= E(|v|) = (1.01 eps + (n+1) 2^-23) |q| |v| + (n+2) 2^-24 |v|^2;
  level 1  -- IF (a^ (1 - delta) - 2 (tau + E_M)) (1 - delta) (1 - 2^-20) > D^_k THEN the re-scored nominees contain the
              true top-k (a "proven" flag is never wrong);
  level 2  -- tau* = (a^ / (1 + delta) - D^_k / (1 - delta)) / 2 - E_M never excludes a true top-k row.
delta = (n + 4) 2^-23 bounds the relative error of the fp32 distances.  The constants are the kernels'; this is a model of
the math, not of the CUDA code: tests/test_gpu_batch_l2.py checks the code."""
import numpy as np
import pytest
import torch

BF16_EPS = 1.03 * 2.0 ** -7
TF32_EPS = 1.25 * 2.0 ** -9


def to_bf16(x):
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(torch.bfloat16).to(torch.float32).numpy()


def to_tf32(x):      # the tensor core reads the top 19 bits of an fp32 operand (10 mantissa bits): truncation
    return (np.ascontiguousarray(x, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def corpus(rng, kind, n, dims):
    if kind == "clustered":      # unit rows around a few centres
        c = rng.standard_normal((int(rng.choice([2, 8, 60])), dims))
        c /= np.linalg.norm(c, axis=1, keepdims=True)
        v = c[rng.integers(0, c.shape[0], n)] + float(rng.choice([0.05, 0.3, 1.0])) / np.sqrt(dims) * rng.standard_normal((n, dims))
        v /= np.linalg.norm(v, axis=1, keepdims=True)
    elif kind == "mixed":        # norms spread over 1e-3 .. 1e3
        v = rng.standard_normal((n, dims)) / np.sqrt(dims) * 10.0 ** rng.uniform(-3, 3, (n, 1))
    else:                        # offset cluster: c + noise with |c| >> noise, far from the origin
        c = rng.standard_normal(dims)
        v = 50.0 * c / np.linalg.norm(c) + rng.standard_normal((n, dims)) / np.sqrt(dims)
    return v.astype(np.float32)


def half_sq(v):
    return (np.float32(0.5) * np.sum(v * v, axis=1, dtype=np.float32)).astype(np.float64)


def distances(q, v):
    """D^: fp32 squares of fp32 differences, fp32 sum (any order is within delta of D)."""
    d = (q[None, :] - v).astype(np.float32)
    return np.sum(d * d, axis=1, dtype=np.float32).astype(np.float64)


def nomination_bound(eps, qn, r, n):
    return (1.01 * eps + (n + 1) * 2.0 ** -23) * qn * r + (n + 2) * 2.0 ** -24 * r * r


def level1(sprime, dhat, k, kprime, slices, rescore):
    """Nominee heaps per row slice, union, the best `rescore` re-scored.  Returns (tau, excluded_any, rescored rows)."""
    n = sprime.size
    bounds = [n * s // slices for s in range(slices + 1)]
    nominees, tau = [], -np.inf
    for s in range(slices):
        idx = np.arange(bounds[s], bounds[s + 1])
        order = idx[np.argsort(-sprime[idx], kind="stable")]
        nominees.extend(order[:kprime].tolist())
        if order.size > kprime:                          # the heap filled up and excluded rows: its root bounds them
            tau = max(tau, sprime[order[kprime - 1]])
    nominees = np.array(nominees)
    nominees = nominees[np.argsort(-sprime[nominees], kind="stable")]
    excluded_any = np.isfinite(tau) or nominees.size > rescore
    if nominees.size > rescore:
        tau = max(tau, sprime[nominees[rescore]])
    rescored = nominees[:rescore]
    return tau, excluded_any, rescored[np.lexsort((rescored, dhat[rescored]))]     # (D^, row) order


@pytest.mark.parametrize("kind", ["clustered", "mixed", "offset"])
@pytest.mark.parametrize("level", ["bf16", "tf32"])
def test_l2_proof_is_never_wrong_and_the_filter_threshold_never_cuts_a_true_result(kind, level):
    rng = np.random.default_rng(["clustered", "mixed", "offset"].index(kind) * 2 + (level == "bf16"))
    rounder, eps = (to_bf16, BF16_EPS) if level == "bf16" else (to_tf32, TF32_EPS)
    proven_cases = unproven_cases = 0
    for case in range(30):
        dims = int(rng.choice([64, 128, 384]))
        n = int(rng.choice([600, 3000]))
        v = corpus(rng, kind, n, dims)
        q = (v[rng.integers(0, n)] + np.float32(rng.choice([0.05, 0.3])) * rng.standard_normal(dims).astype(np.float32)
             * np.float32(np.linalg.norm(v[0]) / np.sqrt(dims))).astype(np.float32)
        k = int(rng.choice([1, 10, 40]))
        kprime, slices = (16, int(rng.choice([4, 18, 37]))) if k <= 10 else (64, int(rng.choice([2, 9])))
        rescore = 256 if k <= 16 else 512
        v64, q64 = v.astype(np.float64), q.astype(np.float64)
        r = np.linalg.norm(v64, axis=1)
        qn, m = float(np.linalg.norm(q64)), float(r.max())
        w = half_sq(v)
        h = v64 @ q64 - 0.5 * r * r
        sprime = rounder(v).astype(np.float64) @ rounder(q).astype(np.float64) - w
        # the nomination bound itself (what E stands for)
        assert np.all(np.abs(sprime - h) <= nomination_bound(eps, qn, r, dims)), (kind, level, case)
        dhat = distances(q, v)
        delta = (dims + 4) * 2.0 ** -23
        truth = np.lexsort((np.arange(n), dhat))[:k]                       # the single-query answer: (D^, row)
        a = float(np.sum(q * q, dtype=np.float32))
        e_m = nomination_bound(eps, qn, m, dims)
        tau, excluded_any, rescored = level1(sprime, dhat, k, kprime, slices, rescore)
        assert rescored.size >= k
        dk = dhat[rescored[k - 1]]
        lhs = (a * (1 - delta) - 2 * (tau + e_m)) * (1 - delta) * (1 - 2.0 ** -20)
        if not excluded_any or lhs > dk:
            proven_cases += 1
            assert rescored[:k].tolist() == truth.tolist(), (kind, level, case, "a proven result missed a true top-k row")
        else:
            unproven_cases += 1
        # filter level: TF32 pass over the fp32 rows with the TF32 threshold
        s_tf32 = to_tf32(v).astype(np.float64) @ to_tf32(q).astype(np.float64) - w
        t = (a / (1 + delta) - dk / (1 - delta)) / 2 - nomination_bound(TF32_EPS, qn, m, dims)
        t = t - abs(t) * 2.0 ** -20 - 1e-30
        assert (s_tf32[truth] > t).all(), (kind, level, case, "the filter threshold cut a true top-k row")
    assert proven_cases + unproven_cases == 30
    if kind == "clustered":
        assert proven_cases >= 10 and unproven_cases >= 1, (proven_cases, unproven_cases)   # both outcomes occur
    if kind == "offset":
        assert unproven_cases >= 25, (proven_cases, unproven_cases)   # |q| M dwarfs the gaps: the exact scan answers
