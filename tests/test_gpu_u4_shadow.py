"""GPU: the 4-bit form of the single-query shadow route (DESIGN 4.1), with `u4_scan_min_bytes` lowered so that small
corpora take it: the stored codes and bound against the numpy model; in every (C, R) shape `launch_u4_scan` compiles the
nominees' score' against the integer model bit for bit and inside the bound, and no left-out row above tau_excl (one CTA
with far more than 256 winners, several CTAs, a ragged last step); the route end to end against the forced fp32 scan; a
refused proof demoting the route to the int8 form and back; appends and removes.
"""
import re
from pathlib import Path

import numpy as np
import pytest

from helpers import unit_rows
from test_gpu_shadow_scan import bits, counts, fp32
from test_u4_proof_model import code_query, code_rows, scores_u4
from wax_b200 import CUDAVectorEngine, VectorMetric

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
COS, DOT = VectorMetric.cosine, VectorMetric.dot
KEY_NONE = np.uint64(0xFFFFFFFFFFFFFFFF)


def _forms():
    src = (ROOT / "wax_b200" / "csrc" / "waxvs_engine.cu").read_text()
    body = re.search(r"static cudaError_t launch_u4_scan\(.*?\n}\n", src, re.S).group(0)
    return [(int(c), int(r)) for c, r in re.findall(r"WAXVS_CASE\((\d+), (\d+)\);", body)]


def _engine(metric, corpus, **opts):
    eng = CUDAVectorEngine(metric, corpus.shape[1])
    eng.add_batch(list(range(corpus.shape[0])), corpus)
    for key, value in dict(shadow_scan_min_bytes=0, u4_scan_min_bytes=0, **opts).items():
        eng.set_option(key, value)
    return eng


def _decode(keys):
    """nominee keys -> (rows, score' as fp32)"""
    keys = keys[keys != KEY_NONE]
    hi = (keys >> np.uint64(32)).astype(np.uint32)
    u = np.where(hi & np.uint32(0x80000000), hi ^ np.uint32(0x80000000), ~hi)
    return (keys & np.uint64(0xFFFFFFFF)).astype(np.int64), -u.view(np.float32)


@pytest.mark.parametrize("dims", [128, 384, 1536])
def test_stored_codes_half_steps_and_bound(dims):
    rng = np.random.default_rng(dims)
    corpus = rng.uniform(-1.0, 1.0, (700, dims)).astype(np.float32)
    corpus[3] = 0.0
    corpus[5] = np.float32(2.0 ** -149) * rng.integers(-5, 6, dims)
    corpus[8] *= np.float32(1e36)
    eng = _engine(DOT, corpus)
    codes, half, rho_max = eng.read_u4_shadow(0, corpus.shape[0])
    want_u, want_h, want_rho = code_rows(corpus)
    assert np.array_equal(half.view(np.uint32), want_h.view(np.uint32))
    assert np.array_equal(codes, want_u)
    assert want_rho.max() <= rho_max <= want_rho.max() * (1 + 1e-6)
    assert eng.counter("u4_shadow_bytes") == corpus.shape[0] * (dims // 2 + 4)
    assert eng.counter("int8_shadow_bytes") == 0, "the int8 shadow is built only when a query takes the int8 form"
    eng.close()


@pytest.mark.parametrize("metric", [COS, DOT])
@pytest.mark.parametrize("form", _forms(), ids=lambda f: "C%d_R%d" % f)
@pytest.mark.parametrize("grid", [1, 5])
def test_nominees_in_every_form(form, metric, grid):
    c, r = form
    dims, n, k = 128 * c, 6001, 10                    # 6001: a ragged last step; grid 1: 2048 list slots, 256 kept
    rng = np.random.default_rng(c * 100 + r + grid)
    corpus = unit_rows(rng, n, dims) if metric is COS else rng.uniform(-1, 1, (n, dims)).astype(np.float32)
    eng = _engine(metric, corpus, u4_rows_per_step=r, grid=grid)
    codes, half, rho_max = eng.read_u4_shadow(0, n)
    for qi in range(2):
        q = rng.standard_normal(dims).astype(np.float32)
        q /= np.linalg.norm(q)
        out = eng.u4_nominations(q, k)
        assert (out["C"], out["R"], out["grid"]) == (c, r, grid)
        rows, got = _decode(out["keys"])
        assert len(set(rows.tolist())) == rows.size == grid * 256
        cq, s_q, rho_q = code_query(q)
        model = scores_u4(codes.astype(np.int64), half, cq, s_q)
        assert np.array_equal(got.view(np.uint32), model[rows].view(np.uint32)), "score' differs from the integer model"
        assert rho_q <= out["rho_q"] <= rho_q * (1 + 1e-6)
        left = np.setdiff1d(np.arange(n), rows)
        assert model[left].max() <= out["tau_excl"], "a left-out row beats tau_excl"
        vhat = corpus if metric is DOT else corpus / np.linalg.norm(corpus.astype(np.float64), axis=1, keepdims=True)
        exact = vhat.astype(np.float64) @ q.astype(np.float64)
        vn = np.linalg.norm(vhat.astype(np.float64), axis=1)
        assert (np.abs(model - exact) <= 1.0001 * (rho_max + out["rho_q"] * (vn + rho_max)) + 1e-6).all()
        want = fp32(eng, lambda: eng.search(q, k))
        if out["ok"]:
            assert bits(out["result"]) == bits(want)
        assert bits(eng.search(q, k)) == bits(want)
    eng.close()


@pytest.mark.parametrize("metric", [COS, DOT])
def test_route_end_to_end_and_lifecycle(metric):
    rng = np.random.default_rng(11)
    n, dims, k = 90_000, 384, 10
    corpus = rng.uniform(-1.0, 1.0, (n, dims))          # uniform elements: the 16 levels cover them evenly
    corpus = (corpus / np.linalg.norm(corpus, axis=1, keepdims=True)).astype(np.float32)
    eng = _engine(metric, corpus)
    qs = unit_rows(rng, 12, dims)
    want = fp32(eng, lambda: [eng.search(q, k) for q in qs])
    (p0, f0), u0 = counts(eng), eng.counter("single_u4_queries")
    got = [eng.search(q, k) for q in qs]
    assert [bits(g) for g in got] == [bits(w) for w in want]
    assert eng.counter("single_u4_queries") - u0 == len(qs)
    (p1, f1) = counts(eng)
    assert (p1 - p0) + (f1 - f0) == len(qs) and p1 - p0 >= len(qs) // 2, "the 4-bit proofs should mostly hold here"
    assert eng.counter("u4_shadow_rows") == n
    extra = unit_rows(rng, 500, dims)
    extra[7] = qs[0]                                   # a new exact match must be found through the extended shadow
    eng.add_batch(list(range(n, n + 500)), extra)
    assert eng.search(qs[0], k)[0][0] == n + 7 and eng.counter("u4_shadow_rows") == n + 500
    eng.remove(n + 7)
    assert bits(eng.search(qs[0], k)) == bits(fp32(eng, lambda: eng.search(qs[0], k)))
    assert eng.counter("u4_shadow_rows") in (n + 7, n + 499)      # the kept prefix, or rebuilt by a 4-bit query
    eng.close()


def test_refused_proof_demotes_to_int8_and_comes_back():
    rng = np.random.default_rng(5)
    n, dims, k = 9000, 384, 10
    base = (rng.choice([-1.0, 1.0], dims) / np.sqrt(dims)).astype(np.float32)        # no outlier element: int8 stays fine
    corpus = (base + 0.01 * rng.standard_normal((n, dims))).astype(np.float32)      # one tight cluster: 4 bits cannot prove
    eng = _engine(COS, corpus, int8_scan_min_bytes=0, grid=2)
    q = base
    want = fp32(eng, lambda: eng.search(q, k))
    (p0, f0), u0, i0 = counts(eng), eng.counter("single_u4_queries"), eng.counter("single_int8_queries")
    assert bits(eng.search(q, k)) == bits(want)
    assert counts(eng) == (p0, f0 + 1) and eng.counter("single_u4_queries") == u0 + 1
    for _ in range(16):                                # the window: the int8 form, never a wrong answer
        assert bits(eng.search(q, k)) == bits(want)
    assert eng.counter("single_u4_queries") == u0 + 1 and eng.counter("single_int8_queries") - i0 >= 1
    for _ in range(600):          # (an int8 proof that fails too opens the fp32 window of its own in between)
        assert bits(eng.search(q, k)) == bits(want)
        if eng.counter("single_u4_queries") >= u0 + 2:
            break
    assert eng.counter("single_u4_queries") >= u0 + 2, "the 4-bit form was not probed again after the window"
    eng.close()
