"""GPU: the single-query 4-bit route (DESIGN 4.1), checked stage by stage (wax_vs_debug_u4_nominations).

When the grid-wide re-score proves a 4-bit query, the guarded fp32 scan returns at entry and nothing checks the answer
afterwards.  So each stage is pinned here on its own, with `u4_scan_min_bytes` lowered so that small corpora take the form:

  1. the stored shadow of both metrics against the numpy model (cosine rows pre-scaled by the cached 1/|v|), and rho_max
     against the residual measured from the stored codes; a non-finite row turns the form off;
  2. in every (C, R) shape `launch_u4_scan` compiles, every schedule and warp / stage option: the nominee layout (a real
     prefix per CTA block of 256, then padding), score' against the integer model bit for bit, every left-out row at or
     below tau_excl, and rows planted at row 0, the last row, every position of a step, claim edges and the ragged last
     step all nominated;
  3. the warp-level cut: a warp whose list fills before its CTA's selection binds must lower tau_excl;
  4. the proof at the warp-list and at the CTA boundary, with a winner whose score' the 4-bit rounding hides;
  5. the proof flag against an fp64 restatement of shadow_rescore_kernel's inequality, swept across its boundary;
  6. the re-score against the fp32 scan restricted to the nominees, bit for bit, over grids up to 264 (block keys read
     from L2) and k in {1, 10, 32};
  7. degenerate queries and score' overflow (+inf, and inf * 0 = NaN, are nominated as +inf and re-scored);
  8. filters and delivery on the route; 9. state carried between queries and contexts; 10. lifecycle and demotion.
Every answer is compared with the forced fp32 scan, ids and score bits.
"""
import threading
import time
import zlib

import numpy as np
import pytest

from helpers import unit_rows
from test_gpu_degenerate_queries import degenerate_queries
from test_gpu_int8_shadow import _special_rows, _vhat
from test_gpu_shadow_nominations import _planted, _risky_rows
from test_gpu_shadow_scan import bits, counts, fp32, routed
from test_gpu_u4_shadow import _decode, _forms
from test_u4_proof_model import code_query, code_rows, scores_u4
from wax_b200 import CUDAVectorEngine, VectorMetric
from wax_b200.engine import InvalidToc

pytestmark = pytest.mark.gpu

COS, DOT = VectorMetric.cosine, VectorMetric.dot
KEY_NONE = np.uint64(0xFFFFFFFFFFFFFFFF)
CTA_KEYS, WARP_KEYS = 256, 128     # kU4CtaNominees; a warp list of the U4 form (E = 4)
SM_BUDGET = 232448 - 4096          # pick_u4_config: the opt-in shared memory minus the kernels' static shared memory
FORMS = _forms()
SCHEDULES = [("auto", dict(chunk_steps=-1, grid=0)), ("auto_grid7", dict(chunk_steps=-1, grid=7)),
             ("static", dict(chunk_steps=0, grid=0))]


def _set(eng, **opts):
    for key, value in opts.items():
        eng.set_option(key, value)


def _engine(metric, corpus, **opts):
    eng = CUDAVectorEngine(metric, corpus.shape[1])
    eng.add_batch(list(range(corpus.shape[0])), corpus)
    _set(eng, shadow_scan_min_bytes=0, u4_scan_min_bytes=0, **opts)
    return eng


def _synth(metric, n, dims, seed, **opts):
    eng = CUDAVectorEngine(metric, dims)
    eng.fill_synthetic(seed, n, normalize=metric is COS)
    _set(eng, shadow_scan_min_bytes=0, u4_scan_min_bytes=0, **opts)
    return eng


def _fits(warps, stages, R, dims):
    """pick_u4_config's ring arithmetic."""
    return warps * stages * (R * (dims // 2 + 4) + 12) + warps * 1024 + 16 <= SM_BUDGET


def _model(eng, q):
    """score' of every row by the integer model from the stored codes (a non-finite score' is nominated as +inf)."""
    codes, half, rho_max = eng.read_u4_shadow(0, eng.count)
    c, s_q, _ = code_query(q)
    with np.errstate(all="ignore"):
        sc = scores_u4(codes.astype(np.int64), half, c, s_q)
    return np.where(np.isfinite(sc), sc, np.float32(np.inf)).astype(np.float32)


def _vmax(corpus):
    return float(np.sqrt(np.einsum("ij,ij->i", corpus.astype(np.float64), corpus.astype(np.float64))).max())


def _check(d, model, allowed=None):
    """Layout, score' bit for bit, and completeness of one read-out.  Returns the nominated rows."""
    n = model.size
    allowed = np.ones(n, bool) if allowed is None else allowed
    keys = d["keys"]
    assert keys.size == d["grid"] * CTA_KEYS
    real = (keys != KEY_NONE).reshape(d["grid"], CTA_KEYS)
    per = real.sum(axis=1)
    assert all(real[b, :per[b]].all() and not real[b, per[b]:].any() for b in range(d["grid"])), \
        "a CTA block is not a real prefix followed by padding"
    rows, got = _decode(keys)
    assert np.all((rows >= 0) & (rows < n)), "a nominee row is out of range"
    assert np.unique(rows).size == rows.size, "a row was nominated twice"
    assert allowed[rows].all(), "a row the filter excludes was nominated"
    assert np.array_equal(got.view(np.uint32), model[rows].view(np.uint32)), "score' differs from the integer model"
    left = allowed.copy()
    left[rows] = False
    tau = d["tau_excl"]
    assert np.all(model[left] <= tau), f"{int((model[left] > tau).sum())} left-out rows above tau_excl"
    if left.any():
        assert tau > -np.inf, "rows were left out, yet tau_excl says none was"
    if allowed.sum() < WARP_KEYS:
        assert tau == -np.inf and not left.any(), "no list can fill, yet a cut was recorded"
    return rows


def _ok_model(d, q, k, metric, vmax=1.0):
    """shadow_rescore_kernel's proof in fp64: (ok, |s_k - tau - eps|, eps)."""
    q32 = q.astype(np.float32)
    with np.errstate(all="ignore"):
        a2 = float(np.sum(q32 * q32, dtype=np.float32))
        qn = float(np.sqrt(np.float32(a2)))
    rho_max, rho_q, tau = d["rho_max"], d["rho_q"], d["tau_excl"]
    excluded = tau > -np.inf
    guard = np.isfinite(a2) and a2 >= 2.0 ** -126
    res = d["result"]
    if len(res) < k:
        return (not excluded) and guard, np.inf, np.inf
    score = res[k - 1][1]
    cos = metric is COS
    dk = float(np.float32(1.0) - np.float32(score)) if cos else -score
    m = 1.0 if cos else vmax
    big_m = 1.0001 if cos else m
    with np.errstate(all="ignore"):
        eps = 1.01 * (qn * rho_max + rho_q * (big_m + rho_max)) + q.size * 2.0 ** -23 * qn * m \
            + 2.0 ** -21 * max(1.0, abs(dk)) * (qn if cos else 1.0)
        s_k = (1.0 - dk) * qn if cos else 1.0 - dk
        if not excluded:
            return guard, np.inf, eps
        ok = bool(np.isfinite(eps) and s_k > tau + eps)
        return ok and guard, abs(s_k - tau - eps), eps


def _check_ok(d, q, k, metric, vmax=1.0):
    ok, margin, eps = _ok_model(d, q, k, metric, vmax)
    if not (margin <= 5e-3 * eps):
        assert d["ok"] == int(ok), f"proof flag {d['ok']}, the inequality says {int(ok)} (margin {margin:.3g}, eps {eps:.3g})"
    return ok


def _check_rescore(eng, d, q, k, rows):
    """The re-score equals the fp32 scan restricted to the nominees (frame id = row here), proven or not."""
    if rows.size == 0:
        return
    want = fp32(eng, lambda: eng.search_filtered(q, k, allow=rows.tolist()))
    assert bits(d["result"]) == bits(want), "the re-score differs from the fp32 scan over the nominees"


def _u4_routed(eng, call, n, proven=None):
    """call() on the route: n queries nominated from the 4-bit shadow (and `proven` of them proven, when given)."""
    u0, (p0, f0) = eng.counter("single_u4_queries"), counts(eng)
    out = call()
    assert eng.counter("single_u4_queries") - u0 == n, "the 4-bit form did not nominate"
    p1, f1 = counts(eng)
    assert (p1 - p0) + (f1 - f0) == n
    if proven is not None:
        assert p1 - p0 == proven, f"{p1 - p0} proofs held, expected {proven}"
    return out


def _plant(rng, eng, q, rows, metric, lo=0.5, hi=0.9):
    """Overwrite `rows` with rows whose cosine with q is lo .. hi (far above every random row)."""
    v = _planted(rng, q, len(rows), metric)
    if (lo, hi) != (0.5, 0.9):
        qh = q.astype(np.float64) / np.linalg.norm(q)
        x = v.astype(np.float64) - (v.astype(np.float64) @ qh)[:, None] * qh[None, :]
        x /= np.linalg.norm(x, axis=1, keepdims=True)
        c = rng.permutation(np.linspace(lo, hi, len(rows)))
        v = (c[:, None] * qh[None, :] + np.sqrt(1 - c * c)[:, None] * x).astype(np.float32)
    eng.add_batch([int(r) for r in rows], v)
    return v


# ---- 1. the stored shadow -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("metric", [COS, DOT], ids=["cos", "dot"])
@pytest.mark.parametrize("dims", [128, 384, 1536])
def test_stored_shadow_both_metrics(metric, dims):
    rng = np.random.default_rng(dims * 3 + (metric is DOT))
    corpus = _special_rows(rng, 700, dims, metric)
    eng = _engine(metric, corpus)
    codes, half, rho_max = eng.read_u4_shadow(0, corpus.shape[0])
    vhat = _vhat(metric, corpus)
    want_u, want_h, _ = code_rows(vhat)
    if metric is DOT:
        assert np.array_equal(half.view(np.uint32), want_h.view(np.uint32)), "half steps"
        assert np.array_equal(codes, want_u), "codes"
    else:                   # the device's 1/|v| may differ from this model's by an ulp: a code may move by one
        assert np.allclose(half, want_h, rtol=2.0 ** -21, atol=0), "half steps of the pre-scaled rows"
        diff = np.abs(codes.astype(np.int32) - want_u.astype(np.int32))
        assert diff.max() <= 1 and (diff > 0).mean() < 1e-3, "codes of the pre-scaled rows"
    assert (codes[[3, 4]] == 8).all() and (half[[3, 4]] == 0).all(), "zero and -0 rows"
    r = vhat.astype(np.float64) - half.astype(np.float64)[:, None] * (2.0 * codes - 15.0)
    rho = np.sqrt(np.einsum("ij,ij->i", r, r)).max()
    slack = 2.0 ** -22 if metric is COS else 0.0      # (the model's v^ may differ from the device's by an ulp)
    assert rho * (1 - 1e-12) - slack <= rho_max <= rho * (1 + 2.0 ** -20) + slack, (rho_max, rho)
    assert eng.counter("u4_shadow_rows") == corpus.shape[0]
    # a non-finite row: rho_max = +inf, and no search takes the 4-bit form
    q = unit_rows(rng, 1, dims)[0]
    bad = corpus[:40].copy()
    bad[9, 1] = np.inf
    eng.add_batch(list(range(10_000, 10_040)), bad)
    assert eng.read_u4_shadow(0, 1)[2] == np.inf
    want = fp32(eng, lambda: eng.search(q, 10))
    u0 = eng.counter("single_u4_queries")
    assert bits(eng.search(q, 10)) == bits(want)
    assert eng.counter("single_u4_queries") == u0, "the 4-bit form answered with an infinite bound"
    eng.close()


# ---- 2. nominee layout and cuts in every form --------------------------------------------------------------------------

@pytest.mark.parametrize("metric", [COS, DOT], ids=["cos", "dot"])
@pytest.mark.parametrize("C,R", FORMS, ids=[f"C{c}_R{r}" for c, r in FORMS])
def test_nominees_and_cuts_in_every_form(C, R, metric):
    dims, n = 128 * C, 20_011
    rng = np.random.default_rng(zlib.crc32(f"u4form{C},{R},{metric.name}".encode()))
    corpus = unit_rows(rng, n, dims)
    if metric is COS:                                  # cosine rows of any norm: the shadow codes v / |v|
        corpus *= np.float32(10.0) ** rng.uniform(-1, 1, (n, 1)).astype(np.float32)
    q = unit_rows(rng, 1, dims)[0]
    eng = _engine(metric, corpus, u4_rows_per_step=R)
    chunks = set()
    for _, sched in SCHEDULES:                         # the claim lengths depend on the options and n only
        for warps in (1, 5, 16):
            _set(eng, u4_warps=warps, u4_stages=2, **sched)
            chunks.add(eng.u4_nominations(q, 10)["chunk_steps"])
    risky = _risky_rows(n, R, chunks)
    extra = rng.permutation(np.setdiff1d(rng.choice(n, 400, replace=False), risky))[:max(0, 64 - risky.size)]
    planted = np.sort(np.concatenate([risky, extra]))
    _plant(rng, eng, q, planted, metric)
    corpus = eng.read_rows(0, n)
    model = _model(eng, q)
    vmax = _vmax(corpus)
    _, _, rho_q = code_query(q)
    i = 0
    for name, sched in SCHEDULES:
        for warps in (1, 5, 16):
            for stages in (2, 3, 4):
                k = (1, 10, 32)[i % 3]
                i += 1
                _set(eng, u4_warps=warps, u4_stages=stages, **sched)
                if not _fits(warps, stages, R, dims):
                    with pytest.raises(InvalidToc, match="rc=-8"):
                        eng.u4_nominations(q, k)
                    continue
                d = eng.u4_nominations(q, k)
                assert (d["C"], d["R"], d["warps"], d["stages"]) == (C, R, warps, stages), d
                assert (d["chunk_steps"] == 0) == (sched["chunk_steps"] == 0), d
                if sched["grid"]:
                    assert d["grid"] == sched["grid"], d
                rows = _check(d, model)
                assert set(planted.tolist()) <= set(rows.tolist()), f"{name}: a planted row was not nominated"
                assert rho_q <= d["rho_q"] <= rho_q * (1 + 1e-6)
                _check_rescore(eng, d, q, k, rows)
                _check_ok(d, q, k, metric, vmax)
    # tail_select does not apply to this form: same nominees (static claims: the same rows per CTA) and answer
    _set(eng, u4_warps=0, u4_stages=0, chunk_steps=0, grid=0)
    outs = []
    for tail in (1, 0):
        _set(eng, tail_select=tail)
        d = eng.u4_nominations(q, 10)
        outs.append((np.sort(d["keys"].reshape(d["grid"], CTA_KEYS), axis=1), bits(d["result"]), d["ok"], d["tau_excl"]))
    assert np.array_equal(outs[0][0], outs[1][0]) and outs[0][1:] == outs[1][1:], "tail_select changed the 4-bit form"
    _set(eng, tail_select=1, chunk_steps=-1)
    want = fp32(eng, lambda: eng.search(q, 10))
    assert bits(_u4_routed(eng, lambda: eng.search(q, 10), 1)) == bits(want)
    eng.close()


def test_rows_per_step_fallbacks():
    """u4_rows_per_step outside r_lo .. r_hi, or not a power of two, falls back to r_hi; in range it is taken."""
    rng = np.random.default_rng(77)
    for C in sorted({c for c, _ in FORMS}):
        rs = [r for c, r in FORMS if c == C]
        r_lo, r_hi = min(rs), max(rs)
        dims = 128 * C
        corpus = unit_rows(rng, 3001, dims)
        q = unit_rows(rng, 1, dims)[0]
        eng = _engine(DOT, corpus)
        want = fp32(eng, lambda: eng.search(q, 10))
        for r in (0, 1, 2, 3, r_lo, r_lo + 1, r_hi, 2 * r_hi, 6, 12, -4):
            expect = r if r_lo <= r <= r_hi and (r & (r - 1)) == 0 else r_hi
            eng.set_option("u4_rows_per_step", r)
            d = eng.u4_nominations(q, 10)
            assert (d["C"], d["R"]) == (C, expect), (r, d)
            _check(d, _model(eng, q))
            assert bits(eng.search(q, 10)) == bits(want)
        eng.close()


# ---- 3. the warp-level cut ---------------------------------------------------------------------------------------------

def _warp_rows(warp, warps, R, n, count):
    """The first `count` rows of the static steps warp, warp + warps, ... (grid 1)."""
    out = []
    step = warp
    while len(out) < count:
        out.extend(range(step * R, min(step * R + R, n)))
        step += warps
    assert out[count - 1] < n
    return np.array(out[:count])


@pytest.mark.parametrize("metric", [COS, DOT], ids=["cos", "dot"])
def test_warp_level_cut_binds(metric):
    """Static claims, grid 1, 16 warps: 200 strong rows only in warp 0's steps.  Warp 0 keeps 128 of them, the CTA's
    selection of 256 does not bind on that warp, so only the warp's cut can bound the 72 strong rows left out.  With the
    strong rows near-tied and k = 32 the proof must refuse."""
    dims, n, R = 384, 16_000, 16
    rng = np.random.default_rng(300 + (metric is DOT))
    corpus = unit_rows(rng, n, dims)
    q = unit_rows(rng, 1, dims)[0]
    eng = _engine(metric, corpus, chunk_steps=0, grid=1, u4_warps=16, u4_rows_per_step=R)
    strong = _warp_rows(0, 16, R, n, 200)
    _plant(rng, eng, q, strong, metric, lo=0.8, hi=0.8002)
    model = _model(eng, q)
    corpus = eng.read_rows(0, n)
    d = eng.u4_nominations(q, 32)
    assert (d["grid"], d["warps"], d["chunk_steps"]) == (1, 16, 0), d
    rows = _check(d, model)
    kept = np.intersect1d(rows, strong)
    assert kept.size == WARP_KEYS, f"warp 0 kept {kept.size} strong rows, its list holds {WARP_KEYS}"
    left = np.setdiff1d(strong, rows)
    assert model[left].max() <= d["tau_excl"], "the warp's cut does not bound the strong rows it left out"
    assert d["ok"] == 0, "a proof with near-tied rows left out of a full warp list"
    _check_ok(d, q, 32, metric, _vmax(corpus))
    _check_rescore(eng, d, q, 32, rows)
    want = fp32(eng, lambda: eng.search(q, 32))
    assert bits(routed(eng, lambda: eng.search(q, 32), proven=0, failed=1)) == bits(want)
    eng.close()


# ---- 4. the proof at both nominee boundaries ---------------------------------------------------------------------------

def _u4_hidden_winner(rng, dims, n_decoys):
    """Dot: q holds integers 1 .. 127 (max 127: s_q = 1, rho_q = 0).  Every special row has v_0 = 16 (h = 1: cells of
    width 2 with centres at the odd integers).  The winner's other components sit 2^-8 below the top of their cells, so
    its score' loses (1 - 2^-8) sum q; the decoys sit on cell centres (exact codes) with exact scores spread over
    (0.15, 0.9) of that loss below the winner's: each decoy's score' beats the winner's, its exact score does not."""
    q = rng.integers(1, 128, dims).astype(np.float64)
    q[0] = 127.0
    e = rng.integers(1, 7, dims).astype(np.float64)
    best = 2 * e - 2.0 ** -8
    base = 2 * e - 1
    best[0] = base[0] = 16.0
    s_best = q @ best
    gap = s_best - q @ base
    decoys = np.empty((n_decoys, dims))
    for i, t in enumerate(np.linspace(0.9, 0.15, n_decoys)):
        row = base.copy()
        for c in rng.permutation(np.arange(1, dims)):
            if q @ row >= s_best - t * gap:
                break
            row[c] += 2.0
        assert s_best - t * gap <= q @ row < s_best
        decoys[i] = row
    return q.astype(np.float32), best.astype(np.float32), decoys.astype(np.float32)


@pytest.mark.parametrize("boundary,decoys", [("warp", 126), ("warp", 127), ("warp", 128), ("warp", 129),
                                             ("cta", 254), ("cta", 255), ("cta", 256), ("cta", 257)])
def test_proof_at_the_nominee_boundaries(boundary, decoys):
    dims, n, R = 384, 30_000, 16
    rng = np.random.default_rng(400 + decoys)
    q, best, rows = _u4_hidden_winner(rng, dims, decoys)
    corpus = unit_rows(rng, n, dims)
    if boundary == "warp":                             # the winner and every decoy in warp 0's steps
        where = _warp_rows(0, 16, R, n, decoys + 1)
        winner, placed = where[0], where[1:]
    else:                                              # spread over the 16 warps: no list holds more than 17
        per = [_warp_rows(w, 16, R, n, decoys // 16 + 2) for w in range(16)]
        winner = per[0][0]
        placed = np.array([per[i % 16][1 + i // 16] for i in range(decoys)])
    corpus[winner] = best
    corpus[placed] = rows
    eng = _engine(DOT, corpus, chunk_steps=0, grid=1, u4_warps=16, u4_rows_per_step=R)
    want = fp32(eng, lambda: eng.search(q, 1))
    assert want[0][0] == winner
    d = eng.u4_nominations(q, 1)
    assert d["rho_q"] == 0.0, "q lies on the int8 grid"
    nominated = _check(d, _model(eng, q))
    limit = WARP_KEYS if boundary == "warp" else CTA_KEYS
    if decoys < limit:
        assert winner in nominated.tolist() and d["result"][0][0] == winner, "the winner is a nominee and the answer"
    else:
        assert winner not in nominated.tolist(), "the construction puts the winner behind the boundary"
        assert d["ok"] == 0, "a proof for a query whose best row was never nominated"
    _check_ok(d, q, 1, DOT, _vmax(corpus))
    _check_rescore(eng, d, q, 1, nominated)
    assert bits(routed(eng, lambda: eng.search(q, 1), proven=d["ok"], failed=1 - d["ok"])) == bits(want)
    eng.close()


# ---- 5. the proof flag against its inequality ---------------------------------------------------------------------------

@pytest.mark.parametrize("metric", [COS, DOT], ids=["cos", "dot"])
def test_proof_flag_against_the_inequality(metric):
    """One CTA; 400 near-copies of a row set tau_excl (the cut falls among them), dot rows have norms up to 3 (max|v| =
    3), and a query with one large component gives rho_q some weight.  One planted row scores tau + t eps, t swept
    across 1: the flag must follow the inequality on both sides."""
    dims, n, R = 384, 8_000, 16
    rng = np.random.default_rng(500 + (metric is DOT))
    corpus = unit_rows(rng, n, dims)
    if metric is DOT:
        corpus *= rng.uniform(0.5, 3.0, (n, 1)).astype(np.float32)
        corpus[17] *= np.float32(3.0) / np.linalg.norm(corpus[17])
    q = unit_rows(rng, 1, dims)[0]
    q[0] = 0.5
    qn = float(np.linalg.norm(q.astype(np.float64)))
    qh = q.astype(np.float64) / qn
    x = rng.standard_normal(dims)
    x -= (x @ qh) * qh
    x /= np.linalg.norm(x)
    r0 = 0.6 * qh + 0.8 * x
    dups = np.sort(rng.choice(np.arange(100, n), 400, replace=False))
    corpus[dups] = (r0[None, :] + 1e-4 * rng.standard_normal((400, dims))).astype(np.float32)
    p = 4321
    assert p not in dups
    eng = _engine(metric, corpus, grid=1, u4_rows_per_step=R)
    y = rng.standard_normal(dims)
    y -= (y @ qh) * qh
    y /= np.linalg.norm(y)

    def plant(score):
        a = score / qn
        norm = 1.0 if metric is COS else 1.5
        v = a * qh + np.sqrt(norm * norm - a * a) * y
        eng.add_batch([p], v[None, :].astype(np.float32))

    plant(0.0)
    d = eng.u4_nominations(q, 1)
    tau, eps = d["tau_excl"], _ok_model(d, q, 1, metric, 3.0)[2]
    assert np.isfinite(tau) and np.isfinite(eps) and d["rho_q"] > 0
    seen = []
    for t in np.r_[np.arange(0.8, 0.97, 0.04), np.arange(0.97, 1.0301, 0.0025), np.arange(1.05, 1.21, 0.05)]:
        plant(tau + t * eps)
        corpus[p] = eng.read_rows(p, 1)[0]
        d = eng.u4_nominations(q, 1)
        assert d["result"][0][0] == p, "the planted row is the best"
        _check(d, _model(eng, q))
        ok = _check_ok(d, q, 1, metric, _vmax(corpus))
        seen.append((round(float(t), 4), d["ok"], ok))
        tau, eps = d["tau_excl"], _ok_model(d, q, 1, metric, _vmax(corpus))[2]
    assert {o for _, o, _ in seen} == {0, 1}, f"the sweep did not cross the boundary: {seen}"
    assert all(o == 0 for t, o, _ in seen if t <= 0.985) and all(o == 1 for t, o, _ in seen if t >= 1.015), seen
    eng.close()


def test_nothing_excluded_proves_whatever_the_bound():
    """<= 256 candidate rows leave nothing out: tau_excl = -inf and the proof holds, even on a dot corpus whose huge row
    makes eps enormous -- whether the candidates are the whole corpus or an allow-list."""
    dims = 384
    rng = np.random.default_rng(510)
    corpus = _special_rows(rng, 5_000, dims, DOT)
    q = unit_rows(rng, 1, dims)[0]
    for n, allow in ((200, None), (5_000, np.sort(rng.choice(5_000, 250, replace=False)))):
        eng = _engine(DOT, corpus[:n])
        for k in (1, 10, 32):
            d = eng.u4_nominations(q, k, allow_rows=allow)
            allowed = None
            if allow is not None:
                allowed = np.zeros(n, bool)
                allowed[allow] = True
            rows = _check(d, _model(eng, q), allowed)
            assert d["tau_excl"] == -np.inf and d["ok"] == 1
            assert np.array_equal(np.sort(rows), np.arange(n) if allow is None else allow)
            _check_rescore(eng, d, q, k, rows)
        eng.close()


# ---- 6. the re-score on its own, over grids -----------------------------------------------------------------------------

@pytest.mark.parametrize("metric", [COS, DOT], ids=["cos", "dot"])
def test_rescore_over_grids_and_k(metric):
    """grid 200 and 264 with k = 32: grid * k * 8 > 48 KiB, the re-score's tail reads the block keys from L2."""
    dims, n = 384, 70_001
    rng = np.random.default_rng(600 + (metric is DOT))
    corpus = unit_rows(rng, n, dims)
    qs = unit_rows(rng, 2, dims)
    eng = _engine(metric, corpus)
    _plant(rng, eng, qs[1], rng.choice(n, 40, replace=False), metric)
    corpus = eng.read_rows(0, n)
    vmax = _vmax(corpus)
    for q in qs:
        model = _model(eng, q)
        for grid in (1, 5, 0, 200, 264):
            eng.set_option("grid", grid)
            for k in (1, 10, 32):
                d = eng.u4_nominations(q, k)
                if grid:
                    assert d["grid"] == grid, d
                rows = _check(d, model)
                _check_rescore(eng, d, q, k, rows)
                _check_ok(d, q, k, metric, vmax)
                want = fp32(eng, lambda: eng.search(q, k))
                if d["ok"]:
                    assert bits(d["result"]) == bits(want)
                assert bits(eng.search(q, k)) == bits(want)
                eng.set_option("u4_scan_min_bytes", 0)        # ends a demotion a refused proof may have opened
    eng.close()


# ---- 7. degenerate queries and overflow ----------------------------------------------------------------------------------

@pytest.mark.parametrize("metric", [COS, DOT], ids=["cos", "dot"])
def test_degenerate_queries(metric):
    dims, n, k = 384, 20_000, 10
    rng = np.random.default_rng(700 + (metric is DOT))
    corpus = np.abs(unit_rows(rng, n, dims))
    eng = _engine(metric, corpus)
    names, qs = degenerate_queries(rng, dims)
    one_hot = np.zeros(dims, np.float32)
    one_hot[5] = 1.0
    extra = [("one_hot", one_hot), ("all_negative", -np.abs(unit_rows(rng, 1, dims)[0])),
             ("huge_1e30", (np.float32(1e30) * unit_rows(rng, 1, dims)[0]).astype(np.float32))]
    names = names + [x for x, _ in extra]
    qs = np.concatenate([qs, np.stack([v for _, v in extra])]).astype(np.float32)
    vmax = _vmax(corpus)
    for name, q in zip(names, qs):
        _set(eng, shadow_scan=1, u4_scan_min_bytes=0)     # clears the skip and demotion windows
        d = eng.u4_nominations(q, k)
        finite = np.isfinite(q).all()
        if finite:
            rows = _check(d, _model(eng, q))
            _check_rescore(eng, d, q, k, rows)
            _check_ok(d, q, k, metric, vmax)
            _, _, rho_q = code_query(q)
            assert rho_q <= d["rho_q"] <= rho_q * (1 + 1e-6) + 2.0 ** -148, name    # (+ subnormal ulps)
        else:
            assert d["rho_q"] == np.inf and d["ok"] == 0, f"{name}: a proof for a non-finite query"
        if not np.any(q):
            assert d["ok"] == 0 and d["rho_q"] == 0.0, f"{name}: the zero query"
        want = fp32(eng, lambda: eng.search(q, k))
        if d["ok"]:
            assert bits(d["result"]) == bits(want), name
        _set(eng, shadow_scan=1, u4_scan_min_bytes=0)
        u0 = eng.counter("single_u4_queries")
        assert bits(eng.search(q, k)) == bits(want), name
        assert eng.counter("single_u4_queries") == u0 + 1, f"{name} did not take the 4-bit form"
    eng.close()


def test_overflowing_score_is_nominated_as_inf():
    """Dot rows of +-1e36 code to +-15 h with h = 6.25e34, and q = 8192 * 127 in every component gives s_q = 8192:
    fl(s_q h) overflows, so score' is +inf, -inf, or inf * 0 = NaN for the row whose integer sum is 0.  Each is
    nominated as +inf and re-scored (its exact fp32 score is not finite either: it never enters the answer).  With
    <= 256 rows nothing is left out and the proof holds; with more the infinite bound refuses it."""
    dims, k = 128, 10
    rng = np.random.default_rng(710)
    corpus = unit_rows(rng, 3_000, dims)
    signs = np.where(np.arange(dims) % 2 == 0, 1.0, -1.0)
    corpus[41] = 1e36 * signs                          # sum c (2u - 15) = 0: score' = inf * 0
    corpus[42] = 1e36 * np.abs(signs)                  # +inf
    corpus[43] = -1e36 * np.abs(signs)                 # -inf
    q = np.full(dims, 8192.0 * 127.0, np.float32)
    for n, proven in ((200, 1), (3_000, 0)):
        eng = _engine(DOT, corpus[:n])
        codes, half, _ = eng.read_u4_shadow(41, 3)
        with np.errstate(over="ignore"):
            assert np.isinf(np.float32(8192.0) * half).all()
        assert (2 * codes[0].astype(np.int64) - 15).sum() == 0
        d = eng.u4_nominations(q, k)
        rows, sc = _decode(d["keys"])
        for r in (41, 42, 43):
            assert r in rows.tolist(), f"row {r}: a non-finite score' was not nominated"
            assert sc[rows.tolist().index(r)] == np.inf, f"row {r}: nominated with score' {sc[rows.tolist().index(r)]}"
        _check(d, _model(eng, q))
        _check_rescore(eng, d, q, k, rows)
        assert d["ok"] == proven
        want = fp32(eng, lambda: eng.search(q, k))
        assert 41 not in [i for i, _ in want]
        if proven:
            assert bits(d["result"]) == bits(want)
        eng.set_option("u4_scan_min_bytes", 0)
        assert bits(routed(eng, lambda: eng.search(q, k), proven=proven, failed=1 - proven)) == bits(want)
        eng.close()


# ---- 8. filters and delivery -----------------------------------------------------------------------------------------------

def test_filters_where_and_delivery_on_the_route(oracle):
    import ctypes as Cc
    import torch
    from test_gpu_where import _attributes
    from wax_b200 import Where, _lib as L, sharded
    n, dims, k = 200_000, 384, 10
    eng = CUDAVectorEngine(COS, dims)
    eng.fill_synthetic(800, n, id_base=3)
    _set(eng, shadow_scan_min_bytes=0, u4_scan_min_bytes=0)
    rng = np.random.default_rng(801)
    qs = oracle.synth_rows(802, 0, 3, dims, normalize=True)
    # 40 strong rows per query, inside the time window below: every k <= 32 answer is strong and proven
    planted = np.sort(rng.choice(np.arange(n // 10 + 10, n // 10 + n // 5 - 10), 120, replace=False))
    perm = rng.permutation(planted)
    for i, q in enumerate(qs):
        _plant(rng, eng, q, perm[40 * i:40 * i + 40] + 3, COS)  # frame id = row + 3
    ids = np.arange(n) + 3
    pids = planted + 3
    deny = np.setdiff1d(rng.choice(ids, 30_000, replace=False), pids).tolist()
    allow = np.union1d(rng.choice(ids, 40_000, replace=False), pids).tolist()      # the row bitset
    for kind, fids in (("deny", deny), ("allow", allow)):
        for kk in (1, 10, 32):
            want = fp32(eng, lambda: [eng.search_filtered(q, kk, **{kind: fids}) for q in qs])
            got = _u4_routed(eng, lambda: [eng.search_filtered(q, kk, **{kind: fids}) for q in qs], 3, proven=3)
            assert [bits(g) for g in got] == [bits(w) for w in want], (kind, kk)
    ts, tags = _attributes(np.random.default_rng(803), n)
    tags[planted] = 0
    eng.set_attributes(ids.astype(np.uint64), ts, tags)
    lat, lon = rng.uniform(9.0, 11.0, n), rng.uniform(19.0, 21.0, n)     # the box below holds ~30 % of the frames
    lat[planted], lon[planted] = 10.0, 20.0
    assert eng.set_locations(ids, lat, lon) == n
    for w in (Where(after=int(ts[n // 10]), before=int(ts[n // 10 + n // 5])), Where(no_tags=3),
              Where(near=(10.0, 20.0, 60_000.0)), Where(near=(10.0, 20.0, 60_000.0), no_tags=3)):
        want = fp32(eng, lambda: [eng.search_where(q, k, w) for q in qs])
        got = _u4_routed(eng, lambda: [eng.search_where(q, k, w) for q in qs], 3, proven=3)
        assert [bits(g) for g in got] == [bits(x) for x in want], w
    want = fp32(eng, lambda: [eng.search(q, k) for q in qs])
    for delivery in (1, 0):
        for inline in (1, 0):
            _set(eng, host_delivery=delivery, inline_query=inline)
            got = _u4_routed(eng, lambda: [eng.search(q, k) for q in qs], 3, proven=3)
            assert [bits(g) for g in got] == [bits(w) for w in want], (delivery, inline)
    stream = torch.cuda.Stream()
    d_q = torch.from_numpy(qs).cuda()
    buf = torch.zeros(len(qs) * k * 24, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    (p0, f0), u0 = counts(eng), eng.counter("single_u4_queries")
    rc = L.lib().wax_vs_search_device(eng.handle, Cc.c_void_p(d_q.data_ptr()), len(qs), k, 0,
                                      Cc.c_void_p(buf.data_ptr()), Cc.c_void_p(stream.cuda_stream))
    assert rc == 0, L.last_error()
    stream.synchronize()
    assert counts(eng) == (p0 + len(qs), f0) and eng.counter("single_u4_queries") == u0 + len(qs)
    cands = buf.cpu().numpy().view(sharded.CAND_DTYPE).reshape(len(qs), k)
    for c, w in zip(cands, want):
        assert [int(x["frame_id"]) for x in c] == [i for i, _ in w]
        assert [float(np.float32(1.0) - x["distance"]) for x in c] == [s for _, s in w]
    # frame ids that differ from rows: remove crowd frames in the middle
    gone = np.setdiff1d(rng.choice(ids[: n // 2], 5_000, replace=False), pids)
    eng.remove_batch(gone.tolist())
    assert eng.count == n - gone.size
    want = fp32(eng, lambda: [eng.search(q, k) for q in qs])
    got = _u4_routed(eng, lambda: [eng.search(q, k) for q in qs], 3, proven=3)
    assert [bits(g) for g in got] == [bits(w) for w in want]
    live = np.setdiff1d(ids, gone)                     # removes keep the order: row = rank among the live frames
    assert all(np.searchsorted(live, g[0][0]) != g[0][0] - 3 for g in got), "frame ids and rows should differ here"
    eng.close()


@pytest.mark.parametrize("metric", [COS, DOT], ids=["cos", "dot"])
def test_few_allowed_rows_of_a_large_corpus(metric):
    """An allow-list of <= 255 rows of a 1 M-row corpus at the risky places: the nominees are exactly the allowed rows,
    nothing is cut and the proof holds, in every schedule."""
    dims, n = 384, 1_000_000
    rng = np.random.default_rng(820 + (metric is DOT))
    q = unit_rows(rng, 1, dims)[0]
    eng = _synth(metric, n, dims, 821)
    chunks, R = set(), None
    for _, sched in SCHEDULES:
        _set(eng, **sched)
        d = eng.u4_nominations(q, 10)
        chunks.add(d["chunk_steps"])
        R = d["R"]
    risky = _risky_rows(n, R, chunks)
    for size in (255, 200):
        extra = rng.permutation(np.setdiff1d(rng.choice(n, 600, replace=False), risky))[:size - risky.size]
        allow = np.sort(np.concatenate([risky, extra]))
        assert allow.size == size
        allowed = np.zeros(n, bool)
        allowed[allow] = True
        for _, sched in SCHEDULES:
            _set(eng, **sched)
            for k in (1, 32):
                d = eng.u4_nominations(q, k, allow_rows=allow)
                rows, _ = _decode(d["keys"])
                assert np.array_equal(np.sort(rows), allow), "the nominees are not exactly the allowed rows"
                assert d["tau_excl"] == -np.inf and d["ok"] == 1
                _check_rescore(eng, d, q, k, rows)
    eng.close()


# ---- 9. state between queries --------------------------------------------------------------------------------------------

def test_state_between_queries():
    """A full query leaves a cut, which the re-score must reset: a following <= 256-row allow-list query reads
    tau_excl = -inf and proves.  The U4 scan's tail has no last CTA, so the re-score also resets the claim counter: a
    dynamic scan after it (U4 or fp32) must see every row."""
    dims, n, k = 384, 60_000, 10
    rng = np.random.default_rng(900)
    corpus = unit_rows(rng, n, dims)
    qs = unit_rows(rng, 3, dims)
    eng = _engine(COS, corpus)
    for i, q in enumerate(qs):
        _plant(rng, eng, q, rng.choice(n, 12, replace=False), COS)
    small = np.sort(rng.choice(n, 200, replace=False))
    allowed = np.zeros(n, bool)
    allowed[small] = True
    want = fp32(eng, lambda: [eng.search(q, k) for q in qs])
    want_small = fp32(eng, lambda: [eng.search_filtered(q, k, allow=small.tolist()) for q in qs])
    for rnd in range(2):
        for sched in ("dynamic", "static", "dynamic"):
            eng.set_option("chunk_steps", -1 if sched == "dynamic" else 0)
            for i, q in enumerate(qs):
                model = _model(eng, q) if rnd == 0 else None
                d = eng.u4_nominations(q, k)
                assert d["tau_excl"] > -np.inf, "a full query over 60 000 rows cuts"
                if model is not None:
                    _check(d, model)
                assert bits(d["result"]) == bits(want[i]) and d["ok"] == 1, (sched, i)
                d = eng.u4_nominations(q, k, allow_rows=small)
                assert d["tau_excl"] == -np.inf and d["ok"] == 1, "a stale cut word from the query before"
                assert np.array_equal(np.sort(_decode(d["keys"])[0]), small)
                assert bits(d["result"]) == bits(want_small[i])
                assert bits(fp32(eng, lambda: eng.search(q, k))) == bits(want[i])
                batch = eng.search_batch(qs, k)
                assert [bits(b) for b in batch] == [bits(w) for w in want]
                assert bits(_u4_routed(eng, lambda: eng.search(q, k), 1, proven=1)) == bits(want[i])
    eng.close()


def test_two_contexts_run_the_route_concurrently():
    dims, n, k, rounds = 384, 80_000, 10, 25
    rng = np.random.default_rng(910)
    corpus = unit_rows(rng, n, dims)
    qs = unit_rows(rng, 4, dims)
    eng = _engine(COS, corpus, int8_scan_min_bytes=0)
    for q in qs:
        _plant(rng, eng, q, rng.choice(n, 12, replace=False), COS)
    want = fp32(eng, lambda: [eng.search(q, k) for q in qs])
    (p0, f0), u0, i0 = counts(eng), eng.counter("single_u4_queries"), eng.counter("single_int8_queries")
    errors, got = [], {0: [], 1: []}

    def worker(t):
        try:
            for r in range(rounds):
                for j in (2 * t, 2 * t + 1):
                    got[t].append((j, eng.search(qs[j], k)))
        except Exception as exc:            # surfaced below
            errors.append(exc)

    threads = [threading.Thread(target=worker, args=(t,)) for t in (0, 1)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    for t in (0, 1):
        assert len(got[t]) == 2 * rounds
        for j, g in got[t]:
            assert bits(g) == bits(want[j]), (t, j)
    total = 4 * rounds
    (p1, f1) = counts(eng)
    assert (p1 - p0) + (f1 - f0) == total, "the proof counts do not add up"
    u, i8 = eng.counter("single_u4_queries") - u0, eng.counter("single_int8_queries") - i0
    assert u + i8 == total and u >= total // 2, (u, i8)
    eng.close()


# ---- 10. lifecycle and demotion ------------------------------------------------------------------------------------------

def test_lifecycle_overwrite_remove_deserialize_fill():
    dims, n, k = 384, 50_000, 10
    rng = np.random.default_rng(1000)
    corpus = unit_rows(rng, n, dims)
    q = unit_rows(rng, 1, dims)[0]
    eng = _engine(COS, corpus)
    _plant(rng, eng, q, rng.choice(np.arange(30_000, n), 12, replace=False), COS)

    def same(proven=1):
        want = fp32(eng, lambda: eng.search(q, k))
        got = _u4_routed(eng, lambda: eng.search(q, k), 1, proven=proven)
        assert bits(got) == bits(want)
        assert eng.counter("u4_shadow_rows") == eng.count
        return got

    same()
    eng.add_batch([777], (q * np.float32(3.0))[None, :])      # overwrite in place: the new best
    assert same()[0][0] == 777
    codes, half, _ = eng.read_u4_shadow(777, 1)
    u, h, _ = code_rows(_vhat(COS, (q * np.float32(3.0))[None, :]))
    assert np.abs(codes.astype(np.int32) - u).max() <= 1 and np.allclose(half, h, rtol=2.0 ** -21)
    eng.remove_batch(list(range(20_000, 20_100)) + [777])     # remove in the middle, then append
    extra = unit_rows(rng, 300, dims)
    extra[5] = q
    eng.add_batch(list(range(10 ** 6, 10 ** 6 + 300)), extra)
    assert same()[0][0] == 10 ** 6 + 5
    other = _engine(COS, unit_rows(rng, 30_000, dims))
    _plant(rng, other, q, rng.choice(30_000, 12, replace=False), COS)
    eng.deserialize(other.serialize())
    other.close()
    assert eng.count == 30_000
    same()
    eng.fill_synthetic(1001, 40_000, normalize=True)
    assert eng.count == 40_000
    want = fp32(eng, lambda: eng.search(q, k))
    u0 = eng.counter("single_u4_queries")
    assert bits(eng.search(q, k)) == bits(want)
    assert eng.counter("single_u4_queries") == u0 + 1 and eng.counter("u4_shadow_rows") == 40_000
    eng.close()


def test_demotion_window_doubles_and_resets():
    """On one tight cluster the 4-bit proof fails: after each failed probe the next window of eligible queries takes
    the int8 form, 16, then 32, then 64; a probe that holds resets the window to 16; setting u4_scan_min_bytes ends it."""
    rng = np.random.default_rng(1100)
    n, dims, k = 9000, 384, 10
    base = (rng.choice([-1.0, 1.0], dims) / np.sqrt(dims)).astype(np.float32)
    corpus = (base + 0.01 * rng.standard_normal((n, dims))).astype(np.float32)
    # a second query with 12 strong rows built from sign vectors like the cluster's (no larger element: the int8 shadow
    # stays fine enough to be the form a demoted query takes)
    q2 = (rng.choice([-1.0, 1.0], dims) / np.sqrt(dims)).astype(np.float32)
    c = np.linspace(0.7, 0.95, 12)[:, None]
    rows2 = rng.choice(n, 12, replace=False)
    eng = _engine(COS, corpus, int8_scan_min_bytes=0, grid=2)
    eng.add_batch(rows2.tolist(), (c * q2[None, :] + np.sqrt(1 - c * c) * base[None, :]).astype(np.float32))
    wants = {0: fp32(eng, lambda: eng.search(base, k)), 1: fp32(eng, lambda: eng.search(q2, k))}
    d = eng.u4_nominations(q2, k)
    assert d["ok"] == 1, "the second query must prove on the 4-bit form"
    assert eng.u4_nominations(base, k)["ok"] == 0, "the cluster query must not"
    eng.set_option("u4_scan_min_bytes", 0)

    def step(which):
        u0, i0, (p0, f0) = eng.counter("single_u4_queries"), eng.counter("single_int8_queries"), counts(eng)
        assert bits(eng.search(q2 if which else base, k)) == bits(wants[which])
        routed_now = eng.counter("single_u4_queries") > u0 or eng.counter("single_int8_queries") > i0
        t0 = time.monotonic()          # the proof counts reach the host mirror without synchronisation: wait for them
        while routed_now and sum(counts(eng)) == p0 + f0 and time.monotonic() - t0 < 1.0:
            time.sleep(1e-4)
        (p1, f1) = counts(eng)
        if eng.counter("single_u4_queries") > u0:
            log.append("u" + ("+" if p1 > p0 else "-"))
        else:
            log.append("i" if eng.counter("single_int8_queries") > i0 else "f")
        return log[-1]

    log = []

    def window():
        """int8 queries until the next 4-bit probe (issued with the cluster query)."""
        n_i = 0
        for _ in range(5000):          # (a failed int8 proof opens a skip window of its own in between)
            e = step(0)
            if e[0] == "u":
                assert e == "u-"
                return n_i
            n_i += e == "i"
        raise AssertionError("no 4-bit probe")

    assert step(0) == "u-"
    assert [window() for _ in range(2)] == [16, 32], " ".join(log)
    n_i = 0
    while n_i < 64:                                    # the third window: 64, then the probe with the proving query
        e = step(0)
        assert e[0] != "u", f"the 4-bit form was probed after {n_i} int8 queries of a 64-query window"
        n_i += e == "i"
    e = step(1)
    while e == "f":
        e = step(1)
    assert e == "u+", "the probe after the window should be the proving query's"
    assert step(0) == "u-"
    assert window() == 16, "a probe that held resets the window to 16"
    assert step(0) == "i"                              # the failed probe opened the next window ...
    eng.set_option("shadow_scan", 1)                   # (closes the skip window a failed int8 proof opens, only that)
    assert step(0) == "i"
    eng.set_option("shadow_scan", 1)
    eng.set_option("u4_scan_min_bytes", 0)
    assert step(0) == "u-", "setting u4_scan_min_bytes ends the window"
    eng.close()
