"""The fp32 scan in every form it compiles, bit for bit (DESIGN 4.1, 4.2).

scan_tma_kernel and scan_ldg_kernel are the exact answer of the engine: the single-query path, the guarded last launch
of every shadow route, the batched levels' fall-backs, the keys-only pass of grouped search and the filtered, where and
sharded searches all end in them.  Here the route is off (shadow_scan = 0), so every search is the fp32 scan alone, and
each row length is run in every form it admits:

  * unrolled lengths (C x 128 elements) in both compiled rows-per-step R, generic lengths (C = 0) in every R of
    {1, 2, 4, 8} whose ring fits the 227 KB of shared memory an H100 CTA may opt into;
  * crossed with the three metrics, k on both sides of the list sizes (32, 128) and of the fused limit, both tails
    (pairwise merges, radix select with the grid's keys staged in shared memory or read from L2), dynamic claims of
    1, 3 and auto steps and static claims, grids of 1, 7 and one CTA per SM, 1 - 3 stages, 1, default and the most
    warps that fit, the L2 hint, the query in the kernel parameters or in device memory, host delivery on and off, and
    a row filter;
  * the direct-load kernel at every length, with 1, 4 and 8 CTAs per SM, and at the lengths no TMA form takes.

wax_vs_debug_last_scan (CUDAVectorEngine.last_scan) reports the form each search actually ran, so a forced option
that silently fell back to the defaults or to the direct-load kernel fails the test.  Every answer must carry the ids
and score bits of the ACC_F32_TREE oracle (the kernels' own accumulation order), computed once per (corpus, query,
metric) -- so every form at one length is bit-identical to every other -- and meet the fp64 tolerance of
test_gpu_parity._check.  After each form one default search runs again: a work counter or ticket the last CTA failed to
reset would change it.

The corpora hold what these kernels get wrong: winners at every row-in-step position (every reduce-scatter owner
lane), at the first and last step of a claim, in the ragged last step and at the last row; rows whose scores rise
with the row (every step inserts into every list: the E = 4 list's flush with more than 32 keys pending); exact
duplicates across steps, warps, claims and the 32 / 33 and 128 list boundaries; NaN and +-Inf rows right before the
ragged step (the reused stage holds non-finite data past n_rows); NaN in the first element of the row after each
winner (the ragged-chunk break at dims % 128 != 0); zero rows, dot rows whose score overflows, and a corpus with
fewer finite rows than k.
"""
import functools
import math

import numpy as np
import pytest
import torch

from wax_b200 import CUDAVectorEngine, InvalidToc, VectorMetric

from helpers import assert_tie_aware_order

pytestmark = pytest.mark.gpu
TOL = 1e-4                              # test_gpu_parity: fp64 score tolerance (x dims for dot and l2)

UNROLLED = {128: (4, 8), 256: (4, 8), 384: (4, 8), 512: (4, 8), 768: (2, 4), 1024: (2, 4), 1536: (1, 2)}
GENERIC = (32, 36, 100, 252, 260, 516, 644, 1000, 2052, 3076, 4096)
# the (C, R) shapes launch_tma compiles, each in three metrics x three modes
COMPILED = [(1, 4), (1, 8), (2, 4), (2, 8), (3, 4), (3, 8), (4, 4), (4, 8), (6, 2), (6, 4), (8, 2), (8, 4), (12, 1),
            (12, 2), (0, 1), (0, 2), (0, 4), (0, 8)]
# pick_tma_config's shared-memory arithmetic: the opt-in limit of an H100 CTA (227 KB) less 4 KB of static shared memory;
# a ring takes warps x stages x (stage + barrier + step slot) + each warp's list, and a generic length its query copy
BUDGET = 232448 - 4096
FUSED_KS = (1, 31, 32, 33, 64, 65, 97, 128)
EMIT_KS = (129, 1000)
KMAX = 1000
DEFAULTS = {"variant": 0, "rows_per_step": 0, "stages": 0, "warps": 0, "grid": 0, "chunk_steps": -1, "l2_hint": 0,
            "fused_k_max": 128, "tail_select": 1, "inline_query": 1, "host_delivery": 1, "ldg_ctas_per_sm": 4,
            "tma_max_dims": 4096}
SEEN = set()                            # (dims, kernel, C, R, metric, mode, tail) of every search run
LENGTHS_RUN = set()


def _unrolled_c(dims):
    return dims // 128 if dims in UNROLLED else 0


def _ring_bytes(dims, R, warps, stages):
    query = dims * 4 + 512 + 32 if dims not in UNROLLED else 0
    return warps * stages * (R * dims * 4 + 8 + 4) + warps * 1024 + 16 + query


def _fits(dims, R, warps=2, stages=2):
    return _ring_bytes(dims, R, warps, stages) <= BUDGET


def _forms(dims):
    return UNROLLED[dims] if dims in UNROLLED else tuple(r for r in (1, 2, 4, 8) if _fits(dims, r))


def _rows(dims):
    return 40_013 if dims <= 2048 else 6_007     # n % 8 = 5 / 7: a ragged last step for every R > 1


@functools.lru_cache(maxsize=None)
def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- corpora ---------------------------------------------------------------------------------------------------------
def _toward(q, u, cos):
    """A unit row whose cosine to the unit q is `cos`, leaning towards u (any direction)."""
    u = u - np.dot(u, q) * q
    u /= np.linalg.norm(u)
    return (cos * q + math.sqrt(max(0.0, 1.0 - cos * cos)) * u).astype(np.float32)


def _winner_rows(n):
    """Every row-in-step position r < 8 (the owner lanes of every R) at the first and the last step of a claim, a claim
    boundary (192 = 8 x 24 rows: a multiple of R x chunk_steps for every R and chunk_steps 1, 3 and 8), a row of the
    ragged last step and the last row."""
    mid, mid2 = 192 * (n // 384), 192 * ((3 * n) // (4 * 192))
    return sorted({*range(8), 191, 192, *range(mid, mid + 8), *range(mid2 - 8, mid2), n - 3, n - 1})


def planted_corpus(oracle, dims, metric, seed):
    n = _rows(dims)
    rng = np.random.default_rng(seed)
    x = oracle.synth_rows(seed, 0, n, dims, normalize=True)
    q = oracle.synth_row(seed + 1, 0, dims, True)
    winners = _winner_rows(n)
    for j, r in enumerate(winners):                       # distinct scores, 0.999 down to ~0.94
        x[r] = _toward(q, rng.standard_normal(dims), 0.999 - 0.002 * j)
    mid = 192 * (n // 384)
    dups = [r for r in [*range(mid + 100, mid + 140), *(1000 + 37 * j for j in range(110))] if r not in winners]
    x[dups] = _toward(q, rng.standard_normal(dims), 0.93)  # ranks 29 .. ~178: cut by k = 32, 33, 64, ..., 129
    for r in (500, 501, n - 30):
        x[r] = 0.0                                        # cosine: distance 1 (USearch zero-norm rule)
    if metric is not VectorMetric.cosine:                 # q.v and |q - v|^2 overflow fp32 (and the fp64 result's cast)
        x[600] = x[601] = np.float32(2e38) * np.where(q >= 0, 1, -1).astype(np.float32)
    bad = (np.nan, np.inf, -np.inf)
    for i, r in enumerate(range(n - 24, n - 1)):          # the steps before the ragged one of every R: NaN and +-Inf
        if r != n - 3:
            x[r] = bad[i % 3]
    for w in winners:                                     # the ragged-chunk break: NaN right after a winner's last element
        if w + 1 < n - 24 and w + 1 not in winners and w + 1 not in dups:
            x[w + 1, 0] = np.nan
    allow = np.ones(n, bool)                              # a row filter: drops every third winner and a run of duplicates
    allow[winners[::3]] = False
    allow[mid + 100:mid + 110] = False
    allow[7777 % n::1013] = False
    return x, q, allow


def monotone_corpus(oracle, dims, seed):
    """Row i scores above row i - 1 in every metric (cos to q rises from 0 to ~0.88, 1e-5 a row at least): every step
    inserts into every list."""
    n = _rows(dims)
    q = oracle.synth_row(seed + 1, 0, dims, True)
    u = oracle.synth_rows(seed, 0, n, dims, normalize=False)
    u -= np.outer(u @ q, q)
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    theta = np.pi / 2 - (np.pi / 2 - 0.5) * np.arange(n) / (n - 1)
    x = (np.cos(theta)[:, None] * q[None, :] + np.sin(theta)[:, None] * u).astype(np.float32)
    return x, q


def sparse_corpus(oracle, dims, seed):
    """Fewer finite rows than k: 100 spread rows, the rest NaN or +-Inf."""
    n = _rows(dims)
    x = np.full((n, dims), np.nan, np.float32)
    x[1::7] = np.inf
    x[2::7] = -np.inf
    keep = np.linspace(0, n - 1, 100).astype(np.int64)
    x[keep] = oracle.synth_rows(seed, 0, 100, dims, normalize=True)
    return x, oracle.synth_row(seed + 1, 0, dims, True)


# ---- the oracle, once per (corpus, query, metric) ---------------------------------------------------------------------
class Truth:
    """The ACC_F32_TREE and fp64 answers of one (corpus, query, metric) at KMAX; the answer for k is their prefix (the
    order distance, row is total).  `allow`: a row filter -- denied rows become NaN rows, which every mode drops."""

    def __init__(self, oracle, metric, corpus, q, allow=None):
        if allow is not None:
            corpus = corpus.copy()
            corpus[~allow] = np.nan
        self.metric, self.dims = metric, corpus.shape[1]
        self.rows, _, self.s = oracle.search(metric.value, corpus, q, KMAX, mode=oracle.ACC_F32_TREE,
                                             threads=oracle.host_threads())
        self.r64, _, self.s64 = oracle.search(metric.value, corpus, q, KMAX + 1, mode=oracle.ACC_F64,
                                              threads=oracle.host_threads())
        self.checked = set()

    def check(self, got, k, what):
        want = min(k, len(self.rows))
        ids = [g[0] for g in got]
        assert ids == self.rows[:want].tolist(), f"{what}: ids differ from the ACC_F32_TREE oracle"
        bits = np.float32([g[1] for g in got]).view(np.uint32)
        assert np.array_equal(bits, self.s[:want].view(np.uint32)), f"{what}: score bits differ"
        if k not in self.checked:      # the fp64 check of these bits (every other form has the same bits)
            self.checked.add(k)
            scale = 1.0 if self.metric is VectorMetric.cosine else float(self.dims)
            s64 = self.s64.astype(np.float64)
            assert np.max(np.abs(np.float64([g[1] for g in got]) - s64[:want]), initial=0.0) <= TOL * scale, what
            assert_tie_aware_order(ids, self.r64[:want].tolist(), s64, 2e-6 * scale)


# ---- one engine, its forms and the read-out ----------------------------------------------------------------------------
class Bench:
    def __init__(self, metric, corpus, q, truth, length_tag):
        self.metric, self.q, self.truth = metric, q, truth
        self.n, self.dims = corpus.shape
        self.tag = length_tag
        self.eng = CUDAVectorEngine(metric, self.dims)
        self.eng.add_batch(np.arange(self.n, dtype=np.uint64), corpus)
        self.eng.set_option("shadow_scan", 0)
        self.opts = dict(DEFAULTS)
        self.set({})

    def close(self):
        self.eng.close()

    def set(self, opts):
        want = dict(DEFAULTS, **opts)
        for key, v in want.items():
            if self.opts.get(key) != v:
                self.eng.set_option(key, v)
        self.opts = want

    def search(self, k, allow=None, truth=None):
        # the filter goes in as a deny-list: it reaches the scan at every corpus size, where an allow-list of at most
        # 16 384 rows is scored by the gather path instead (plan_filtered)
        got = (self.eng.search(self.q, k) if allow is None
               else self.eng.search_filtered(self.q, k, deny=np.flatnonzero(~allow).tolist()))
        form = self.eng.last_scan()
        what = f"{self.tag} {self.metric.name} k={k} {self.opts_diff()} ran {form}"
        (truth or self.truth).check(got, k, what)
        self.expect(form, k, filtered=allow is not None, what=what)
        SEEN.add((self.dims, form["kernel"], form["C"], form["R"], self.metric.name, form["mode"], form["tail"]))
        return form

    def opts_diff(self):
        return {k: v for k, v in self.opts.items() if DEFAULTS[k] != v}

    def expect(self, form, k, filtered, what):
        """The form the options ask for, field by field."""
        o, dims = self.opts, self.dims
        k_eff = min(k, self.n)
        emit = k_eff > o["fused_k_max"]
        mode = 2 if emit else (0 if k_eff <= 32 else 1)
        tma = o["variant"] != 2 and dims % 4 == 0 and dims >= 32 and (dims in UNROLLED or dims <= o["tma_max_dims"])
        if tma and o["rows_per_step"]:     # an explicit warp count is kept; auto warps shrink to 2 before giving up
            tma = _fits(dims, o["rows_per_step"], o["warps"] or 2, o["stages"] or 2)
        assert form["kernel"] == (1 if tma else 2), what
        assert form["mode"] == mode, what
        assert form["grid"] >= 1 and (not o["grid"] or form["grid"] == o["grid"]), what
        if not tma:
            assert (form["C"], form["R"], form["warps"], form["stages"], form["chunk_steps"], form["tail"],
                    form["inline_query"]) == (0, 1, 8, 0, 0, 0, 0), what
            if not o["grid"]:
                assert form["grid"] == min(_sm_count() * o["ldg_ctas_per_sm"], (self.n + 7) // 8), what
            return
        assert form["C"] == _unrolled_c(dims), what
        if o["rows_per_step"]:
            assert form["R"] == o["rows_per_step"], what
        if o["warps"]:
            assert form["warps"] == o["warps"], what
        assert form["stages"] == (o["stages"] or 2), what
        steps = (self.n + form["R"] - 1) // form["R"]
        if not o["grid"]:
            assert form["grid"] == min(_sm_count(), (steps + form["warps"] - 1) // form["warps"]), what
        if emit:
            chunk = 0
        elif o["chunk_steps"] < 0:
            chunk = max(1, min(8, steps // (form["grid"] * form["warps"] * 2)))
        else:
            chunk = o["chunk_steps"]
        assert form["chunk_steps"] == chunk, what
        if emit or not o["tail_select"]:
            tail = 0
        else:   # finish_topk_select's own test: the grid's k keys per CTA fit the idle ring
            ring = form["warps"] * form["stages"] * form["R"] * dims * 4
            tail = 1 if form["grid"] * k_eff * 8 <= ring else 2
        assert form["tail"] == tail, what
        inline = (not filtered and o["host_delivery"] and o["inline_query"] and not emit and dims <= 512)
        assert form["inline_query"] == int(bool(inline)), what

    def run(self, opts, ks, allow=None, truth=None):
        """The searches of one form, then one default search: the form must leave the scratch state as it found it."""
        self.set(opts)
        forms = [self.search(k, allow, truth) for k in ks]
        self.set({})
        self.search(32)
        return forms


def _max_warps(dims, R, stages=2):
    return max(w for w in range(1, 17) if _ring_bytes(dims, R, w, stages) <= BUDGET)


def _every_setting(b, dims, R, allow, filtered_truth):
    """Every setting crossed with the form (dims, R) on the planted corpus."""
    f = {"variant": 1, "rows_per_step": R}
    tails = set()
    for opts, ks in (
            ({}, FUSED_KS + EMIT_KS),
            ({"fused_k_max": 32}, (33, 64, 65, 97, 128)),       # 33 .. 128 through emit + select
            ({"tail_select": 0}, (1, 32, 33, 128)),
            ({"grid": 7}, (1, 32, 128)),
            ({"warps": 1, "stages": 1}, (1, 33, 128)),          # a tiny ring: the grid's keys are read from L2
            ({"chunk_steps": 1}, (32, 97)),
            ({"chunk_steps": 3}, (31, 65)),
            ({"chunk_steps": 0}, (32, 128)),                    # static claims
            ({"grid": 1}, (1, 128)),
            ({"stages": 1}, (32, 64)),
            ({"l2_hint": 1}, (32, 128)),
            ({"inline_query": 0}, (32,)),
            ({"host_delivery": 0}, (32, 128))):
        tails |= {form["tail"] for form in b.run({**f, **opts}, ks)}
    if _fits(dims, R, 2, 3):
        b.run({**f, "stages": 3}, (33,))
    w = _max_warps(dims, R)
    b.run({**f, "warps": w}, (32, 128))
    if w < 16:      # one warp more does not fit: refused, not quietly run in another form
        b.set({**f, "warps": w + 1})
        with pytest.raises(InvalidToc, match=r"rc=-8"):
            b.eng.search(b.q, 32)
        b.set({})
    b.run(f, (32, 128), allow=allow, truth=filtered_truth)
    return tails


@pytest.mark.parametrize("dims", sorted([*UNROLLED, *GENERIC]))
def test_every_form_at_length(oracle, dims):
    n = _rows(dims)
    forms = _forms(dims)
    print(f"\n{dims} dims, {n} rows: R in {forms}")
    for mi, metric in enumerate(VectorMetric):
        seed = 9000 + 10 * dims + mi
        corpus, q, allow = planted_corpus(oracle, dims, metric, seed)
        truth, filtered = Truth(oracle, metric, corpus, q), Truth(oracle, metric, corpus, q, allow)
        b = Bench(metric, corpus, q, truth, f"{dims}d planted")
        try:
            tails = set()
            for R in forms:
                tails |= _every_setting(b, dims, R, allow, filtered)
            assert {1, 2} <= tails, f"{dims} {metric.name}: both select-tail branches must run, got {tails}"
            for R in (1, 2, 4, 8):       # a ring that does not fit: the direct-load kernel, or refused when forced
                if dims in UNROLLED or R in forms:
                    continue
                b.run({"rows_per_step": R}, (32, 1000))
                b.set({"variant": 1, "rows_per_step": R})
                with pytest.raises(InvalidToc, match=r"rc=-8"):
                    b.eng.search(q, 32)
                b.set({})
            for ctas in (1, 4, 8):         # the direct-load kernel, same bits
                b.run({"variant": 2, "ldg_ctas_per_sm": ctas}, (1, 32, 33, 128, 1000))
        finally:
            b.close()
        for name, (corpus, q) in (("monotone", monotone_corpus(oracle, dims, seed)),
                                  ("sparse", sparse_corpus(oracle, dims, seed))):
            b = Bench(metric, corpus, q, Truth(oracle, metric, corpus, q), f"{dims}d {name}")
            try:
                for R in forms:
                    f = {"variant": 1, "rows_per_step": R}
                    b.run(f, FUSED_KS + EMIT_KS)
                    b.run({**f, "fused_k_max": 32}, (33, 97, 128))
                    b.run({**f, "tail_select": 0}, (32, 128))
                    b.run({**f, "warps": 1, "stages": 1}, (32, 128))
                    b.run({**f, "chunk_steps": 0}, (32, 128))
                    b.run({**f, "grid": 7, "chunk_steps": 1}, (33, 128))
                b.run({"variant": 2}, (32, 128, 1000))
            finally:
                b.close()
    here = [s[1:] for s in SEEN if s[0] == dims]
    for metric in VectorMetric:
        for R in forms:
            modes = {s[4] for s in here if s[:3] == (1, _unrolled_c(dims), R) and s[3] == metric.name}
            assert modes == {0, 1, 2}, (dims, R, metric.name, modes)
    ran = sorted({(s[1], s[2], s[4], s[5]) for s in here if s[0] == 1})
    print("  (C, R, mode, tail) ran:", ran)
    LENGTHS_RUN.add(dims)


def _plain_corpus(oracle, dims, n, seed):
    x = oracle.synth_rows(seed, 0, n, dims, normalize=True)
    x[n // 3] = x[n // 2]                       # an exact duplicate
    x[n // 5] = 0.0
    x[n // 7, dims // 2] = np.nan
    return x, oracle.synth_row(seed + 1, 0, dims, True)


@pytest.mark.parametrize("dims", [1, 3, 5, 31, 33, 127, 4099, 10_001, 65_537])
def test_direct_load_lengths(oracle, dims):
    """Lengths no TMA form takes (dims % 4 != 0): the direct-load kernel alone; forcing the TMA kernel is refused."""
    n = 301
    for mi, metric in enumerate(VectorMetric):
        corpus, q = _plain_corpus(oracle, dims, n, 7000 + dims + mi)
        b = Bench(metric, corpus, q, Truth(oracle, metric, corpus, q), f"{dims}d direct")
        try:
            for ctas in (1, 4, 8):
                b.run({"ldg_ctas_per_sm": ctas}, (1, 32, 33, 128, 129, 1000))
            b.run({"grid": 1}, (1, 128))
            b.set({"variant": 1})
            with pytest.raises(InvalidToc, match=r"rc=-8"):
                b.eng.search(q, 32)
            b.set({})
        finally:
            b.close()


def test_tma_max_dims(oracle):
    """tma_max_dims moves the generic TMA shape's limit: raised to 8 192, C = 0 runs 6 000 and 8 192 dims with the
    direct-load kernel's bits; at 0 every generic length goes direct-load, and the unrolled lengths stay TMA."""
    for dims in (6000, 8192):
        corpus, q = _plain_corpus(oracle, dims, 2003, 7100 + dims)
        for metric in VectorMetric:
            b = Bench(metric, corpus, q, Truth(oracle, metric, corpus, q), f"{dims}d long")
            try:
                b.run({}, (32, 128, 1000))                      # default limit 4 096: direct-load
                b.set({"variant": 1})
                with pytest.raises(InvalidToc, match=r"rc=-8"):
                    b.eng.search(q, 32)
                forms = b.run({"variant": 1, "tma_max_dims": 8192}, FUSED_KS + EMIT_KS)
                assert all((f["kernel"], f["C"], f["R"]) == (1, 0, 1) for f in forms)
                b.run({"variant": 1, "tma_max_dims": 8192, "tail_select": 0, "grid": 7}, (33, 128))
                b.run({"variant": 2, "tma_max_dims": 8192}, (32, 128, 1000))
            finally:
                b.close()
    for dims in (100, 1000, 384):
        corpus, q = _plain_corpus(oracle, dims, 5003, 7200 + dims)
        b = Bench(VectorMetric.cosine, corpus, q, Truth(oracle, VectorMetric.cosine, corpus, q), f"{dims}d")
        try:
            forms = b.run({"tma_max_dims": 0}, (32, 128))
            assert all(f["kernel"] == (1 if dims in UNROLLED else 2) for f in forms)
            if dims not in UNROLLED:
                b.set({"variant": 1, "tma_max_dims": 0})
                with pytest.raises(InvalidToc, match=r"rc=-8"):
                    b.eng.search(q, 32)
        finally:
            b.close()


def test_every_compiled_form_ran():
    """The union of the length tests: every (C, R) of launch_tma's switch in every metric and mode, both select tails."""
    missing = sorted({*UNROLLED, *GENERIC} - LENGTHS_RUN)
    if missing:
        pytest.skip(f"lengths not run in this session: {missing}")
    tma = {s[1:] for s in SEEN if s[1] == 1}
    for C, R in COMPILED:
        for metric in VectorMetric:
            for mode in (0, 1, 2):
                assert any(s[1:5] == (C, R, metric.name, mode) for s in tma), (C, R, metric.name, mode)
    assert {1, 2} <= {s[5] for s in tma}
    print("\nforms run (C, R, mode, tail):")
    for form in sorted({(s[1], s[2], s[4], s[5]) for s in tma}):
        print("  ", form)
