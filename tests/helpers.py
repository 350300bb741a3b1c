"""Shared test helpers: a list-based model of the engine's mutation semantics, comparators, test corpora."""
from __future__ import annotations

import json
from pathlib import Path

import numpy as np

GOLDEN = Path(__file__).resolve().parent / "golden"


class EngineModel:
    """Reference mutation semantics (MetalVectorEngine.swift:330-444) on plain Python lists:
    upsert by frameId (overwrite in place, else append), order-preserving remove, no-op for unknown ids.
    Search goes through the oracle."""

    def __init__(self, oracle, metric: int, dims: int):
        self.o, self.metric, self.dims = oracle, metric, dims
        self.ids: list[int] = []
        self.rows: list[np.ndarray] = []

    def add(self, frame_id, vector):
        v = np.asarray(vector, np.float32)
        assert v.size == self.dims
        if frame_id in self.ids:
            self.rows[self.ids.index(frame_id)] = v
        else:
            self.ids.append(frame_id)
            self.rows.append(v)

    def add_batch(self, frame_ids, vectors):
        for i, v in zip(frame_ids, vectors):
            self.add(i, v)

    def remove(self, frame_id):
        if frame_id in self.ids:
            idx = self.ids.index(frame_id)
            del self.ids[idx]
            del self.rows[idx]

    def corpus(self):
        return np.stack(self.rows).astype(np.float32) if self.rows else np.zeros((0, self.dims), np.float32)

    def search(self, query, top_k, mode=None):
        mode = self.o.ACC_F32_TREE if mode is None else mode
        if not self.rows:
            return []
        rows, d, s = self.o.search(self.metric, self.corpus(), query, top_k, mode=mode)
        return [(self.ids[int(r)], float(sc)) for r, sc in zip(rows, s)]


def assert_tie_aware_order(got_ids, ref_ids, ref_scores_f64, tol):
    """ids must match position by position, except inside groups whose fp64-oracle scores are within `tol`
    of each other (where fp32 rounding order may legitimately permute neighbours)."""
    got_ids, ref_ids = list(got_ids), list(ref_ids)
    assert len(got_ids) == len(ref_ids)
    i = 0
    n = len(ref_ids)
    while i < n:
        j = i
        while j + 1 < n and abs(ref_scores_f64[j + 1] - ref_scores_f64[j]) <= tol:
            j += 1
        # positions i..j form a near-tie group; the last group may also trade members with rank n+1.. if the
        # boundary is a near tie -- callers pass one extra reference row to detect that.
        assert sorted(got_ids[i:j + 1]) == sorted(ref_ids[i:j + 1]) or j == n - 1, (
            f"order differs outside a near-tie at ranks {i}..{j}: got {got_ids[i:j + 1]} ref {ref_ids[i:j + 1]}")
        i = j + 1


def load_json(name):
    return json.loads((GOLDEN / name).read_text())


def unit_rows(rng, n, dims):
    x = rng.standard_normal((n, dims))
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


def hidden_winner(rng, dims, n, bf16, n_decoys, scale_log2=0):
    """Dot query q and a corpus whose first 1 + n_decoys rows (one slice: the first tile) are the true best row (row 0)
    and decoys.  q and the decoys have components exactly representable in bf16 (hence TF32), so their score' is exact
    up to accumulation; the best row's components sit just below a TF32 rounding midpoint that lies just below a bf16
    midpoint, so TF32 (rounded or truncated) loses ~2^-11 and bf16 ~2^-8 of every component: its score' drops below
    every decoy, whose exact scores are spread over (0.1, 0.9) of that loss below the best score.  The other rows are
    unrelated unit rows.  Rows 0..n_decoys are scaled by 2^scale_log2 (exact)."""
    q = 1.0 + rng.integers(0, 4, dims) * 2.0 ** -7
    lo = 1.0 + rng.integers(0, 4, dims) * 2.0 ** -7                     # the bf16 value the best row rounds down to
    best = (lo + 2.0 ** -8 - 2.0 ** -11) * (1.0 - 2.0 ** -18)
    s_best = q @ best
    rounded = lo if bf16 else lo + 2.0 ** -8 - 2.0 ** -10                # the operand the tensor cores see
    gap = s_best - q @ rounded
    decoys = np.empty((n_decoys, dims))
    for i, t in enumerate(np.linspace(0.9, 0.15, n_decoys)):
        row = lo.copy()
        for c in rng.permutation(dims):                                 # exact 2^-7 steps up to the target score
            if q @ row >= s_best - t * gap:
                break
            row[c] += 2.0 ** -7
        assert s_best - t * gap <= q @ row < s_best
        decoys[i] = row
    corpus = unit_rows(rng, n, dims)
    corpus[0] = best
    corpus[1:1 + n_decoys] = decoys
    corpus[:1 + n_decoys] *= np.float32(2.0 ** scale_log2)
    return q.astype(np.float32)[None, :], corpus
