#!/usr/bin/env python
"""CPU model (no GPU, no oracle): how often can level 1 of the batched path NOT prove a query of BASELINE configs[4]
(10 M x 768 un-normalised rows, top-100 dot; on a 132-SM H100 two query groups share the SMs, 66 row slices of
151 515 rows) as a function of the nominee heap size per
(slice, query) and of the number of nominees the finish kernel re-scores?

Scores of a unit query against uniform[-1,1]^768 rows are ~ N(0, 1/3); only the upper tail matters, so each slice's top-H
scores are drawn from the exact order statistics (cumulative exponential spacings -> uniform order statistics -> normal
quantiles).  The proof needs  s_k > max(max over slices of the slice's H-th best, the (R+1)-th nominee) + eps  with
eps = 1.03 * 2^-7 * |q| * max|v| (+ accumulation slack), |q| = 1, max|v| ~ 16.  bf16 noise on the nominee ORDER is ignored
(it adds a little), so the model is a lower bound on the failure rate.  This is the Poisson tail argument behind the
engine's heap-size cost model (pick_heap in wax_b200/csrc/waxvs_engine.cu)."""
import sys

import numpy as np
from scipy.stats import norm

S, n, k = 66, 151_515, 100
sigma = np.sqrt(1 / 3)
eps = (1.03 * 2 ** -7 * 1.01) * 1.0 * 16.0 + 768 * 2 ** -23 * 16
trials = int(sys.argv[1]) if len(sys.argv) > 1 else 20_000
rng = np.random.default_rng(0)


def trial(H, R):
    e = rng.exponential(size=(S, H)).cumsum(axis=1) / n
    z = norm.isf(e) * sigma                      # each slice's H best scores, descending
    roots = z[:, H - 1]
    allv = np.sort(z.ravel())[::-1]
    sk = allv[k - 1]
    by_root = sk > roots.max() + eps
    by_r = allv.size <= R or sk > allv[R] + eps
    return by_root and by_r, by_root, by_r


for H, R in [(16, 1024), (20, 1024), (24, 1024), (24, 512), (32, 1024), (64, 1024)]:
    r = np.array([trial(H, R) for _ in range(trials)])
    print(f"heap {H:2d} rescore {R:4d}: unproven {1 - r[:, 0].mean():.5f}  (slice-root bound {1 - r[:, 1].mean():.5f}, "
          f"(R+1)-th nominee bound {1 - r[:, 2].mean():.5f})  of {trials} trials")
