"""Regenerates the error-budget table of DESIGN.md §4c on the CPU (no GPU needed): the exact emulation of the digit engine
(tests/digit_emulation.py) on the headline model (N = 4096, D = 10, Matern52, Ackley-10 data of bench.py), 256 random candidates.

    python tools/digit_error_study.py [N]      # ~1 minute at N = 4096 on 8 cores
"""
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import scipy.linalg as sl

from oracle import gp_oracle as o  # checker side only
from tests import digit_emulation as de

N = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
D = 10
rng = np.random.default_rng(0)
X = rng.uniform(size=(N, D))
y = o.ackley(X).reshape(-1)
var = float(np.var(y))
ls = np.full(D, 0.2 * math.sqrt(D))
K = o.kernel_matrix("matern52", X, X, var, ls) + 0.01 * var * np.eye(N)
Linv = sl.solve_triangular(np.linalg.cholesky(K), np.eye(N), lower=True)
Ks = o.kernel_matrix("matern52", X, np.random.default_rng(1).uniform(size=(256, D)), var, ls)
rows = [
    ("round 1: power-of-two scales with two spare bits, 6 digits, pairs p+q <= 7", dict(SA=6, SB=6, R=7, tight=False, centre=False)),
    ("same, pairs p+q <= 6", dict(SA=6, SB=6, R=6, tight=False, centre=False)),
    ("+ tight scales", dict(SA=6, SB=6, R=6, tight=True, centre=False)),
    ("+ centred K*", dict(SA=6, SB=6, R=6, tight=True, centre=True)),
    ("5 digits, pairs p+q <= 6 (the shipped mode)", dict(SA=5, SB=5, R=6)),
    ("K* cut to 4 digits (DESIGN section 7, not taken)", dict(SA=5, SB=4, R=6)),
    ("Linv cut to 4 digits", dict(SA=4, SB=5, R=6)),
    ("fp32 handles: 3 digits, pairs p+q <= 4", dict(SA=3, SB=3, R=4)),
    ("fp32 handles: 4 digits, pairs p+q <= 5", dict(SA=4, SB=4, R=5)),
]
print(f"N = {N}, sigma_f^2 = {var:.4f}, max row scale = {de.tight_row_scales(Linv)[0].max():.3f}")
print("| variant | products | max |dvar|/sigma_f^2 | rms |")
print("|---|---|---|---|")
for name, kw in rows:
    mx, rms, n = de.variance_error(Linv, Ks, var, **kw)
    print(f"| {name} | {n} | {mx:.2e} | {rms:.2e} |")
for S in (5, 4, 3):
    print(f"a-priori estimate (single_pass_estimate) for S = {S}: {de.apriori_estimate(var, de.tight_row_scales(Linv)[0].max(), N, S):.2e}")
