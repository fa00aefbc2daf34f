"""CPU pins of the digit engine's error budget (DESIGN.md §4c) through the exact emulation in tests/digit_emulation.py:
what the 15-product single-pass mode costs in accuracy, that the a-priori estimate which admits it covers what is measured, and
the alternatives that were examined and dropped (DESIGN.md §7)."""
import math

import numpy as np
import pytest

from oracle import gp_oracle as o
from tests import digit_emulation as de

BAR = 1e-9  # |Δvar| <= 1e-9 σ_f² (stated fp64 tolerance of the variance)


def _model(kind, N, D, noise_frac, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.uniform(size=(N, D))
    y = (o.hartmann_6(X) if D == 6 else o.ackley(X)).reshape(-1)
    var = float(np.var(y))
    ls = np.full(D, 0.2 * math.sqrt(D))
    K = o.kernel_matrix(kind, X, X, var, ls) + noise_frac * var * np.eye(N)
    L = np.linalg.cholesky(K)
    import scipy.linalg as sl

    Linv = sl.solve_triangular(L, np.eye(N), lower=True)
    Xc = np.random.default_rng(seed + 1).uniform(size=(96, D))
    return Linv, o.kernel_matrix(kind, X, Xc, var, ls), var


def test_balanced_digits_are_exact_and_match_the_byte_trick():
    rng = np.random.default_rng(0)
    for S in (3, 4, 5, 6):
        lim = int(0.498 * 2 ** (8 * S))
        v = rng.integers(-lim, lim, size=5000)
        d = de.balanced_digits(v, S)
        assert all(x.min() >= -128 and x.max() <= 127 for x in d)
        recon = sum(d[p].astype(np.int64) * 256 ** (S - 1 - p) for p in range(S))
        np.testing.assert_array_equal(recon, v)
        b = de.digit_bytes(v, S)  # least significant first
        for p in range(S):
            np.testing.assert_array_equal(b[S - 1 - p].astype(np.int64), d[p].astype(np.int64))
    with pytest.raises(OverflowError):
        de.balanced_digits(np.array([2 ** 40]), 5)  # 0.5 2^40 is the first value that needs a sixth digit


def test_all_pairs_reproduce_the_fp64_product():
    Linv, Ks, var = _model("matern52", 256, 6, 1e-2)
    A, nprod = de.digit_gemm(Linv, Ks, var, SA=6, SB=6, R=12)
    assert nprod == 36
    scale = np.abs(Linv).max(axis=1)[:, None] * var
    assert np.abs(A - Linv @ Ks).max() / scale.max() < 1e-13  # 48-bit operands: only their rounding is left


@pytest.mark.parametrize("kind", ["rbf", "matern12", "matern32", "matern52"])
def test_fifteen_products_meet_the_bar_and_the_estimate_covers_them(kind):
    N = 512
    Linv, Ks, var = _model(kind, N, 6, 1e-2)
    mx, rms, nprod = de.variance_error(Linv, Ks, var)  # 5 digits, pairs p + q <= 6
    assert nprod == 15
    est = de.apriori_estimate(var, de.tight_row_scales(Linv)[0].max(), N, 5)
    assert mx < BAR / 3, (kind, mx)
    assert est <= 3e-10, (kind, est)  # the mode is admitted for the default noise level ...
    assert mx <= 3.0 * est and est <= 100.0 * mx, (kind, mx, est)  # ... by an estimate of the right size
    # the 21 products of the six-digit mode (the same tight scales and centred K*, pairs p + q <= 7): two orders tighter
    mx21, _, n21 = de.variance_error(Linv, Ks, var, SA=6, SB=6, R=7)
    assert n21 == 21 and mx21 < mx / 100


def test_what_tight_scales_and_the_centred_kstar_buy():
    Linv, Ks, var = _model("matern52", 768, 10, 1e-2)
    loose, _, n = de.variance_error(Linv, Ks, var, SA=6, SB=6, R=6, tight=False, centre=False)
    tight, _, _ = de.variance_error(Linv, Ks, var, SA=6, SB=6, R=6, tight=True, centre=False)
    both, _, _ = de.variance_error(Linv, Ks, var, SA=6, SB=6, R=6, tight=True, centre=True)
    five, _, n5 = de.variance_error(Linv, Ks, var, SA=5, SB=5, R=6)
    assert n == 15 and n5 == 15
    # N = 4096 headline data (tools/digit_error_study.py): 1.4e-9 -> 1.4e-10 -> 1.0e-10
    assert tight < loose / 3 and both < tight and both < loose / 4
    assert five < 1.5 * both  # the sixth digit buys nothing once the pairs stop at p + q <= 6


def test_low_noise_model_is_refused_by_the_estimate():
    # an RBF model with noise σ_f²/1e5 has rows of Linv up to ~300/σ_f: the 15-product error approaches the bar and the
    # a-priori estimate (which only sees the row scales) must keep such a handle on 6 digits (21 products)
    N = 400
    Linv, Ks, var = _model("rbf", N, 6, 1e-5)
    est = de.apriori_estimate(var, de.tight_row_scales(Linv)[0].max(), N, 5)
    mx, _, _ = de.variance_error(Linv, Ks, var)
    assert est > 3e-10 and mx <= 3.0 * est


def test_fp32_handles_three_digits_meet_the_fp32_bar():
    N = 512
    Linv, Ks, var = _model("matern52", N, 6, 1e-2)
    mx, _, nprod = de.variance_error(Linv, Ks, var, SA=3, SB=3, R=4)
    assert nprod == 6 and mx < 1e-4 / 3
    assert mx <= 3.0 * de.apriori_estimate(var, de.tight_row_scales(Linv)[0].max(), N, 3)


def test_asymmetric_digit_counts_examined_in_design_section_7():
    # K* cut to 4 digits (14 products) roughly doubles the error; cutting Linv instead costs two orders of magnitude
    Linv, Ks, var = _model("matern52", 768, 10, 1e-2)
    sym, _, _ = de.variance_error(Linv, Ks, var)
    kcut, _, n14 = de.variance_error(Linv, Ks, var, SA=5, SB=4, R=6)
    lcut, _, _ = de.variance_error(Linv, Ks, var, SA=4, SB=5, R=6)
    assert n14 == 14
    assert sym < kcut < 20 * sym
    assert lcut > 20 * sym
