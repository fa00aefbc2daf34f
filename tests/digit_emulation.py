"""CPU emulation of the int8 digit engine (trieste_b200/csrc/ozaki5.cuh, ozaki.cuh, int8_engines.cu) — TEST INFRASTRUCTURE.

The int8 tensor-core engine evaluates the fp64 product ``A = Linv · K*`` as exact integer digit GEMMs.  Everything it does is
integer arithmetic on balanced base-256 digits plus a handful of fp64 operations in the epilogue, so NumPy can replay it
exactly on the CPU (digit products of K <= 16384 terms stay below 2^31, far inside fp64's 2^53 exact-integer range):

  * ``tight_row_scales``      ozaki.cuh ``rowstats_kernel`` (tight split): rowscale[n] = max_k |Linv[n,k]| / FILL, rowsum[n]
  * ``balanced_digits``       ozaki.cuh ``digit_bytes`` / ``digits_kernel``: v = rint(x / scale · 2^(8S)) = Σ_p d_p 256^(S-p)
  * ``digit_bytes``           the carry-free byte trick ``(v + 0x80..80) ^ 0x80..80`` the kernels use to cut the digits
  * ``centred_kstar_digits``  ozaki5.cuh ``kstar_digits_kernel`` + int8_engines.cu ``centre_int / h_eff``: integer centre
  * ``digit_gemm``            digit_gemm.cuh ``digit_gemm_kernel`` (pairs p + q <= R share the level accumulator T_{p+q}) and
                              its epilogue (Horner over the levels, row scale, row-sum term)
  * ``apriori_estimate``      int8_engines.cu ``single_pass_estimate``: the admission test of the 15-product mode

It is how the error budget of DESIGN.md §4c was established (tools/digit_error_study.py regenerates that table) and it lets the
CPU suite pin the budget without a GPU (tests/test_digit_emulation.py).  Nothing in the product imports this module."""
from __future__ import annotations

import math

import numpy as np

FILL = 0.4975  # ozaki.cuh: |x̂| bound (the largest 5-digit balanced value is 0.49804)


def tight_row_scales(Linv: np.ndarray):
    mx = np.abs(Linv).max(axis=1)
    return np.where(mx > 0, mx / FILL, 1.0), Linv.sum(axis=1)


def balanced_digits(v: np.ndarray, S: int):
    """int64 v -> S balanced base-256 digits, most significant first, each in [-128, 127]; raises if v needs more digits."""
    v = v.astype(np.int64).copy()
    out = []
    for _ in range(S):
        lo = ((v + 128) & 255) - 128
        out.append(lo.astype(np.float64))
        v = (v - lo) >> 8
    if np.any(v != 0):
        raise OverflowError("value does not fit the requested number of balanced digits")
    return out[::-1]


def digit_bytes(v: np.ndarray, S: int) -> np.ndarray:
    """The kernels' carry-free cut: the int8 digits are the low S bytes of (v + 0x80..80) ^ 0x80..80; returns [S, ...] int8,
    least significant digit first (byte 0)."""
    K = np.uint64(int("80" * S, 16))
    w = (v.astype(np.int64).view(np.uint64) + K) ^ K
    return np.stack([((w >> np.uint64(8 * b)) & np.uint64(0xFF)).astype(np.uint8).view(np.int8) for b in range(S)])


def centred_kstar_digits(Ks: np.ndarray, variance: float, S: int):
    """K* = h_eff + K̃ with the INTEGER centre c = rint(FILL 2^(8S)) in digit units (no rounding bias): returns
    (digits of K̃ / sB, sB, h_eff), sB = (variance / 2) / FILL."""
    h = 0.5 * variance
    sB = h / FILL
    inv = 2.0 ** (8 * S) / sB
    centre = np.rint(FILL * 2.0 ** (8 * S))
    v = np.rint(Ks * inv).astype(np.int64) - np.int64(centre)
    return balanced_digits(v, S), sB, h * centre / (FILL * 2.0 ** (8 * S))


def digit_gemm(Linv: np.ndarray, Ks: np.ndarray, variance: float, SA: int = 5, SB: int = 5, R: int = 6,
               tight: bool = True, centre: bool = True):
    """Emulated A = Linv K* with SA digits of Linv, SB digits of K* and the digit pairs p + q <= R.
    Returns (A, number of digit products).  ``tight=False`` / ``centre=False`` reproduce round 1's power-of-two scales with two
    spare bits and the uncentred K* (for the error-budget table)."""
    N = Linv.shape[0]
    if tight:
        sA, rowsum = tight_row_scales(Linv)
    else:
        mx = np.abs(Linv).max(axis=1)
        mx[mx == 0] = 1.0
        sA, rowsum = 2.0 ** (np.ceil(np.log2(mx)) + 2), Linv.sum(axis=1)
    dA = balanced_digits(np.rint(Linv / sA[:, None] * 2.0 ** (8 * SA)), SA)
    if centre:
        dB, sB, h_eff = centred_kstar_digits(Ks, variance, SB)
    else:
        sB, h_eff = (variance / FILL if tight else 2.0 ** (math.ceil(math.log2(variance)) + 2)), 0.0
        dB = balanced_digits(np.rint(Ks / sB * 2.0 ** (8 * SB)), SB)
    levels = {}
    nprod = 0
    for p in range(1, SA + 1):
        for q in range(1, SB + 1):
            if p + q <= R:
                t = dA[p - 1] @ dB[q - 1]  # exact: |t| <= N 2^14 < 2^53
                levels[p + q] = levels.get(p + q, 0.0) + t
                nprod += 1
    assert max(np.abs(t).max() for t in levels.values()) < 2.0 ** 31, "int32 accumulator headroom"
    rs = sorted(levels)
    v = levels[rs[-1]]
    for r in rs[-2::-1]:  # Horner, least significant level first, exactly as the epilogue: v = v 2^-8 + T_r
        gap = rs[rs.index(r) + 1] - r
        v = v * 2.0 ** (-8 * gap) + levels[r]
    A = v * (sA[:, None] * sB * 2.0 ** (-8 * rs[0])) + (h_eff * rowsum)[:, None]
    return A, nprod


def apriori_estimate(variance: float, max_rowscale: float, N: int, S: int) -> float:
    """int8_engines.cu ``single_pass_estimate``: max |Δvar| / σ_f² when the levels r > S + 1 are dropped."""
    sB = 0.5 * variance / FILL
    return 1.6 * math.sqrt(variance) * max_rowscale * sB * math.sqrt(6.0 * N) * (65536.0 / 12.0) * 2.0 ** (-8 * (S + 2)) / variance


def variance_error(Linv: np.ndarray, Ks: np.ndarray, variance: float, **kw):
    """max and rms of |Σ_n A_emulated² − Σ_n A_exact²| / σ_f² over the candidate columns, and the product count."""
    A, nprod = digit_gemm(Linv, Ks, variance, **kw)
    At = Linv @ Ks
    d = (A * A).sum(axis=0) - (At * At).sum(axis=0)
    return float(np.abs(d).max() / variance), float(np.sqrt((d * d).mean()) / variance), nprod
