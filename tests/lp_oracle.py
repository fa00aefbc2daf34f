"""NumPy restatement of local penalisation (trieste 4.2.1 acquisition/function/greedy_batch.py:54-388) for the tests.

Written from the published algorithm (Gonzalez et al. 2016, soft; Alvi et al. 2019, hard) at the reference's call sites, on
top of the GP oracle (``oracle/gp_oracle.py``); the device code never imports it.  Citations are to greedy_batch.py.
"""
from __future__ import annotations

import math

import numpy as np
from scipy import special as ssp

from oracle import gp_oracle as o

SOFT, HARD = "soft", "hard"


def lipschitz_and_eta(m: o.GPRModel, points: np.ndarray):
    """:206-230: L = max over the points of ||d mean / d x||_2 and eta = min of the mean; L < 1e-5 ('flat' model) -> 10."""
    dmean, _ = o.posterior_gradients(m, points)
    mean, _ = o.predict(m, points)
    L = float(np.max(np.sqrt(np.sum(dmean * dmean, axis=1))))
    if L < 1e-5:
        L = 10.0
    return L, float(np.min(mean))


def penalizer_state(m: o.GPRModel, pending: np.ndarray, L: float, eta: float):
    """:272-312: radius_j = (mean(x_j) - eta) / L, scale_j = sqrt(var(x_j)) / L (variance clipped at 1e-12 by predict)."""
    mean, var = o.predict(m, pending)
    return (mean[:, 0] - eta) / L, np.sqrt(var[:, 0]) / L


def _distances(x: np.ndarray, pending: np.ndarray):
    diff = x[:, None, :] - pending[None, :, :]  # [M, P, D]
    return np.sqrt(np.sum(diff * diff, axis=-1)), diff


def penalty(kind: str, x: np.ndarray, pending: np.ndarray, radius: np.ndarray, scale: np.ndarray) -> np.ndarray:
    """soft (:340-354): prod_j Phi((d_j - radius_j) / scale_j); hard (:374-388): prod_j ((d_j / (radius_j + scale_j))^-5 + 1)^-1/5.
    x [M, D] -> [M]."""
    dist, _ = _distances(x, pending)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        if kind == SOFT:
            f = o.ndtr((dist - radius[None, :]) / scale[None, :])
        else:
            f = np.power(np.power(dist / (radius + scale)[None, :], -5.0) + 1.0, -0.2)
    return np.prod(f, axis=-1)


def penalty_gradient(kind: str, x: np.ndarray, pending: np.ndarray, radius: np.ndarray, scale: np.ndarray):
    """(penalty [M], d penalty / d x [M, D]) by the product rule pen * sum_j d log f_j / d x.  d log f_j / d d_j: soft
    phi(z)/Phi(z) / scale_j (formed as exp(log phi - log Phi)); hard 1 / (d_j (1 + u_j^5)), u_j = d_j / (radius_j + scale_j).
    The gradient of d_j at d_j = 0 is taken as 0, and where the penalty is 0 so is its gradient."""
    dist, diff = _distances(x, pending)
    pen = penalty(kind, x, pending, radius, scale)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        if kind == SOFT:
            z = (dist - radius[None, :]) / scale[None, :]
            dlog = np.exp(-0.5 * z * z - 0.5 * math.log(2.0 * math.pi) - ssp.log_ndtr(z)) / scale[None, :]
        else:
            u = dist / (radius + scale)[None, :]
            dlog = 1.0 / (dist * (1.0 + u**5))
        w = np.where(dist > 0.0, dlog / dist, 0.0)  # d log f_j / d x = w (x - x_j)
    glog = np.einsum("mp,mpd->md", w, diff)
    gpen = np.where(pen[:, None] == 0.0, 0.0, pen[:, None] * glog)
    return pen, gpen


def penalized(base: np.ndarray, pen: np.ndarray) -> np.ndarray:
    """PenalizedAcquisition.__call__ (:265-269): exp(log base + log pen)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.exp(np.log(base) + np.log(pen))


def penalized_ei_value_and_gradient(m: o.GPRModel, x: np.ndarray, eta: float, kind: str, pending, radius, scale):
    """Penalised EI and its gradient pen grad(EI) + EI grad(pen) (the product rule's finite limit where the log form is
    NaN).  x [M, D] -> ([M], [M, D])."""
    ei, gei = o.ei_gradient(m, x, eta)
    pen, gpen = penalty_gradient(kind, x, pending, radius, scale)
    val = penalized(ei[:, 0], pen)
    grad = pen[:, None] * gei + np.where(gpen == 0.0, 0.0, ei * gpen)
    return val, grad


def seeded_space(lower, upper, seed: int):
    """A Box whose ``sample`` draws from seed, seed + 1, ... and records every draw, so that a test sees the same
    Lipschitz samples as the builder."""
    import trieste_b200 as tb

    class SeededBox(tb.Box):
        def __init__(self):
            super().__init__(lower, upper)
            self.drawn = []

        def sample(self, num_samples, seed_=None):
            s = tb.Box.sample(self, num_samples, seed=seed + len(self.drawn))
            self.drawn.append(s)
            return s

    return SeededBox()
