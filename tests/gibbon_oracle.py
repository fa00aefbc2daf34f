"""NumPy restatement of GIBBON (trieste 4.2.1 acquisition/function/entropy.py:236-618) for the tests.

Written from the published method (Moss et al. 2021, modified for minimisation) at the reference's call sites, on top of
the GP oracle (``oracle/gp_oracle.py``); the device code never imports it.  Citations are to entropy.py.
"""
from __future__ import annotations

import math

import numpy as np
from scipy import linalg as sla
from scipy.special import log_ndtr

from oracle import gp_oracle as o

CLAMP_LB = 1e-8  # entropy.py:47


def quality_term(mean, var, samples, noise):
    """:479-500.  mean, var [M,1] (var clipped by predict); samples [S,1] -> [M,1]:
    -1/2 mean_s log(1 + rho^2 r_s (gamma_s - r_s)), rho^2 = var / (var + noise), r = exp(log_prob(gamma) - log_cdf(-gamma))."""
    yvar = var + noise
    rho2 = var / yvar
    fsd = np.maximum(np.sqrt(var), CLAMP_LB)
    gamma = (np.asarray(samples, dtype=np.float64).reshape(1, -1) - mean) / fsd  # [M, S]
    log_minus_cdf = log_ndtr(-gamma)
    ratio = np.exp(-0.5 * gamma * gamma - 0.5 * math.log(2.0 * math.pi) - log_minus_cdf)
    inner = 1 + rho2 * ratio * (gamma - ratio)
    return -0.5 * np.mean(np.log(inner), axis=1, keepdims=True)


def repulsion_weight(m_pending: int, rescaled: bool) -> float:
    """:611-616: (1 / m)^2 with rescaled_repulsion, m the current number of pending points."""
    return (1.0 / m_pending) ** 2 if rescaled else 1.0


def repulsion_term(m: o.GPRModel, x: np.ndarray, pending: np.ndarray, rescaled: bool = True):
    """:586-618 line by line.  x [M, D], pending [m, D] -> [M, 1]."""
    _, fvar = o.predict(m, x)
    yvar = fvar + m.noise
    _, B = o.predict_joint(m, pending)  # [1, m, m]
    L = np.linalg.cholesky(B[0] + m.noise * np.eye(pending.shape[0]))
    A = o.covariance_between_points(m, x, pending)[0]  # [M, m]
    L_inv_A = sla.solve_triangular(L, A.T, lower=True)  # [m, M]
    V_det = yvar - np.sum(L_inv_A * L_inv_A, axis=0)[:, None]
    repulsion = 0.5 * (np.log(V_det) - np.log(yvar))
    return repulsion_weight(pending.shape[0], rescaled) * repulsion


def gibbon(m: o.GPRModel, x, samples, pending, rescaled: bool = True):
    """GibbonAcquisition.__call__ (:435-436): diversity + quality."""
    mean, var = o.predict(m, x)
    return repulsion_term(m, x, pending, rescaled) + quality_term(mean, var, samples, m.noise)


# ---- gradients (what tfp.math.value_and_gradient takes of the above) ----
def _dk(m: o.GPRModel, x: np.ndarray, z: np.ndarray):
    """d k(x_i, z_j) / d x_i: [M, n, D]."""
    diff = (x[:, None, :] - z[None, :, :]) / m.lengthscales
    r2 = np.sum(diff * diff, axis=-1)
    return o._kernel_dr2(m.kind, r2, m.variance)[:, :, None] * 2.0 * diff / m.lengthscales


def quality_value_and_gradient(m: o.GPRModel, x: np.ndarray, samples):
    """Analytic: with h = r (gamma - r), r' = r (r - gamma), I = 1 + rho^2 h the per-sample term is -log(I)/2, so
    dq = -(rho^2 h' dgamma + h drho^2) / (2 I); the variance path is cut where predict clips it."""
    mean, var = o.predict(m, x)
    dmean, dvar = o.posterior_gradients(m, x)
    dvar = np.where(var <= o.VAR_CLIP, 0.0, dvar)
    noise = m.noise
    yvar = var + noise
    rho2 = var / yvar
    sd = np.sqrt(var)
    gamma = (np.asarray(samples, dtype=np.float64).reshape(1, -1) - mean) / sd
    r = np.exp(-0.5 * gamma * gamma - 0.5 * math.log(2.0 * math.pi) - log_ndtr(-gamma))
    h = r * (gamma - r)
    dr = r * (r - gamma)
    dh = dr * (gamma - r) + r * (1.0 - dr)
    inner = 1.0 + rho2 * h
    dq_dgamma = -0.5 * rho2 * dh / inner  # [M, S]
    dq_drho2 = -0.5 * h / inner
    # dgamma/dx = -dmean/sd - gamma dvar / (2 var); drho2/dx = noise / yvar^2 dvar
    dgamma_dm = -1.0 / sd
    g = (np.mean(dq_dgamma * dgamma_dm, axis=1, keepdims=True) * dmean
         + np.mean(-dq_dgamma * gamma / (2.0 * var) + dq_drho2 * noise / (yvar * yvar), axis=1, keepdims=True) * dvar)
    return quality_term(mean, var, samples, noise), g


def repulsion_value_and_gradient(m: o.GPRModel, x: np.ndarray, pending: np.ndarray, rescaled: bool = True):
    """R = w/2 (log V_det - log yvar), V_det = yvar - |u|^2, u = L_B^-1 c(x):
    dR = w/2 ((dvar - d|u|^2) / V_det - dvar / yvar), d|u|^2 = 2 s^T dc, s = L_B^-T u,
    dc_j = dk(x, p_j) - dk(x, X) K^-1 k(X, p_j)."""
    _, var = o.predict(m, x)
    _, dvar = o.posterior_gradients(m, x)
    dvar = np.where(var <= o.VAR_CLIP, 0.0, dvar)
    yvar = var + m.noise
    _, B = o.predict_joint(m, pending)
    LB = np.linalg.cholesky(B[0] + m.noise * np.eye(pending.shape[0]))
    c = o.covariance_between_points(m, x, pending)[0]  # [M, m]
    u = sla.solve_triangular(LB, c.T, lower=True)  # [m, M]
    s = sla.solve_triangular(LB.T, u, lower=False)  # [m, M]
    W = sla.cho_solve((m.L, True), o.kernel_matrix(m.kind, m.X, pending, m.variance, m.lengthscales))  # [N, m]
    dc = _dk(m, x, pending) - np.einsum("mnd,nj->mjd", _dk(m, x, m.X), W)  # [M, m, D]
    duu = 2.0 * np.einsum("jm,mjd->md", s, dc)
    V_det = yvar - np.sum(u * u, axis=0)[:, None]
    w = repulsion_weight(pending.shape[0], rescaled)
    val = w * 0.5 * (np.log(V_det) - np.log(yvar))
    grad = w * 0.5 * ((dvar - duu) / V_det - dvar / yvar)
    return val, grad


def gibbon_value_and_gradient(m: o.GPRModel, x, samples, pending, rescaled: bool = True):
    qv, qg = quality_value_and_gradient(m, x, samples)
    rv, rg = repulsion_value_and_gradient(m, x, pending, rescaled)
    return rv + qv, rg + qg


def augmented_repulsion(m: o.GPRModel, x: np.ndarray, pending: np.ndarray, rescaled: bool = True):
    """The same term written through the model conditioned on (noisy) observations at the pending points:
    V_det = noise + var_aug(x), so R = w/2 log((noise + var_aug) / (noise + var)); the observed values do not matter."""
    _, var = o.predict(m, x)
    _, var_aug = o.conditional_predict_f(m, x, pending, np.zeros((pending.shape[0], 1)))
    return repulsion_weight(pending.shape[0], rescaled) * 0.5 * np.log((m.noise + var_aug) / (m.noise + var))
