"""NumPy restatement of the active-learning acquisitions of trieste/acquisition/function/active_learning.py and of their
gradients: the feasibility criteria (:220-245), BALD (:504-513) and the predictive variance (:98-108), single queries and
q-batches.  Values follow the reference's operation order (tfp's ``ndtr`` for Phi, ``exp(log_prob)`` for phi).  Gradients
are analytic: d/dmean and d/dvar of each tail, mapped to d/dx through the posterior gradients; for the q-batch predictive
variance, Sigma_bar = det(M) M^-1 (M = cov + jitter 1 1^T) through the Jacobians of the joint mean and covariance."""
from __future__ import annotations

import math

import numpy as np
import scipy.linalg as sla

from oracle import gp_oracle as o

BALD_C2 = (math.pi * math.log(2.0)) / 2


def _prob(t):
    """tfp Normal(0, 1).prob: exp(log_prob)"""
    return np.exp(-0.5 * t * t - 0.5 * math.log(2.0 * math.pi))


def feasibility(mean, var, threshold, alpha, delta):
    """bichon_ranjan_criterion (:220-245)"""
    stdev = np.sqrt(var)
    t = (threshold - mean) / stdev
    t_plus, t_minus = t + alpha, t - alpha
    if delta == 1:
        G = (alpha * (o.ndtr(t_plus) - o.ndtr(t_minus)) - t * (2 * o.ndtr(t) - o.ndtr(t_plus) - o.ndtr(t_minus))
             - (2 * _prob(t) - _prob(t_plus) - _prob(t_minus)))
        return G * stdev
    G = ((alpha**2 - 1 - t**2) * (o.ndtr(t_plus) - o.ndtr(t_minus)) - 2 * t * (_prob(t_plus) - _prob(t_minus))
         + t_plus * _prob(t_plus) - t_minus * _prob(t_minus))
    return G * var


def feasibility_partials(mean, var, threshold, alpha, delta, clipped=None):
    """d/dmean, d/dvar of :func:`feasibility`; d/dvar = 0 where ``clipped``"""
    s = np.sqrt(var)
    t = (threshold - mean) / s
    tp, tm = t + alpha, t - alpha
    A = o.ndtr(tp) - o.ndtr(tm)
    B = _prob(tp) - _prob(tm)
    if delta == 1:
        dm = 2 * o.ndtr(t) - o.ndtr(tp) - o.ndtr(tm)
        dv = (alpha * A - (2 * _prob(t) - _prob(tp) - _prob(tm))) / (2 * s)
    else:
        dm = 2 * s * (t * A + B)
        dv = feasibility(mean, var, threshold, alpha, 2) / var + t * (t * A + B)
    return dm, _zero_where(dv, clipped)


def bald(mean, var, jitter):
    """bayesian_active_learning_by_disagreement.__call__ (:504-513)"""
    variance = np.maximum(var, jitter)
    p = o.ndtr(mean / np.sqrt(variance + 1))
    Ef = (np.sqrt(BALD_C2) / np.sqrt(variance + BALD_C2)) * np.exp(-(mean**2) / (2 * (variance + BALD_C2)))
    return -p * np.log(p + jitter) - (1 - p) * np.log(1 - p + jitter) - Ef


def bald_partials(mean, var, jitter, clipped=None):
    """d/dmean, d/dvar of :func:`bald`; d/dvar = 0 where var < jitter (tf.maximum) or ``clipped``"""
    v = np.maximum(var, jitter)
    sv = np.sqrt(v + 1)
    u = mean / sv
    p, fu = o.ndtr(u), _prob(u)
    vc = v + BALD_C2
    E = np.sqrt(BALD_C2) / np.sqrt(vc) * np.exp(-mean * mean / (2 * vc))
    dh = -np.log(p + jitter) - p / (p + jitter) + np.log(1 - p + jitter) + (1 - p) / (1 - p + jitter)
    dm = dh * fu / sv + E * mean / vc
    dv = -dh * fu * u / (2 * (v + 1)) - E * (mean * mean / (2 * vc * vc) - 1 / (2 * vc))
    return dm, _zero_where(np.where(var < jitter, 0.0, dv), clipped)


def predictive_variance_single(mean, var, jitter):
    """predictive_variance at q = 1: exp(logdet([[var + jitter]])) = var + jitter"""
    return var + jitter


def predictive_variance_single_partials(mean, var, jitter, clipped=None):
    return np.zeros_like(mean), _zero_where(np.ones_like(var), clipped)


def _zero_where(dv, clipped):
    return dv if clipped is None else np.where(clipped, 0.0, dv)


def single_query(om, Xq, value, partials, *args):
    """value [M, 1] and d value / d x [M, D] of a single-query tail ``value(mean, var, *args)`` at Xq [M, D], its variance
    partial zeroed where the posterior variance is clipped at 1e-12"""
    mean, var = o.predict(om, Xq)
    clipped = o.predict_f(om, Xq)[1] < o.VAR_CLIP
    dm, dv = partials(mean, var, *args, clipped=clipped)
    gm, gv = o.posterior_gradients(om, Xq)
    return value(mean, var, *args), dm * gm + dv * gv


def pv_matrix(cov, jitter):
    """the reference's cov + jitter: the scalar is broadcast to every entry"""
    return cov + jitter


def predictive_variance(om, Xb, jitter):
    """predictive_variance (:98-108) of query batches Xb [B, q, D] -> [B, 1]: exp(2 sum log diag chol(cov + jitter))"""
    _, cov = o.predict_joint(om, Xb)  # [B, 1, q, q]
    L = np.linalg.cholesky(pv_matrix(cov[:, 0], jitter))
    return np.exp(2.0 * np.log(np.diagonal(L, axis1=-2, axis2=-1)).sum(-1))[:, None]


def joint_reverse(om, Xb, g_mean, s_bar):
    """d/dx of a function of the joint posterior (mean [q], cov [q, q]) of one batch Xb [q, D], given its adjoints g_mean [q]
    and s_bar [q, q] (d f / d cov_jk, entries taken as independent):
      d/dx_j = g_mean_j dmean_j/dx_j + sum_k (s_bar_jk + s_bar_kj) J_jk,
      J_jk = d cov_jk / d x_j through the first argument = dk(x_j, x_k)/dx_j - (dk(x_j, X)/dx_j)^T K^-1 k(X, x_k)
    (k(x, x) is constant, so J_jj is the posterior part only, and d cov_jj / dx_j = 2 J_jj)."""
    ls = om.lengthscales
    q = Xb.shape[0]
    diff_n = (Xb[:, None, :] - om.X[None, :, :]) / ls  # [q, N, D]
    dk_n = o._kernel_dr2(om.kind, np.square(diff_n).sum(-1), om.variance)[:, :, None] * 2.0 * diff_n / ls
    diff_q = (Xb[:, None, :] - Xb[None, :, :]) / ls  # [q, q, D]
    dk_q = o._kernel_dr2(om.kind, np.square(diff_q).sum(-1), om.variance)[:, :, None] * 2.0 * diff_q / ls
    dk_q[np.arange(q), np.arange(q)] = 0.0
    alpha = sla.cho_solve((om.L, True), om.err, check_finite=False)[:, 0]
    V = sla.cho_solve((om.L, True), o.kernel_matrix(om.kind, om.X, Xb, om.variance, ls), check_finite=False)  # [N, q]
    dmean = np.einsum("jnd,n->jd", dk_n, alpha)
    J = dk_q - np.einsum("jnd,nk->jkd", dk_n, V)
    return g_mean[:, None] * dmean + np.einsum("jk,jkd->jd", s_bar + s_bar.T, J)


def predictive_variance_gradient(om, Xb, jitter):
    """value and d/dx [q, D] of :func:`predictive_variance` for one batch Xb [q, D]: Sigma_bar = det(M) M^-1"""
    _, cov = o.predict_joint(om, Xb[None])
    M = pv_matrix(cov[0, 0], jitter)
    L = np.linalg.cholesky(M)
    det = np.exp(2.0 * np.log(np.diag(L)).sum())
    s_bar = det * sla.cho_solve((L, True), np.eye(Xb.shape[0]))
    return det, joint_reverse(om, Xb, np.zeros(Xb.shape[0]), s_bar)
