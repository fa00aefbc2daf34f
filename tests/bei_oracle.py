"""NumPy restatement of BatchExpectedImprovement (trieste 4.2.1 acquisition/function/function.py:1281-1805) and of
MultivariateNormalCDF (acquisition/function/utils.py:29-199), with a hand-written reverse pass.

The forward functions follow the reference's tensor algebra literally (the delta masks of ``_compute_Sigma``, the ragged
mask of ``_compute_c``, the blocks of ``_compute_R``); the reverse pass is written per q-batch and per CDF and is checked
against central finite differences.  Sobol points are passed in as ``w [S, >= Q-1]`` (column j serves every dimension)."""
from __future__ import annotations

import numpy as np
import scipy.linalg as sla
from scipy.special import ndtr, ndtri
from scipy.stats import norm

from oracle import gp_oracle as o

BEI_JITTER = 1e-6  # function.py:1776-1783 (hard-coded) and MultivariateNormalCDF's default jitter (utils.py:114)


# ---- MultivariateNormalCDF.__call__ (utils.py:109-199) ----
def mvn_cdf(x, mean, cov, w, jitter=BEI_JITTER):
    """x, mean [B, Q], cov [B, Q, Q], w [S, >= Q-1] -> [B]."""
    x, mean, cov = (np.asarray(a, dtype=np.float64) for a in (x, mean, cov))
    B, Q = x.shape
    C = np.linalg.cholesky(cov + jitter * np.eye(Q)[None])
    S = w.shape[0]
    b = x - mean
    e = np.zeros((B, S, Q))
    f = np.zeros((B, S, Q))
    y = np.zeros((B, S, Q))
    e[:, :, 0] = ndtr(b[:, None, 0] / (C[:, None, 0, 0] + 1e-12))
    f[:, :, 0] = e[:, :, 0]
    for i in range(1, Q):
        y[:, :, i - 1] = ndtri(1e-6 + (1 - 2e-6) * w[None, :, i - 1] * e[:, :, i - 1])
        t = np.sum(C[:, None, i, :i] * y[:, :, :i], axis=-1)
        e[:, :, i] = ndtr((b[:, None, i] - t) / (C[:, None, i, i] + 1e-12))
        f[:, :, i] = e[:, :, i] * f[:, :, i - 1]
    return f[:, :, -1].mean(-1)


# ---- batch_expected_improvement._compute_batch_expected_improvement (function.py:1651-1745) ----
def _compute_bm(mean, threshold):
    B, Q = mean.shape
    b = np.zeros((B, Q, Q)) - threshold[:, None, None] * np.eye(Q)[None]
    m = mean[:, None, :] - mean[:, :, None]
    m = m - mean[:, :, None] * np.eye(Q)[None]
    return b, m


def _delta(idx, dim):
    d = np.ones((dim, dim))
    d[idx, :] = 0.0
    return d


def _compute_Sigma(cov):
    B, Q, _ = cov.shape
    out = np.empty((B, Q, Q, Q))
    for q in range(Q):
        diq, dqj = _delta(q, Q), _delta(q, Q).T
        out[:, q] = cov * diq * dqj - cov[:, :, q:q + 1] * diq - cov[:, q:q + 1, :] * dqj + cov[:, q:q + 1, q:q + 1]
    return out


def _compute_c(diff, Sig):
    BQ, Q = diff.shape
    ratio = Sig / np.diagonal(Sig, axis1=1, axis2=2)[:, :, None]
    c = diff[:, None, :] - diff[:, :, None] * ratio
    return c[:, ~np.eye(Q, dtype=bool)].reshape(BQ, Q, Q - 1)


def _compute_R(Sig):
    BQ, Q, _ = Sig.shape
    R_whole = Sig[:, None, :, :] - Sig[:, :, :, None] * Sig[:, :, None, :] / np.diagonal(Sig, axis1=1, axis2=2)[:, :, None, None]
    R = np.empty((BQ, Q, Q - 1, Q - 1))
    for q in range(Q):
        keep = np.arange(Q) != q
        R[:, q] = R_whole[:, q][:, keep][:, :, keep]
    return R


def compute_bei(mean, cov, threshold, w):
    """mean [B, Q], cov [B, Q, Q], threshold [B] in the maximisation form -> ei [B]."""
    B, Q = mean.shape
    b, m = _compute_bm(mean, threshold)
    Sigma = _compute_Sigma(cov)
    b_r, m_r, Sig_r = b.reshape(B * Q, Q), m.reshape(B * Q, Q), Sigma.reshape(B * Q, Q, Q)
    p = mvn_cdf(b_r - m_r, np.zeros((B * Q, Q)), Sig_r, w).reshape(B, Q)
    c = _compute_c(b_r - m_r, Sig_r)
    R = _compute_R(Sig_r)
    Phi = mvn_cdf(c.reshape(B * Q * Q, Q - 1), np.zeros((B * Q * Q, Q - 1)), R.reshape(B * Q * Q, Q - 1, Q - 1), w).reshape(B, Q, Q)
    S_diag = np.diagonal(Sigma, axis1=2, axis2=3)
    pdf = norm.pdf(b, loc=m, scale=np.sqrt(S_diag))
    Sigma_diag = np.transpose(np.diagonal(np.transpose(Sigma, (0, 2, 1, 3)), axis1=2, axis2=3), (0, 2, 1))
    T = np.tile(threshold[:, None], (1, Q))
    return np.sum((mean - T) * p + np.sum(Sigma_diag * pdf * Phi, axis=2), axis=1)


def batch_expected_improvement(mean, cov, eta, w):
    """``__call__`` (function.py:1747-1805) from the joint posterior: mean [B, q], cov [B, q, q] -> [B]."""
    mean = np.asarray(mean, dtype=np.float64)
    cov = np.asarray(cov, dtype=np.float64) + BEI_JITTER * np.eye(mean.shape[1])[None]
    return compute_bei(-mean, cov, -np.full(mean.shape[0], float(eta)), w)


def batch_expected_improvement_at(m: o.GPRModel, Xq, eta, w):
    """Xq [B, q, D] -> [B] through the oracle GP's predict_joint."""
    mean, cov = o.predict_joint(m, Xq)
    return batch_expected_improvement(mean[..., 0], cov[:, 0], eta, w)


# ---- reverse pass ----
def _chol_backward(L, Lbar):
    """tf.linalg.cholesky's gradient (Murray 2016): L^-T sym(Phi(L^T Lbar)) L^-1."""
    P = np.tril(L.T @ Lbar)
    P[np.diag_indices(L.shape[0])] *= 0.5
    M = 0.5 * (P + P.T)
    return sla.solve_triangular(L.T, sla.solve_triangular(L.T, M, lower=False).T, lower=False).T


def mvn_cdf_backward(bvec, A, w, gbar):
    """One CDF P(X <= bvec), X ~ N(0, A + jitter I), and the adjoints of bvec and A for the seed gbar on its value."""
    n = len(bvec)
    L = np.linalg.cholesky(A + BEI_JITTER * np.eye(n))
    S = w.shape[0]
    lp = np.diag(L) + 1e-12
    z, e, y = np.zeros((S, n)), np.zeros((S, n)), np.zeros((S, n))
    z[:, 0] = bvec[0] / lp[0]
    e[:, 0] = ndtr(z[:, 0])
    for i in range(1, n):
        y[:, i - 1] = ndtri(1e-6 + (1 - 2e-6) * w[:, i - 1] * e[:, i - 1])
        z[:, i] = (bvec[i] - y[:, :i] @ L[i, :i]) / lp[i]
        e[:, i] = ndtr(z[:, i])
    value = np.prod(e, axis=1).mean()
    seed = gbar / S
    ybar = np.zeros((S, n))
    Lbar = np.zeros((n, n))
    bbar = np.zeros(n)
    for i in reversed(range(n)):
        ebar = seed * np.prod(np.delete(e, i, axis=1), axis=1)  # d f / d e_i without dividing by e_i
        if i < n - 1:
            ebar = ebar + ybar[:, i] * (1 - 2e-6) * w[:, i] / norm.pdf(y[:, i])
        zbar = ebar * norm.pdf(z[:, i])
        bbar[i] = zbar.sum() / lp[i]
        Lbar[i, i] = -(zbar * z[:, i]).sum() / lp[i]
        Lbar[i, :i] = -(zbar[:, None] * y[:, :i]).sum(0) / lp[i]
        ybar[:, :i] -= zbar[:, None] * L[i, :i][None, :] / lp[i]
    return value, bbar, _chol_backward(L, Lbar)


def bei_adjoints(mean, cov, eta, w):
    """One q-batch: mean [q], cov [q, q] -> (value, d value / d mean [q], sym(d value / d cov) [q, q])."""
    q = len(mean)
    mu, T = -np.asarray(mean, dtype=np.float64), -float(eta)
    C = np.asarray(cov, dtype=np.float64) + BEI_JITTER * np.eye(q)
    covbar, mubar, value = np.zeros((q, q)), np.zeros(q), 0.0
    for k in range(q):
        diq, dqj = _delta(k, q), _delta(k, q).T
        S = C * diq * dqj - C[:, k:k + 1] * diq - C[k:k + 1, :] * dqj + C[k, k]
        d = np.where(np.arange(q) == k, -T + mu[k], -(mu - mu[k]))
        Sbar, dbar = np.zeros((q, q)), np.zeros(q)
        p, bb, Ab = mvn_cdf_backward(d, S, w, mu[k] - T)
        value += (mu[k] - T) * p
        mubar[k] += p
        Sbar += Ab
        dbar += bb
        for i in range(q):
            idx = np.arange(q) != i
            sii, s = S[i, i], S[i, idx]
            c = d[idx] - d[i] * s / sii
            R = S[np.ix_(idx, idx)] - np.outer(s, s) / sii
            pdf = norm.pdf(d[i] / np.sqrt(sii)) / np.sqrt(sii)
            sik = S[i, k]
            g, cb, Rb = mvn_cdf_backward(c, R, w, sik * pdf)
            value += sik * pdf * g
            Sbar[i, k] += pdf * g
            pb = sik * g
            dbar[i] += pb * pdf * (-d[i] / sii)
            Sbar[i, i] += pb * pdf * (0.5 * d[i] ** 2 / sii ** 2 - 0.5 / sii)
            dbar[idx] += cb
            dbar[i] -= cb @ s / sii
            Sbar[i, idx] -= cb * d[i] / sii
            Sbar[i, i] += (cb @ s) * d[i] / sii ** 2
            Sbar[np.ix_(idx, idx)] += Rb
            Sbar[i, idx] -= (Rb @ s + Rb.T @ s) / sii
            Sbar[i, i] += s @ Rb @ s / sii ** 2
        covbar += Sbar * diq * dqj
        covbar[:, k] -= (Sbar * diq).sum(1)
        covbar[k, :] -= (Sbar * dqj).sum(0)
        covbar[k, k] += Sbar.sum()
        mubar[k] += dbar.sum()
        notk = np.arange(q) != k
        mubar[notk] -= dbar[notk]
    return value, -mubar, 0.5 * (covbar + covbar.T)


def bei_gradient(m: o.GPRModel, Xb, eta, w):
    """Value and d / dX of the batch EI of ONE query batch Xb [q, D] through the oracle GP (the assembly of
    gp_oracle.batch_mc_ei_gradient from the mean and covariance adjoints)."""
    Xb = np.asarray(Xb, dtype=np.float64)
    q, D = Xb.shape
    mean, cov = o.predict_joint(m, Xb[None])
    value, G_mu, Sbar = bei_adjoints(mean[0, :, 0], cov[0, 0], eta, w)
    ls = m.lengthscales
    Xt, Xq = m.X / ls, Xb / ls
    diff_n = Xq[:, None, :] - Xt[None, :, :]
    dk_n = o._kernel_dr2(m.kind, np.square(diff_n).sum(-1), m.variance)[:, :, None] * 2.0 * diff_n / ls
    alpha = sla.cho_solve((m.L, True), m.err, check_finite=False)[:, 0]
    V = sla.cho_solve((m.L, True), o.kernel_matrix(m.kind, m.X, Xb, m.variance, ls), check_finite=False)
    diff_q = Xq[:, None, :] - Xq[None, :, :]
    dk_q = o._kernel_dr2(m.kind, np.square(diff_q).sum(-1), m.variance)[:, :, None] * 2.0 * diff_q / ls
    dk_q[np.arange(q), np.arange(q)] = 0.0
    grad = np.zeros((q, D))
    for j in range(q):
        wv = G_mu[j] * alpha - 2.0 * (V @ Sbar[j])
        grad[j] = dk_n[j].T @ wv + 2.0 * (Sbar[j][:, None] * dk_q[j]).sum(0)
    return value, grad
