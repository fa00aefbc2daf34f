"""NumPy restatement of the trajectories' values and input gradients that continuous Thompson sampling
(trieste acquisition/function/continuous_thompson_sampling.py) differentiates through (models/gpflow/sampler.py:858-953,
809-855), for the tests.  Written from the formulas on top of the GP oracle (``oracle/gp_oracle.py``); the device code
never imports it.

  f_b(x) = s sum_f theta_bf cos(a_f) + m + sum_j v_bj k(x, x_j),   a_f = w_f . (x / l) + c_f,   s = sqrt(2 sigma^2 / F)
  grad f_b(x) = -s sum_f theta_bf sin(a_f) w_f / l + sum_j v_bj 2 k'(r2_j) (x - x_j) / l^2
"""
from __future__ import annotations

import math

import numpy as np

from oracle import gp_oracle as o


def _paired(Xq: np.ndarray, W, b, theta, variance, lengthscales, mean_const, canonical=None):
    """Xq [M, B, D], theta [B, F]; canonical = (kind, X [N, D], v [B, N]) or None -> (values [M, B], grads [M, B, D])."""
    M, B, D = Xq.shape
    F = W.shape[0]
    ls = np.broadcast_to(np.asarray(lengthscales, dtype=np.float64), (D,))
    s = math.sqrt(2.0 * variance / F)
    vals = np.empty((M, B))
    grads = np.empty((M, B, D))
    for bb in range(B):
        x = Xq[:, bb, :] / ls  # [M, D]
        a = x @ W.T + b  # [M, F]
        vals[:, bb] = s * (np.cos(a) @ theta[bb]) + mean_const
        grads[:, bb] = -s * ((np.sin(a) * theta[bb]) @ W) / ls
        if canonical is not None:
            kind, X, v = canonical
            xs = X / ls
            diff = x[:, None, :] - xs[None, :, :]  # [M, N, D]
            r2 = np.sum(diff * diff, axis=-1)
            vals[:, bb] += o.kernel_from_r2(kind, r2, variance) @ v[bb]
            w = 2.0 * o._kernel_dr2(kind, r2, variance) * v[bb][None, :]  # [M, N]
            grads[:, bb] += np.einsum("mn,mnd->md", w, diff) / ls
    return vals, grads


def rff_value_and_gradient(Xq, W, b, theta, variance, lengthscales, mean_const):
    """The RFF trajectory of ``oracle.rff_trajectory`` and its input gradient: Xq [M, B, D] -> ([M, B], [M, B, D])."""
    return _paired(Xq, W, b, theta, variance, lengthscales, mean_const)


def decoupled_value_and_gradient(m: o.GPRModel, Xq, W, b, prior_w, v):
    """The decoupled trajectory of ``oracle.decoupled_trajectory`` and its input gradient."""
    return _paired(Xq, W, b, prior_w, m.variance, m.lengthscales, m.mean_const, canonical=(m.kind, m.X, v))
