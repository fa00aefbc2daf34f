"""Shared test helpers: build matching (oracle model, native model) pairs."""
from __future__ import annotations

import dataclasses

import numpy as np

from oracle import gp_oracle as o

KERNEL_CLASSES = {"rbf": "SquaredExponential", "matern12": "Matern12", "matern32": "Matern32", "matern52": "Matern52"}


def native_from_oracle(om, **kw):
    import trieste_b200 as tb

    kcls = getattr(tb, KERNEL_CLASSES[om.kind])
    spec = tb.GPRSpec((om.X, om.y), kcls(om.variance, om.lengthscales), tb.Constant(om.mean_const), om.noise)
    return tb.GaussianProcessRegression(spec, **kw)


def model_pair(objective, N, D, kind="matern52", seed=0, noise=None, engine=None):
    om = o.synthetic_model(objective, N, D, kind=kind, seed=seed, noise=noise)
    nm = native_from_oracle(om)
    if engine is not None:
        nm.set_engine(engine)
    return om, nm


def candidates(M, D, seed=1):
    return np.random.default_rng(seed).uniform(size=(M, D))


def exact_square_dist(X1, X2, lengthscales):
    """r^2 from explicit differences, a drop-in for ``o.scaled_square_dist``: exactly 0 where two points coincide.  The
    oracle's expansion form leaves O(1e-16) there, which Matern-12's sqrt turns into an O(1e-8) error of k(x, x)."""
    d = (X1[:, None, :] - X2[None, :, :]) / lengthscales
    return np.einsum("mnd,mnd->mn", d, d)


def with_exact_cholesky(om):
    """The oracle model with L = chol(K + noise I) of the difference-form Gram (the library's), everything else unchanged.
    For the smooth kernels this changes L at the 1e-16 level; for Matern-12 it removes the oracle's own 1e-8 error."""
    K = o.kernel_from_r2(om.kind, exact_square_dist(om.X, om.X, om.lengthscales), om.variance)
    K[np.diag_indices_from(K)] += om.noise
    return dataclasses.replace(om, L=np.linalg.cholesky(K))
