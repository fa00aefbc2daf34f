"""NumPy expected hypervolume improvement: the reference's literal form (acquisition/function/multi_objective.py:188-250,
the sum over all 2^L picks of (psi difference, nu) per objective), the product-of-sums form the device evaluates, the
analytic partials in (mean, var) and a Monte-Carlo hypervolume improvement.  Test infrastructure only."""
from itertools import product

import numpy as np
from scipy import special as ssp

CLIP = 1e10  # multi_objective.py:215


def _pdf(z):
    return np.exp(-0.5 * z * z) / np.sqrt(2.0 * np.pi)


def _cdf(z):
    return ssp.ndtr(z)


def _terms(mean, var, lower, upper):
    """mean, var [M, L]; lower, upper [K, L] -> a, b, m, s, broadcast to [M, K, L]"""
    m = -np.asarray(mean, dtype=np.float64)[:, None, :]
    s = np.sqrt(np.asarray(var, dtype=np.float64))[:, None, :]
    a = -np.asarray(upper, dtype=np.float64)[None]
    b = np.minimum(-np.asarray(lower, dtype=np.float64), CLIP)[None]
    return a, b, m, s


def _psi(a, c, m, s):
    z = (c - m) / s
    return s * _pdf(z) + (m - a) * (1.0 - _cdf(z))


def ehvi_literal(mean, var, lower, upper):
    """the reference's form: sum over cells and over the 2^L picks of prod_l (psi difference or nu) -> [M]"""
    a, b, m, s = _terms(mean, var, lower, upper)
    diff = np.maximum(_psi(a, a, m, s) - _psi(a, b, m, s), 0.0)
    nu = (b - a) * (1.0 - _cdf((b - m) / s))
    stacked = np.stack([diff, nu], axis=-2)  # [M, K, 2, L]
    L = diff.shape[-1]
    total = np.zeros(diff.shape[0])
    for pick in product([0, 1], repeat=L):
        f = np.ones(diff.shape[:2])
        for l, c in enumerate(pick):
            f = f * stacked[:, :, c, l]
        total = total + f.sum(axis=1)
    return total


def ehvi_factors(mean, var, lower, upper):
    """g_kl = max(psi(a, a) - psi(a, b), 0) + nu and its partials in (m, s), each [M, K, L]"""
    a, b, m, s = _terms(mean, var, lower, upper)
    za, zb = (a - m) / s, (b - m) / s
    pa, pb, qa, qb = _pdf(za), _pdf(zb), 1.0 - _cdf(za), 1.0 - _cdf(zb)
    diff = (s * pa + (m - a) * qa) - (s * pb + (m - a) * qb)
    w = b - a
    nu = w * qb
    on = diff >= 0.0  # tf.maximum passes the gradient to its first argument when x >= y
    gm = w * pb / s + np.where(on, qa - (pb * w / s + qb), 0.0)
    gs = w * pb * zb / s + np.where(on, pa - pb * (1.0 + zb * w / s), 0.0)
    return np.maximum(diff, 0.0) + nu, gm, gs, s


def _in_blocks(f, arrays, K, L):
    """f over row blocks of the [M, ...] arrays, its outputs concatenated: the [M, K, L] intermediates stay near 32 MB
    each, whatever the cell and candidate counts"""
    rows = max(1, (1 << 22) // max(1, K * L))
    M = len(arrays[0])
    if M <= rows:
        return f(*arrays)
    parts = [f(*(a[i:i + rows] for a in arrays)) for i in range(0, M, rows)]
    if isinstance(parts[0], tuple):
        return tuple(np.concatenate(p) for p in zip(*parts))
    return np.concatenate(parts)


def ehvi(mean, var, lower, upper):
    """the product-of-sums form: sum_k prod_l g_kl -> [M]"""
    def one(mean, var):
        return np.prod(ehvi_factors(mean, var, lower, upper)[0], axis=-1).sum(axis=-1)

    return _in_blocks(one, (np.asarray(mean), np.asarray(var)), *np.shape(lower))


def ehvi_partials(mean, var, lower, upper, var_clipped=None):
    """d EHVI / d mean and d EHVI / d var, each [M, L]; zero in var where the variance was clipped"""
    arrays = (np.asarray(mean), np.asarray(var))
    if var_clipped is not None:
        arrays += (np.broadcast_to(var_clipped, arrays[0].shape),)
    return _in_blocks(lambda *a: _partials(*a[:2], lower, upper, *a[2:]), arrays, *np.shape(lower))


def _partials(mean, var, lower, upper, var_clipped=None):
    g, gm, gs, s = ehvi_factors(mean, var, lower, upper)
    L = g.shape[-1]
    others = np.stack([np.prod(np.delete(g, l, axis=-1), axis=-1) for l in range(L)], axis=-1)  # [M, K, L]
    dm = (others * gm).sum(axis=1)
    ds = (others * gs).sum(axis=1)
    dvar = ds / (2.0 * s[:, 0, :])
    if var_clipped is not None:
        dvar = np.where(var_clipped, 0.0, dvar)
    return -dm, dvar


def ehvi_gradient(models, Xq, lower, upper, predict, posterior_gradients):
    """d EHVI / d x [M, D] of oracle models (one per objective) through their posterior gradients"""
    means, vars_ = zip(*(predict(m, Xq) for m in models))
    mean, var = np.concatenate(means, axis=1), np.concatenate(vars_, axis=1)
    dmu, dvar = ehvi_partials(mean, var, lower, upper)
    grad = np.zeros_like(np.asarray(Xq, dtype=np.float64))
    for l, m in enumerate(models):
        gm, gv = posterior_gradients(m, Xq)
        grad += dmu[:, l:l + 1] * gm + dvar[:, l:l + 1] * gv
    return grad


def hypervolume_improvement_mc(mean, var, lower, upper, n, seed=0):
    """Monte-Carlo EHVI of one candidate (mean, var [L]): the volume of the cells below each sampled point, averaged"""
    rng = np.random.default_rng(seed)
    y = np.asarray(mean)[None, :] + np.sqrt(np.asarray(var))[None, :] * rng.standard_normal((n, len(mean)))
    lo, up = np.asarray(lower)[None], np.asarray(upper)[None]
    ext = np.clip(up - np.maximum(lo, y[:, None, :]), 0.0, None)  # [n, K, L]
    return float(np.prod(ext, axis=-1).sum(axis=-1).mean())
