"""NumPy HIPPO penalty (trieste acquisition/function/multi_objective.py:664-758), its partials in the candidate's member
means, and the penalised EHVI value and gradient built on tests/ehvi_oracle.py.  Test infrastructure only."""
import numpy as np

from tests import ehvi_oracle as eo


def _factors(mean, pmean, pvar):
    """w_p = (2/pi) atan(d_p) [M, P], w'_p [M, P], and dd_p/dmean [M, P, L] (0 at d_p = 0)"""
    mean, pmean, pvar = (np.asarray(a, dtype=np.float64) for a in (mean, pmean, pvar))
    diff = mean[:, None, :] - pmean[None]
    z = diff / np.sqrt(pvar)[None]
    d = np.sqrt(np.sum(z * z, axis=-1))
    w = (2.0 / np.pi) * np.arctan(d)
    dw = (2.0 / np.pi) / (1.0 + d * d)
    with np.errstate(divide="ignore", invalid="ignore"):
        dd = np.where(d[..., None] > 0.0, diff / (pvar[None] * d[..., None]), 0.0)
    return w, dw, dd


def penalty(mean, pmean, pvar):
    """mean [M, L]; pending means and variances [P, L] -> prod_p (2/pi) atan(d_p) [M]"""
    return np.prod(_factors(mean, pmean, pvar)[0], axis=-1)


def penalty_partials(mean, pmean, pvar):
    """d pen / d mean [M, L]: sum_p (prod_{q != p} w_q) w'_p dd_p/dmean, with no division by a factor"""
    w, dw, dd = _factors(mean, pmean, pvar)
    P = w.shape[1]
    others = np.stack([np.prod(np.delete(w, p, axis=1), axis=1) for p in range(P)], axis=1)  # [M, P]
    return np.sum((others * dw)[..., None] * dd, axis=1)


def value(mean, var, lower, upper, pmean, pvar):
    """EHVI x penalty [M]"""
    return eo.ehvi(mean, var, lower, upper) * penalty(mean, pmean, pvar)


def partials(mean, var, lower, upper, pmean, pvar):
    """d value / d mean and d value / d var [M, L]"""
    e = eo.ehvi(mean, var, lower, upper)
    de_mu, de_var = eo.ehvi_partials(mean, var, lower, upper)
    pen = penalty(mean, pmean, pvar)
    return pen[:, None] * de_mu + e[:, None] * penalty_partials(mean, pmean, pvar), pen[:, None] * de_var


def gradient(models, Xq, lower, upper, pmean, pvar, predict, posterior_gradients):
    """d value / d x [M, D] of oracle models (one per objective): pen grad EHVI + EHVI sum_l dpen/dmean_l grad mean_l"""
    means, vars_ = zip(*(predict(m, Xq) for m in models))
    mean, var = np.concatenate(means, axis=1), np.concatenate(vars_, axis=1)
    pen = penalty(mean, pmean, pvar)
    dpen = penalty_partials(mean, pmean, pvar)
    grad = pen[:, None] * eo.ehvi_gradient(models, Xq, lower, upper, predict, posterior_gradients)
    e = eo.ehvi(mean, var, lower, upper)
    for l, m in enumerate(models):
        grad += (e * dpen[:, l])[:, None] * posterior_gradients(m, Xq)[0]
    return grad
