"""NumPy restatement of the reducers over single-query acquisitions (trieste/acquisition/combination.py: Sum, Product;
function/function.py:1914-1990: MakePositive) and their gradients.  Each term is a fused kind on an oracle model; its
value and d/d(mean, var) come from oracle/gp_oracle.py and tests/al_oracle.py, d/dvar zero where the posterior variance
is clipped.  Terms combine in term order; the product's coefficients are prefix x suffix products of the other values,
the softplus's is sigmoid(v)."""
from __future__ import annotations

import math

import numpy as np

from oracle import gp_oracle as o
from tests import al_oracle as al


def _pdf(z):
    return np.exp(-0.5 * z * z) / math.sqrt(2.0 * math.pi)


def kind_value_partials(kind, mean, var, param=0.0, alpha=None, noise=None, samples=None):
    """(value, d/dmean, d/dvar) of one kind at (mean, var) [M, 1], variance already clipped"""
    s = np.sqrt(var)
    if kind == "ei":
        z = (param - mean) / s
        return o.expected_improvement(mean, var, param), -o.ndtr(z), _pdf(z) / (2 * s)
    if kind == "log_ei":
        z = (param - mean) / s
        v = o.log_expected_improvement(mean, var, param)
        import scipy.special as ssp

        log_h = v - np.log(s)
        return v, -np.exp(ssp.log_ndtr(z) - log_h) / s, np.exp(-0.5 * z * z - 0.5 * math.log(2 * math.pi) - log_h) / (2 * var)
    if kind == "pbt":
        z = (param - mean) / s
        return o.ndtr(z), -_pdf(z) / s, -_pdf(z) * z / (2 * var)
    if kind == "lcb":
        return mean - param * s, np.ones_like(mean), -param / (2 * s)
    if kind == "neg_lcb":
        return -(mean - param * s), -np.ones_like(mean), param / (2 * s)
    if kind == "aei":
        z = (param - mean) / s
        ei = o.expected_improvement(mean, var, param)
        tv = noise + var
        aug = 1.0 - math.sqrt(noise) / np.sqrt(tv)
        return (o.augmented_expected_improvement(mean, var, param, noise), -o.ndtr(z) * aug,
                _pdf(z) / (2 * s) * aug + ei * 0.5 * math.sqrt(noise) / (tv * np.sqrt(tv)))
    if kind == "mes":
        from scipy.special import log_ndtr

        sd = np.maximum(s, o.MES_CLAMP_LB)
        gamma = (np.asarray(samples).reshape(1, -1) - mean) / sd
        r = np.exp(-0.5 * gamma * gamma - 0.5 * math.log(2 * math.pi) - log_ndtr(-gamma))
        dg = 0.5 * r - 0.5 * gamma * r * (r - gamma)
        return (o.min_value_entropy_search(mean, var, samples), -dg.mean(axis=1, keepdims=True) / sd,
                -(dg * gamma).mean(axis=1, keepdims=True) / (2 * var))
    if kind in ("bichon", "ranjan"):
        delta = 1 if kind == "bichon" else 2
        dm, dv = al.feasibility_partials(mean, var, param, alpha, delta)
        return al.feasibility(mean, var, param, alpha, delta), dm, dv
    if kind == "bald":
        dm, dv = al.bald_partials(mean, var, param)
        return al.bald(mean, var, param), dm, dv
    if kind == "pv":
        dm, dv = al.predictive_variance_single_partials(mean, var, param)
        return al.predictive_variance_single(mean, var, param), dm, dv
    raise ValueError(kind)


def combine(op, values):
    """the reduced value and the coefficient of each term's partials"""
    T = len(values)
    if op == "softplus":
        assert T == 1
        v = values[0]
        with np.errstate(over="ignore"):
            return np.log(1 + np.exp(v)), [1.0 / (1.0 + np.exp(-v))]
    if op == "sum":
        out = values[0]
        for v in values[1:]:
            out = out + v
        return out, [np.ones_like(values[0])] * T
    out = values[0]
    for v in values[1:]:
        out = out * v
    pre, acc = [], np.ones_like(values[0])
    for v in values:
        pre.append(acc)
        acc = acc * v
    coef, acc = [None] * T, np.ones_like(values[0])
    for k in range(T - 1, -1, -1):
        coef[k] = pre[k] * acc
        acc = acc * values[k]
    return out, coef


def term_moments(om, X):
    """posterior mean and clipped variance [M, 1], and where the variance was clipped"""
    mean, var = o.predict(om, X)
    clipped = o.predict_f(om, X)[1] < o.VAR_CLIP
    return mean, var, clipped


def reduction(op, terms, X):
    """terms: (kind, oracle model, kwargs of kind_value_partials without noise).  Returns (value [M, 1], d value / d x
    [M, D], {id(model): |d value / d var_model| [M, 1]})."""
    vals, parts = [], []
    for kind, om, kw in terms:
        mean, var, clipped = term_moments(om, X)
        v, dm, dv = kind_value_partials(kind, mean, var, noise=om.noise, **kw)
        vals.append(v)
        parts.append((om, dm, np.where(clipped, 0.0, dv)))
    value, coef = combine(op, vals)
    grad = np.zeros_like(X, dtype=np.float64)
    dvar = {}
    for c, (om, dm, dv) in zip(coef, parts):
        gm, gv = o.posterior_gradients(om, X)
        grad = grad + c * dm * gm + c * dv * gv
        dvar[id(om)] = dvar.get(id(om), 0.0) + c * dv
    return value, grad, {k: np.abs(v) for k, v in dvar.items()}
