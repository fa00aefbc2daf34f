"""Synthetic objectives used to build the BASELINE configs — NumPy restatements of
trieste/objectives/single_objectives.py (branin :83-107, ackley_5 :433-458 generalised to d dims,
hartmann_6 :476-501).  Input generators only; not on the per-candidate path."""
from __future__ import annotations

import math

import numpy as np


def branin(x):
    x = np.asarray(x, dtype=np.float64)
    x0 = x[..., :1] * 15.0 - 5.0
    x1 = x[..., 1:] * 15.0
    b = 5.1 / (4 * math.pi**2)
    c = 5 / math.pi
    t = 1 / (8 * math.pi)
    return (x1 - b * x0**2 + c * x0 - 6) ** 2 + 10 * (1 - t) * np.cos(x0) + 10


def scaled_branin(x):
    x = np.asarray(x, dtype=np.float64)
    x0 = x[..., :1] * 15.0 - 5.0
    x1 = x[..., 1:] * 15.0
    b = 5.1 / (4 * math.pi**2)
    c = 5 / math.pi
    t = 1 / (8 * math.pi)
    return (1 / 51.95) * ((x1 - b * x0**2 + c * x0 - 6) ** 2 + 10 * (1 - t) * np.cos(x0) - 44.81)


def ackley(x):
    x = np.asarray(x, dtype=np.float64)
    d = x.shape[-1]
    x = (x - 0.5) * (32.768 * 2.0)
    e1 = -0.2 * np.sqrt((1.0 / d) * np.square(x).sum(-1))
    e2 = (1.0 / d) * np.cos(2.0 * math.pi * x).sum(-1)
    return (-20.0 * np.exp(e1) - np.exp(e2) + 20.0 + math.e)[..., None]


_H6_A = np.array(
    [[10.0, 3.0, 17.0, 3.5, 1.7, 8.0], [0.05, 10.0, 17.0, 0.1, 8.0, 14.0], [3.0, 3.5, 1.7, 10.0, 17.0, 8.0], [17.0, 8.0, 0.05, 10.0, 0.1, 14.0]]
)
_H6_P = np.array(
    [
        [0.1312, 0.1696, 0.5569, 0.0124, 0.8283, 0.5886],
        [0.2329, 0.4135, 0.8307, 0.3736, 0.1004, 0.9991],
        [0.2348, 0.1451, 0.3522, 0.2883, 0.3047, 0.6650],
        [0.4047, 0.8828, 0.8732, 0.5743, 0.1091, 0.0381],
    ]
)


def hartmann_6(x):
    x = np.asarray(x, dtype=np.float64)
    a = np.array([1.0, 1.2, 3.0, 3.2])
    inner = -(_H6_A * (x[..., None, :] - _H6_P) ** 2).sum(-1)
    return -(a * np.exp(inner)).sum(-1, keepdims=True)


# ---- multi-objective (trieste/objectives/multi_objectives.py): minimisation, values [..., L] ----
def vlmop2(x, d: int):
    """VLMOP2 (:60-73): 1 - exp(-|x - 1/sqrt(d)|^2) and 1 - exp(-|x + 1/sqrt(d)|^2), on [-2, 2]^d."""
    x = np.asarray(x, dtype=np.float64)
    if x.shape[-1] != d:
        raise ValueError(f"x must have trailing dimension {d}, got {x.shape}")
    t = 1.0 / math.sqrt(d)
    y1 = 1.0 - np.exp(-np.sum((x - t) ** 2, axis=-1))
    y2 = 1.0 - np.exp(-np.sum((x + t) ** 2, axis=-1))
    return np.stack([y1, y2], axis=-1)


def vlmop2_pareto_optimal_points(n: int, d: int):
    """n points of the VLMOP2 Pareto front (:88-92): the images of the segment x_i = s, s in [-1/sqrt(d), 1/sqrt(d)]."""
    if n <= 0:
        raise ValueError(f"n must be positive, got {n}")
    t = 1.0 / math.sqrt(d)
    x = np.tile(np.linspace(-t, t, n)[:, None], (1, d))
    return vlmop2(x, d)


def dtlz2(x, m: int, d: int):
    """DTLZ2 (:184-212) with m objectives on [0, 1]^d (d > m): objective i is
    (1 + g) prod_{j < m-1-i} cos(pi x_j / 2), times sin(pi x_{m-1-i} / 2) for i > 0, with g = sum_{j >= m-1} (x_j - 1/2)^2."""
    x = np.asarray(x, dtype=np.float64)
    if x.shape[-1] != d:
        raise ValueError(f"x must have trailing dimension {d}, got {x.shape}")
    if not 0 < m < d:
        raise ValueError(f"need 0 < m < d, got m = {m}, d = {d}")
    g = np.sum((x[..., m - 1:] - 0.5) ** 2, axis=-1)
    cos = np.cos(0.5 * math.pi * x)
    out = []
    for i in range(m):
        y = 1.0 + g
        y = y * np.prod(cos[..., : m - 1 - i], axis=-1)
        if i > 0:
            y = y * np.sin(0.5 * math.pi * x[..., m - 1 - i])
        out.append(y)
    return np.stack(out, axis=-1)


def dtlz2_pareto_optimal_points(n: int, m: int, seed=None):
    """n points of the DTLZ2 Pareto front (:226-230): the positive orthant of the unit sphere in m objectives."""
    if m < 2:
        raise ValueError(f"need at least two objectives, got {m}")
    r = np.random.default_rng(seed).standard_normal((n, m))
    return np.abs(r / np.linalg.norm(r, axis=-1, keepdims=True))
