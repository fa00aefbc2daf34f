"""Pareto dominance (trieste acquisition/multi_objective/dominance.py:23-70), in NumPy: once per BO step on the host."""
from __future__ import annotations

from typing import Tuple

import numpy as np

_BLOCK = 1024  # rows compared against all others at a time: bounds the [block, N, L] comparison


def non_dominated(observations) -> Tuple[np.ndarray, np.ndarray]:
    """The non-dominated points of ``observations`` [N, L] (minimisation) and the mask [N] of which rows they are.

    Row i is dominated when some row is <= it in every objective and < it in one.  Duplicates of a non-dominated point
    are all kept.  The front lists the non-dominated rows in their input order."""
    obs = np.asarray(observations, dtype=np.float64)
    if obs.ndim != 2:
        raise ValueError(f"observations must have shape [N, L], got {obs.shape}")
    n = obs.shape[0]
    mask = np.ones(n, dtype=bool)
    for i0 in range(0, n, _BLOCK):
        blk = obs[i0:i0 + _BLOCK]  # [b, L]
        le = np.all(obs[None, :, :] <= blk[:, None, :], axis=-1)  # [b, N]: row j <= row i everywhere
        lt = np.any(obs[None, :, :] < blk[:, None, :], axis=-1)
        mask[i0:i0 + _BLOCK] = ~np.any(le & lt, axis=1)
    return obs[mask], mask
