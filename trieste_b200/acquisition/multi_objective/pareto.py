"""Pareto fronts and their hypervolume (trieste acquisition/multi_objective/pareto.py:29-80, 270-287), in NumPy."""
from __future__ import annotations

import numpy as np

from .dominance import non_dominated
from .partition import prepare_default_non_dominated_partition_bounds


class Pareto:
    """The Pareto front of ``observations`` [N, L] (L >= 2), or the observations themselves when they are known to be
    non-dominated."""

    def __init__(self, observations, already_non_dominated: bool = False):
        obs = np.asarray(observations, dtype=np.float64)
        if obs.ndim != 2:
            raise ValueError(f"observations must have rank 2, got shape {obs.shape}")
        if obs.shape[-1] < 2:
            raise ValueError(f"observations need at least two objectives, got shape {obs.shape}")
        self.front = obs if already_non_dominated else non_dominated(obs)[0]

    def hypervolume_indicator(self, reference) -> float:
        """Volume of the region the front dominates below ``reference`` [L]: the box [min(front) - 1, reference] less the
        cells of its non-dominated partition.  Raises ValueError for an empty front, a reference that is not of shape
        [L], and a reference below any front point in some objective (below the front's anti-ideal point)."""
        if self.front.size == 0:
            raise ValueError("empty front cannot be used to calculate hypervolume indicator")
        anti = self.front.min(axis=0) - 1.0
        lower, upper = prepare_default_non_dominated_partition_bounds(reference, self.front, anti)
        ref = np.asarray(reference, dtype=np.float64)
        return float(np.prod(ref - anti) - np.sum(np.prod(upper - lower, axis=1)))


def get_reference_point(observations) -> np.ndarray:
    """The default reference point of a set of observations [N, L]: the worst point of their front plus twice its
    range over the front's size, max(front) + 2 (max(front) - min(front)) / |front|."""
    obs = np.asarray(observations, dtype=np.float64)
    if obs.size == 0:
        raise ValueError("empty observations cannot be used to calculate reference point")
    front = Pareto(obs).front
    hi, lo = front.max(axis=-2), front.min(axis=-2)
    return hi + 2.0 * (hi - lo) / front.shape[-2]
