"""Partitions of the region a Pareto front does not dominate into hyper-rectangular cells (trieste
acquisition/multi_objective/partition.py:28-393), in NumPy: once per BO step on the host.

Both partitions describe each cell by indices into the pseudo front ``[anti_reference, front..., reference]`` and resolve
them against the two corner points only in :meth:`partition_bounds`, so one partition serves any reference pair."""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np

from .dominance import non_dominated

ANTI_REFERENCE_DEFAULT = -1e10  # partition.py:62, acts as -inf
JITTER = 1e-6  # trieste utils/misc.py DEFAULTS.JITTER: tolerance of the divide-and-conquer cell tests


def _vector(x, name: str, L: Optional[int] = None) -> np.ndarray:
    v = np.asarray(x, dtype=np.float64)
    if v.ndim != 1 or (L is not None and v.shape[0] != L):
        want = f"[{L}]" if L is not None else "[L]"
        raise ValueError(f"{name} must have shape {want}, got {v.shape}")
    return v


def prepare_default_non_dominated_partition_bounds(reference, observations=None, anti_reference=None
                                                   ) -> Tuple[np.ndarray, np.ndarray]:
    """Lower and upper bounds [K, L] of the cells that partition the region between ``anti_reference`` and ``reference``
    not dominated by the front ``observations`` [N, L]: the exact staircase for L = 2, divide and conquer for L > 2.
    Without observations (None or empty) the single cell [anti_reference, reference].  The default anti-reference is
    -1e10 in every objective."""
    ref = _vector(reference, "reference")
    L = ref.shape[0]
    obs = None if observations is None else np.asarray(observations, dtype=np.float64)
    empty = obs is None or obs.size == 0
    if anti_reference is None:
        anti = np.full(L, ANTI_REFERENCE_DEFAULT)
        if np.any(ref < anti):
            raise ValueError(f"reference point: {ref} containing at least one value below default anti-reference point "
                             "([-1e10, ..., -1e10]), try specify a lower anti-reference point.")
        if not empty and np.any(obs < anti):
            raise ValueError(f"observations: {obs} containing at least one value below default anti-reference point "
                             "([-1e10, ..., -1e10]), try specify a lower anti-reference point.")
    else:
        anti = _vector(anti_reference, "anti_reference", L)
    if empty:
        if np.any(anti > ref):
            raise ValueError(f"anti_reference point: {anti} contains at least one value larger than reference point: {ref}")
        return anti[None].copy(), ref[None].copy()
    if obs.ndim != 2 or obs.shape[-1] != L:
        raise ValueError(f"observations must have shape [N, {L}], got {obs.shape}")
    part = DividedAndConquerNonDominated(obs) if L > 2 else ExactPartition2dNonDominated(obs)
    return part.partition_bounds(anti, ref)


class _BoundIndexPartition:
    front: np.ndarray
    _lower_idx: np.ndarray  # [K, L] indices into the pseudo front, per objective
    _upper_idx: np.ndarray

    def __init__(self, front):
        f = np.asarray(front, dtype=np.float64)
        if f.ndim != 2:
            raise ValueError(f"front must have shape [N, L], got {f.shape}")
        if not np.all(non_dominated(f)[1]):
            raise ValueError(f"\ninput {f} contains dominated points")
        self.front = f

    def partition_bounds(self, anti_reference, reference) -> Tuple[np.ndarray, np.ndarray]:
        """Lower and upper bounds [K, L] of the cells for this pair of corner points."""
        L = self.front.shape[1]
        anti = _vector(anti_reference, "anti_reference", L)
        ref = _vector(reference, "reference", L)
        if np.any(ref < self.front):
            raise ValueError(f"reference point {ref} is below the anti-ideal point of the front")
        if np.any(self.front < anti):
            raise ValueError(f"the front has points below the anti-reference point {anti}")
        pseudo = np.concatenate([anti[None], self.front, ref[None]], axis=0)
        cols = np.arange(L)[None, :]
        return pseudo[self._lower_idx, cols], pseudo[self._upper_idx, cols]


class ExactPartition2dNonDominated(_BoundIndexPartition):
    """The exact partition for two objectives: with the front sorted by the first objective (so the second descends),
    cell i spans [x_i, x_{i+1}] x [anti_2, y_i], where x_0 = anti_1, x_{n+1} = ref_1 and y_0 = ref_2."""

    def __init__(self, front):
        super().__init__(front)
        self.front = self.front[np.argsort(self.front[:, 0], kind="stable")]
        n = self.front.shape[0]
        i = np.arange(n + 1)
        self._lower_idx = np.stack([i, np.zeros_like(i)], axis=1)
        self._upper_idx = np.stack([i + 1, np.where(i == 0, n + 1, i)], axis=1)


class DividedAndConquerNonDominated(_BoundIndexPartition):
    """Divide and conquer over the grid of the front's coordinate ranks (Couckuyt et al. 2012).  A grid cell is taken
    when no front point weakly dominates its upper corner, dropped when one dominates its lower corner, and otherwise
    halved along its longest edge (in ranks).  ``threshold`` > 0 also drops cells whose volume is at most that fraction
    of the front's bounding box, which makes the partition approximate."""

    def __init__(self, front, threshold: float = 0):
        super().__init__(front)
        f = self.front
        n, L = f.shape
        order = np.argsort(f, axis=0, kind="stable") + 1  # rank r of objective l -> row of the pseudo front
        rank_to_row = np.concatenate([np.zeros((1, L), dtype=np.int64), order, np.full((1, L), n + 1)], axis=0)
        lo_pt, hi_pt = f.min(axis=0) - 1, f.max(axis=0) + 1
        pseudo = np.concatenate([lo_pt[None], f, hi_pt[None]], axis=0)
        total = np.prod(hi_pt - lo_pt)
        cols = np.arange(L)
        lower_idx, upper_idx = [], []
        stack = [(np.zeros(L, dtype=np.int64), np.full(L, n + 1, dtype=np.int64))]
        while stack:
            lo, hi = stack.pop()
            li, ui = rank_to_row[lo, cols], rank_to_row[hi, cols]
            lower, upper = pseudo[li, cols], pseudo[ui, cols]
            accepted = np.all(np.any(upper - JITTER < f, axis=1))
            if accepted:
                lower_idx.append(li)
                upper_idx.append(ui)
                continue
            if not np.all(np.any(lower + JITTER < f, axis=1)):
                continue  # dominated
            dist = hi - lo
            if np.any(dist > 1) and np.prod(upper - lower) / total > threshold:
                d = int(np.argmax(dist))
                half = int(np.round(dist[d] / 2.0))
                first_hi = hi.copy()
                first_hi[d] -= half
                second_lo = lo.copy()
                second_lo[d] += dist[d] - half
                stack.append((lo, first_hi))
                stack.append((second_lo, hi))
        empty = np.zeros((0, L), dtype=np.int64)
        self._lower_idx = np.array(lower_idx, dtype=np.int64) if lower_idx else empty
        self._upper_idx = np.array(upper_idx, dtype=np.int64) if upper_idx else empty
