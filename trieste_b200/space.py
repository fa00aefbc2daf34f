"""Minimal search spaces: ``Box`` with i.i.d. uniform sampling (trieste/space.py:843-867), ``DiscreteSearchSpace`` and
``TaggedMultiSearchSpace`` (space.py:1410-1513, the acquisition space of the batch trust-region rules).  Only what the
acquisition optimisers of the hot path need."""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np


class SearchSpace:
    dimension: int

    def sample(self, num_samples: int, seed: Optional[int] = None) -> np.ndarray:  # pragma: no cover
        raise NotImplementedError

    @property
    def has_constraints(self) -> bool:
        return False


class Box(SearchSpace):
    def __init__(self, lower: Sequence[float], upper: Sequence[float]):
        self.lower = np.atleast_1d(np.asarray(lower, dtype=np.float64))
        self.upper = np.atleast_1d(np.asarray(upper, dtype=np.float64))
        if self.lower.shape != self.upper.shape or self.lower.ndim != 1 or self.lower.size == 0:
            raise ValueError(f"lower and upper must be non-empty 1-D of equal shape, got {self.lower.shape}, {self.upper.shape}")
        if np.any(self.lower > self.upper):
            raise ValueError("lower bound must not exceed upper bound")
        self._rng = np.random.default_rng()

    def __repr__(self) -> str:
        return f"Box({self.lower!r}, {self.upper!r})"

    @property
    def dimension(self) -> int:
        return int(self.lower.shape[0])

    def __pow__(self, n: int) -> "Box":
        """Cartesian power, as used by ``batchify_joint`` (acquisition/optimizer.py:924)."""
        return Box(np.tile(self.lower, n), np.tile(self.upper, n))

    def __mul__(self, other: "Box") -> "Box":
        return Box(np.concatenate([self.lower, other.lower]), np.concatenate([self.upper, other.upper]))

    def sample(self, num_samples: int, seed: Optional[int] = None) -> np.ndarray:
        if num_samples < 0:
            raise ValueError(f"num_samples must be non-negative, got {num_samples}")
        rng = self._rng if seed is None else np.random.default_rng(seed)
        u = rng.uniform(size=(num_samples, self.dimension))
        return self.lower + u * (self.upper - self.lower)

    def contains(self, x: np.ndarray) -> np.ndarray:
        x = np.asarray(x)
        return np.all((x >= self.lower) & (x <= self.upper), axis=-1)


class DiscreteSearchSpace(SearchSpace):
    def __init__(self, points: np.ndarray):
        self.points = np.asarray(points, dtype=np.float64)
        if self.points.ndim != 2:
            raise ValueError(f"points must be rank 2, got {self.points.shape}")
        self._rng = np.random.default_rng()

    @property
    def dimension(self) -> int:
        return int(self.points.shape[1])

    def sample(self, num_samples: int, seed: Optional[int] = None) -> np.ndarray:
        rng = self._rng if seed is None else np.random.default_rng(seed)
        if num_samples >= len(self.points):
            return self.points
        return self.points[rng.choice(len(self.points), size=num_samples, replace=False)]


class TaggedMultiSearchSpace(SearchSpace):
    """space.py:1121-1231, 1410-1513: independent subspaces of one dimension D, each with a unique tag.  Accessed all at
    once, the subspaces add an axis: ``lower`` / ``upper`` are [S, D] and ``sample(n)`` is [n, S, D] (column s drawn from
    subspace s), so an optimiser of a function vectorised over V = k * S columns searches column v in subspace v mod S."""

    def __init__(self, spaces: Sequence[SearchSpace], tags: Optional[Sequence[str]] = None):
        if len(spaces) == 0:
            raise ValueError(f"At least one subspace is required but received {len(spaces)}.")
        dims = [int(space.dimension) for space in spaces]
        if len(set(dims)) != 1:
            raise ValueError(f"All subspaces must have the same dimension but received {dims}.")
        if tags is None:
            tags = [str(index) for index in range(len(spaces))]
        elif len(tags) != len(spaces):
            raise ValueError(
                f"Number of tags must match number of subspaces but received {len(tags)} tags and {len(spaces)} subspaces."
            )
        elif len(set(tags)) != len(tags):
            raise ValueError(f"Subspace names must be unique but received {tags}.")
        self._spaces = dict(zip(tags, spaces))
        self._tags = tuple(tags)

    def __repr__(self) -> str:
        return f"TaggedMultiSearchSpace({[self._spaces[t] for t in self._tags]!r}, {self._tags!r})"

    @property
    def subspace_tags(self) -> tuple:
        return self._tags

    def get_subspace(self, tag: str) -> SearchSpace:
        if tag not in self._spaces:
            raise ValueError(
                f"Attempted to access a subspace that does not exist. This space only contains subspaces with the tags "
                f"{self._tags} but received {tag}."
            )
        return self._spaces[tag]

    @property
    def dimension(self) -> int:
        return int(self._spaces[self._tags[0]].dimension)

    @property
    def lower(self) -> np.ndarray:
        return np.stack([np.asarray(self._spaces[t].lower, dtype=np.float64) for t in self._tags])

    @property
    def upper(self) -> np.ndarray:
        return np.stack([np.asarray(self._spaces[t].upper, dtype=np.float64) for t in self._tags])

    def sample(self, num_samples: int, seed: Optional[int] = None) -> np.ndarray:
        """[num_samples, S, D].  A ``seed`` s seeds subspace i with s + i, so that the subspaces draw different uniforms
        (the reference sets one global TensorFlow seed before drawing all of them)."""
        if num_samples < 0:
            raise ValueError(f"num_samples must be non-negative, got {num_samples}")
        seeds = [None] * len(self._tags) if seed is None else [seed + i for i in range(len(self._tags))]
        return np.stack([self._spaces[t].sample(num_samples, seed=sd) for t, sd in zip(self._tags, seeds)], axis=1)

    def contains(self, x: np.ndarray) -> np.ndarray:
        """A point is a member when it lies in any of the subspaces."""
        return np.any([self._spaces[t].contains(x) for t in self._tags], axis=0)
