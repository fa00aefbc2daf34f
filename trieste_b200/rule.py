"""Acquisition rules — mirrors trieste/acquisition/rule.py (``EfficientGlobalOptimization`` :209-399,
``DiscreteThompsonSampling`` :879-994, and the box trust regions: ``SingleObjectiveTrustRegionBox`` / ``TREGOBox`` /
``TURBOBox`` :1569-2218 with ``BatchTrustRegionBox`` :1261-1566, 1863-1920).  Rules are per-BO-step orchestration on the
host; each region's acquisition runs through the same device paths as a plain ``Box``.  Local models and datasets
(``LocalizedTag``), discrete, product and categorical regions and the asynchronous rules are out of scope."""
from __future__ import annotations

import copy
from typing import Mapping, Optional, Sequence, Tuple, Union

import numpy as np

from .acquisition.function import ExpectedImprovement
from .acquisition.interface import (
    OBJECTIVE,
    AcquisitionFunctionBuilder,
    GreedyAcquisitionFunctionBuilder,
    SingleModelAcquisitionBuilder,
    SingleModelGreedyAcquisitionBuilder,
    VectorizedAcquisitionFunctionBuilder,
)
from .acquisition.optimizer import automatic_optimizer_selector, batchify_joint, batchify_vectorize
from .acquisition.sampler import ExactThompsonSampler, ThompsonSamplerFromTrajectory  # noqa: F401
from .data import Dataset
from .space import Box, SearchSpace, TaggedMultiSearchSpace


class EfficientGlobalOptimization:
    """rule.py:209-399: build (or update in place) the acquisition function, then maximise it."""

    def __init__(self, builder=None, optimizer=None, num_query_points: int = 1):
        if num_query_points <= 0:
            raise ValueError(f"Number of query points must be greater than 0, got {num_query_points}")
        if builder is None:
            if num_query_points != 1:
                raise ValueError("a batch acquisition builder must be given for num_query_points > 1")
            builder = ExpectedImprovement()
        if optimizer is None:
            optimizer = automatic_optimizer_selector
        if isinstance(builder, (SingleModelAcquisitionBuilder, SingleModelGreedyAcquisitionBuilder)):
            builder = builder.using(OBJECTIVE)
        if num_query_points > 1:  # rule.py:291-301
            if isinstance(builder, VectorizedAcquisitionFunctionBuilder):
                optimizer = batchify_vectorize(optimizer, num_query_points)  # batch elements optimised independently
            elif isinstance(builder, AcquisitionFunctionBuilder):
                optimizer = batchify_joint(optimizer, num_query_points)  # ... jointly over space ** q
            # a GreedyAcquisitionFunctionBuilder collects the batch sequentially in acquire()
        self._builder = builder
        self._optimizer = optimizer
        self._num_query_points = num_query_points
        self._acquisition_function = None

    def __repr__(self) -> str:
        return f"EfficientGlobalOptimization({self._builder!r}, {self._optimizer!r}, {self._num_query_points!r})"

    @property
    def acquisition_function(self):
        return self._acquisition_function

    def acquire(self, search_space: SearchSpace, models: Mapping[str, object],
                datasets: Optional[Mapping[str, Dataset]] = None) -> np.ndarray:
        if self._acquisition_function is None:
            self._acquisition_function = self._builder.prepare_acquisition_function(models, datasets=datasets)
        else:
            self._acquisition_function = self._builder.update_acquisition_function(
                self._acquisition_function, models, datasets=datasets
            )
        points = self._optimizer(search_space, self._acquisition_function)
        if isinstance(self._builder, GreedyAcquisitionFunctionBuilder):
            for _ in range(self._num_query_points - 1):  # rule.py:371-385: greedily allocate the remaining batch elements
                self._acquisition_function = self._builder.update_acquisition_function(
                    self._acquisition_function, models, datasets=datasets, pending_points=points, new_optimization_step=False
                )
                chosen_point = self._optimizer(search_space, self._acquisition_function)
                points = np.concatenate([points, chosen_point], axis=0)
        return points

    def acquire_single(self, search_space, model, dataset=None):
        return self.acquire(search_space, {OBJECTIVE: model}, None if dataset is None else {OBJECTIVE: dataset})


class DiscreteThompsonSampling:
    """rule.py:879-994: sample ``num_search_space_samples`` candidates, pick ``num_query_points`` by
    Thompson sampling from trajectories."""

    def __init__(self, num_search_space_samples: int, num_query_points: int, thompson_sampler=None):
        if not num_search_space_samples > 0:
            raise ValueError(f"Search space must be greater than 0, got {num_search_space_samples}")
        if not num_query_points > 0:
            raise ValueError(f"Number of query points must be greater than 0, got {num_query_points}")
        if thompson_sampler is not None:
            if thompson_sampler.sample_min_value:
                raise ValueError(
                    "Thompson sampling requires a thompson_sampler that samples minimizers, not just minimum values. "
                    "However the passed sampler has sample_min_value=True."
                )
        else:
            # rule.py:942-943: the reference default — exact joint samples, O(M^3) in the candidate count; pass
            # ThompsonSamplerFromTrajectory() for large candidate sets (BASELINE config 4)
            thompson_sampler = ExactThompsonSampler(sample_min_value=False)
        self._thompson_sampler = thompson_sampler
        self._num_search_space_samples = num_search_space_samples
        self._num_query_points = num_query_points

    def __repr__(self) -> str:
        return f"DiscreteThompsonSampling({self._num_search_space_samples!r}, {self._num_query_points!r}, {self._thompson_sampler!r})"

    def acquire(self, search_space: SearchSpace, models, datasets=None) -> np.ndarray:
        if OBJECTIVE not in models:
            raise ValueError(f"dict of models must contain the single key {OBJECTIVE}, got keys {list(models.keys())}")
        query_points = search_space.sample(self._num_search_space_samples)
        return self._thompson_sampler.sample(models[OBJECTIVE], self._num_query_points, query_points)

    def acquire_single(self, search_space, model, dataset=None):
        return self.acquire(search_space, {OBJECTIVE: model}, None if dataset is None else {OBJECTIVE: dataset})


# ---------------------------------------------------------------------------------------------------
# box trust regions (rule.py:1039-1236, 1569-2218)
# ---------------------------------------------------------------------------------------------------
def _objective_dataset(datasets: Optional[Mapping[str, Dataset]]) -> Dataset:
    if datasets is None or len(datasets) != 1 or next(iter(datasets)) != OBJECTIVE:
        raise ValueError("a single OBJECTIVE dataset must be provided")
    return next(iter(datasets.values()))


class UpdatableTrustRegionBox(Box):
    """rule.py:1780-1820: a box with a centre ``location`` inside a global ``Box``; ``lower`` / ``upper`` are the current
    bounds of the region.  Subclasses set ``_initialized`` in ``initialize`` and move the bounds in ``update``."""

    def __init__(self, global_search_space: Box, region_index: Optional[int] = None):
        Box.__init__(self, global_search_space.lower, global_search_space.upper)
        self._global_search_space = global_search_space
        self.region_index = region_index
        self._initialized = False

    @property
    def global_search_space(self) -> Box:
        return self._global_search_space

    @property
    def requires_initialization(self) -> bool:
        return not self._initialized

    def _init_location(self, location_candidate: Optional[np.ndarray] = None) -> None:
        if location_candidate is not None:
            self.location = np.asarray(location_candidate, dtype=np.float64)
        else:
            self.location = self.global_search_space.sample(1)[0]

    def _get_bounds_within_distance(self, eps) -> Tuple[np.ndarray, np.ndarray]:
        lower = np.maximum(self.global_search_space.lower, self.location - eps)
        upper = np.minimum(self.global_search_space.upper, self.location + eps)
        return lower, upper


class SingleObjectiveTrustRegionBox(UpdatableTrustRegionBox):
    """rule.py:1585-1777, 1823-1860 (``HypercubeTrustRegion`` for a box): the region is ``location ± eps`` clipped to the
    global box, ``eps`` starting at ``zeta`` times the global widths.  A step succeeds when the best observation inside
    the region beats the previous best by ``kappa`` times the region's volume; ``eps`` then grows by ``1 / beta`` and the
    centre moves to that observation, otherwise ``eps`` shrinks by ``beta``.  Below ``min_eps`` the region re-initialises."""

    def __init__(self, global_search_space: Box, beta: float = 0.7, kappa: float = 1e-4, zeta: float = 0.5,
                 min_eps: float = 1e-2, region_index: Optional[int] = None):
        UpdatableTrustRegionBox.__init__(self, global_search_space, region_index)
        self._beta = beta
        self._kappa = kappa
        self._zeta = zeta
        self._min_eps = min_eps
        self._step_is_success = False
        self._init_location()
        self._init_eps()
        self._update_domain()
        self._y_min = np.inf

    def __repr__(self) -> str:
        return (f"{type(self).__name__}({self.global_search_space!r}, {self._beta!r}, {self._kappa!r}, {self._zeta!r}, "
                f"{self._min_eps!r}, {self.region_index!r})")

    def _init_eps(self) -> None:
        self.eps = self._zeta * (self.global_search_space.upper - self.global_search_space.lower)

    def _update_domain(self) -> None:
        self.lower, self.upper = self._get_bounds_within_distance(self.eps)

    @property
    def requires_initialization(self) -> bool:
        return not self._initialized or bool(np.any(self.eps < self._min_eps))

    def initialize(self, models=None, datasets: Optional[Mapping[str, Dataset]] = None,
                   location_candidate: Optional[np.ndarray] = None) -> None:
        self._init_location(location_candidate)
        self._step_is_success = False
        self._init_eps()
        self._update_domain()
        self._y_min = np.inf  # the first update always succeeds
        self._initialized = True

    def update(self, models=None, datasets: Optional[Mapping[str, Dataset]] = None) -> None:
        x_min, y_min = self.get_dataset_min(datasets)
        tr_volume = np.prod(self.upper - self.lower)
        self._step_is_success = bool(y_min < self._y_min - self._kappa * tr_volume)
        self.eps = self.eps / self._beta if self._step_is_success else self.eps * self._beta
        if self._step_is_success:
            self.location = x_min
            self._y_min = y_min
        self._update_domain()

    def get_values_min(self, query_points: np.ndarray, values: np.ndarray, num_query_points: Optional[int] = None,
                       in_region_only: bool = True) -> Tuple[np.ndarray, float]:
        """rule.py:1711-1750: (point, value) of the smallest value, optionally of the latest points and inside the
        region only (+inf when none is inside)."""
        qps = np.asarray(query_points) if num_query_points is None else np.asarray(query_points)[-num_query_points:]
        vals = np.asarray(values)[-len(qps):, 0]
        if in_region_only:
            vals = np.where(self.contains(qps), vals, np.inf)
        ix = int(np.argmin(vals))
        return qps[ix], float(vals[ix])

    def get_dataset_min(self, datasets: Optional[Mapping[str, Dataset]]) -> Tuple[np.ndarray, float]:
        dataset = _objective_dataset(datasets)
        return self.get_values_min(dataset.query_points, dataset.observations, in_region_only=True)


class TREGOBox(SingleObjectiveTrustRegionBox):
    """rule.py:1923-2035 (TREGO, Diouane et al. 2022): alternates global steps over the whole space with local steps in
    the trust region.  A success returns to (or stays in) global mode; a failure switches mode.  ``eps`` only changes
    after a local step, and the best point is taken over the whole (global) dataset."""

    def __init__(self, global_search_space: Box, beta: float = 0.7, kappa: float = 1e-4, zeta: float = 0.5,
                 min_eps: float = 1e-2, region_index: Optional[int] = None):
        self._is_global = False
        super().__init__(global_search_space, beta, kappa, zeta, min_eps, region_index)

    @property
    def eps(self):
        return self._eps

    @eps.setter
    def eps(self, eps) -> None:
        if not self._is_global:  # the size is frozen in global mode
            self._eps = eps

    def _update_domain(self) -> None:
        self._is_global = self._step_is_success or not self._is_global
        if self._is_global:
            self.lower, self.upper = self.global_search_space.lower, self.global_search_space.upper
        else:
            super()._update_domain()

    def initialize(self, models=None, datasets=None, location_candidate=None) -> None:
        # global mode at the first initialisation, local mode at re-initialisations (_update_domain flips the mode)
        self._is_global = self._initialized
        super().initialize(models, datasets, location_candidate)

    def get_dataset_min(self, datasets: Optional[Mapping[str, Dataset]]) -> Tuple[np.ndarray, float]:
        dataset = _objective_dataset(datasets)
        return self.get_values_min(dataset.query_points, dataset.observations, in_region_only=False)


class TURBOBox(UpdatableTrustRegionBox):
    """rule.py:2038-2218 (TuRBO, Eriksson et al. 2019): a box of side ``L`` centred on the best observation, stretched
    by the model's lengthscales at fixed volume.  ``success_tolerance`` consecutive improvements double ``L`` (up to
    ``L_max``), ``failure_tolerance`` consecutive failures halve it, and below ``L_min`` the region restarts at
    ``L_init``.  Unset lengths follow the reference's heuristics from the widest side of the global box."""

    def __init__(self, global_search_space: Box, L_min: Optional[float] = None, L_init: Optional[float] = None,
                 L_max: Optional[float] = None, success_tolerance: int = 3, failure_tolerance: Optional[int] = None,
                 region_index: Optional[int] = None):
        super().__init__(global_search_space, region_index)
        self._init_location()
        width = float(np.max(global_search_space.upper - global_search_space.lower))
        L_min = 0.5**7 * width if L_min is None else L_min
        L_init = 0.8 * width if L_init is None else L_init
        L_max = 1.6 * width if L_max is None else L_max
        if L_min <= 0:
            raise ValueError(f"L_min must be postive, got {L_min}")
        if L_init <= 0:
            raise ValueError(f"L_init must be postive, got {L_init}")
        if L_max <= 0:
            raise ValueError(f"L_max must be postive, got {L_max}")
        self.L_min, self.L_init, self.L_max = L_min, L_init, L_max
        self.L = L_init
        self.success_tolerance = success_tolerance
        self.failure_tolerance = failure_tolerance if failure_tolerance is not None else global_search_space.dimension
        self.success_counter = 0
        self.failure_counter = 0
        if self.success_tolerance <= 0:
            raise ValueError(f"success tolerance must be an integer greater than 0, got {self.success_tolerance}")
        if self.failure_tolerance <= 0:
            raise ValueError(f"success tolerance must be an integer greater than 0, got {self.failure_tolerance}")
        self.y_min = np.inf
        self.tr_width = global_search_space.upper - global_search_space.lower
        self._update_domain()

    def __repr__(self) -> str:
        return (f"TURBOBox({self.global_search_space!r}, {self.L_min!r}, {self.L_init!r}, {self.L_max!r}, "
                f"{self.success_tolerance!r}, {self.failure_tolerance!r}, {self.region_index!r})")

    def _set_tr_width(self, models=None) -> None:
        if models is None or len(models) != 1 or next(iter(models)) != OBJECTIVE:
            raise ValueError("a single OBJECTIVE model must be provided")
        model = next(iter(models.values()))
        D = self.global_search_space.dimension
        lengthscales = np.broadcast_to(np.asarray(model.get_kernel().lengthscales, dtype=np.float64), (D,))
        self.tr_width = lengthscales * self.L / np.prod(lengthscales) ** (1.0 / D)  # volume L^D

    def _update_domain(self) -> None:
        self.lower = np.maximum(self.global_search_space.lower, self.location - self.tr_width / 2.0)
        self.upper = np.minimum(self.global_search_space.upper, self.location + self.tr_width / 2.0)

    def initialize(self, models=None, datasets: Optional[Mapping[str, Dataset]] = None) -> None:
        x_min, self.y_min = self.get_dataset_min(datasets)
        self.location = x_min
        self.L, self.failure_counter, self.success_counter = self.L_init, 0, 0
        self._set_tr_width(models)
        self._update_domain()
        self._initialized = True

    def update(self, models=None, datasets: Optional[Mapping[str, Dataset]] = None) -> None:
        x_min, y_min = self.get_dataset_min(datasets)
        self.location = x_min
        step_is_success = y_min < self.y_min - 1e-10
        self.y_min = y_min
        self.failure_counter = 0 if step_is_success else self.failure_counter + 1
        self.success_counter = self.success_counter + 1 if step_is_success else 0
        if self.success_counter == self.success_tolerance:
            self.L *= 2.0
            self.success_counter = 0
        elif self.failure_counter == self.failure_tolerance:
            self.L *= 0.5
            self.failure_counter = 0
        self.L = min(self.L, self.L_max)
        if self.L < self.L_min:  # too small: start again
            self.L, self.failure_counter, self.success_counter = self.L_init, 0, 0
        self._set_tr_width(models)
        self._update_domain()

    def get_dataset_min(self, datasets: Optional[Mapping[str, Dataset]]) -> Tuple[np.ndarray, float]:
        dataset = _objective_dataset(datasets)
        ix = int(np.argmin(dataset.observations[:, 0]))
        return dataset.query_points[ix], float(dataset.observations[ix, 0])


def get_unique_points_mask(points: np.ndarray, tolerance: float = 1e-6) -> np.ndarray:
    """acquisition/utils.py:211-255: greedy cover — a point is kept unless it lies within ``tolerance`` (Euclidean) of
    an earlier kept point."""
    points = np.asarray(points, dtype=np.float64)
    mask = np.zeros(len(points), dtype=bool)
    for i in range(len(points)):
        mask[i] = not np.any(np.linalg.norm(points[:i][mask[:i]] - points[i], axis=-1) <= tolerance)
    return mask


class BatchTrustRegionBox:
    """rule.py:1261-1566, 1863-1920: one query batch per trust region, the regions updated from the data between steps.

    The rule keeps its regions: the first ``acquire`` initialises them (the reference's first ``filter_datasets``);
    every later call first updates them from the datasets it receives — re-initialising regions that have shrunk below
    their minimum size or share a centre with an earlier region — and then acquires.  With an
    ``EfficientGlobalOptimization`` base rule the acquisition runs once over a ``TaggedMultiSearchSpace`` of the
    regions, column v of a vectorised function searching region v mod S; any other base rule is deep-copied once per
    region and run inside it.  ``acquire`` returns the [q, S, D] points flattened to [q * S, D]."""

    def __init__(self, init_subspaces: Union[None, UpdatableTrustRegionBox, Sequence[UpdatableTrustRegionBox]] = None,
                 rule=None):
        self._init_subspaces = None
        self._tags = None
        if init_subspaces is not None:
            if not isinstance(init_subspaces, Sequence):
                init_subspaces = [init_subspaces]
            self._init_subspaces = tuple(init_subspaces)
            for index, subspace in enumerate(self._init_subspaces):
                subspace.region_index = index
            self._tags = tuple(str(index) for index in range(len(self._init_subspaces)))
        self._rule = rule
        self._rules = None  # one deep copy of the base rule per region, when the base rule is run per region
        self._subspaces: Optional[Tuple[UpdatableTrustRegionBox, ...]] = None  # the current regions

    def __repr__(self) -> str:
        return f"BatchTrustRegionBox({self._init_subspaces!r}, {self._rule!r})"

    @property
    def num_local_datasets(self) -> int:
        assert self._init_subspaces is not None, "the subspaces have not been initialized"
        return len(self._init_subspaces)

    @property
    def subspaces(self) -> Optional[Tuple[UpdatableTrustRegionBox, ...]]:
        """The current regions (``None`` before the first ``acquire``)."""
        return self._subspaces

    def initialize_subspaces(self, search_space: SearchSpace) -> None:
        """rule.py:1869-1890: without initial regions, one ``SingleObjectiveTrustRegionBox`` per query point of an EGO
        base rule (one otherwise)."""
        if self._init_subspaces is None:
            num_query_points = self._rule._num_query_points if isinstance(self._rule, EfficientGlobalOptimization) else 1
            if not isinstance(search_space, Box):
                raise ValueError(f"search space should be a Box, got {type(search_space)}")
            self._init_subspaces = tuple(
                SingleObjectiveTrustRegionBox(search_space, region_index=i) for i in range(num_query_points)
            )
            self._tags = tuple(str(index) for index in range(num_query_points))

    def get_initialize_subspaces_mask(self, subspaces, models, datasets=None) -> np.ndarray:
        """rule.py:1911-1920: re-initialise the regions whose centres duplicate an earlier region's."""
        centres = np.stack([np.asarray(subspace.location, dtype=np.float64) for subspace in subspaces])
        return ~get_unique_points_mask(centres, tolerance=1e-6)

    def maybe_initialize_subspaces(self, subspaces, models, datasets=None) -> None:
        mask = self.get_initialize_subspaces_mask(subspaces, models, datasets)
        for ix, subspace in enumerate(subspaces):
            if mask[ix]:
                subspace.initialize(models, datasets)

    def update_subspaces(self, models, datasets) -> None:
        """rule.py:1501-1533 for global data: initialise or update every region, then re-initialise duplicates."""
        if self._subspaces is None:
            self._subspaces = copy.deepcopy(self._init_subspaces)  # leave the caller's regions untouched
        for subspace in self._subspaces:
            if subspace.requires_initialization:
                subspace.initialize(models, datasets)
            else:
                subspace.update(models, datasets)
        self.maybe_initialize_subspaces(self._subspaces, models, datasets)

    def acquire(self, search_space: SearchSpace, models: Mapping[str, object],
                datasets: Optional[Mapping[str, Dataset]] = None) -> np.ndarray:
        for subspace in self._init_subspaces or ():
            glob = subspace.global_search_space
            if not (isinstance(search_space, Box) and np.array_equal(glob.lower, search_space.lower)
                    and np.array_equal(glob.upper, search_space.upper)):
                raise ValueError(
                    "The global search space of the subspaces should be the same as the search space passed to the "
                    "BatchTrustRegionBox acquisition rule. If you want to change the global search space, you should "
                    "recreate the rule. Note: all subspaces should be initialized with the same global search space."
                )
        self.initialize_subspaces(search_space)
        if self._rule is None:  # rule.py:1354-1362
            if isinstance(self._init_subspaces[0], TURBOBox):
                self._rule = DiscreteThompsonSampling(min(100 * search_space.dimension, 5000), 1)
            else:
                self._rule = EfficientGlobalOptimization()
        if self._rules is None and not isinstance(self._rule, EfficientGlobalOptimization):
            self._rules = [copy.deepcopy(self._rule) for _ in self._tags]
        self.update_subspaces(models, datasets)
        subspaces = self._subspaces
        if self._rules is not None:
            points = np.stack([rule.acquire(subspace, models, datasets) for subspace, rule in zip(subspaces, self._rules)],
                              axis=1)
        else:
            points = self._rule.acquire(TaggedMultiSearchSpace(subspaces, self._tags), models, datasets)
        points = np.asarray(points).reshape(-1, len(subspaces), points.shape[-1])  # [q, S, D]
        return points.reshape(-1, points.shape[-1])
