"""Acquisition rules — mirrors trieste/acquisition/rule.py (``EfficientGlobalOptimization`` :209-399,
``DiscreteThompsonSampling`` :879-994, and the box trust regions: ``SingleObjectiveTrustRegionBox`` / ``TREGOBox`` /
``TURBOBox`` :1569-2218 with ``BatchTrustRegionBox`` :1261-1566, 1863-1920).  Rules are per-BO-step orchestration on the
host; each region's acquisition runs through the same device paths as a plain ``Box``.  Regions may have local models and
datasets (``LocalizedTag``, rule.py:1099-1232, 1364-1435, 1501-1566); discrete, product and categorical regions and the
asynchronous rules are out of scope."""
from __future__ import annotations

import copy
from collections import Counter
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
from .utils import LocalizedTag


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
        base_optimizer = optimizer  # before batchify: BatchTrustRegionBox's batched local-model route vectorises it itself
        if num_query_points > 1:  # rule.py:291-301
            if isinstance(builder, VectorizedAcquisitionFunctionBuilder):
                optimizer = batchify_vectorize(optimizer, num_query_points)  # batch elements optimised independently
            elif isinstance(builder, AcquisitionFunctionBuilder):
                optimizer = batchify_joint(optimizer, num_query_points)  # ... jointly over space ** q
            # a GreedyAcquisitionFunctionBuilder collects the batch sequentially in acquire()
        self._builder = builder
        self._base_optimizer = base_optimizer
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
    if datasets is None or len(datasets) != 1 or LocalizedTag.from_tag(next(iter(datasets))).global_tag != OBJECTIVE:
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

    def _get_tags(self, tags):
        """rule.py:1099-1114: (global parts of this region's local tags, global tags without a local tag here)."""
        local_gtags, global_tags = set(), set()
        for tag in tags:
            ltag = LocalizedTag.from_tag(tag)
            if not ltag.is_local:
                global_tags.add(tag)
            elif ltag.local_index == self.region_index:
                local_gtags.add(ltag.global_tag)
        return local_gtags, global_tags - local_gtags

    def select_in_region(self, mapping):
        """rule.py:1177-1206: the items of this region — for each tag its local item of this region's index, else the
        global one (only the global items without an index); None when there are none."""
        if mapping is None:
            _mapping = {}
        elif self.region_index is None:
            _mapping = {tag: item for tag, item in mapping.items() if not LocalizedTag.from_tag(tag).is_local}
        else:
            local_gtags, global_tags = self._get_tags(set(mapping))
            _mapping = {}
            for tag in local_gtags:
                ltag = LocalizedTag(tag, self.region_index)
                _mapping[ltag] = mapping[ltag]
            for tag in global_tags:
                _mapping[tag] = mapping[tag]
        return _mapping if _mapping else None

    def get_datasets_filter_mask(self, datasets):
        """rule.py:1208-1232: for each of this region's local datasets, the mask of its points inside the region."""
        assert self.region_index is not None, "the region_index should be set for filtering local datasets"
        if datasets is None:
            return None
        return {
            tag: self.contains(np.asarray(dataset.query_points))
            for tag, dataset in datasets.items()
            if LocalizedTag.from_tag(tag).local_index == self.region_index
        }


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
        x_min, y_min = self.get_dataset_min(self.select_in_region(datasets))
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

    def get_datasets_filter_mask(self, datasets):
        """rule.py:2003-2020: TREGO keeps its whole local dataset."""
        assert self.region_index is not None, "the region_index should be set for filtering local datasets"
        if datasets is None:
            return None
        return {
            tag: np.ones(np.asarray(dataset.query_points).shape[:-1], dtype=bool)
            for tag, dataset in datasets.items()
            if LocalizedTag.from_tag(tag).local_index == self.region_index
        }


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
        if models is None or len(models) != 1 or LocalizedTag.from_tag(next(iter(models))).global_tag != OBJECTIVE:
            raise ValueError("a single OBJECTIVE model must be provided")
        model = next(iter(models.values()))
        D = self.global_search_space.dimension
        lengthscales = np.broadcast_to(np.asarray(model.get_kernel().lengthscales, dtype=np.float64), (D,))
        self.tr_width = lengthscales * self.L / np.prod(lengthscales) ** (1.0 / D)  # volume L^D

    def _update_domain(self) -> None:
        self.lower = np.maximum(self.global_search_space.lower, self.location - self.tr_width / 2.0)
        self.upper = np.minimum(self.global_search_space.upper, self.location + self.tr_width / 2.0)

    def initialize(self, models=None, datasets: Optional[Mapping[str, Dataset]] = None) -> None:
        x_min, self.y_min = self.get_dataset_min(self.select_in_region(datasets))
        self.location = x_min
        self.L, self.failure_counter, self.success_counter = self.L_init, 0, 0
        self._set_tr_width(self.select_in_region(models))
        self._update_domain()
        self._initialized = True

    def update(self, models=None, datasets: Optional[Mapping[str, Dataset]] = None) -> None:
        x_min, y_min = self.get_dataset_min(self.select_in_region(datasets))
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
        self._set_tr_width(self.select_in_region(models))
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

    The rule keeps its regions.  With global models and datasets only, the first ``acquire`` initialises them (the
    reference's first ``filter_datasets``) and every later call first updates them from the datasets it receives —
    re-initialising regions that have shrunk below their minimum size or share a centre with an earlier region — and then
    acquires.  With local datasets (``LocalizedTag``, see ``with_local_datasets``) ``filter_datasets`` updates the regions
    and ``acquire`` only acquires, as in the reference.

    With an ``EfficientGlobalOptimization`` base rule and global models the acquisition runs once over a
    ``TaggedMultiSearchSpace`` of the regions, column v of a vectorised function searching region v mod S.  Otherwise the
    base rule is deep-copied once per region and each copy acquires inside its region with that region's models and
    datasets under their global tags.  With local models, an ``EfficientGlobalOptimization`` base rule whose builder is
    not greedy and region functions that all maximise on the device (a fused single-query function on a model of its
    own, or the negated trajectories of ``ParallelContinuousThompsonSampling``), the regions' functions are stacked into
    one function over V = k * S columns and the base optimiser runs once over the regions, every region's L-BFGS in one
    device call (``tb_acq_maximize_models`` / ``tb_rff_maximize_models``).  ``acquire`` returns the [q, S, D] points
    flattened to [q * S, D]."""

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
        self._filtered = {}  # the local datasets of the last filter_datasets

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

    def filter_datasets(self, models, datasets):
        """rule.py:1501-1566: update the regions from ``datasets`` (as ``update_subspaces``), then keep the points of each
        local dataset that lie inside its own region (TREGO keeps them all); global datasets pass through unchanged.

        Deviation: a local dataset that filtering would leave empty (a region re-initialised away from all of its
        points) keeps the dataset it had after the previous filtering — the first time, the one it was given — so its
        model stays as it is.  The reference conditions that region's GPR on no data and searches it under the prior;
        the device GPR needs at least one point."""
        self.update_subspaces(models, datasets)
        used_masks = {
            tag: np.zeros(np.asarray(dataset.query_points).shape[:-1], dtype=bool)
            for tag, dataset in datasets.items()
            if LocalizedTag.from_tag(tag).is_local
        }
        for subspace in self._subspaces:
            in_region_masks = subspace.get_datasets_filter_mask(datasets)
            for tag, in_region in (in_region_masks or {}).items():
                used_masks[tag] = used_masks[tag] | np.asarray(in_region, dtype=bool)
        filtered = {}
        for tag, used_mask in used_masks.items():
            dataset = datasets[tag]
            if used_mask.any():
                filtered[tag] = Dataset(np.asarray(dataset.query_points)[used_mask],
                                        np.asarray(dataset.observations)[used_mask])
            else:
                filtered[tag] = self._filtered.get(tag, dataset)
        self._filtered = dict(filtered)
        for tag, dataset in datasets.items():
            if not LocalizedTag.from_tag(tag).is_local:
                filtered[tag] = dataset
        return filtered

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
        num_local_models = Counter(
            LocalizedTag.from_tag(tag).global_tag for tag in models if LocalizedTag.from_tag(tag).is_local
        )
        num_local_models_vals = set(num_local_models.values())
        if len(num_local_models_vals) > 1:
            raise ValueError(f"The number of local models should be the same for all tags, got {num_local_models}")
        _num_local_models = sum(num_local_models_vals)
        num_subspaces = len(self._tags)
        if _num_local_models not in (0, num_subspaces):
            raise ValueError(
                f"When using local models, the number of subspaces {num_subspaces} should be equal to the number of "
                f"local models {_num_local_models}"
            )
        if self._rules is None and not (_num_local_models == 0 and isinstance(self._rule, EfficientGlobalOptimization)):
            self._rules = [copy.deepcopy(self._rule) for _ in self._tags]
        local_data = any(LocalizedTag.from_tag(tag).is_local for tag in (datasets or {}))
        if not (local_data or _num_local_models) or self._subspaces is None:
            self.update_subspaces(models, datasets)  # with local data, filter_datasets has updated the regions
        subspaces = self._subspaces
        if self._rules is not None:
            per_region = [
                (_global_tags(subspace.select_in_region(models)), _global_tags(subspace.select_in_region(datasets)))
                for subspace in subspaces
            ]
            if _num_local_models and isinstance(self._rule, EfficientGlobalOptimization) and not isinstance(
                self._rule._builder, GreedyAcquisitionFunctionBuilder
            ):
                points = self._acquire_local_ego(subspaces, per_region)
            else:
                points = np.stack([rule.acquire(subspace, m, d) for subspace, rule, (m, d)
                                   in zip(subspaces, self._rules, per_region)], axis=1)
        else:
            global_datasets = None if datasets is None else {
                tag: dataset for tag, dataset in datasets.items() if not LocalizedTag.from_tag(tag).is_local
            }
            points = self._rule.acquire(TaggedMultiSearchSpace(subspaces, self._tags), models, global_datasets)
        points = np.asarray(points).reshape(-1, len(subspaces), points.shape[-1])  # [q, S, D]
        return points.reshape(-1, points.shape[-1])

    def _acquire_local_ego(self, subspaces, per_region) -> np.ndarray:
        """EfficientGlobalOptimization.acquire of every region's copy (a builder that is not greedy), with the
        maximisation batched over the regions when their functions allow it (``_RegionStack``).  Returns [q, S, D]."""
        functions = []
        for rule, (models, datasets) in zip(self._rules, per_region):
            if rule._acquisition_function is None:
                rule._acquisition_function = rule._builder.prepare_acquisition_function(models, datasets=datasets)
            else:
                rule._acquisition_function = rule._builder.update_acquisition_function(
                    rule._acquisition_function, models, datasets=datasets
                )
            functions.append(rule._acquisition_function)
        k = self._rule._num_query_points
        stack = _RegionStack.of(functions, k)
        if stack is None:
            return np.stack([rule._optimizer(subspace, fn) for subspace, rule, fn in zip(subspaces, self._rules, functions)],
                            axis=1)
        S = len(subspaces)
        points = self._rule._base_optimizer(TaggedMultiSearchSpace(subspaces, self._tags), (stack, k * S))  # [k * S, D]
        return np.asarray(points).reshape(k, S, -1)


def _global_tags(mapping):
    """rule.py:1422-1432: a region's items under their global tags (single-model builders expect OBJECTIVE)."""
    if mapping is None:
        return None
    return {LocalizedTag.from_tag(tag).global_tag: item for tag, item in mapping.items()}


class _RegionStack:
    """S regions' acquisition functions as one function vectorised over V = k * S columns: column v is column v // S of
    region v % S's function, searched inside region v % S (the round robin of a ``TaggedMultiSearchSpace``).  Values and
    gradients call each region's function on its own columns.  ``maximize_from`` runs every region's multi-start L-BFGS in
    one device call: ``tb_acq_maximize_models`` for fused single-query functions (k = 1) on S distinct model handles,
    ``tb_rff_maximize_models`` for the negated trajectories of S distinct trajectory handles of k trajectories each."""

    def __init__(self, functions, k: int, kind: str):
        self._fns = list(functions)
        self._S = len(self._fns)
        self._k = k
        self._kind = kind

    @staticmethod
    def of(functions, k: int):
        """The stack of ``functions``, or None when some function cannot be maximised this way."""
        from .acquisition.function import _FusedSingleQuery

        if k == 1 and all(isinstance(f, _FusedSingleQuery)
                          and type(f)._native_maximize is _FusedSingleQuery._native_maximize for f in functions):
            handles = {f._model.handle.value for f in functions}
            if len(handles) == len(functions) and len({f._model.dtype for f in functions}) == 1:
                return _RegionStack(functions, k, "acq")
        if all(hasattr(f, "minimize_from") and hasattr(f, "maximize_from") for f in functions):
            if len({f._h.value for f in functions}) == len(functions):
                return _RegionStack(functions, k, "rff")
        return None

    def _columns(self, x, s):
        return x[..., s::self._S, :]

    def __call__(self, x):
        x = np.asarray(x)
        out = np.empty(x.shape[:-1])
        for s, f in enumerate(self._fns):
            out[..., s::self._S] = np.asarray(f(self._columns(x, s))).reshape(out[..., s::self._S].shape)
        return out

    def value_and_gradient(self, x):
        x = np.asarray(x)
        vals, grads = np.empty(x.shape[:-1]), np.empty(x.shape)
        for s, f in enumerate(self._fns):
            v, g = f.value_and_gradient(self._columns(x, s))
            vals[..., s::self._S] = np.asarray(v).reshape(vals[..., s::self._S].shape)
            grads[..., s::self._S, :] = np.asarray(g).reshape(grads[..., s::self._S, :].shape)
        return vals, grads

    def maximize_from(self, starts, lower, upper, *, maxcor: int = 10, maxiter: int = 15000, maxls: int = 20,
                      gtol: float = 1e-5, ftol: float = 2.220446049250313e-09):
        """starts [R, V, D] ([P, D] when V = 1), one box [D] or the regions' boxes [S, D] -> (success, maximised values,
        x, nfev) shaped like the starts without their last axis."""
        import ctypes as C

        from . import _lib

        x0 = np.asarray(starts, dtype=np.float64)
        flat = x0.ndim == 2
        if flat:
            x0 = x0[:, None, :]
        x0 = np.ascontiguousarray(x0)
        R, V, D = x0.shape
        S = self._S
        if V != self._k * S:
            raise ValueError(f"starts must have {self._k * S} columns, got {V}")
        lo, up = (np.ascontiguousarray(np.broadcast_to(np.atleast_2d(np.asarray(b, dtype=np.float64)), (S, D)))
                  for b in (lower, upper))
        x, f = np.empty((R, V, D)), np.empty((R, V))
        ok, nfev = np.zeros((R, V), dtype=np.int32), np.zeros((R, V), dtype=np.int64)
        tail = (int(maxcor), int(maxiter), int(maxls), float(gtol), float(ftol), x.ctypes.data, f.ctypes.data,
                ok.ctypes.data, nfev.ctypes.data)
        if self._kind == "acq":
            for fn in self._fns:
                fn._before_call()
                fn._model._check_dim(x0)
            handles = (C.c_void_p * S)(*[fn._model.handle.value for fn in self._fns])
            acq = np.array([fn._acq for fn in self._fns], dtype=np.int32)
            param = np.array([fn._param for fn in self._fns], dtype=np.float64)
            _lib.check(_lib.lib().tb_acq_maximize_models(handles, acq.ctypes.data, param.ctypes.data, S, lo.ctypes.data,
                                                         up.ctypes.data, x0.ctypes.data, R, *tail))
        else:
            for s, fn in enumerate(self._fns):
                fn._model._check_dim(x0)
                fn._batch(x0[:1, s::S])  # fixes the batch size k and draws the weights on first use
            handles = (C.c_void_p * S)(*[fn._h.value for fn in self._fns])
            _lib.check(_lib.lib().tb_rff_maximize_models(handles, S, lo.ctypes.data, up.ctypes.data, x0.ctypes.data, R,
                                                         *tail))
        if flat:
            return ok[:, 0].astype(bool), f[:, 0], x[:, 0, :], nfev[:, 0]
        return ok.astype(bool), f, x, nfev
