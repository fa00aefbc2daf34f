"""Minimal Bayesian-optimisation driver — the shape of ``BayesianOptimizer.optimize``
(trieste/bayesian_optimizer.py:570-883) for the single-model, single-objective case of the README example
(README.md:33-66): per step ``rule.acquire`` -> observer -> ``model.update`` / ``model.optimize``; and for mappings of
datasets and models keyed by tags, including the ``LocalizedTag`` local datasets and models of a ``BatchTrustRegionBox``
(bayesian_optimizer.py:676-840).  The reference's history records, checkpointing and TensorBoard logging are orchestration
and out of scope (SURVEY.md §2 row 17)."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, List, Mapping, Optional

import numpy as np

from .acquisition.interface import OBJECTIVE
from .data import Dataset
from .acquisition.utils import with_local_datasets
from .rule import EfficientGlobalOptimization
from .space import SearchSpace
from .utils import LocalizedTag, get_value_for_tag, ignoring_local_tags


@dataclass
class OptimizationResult:
    dataset: Dataset
    model: object
    history: List[np.ndarray] = field(default_factory=list)  # query points of every step
    error: Optional[BaseException] = None
    datasets: Optional[Mapping] = None  # every dataset and model by tag, when optimize was given mappings
    models: Optional[Mapping] = None

    def try_get_final_datasets(self) -> Mapping:
        """bayesian_optimizer.py:241-248: the final datasets by tag (local ones included)."""
        if self.error is not None:
            raise self.error
        return self.datasets if self.datasets is not None else {OBJECTIVE: self.dataset}

    def try_get_final_models(self) -> Mapping:
        """bayesian_optimizer.py:286-293: the final models by tag (local ones included)."""
        if self.error is not None:
            raise self.error
        return self.models if self.models is not None else {OBJECTIVE: self.model}

    def try_get_final_dataset(self) -> Dataset:
        if self.error is not None:
            raise self.error
        if self.datasets is not None:  # bayesian_optimizer.py:250-264: the single global dataset
            datasets = ignoring_local_tags(self.datasets)
            if len(datasets) != 1:
                raise ValueError(f"Expected a single dataset, found {len(datasets)}")
            return next(iter(datasets.values()))
        return self.dataset

    def try_get_optimal_point(self):
        """(query point, observation, index) of the best observation (bayesian_optimizer.py:260-280)."""
        ds = self.try_get_final_dataset()
        i = int(np.argmin(ds.observations[:, 0]))
        return ds.query_points[i], ds.observations[i], i


class BayesianOptimizer:
    def __init__(self, observer: Callable[[np.ndarray], np.ndarray], search_space: SearchSpace):
        self._observer = observer
        self._search_space = search_space

    def optimize(self, num_steps: int, dataset: Dataset, model, acquisition_rule=None) -> OptimizationResult:
        """``dataset`` and ``model``: one dataset and model (the objective's), or mappings of datasets and models by tag."""
        if num_steps < 0:
            raise ValueError(f"num_steps must be at least 0, got {num_steps}")
        if isinstance(dataset, Mapping) or isinstance(model, Mapping):
            return self._optimize_tagged(num_steps, dataset, model, acquisition_rule)
        rule = acquisition_rule if acquisition_rule is not None else EfficientGlobalOptimization()
        history: List[np.ndarray] = []
        try:  # the reference records the exception and returns the history so far (bayesian_optimizer.py:855-875)
            for _ in range(num_steps):
                query_points = rule.acquire(self._search_space, {OBJECTIVE: model}, {OBJECTIVE: dataset})
                observations = np.asarray(self._observer(query_points), dtype=np.float64).reshape(len(query_points), -1)
                dataset = dataset + Dataset(np.asarray(query_points, dtype=np.float64), observations)
                model.update(dataset)
                model.optimize(dataset)
                history.append(np.asarray(query_points))
        except Exception as e:  # noqa: BLE001
            return OptimizationResult(dataset, model, history, e)
        return OptimizationResult(dataset, model, history)

    def _optimize_tagged(self, num_steps: int, datasets, models, rule) -> OptimizationResult:
        """bayesian_optimizer.py:676-840 with mappings.  A rule with local datasets (``BatchTrustRegionBox``) gets them
        (``with_local_datasets``) at the first step and filters the datasets (``filter_datasets``) before every
        acquisition; region s's points (rows s, s + S, ... of the [q * S, D] batch) go to its local datasets and every
        point to the global ones.  Each model is updated with its own dataset, the local one when it has one."""
        if not isinstance(datasets, Mapping) or not isinstance(models, Mapping):
            raise ValueError("datasets and models must both be mappings by tag, or both a single dataset and model")
        datasets_keys = {LocalizedTag.from_tag(tag).global_tag for tag in datasets.keys()}
        models_keys = {LocalizedTag.from_tag(tag).global_tag for tag in models.keys()}
        if datasets_keys != models_keys:
            raise ValueError(
                f"datasets and models should contain the same keys. Got {datasets_keys} and {models_keys} respectively."
            )
        if not datasets:
            raise ValueError("dicts of datasets and models must be populated.")
        if rule is None:
            if datasets.keys() != {OBJECTIVE}:
                raise ValueError(
                    f"Default acquisition rule EfficientGlobalOptimization requires tag {OBJECTIVE!r}, got keys "
                    f"{datasets.keys()}"
                )
            rule = EfficientGlobalOptimization()
        # a rule with local datasets (the reference's LocalDatasetsAcquisitionRule), such as BatchTrustRegionBox
        regions = all(hasattr(type(rule), a) for a in ("num_local_datasets", "initialize_subspaces", "filter_datasets"))
        datasets, models = dict(datasets), dict(models)
        history: List[np.ndarray] = []

        def filtered():
            return rule.filter_datasets(models, datasets) if regions else datasets

        def fit(by_tag) -> None:
            for tag, model in models.items():
                _, ds = get_value_for_tag(by_tag, tag, LocalizedTag.from_tag(tag).global_tag)
                model.update(ds)
                model.optimize(ds)

        try:
            for step in range(1, num_steps + 1):
                if step == 1:
                    if regions:
                        rule.initialize_subspaces(self._search_space)
                        datasets = with_local_datasets(datasets, rule.num_local_datasets)
                    current = filtered()
                    fit(current)
                query_points = np.asarray(rule.acquire(self._search_space, models, current), dtype=np.float64)
                output = self._observer(query_points)
                if isinstance(output, Dataset):
                    output = {OBJECTIVE: output}
                elif not isinstance(output, Mapping):
                    observations = np.asarray(output, dtype=np.float64).reshape(len(query_points), -1)
                    output = {OBJECTIVE: Dataset(query_points, observations)}
                S = rule.num_local_datasets if regions else 0
                for tag, new in output.items():
                    datasets[tag] = datasets[tag] + new
                    for s in range(S):  # objectives/utils.py:78-104: region s's rows to its local dataset
                        ltag = LocalizedTag(tag, s)
                        if ltag in datasets and ltag not in output:
                            qp, obs = np.asarray(new.query_points), np.asarray(new.observations)
                            datasets[ltag] = datasets[ltag] + Dataset(qp[s::S], obs[s::S])
                current = filtered()
                for tag, model in models.items():
                    model.update(current[tag])
                    model.optimize(current[tag])
                history.append(query_points)
        except Exception as e:  # noqa: BLE001
            return self._tagged_result(datasets, models, history, e)
        return self._tagged_result(datasets, models, history, None)

    @staticmethod
    def _tagged_result(datasets, models, history, error) -> OptimizationResult:
        glob_ds, glob_m = ignoring_local_tags(datasets), ignoring_local_tags(models)
        dataset = next(iter(glob_ds.values())) if len(glob_ds) == 1 else None
        model = next(iter(glob_m.values())) if len(glob_m) == 1 else None
        return OptimizationResult(dataset, model, history, error, datasets=datasets, models=models)
