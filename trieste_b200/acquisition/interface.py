"""Acquisition-side protocol — mirrors trieste/acquisition/interface.py:27-157.

``AcquisitionFunction``: callable ``[..., B, D] -> [..., 1]``.  Builders keep the reference's
``prepare_acquisition_function`` / ``update_acquisition_function`` contract, including returning
the *same* function object from ``update`` (tests assert identity, test_function.py:196).
"""
from __future__ import annotations

import copy
from abc import ABC, abstractmethod
from typing import Callable, Generic, Mapping, Optional, TypeVar

from ..data import Dataset

Tag = str
OBJECTIVE: Tag = "OBJECTIVE"  # trieste/observer.py:42
AcquisitionFunction = Callable[..., object]
M_contra = TypeVar("M_contra")


class AcquisitionFunctionClass(ABC):
    """interface.py:41-49."""

    @abstractmethod
    def __call__(self, x):
        ...


class AcquisitionFunctionBuilder(Generic[M_contra], ABC):
    """interface.py:52-87."""

    @abstractmethod
    def prepare_acquisition_function(self, models: Mapping[Tag, M_contra], datasets: Optional[Mapping[Tag, Dataset]] = None):
        ...

    def update_acquisition_function(self, function, models, datasets=None):
        return self.prepare_acquisition_function(models, datasets=datasets)


class SingleModelAcquisitionBuilder(Generic[M_contra], ABC):
    """interface.py:90-157 — ``using(tag)`` adapts to the multi-model builder interface."""

    def using(self, tag: Tag) -> AcquisitionFunctionBuilder:
        single = self

        class _Anon(AcquisitionFunctionBuilder):
            def prepare_acquisition_function(self, models, datasets=None):
                return single.prepare_acquisition_function(models[tag], dataset=None if datasets is None else datasets[tag])

            def update_acquisition_function(self, function, models, datasets=None):
                return single.update_acquisition_function(function, models[tag], dataset=None if datasets is None else datasets[tag])

            def __repr__(self) -> str:
                return f"{single!r} using tag {tag!r}"

            def __deepcopy__(self, memo):  # a copy wraps a copy of the builder and its state (one per trust region)
                return copy.deepcopy(single, memo).using(tag)

        return _Anon()

    @abstractmethod
    def prepare_acquisition_function(self, model: M_contra, dataset: Optional[Dataset] = None):
        ...

    def update_acquisition_function(self, function, model: M_contra, dataset: Optional[Dataset] = None):
        return self.prepare_acquisition_function(model, dataset=dataset)


class GreedyAcquisitionFunctionBuilder(Generic[M_contra], ABC):
    """interface.py:160-214: builds a function for greedily collected batches; ``pending_points`` [M, D] are the
    points already chosen for the current batch (``None`` on the first call of a step)."""

    @abstractmethod
    def prepare_acquisition_function(self, models: Mapping[Tag, M_contra], datasets: Optional[Mapping[Tag, Dataset]] = None,
                                     pending_points=None):
        ...

    def update_acquisition_function(self, function, models, datasets=None, pending_points=None,
                                    new_optimization_step: bool = True):
        return self.prepare_acquisition_function(models, datasets=datasets, pending_points=pending_points)


class SingleModelGreedyAcquisitionBuilder(Generic[M_contra], ABC):
    """interface.py:217-308."""

    def using(self, tag: Tag) -> GreedyAcquisitionFunctionBuilder:
        single = self

        class _Anon(GreedyAcquisitionFunctionBuilder):
            def prepare_acquisition_function(self, models, datasets=None, pending_points=None):
                return single.prepare_acquisition_function(
                    models[tag], dataset=None if datasets is None else datasets[tag], pending_points=pending_points)

            def update_acquisition_function(self, function, models, datasets=None, pending_points=None,
                                            new_optimization_step: bool = True):
                return single.update_acquisition_function(
                    function, models[tag], dataset=None if datasets is None else datasets[tag],
                    pending_points=pending_points, new_optimization_step=new_optimization_step)

            def __repr__(self) -> str:
                return f"{single!r} using tag {tag!r}"

            def __deepcopy__(self, memo):  # a copy wraps a copy of the builder and its state (one per trust region)
                return copy.deepcopy(single, memo).using(tag)

        return _Anon()

    @abstractmethod
    def prepare_acquisition_function(self, model: M_contra, dataset: Optional[Dataset] = None, pending_points=None):
        ...

    def update_acquisition_function(self, function, model: M_contra, dataset: Optional[Dataset] = None, pending_points=None,
                                    new_optimization_step: bool = True):
        return self.prepare_acquisition_function(model, dataset=dataset, pending_points=pending_points)


class VectorizedAcquisitionFunctionBuilder(AcquisitionFunctionBuilder[M_contra]):
    """interface.py:311-316: functions that return one value per query point of the batch, ``[..., B, D] -> [..., B]``."""


class SingleModelVectorizedAcquisitionBuilder(SingleModelAcquisitionBuilder[M_contra]):
    """interface.py:319-363."""

    def using(self, tag: Tag) -> AcquisitionFunctionBuilder:
        single = self

        class _Anon(VectorizedAcquisitionFunctionBuilder):
            def prepare_acquisition_function(self, models, datasets=None):
                return single.prepare_acquisition_function(models[tag], dataset=None if datasets is None else datasets[tag])

            def update_acquisition_function(self, function, models, datasets=None):
                return single.update_acquisition_function(function, models[tag], dataset=None if datasets is None else datasets[tag])

            def __repr__(self) -> str:
                return f"{single!r} using tag {tag!r}"

            def __deepcopy__(self, memo):  # a copy wraps a copy of the builder and its state (one per trust region)
                return copy.deepcopy(single, memo).using(tag)

        return _Anon()
