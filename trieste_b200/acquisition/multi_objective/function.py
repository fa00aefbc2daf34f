"""Expected hypervolume improvement (trieste acquisition/function/multi_objective.py:49-250) over a stack of native GPs.

The builder computes the reference point, the Pareto front of the posterior means at the data and its non-dominated
partition on the host, once per BO step.  Per candidate, each objective's posterior and the EHVI over all cells run on
the device (``tb_ehvi_*``, csrc/ehvi.cuh)."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from ... import _lib
from ...data import Dataset
from ...models import GaussianProcessRegression, ModelStack
from ..function import _check_populated, _FusedSingleQuery, _to_host
from ..interface import SingleModelAcquisitionBuilder
from .pareto import Pareto, get_reference_point
from .partition import prepare_default_non_dominated_partition_bounds


def _native_members(model) -> tuple:
    """The members of a stack the fused EHVI path runs on: native GPRs of one output each, distinct, on one device with
    one dtype and one input dimension."""
    if not isinstance(model, ModelStack):
        raise ValueError(f"ExpectedHypervolumeImprovement needs a trieste_b200.ModelStack of native models; received {model!r}")
    members = model.models
    if any(not isinstance(m, GaussianProcessRegression) for m in members):
        raise ValueError("ExpectedHypervolumeImprovement needs every stack member to be a trieste_b200.GaussianProcessRegression")
    if any(e != 1 for e in model.event_sizes):
        raise ValueError(f"ExpectedHypervolumeImprovement needs one output per stack member; got event sizes {model.event_sizes}")
    if len({id(m) for m in members}) != len(members):
        raise ValueError("the stack members must be distinct models")
    if len({m.device for m in members}) != 1 or len({m.dtype for m in members}) != 1:
        raise ValueError("the stack members must be on one device and have one dtype")
    if len({m.get_internal_data().query_points.shape[-1] for m in members}) != 1:
        raise ValueError("the stack members must have one input dimension")
    if not 2 <= len(members) <= 8:
        raise ValueError(f"ExpectedHypervolumeImprovement supports 2 to 8 objectives on the device; got {len(members)}")
    return members


class expected_hv_improvement(_FusedSingleQuery):
    """EHVI over the cells ``partition_bounds`` = (lower, upper) [K, L] of the non-dominated region, for a stack of L
    native one-output GPRs.  Shapes as the reference: ``x [..., 1, D] -> [..., 1]``.  The object owns a ``tb_ehvi`` and
    keeps the member models alive with it, so their handles outlive it."""

    def __init__(self, model, partition_bounds):
        self._members = _native_members(model)
        self._model = self._members[0]  # dtype and input checks of the shape handling
        self._param = 0.0
        h = C.c_void_p()
        handles = (C.c_void_p * len(self._members))(*[m.handle.value for m in self._members])
        _lib.check(_lib.lib().tb_ehvi_create(C.byref(h), handles, len(self._members)))
        self._h = h
        self.update(partition_bounds)

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            try:
                _lib.lib().tb_ehvi_destroy(h)
            except Exception:  # pragma: no cover
                pass
            self._h = None

    def update(self, partition_bounds) -> None:
        """New cells (lower, upper) [K, L]; the function object stays the same."""
        lower = np.ascontiguousarray(_to_host(partition_bounds[0]), dtype=np.float64)
        upper = np.ascontiguousarray(_to_host(partition_bounds[1]), dtype=np.float64)
        L = len(self._members)
        if lower.ndim != 2 or lower.shape != upper.shape or lower.shape[1] != L:
            raise ValueError(f"partition bounds must be two [K, {L}] arrays, got {lower.shape} and {upper.shape}")
        _lib.check(_lib.lib().tb_ehvi_set_cells(self._h, lower.ctypes.data, upper.ctypes.data, lower.shape[0]))
        self._lower, self._upper = lower, upper

    @property
    def partition_bounds(self):
        return self._lower, self._upper

    def _native_eval(self, px, M, po, pg) -> int:
        return _lib.lib().tb_ehvi_eval(self._h, px, M, po, pg)

    def _native_argmax(self, px, M, best, idx) -> int:
        return _lib.lib().tb_ehvi_argmax(self._h, px, M, None, best, idx)

    def _native_maximize(self, lo, up, x0, P, *args) -> int:
        return _lib.lib().tb_ehvi_maximize(self._h, lo, up, x0, P, *args)


class ExpectedHypervolumeImprovement(SingleModelAcquisitionBuilder):
    """multi_objective.py:49-142.  ``reference_point_spec``: a callable of the posterior means at the data [N, L]
    returning the reference point [L] (default :func:`get_reference_point`), or a fixed reference point."""

    def __init__(self, reference_point_spec=get_reference_point):
        if callable(reference_point_spec):
            self._ref_point_spec = reference_point_spec
        else:
            self._ref_point_spec = np.asarray(reference_point_spec, dtype=np.float64)
        self._ref_point = None

    def __repr__(self) -> str:
        if callable(self._ref_point_spec):
            return f"ExpectedHypervolumeImprovement({self._ref_point_spec.__name__})"
        return f"ExpectedHypervolumeImprovement({self._ref_point_spec!r})"

    def _partition_bounds(self, model, dataset: Optional[Dataset]):
        dataset = _check_populated(dataset)
        mean = np.asarray(_to_host(model.predict(dataset.query_points)[0]), dtype=np.float64)
        spec = self._ref_point_spec
        self._ref_point = np.asarray(spec(mean) if callable(spec) else spec, dtype=np.float64)
        front = Pareto(mean).front
        screened = front[np.all(front <= self._ref_point, axis=-1)]
        return prepare_default_non_dominated_partition_bounds(self._ref_point, screened)

    def prepare_acquisition_function(self, model, dataset: Optional[Dataset] = None):
        return expected_hv_improvement(model, self._partition_bounds(model, dataset))

    def update_acquisition_function(self, function, model, dataset: Optional[Dataset] = None):
        if not isinstance(function, expected_hv_improvement):
            raise ValueError(f"expected an expected_hv_improvement function, got {function!r}")
        function.update(self._partition_bounds(model, dataset))
        return function
