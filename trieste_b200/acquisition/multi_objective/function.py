"""Expected hypervolume improvement (trieste acquisition/function/multi_objective.py:49-250) over a stack of native GPs,
and HIPPO's greedy batches over it (:506-758).

The builder computes the reference point, the Pareto front of the posterior means at the data and its non-dominated
partition on the host, once per BO step.  Per candidate, each objective's posterior and the EHVI over all cells run on
the device (``tb_ehvi_*``, csrc/ehvi.cuh).  HIPPO's penalty around the pending points, in objective space, is evaluated in
the same kernel from the members' means, so the penalised function has EHVI's value, gradient, argmax and device L-BFGS
paths at O(P L) extra work per candidate for P pending points."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from ... import _lib
from ...data import Dataset
from ...models import GaussianProcessRegression, ModelStack
from ..function import _check_populated, _FusedSingleQuery, _to_host
from ..interface import OBJECTIVE, AcquisitionFunctionBuilder, GreedyAcquisitionFunctionBuilder, SingleModelAcquisitionBuilder
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

    def _before_call(self) -> None:
        # a hippo_penalized_ehvi may share the handle and have left its penalty there
        _lib.check(_lib.lib().tb_ehvi_set_penalty(self._h, None, None, 0))

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


def _check_objective_data(datasets, tag) -> None:
    """multi_objective.py:567-573 and :601-607"""
    if datasets is None or tag not in datasets or datasets[tag] is None:
        raise ValueError(f"{tag} dataset must be populated.")
    if len(datasets[tag]) == 0:
        raise ValueError(f"{tag} dataset must be populated.")


class hippo_penalizer:
    """multi_objective.py:664-758: the pending points p with their means mu_pl and variances v_pl from ``model.predict``
    (any model with ``predict``; fixed until :meth:`update`).  A candidate x with means mean_l(x) is penalised by
    ``prod_p (2/pi) atan(d_p(x))``, ``d_p(x) = sqrt(sum_l ((mean_l(x) - mu_pl) / sqrt(v_pl))^2)``: 0 at a pending point, towards
    1 far from all of them in objective space, independent of the candidate's variances.  :meth:`__call__` evaluates it from
    ``model.predict`` on the host; a :class:`hippo_penalized_ehvi` evaluates it on the device instead."""

    def __init__(self, model, pending_points):
        self._model = model
        self.update(pending_points)

    def update(self, pending_points) -> None:
        """multi_objective.py:712-725: new pending points, re-predicted with the model."""
        if pending_points is None or len(pending_points) == 0:
            raise ValueError("pending_points must not be None or empty")
        pts = np.asarray(_to_host(pending_points), dtype=np.float64)
        if pts.ndim != 2:
            raise ValueError(f"pending_points must have rank 2, got shape {pts.shape}")
        mean, var = self._model.predict(pts)
        mean = np.ascontiguousarray(_to_host(mean), dtype=np.float64)
        var = np.ascontiguousarray(_to_host(var), dtype=np.float64)
        if mean.ndim != 2 or mean.shape != var.shape or mean.shape[0] != pts.shape[0]:
            raise ValueError(f"the model's predict must return [P, L] means and variances, got {mean.shape} and {var.shape}")
        self._pending_points = pts
        self._pending_means = mean
        self._pending_vars = var

    def __call__(self, x):
        """x [N, 1, D] -> the penalty [N, 1]"""
        if len(getattr(x, "shape", ())) != 3 or x.shape[1] != 1:
            raise ValueError(f"This penalization function cannot be calculated for batches of points; got shape {tuple(x.shape)}")
        mean = np.asarray(_to_host(self._model.predict(x[:, 0, :])[0]), dtype=np.float64)
        z = (mean[:, None, :] - self._pending_means[None]) / np.sqrt(self._pending_vars)[None]  # [N, P, L]
        d = np.sqrt(np.sum(z * z, axis=-1))
        return np.prod((2.0 / np.pi) * np.arctan(d), axis=-1)[:, None]

    def _push(self, h) -> None:
        m = self._pending_means
        _lib.check(_lib.lib().tb_ehvi_set_penalty(h, m.ctypes.data, self._pending_vars.ctypes.data, m.shape[0]))


class hippo_penalized_ehvi(_FusedSingleQuery):
    """HIPPO's ``penalized_acquisition`` (multi_objective.py:637-647) over :class:`expected_hv_improvement`: the EHVI
    times the :class:`hippo_penalizer` penalty, evaluated in the EHVI kernel on the base function's ``tb_ehvi``.  The
    reference's ``exp(log EHVI + log pen)`` is computed as the product (the same value up to rounding); where that log form
    has a NaN gradient (EHVI 0, penalty 0, or x at a pending point, where the gradient of the norm is taken as 0) this
    returns the finite limit of the product rule.  The penalty is pushed to the handle before every launch, and the base
    function removes it before its own, so the two never see each other's state."""

    def __init__(self, base_acquisition_function, penalization):
        if type(base_acquisition_function) is not expected_hv_improvement:
            raise ValueError(f"HIPPO supports expected_hv_improvement base functions; received {base_acquisition_function!r}")
        if not isinstance(penalization, hippo_penalizer):
            raise ValueError(f"expected a hippo_penalizer, received {penalization!r}")
        self._base = base_acquisition_function
        self._penalization = penalization
        self._model = base_acquisition_function._model
        self._param = 0.0

    def _before_call(self) -> None:
        L = len(self._base._members)
        if self._penalization._pending_means.shape[1] != L:
            raise ValueError(f"the penaliser's model has {self._penalization._pending_means.shape[1]} outputs, the stack {L}")
        self._penalization._push(self._base._h)

    def _native_eval(self, px, M, po, pg) -> int:
        return self._base._native_eval(px, M, po, pg)

    def _native_argmax(self, px, M, best, idx) -> int:
        return self._base._native_argmax(px, M, best, idx)

    def _native_maximize(self, lo, up, x0, P, *args) -> int:
        return self._base._native_maximize(lo, up, x0, P, *args)


class HIPPO(GreedyAcquisitionFunctionBuilder):
    """multi_objective.py:506-661: greedy batches for multi-objective BO, each greedy step penalising the base function
    around the points already chosen, by their distance in objective space (:class:`hippo_penalizer`).  Without pending
    points the base function itself is returned; with them one penalised function, updated in place at later greedy steps
    and BO steps.  Supported base: :class:`ExpectedHypervolumeImprovement` (default), given as is or through ``.using``."""

    def __init__(self, objective_tag=OBJECTIVE, base_acquisition_function_builder=None):
        self._objective_tag = objective_tag
        base = base_acquisition_function_builder
        if base is None:
            base = ExpectedHypervolumeImprovement()
        if isinstance(base, SingleModelAcquisitionBuilder):
            if not isinstance(base, ExpectedHypervolumeImprovement):
                raise ValueError(f"HIPPO supports the ExpectedHypervolumeImprovement base builder; received {base!r}")
            base = base.using(objective_tag)
        elif not isinstance(base, AcquisitionFunctionBuilder):
            raise ValueError(f"HIPPO supports the ExpectedHypervolumeImprovement base builder; received {base!r}")
        self._base_builder = base
        self._base_acquisition_function: Optional[expected_hv_improvement] = None
        self._penalization: Optional[hippo_penalizer] = None
        self._penalized_acquisition: Optional[hippo_penalized_ehvi] = None

    def __repr__(self) -> str:
        return f"HIPPO({self._objective_tag!r}, {self._base_builder!r})"

    def prepare_acquisition_function(self, models, datasets=None, pending_points=None):
        """multi_objective.py:548-580."""
        _check_objective_data(datasets, self._objective_tag)
        acq = self._update_base_acquisition_function(models, datasets)
        if pending_points is not None and len(pending_points) != 0:
            acq = self._update_penalization(acq, models[self._objective_tag], pending_points)
        return acq

    def update_acquisition_function(self, function, models, datasets=None, pending_points=None,
                                    new_optimization_step: bool = True):
        """multi_objective.py:582-621."""
        _check_objective_data(datasets, self._objective_tag)
        if self._base_acquisition_function is None:
            raise ValueError("HIPPO: prepare_acquisition_function must be called before update_acquisition_function")
        if new_optimization_step:
            self._update_base_acquisition_function(models, datasets)
        if pending_points is None or len(pending_points) == 0:
            return self._base_acquisition_function
        return self._update_penalization(function, models[self._objective_tag], pending_points)

    def _update_penalization(self, function, model, pending_points):
        """multi_objective.py:623-649."""
        pts = np.asarray(_to_host(pending_points))
        if pts.ndim != 2:
            raise ValueError(f"pending_points must have rank 2, got shape {pts.shape}")
        if self._penalized_acquisition is not None:
            self._penalization.update(pts)
            return self._penalized_acquisition
        self._penalization = hippo_penalizer(model, pts)
        self._penalized_acquisition = hippo_penalized_ehvi(self._base_acquisition_function, self._penalization)
        return self._penalized_acquisition

    def _update_base_acquisition_function(self, models, datasets):
        """multi_objective.py:651-661."""
        if self._base_acquisition_function is None:
            fn = self._base_builder.prepare_acquisition_function(models, datasets)
        else:
            fn = self._base_builder.update_acquisition_function(self._base_acquisition_function, models, datasets)
        if type(fn) is not expected_hv_improvement:
            raise ValueError(f"HIPPO supports expected_hv_improvement base functions; the base builder returned {fn!r}")
        self._base_acquisition_function = fn
        return fn
