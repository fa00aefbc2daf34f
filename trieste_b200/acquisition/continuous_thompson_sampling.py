"""Continuous Thompson sampling — mirrors trieste/acquisition/function/continuous_thompson_sampling.py
(``GreedyContinuousThompsonSampling`` :33-111, ``ParallelContinuousThompsonSampling`` :114-186,
``negate_trajectory_function`` :196-250).

Each builder returns the negative of trajectories sampled from the model, so that the acquisition optimisers (maximisers)
return the trajectories' minimisers.  With the default ``select_output`` the negated trajectory also offers
``value_and_gradient`` (one paired CUDA launch per call: point (n, b) under trajectory b only) and ``maximize_from``
(the multi-start L-BFGS of every trajectory on the device, ``tb_rff_maximize``), so the continuous optimiser never leaves
the GPU between iterations; its cost grows linearly in the batch size B, with no q x q joint algebra.
"""
from __future__ import annotations

import functools
import inspect
from typing import Callable, Optional

from ..data import Dataset
from .interface import SingleModelGreedyAcquisitionBuilder, SingleModelVectorizedAcquisitionBuilder
from .utils import select_nth_output


def _require_trajectory_sampler(model) -> None:
    if not hasattr(model, "trajectory_sampler"):
        raise ValueError(
            f"Thompson sampling from trajectory only supports models with a trajectory_sampler method; received {model!r}"
        )


class GreedyContinuousThompsonSampling(SingleModelGreedyAcquisitionBuilder):
    """continuous_thompson_sampling.py:33-111: one negated trajectory per greedy step, resampled between the steps of a
    batch and rebuilt from the updated model at each new optimisation step."""

    def __init__(self, select_output: Callable = select_nth_output):
        self._select_output = select_output

    def __repr__(self) -> str:
        return f"GreedyContinuousThompsonSampling({self._select_output!r})"

    def prepare_acquisition_function(self, model, dataset: Optional[Dataset] = None, pending_points=None):
        _require_trajectory_sampler(model)
        self._trajectory_sampler = model.trajectory_sampler()
        function = self._trajectory_sampler.get_trajectory()
        return negate_trajectory_function(function, self._select_output)

    def update_acquisition_function(self, function, model, dataset: Optional[Dataset] = None, pending_points=None,
                                    new_optimization_step: bool = True):
        if new_optimization_step:  # update the sampler and resample the trajectory
            new_function = self._trajectory_sampler.update_trajectory(function)
        else:  # only resample the trajectory
            new_function = self._trajectory_sampler.resample_trajectory(function)
        if new_function is not function:
            function = negate_trajectory_function(new_function, self._select_output)
        return function


class ParallelContinuousThompsonSampling(SingleModelVectorizedAcquisitionBuilder):
    """continuous_thompson_sampling.py:114-186: B negated trajectories, one per batch element, maximised independently
    (``batchify_vectorize``)."""

    def __init__(self, select_output: Callable = select_nth_output):
        self._select_output = select_output

    def __repr__(self) -> str:
        return f"ParallelContinuousThompsonSampling({self._select_output!r})"

    def prepare_acquisition_function(self, model, dataset: Optional[Dataset] = None):
        _require_trajectory_sampler(model)
        self._trajectory_sampler = model.trajectory_sampler()
        self._trajectory = self._trajectory_sampler.get_trajectory()
        self._negated_trajectory = negate_trajectory_function(self._trajectory, self._select_output)
        return self._negated_trajectory

    def update_acquisition_function(self, function, model, dataset: Optional[Dataset] = None):
        if function is not self._negated_trajectory:
            raise ValueError("Wrong trajectory function passed into update_acquisition_function")
        new_function = self._trajectory_sampler.update_trajectory(self._trajectory)
        if new_function is not self._trajectory:  # negate again when not updated in place
            self._trajectory = new_function
            self._negated_trajectory = negate_trajectory_function(new_function, self._select_output)
        return self._negated_trajectory


class _Unavailable:
    """A method the negated trajectory does not offer: ``hasattr`` is False, so the optimisers take their generic routes."""

    def __get__(self, obj, objtype=None):
        raise AttributeError("only the negated trajectory with the default select_output offers this method")


def negate_trajectory_function(function, select_output: Optional[Callable] = None, function_type=None):
    """continuous_thompson_sampling.py:196-250: ``-1 * select_output(function(x))``.  A trajectory object keeps its
    methods (``update``, ``resample``): its class is swapped in place for a subclass named ``NegatedTrajectory``; a plain
    function is wrapped.  With ``select_output=select_nth_output`` the negated object also negates ``value_and_gradient``
    ([N, B, D] -> ([N, B], [N, B, D])) and offers ``maximize_from`` (device L-BFGS, starts [R, B, D], or [P, D] when
    B = 1) and, for B = 1, ``fused_argmax`` over a candidate set; a custom ``select_output`` gets ``__call__`` only."""
    if inspect.isfunction(function) or inspect.ismethod(function) or isinstance(function, functools.partial):

        def negated_trajectory(x):
            if select_output is not None:
                return -1.0 * select_output(function(x))
            return -1.0 * function(x)

        return negated_trajectory

    base = function_type or type(function)
    native = select_output is select_nth_output and hasattr(base, "minimize_from")

    class NegatedTrajectory(base):  # type: ignore[misc, valid-type]
        def __call__(self, x):
            if select_output is not None:
                return -1.0 * select_output(super().__call__(x))
            return -1.0 * super().__call__(x)

        if native:

            def value_and_gradient(self, x):
                """x [N, B, D] -> (-f_b [N, B], -grad f_b [N, B, D])."""
                vals, grads = super().value_and_gradient(x)
                return -1.0 * vals[..., 0], -1.0 * grads

            def maximize_from(self, starts, lower, upper, **options):
                """Maximise -f_b from starts [R, B, D] ([P, D] for B = 1) on the device; returns (success, -f_b, x,
                nfev) shaped like the starts without their last axis."""
                flat = getattr(starts, "ndim", 0) == 2
                if flat:
                    starts = starts[:, None, :]
                ok, f, x, nfev = self.minimize_from(starts, lower, upper, **options)
                if flat:
                    return ok[:, 0], -1.0 * f[:, 0], x[:, 0, :], nfev[:, 0]
                return ok, -1.0 * f, x, nfev

            def fused_argmax(self, points):
                """points [M, D] -> (first index of the largest -f, that value), for a trajectory of batch size 1."""
                if self._initialized and self._batch_size != 1:
                    raise ValueError(f"fused_argmax needs a trajectory of batch size 1, got {self._batch_size}")
                mv, mi = self.argmin_over(points)
                return int(mi[0]), -1.0 * float(mv[0])

        else:
            value_and_gradient = _Unavailable()
            maximize_from = _Unavailable()
            fused_argmax = _Unavailable()

    function.__class__ = NegatedTrajectory
    return function
