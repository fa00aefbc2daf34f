"""Analytic and Monte-Carlo single-objective acquisition functions of the hot path — mirrors
trieste/acquisition/function/function.py (EI :96-223, LCB :328-418, batch MC-EI :1074-1186, batch EI :1189-1805).

Each callable keeps the reference's shape contract (``x: [..., 1, D] -> [..., 1]``; batch
functions ``[..., B, D] -> [..., 1]``) but evaluates predict + tail in ONE pass of fused GPU
kernels behind the C-ABI instead of ``model.predict`` followed by separate elementwise ops.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from .. import _lib
from ..data import Dataset
from ..models import GaussianProcessRegression, _flatten_leading, _ptr
from .interface import (AcquisitionFunctionClass, SingleModelAcquisitionBuilder, SingleModelGreedyAcquisitionBuilder,
                        SingleModelVectorizedAcquisitionBuilder)

JITTER = 1e-6  # trieste/utils/misc.py:183


def _check_populated(dataset: Optional[Dataset]) -> Dataset:
    if dataset is None:
        raise ValueError("Dataset must be populated.")
    if len(dataset) == 0:
        raise ValueError("Dataset must be populated.")
    return dataset


def _to_host(x) -> np.ndarray:
    return x.detach().cpu().numpy() if hasattr(x, "detach") else np.asarray(x)


def _require_native(model) -> GaussianProcessRegression:
    if not isinstance(model, GaussianProcessRegression):
        raise ValueError(
            f"trieste_b200 acquisition functions need a trieste_b200.GaussianProcessRegression model; received {model!r}"
        )
    return model


class _FusedSingleQuery(AcquisitionFunctionClass):
    """Common machinery: squeeze the B=1 axis, run the fused kernel chain, restore shapes."""

    _acq: int = -1

    def __init__(self, model: GaussianProcessRegression, param: float):
        self._model = _require_native(model)
        self._param = float(param)

    def _before_call(self) -> None:
        """state that lives in the native handle and must be current before a launch (none by default)"""

    # the native calls behind the shape handling below; a function over several handles overrides all three
    def _native_eval(self, px, M, po, pg) -> int:
        return _lib.lib().tb_acq_eval(self._model.handle, self._acq, self._param, px, M, po, pg)

    def _native_argmax(self, px, M, best, idx) -> int:
        return _lib.lib().tb_acq_argmax(self._model.handle, self._acq, self._param, px, M, None, best, idx)

    def _native_maximize(self, lo, up, x0, P, *args) -> int:
        return _lib.lib().tb_acq_maximize(self._model.handle, self._acq, self._param, lo, up, x0, P, *args)

    def _squeeze(self, x):
        self._before_call()
        x, _ = _lib.as_contiguous(x, self._model.dtype)
        if x.ndim < 2 or x.shape[-2] != 1:
            raise ValueError(
                f"This acquisition function only supports batch sizes of one; got input of shape {tuple(x.shape)}"
            )
        self._model._check_dim(x)
        return _flatten_leading(x.reshape(tuple(x.shape[:-2]) + (x.shape[-1],)), 1)

    def __call__(self, x):
        flat, lead = self._squeeze(x)
        M = flat.shape[0]
        out, po = _lib.empty_like_kind(flat, (M, 1), self._model.dtype)
        _lib.check(self._native_eval(_ptr(flat), M, po, None))
        return out.reshape(lead + (1,))

    def value_and_gradient(self, x):
        """``tfp.math.value_and_gradient(fn, x)`` as used at acquisition/optimizer.py:621-629:
        returns (values [..., 1], d values / d x [..., 1, D])."""
        flat, lead = self._squeeze(x)
        M, D = flat.shape
        out, po = _lib.empty_like_kind(flat, (M, 1), self._model.dtype)
        grad, pg = _lib.empty_like_kind(flat, (M, D), self._model.dtype)
        _lib.check(self._native_eval(_ptr(flat), M, po, pg))
        return out.reshape(lead + (1,)), grad.reshape(lead + (1, D))

    def maximize_from(self, starts, lower, upper, *, maxcor: int = 10, maxiter: int = 15000, maxls: int = 20,
                      gtol: float = 1e-5, ftol: float = 2.220446049250313e-09):
        """Device-side multi-start projected L-BFGS (``tb_acq_maximize``): every row of ``starts`` [P, D] is an
        independent local maximisation inside the box — the work of ``_perform_parallel_continuous_optimization`` and its
        SciPy greenlets (optimizer.py:566-745) without leaving the GPU between iterations.
        Returns (success [P] bool, values [P], x [P, D], nfev [P]); fp64 like the reference's SciPy side."""
        self._before_call()
        x0 = np.ascontiguousarray(_to_host(starts), dtype=np.float64)
        if x0.ndim != 2:
            raise ValueError(f"starts must be [P, D], got {x0.shape}")
        self._model._check_dim(x0)
        P, D = x0.shape
        lo = np.ascontiguousarray(np.broadcast_to(np.asarray(lower, dtype=np.float64), (D,)))
        up = np.ascontiguousarray(np.broadcast_to(np.asarray(upper, dtype=np.float64), (D,)))
        x = np.empty((P, D))
        f = np.empty(P)
        ok = np.zeros(P, dtype=np.int32)
        nfev = np.zeros(P, dtype=np.int64)
        _lib.check(
            self._native_maximize(
                lo.ctypes.data, up.ctypes.data, x0.ctypes.data, P, int(maxcor), int(maxiter), int(maxls), float(gtol),
                float(ftol), x.ctypes.data, f.ctypes.data, ok.ctypes.data, nfev.ctypes.data,
            )
        )
        return ok.astype(bool), f, x, nfev

    def fused_argmax(self, points):
        """points [M, D] -> (first-max index, value) without writing the M values to HBM
        (generate_random_search_optimizer / _get_max_discrete_points, optimizer.py:124-150)."""
        self._before_call()
        pts, _ = _lib.as_contiguous(points, self._model.dtype)
        if pts.ndim != 2:
            raise ValueError(f"points must be [M, D], got {tuple(pts.shape)}")
        self._model._check_dim(pts)
        best = C.c_double() if self._model.dtype == np.float64 else C.c_float()
        idx = C.c_int64()
        _lib.check(self._native_argmax(_ptr(pts), pts.shape[0], C.byref(best), C.byref(idx)))
        return int(idx.value), float(best.value)


class expected_improvement(_FusedSingleQuery):
    """function.py:190-223: ``(eta - mean) * cdf(eta) + variance * pdf(eta)``."""

    _acq = _lib.ACQ_EI

    def __init__(self, model, eta):
        super().__init__(model, float(np.asarray(eta).reshape(-1)[0]))

    def update(self, eta) -> None:
        self._param = float(np.asarray(eta).reshape(-1)[0])

    @property
    def eta(self) -> float:
        return self._param


class log_expected_improvement(expected_improvement):
    """log of :class:`expected_improvement`.  ABSENT in the reference at this commit (SURVEY.md §8 a8);
    defined here (numerically stable for z << 0); parity unpinned."""

    _acq = _lib.ACQ_LOG_EI


class augmented_expected_improvement(expected_improvement):
    """function.py:283-325: EI times ``1 - sqrt(noise) / sqrt(noise + variance)`` (Huang et al. 2006); the noise
    variance is the model's likelihood variance, read from the native handle on every call (the reference re-assigns it
    in ``update``, :306-309)."""

    _acq = _lib.ACQ_AEI


class min_value_entropy_search(_FusedSingleQuery):
    """entropy.py:166-213: information gain about the objective minimum y* from evaluating at x, averaged over samples
    of y* (Wang & Jegelka 2017, adapted for minimisation).  The samples are pushed to the native handle before every
    launch (two functions may share one model)."""

    _acq = _lib.ACQ_MES

    def __init__(self, model, samples):
        super().__init__(model, 0.0)
        self.update(samples)

    def update(self, samples) -> None:
        s = np.asarray(samples, dtype=np.float64)
        if s.ndim != 2:
            raise ValueError(f"samples must have rank two, got shape {s.shape}")
        if s.shape[0] == 0:
            raise ValueError("samples must not be empty")
        self._samples = np.ascontiguousarray(s.reshape(-1))

    @property
    def samples(self) -> np.ndarray:
        return self._samples[:, None]

    def _before_call(self) -> None:
        _push_min_value_samples(self._model, self._samples)


def _push_min_value_samples(model: GaussianProcessRegression, samples: np.ndarray) -> None:
    _lib.check(
        _lib.lib().tb_acq_set_min_value_samples(model.handle, samples.ctypes.data_as(C.POINTER(C.c_double)), int(samples.size))
    )


class _lcb(_FusedSingleQuery):
    def __init__(self, model, beta: float, negate: bool):
        if beta < 0:
            raise ValueError("Standard deviation scaling parameter beta must not be negative")
        super().__init__(model, beta)
        self._acq = _lib.ACQ_NEG_LCB if negate else _lib.ACQ_LCB


def lower_confidence_bound(model, beta: float):
    """function.py:389-418: ``mean - beta * sqrt(variance)``."""
    return _lcb(model, beta, negate=False)


def _eta_from_model(model, dataset: Dataset, search_space=None) -> float:
    """function.py:133-149: eta = min over the FEASIBLE training inputs of the posterior mean; with a constrained search
    space only the query points that satisfy the constraints count, and if none does eta = max of the mean."""
    _require_native(model)
    mean, _ = model.predict(np.asarray(dataset.query_points))
    mean = np.asarray(_to_host(mean))
    if search_space is not None and getattr(search_space, "has_constraints", False):
        feasible = np.asarray(search_space.is_feasible(np.asarray(dataset.query_points)), dtype=bool).reshape(-1)
        if not feasible.any():
            return float(np.max(mean, axis=0)[0])
        mean = mean[feasible]
    return float(np.min(mean, axis=0)[0])


class probability_below_threshold(_FusedSingleQuery):
    """function.py:481-513: ``Normal(mean, sqrt(var)).cdf(threshold)``."""

    _acq = _lib.ACQ_PBT

    def __init__(self, model, threshold):
        if np.ndim(threshold) != 0 and np.size(threshold) != 1:
            raise ValueError("threshold must be a scalar")
        super().__init__(model, float(np.asarray(threshold).reshape(-1)[0]))

    def update(self, threshold) -> None:
        self._param = float(np.asarray(threshold).reshape(-1)[0])


class ProbabilityOfImprovement(SingleModelAcquisitionBuilder):
    """function.py:47-93: probability of improving on eta = min posterior mean at the observed points."""

    def __repr__(self) -> str:
        return "ProbabilityOfImprovement()"

    def prepare_acquisition_function(self, model, dataset: Optional[Dataset] = None):
        dataset = _check_populated(dataset)
        return probability_below_threshold(model, _eta_from_model(model, dataset))

    def update_acquisition_function(self, function, model, dataset: Optional[Dataset] = None):
        dataset = _check_populated(dataset)
        if not isinstance(function, probability_below_threshold):
            raise ValueError(f"expected a probability_below_threshold function, got {function!r}")
        function.update(_eta_from_model(model, dataset))
        return function


class ProbabilityOfFeasibility(SingleModelAcquisitionBuilder):
    """function.py:421-478: probability that the constraint model is below ``threshold``."""

    def __init__(self, threshold: float):
        if np.ndim(threshold) != 0:
            raise ValueError("threshold must be a scalar")
        self._threshold = float(threshold)

    def __repr__(self) -> str:
        return f"ProbabilityOfFeasibility({self._threshold!r})"

    @property
    def threshold(self) -> float:
        return self._threshold

    def prepare_acquisition_function(self, model, dataset: Optional[Dataset] = None):
        return probability_below_threshold(model, self._threshold)

    def update_acquisition_function(self, function, model, dataset: Optional[Dataset] = None):
        return function  # no need to update anything (function.py:470-478)


class ExpectedImprovement(SingleModelAcquisitionBuilder):
    """function.py:96-187."""

    _fn_class = expected_improvement

    def __init__(self, search_space=None):
        self._search_space = search_space

    def __repr__(self) -> str:
        return f"{type(self).__name__}({self._search_space!r})"

    def prepare_acquisition_function(self, model, dataset: Optional[Dataset] = None):
        dataset = _check_populated(dataset)
        return self._fn_class(model, _eta_from_model(model, dataset, self._search_space))

    def update_acquisition_function(self, function, model, dataset: Optional[Dataset] = None):
        dataset = _check_populated(dataset)
        if not isinstance(function, self._fn_class):
            raise ValueError(f"expected a {self._fn_class.__name__} function, got {function!r}")
        function.update(_eta_from_model(model, dataset, self._search_space))  # same object: no re-build
        return function


class LogExpectedImprovement(ExpectedImprovement):
    _fn_class = log_expected_improvement


class MinValueEntropySearch(SingleModelAcquisitionBuilder):
    """entropy.py:52-164.  The min-value samples come from ``min_value_sampler`` evaluated on the data plus
    ``grid_size`` random points of the search space (:134-137).  Default as in the reference (:111):
    ``ExactThompsonSampler(sample_min_value=True)`` — joint samples over all N + grid_size points, drawn on the device
    (``tb_gp_sample_joint``); above its 16384-point limit the :class:`GumbelSampler` takes over.  Any sampler with
    ``sample_min_value=True`` can be passed (``GumbelSampler``, ``ThompsonSamplerFromTrajectory``)."""

    def __init__(self, search_space, num_samples: int = 5, grid_size: int = 1000, min_value_sampler=None, seed=None):
        if num_samples <= 0:
            raise ValueError(f"num_samples must be positive, got {num_samples}")
        if grid_size <= 0:
            raise ValueError(f"grid_size must be positive, got {grid_size}")
        if min_value_sampler is not None:
            if not min_value_sampler.sample_min_value:
                raise ValueError(
                    "Minvalue Entropy Search requires a min_value_sampler that samples minimum values, "
                    "however the passed sampler has sample_min_value=False."
                )
        self._seed = seed
        self._draws = 0
        self._min_value_sampler = min_value_sampler  # None: chosen per draw (see _draw)
        self._search_space = search_space
        self._num_samples = num_samples
        self._grid_size = grid_size

    def __repr__(self) -> str:
        return (f"MinValueEntropySearch({self._search_space!r}, {self._num_samples!r}, {self._grid_size!r}, "
                f"{self._min_value_sampler!r})")

    MAX_EXACT_POINTS = 16384  # tb_gp_sample_joint's limit on the jointly sampled point set

    def _draw(self, model, dataset: Dataset) -> np.ndarray:
        grid = np.asarray(self._search_space.sample(self._grid_size))
        query_points = np.concatenate([np.asarray(dataset.query_points, dtype=grid.dtype), grid], axis=0)
        sampler = self._min_value_sampler
        # a seeded builder is reproducible: draw k of the builder uses seed + k for the samplers that take a per-call seed
        draw_seed = None if self._seed is None else int(self._seed) + self._draws
        self._draws += 1
        if sampler is None:
            # entropy.py:111: the reference default is ExactThompsonSampler(sample_min_value=True) — joint samples over the
            # data and the grid; beyond the device path's point limit the Gumbel sampler (marginals only) takes over
            from .sampler import ExactThompsonSampler, GumbelSampler

            if query_points.shape[0] <= self.MAX_EXACT_POINTS:
                return ExactThompsonSampler(sample_min_value=True).sample(model, self._num_samples, query_points, seed=draw_seed)
            sampler = GumbelSampler(sample_min_value=True, seed=draw_seed)
        return sampler.sample(model, self._num_samples, query_points)

    def prepare_acquisition_function(self, model, dataset: Optional[Dataset] = None):
        dataset = _check_populated(dataset)
        return min_value_entropy_search(model, self._draw(model, dataset))

    def update_acquisition_function(self, function, model, dataset: Optional[Dataset] = None):
        dataset = _check_populated(dataset)
        if not isinstance(function, min_value_entropy_search):
            raise ValueError(f"expected a min_value_entropy_search function, got {function!r}")
        function.update(self._draw(model, dataset))
        return function


class gibbon_quality_term(_FusedSingleQuery):
    """entropy.py:439-500: the information each single point gives about the objective minimum y*,
    ``-1/2 mean_s log(1 + rho^2 r_s (gamma_s - r_s))`` with ``rho^2 = var / (var + noise)`` and gamma, r as for MES.  The
    samples (rank two, non-empty) are pushed to the native handle before every launch."""

    _acq = _lib.ACQ_GIBBON_QUALITY

    def __init__(self, model, samples):
        super().__init__(model, 0.0)
        self.update(samples)

    def update(self, samples) -> None:
        s = np.asarray(_to_host(samples), dtype=np.float64)
        if s.ndim != 2:
            raise ValueError(f"samples must have rank two, got shape {s.shape}")
        if s.shape[0] == 0:
            raise ValueError("samples must not be empty")
        self._samples = np.ascontiguousarray(s.reshape(-1))

    @property
    def samples(self) -> np.ndarray:
        return self._samples[:, None]

    def _before_call(self) -> None:
        _push_min_value_samples(self._model, self._samples)


class gibbon_repulsion_term(_FusedSingleQuery):
    """entropy.py:503-618: ``w/2 (log V_det - log yvar)``, the log-determinant gain of adding x to the m pending points,
    ``V_det = yvar - c(x)^T (B + noise I)^-1 c(x)`` with c the posterior covariance between x and the pending points and B
    theirs; ``w = (1/m)^2`` with ``rescaled_repulsion``, else 1.  The device derives K^-1 k(X, P) and the Cholesky factor of
    B + noise I once per pending set and posterior; the pending points are pushed before every launch."""

    _acq = _lib.ACQ_GIBBON_REPULSION

    def __init__(self, model, pending_points, rescaled_repulsion: bool = True):
        super().__init__(model, 0.0)
        self._rescaled_repulsion = bool(rescaled_repulsion)
        self.update(pending_points)

    def update(self, pending_points, lipschitz_constant=None, eta=None) -> None:
        """entropy.py:594-601: only the pending points change; the other arguments are those of the penalisation protocol."""
        p = np.asarray(_to_host(pending_points), dtype=np.float64)
        if p.ndim != 2:
            raise ValueError(f"pending_points must have rank 2, got shape {p.shape}")
        if p.shape[0] == 0:
            raise ValueError("pending_points must not be empty")
        self._model._check_dim(p)
        self._pending = np.ascontiguousarray(p)

    @property
    def pending_points(self) -> np.ndarray:
        return self._pending

    @property
    def weight(self) -> float:
        return (1.0 / self._pending.shape[0]) ** 2 if self._rescaled_repulsion else 1.0

    def _before_call(self) -> None:
        _lib.check(
            _lib.lib().tb_acq_set_gibbon_repulsion(
                self._model.handle, self._pending.ctypes.data, int(self._pending.shape[0]), float(self.weight)
            )
        )


class GibbonAcquisition(_FusedSingleQuery):
    """entropy.py:422-436: ``diversity_term(x) + quality_term(x)``, both evaluated in the same fused launch."""

    _acq = _lib.ACQ_GIBBON

    def __init__(self, quality_term: gibbon_quality_term, diversity_term: gibbon_repulsion_term):
        if not isinstance(quality_term, gibbon_quality_term) or not isinstance(diversity_term, gibbon_repulsion_term):
            raise ValueError("GibbonAcquisition needs a gibbon_quality_term and a gibbon_repulsion_term")
        if quality_term._model is not diversity_term._model:
            raise ValueError("the quality and repulsion terms of GibbonAcquisition must share one model")
        super().__init__(quality_term._model, 0.0)
        self._quality_term = quality_term
        self._diversity_term = diversity_term

    def _before_call(self) -> None:
        self._quality_term._before_call()
        self._diversity_term._before_call()


class GIBBON(SingleModelGreedyAcquisitionBuilder):
    """entropy.py:236-419: greedy batches by GIBBON (Moss et al. 2021), modified for minimisation.  The min-value samples
    are drawn as :class:`MinValueEntropySearch` draws them (its ``_draw``: exact Thompson sampling over the data and
    ``grid_size`` search-space points by default, Gumbel above the exact sampler's point limit); ``seed`` makes the draws
    reproducible.  Without pending points the builder returns the quality term, otherwise one :class:`GibbonAcquisition`
    object that is updated in place at every later greedy step."""

    def __init__(self, search_space, num_samples: int = 5, grid_size: int = 1000, min_value_sampler=None,
                 rescaled_repulsion: bool = True, seed=None):
        if min_value_sampler is not None and not min_value_sampler.sample_min_value:
            raise ValueError(
                "GIBBON requires a min_value_sampler that samples minimum values, however the passed sampler has "
                "sample_min_value=False."
            )
        # validates num_samples and grid_size, and owns the draws
        self._min_value_draws = MinValueEntropySearch(search_space, num_samples, grid_size, min_value_sampler, seed=seed)
        self._search_space = search_space
        self._num_samples = num_samples
        self._grid_size = grid_size
        self._min_value_sampler = min_value_sampler
        self._rescaled_repulsion = bool(rescaled_repulsion)
        self._min_value_samples: Optional[np.ndarray] = None
        self._quality_term: Optional[gibbon_quality_term] = None
        self._diversity_term: Optional[gibbon_repulsion_term] = None
        self._gibbon_acquisition: Optional[GibbonAcquisition] = None

    def __repr__(self) -> str:
        return (f"GIBBON({self._search_space!r}, {self._num_samples!r}, {self._grid_size!r}, {self._min_value_sampler!r}, "
                f"{self._rescaled_repulsion!r})")

    def prepare_acquisition_function(self, model, dataset: Optional[Dataset] = None, pending_points=None):
        """entropy.py:315-341."""
        _require_native(model)
        dataset = _check_populated(dataset)
        acq = self._update_quality_term(dataset, model)
        if pending_points is not None and len(pending_points) != 0:
            acq = self._update_repulsion_term(acq, dataset, model, pending_points)
        return acq

    def update_acquisition_function(self, function, model, dataset: Optional[Dataset] = None, pending_points=None,
                                    new_optimization_step: bool = True):
        """entropy.py:343-374: new samples at a new optimisation step; the quality term alone without pending points."""
        dataset = _check_populated(dataset)
        if self._quality_term is None:
            raise ValueError("GIBBON: prepare_acquisition_function must be called before update_acquisition_function")
        if new_optimization_step:
            self._update_quality_term(dataset, model)
        if pending_points is None:
            return self._quality_term
        return self._update_repulsion_term(function, dataset, model, pending_points)

    def _update_repulsion_term(self, function, dataset: Dataset, model, pending_points):
        """entropy.py:376-401: the same GibbonAcquisition object once it exists."""
        pts = np.asarray(_to_host(pending_points))
        if pts.ndim != 2:
            raise ValueError(f"pending_points must have rank 2, got shape {pts.shape}")
        if self._gibbon_acquisition is not None and isinstance(self._diversity_term, gibbon_repulsion_term):
            self._diversity_term.update(pts)
            return self._gibbon_acquisition
        self._diversity_term = gibbon_repulsion_term(model, pts, rescaled_repulsion=self._rescaled_repulsion)
        self._gibbon_acquisition = GibbonAcquisition(self._quality_term, self._diversity_term)
        return self._gibbon_acquisition

    def _update_quality_term(self, dataset: Dataset, model):
        """entropy.py:403-419."""
        _require_native(model)
        dataset = _check_populated(dataset)
        self._min_value_samples = self._min_value_draws._draw(model, dataset)
        if self._quality_term is not None:
            self._quality_term.update(self._min_value_samples)
        else:
            self._quality_term = gibbon_quality_term(model, self._min_value_samples)
        return self._quality_term


class AugmentedExpectedImprovement(ExpectedImprovement):
    """function.py:225-280: eta = min posterior mean at the data, as for EI."""

    _fn_class = augmented_expected_improvement

    def __init__(self):
        super().__init__(None)

    def __repr__(self) -> str:
        return "AugmentedExpectedImprovement()"


class NegativeLowerConfidenceBound(SingleModelAcquisitionBuilder):
    """function.py:328-372: negated LCB so that maximisation minimises the bound."""

    def __init__(self, beta: float = 1.96):
        if beta < 0:
            raise ValueError(f"Confidence parameter's standard deviation scaling must not be negative, got {beta}")
        self._beta = beta

    def __repr__(self) -> str:
        return f"NegativeLowerConfidenceBound({self._beta!r})"

    def prepare_acquisition_function(self, model, dataset: Optional[Dataset] = None):
        return _lcb(model, self._beta, negate=True)

    def update_acquisition_function(self, function, model, dataset: Optional[Dataset] = None):
        return function  # no dependence on data (function.py:361-372)


class MakePositive(SingleModelAcquisitionBuilder):
    """function.py:1914-1990: ``log(1 + exp(f))`` of the base builder's function f, so that every value is positive (as
    local penalisation needs of its base function).  Over a fused single-query function it runs on the device as a
    one-term reduction (acquisition/combination.py), with ``value_and_gradient``, ``fused_argmax`` and ``maximize_from``;
    over any other function with ``value_and_gradient`` the gradient is sigmoid(f) times the base gradient."""

    def __init__(self, base_acquisition_function_builder: SingleModelAcquisitionBuilder) -> None:
        self._base_builder = base_acquisition_function_builder

    def __repr__(self) -> str:
        return f"MakePositive({self._base_builder})"

    def _wrap(self):
        from .combination import REDUCE_SOFTPLUS, _softplus, reduce_functions

        return reduce_functions(REDUCE_SOFTPLUS, lambda inputs: _softplus(inputs[0]), (self._base_function,))

    def prepare_acquisition_function(self, model, dataset: Optional[Dataset] = None):
        self._base_function = self._base_builder.prepare_acquisition_function(model, dataset)
        return self._wrap()

    def update_acquisition_function(self, function, model, dataset: Optional[Dataset] = None):
        """function.py:1967-1990: the same function when the base builder updated its function in place."""
        up_fn = self._base_builder.update_acquisition_function(self._base_function, model, dataset)
        if up_fn is self._base_function:
            return function
        self._base_function = up_fn
        return self._wrap()


class multiple_optimism_lower_confidence_bound(AcquisitionFunctionClass):
    """function.py:1857-1911 (MOLCB, Torossian et al. 2020): a VECTORISED function ``[..., B, D] -> [..., B]``; column b is
    the negated lower confidence bound ``-mean + beta_b sqrt(var)`` with ``beta_b = 5 d Phi^-1(0.5 + 0.5 b / (B + 1))``, b = 1..B,
    fixed at the first call (a later call with another batch size is an error, as in the reference).  Each column runs the
    fused predict + NegLCB kernels with its own beta (value and gradient), so ``batchify_vectorize`` optimises the B
    columns independently."""

    def __init__(self, model, search_space_dim: int):
        if search_space_dim <= 0:
            raise ValueError(f"search_space_dim must be positive, got {search_space_dim}")
        self._model = _require_native(model)
        self._search_space_dim = int(search_space_dim)
        self._betas: Optional[np.ndarray] = None  # [B], lazily initialised
        self._columns = []

    @property
    def betas(self) -> Optional[np.ndarray]:
        return self._betas

    def _prepare(self, x):
        if len(x.shape) < 2:
            raise ValueError(f"expected [..., B, D] query batches, got shape {tuple(x.shape)}")
        B = int(x.shape[-2])
        if B <= 0:
            raise ValueError("batch size must be positive")
        if self._betas is None:
            from statistics import NormalDist

            spread = 0.5 + 0.5 * np.arange(1, B + 1, dtype=np.float64) / (B + 1.0)
            self._betas = 5.0 * self._search_space_dim * np.array([NormalDist().inv_cdf(p) for p in spread])
            self._columns = [_lcb(self._model, float(b), negate=True) for b in self._betas]
        elif B != self._betas.shape[0]:
            raise ValueError(
                f"{type(self).__name__} requires a fixed batch size. Got batch size {B} but previous batch size was "
                f"{self._betas.shape[0]}."
            )
        return B

    def __call__(self, x):
        x = x if hasattr(x, "shape") else np.asarray(x)
        B = self._prepare(x)
        cols = [_to_host(self._columns[b](x[..., b : b + 1, :])) for b in range(B)]  # each [..., 1]
        return np.concatenate(cols, axis=-1)

    def value_and_gradient(self, x):
        """[..., B, D] -> (values [..., B], gradients [..., B, D]); column b only depends on x[..., b, :]."""
        x = x if hasattr(x, "shape") else np.asarray(x)
        B = self._prepare(x)
        vals, grads = [], []
        for b in range(B):
            v, g = self._columns[b].value_and_gradient(x[..., b : b + 1, :])
            vals.append(_to_host(v))
            grads.append(_to_host(g))
        return np.concatenate(vals, axis=-1), np.concatenate(grads, axis=-2)


class MultipleOptimismNegativeLowerConfidenceBound(SingleModelVectorizedAcquisitionBuilder):
    """function.py:1808-1854: builder of :class:`multiple_optimism_lower_confidence_bound`; nothing to update between
    steps."""

    def __init__(self, search_space):
        self._search_space = search_space

    def __repr__(self) -> str:
        return f"MultipleOptimismNegativeLowerConfidenceBound({self._search_space!r})"

    def prepare_acquisition_function(self, model, dataset: Optional[Dataset] = None):
        return multiple_optimism_lower_confidence_bound(model, self._search_space.dimension)

    def update_acquisition_function(self, function, model, dataset: Optional[Dataset] = None):
        if not isinstance(function, multiple_optimism_lower_confidence_bound):
            raise ValueError(f"expected a multiple_optimism_lower_confidence_bound function, got {function!r}")
        return function  # nothing to update


class batch_monte_carlo_expected_improvement(AcquisitionFunctionClass):
    """function.py:1150-1186: mean over S reparametrised joint samples of
    ``max(eta - min_q sample, 0)``."""

    def __init__(self, sample_size: int, model, eta, jitter: float):
        if not hasattr(model, "reparam_sampler"):
            raise ValueError(
                "The batch Monte-Carlo expected improvement acquisition function only supports models that "
                f"implement a reparam_sampler method; received {model!r}"
            )
        self._sample_size = sample_size
        self._model = _require_native(model)
        self._sampler = model.reparam_sampler(sample_size)
        self._eta = float(np.asarray(eta).reshape(-1)[0])
        self._jitter = jitter

    def update(self, eta) -> None:
        self._eta = float(np.asarray(eta).reshape(-1)[0])
        self._sampler.reset_sampler()

    def __call__(self, x):
        x, _ = _lib.as_contiguous(x, self._model.dtype)
        if x.ndim < 2:
            raise ValueError(f"expected [..., B, D] query batches, got shape {tuple(x.shape)}")
        self._model._check_dim(x)
        flat, lead = _flatten_leading(x, 2)
        nb, q = flat.shape[0], flat.shape[1]
        eps = np.ascontiguousarray(self._sampler._get_eps(q), dtype=self._model.dtype)  # [q, S] host, fixed until reset
        out, po = _lib.empty_like_kind(flat, (nb, 1), self._model.dtype)
        _lib.check(
            _lib.lib().tb_acq_batch_mc_ei(
                self._model.handle, _ptr(flat), nb, q, eps.ctypes.data, eps.shape[1], self._eta, self._jitter, po
            )
        )
        return out.reshape(lead + (1,))

    def value_and_gradient(self, x):
        """[..., B, D] -> (values [..., 1], d values / d x [..., B, D]): the reverse pass TensorFlow's autodiff performs
        when the reference maximises this function over ``space ** B`` (batchify_joint, optimizer.py:897-936)."""
        x, _ = _lib.as_contiguous(x, self._model.dtype)
        if x.ndim < 2:
            raise ValueError(f"expected [..., B, D] query batches, got shape {tuple(x.shape)}")
        self._model._check_dim(x)
        flat, lead = _flatten_leading(x, 2)
        nb, q, D = flat.shape
        eps = np.ascontiguousarray(self._sampler._get_eps(q), dtype=self._model.dtype)
        out, po = _lib.empty_like_kind(flat, (nb, 1), self._model.dtype)
        grad, pg = _lib.empty_like_kind(flat, (nb, q, D), self._model.dtype)
        _lib.check(
            _lib.lib().tb_acq_batch_mc_ei_grad(
                self._model.handle, _ptr(flat), nb, q, eps.ctypes.data, eps.shape[1], self._eta, self._jitter, po, pg
            )
        )
        return out.reshape(lead + (1,)), grad.reshape(lead + (q, D))


class monte_carlo_expected_improvement(batch_monte_carlo_expected_improvement):
    """function.py:883-920: ``mean_S max(eta - f_s(x), 0)`` over reparametrised samples, batch size one.  For a GPR the
    reference's ``model.reparam_sampler`` is the batch sampler (models.py:325-331), so this is the q = 1 case of the
    batch kernel chain."""

    def __call__(self, x):
        x_arr = x if hasattr(x, "shape") else np.asarray(x)
        if len(x_arr.shape) < 2 or x_arr.shape[-2] != 1:
            raise ValueError(
                f"This acquisition function only supports batch sizes of one; got input of shape {tuple(x_arr.shape)}"
            )
        return super().__call__(x)


class MonteCarloExpectedImprovement(SingleModelAcquisitionBuilder):
    """function.py:782-880: eta = min over the data of the sample mean at each training input."""

    def __init__(self, sample_size: int, *, jitter: float = JITTER):
        if sample_size <= 0:
            raise ValueError(f"sample_size must be positive, got {sample_size}")
        if jitter < 0:
            raise ValueError(f"jitter must be non-negative, got {jitter}")
        self._sample_size = sample_size
        self._jitter = jitter

    def __repr__(self) -> str:
        return f"MonteCarloExpectedImprovement({self._sample_size!r}, jitter={self._jitter!r})"

    def _eta(self, sampler, dataset: Dataset):
        x = np.asarray(dataset.query_points)
        samples = sampler.sample(x[..., None, :], jitter=self._jitter)  # [N, S, 1, 1]
        return np.min(np.mean(samples, axis=-3), axis=0)

    def prepare_acquisition_function(self, model, dataset: Optional[Dataset] = None):
        if not hasattr(model, "reparam_sampler"):
            raise ValueError(
                f"MonteCarloExpectedImprovement only supports models with a reparam_sampler method; received {model!r}"
            )
        dataset = _check_populated(dataset)
        fn = monte_carlo_expected_improvement(self._sample_size, model, 0.0, self._jitter)
        fn._eta = float(np.asarray(self._eta(fn._sampler, dataset)).reshape(-1)[0])
        return fn

    def update_acquisition_function(self, function, model, dataset: Optional[Dataset] = None):
        dataset = _check_populated(dataset)
        if not isinstance(function, monte_carlo_expected_improvement):
            raise ValueError(f"expected a monte_carlo_expected_improvement, got {function!r}")
        function._sampler.reset_sampler()
        function._eta = float(np.asarray(self._eta(function._sampler, dataset)).reshape(-1)[0])
        return function


class BatchMonteCarloExpectedImprovement(SingleModelAcquisitionBuilder):
    """function.py:1074-1147."""

    def __init__(self, sample_size: int, *, jitter: float = JITTER):
        if sample_size <= 0:
            raise ValueError(f"sample_size must be positive, got {sample_size}")
        if jitter < 0:
            raise ValueError(f"jitter must be non-negative, got {jitter}")
        self._sample_size = sample_size
        self._jitter = jitter

    def __repr__(self) -> str:
        return f"BatchMonteCarloExpectedImprovement({self._sample_size!r}, jitter={self._jitter!r})"

    def prepare_acquisition_function(self, model, dataset: Optional[Dataset] = None):
        dataset = _check_populated(dataset)
        mean, _ = model.predict(np.asarray(dataset.query_points))
        if mean.shape[-1] != 1:
            raise ValueError("Expected model with event shape [1].")
        eta = np.min(mean, axis=0)
        return batch_monte_carlo_expected_improvement(self._sample_size, model, eta, self._jitter)

    def update_acquisition_function(self, function, model, dataset: Optional[Dataset] = None):
        dataset = _check_populated(dataset)
        if not isinstance(function, batch_monte_carlo_expected_improvement):
            raise ValueError(f"expected a batch_monte_carlo_expected_improvement, got {function!r}")
        mean, _ = model.predict(np.asarray(dataset.query_points))
        function.update(np.min(mean, axis=0))
        return function


class batch_expected_improvement(AcquisitionFunctionClass):
    """function.py:1281-1805: the multi-point EI of Chevalier & Ginsbourger, its multivariate-normal CDFs by Genz's QMC
    recursion over ``sample_size`` Sobol points, evaluated on the device (``tb_acq_batch_ei``).  As in the reference, the
    points and the batch size q are fixed by the first call: ``update`` draws a new skip but changes only ``eta``, and
    a call with another q — or with q = 1, where the reference's dimension-(q-1) CDF cannot be built — raises."""

    def __init__(self, sample_size: int, model, eta, jitter: float, seed: Optional[int] = None):
        self._sample_size = int(sample_size)
        self._jitter = jitter  # validated and kept, never used (the reference hard-codes 1e-6, :1776-1783)
        self._model = _require_native(model)
        self._eta = float(np.asarray(eta).reshape(-1)[0])
        self._rng = np.random.default_rng(seed)
        self._num_sobol_skip = self._draw_skip()
        self._q: Optional[int] = None
        self._w: Optional[np.ndarray] = None  # [q-1, S], drawn at the first call

    def _draw_skip(self) -> int:
        return int(np.floor(1e9 * self._rng.random(dtype=np.float32)))  # :1306, :1313

    def update(self, eta) -> None:
        self._eta = float(np.asarray(eta).reshape(-1)[0])
        self._num_sobol_skip = self._draw_skip()

    @property
    def eta(self) -> float:
        return self._eta

    def _prepare(self, x):
        x, _ = _lib.as_contiguous(x, self._model.dtype)
        if x.ndim < 2:
            raise ValueError(f"expected [..., B, D] query batches, got shape {tuple(x.shape)}")
        self._model._check_dim(x)
        flat, lead = _flatten_leading(x, 2)
        q = flat.shape[1]
        if self._q is None:
            self._q = q
        if q != self._q:
            raise ValueError(f"batch_expected_improvement was first called with batch size {self._q}; got {q}")
        if q < 2:
            raise ValueError("batch_expected_improvement needs a batch size of at least 2 (its CDFs have dimension q - 1)")
        if self._w is None:
            from ..sampler import sobol_points

            self._w = np.ascontiguousarray(sobol_points(self._sample_size, q - 1, self._num_sobol_skip).T)
        return flat, lead

    def __call__(self, x):
        flat, lead = self._prepare(x)
        nb, q = flat.shape[0], flat.shape[1]
        out, po = _lib.empty_like_kind(flat, (nb, 1), self._model.dtype)
        _lib.check(_lib.lib().tb_acq_batch_ei(self._model.handle, _ptr(flat), nb, q, self._w.ctypes.data,
                                              self._sample_size, self._eta, po))
        return out.reshape(lead + (1,))

    def value_and_gradient(self, x):
        """[..., B, D] -> (values [..., 1], d values / d x [..., B, D]), the reverse pass of ``__call__``."""
        flat, lead = self._prepare(x)
        nb, q, D = flat.shape
        out, po = _lib.empty_like_kind(flat, (nb, 1), self._model.dtype)
        grad, pg = _lib.empty_like_kind(flat, (nb, q, D), self._model.dtype)
        _lib.check(_lib.lib().tb_acq_batch_ei_grad(self._model.handle, _ptr(flat), nb, q, self._w.ctypes.data,
                                                   self._sample_size, self._eta, po, pg))
        return out.reshape(lead + (1,)), grad.reshape(lead + (q, D))


class BatchExpectedImprovement(SingleModelAcquisitionBuilder):
    """function.py:1189-1278: eta = min over the data of the posterior mean.  ``seed`` makes the Sobol skip draws
    reproducible."""

    def __init__(self, sample_size: int, *, jitter: float = JITTER, seed: Optional[int] = None):
        if sample_size <= 0:
            raise ValueError(f"sample_size must be positive, got {sample_size}")
        if jitter < 0:
            raise ValueError(f"jitter must be non-negative, got {jitter}")
        self._sample_size = sample_size
        self._jitter = jitter
        self._seed = seed

    def __repr__(self) -> str:
        return f"BatchExpectedImprovement({self._sample_size!r}, jitter={self._jitter!r})"

    @staticmethod
    def _eta(model, dataset: Optional[Dataset]) -> float:
        dataset = _check_populated(dataset)
        mean, _ = model.predict(np.asarray(dataset.query_points))
        if mean.shape[-1] != 1:
            raise ValueError("Expected model with event shape [1].")
        return float(np.min(mean, axis=0)[0])

    def prepare_acquisition_function(self, model, dataset: Optional[Dataset] = None):
        return batch_expected_improvement(self._sample_size, model, self._eta(model, dataset), self._jitter, seed=self._seed)

    def update_acquisition_function(self, function, model, dataset: Optional[Dataset] = None):
        eta = self._eta(model, dataset)
        if not isinstance(function, batch_expected_improvement):
            raise ValueError(f"expected a batch_expected_improvement function, got {function!r}")
        function.update(eta)
        return function
