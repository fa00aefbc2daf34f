"""Greedy batch builders, mirrors trieste/acquisition/function/greedy_batch.py.

``LocalPenalization`` (:54-247) and its penalisers (:250-388): each greedy step multiplies the single-point acquisition
function by a penalty around the points already chosen for the batch (Gonzalez et al. 2016; Alvi et al. 2019).  The
penalty is evaluated in the fused acquisition tail on the device (``TB_ACQ_PENALIZED``), so the penalised function has
the base function's value, gradient, argmax and device L-BFGS paths, at O(P D) extra work per candidate for P pending
points; nothing is appended to the model or refactorised between greedy steps.

``Fantasizer`` — greedy batches with any single-point acquisition function, :415-607 (builder) and :630-770
(``_fantasized_model``).

Every time a point of the batch has been chosen, its observation is "fantasised" (kriging believer: the model mean;
"sample": a posterior sample) and the model is conditioned on it.  For an exact GPR that conditional posterior IS the
posterior of the same GPR with the pending points appended to its data (Chevalier et al. 2014, eqs. 8-10; the reference
evaluates it through ``conditional_predict_*``, models/gpflow/models.py:355-525).  The device-resident form therefore keeps a
second device-resident model whose posterior cache is the base model's cache EXTENDED by the pending rows
(``tb_gp_append_data``, O(m N^2) per greedy step instead of conditioning every prediction on the host), so the fantasised
model runs the same fused predict + acquisition kernels — including the device-side multi-start optimiser — as the base
model."""
from __future__ import annotations

from typing import Mapping, Optional

import numpy as np

from .. import _lib
from ..data import Dataset
from ..models import GaussianProcessRegression, GPRSpec
from .function import (
    ExpectedImprovement,
    MinValueEntropySearch,
    _check_populated,
    _FusedSingleQuery,
    _require_native,
    _to_host,
    expected_improvement,
    min_value_entropy_search,
)
from .interface import (
    OBJECTIVE,
    AcquisitionFunctionBuilder,
    GreedyAcquisitionFunctionBuilder,
    SingleModelAcquisitionBuilder,
    SingleModelGreedyAcquisitionBuilder,
    Tag,
)


class local_penalizer:
    """greedy_batch.py:272-312: the pending points x_j with ``radius_j = (mean(x_j) - eta) / L`` and
    ``scale_j = sqrt(var(x_j)) / L`` from ``model.predict`` (variance clipped at 1e-12).  The state is pushed to the model's
    native handle before every launch of a :class:`PenalizedAcquisition`, which evaluates the penalty on the device."""

    _kind: int = 0

    def __init__(self, model, pending_points, lipschitz_constant, eta):
        self._model = _require_native(model)
        self.update(pending_points, lipschitz_constant, eta)

    def update(self, pending_points, lipschitz_constant, eta) -> None:
        """greedy_batch.py:302-312."""
        pts = np.asarray(_to_host(pending_points), dtype=np.float64)
        if pts.ndim != 2:
            raise ValueError(f"pending_points must have rank 2, got shape {pts.shape}")
        if pts.shape[0] == 0:
            raise ValueError("pending_points must not be empty")
        self._model._check_dim(pts)
        mean, var = self._model.predict(pts)
        mean = np.asarray(_to_host(mean), dtype=np.float64)[:, 0]
        var = np.asarray(_to_host(var), dtype=np.float64)[:, 0]
        L = float(np.asarray(lipschitz_constant).reshape(-1)[0])
        eta = float(np.asarray(eta).reshape(-1)[0])
        self._pending_points = np.ascontiguousarray(pts)
        self._radius = np.ascontiguousarray((mean - eta) / L)
        self._scale = np.ascontiguousarray(np.sqrt(var) / L)

    @property
    def pending_points(self) -> np.ndarray:
        return self._pending_points

    @property
    def radius(self) -> np.ndarray:
        return self._radius

    @property
    def scale(self) -> np.ndarray:
        return self._scale

    def _push(self) -> None:
        _lib.check(
            _lib.lib().tb_acq_set_penalization(
                self._model.handle, self._kind, self._pending_points.ctypes.data, int(self._pending_points.shape[0]),
                self._radius.ctypes.data, self._scale.ctypes.data,
            )
        )


class soft_local_penalizer(local_penalizer):
    """greedy_batch.py:315-354 (Gonzalez et al. 2016): ``prod_j Phi((||x - x_j|| - radius_j) / scale_j)``."""

    _kind = _lib.PEN_SOFT


class hard_local_penalizer(local_penalizer):
    """greedy_batch.py:357-388 (Alvi et al. 2019): ``prod_j ((||x - x_j|| / (radius_j + scale_j))^-5 + 1)^(-1/5)``."""

    _kind = _lib.PEN_HARD


class PenalizedAcquisition(_FusedSingleQuery):
    """greedy_batch.py:250-269: ``exp(log base(x) + log penalty(x))``, evaluated as the base value times the penalty in
    the fused tail (NaN where the base value is negative, as the logarithm gives).  Gradients follow the product rule
    ``pen grad(base) + base grad(pen)``.  Where the reference's log-space form has a NaN gradient (base value 0, penalty 0,
    or x at a pending point, where the gradient of the norm is undefined and taken as 0) this returns the finite limit of
    the product rule instead.  The base function's handle state and the penalty are pushed before every launch, so other
    functions on the same model are not disturbed."""

    def __init__(self, base_acquisition_function, penalization):
        if type(base_acquisition_function) not in (expected_improvement, min_value_entropy_search):
            raise ValueError(
                "PenalizedAcquisition supports expected_improvement and min_value_entropy_search base functions; "
                f"received {base_acquisition_function!r}"
            )
        if not isinstance(penalization, local_penalizer):
            raise ValueError(
                "PenalizedAcquisition supports soft_local_penalizer and hard_local_penalizer penalties; "
                f"received {penalization!r}"
            )
        super().__init__(base_acquisition_function._model, base_acquisition_function._param)
        self._base_acquisition_function = base_acquisition_function
        self._penalization = penalization
        self._acq = base_acquisition_function._acq | _lib.ACQ_PENALIZED

    def _before_call(self) -> None:
        base = self._base_acquisition_function
        self._param = base._param  # the base builder may have updated eta in place
        base._before_call()
        self._penalization._push()


_PENALIZERS = (soft_local_penalizer, hard_local_penalizer)


class LocalPenalization(SingleModelGreedyAcquisitionBuilder):
    """greedy_batch.py:54-247.  The Lipschitz constant ``L = max ||grad mean||`` and ``eta = min mean`` over
    ``num_samples`` search-space samples plus the data's query points are estimated at every new optimisation step
    (``L = 10`` for a flat model, L < 1e-5) and kept between the greedy steps of one batch.  The gradient of the mean comes
    from :meth:`GaussianProcessRegression.mean_gradient`, without the variance machinery.

    Supported: base builders :class:`ExpectedImprovement` (default) and :class:`MinValueEntropySearch`; penalisers
    :class:`soft_local_penalizer` (default) and :class:`hard_local_penalizer`."""

    def __init__(self, search_space, num_samples: int = 500, penalizer=None, base_acquisition_function_builder=None):
        if num_samples <= 0:
            raise ValueError(f"num_samples must be positive, got {num_samples}")
        penalizer = soft_local_penalizer if penalizer is None else penalizer
        if penalizer not in _PENALIZERS:
            raise ValueError(f"penalizer must be soft_local_penalizer or hard_local_penalizer, got {penalizer!r}")
        if base_acquisition_function_builder is None:
            base_acquisition_function_builder = ExpectedImprovement()
        if type(base_acquisition_function_builder) not in (ExpectedImprovement, MinValueEntropySearch):
            raise ValueError(
                "LocalPenalization supports the ExpectedImprovement and MinValueEntropySearch base builders; "
                f"received {base_acquisition_function_builder!r}"
            )
        self._search_space = search_space
        self._num_samples = int(num_samples)
        self._lipschitz_penalizer = penalizer
        self._base_builder = base_acquisition_function_builder
        self._lipschitz_constant: Optional[float] = None
        self._eta: Optional[float] = None
        self._base_acquisition_function = None
        self._penalization: Optional[local_penalizer] = None
        self._penalized_acquisition: Optional[PenalizedAcquisition] = None

    def __repr__(self) -> str:
        return (f"LocalPenalization({self._search_space!r}, {self._num_samples!r}, {self._lipschitz_penalizer.__name__}, "
                f"{self._base_builder!r})")

    @property
    def lipschitz_constant(self) -> Optional[float]:
        return self._lipschitz_constant

    @property
    def eta(self) -> Optional[float]:
        return self._eta

    def prepare_acquisition_function(self, model, dataset: Optional[Dataset] = None, pending_points=None):
        """greedy_batch.py:125-147."""
        dataset = _check_populated(dataset)
        acq = self._update_base_acquisition_function(dataset, model)
        if pending_points is not None and len(pending_points) != 0:
            acq = self._update_penalization(acq, dataset, model, pending_points)
        return acq

    def update_acquisition_function(self, function, model, dataset: Optional[Dataset] = None, pending_points=None,
                                    new_optimization_step: bool = True):
        """greedy_batch.py:149-181: the same penalised object is returned at every greedy step."""
        dataset = _check_populated(dataset)
        if self._base_acquisition_function is None:
            raise ValueError("LocalPenalization: prepare_acquisition_function must be called before update_acquisition_function")
        if new_optimization_step:
            self._update_base_acquisition_function(dataset, model)
        if pending_points is None or len(pending_points) == 0:
            return self._base_acquisition_function
        return self._update_penalization(function, dataset, model, pending_points)

    def _update_penalization(self, function, dataset: Dataset, model, pending_points):
        """greedy_batch.py:183-204."""
        pts = np.asarray(_to_host(pending_points))
        if pts.ndim != 2:
            raise ValueError(f"pending_points must have rank 2, got shape {pts.shape}")
        if self._penalized_acquisition is not None:
            self._penalization.update(pts, self._lipschitz_constant, self._eta)
            return self._penalized_acquisition
        self._penalization = self._lipschitz_penalizer(model, pts, self._lipschitz_constant, self._eta)
        self._penalized_acquisition = PenalizedAcquisition(self._base_acquisition_function, self._penalization)
        return self._penalized_acquisition

    def _get_lipschitz_estimate(self, model, sampled_points):
        """greedy_batch.py:206-217: (max ||grad mean||_2, min mean) over the points."""
        mean, grad = model.mean_gradient(sampled_points)
        mean = np.asarray(_to_host(mean), dtype=np.float64)
        grad = np.asarray(_to_host(grad), dtype=np.float64)
        return float(np.max(np.linalg.norm(grad, axis=1))), float(np.min(mean))

    def _update_base_acquisition_function(self, dataset: Dataset, model):
        """greedy_batch.py:219-247."""
        model = _require_native(model)
        samples = np.asarray(self._search_space.sample(self._num_samples))
        query_points = np.asarray(dataset.query_points)
        samples = np.concatenate([query_points, samples.astype(query_points.dtype, copy=False)], axis=0)
        lipschitz_constant, eta = self._get_lipschitz_estimate(model, samples)
        if lipschitz_constant < 1e-5:  # :224-225, numerical stability for 'flat' models
            lipschitz_constant = 10.0
        self._lipschitz_constant = lipschitz_constant
        self._eta = eta
        if self._base_acquisition_function is not None:
            # :231-236: later steps go through the base builder's own update, which resets EI's eta to the builder's value
            # (min of the mean over the data only) instead of the eta above (samples and data)
            self._base_acquisition_function = self._base_builder.update_acquisition_function(
                self._base_acquisition_function, model, dataset=dataset)
        elif isinstance(self._base_builder, ExpectedImprovement):  # :237-241: the first EI reuses the eta estimate above
            self._base_acquisition_function = expected_improvement(model, self._eta)
        else:
            self._base_acquisition_function = self._base_builder.prepare_acquisition_function(model, dataset=dataset)
        return self._base_acquisition_function


def _generate_fantasized_data(fantasize_method: str, model, pending_points) -> Dataset:
    """greedy_batch.py:572-594."""
    pending_points = np.asarray(pending_points)
    if fantasize_method == "KB":
        fantasized_obs, _ = model.predict(pending_points)
    elif fantasize_method == "sample":
        fantasized_obs = model.sample(pending_points, num_samples=1)[0]
    else:
        raise NotImplementedError(f"fantasize_method must be KB or sample, received {fantasize_method!r}")
    return Dataset(pending_points, np.asarray(fantasized_obs))


class _fantasized_model(GaussianProcessRegression):
    """greedy_batch.py:630-770: the base model conditioned on additional (fantasised) data.  A native model of its own:
    data = base data + fantasised rows, same kernel / mean function / noise."""

    def __init__(self, model: GaussianProcessRegression, fantasized_data: Dataset):
        if not isinstance(model, GaussianProcessRegression):
            raise NotImplementedError(
                "Fantasizer only works with FastUpdateModel models that also support predict_joint, get_kernel and "
                f"get_observation_noise; received {model!r}"
            )
        self._base = model
        self._fantasized = self._check(fantasized_data)
        super().__init__(self._spec_from_base(), device=model.device, num_rff_features=model._num_rff_features,
                         use_decoupled_sampler=model._use_decoupled_sampler)
        if hasattr(model, "_engine"):
            self.set_engine(model._engine)

    def _check(self, data: Dataset) -> Dataset:
        X, Y = np.asarray(data.query_points), np.asarray(data.observations)
        if X.ndim != 2 or Y.ndim != 2 or Y.shape != (X.shape[0], 1):
            raise ValueError(
                f"fantasized data must have query_points [M, D] and observations [M, 1], got {X.shape} and {Y.shape}")
        return Dataset(X, Y)

    def _joined(self):
        base = self._base.get_internal_data()
        dt = self._base.dtype
        X = np.concatenate([np.asarray(base.query_points, dtype=dt), np.asarray(self._fantasized.query_points, dtype=dt)], axis=0)
        Y = np.concatenate([np.asarray(base.observations, dtype=dt), np.asarray(self._fantasized.observations, dtype=dt)], axis=0)
        return X, Y

    def _hyper_key(self):
        k = self._base.get_kernel()
        return (k.kind, float(k.variance), tuple(np.asarray(k.lengthscales, dtype=np.float64).reshape(-1)),
                float(self._base.get_observation_noise()), float(self._base.get_mean_function().c))

    def _spec_from_base(self) -> GPRSpec:
        self._key = self._hyper_key()
        return GPRSpec(self._joined(), self._base.get_kernel(), self._base.get_mean_function(), self._base.get_observation_noise())

    def update_fantasized_data(self, fantasized_data: Dataset) -> None:
        """greedy_batch.py:656-661.  The data become base + new fantasised rows: when that extends what this model already
        holds (kriging believer within one BO step: earlier pending points keep their values) the cached factors grow by a
        rank-m append; otherwise (new BO step, "sample") the cache is rebuilt."""
        self._fantasized = self._check(fantasized_data)
        if self._hyper_key() != self._key:  # the base model was re-trained: take its hyper-parameters
            self._key = self._hyper_key()
            self._spec.kernel = self._base.get_kernel()
            self._spec.mean_function = self._base.get_mean_function()
            self._spec.noise_variance = self._base.get_observation_noise()
            self._push_hyper()
        X, Y = self._joined()
        self.update(Dataset(X, Y))
        self.optimize(Dataset(X, Y))  # refreshes the cache only when update() could not append


class Fantasizer(GreedyAcquisitionFunctionBuilder):
    """greedy_batch.py:415-569."""

    def __init__(self, base_acquisition_function_builder=None, fantasize_method: str = "KB"):
        if fantasize_method not in ("KB", "sample"):
            raise ValueError(f"fantasize_method must be 'KB' or 'sample', got {fantasize_method!r}")
        if base_acquisition_function_builder is None:
            base_acquisition_function_builder = ExpectedImprovement()
        if isinstance(base_acquisition_function_builder, SingleModelAcquisitionBuilder):
            base_acquisition_function_builder = base_acquisition_function_builder.using(OBJECTIVE)
        self._builder: AcquisitionFunctionBuilder = base_acquisition_function_builder
        self._fantasize_method = fantasize_method
        self._base_acquisition_function = None
        self._fantasized_acquisition = None
        self._fantasized_models: Mapping[Tag, _fantasized_model] = {}

    def __repr__(self) -> str:
        return f"Fantasizer({self._builder!r}, {self._fantasize_method!r})"

    def _update_base_acquisition_function(self, models, datasets):
        if self._base_acquisition_function is not None:
            self._base_acquisition_function = self._builder.update_acquisition_function(
                self._base_acquisition_function, models, datasets)
        else:
            self._base_acquisition_function = self._builder.prepare_acquisition_function(models, datasets)
        return self._base_acquisition_function

    def _update_fantasized_acquisition_function(self, models, datasets, pending_points):
        pending_points = np.asarray(pending_points)
        if pending_points.ndim != 2:
            raise ValueError(f"pending_points must have rank 2, got shape {pending_points.shape}")
        fantasized_data = {
            tag: _generate_fantasized_data(self._fantasize_method, model, pending_points) for tag, model in models.items()
        }
        if datasets is None:
            datasets = fantasized_data
        else:
            datasets = {tag: data + fantasized_data[tag] for tag, data in datasets.items()}
        if self._fantasized_acquisition is None:
            self._fantasized_models = {tag: _fantasized_model(model, fantasized_data[tag]) for tag, model in models.items()}
            self._fantasized_acquisition = self._builder.prepare_acquisition_function(self._fantasized_models, datasets)
        else:
            for tag, model in self._fantasized_models.items():
                if model._base is not models[tag]:
                    raise ValueError("Fantasizer was prepared with a different model object for tag " + repr(tag))
                model.update_fantasized_data(fantasized_data[tag])
            self._fantasized_acquisition = self._builder.update_acquisition_function(
                self._fantasized_acquisition, self._fantasized_models, datasets)
        return self._fantasized_acquisition

    def prepare_acquisition_function(self, models, datasets=None, pending_points=None):
        for model in models.values():
            if not isinstance(model, GaussianProcessRegression):
                raise NotImplementedError(
                    "Fantasizer only works with FastUpdateModel models that also support predict_joint, get_kernel and "
                    f"get_observation_noise; received {model!r}"
                )
        if pending_points is None:
            return self._update_base_acquisition_function(models, datasets)
        return self._update_fantasized_acquisition_function(models, datasets, pending_points)

    def update_acquisition_function(self, function, models, datasets=None, pending_points=None,
                                    new_optimization_step: bool = True):
        if pending_points is None:
            return self._update_base_acquisition_function(models, datasets)
        return self._update_fantasized_acquisition_function(models, datasets, pending_points)
