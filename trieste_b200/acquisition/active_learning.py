"""Active-learning acquisition functions — mirrors trieste/acquisition/function/active_learning.py (PredictiveVariance
:36-110, ExpectedFeasibility :113-247, BayesianActiveLearningByDisagreement :418-513).

Single queries run the fused predict + tail chain of the other analytic functions, so values, gradients, ``fused_argmax``
and the device L-BFGS (``maximize_from``) all stay on the GPU.  Query batches of :func:`predictive_variance` (q >= 2)
run the joint-posterior chain of batch MC-EI with a log-determinant tail (``tb_acq_predictive_variance``), value and
gradient, which is what ``batchify_joint`` maximises over ``space ** q``.

Deviations from the reference:

- the query batch of :func:`predictive_variance` is bounded by 1 <= q <= 32 (the reference has no bound);
- ``tf.debugging.check_numerics`` on the feasibility criteria's G (active_learning.py:233, :242) is not reproduced.  With the
  tail's clipped variance (>= 1e-12) and finite inputs G is finite; non-finite inputs follow the NaN semantics of every
  other kind through the argmax and the L-BFGS;
- ``IntegratedVarianceReduction`` (:250-415) is not provided;
- argument errors are ``ValueError`` (the reference raises ``InvalidArgumentError`` for some of them).
"""
from __future__ import annotations

from typing import Optional

import numpy as np

from .. import _lib
from ..data import Dataset
from ..models import _flatten_leading, _ptr
from .function import JITTER, _FusedSingleQuery
from .interface import SingleModelAcquisitionBuilder


class PredictiveVariance(SingleModelAcquisitionBuilder):
    """active_learning.py:36-83: the determinant of the predictive covariance over the batch points; for a batch of size
    one, the predictive variance."""

    def __init__(self, jitter: float = JITTER) -> None:
        self._jitter = jitter

    def __repr__(self) -> str:
        return f"PredictiveVariance(jitter={self._jitter!r})"

    def prepare_acquisition_function(self, model, dataset: Optional[Dataset] = None):
        return predictive_variance(model, self._jitter)

    def update_acquisition_function(self, function, model, dataset: Optional[Dataset] = None):
        return function  # no need to update anything (:72-83)


class predictive_variance(_FusedSingleQuery):
    """active_learning.py:86-110: ``exp(logdet(cov + jitter))`` of the joint posterior of each query batch ``[..., q, D]``.
    As in the reference the jitter is added to every entry of the covariance, not only to its diagonal.  q = 1 runs the
    fused single-query kind (value ``var + jitter``, with ``fused_argmax`` and ``maximize_from``); q >= 2 the joint chain."""

    _acq = _lib.ACQ_PREDICTIVE_VARIANCE

    def __init__(self, model, jitter: float):
        super().__init__(model, jitter)

    @property
    def jitter(self) -> float:
        return self._param

    @staticmethod
    def _single(x) -> bool:
        shape = x.shape if hasattr(x, "shape") else np.shape(x)
        return len(shape) >= 2 and shape[-2] == 1

    def _batches(self, x):
        x, _ = _lib.as_contiguous(x, self._model.dtype)
        if x.ndim < 2:
            raise ValueError(f"expected [..., B, D] query batches, got shape {tuple(x.shape)}")
        self._model._check_dim(x)
        return _flatten_leading(x, 2)

    def __call__(self, x):
        if self._single(x):
            return super().__call__(x)
        flat, lead = self._batches(x)
        nb, q = flat.shape[0], flat.shape[1]
        out, po = _lib.empty_like_kind(flat, (nb, 1), self._model.dtype)
        _lib.check(_lib.lib().tb_acq_predictive_variance(self._model.handle, _ptr(flat), nb, q, self._param, po, None))
        return out.reshape(lead + (1,))

    def value_and_gradient(self, x):
        """[..., B, D] -> (values [..., 1], d values / d x [..., B, D]), what ``tfp.math.value_and_gradient`` returns through
        ``batchify_joint`` (optimizer.py:621-629, 897-936)."""
        if self._single(x):
            return super().value_and_gradient(x)
        flat, lead = self._batches(x)
        nb, q, D = flat.shape
        out, po = _lib.empty_like_kind(flat, (nb, 1), self._model.dtype)
        grad, pg = _lib.empty_like_kind(flat, (nb, q, D), self._model.dtype)
        _lib.check(_lib.lib().tb_acq_predictive_variance(self._model.handle, _ptr(flat), nb, q, self._param, po, pg))
        return out.reshape(lead + (1,)), grad.reshape(lead + (q, D))


def _check_feasibility_args(threshold, alpha, delta) -> None:
    """active_learning.py:132-136"""
    if np.ndim(threshold) != 0:
        raise ValueError(f"threshold must be a scalar, got shape {np.shape(threshold)}")
    if np.ndim(alpha) != 0:
        raise ValueError(f"alpha must be a scalar, got shape {np.shape(alpha)}")
    if not float(alpha) > 0.0:
        raise ValueError("Parameter alpha must be positive.")
    if not np.isfinite(float(alpha)):
        raise ValueError("Parameter alpha must be finite.")
    if np.ndim(delta) != 0 or delta not in [1, 2]:
        raise ValueError(f"delta must be 1 (bichon) or 2 (ranjan), got {delta!r}")


class ExpectedFeasibility(SingleModelAcquisitionBuilder):
    """active_learning.py:113-169: the bichon (delta = 1) or ranjan (delta = 2) criterion for finding the contour
    f(x) = threshold of a failure or feasibility region."""

    def __init__(self, threshold: float, alpha: float = 1, delta: int = 1) -> None:
        _check_feasibility_args(threshold, alpha, delta)
        self._threshold = threshold
        self._alpha = alpha
        self._delta = delta

    def __repr__(self) -> str:
        return (
            f"ExpectedFeasibility(threshold={self._threshold!r}, alpha={self._alpha!r},"
            f" delta={self._delta!r})"
        )

    def prepare_acquisition_function(self, model, dataset: Optional[Dataset] = None):
        return bichon_ranjan_criterion(model, self._threshold, self._alpha, self._delta)

    def update_acquisition_function(self, function, model, dataset: Optional[Dataset] = None):
        return function  # no need to update anything (:163-169)


class bichon_ranjan_criterion(_FusedSingleQuery):
    """active_learning.py:172-247: ``E[max(0, (alpha s(x))^delta - |T - m(x)|^delta)]`` in closed form, ``G_1 s`` (bichon)
    or ``G_2 var`` (ranjan), batch size one.  alpha is pushed to the native handle before every launch, so several
    functions on one model never see each other's alpha."""

    def __init__(self, model, threshold: float, alpha: float, delta: int):
        _check_feasibility_args(threshold, alpha, delta)
        super().__init__(model, float(threshold))
        self._alpha = float(alpha)
        self._delta = int(delta)
        self._acq = _lib.ACQ_FEASIBILITY_BICHON if self._delta == 1 else _lib.ACQ_FEASIBILITY_RANJAN

    @property
    def threshold(self) -> float:
        return self._param

    @property
    def alpha(self) -> float:
        return self._alpha

    @property
    def delta(self) -> int:
        return self._delta

    def _before_call(self) -> None:
        _lib.check(_lib.lib().tb_acq_set_feasibility(self._model.handle, self._alpha))


class BayesianActiveLearningByDisagreement(SingleModelAcquisitionBuilder):
    """active_learning.py:418-460: the information gain of the predictive entropy (Houlsby et al. 2011)."""

    def __init__(self, jitter: float = JITTER) -> None:
        self._jitter = jitter

    def __repr__(self) -> str:
        return f"BayesianActiveLearningByDisagreement(jitter={self._jitter!r})"

    def prepare_acquisition_function(self, model, dataset: Optional[Dataset] = None):
        return bayesian_active_learning_by_disagreement(model, self._jitter)

    def update_acquisition_function(self, function, model, dataset: Optional[Dataset] = None):
        return function  # no need to update anything (:449-460)


class bayesian_active_learning_by_disagreement(_FusedSingleQuery):
    """active_learning.py:463-513: ``h(Phi(m / sqrt(v + 1))) - sqrt(C2)/sqrt(v + C2) exp(-m^2 / (2 (v + C2)))`` with
    ``v = max(var, jitter)``, ``C2 = pi log(2) / 2`` and ``h(p) = -p log(p + jitter) - (1 - p) log(1 - p + jitter)``, batch
    size one."""

    _acq = _lib.ACQ_BALD

    def __init__(self, model, jitter: float):
        if not jitter > 0:
            raise ValueError("Jitter must be positive.")
        super().__init__(model, jitter)

    @property
    def jitter(self) -> float:
        return self._param


__all__ = [
    "BayesianActiveLearningByDisagreement",
    "ExpectedFeasibility",
    "PredictiveVariance",
    "bayesian_active_learning_by_disagreement",
    "bichon_ranjan_criterion",
    "predictive_variance",
]
