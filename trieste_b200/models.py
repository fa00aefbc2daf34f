"""Model side of the drop-in boundary.

``GaussianProcessRegression`` mirrors trieste's wrapper of the same name
(trieste/models/gpflow/models.py:69-526) together with the ``GPflowPredictor`` posterior cache
(trieste/models/gpflow/interface.py:89-133).  It satisfies the structural protocols
``ProbabilisticModel`` / ``SupportsPredictJoint`` / ``HasReparamSampler`` / ``HasTrajectorySampler``
/ ``TrainableProbabilisticModel`` (trieste/models/interfaces.py:38-327) by method name, argument
meaning and output shape.  All arithmetic runs on the GPU behind the C-ABI; arrays may be NumPy
(host, staged per call) or ``torch.cuda`` tensors (device-resident, zero-copy).
"""
from __future__ import annotations

import copy
import ctypes as C
import math
from typing import Optional, Tuple

import numpy as np

from . import _lib
from .data import Dataset
from .kernels import Constant, Matern52, Stationary
from .space import SearchSpace

# builders.py:41-82
KERNEL_LENGTHSCALE = 0.2
SIGNAL_NOISE_RATIO_LIKELIHOOD = 10.0


class GPRSpec:
    """What ``gpflow.models.GPR(data, kernel, mean_function, noise_variance)`` carries."""

    def __init__(self, data, kernel: Stationary, mean_function: Optional[Constant] = None, noise_variance: float = 1.0):
        if isinstance(data, Dataset):
            data = data.astuple()
        # dtype follows the model data (fp64 default, fp32 supported end to end: builders.py:41,
        # tests/integration/test_bayesian_optimization.py:641-658)
        x0 = data[0].detach().cpu().numpy() if _lib.is_torch(data[0]) else np.asarray(data[0])
        self.dtype = np.float32 if x0.dtype == np.float32 else np.float64
        self.X = np.ascontiguousarray(np.asarray(x0, dtype=self.dtype))
        self.Y = np.ascontiguousarray(np.asarray(data[1], dtype=self.dtype))
        self.kernel = kernel
        self.mean_function = mean_function if mean_function is not None else Constant(0.0)
        self.noise_variance = float(noise_variance)


def build_gpr(
    data: Dataset,
    search_space: Optional[SearchSpace] = None,
    kernel_priors: bool = True,
    likelihood_variance: Optional[float] = None,
    trainable_likelihood: bool = False,
    kernel: Optional[Stationary] = None,
) -> GPRSpec:
    """``build_gpr`` defaults (trieste/models/gpflow/builders.py:85-155): Matern52, constant mean
    = mean(y), kernel variance = Var(y), lengthscales 0.2 * (upper - lower) * sqrt(D) (:413-423),
    noise = Var(y) / 10^2 unless given (:432-443).  Priors only matter for hyper-parameter
    training, which is out of scope here."""
    dt = np.float32 if np.asarray(data.query_points).dtype == np.float32 else np.float64
    X, Y = np.asarray(data.query_points, dtype=dt), np.asarray(data.observations, dtype=dt)
    if X.shape[0] == 0:
        raise ValueError("Dataset must be populated.")
    variance = float(np.var(Y))
    if variance <= 0:
        variance = 1.0
    mean = float(np.mean(Y))
    D = X.shape[-1]
    if kernel is None:
        if search_space is not None:
            rng_ = np.asarray(search_space.upper) - np.asarray(search_space.lower)
            ls = KERNEL_LENGTHSCALE * rng_ * math.sqrt(D)
            ls = np.where(rng_ == 0, 1.0, ls)
        else:
            ls = np.full(D, KERNEL_LENGTHSCALE * math.sqrt(D))
        kernel = Matern52(variance=variance, lengthscales=ls)
    if likelihood_variance is None:
        noise = variance / SIGNAL_NOISE_RATIO_LIKELIHOOD**2
    else:
        if likelihood_variance <= 0:
            raise ValueError("likelihood_variance must be positive")
        noise = float(likelihood_variance)
    return GPRSpec((X, Y), kernel, Constant(mean), noise)


def _flatten_leading(x, keep: int):
    """[..., k1..k_keep] -> ([prod, k...], leading_shape)."""
    lead = tuple(x.shape[: x.ndim - keep])
    return x.reshape((-1,) + tuple(x.shape[x.ndim - keep :])), lead


class GaussianProcessRegression:
    """H100-native exact GPR posterior.  Construct from a :class:`GPRSpec` (or ``build_gpr(...)``)."""

    def __init__(self, model: GPRSpec, device: int = 0, num_rff_features: int = 1000, use_decoupled_sampler: bool = True):
        _lib.require_gpu()
        if num_rff_features <= 0:
            raise ValueError(f"num_rff_features must be greater or equal to zero, got {num_rff_features}.")
        self._spec = model
        self._device = device
        self._num_rff_features = num_rff_features
        self._use_decoupled_sampler = use_decoupled_sampler
        h = C.c_void_p()
        self._dtype = model.dtype
        _lib.check(_lib.lib().tb_gp_create(C.byref(h), device, _lib.TB_F32 if self._dtype == np.float32 else _lib.TB_F64))
        self._h = h
        self._push_data()
        self._push_hyper()
        self.update_posterior_cache()

    # ---- handle plumbing ---------------------------------------------------------------------
    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            try:
                _lib.lib().tb_gp_destroy(h)
            except Exception:  # pragma: no cover
                pass
            self._h = None

    def __deepcopy__(self, memo):
        """A model with its own device handle, data, hyper-parameters, engine and posterior cache (``copy_to_local_models``
        conditions each copy on its own local data)."""
        new = GaussianProcessRegression(copy.deepcopy(self._spec, memo), self._device, self._num_rff_features,
                                        self._use_decoupled_sampler)
        memo[id(self)] = new
        if hasattr(self, "_engine"):
            new.set_engine(self._engine)
        return new

    @property
    def handle(self) -> C.c_void_p:
        return self._h

    @property
    def device(self) -> int:
        return self._device

    @property
    def dtype(self):
        return self._dtype

    def _push_data(self) -> None:
        X, Y = self._spec.X, self._spec.Y
        if X.ndim != 2 or Y.ndim != 2 or Y.shape[1] != 1 or X.shape[0] != Y.shape[0]:
            raise ValueError(f"expected query_points [N, D] and observations [N, 1], got {X.shape} and {Y.shape}")
        if X.shape[0] == 0:
            raise ValueError("Dataset must be populated.")
        y = np.ascontiguousarray(Y[:, 0])
        self._cache_current = False
        _lib.check(_lib.lib().tb_gp_set_data(self._h, X.ctypes.data, y.ctypes.data, X.shape[0], X.shape[1]))

    def _push_hyper(self) -> None:
        k = self._spec.kernel
        ls = np.ascontiguousarray(k.lengthscales, dtype=np.float64)
        self._cache_current = False
        _lib.check(
            _lib.lib().tb_gp_set_hyper(
                self._h,
                _lib.KERNEL_IDS[k.kind],
                k.variance,
                ls.ctypes.data_as(C.POINTER(C.c_double)),
                int(ls.size),
                self._spec.noise_variance,
                self._spec.mean_function.c,
            )
        )

    def set_engine(self, engine: str) -> None:
        """Engine of the variance GEMM (predict / EI / LCB / log-EI / argmax): ``"fp64"`` = native DMMA,
        ``"int8"`` = fp64-accurate Ozaki splitting on the INT8 tensor cores (same stated tolerances)."""
        if engine not in ("fp64", "int8", "int8x21"):
            raise ValueError(f"engine must be 'fp64', 'int8' or 'int8x21', got {engine!r}")
        # "int8" picks the number of digit products (15 or 21; fp32 models 6 or 10) from the a-priori error estimate of the
        # cache; "int8x21" pins six digits (21 products)
        _lib.check(_lib.lib().tb_gp_set_engine(self._h, {"fp64": 0, "int8": 1, "int8x21": 2}[engine]))
        self._engine = engine

    @property
    def engine(self) -> str:
        return getattr(self, "_engine", "int8")  # the handle's default until set_engine is called

    def engine_info(self) -> Tuple[int, float]:
        """(int8 digit products per k-step of the variance GEMM — 15 / 21, fp32 models 6 / 10, 0 = native fp64 engine —,
        a-priori estimate of max |Δvar| / σ_f² of a reduced mode)."""
        n, est = C.c_int(0), C.c_double(0.0)
        _lib.check(_lib.lib().tb_gp_engine_info(self._h, C.byref(n), C.byref(est)))
        return n.value, est.value

    def update_posterior_cache(self) -> None:
        """interface.py:108-112 — must follow any change of data or hyper-parameters."""
        self._cache_current = False
        _lib.check(_lib.lib().tb_gp_update_posterior_cache(self._h))
        self._cache_current = True

    # ---- ProbabilisticModel ------------------------------------------------------------------
    def predict(self, query_points) -> Tuple[np.ndarray, np.ndarray]:
        """[..., D] -> (mean [..., 1], var [..., 1]), variance clipped to >= 1e-12
        (interfaces.py:55-64; interface.py:119-124)."""
        x, _ = _lib.as_contiguous(query_points, self._dtype)
        self._check_dim(x)
        flat, lead = _flatten_leading(x, 1)
        M = flat.shape[0]
        mean, pm = _lib.empty_like_kind(flat, (M, 1), self._dtype)
        var, pv = _lib.empty_like_kind(flat, (M, 1), self._dtype)
        _lib.check(_lib.lib().tb_gp_predict(self._h, _ptr(flat), M, pm, pv))
        return mean.reshape(lead + (1,)), var.reshape(lead + (1,))

    def mean_gradient(self, query_points) -> Tuple[np.ndarray, np.ndarray]:
        """[..., D] -> (mean [..., 1], d mean / d x [..., D]): the posterior mean and the gradient the reference takes of it
        with a GradientTape for the Lipschitz estimate of local penalisation (greedy_batch.py:207-217).  No variance is
        formed: one pass over the training rows per point."""
        x, _ = _lib.as_contiguous(query_points, self._dtype)
        self._check_dim(x)
        flat, lead = _flatten_leading(x, 1)
        M, D = flat.shape
        mean, pm = _lib.empty_like_kind(flat, (M, 1), self._dtype)
        grad, pg = _lib.empty_like_kind(flat, (M, D), self._dtype)
        _lib.check(_lib.lib().tb_gp_mean_gradient(self._h, _ptr(flat), M, pm, pg))
        return mean.reshape(lead + (1,)), grad.reshape(lead + (D,))

    def predict_joint(self, query_points) -> Tuple[np.ndarray, np.ndarray]:
        """[..., B, D] -> (mean [..., B, 1], cov [..., 1, B, B]) (interfaces.py:133-140;
        interface.py:126-133)."""
        x, _ = _lib.as_contiguous(query_points, self._dtype)
        if x.ndim < 2:
            raise ValueError(f"predict_joint needs query points of rank >= 2, got shape {tuple(x.shape)}")
        self._check_dim(x)
        flat, lead = _flatten_leading(x, 2)
        nb, q = flat.shape[0], flat.shape[1]
        mean, pm = _lib.empty_like_kind(flat, (nb, q, 1), self._dtype)
        cov, pc = _lib.empty_like_kind(flat, (nb, 1, q, q), self._dtype)
        _lib.check(_lib.lib().tb_gp_predict_joint(self._h, _ptr(flat), nb, q, pm, pc))
        return mean.reshape(lead + (q, 1)), cov.reshape(lead + (1, q, q))

    def covariance_between_points(self, query_points_1, query_points_2) -> np.ndarray:
        """[..., N, D], [M, D] -> [..., 1, N, M]: posterior covariance between two sets of points,
        ``K12 - Kx1 (K + noise I)^-1 Kx2`` (models.py:188-254; SupportsCovarianceBetweenPoints, interfaces.py:143-163)."""
        x1 = np.ascontiguousarray(np.asarray(query_points_1, dtype=self._dtype))
        x2 = np.ascontiguousarray(np.asarray(query_points_2, dtype=self._dtype))
        if x1.ndim < 2 or x2.ndim != 2:
            raise ValueError(f"expected query_points_1 [..., N, D] and query_points_2 [M, D], got {x1.shape} and {x2.shape}")
        self._check_dim(x1)
        self._check_dim(x2)
        lead, n, m = x1.shape[:-2], x1.shape[-2], x2.shape[0]
        flat = x1.reshape(-1, x1.shape[-1])
        out = np.empty((flat.shape[0], m), dtype=self._dtype)
        if flat.shape[0] and m:
            _lib.check(
                _lib.lib().tb_gp_covariance_between_points(self._h, flat.ctypes.data, flat.shape[0], x2.ctypes.data, m, out.ctypes.data)
            )
        return out.reshape(lead + (n, m))[..., None, :, :]

    # ---- conditioning on additional (fantasised) data: models.py:355-525 ------------------------------
    def _conditional_parts(self, query_points, additional_data: Dataset):
        xq = np.ascontiguousarray(np.asarray(query_points, dtype=self._dtype))
        xa = np.ascontiguousarray(np.asarray(additional_data.query_points, dtype=self._dtype))
        ya = np.asarray(additional_data.observations, dtype=np.float64)
        if xq.ndim != 2 or xa.ndim < 2 or ya.shape != xa.shape[:-1] + (1,):
            raise ValueError(
                "additional_data must have query_points with shape [..., N, D] and observations with shape [..., N, 1], "
                f"and query_points should have shape [M, D]; got {xa.shape}, {ya.shape} and {xq.shape}"
            )
        self._check_dim(xq)
        self._check_dim(xa)
        n2 = xa.shape[-2]
        lead = xa.shape[:-2]
        flat_a = xa.reshape(-1, xa.shape[-1])
        # posterior moments of the additional points (joint, per leading batch) and their covariance with the queries;
        # all O(N^2)-per-point work is on the device, the N2 x N2 algebra below is host arithmetic
        xa3 = xa.reshape((-1, n2, xa.shape[-1]))
        nbatch = xa3.shape[0]
        if n2 <= 32:  # the batched joint kernels (the reference calls predict_joint here too, models.py:383-385)
            mean_add, cov_add = self.predict_joint(xa3)
            mean_add = np.asarray(mean_add, dtype=np.float64)[..., 0]  # [B, N2]
            cov_add = np.asarray(cov_add, dtype=np.float64)[:, 0]  # [B, N2, N2]
        else:
            mean_add = np.asarray(self.predict(flat_a)[0], dtype=np.float64).reshape(nbatch, n2)
            cov_add = np.stack([np.asarray(self.covariance_between_points(xa3[b], xa3[b]), dtype=np.float64)[0]
                                for b in range(nbatch)])
        limit = 16384 - flat_a.shape[0]
        if limit < 1:
            raise ValueError("too many additional points (at most 16383 over all leading dimensions)")
        cross = [np.asarray(self.covariance_between_points(flat_a, xq[i:i + limit]), dtype=np.float64)[0]
                 for i in range(0, xq.shape[0], limit)]
        cov_cross = np.concatenate(cross, axis=-1).reshape(nbatch, n2, xq.shape[0])  # [B, N2, M]
        L_add = np.linalg.cholesky(cov_add + self._spec.noise_variance * np.eye(n2))
        A = np.linalg.solve(L_add, cov_cross)  # [B, N2, M]
        AM = np.linalg.solve(L_add, (ya.reshape(nbatch, n2) - mean_add)[..., None])  # [B, N2, 1]
        return xq, lead, A, AM

    def conditional_predict_f(self, query_points, additional_data: Dataset):
        """Marginal posterior at ``query_points`` [M, D] conditioned on the model's data AND ``additional_data``
        ([..., N, D], [..., N, 1]) by the exact update formulas (models.py:355-425; Chevalier et al. 2014, eqs. 8-10):
        returns (mean [..., M, 1], var [..., M, 1])."""
        xq, lead, A, AM = self._conditional_parts(query_points, additional_data)
        mean_qp, var_qp = self.predict(xq)
        mean_qp, var_qp = np.asarray(mean_qp, dtype=np.float64)[:, 0], np.asarray(var_qp, dtype=np.float64)[:, 0]
        var_new = var_qp[None, :] - np.sum(A * A, axis=-2)  # [B, M]
        mean_new = mean_qp[None, :] + np.einsum("bnm,bn->bm", A, AM[..., 0])
        shape = lead + (xq.shape[0], 1)
        return mean_new.reshape(shape).astype(self._dtype), var_new.reshape(shape).astype(self._dtype)

    def conditional_predict_joint(self, query_points, additional_data: Dataset):
        """Joint posterior at ``query_points`` [M, D] conditioned on ``additional_data`` (models.py:427-500):
        returns (mean [..., M, 1], cov [..., 1, M, M]); M at most 8192."""
        xq, lead, A, AM = self._conditional_parts(query_points, additional_data)
        cov_qp = np.asarray(self.covariance_between_points(xq, xq), dtype=np.float64)[0]  # [M, M]
        mean_qp = np.asarray(self.predict(xq)[0], dtype=np.float64)[:, 0]
        cov_new = cov_qp[None] - np.einsum("bnm,bnk->bmk", A, A)
        mean_new = mean_qp[None, :] + np.einsum("bnm,bn->bm", A, AM[..., 0])
        M = xq.shape[0]
        return (mean_new.reshape(lead + (M, 1)).astype(self._dtype), cov_new.reshape(lead + (1, M, M)).astype(self._dtype))

    def conditional_predict_f_sample(self, query_points, additional_data: Dataset, num_samples: int, seed: Optional[int] = None):
        """models.py:490-509: ``num_samples`` joint samples at ``query_points`` [M, D] conditioned on ``additional_data``
        — gpflow ``sample_mvn`` on :meth:`conditional_predict_joint` (full covariance + jitter 1e-6, Cholesky,
        mean + L z).  Returns [..., num_samples, M, 1]."""
        if num_samples <= 0:
            raise ValueError(f"num_samples must be positive, got {num_samples}")
        mean, cov = self.conditional_predict_joint(query_points, additional_data)  # [..., M, 1], [..., 1, M, M]
        mean = np.asarray(mean, dtype=np.float64)[..., 0]  # [..., M]
        cov = np.asarray(cov, dtype=np.float64)[..., 0, :, :]  # [..., M, M]
        M = mean.shape[-1]
        L = np.linalg.cholesky(cov + 1e-6 * np.eye(M))
        z = np.random.default_rng(seed).standard_normal(mean.shape[:-1] + (num_samples, M))
        samples = mean[..., None, :] + np.einsum("...ij,...sj->...si", L, z)  # [..., S, M]
        return samples[..., None].astype(self._dtype)

    def conditional_predict_y(self, query_points, additional_data: Dataset):
        """models.py:502-525: :meth:`conditional_predict_f` plus the observation noise."""
        mean, var = self.conditional_predict_f(query_points, additional_data)
        return mean, var + self._spec.noise_variance

    def predict_y(self, query_points):
        """Gaussian likelihood: adds the observation noise to the variance (models.py:126-131)."""
        mean, var = self.predict(query_points)
        return mean, var + self._spec.noise_variance

    def sample(self, query_points, num_samples: int, seed: Optional[int] = None):
        """[..., N, D] -> [..., S, N, 1]: joint samples (interface.py:135-138 -> gpflow predict_f_samples: full covariance
        + jitter 1e-6, Cholesky, mean + L z).  Sets of up to 32 points go through the batched ``predict_joint`` kernels,
        larger ones (the ExactThompsonSampler's case) through ``tb_gp_sample_joint`` — covariance and Cholesky on the
        device, one set at a time."""
        if num_samples <= 0:
            raise ValueError(f"num_samples must be positive, got {num_samples}")
        x = np.asarray(query_points, dtype=self._dtype)
        if x.ndim < 2:
            raise ValueError(f"query points must have rank >= 2, got shape {x.shape}")
        self._check_dim(x)
        q = x.shape[-2]
        rng = np.random.default_rng(seed)
        if q <= 32:
            from .sampler import _reparam_sample

            return _reparam_sample(self, x, rng.standard_normal((q, num_samples)), 1e-6)
        flat = np.ascontiguousarray(x.reshape((-1,) + x.shape[-2:]))
        out = np.empty((flat.shape[0], num_samples, q), dtype=self._dtype)
        for i in range(flat.shape[0]):
            z = np.ascontiguousarray(rng.standard_normal((num_samples, q)))
            _lib.check(
                _lib.lib().tb_gp_sample_joint(self._h, flat[i].ctypes.data, q, z.ctypes.data, num_samples, 1e-6, out[i].ctypes.data)
            )
        return out.reshape(x.shape[:-2] + (num_samples, q, 1))

    def log(self, dataset: Optional[Dataset] = None) -> None:
        """TensorBoard summaries in the reference (models/utils.py:33-107): observability only."""

    # ---- TrainableProbabilisticModel -----------------------------------------------------------
    APPEND_MAX = 64  # tb_gp_append_data handles up to this many new rows per call

    def update(self, dataset: Dataset) -> None:
        """models.py:171-186: swap the data, refresh the posterior cache.  When the new data set is the old one plus a
        few appended rows (the BO loop's case, bayesian_optimizer.py:786-800) the cached factors are extended in
        O(m N^2) by ``tb_gp_append_data`` instead of being rebuilt in O(N^3)."""
        X = np.ascontiguousarray(np.asarray(dataset.query_points, dtype=self._dtype))
        Y = np.ascontiguousarray(np.asarray(dataset.observations, dtype=self._dtype))
        if X.ndim != 2 or X.shape[-1] != self._spec.X.shape[-1]:
            raise ValueError(f"new query points must be [N, {self._spec.X.shape[-1]}], got {X.shape}")
        n0 = self._spec.X.shape[0]
        m = X.shape[0] - n0
        appended = (
            getattr(self, "_cache_current", False) and 0 < m <= self.APPEND_MAX and Y.shape[0] == X.shape[0]
            and np.array_equal(X[:n0], self._spec.X) and np.array_equal(Y[:n0], self._spec.Y)
        )
        self._spec.X, self._spec.Y = X, Y
        self.last_update_appended = bool(appended)
        if appended:
            xn = np.ascontiguousarray(X[n0:])
            yn = np.ascontiguousarray(Y[n0:].reshape(-1))
            try:
                _lib.check(_lib.lib().tb_gp_append_data(self._h, xn.ctypes.data, yn.ctypes.data, m))
                return
            except Exception:
                self._cache_current = False
                raise
        self._push_data()
        self.update_posterior_cache()

    def optimize(self, dataset: Dataset) -> None:
        """Hyper-parameter training (models.py:256-292) is the once-per-step model fit and is OUT OF
        SCOPE of this engine (SURVEY.md §2 row 6): hyper-parameters are set through
        :meth:`set_hyperparameters`; the cache refresh that follows training in the reference
        (models.py:290-291) is kept — and skipped when the cache already matches the data and hyper-parameters (e.g. right
        after an appending :meth:`update`)."""
        if not getattr(self, "_cache_current", False):
            self.update_posterior_cache()

    def set_hyperparameters(self, kernel: Optional[Stationary] = None, noise_variance: Optional[float] = None,
                            mean_constant: Optional[float] = None) -> None:
        if kernel is not None:
            self._spec.kernel = kernel
        if noise_variance is not None:
            self._spec.noise_variance = float(noise_variance)
        if mean_constant is not None:
            self._spec.mean_function = Constant(mean_constant)
        self._push_hyper()
        self.update_posterior_cache()

    # ---- getters used by samplers (interfaces.py:166-225) -------------------------------------------
    def get_kernel(self) -> Stationary:
        return self._spec.kernel

    def get_mean_function(self) -> Constant:
        return self._spec.mean_function

    def get_observation_noise(self) -> float:
        return self._spec.noise_variance

    def get_internal_data(self) -> Dataset:
        return Dataset(self._spec.X, self._spec.Y)

    def get_cholesky(self) -> np.ndarray:
        N = self._spec.X.shape[0]
        out = np.empty((N, N), dtype=self._dtype)
        _lib.check(_lib.lib().tb_gp_get_cholesky(self._h, out.ctypes.data))
        return out

    # ---- samplers --------------------------------------------------------------------------------
    def reparam_sampler(self, num_samples: int):
        """interface.py:189-195 -> BatchReparametrizationSampler."""
        from .sampler import BatchReparametrizationSampler

        return BatchReparametrizationSampler(num_samples, self)

    def trajectory_sampler(self):
        """models.py:323-345: decoupled sampler by default, plain RFF with ``use_decoupled_sampler=False``."""
        from .sampler import DecoupledTrajectorySampler, RandomFourierFeatureTrajectorySampler

        if self._use_decoupled_sampler:
            return DecoupledTrajectorySampler(self, self._num_rff_features)
        return RandomFourierFeatureTrajectorySampler(self, self._num_rff_features)

    # ---- helpers -----------------------------------------------------------------------------------
    def _check_dim(self, x) -> None:
        D = self._spec.X.shape[-1]
        if x.ndim < 1 or x.shape[-1] != D:
            raise ValueError(f"query points must have trailing dimension {D}, got shape {tuple(x.shape)}")


def _ptr(a) -> int:
    return a.data_ptr() if _lib.is_torch(a) else a.ctypes.data


class ModelStack:
    """Independent models side by side along the output axis (interfaces.py:337-397): ``ModelStack((m1, 1), (m2, 1))``.
    ``predict`` and ``sample`` concatenate the members' outputs along the last axis in member order."""

    def __init__(self, model_with_event_size, *models_with_event_sizes):
        pairs = (model_with_event_size,) + models_with_event_sizes
        self._models, self._event_sizes = (tuple(x) for x in zip(*pairs))

    @property
    def models(self):
        return self._models

    @property
    def event_sizes(self):
        return self._event_sizes

    def predict(self, query_points):
        means, vars_ = zip(*(m.predict(query_points) for m in self._models))
        return _concat_last(means), _concat_last(vars_)

    def sample(self, query_points, num_samples: int):
        return _concat_last([m.sample(query_points, num_samples) for m in self._models])

    def log(self, dataset: Optional[Dataset] = None) -> None:
        for m in self._models:
            m.log(dataset)


class TrainableModelStack(ModelStack):
    """A :class:`ModelStack` of trainable members (interfaces.py:400-443): ``update`` and ``optimize`` give member i the
    observation columns of its event."""

    def _split(self, dataset: Dataset):
        obs = np.asarray(dataset.observations)
        edges = np.cumsum(self._event_sizes)[:-1]
        return [Dataset(dataset.query_points, o) for o in np.split(obs, edges, axis=-1)]

    def update(self, dataset: Dataset) -> None:
        for m, d in zip(self._models, self._split(dataset)):
            m.update(d)

    def optimize(self, dataset: Dataset):
        return [m.optimize(d) for m, d in zip(self._models, self._split(dataset))]


def _concat_last(parts):
    if _lib.is_torch(parts[0]):
        import torch

        return torch.cat(list(parts), dim=-1)
    return np.concatenate([np.asarray(p) for p in parts], axis=-1)
