"""Model-side samplers — mirrors trieste/models/gpflow/sampler.py
(BatchReparametrizationSampler :167-287, RandomFourierFeatureTrajectorySampler :452-591,
ResampleableRandomFourierFeatureFunctions :741-806, feature_decomposition_trajectory :858-953)."""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional

import numpy as np

from . import _lib
from .models import GaussianProcessRegression, _flatten_leading, _ptr

JITTER = 1e-6


def _reparam_sample(model: GaussianProcessRegression, at, eps: np.ndarray, jitter: float):
    """at [..., q, D], eps [q, S] -> samples [..., S, q, 1]."""
    x, _ = _lib.as_contiguous(at, model.dtype)
    flat, lead = _flatten_leading(x, 2)
    nb, q = flat.shape[0], flat.shape[1]
    S = eps.shape[1]
    eps = np.ascontiguousarray(eps, dtype=model.dtype)
    out, po = _lib.empty_like_kind(flat, (nb, S, q), model.dtype)
    _lib.check(_lib.lib().tb_gp_reparam_sample(model.handle, _ptr(flat), nb, q, eps.ctypes.data, S, jitter, po))
    return out.reshape(lead + (S, q, 1))


def qmc_normal_samples(num_samples: int, n_sample_dim: int, skip: int = 0, dtype=np.float64) -> np.ndarray:
    """sampler.py:53-79: ``num_samples`` points of the (unscrambled, Joe-Kuo) Sobol sequence in ``n_sample_dim`` dimensions,
    skipping the first ``skip``, mapped through the standard normal quantile.  ``tf.math.sobol_sample`` never returns the
    origin (its quantile would be -inf), so the sequence starts at the first non-zero point; SciPy's generator uses the same
    direction numbers and Gray-code order.  The exact point order of TensorFlow's kernel cannot be checked here (parity
    unpinned); what the samplers rely on — low-discrepancy, deterministic, disjoint blocks for successive ``skip`` values —
    holds by construction."""
    if num_samples == 0 or n_sample_dim == 0:
        return np.zeros((num_samples, n_sample_dim), dtype=dtype)
    from scipy.special import ndtri
    from scipy.stats import qmc

    gen = qmc.Sobol(d=int(n_sample_dim), scramble=False)
    gen.fast_forward(int(skip) + 1)  # + 1: never the origin
    return ndtri(gen.random(int(num_samples))).astype(dtype)


def sobol_points(num_samples: int, dim: int, skip: int = 0) -> np.ndarray:
    """``tf.math.sobol_sample(dim, num_samples, skip=skip)`` as MultivariateNormalCDF draws it (utils.py:147-152):
    [num_samples, dim] points of the unscrambled Sobol sequence, on the convention of :func:`qmc_normal_samples` (first
    point after ``fast_forward(skip + 1)``, never the origin) but without the normal quantile.  Column j is the same
    sequence whatever ``dim`` is, so a dimension-(q-1) draw holds the points of every CDF of dimension q or q-1.
    ``fast_forward`` is linear in ``skip`` (about 2 s at the largest skip, 1e9)."""
    if num_samples == 0 or dim == 0:
        return np.zeros((num_samples, dim))
    from scipy.stats import qmc

    gen = qmc.Sobol(d=int(dim), scramble=False)
    gen.fast_forward(int(skip) + 1)
    return gen.random(int(num_samples))


class IndependentReparametrizationSampler:
    """sampler.py:82-164: ``x -> mu(x) + eps * sigma(x)`` with base samples eps [S, 1] fixed until
    :meth:`reset_sampler`; batch size one only.  One batched GPU ``predict`` per call; the S-fold broadcast is host
    arithmetic on the [..., 1] outputs.  ``qmc=True`` draws the base samples from the Sobol sequence (:func:`qmc_normal_samples`);
    ``qmc_skip`` advances the class-wide ``skip`` counter so that different samplers use different points (:90-117)."""

    skip: int = 0  # number of Sobol points already handed out (sampler.py:93-94: shared by both sampler classes)

    def __init__(self, sample_size: int, model, qmc: bool = False, qmc_skip: bool = True, seed: Optional[int] = None):
        if sample_size <= 0:
            raise ValueError(f"sample_size must be positive, got {sample_size}")
        self._sample_size = sample_size
        self._model = model
        self._qmc = qmc
        self._qmc_skip = qmc_skip
        self._rng = np.random.default_rng(seed)
        self._eps: Optional[np.ndarray] = None  # [S, 1]
        self._initialized = False

    def set_eps(self, eps) -> None:
        eps = np.asarray(eps, dtype=np.float64).reshape(-1, 1)
        if eps.shape[0] != self._sample_size:
            raise ValueError(f"eps must hold {self._sample_size} base samples, got {eps.shape[0]}")
        self._eps = eps
        self._initialized = True

    def sample(self, at, *, jitter: float = JITTER):
        """at [..., 1, D] -> [..., S, 1, 1]."""
        shape = tuple(np.shape(at))
        if len(shape) < 2 or shape[-2] != 1:
            raise ValueError(f"IndependentReparametrizationSampler only supports batch sizes of one, got shape {shape}")
        if jitter < 0:
            raise ValueError(f"jitter must be non-negative, got {jitter}")
        x = at.detach().cpu().numpy() if hasattr(at, "detach") else np.asarray(at)
        mean, var = self._model.predict(x[..., None, :, :])  # [..., 1, 1, 1]
        mean, var = np.asarray(mean, dtype=np.float64), np.asarray(var, dtype=np.float64)
        if not self._initialized or self._eps is None:
            if self._qmc:  # sampler.py:140-148
                skip = 0
                if self._qmc_skip:
                    skip = IndependentReparametrizationSampler.skip
                    IndependentReparametrizationSampler.skip = skip + self._sample_size
                self._eps = qmc_normal_samples(self._sample_size, 1, skip)
            else:
                self._eps = self._rng.standard_normal((self._sample_size, 1))
            self._initialized = True
        return mean + np.sqrt(var + jitter) * self._eps[:, None, :]  # [..., S, 1, 1]

    def reset_sampler(self) -> None:
        self._initialized = False


class BatchReparametrizationSampler:
    """sampler.py:167-287.  The base samples ``eps`` [L=1, q, S] are drawn once (NumPy generator —
    the reference uses tf.random.normal; RNG streams are never bit-compatible, so ``eps`` can also be
    injected with :meth:`set_eps`) and stay fixed until :meth:`reset_sampler`."""

    def __init__(self, sample_size: int, model: GaussianProcessRegression, qmc: bool = False, qmc_skip: bool = True,
                 seed: Optional[int] = None):
        if sample_size <= 0:
            raise ValueError(f"sample_size must be positive, got {sample_size}")
        if not hasattr(model, "predict_joint"):
            raise ValueError(f"BatchReparametrizationSampler only works with models that support predict_joint; received {model!r}")
        self._sample_size = sample_size
        self._model = model
        self._qmc = qmc
        self._qmc_skip = qmc_skip
        self._rng = np.random.default_rng(seed)
        self._eps: Optional[np.ndarray] = None  # [q, S]
        self._initialized = False

    def set_eps(self, eps: np.ndarray) -> None:
        eps = np.ascontiguousarray(np.asarray(eps, dtype=np.float64))
        if eps.ndim == 3:
            eps = eps[0]
        if eps.ndim != 2 or eps.shape[1] != self._sample_size:
            raise ValueError(f"eps must be [q, {self._sample_size}], got {eps.shape}")
        self._eps = eps
        self._initialized = True

    def _get_eps(self, batch_size: int) -> np.ndarray:
        if batch_size <= 0:
            raise ValueError("batch size must be positive")
        if not self._initialized or self._eps is None:
            if self._qmc:  # sampler.py:241-254: S points in batch_size dimensions, stored [q, S]
                skip = 0
                if self._qmc_skip:
                    skip = IndependentReparametrizationSampler.skip
                    IndependentReparametrizationSampler.skip = skip + self._sample_size
                self._eps = np.ascontiguousarray(qmc_normal_samples(self._sample_size, batch_size, skip).T)
            else:
                self._eps = self._rng.standard_normal((batch_size, self._sample_size))
            self._initialized = True
        if self._eps.shape[0] != batch_size:
            raise ValueError(
                f"{type(self).__name__} requires a fixed batch size. Got batch size {batch_size} but previous "
                f"batch size was {self._eps.shape[0]}."
            )
        return self._eps

    def sample(self, at, *, jitter: float = JITTER):
        """at [..., B, D] -> [..., S, B, 1]."""
        if np.ndim(at) < 2:
            raise ValueError("at must have rank >= 2")
        if jitter < 0:
            raise ValueError(f"jitter must be non-negative, got {jitter}")
        eps = self._get_eps(int(np.shape(at)[-2]))
        return _reparam_sample(self._model, at, eps, jitter)

    def reset_sampler(self) -> None:
        self._initialized = False


# ---------------------------------------------------------------------------------------------------
# Random Fourier features (sampler.py:452-591, 741-806, 858-953)
# ---------------------------------------------------------------------------------------------------
def top_k(values, k: int, device: Optional[int] = None):
    """tf.math.top_k over a 1-D score vector (values desc, ties -> lower index): returns
    (top_values [k], top_indices [k]); NumPy in -> NumPy out, torch.cuda in -> torch.cuda out.  ``device``: the GPU that sorts a
    host vector — default: the process's current CUDA device (one process per GPU: the rank's own)."""
    v, pv = _lib.as_f64_contiguous(values)
    if v.ndim != 1:
        raise ValueError(f"values must be 1-D, got shape {tuple(v.shape)}")
    M = int(v.shape[0])
    if M == 0 or k <= 0:
        raise ValueError("top_k needs a non-empty input and k >= 1")
    k = min(int(k), M)
    tv, ptv = _lib.empty_like_kind(v, (k,))
    ti, pti = _lib.empty_like_kind(v, (k,), dtype=np.int64)
    if _lib.is_torch(v):
        device = v.device.index or 0
    elif device is None:
        import torch

        device = torch.cuda.current_device() if torch.cuda.is_available() else 0
    _lib.check(_lib.lib().tb_topk(device, _lib.TB_F64, pv, M, k, ptv, C.cast(pti, C.POINTER(C.c_int64))))
    return tv, ti


class ResampleableRandomFourierFeatureFunctions:
    """sampler.py:741-806 on top of gpflux ``RandomFourierFeaturesCosine``:
    phi(x) = sqrt(2 variance / F) cos((x / l) W^T + b); W ~ N(0, I) for RBF, multivariate Student-t
    (nu = 2p + 1) for Matern-p/2; b ~ U[0, 2 pi).  ``resample`` redraws both in place."""

    def __init__(self, model: GaussianProcessRegression, n_components: int, seed: Optional[int] = None):
        for name in ("get_kernel", "get_observation_noise", "get_internal_data"):
            if not hasattr(model, name):
                raise NotImplementedError(
                    "ResampleableRandomFourierFeatureFunctions only work with models that support "
                    f"get_kernel, get_observation_noise and get_internal_data; but received {model!r}."
                )
        if n_components <= 0:
            raise ValueError("n_components must be positive")
        self._model = model
        self.n_components = int(n_components)
        self._rng = np.random.default_rng(seed)
        self.W: np.ndarray = np.empty((0, 0))
        self.b: np.ndarray = np.empty((0,))
        self.resample()

    def set_weights(self, W: np.ndarray, b: np.ndarray) -> None:
        """Inject W [F, D], b [F] (RNG streams of the reference cannot be reproduced bit-for-bit)."""
        self.W = np.ascontiguousarray(W, dtype=np.float64)
        self.b = np.ascontiguousarray(b, dtype=np.float64)

    def resample(self) -> None:
        kernel = self._model.get_kernel()
        D = self._model.get_internal_data().query_points.shape[-1]
        F = self.n_components
        W = self._rng.standard_normal((F, D))
        if kernel.kind != "rbf":
            nu = {"matern12": 1.0, "matern32": 3.0, "matern52": 5.0}[kernel.kind]
            W = W / np.sqrt(self._rng.chisquare(nu, size=(F, 1)) / nu)
        self.W = W
        self.b = self._rng.uniform(0.0, 2.0 * math.pi, size=(F,))

    def __call__(self, X) -> np.ndarray:
        """Feature matrix phi(X) [n, F] — only ever needed at the n training inputs (theta posterior,
        once per trajectory); evaluated on the GPU through torch (plumbing: dense matmul + cos)."""
        import torch

        k = self._model.get_kernel()
        dev = torch.device("cuda", self._model.device)
        x = torch.as_tensor(np.asarray(X, dtype=np.float64), device=dev) / torch.as_tensor(
            np.broadcast_to(k.lengthscales, (np.shape(X)[-1],)).copy(), device=dev
        )
        W = torch.as_tensor(self.W, device=dev)
        b = torch.as_tensor(self.b, device=dev)
        return math.sqrt(2.0 * k.variance / self.n_components) * torch.cos(x @ W.T + b)


class feature_decomposition_trajectory:
    """sampler.py:858-953: f(x) = phi(x) . theta + m(x) for a batch of B trajectories (B fixed by the
    first call); ``[N, B, D] -> [N, B, 1]``.  The cos-feature projection runs in one CUDA kernel
    that never materialises the [N*B, F] feature matrix; for B > 1 each point is evaluated under its own trajectory only
    (``tb_rff_eval_paired``), which also gives ``value_and_gradient`` and the device L-BFGS of ``minimize_from``."""

    def __init__(self, feature_functions: ResampleableRandomFourierFeatureFunctions, weight_sampler, model):
        self._feature_functions = feature_functions
        self._weight_sampler = weight_sampler
        self._model = model
        self._initialized = False
        self._batch_size = 0
        self._weights_sample: Optional[np.ndarray] = None  # [B, F]
        h = C.c_void_p()
        _lib.check(_lib.lib().tb_rff_create(C.byref(h), model.device))
        self._h = h
        self._push_features()

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            try:
                _lib.lib().tb_rff_destroy(h)
            except Exception:  # pragma: no cover
                pass
            self._h = None

    def _push_features(self) -> None:
        ff = self._feature_functions
        k = self._model.get_kernel()
        D = ff.W.shape[1]
        ls = np.ascontiguousarray(np.broadcast_to(k.lengthscales, (D,)), dtype=np.float64)
        dp = C.POINTER(C.c_double)
        _lib.check(
            _lib.lib().tb_rff_set(
                self._h, ff.W.ctypes.data_as(dp), ff.b.ctypes.data_as(dp), ff.W.shape[0], D, ls.ctypes.data_as(dp),
                k.variance, self._model.get_mean_function().c,
            )
        )

    def _push_theta(self) -> None:
        th = np.ascontiguousarray(self._weights_sample, dtype=np.float64)
        _lib.check(_lib.lib().tb_rff_set_theta(self._h, th.ctypes.data_as(C.POINTER(C.c_double)), th.shape[0]))

    def _batch(self, x):
        """x [N, B, D] as a contiguous fp64 array; the first call fixes the batch size B and draws the weights."""
        x, _ = _lib.as_f64_contiguous(x)
        if x.ndim != 3:
            raise ValueError(f"trajectory inputs must be [N, B, D], got shape {tuple(x.shape)}")
        B = x.shape[1]
        if not self._initialized:
            self._batch_size = B
            self.resample()
            self._initialized = True
        if B != self._batch_size:
            raise ValueError(
                f"This trajectory only supports batch sizes of {self._batch_size}. If you wish to change the batch "
                "size you must get a new trajectory by calling the get_trajectory method of the trajectory sampler."
            )
        return x

    def __call__(self, x):
        x = self._batch(x)
        N, B, D = x.shape
        if B == 1:
            flat = x.reshape(N, D)
            out, po = _lib.empty_like_kind(flat, (N, 1))
            _lib.check(_lib.lib().tb_rff_eval(self._h, _ptr(flat), N, po, None, None))
            return out.reshape(N, 1, 1)
        # B > 1: point (n, b) under trajectory b only, one paired launch per chunk
        out, po = _lib.empty_like_kind(x, (N, B, 1))
        _lib.check(_lib.lib().tb_rff_eval_paired(self._h, _ptr(x), N, B, po, None))
        return out

    def value_and_gradient(self, x):
        """x [N, B, D] -> (f_b(x_nb) [N, B, 1], grad_x f_b(x_nb) [N, B, D]): each point under its own trajectory."""
        x = self._batch(x)
        N, B, D = x.shape
        out, po = _lib.empty_like_kind(x, (N, B, 1))
        grad, pg = _lib.empty_like_kind(x, (N, B, D))
        _lib.check(_lib.lib().tb_rff_eval_paired(self._h, _ptr(x), N, B, po, pg))
        return out, grad

    def minimize_from(self, starts, lower, upper, *, maxcor: int = 10, maxiter: int = 15000, maxls: int = 20,
                      gtol: float = 1e-5, ftol: float = 2.220446049250313e-09):
        """Device-side multi-start projected L-BFGS (``tb_rff_maximize_boxes`` on -f_b): start (i, b) of ``starts``
        [R, B, D] minimises trajectory b inside its box, with SciPy's option names and defaults.  ``lower`` / ``upper`` are
        one box [D] or ``nbox`` boxes [nbox, D] with nbox dividing B; column b uses box ``b % nbox`` (the round robin of a
        multi-region search space).  Returns (success [R, B] bool, f_b at the end points [R, B], x [R, B, D], nfev [R, B]).
        The negated trajectory of the continuous Thompson-sampling builders offers it as ``maximize_from``."""
        x0 = starts.detach().cpu().numpy() if hasattr(starts, "detach") else starts
        x0 = np.ascontiguousarray(x0, dtype=np.float64)
        if x0.ndim != 3:
            raise ValueError(f"starts must be [R, B, D], got {x0.shape}")
        self._batch(x0[:1])
        R, B, D = x0.shape
        lo, up = (np.atleast_2d(np.asarray(v, dtype=np.float64)) for v in (lower, upper))
        nbox = max(lo.shape[0], up.shape[0])
        lo = np.ascontiguousarray(np.broadcast_to(lo, (nbox, D)))
        up = np.ascontiguousarray(np.broadcast_to(up, (nbox, D)))
        x = np.empty((R, B, D))
        f = np.empty((R, B))
        ok = np.zeros((R, B), dtype=np.int32)
        nfev = np.zeros((R, B), dtype=np.int64)
        _lib.check(
            _lib.lib().tb_rff_maximize_boxes(
                self._h, lo.ctypes.data, up.ctypes.data, nbox, x0.ctypes.data, R, int(maxcor), int(maxiter), int(maxls),
                float(gtol), float(ftol), x.ctypes.data, f.ctypes.data, ok.ctypes.data, nfev.ctypes.data,
            )
        )
        return ok.astype(bool), -f, x, nfev

    def argmin_over(self, candidates):
        """Fused evaluate + argmin of every trajectory over one shared candidate set [M, D]:
        returns (min_values [B], min_indices [B]) without writing the [M, B] values
        (ThompsonSamplerFromTrajectory, acquisition/sampler.py:262-271)."""
        pts, _ = _lib.as_f64_contiguous(candidates)
        if pts.ndim != 2:
            raise ValueError(f"candidates must be [M, D], got {tuple(pts.shape)}")
        if not self._initialized:
            self._batch_size = 1
            self.resample()
            self._initialized = True
        B = self._batch_size
        mv = np.empty(B, dtype=np.float64)
        mi = np.empty(B, dtype=np.int64)
        _lib.check(
            _lib.lib().tb_rff_eval(
                self._h, _ptr(pts), pts.shape[0], None, mv.ctypes.data_as(C.POINTER(C.c_double)),
                mi.ctypes.data_as(C.POINTER(C.c_int64)),
            )
        )
        return mv, mi

    def resample(self) -> None:
        self._weights_sample = np.asarray(self._weight_sampler(self._batch_size))[..., 0]  # [B, F]
        self._push_theta()

    def update(self, weight_sampler) -> None:
        self._weight_sampler = weight_sampler
        self._push_features()
        self.resample()


class RandomFourierFeatureTrajectorySampler:
    """sampler.py:452-591: theta posterior in design space when F < n (:529-557), gram space
    otherwise (:559-591); ``get_trajectory`` / ``resample_trajectory`` / ``update_trajectory``
    (sampler.py:386-450).  The once-per-trajectory O(min(n,F)^3) linear algebra runs on the GPU
    through torch's cuSOLVER/cuBLAS bindings (library calls off the per-candidate path)."""

    def __init__(self, model: GaussianProcessRegression, num_features: int = 1000, seed: Optional[int] = None):
        for name in ("get_kernel", "get_observation_noise", "get_internal_data"):
            if not hasattr(model, name):
                raise NotImplementedError(
                    "RandomFourierFeatureTrajectorySampler only works with models with get_kernel, "
                    f"get_observation_noise and get_internal_data methods; but received {model!r}."
                )
        if num_features <= 0:
            raise ValueError("num_features must be positive")
        if len(model.get_internal_data()) == 0:
            raise ValueError("Dataset must be populated.")
        self._model = model
        self._num_features = num_features
        self._rng = np.random.default_rng(seed)
        self._feature_functions = ResampleableRandomFourierFeatureFunctions(model, num_features, seed=None if seed is None else seed + 1)
        self._weight_sampler = None

    def __repr__(self) -> str:
        return f"{type(self).__name__}({self._model!r}, {self._num_features!r})"

    def theta_posterior(self):
        """(mean [F], chol_cov [F, F]) as torch.cuda float64 tensors."""
        import torch

        data = self._model.get_internal_data()
        n = len(data)
        dev = torch.device("cuda", self._model.device)
        phi = self._feature_functions(data.query_points)  # [n, F] cuda
        noise = self._model.get_observation_noise()
        resid = torch.as_tensor(
            np.asarray(data.observations, dtype=np.float64) - self._model.get_mean_function()(data.query_points), device=dev
        )
        F = self._num_features
        eye = lambda m: torch.eye(m, dtype=torch.float64, device=dev)  # noqa: E731
        if F < n:  # design space (sampler.py:529-557)
            Dm = phi.T @ phi + noise * eye(F)
            L = torch.linalg.cholesky(Dm)
            D_inv = torch.cholesky_solve(eye(F), L)
            mean = (D_inv @ (phi.T @ resid))[:, 0]
            chol_cov = torch.linalg.cholesky(D_inv * noise)
        else:  # gram space (sampler.py:559-591)
            G = phi @ phi.T + noise * eye(n)
            L = torch.linalg.cholesky(G)
            L_inv_phi = torch.linalg.solve_triangular(L, phi, upper=False)
            L_inv_y = torch.linalg.solve_triangular(L, resid, upper=False)
            mean = (L_inv_phi.T @ L_inv_y)[:, 0]
            cov = eye(F) - L_inv_phi.T @ L_inv_phi
            chol_cov = torch.linalg.cholesky(cov)
        return mean, chol_cov

    def _prepare_weight_sampler(self):
        import torch

        mean, chol = self.theta_posterior()

        def sample(b: int) -> np.ndarray:  # [B] -> [B, F, 1]
            z = torch.as_tensor(self._rng.standard_normal((b, mean.shape[0])), device=mean.device)
            return (mean[None, :] + z @ chol.T).cpu().numpy()[..., None]

        return sample

    def get_trajectory(self) -> feature_decomposition_trajectory:
        self._weight_sampler = self._prepare_weight_sampler()
        return feature_decomposition_trajectory(self._feature_functions, self._weight_sampler, self._model)

    def resample_trajectory(self, trajectory: feature_decomposition_trajectory) -> feature_decomposition_trajectory:
        if not isinstance(trajectory, feature_decomposition_trajectory):
            raise ValueError("trajectory must be a feature_decomposition_trajectory")
        trajectory.resample()
        return trajectory

    def update_trajectory(self, trajectory: feature_decomposition_trajectory) -> feature_decomposition_trajectory:
        if not isinstance(trajectory, feature_decomposition_trajectory):
            raise ValueError("trajectory must be a feature_decomposition_trajectory")
        self._feature_functions.resample()
        self._weight_sampler = self._prepare_weight_sampler()
        trajectory.update(self._weight_sampler)
        return trajectory


# ---------------------------------------------------------------------------------------------------
# Decoupled (pathwise) sampling (sampler.py:594-738, 809-855) — the reference's default for GPR
# (models.py:342-345): f(x) = phi(x) w + sum_j v_j k(x, x_j) + m(x)
# ---------------------------------------------------------------------------------------------------
class decoupled_trajectory(feature_decomposition_trajectory):
    """``feature_decomposition_trajectory`` over F RFF features + N canonical features ``k(., x_j)``; the weight
    sampler returns ``(w [B, F], v [B, N])``."""

    def resample(self) -> None:
        w, v = self._weight_sampler(self._batch_size)
        self._weights_sample = np.ascontiguousarray(w, dtype=np.float64)
        self._canonical_weights = np.ascontiguousarray(v, dtype=np.float64)
        self._push_theta()
        data = self._model.get_internal_data()
        X = np.ascontiguousarray(np.asarray(data.query_points, dtype=np.float64))
        dp = C.POINTER(C.c_double)
        _lib.check(
            _lib.lib().tb_rff_set_canonical(
                self._h, _lib.KERNEL_IDS[self._model.get_kernel().kind], X.ctypes.data_as(dp), X.shape[0],
                self._canonical_weights.ctypes.data, self._canonical_weights.shape[0],
            )
        )


class DecoupledTrajectorySampler:
    """sampler.py:594-738 (exact-GP branch :668-677): prior part through RFF weights ``w ~ N(0, I)``, data
    update through canonical weights ``v = (K + noise I)^-1 (y - m + sqrt(noise) eps - phi(X) w)`` — the solve
    reuses the model's cached Cholesky factor on the GPU (``tb_gp_kinv_apply``)."""

    def __init__(self, model: GaussianProcessRegression, num_features: int = 1000, seed: Optional[int] = None):
        for name in ("get_kernel", "get_observation_noise", "get_internal_data"):
            if not hasattr(model, name):
                raise NotImplementedError(
                    "DecoupledTrajectorySampler only works with models that either support get_kernel, "
                    f"get_observation_noise and get_internal_data or support get_kernel and get_inducing_variables; but received {model!r}."
                )
        if num_features <= 0:
            raise ValueError("num_features must be positive")
        if len(model.get_internal_data()) == 0:
            raise ValueError("Dataset must be populated.")
        self._model = model
        self._num_features = num_features
        self._rng = np.random.default_rng(seed)
        self._feature_functions = ResampleableRandomFourierFeatureFunctions(model, num_features, seed=None if seed is None else seed + 1)
        self._weight_sampler = None

    def __repr__(self) -> str:
        return f"{type(self).__name__}({self._model!r}, {self._num_features!r})"

    def canonical_weights(self, prior_w: np.ndarray, eps: np.ndarray) -> np.ndarray:
        """v [B, N] for given prior weights w [B, F] and noise draws eps [B, N]."""
        import torch

        data = self._model.get_internal_data()
        dev = torch.device("cuda", self._model.device)
        phi_Z = self._feature_functions(data.query_points)  # [N, F] on the GPU
        resid = np.asarray(data.observations, dtype=np.float64) - self._model.get_mean_function()(data.query_points)  # [N, 1]
        u = torch.as_tensor(resid[:, 0][None, :] + math.sqrt(self._model.get_observation_noise()) * np.asarray(eps), device=dev)
        diff = (u - torch.as_tensor(np.asarray(prior_w), device=dev) @ phi_Z.T).contiguous()  # [B, N]
        out = torch.empty_like(diff)
        _lib.sync_torch_stream(diff)  # diff was produced on torch's stream; the library reads it on the handle's stream
        _lib.check(_lib.lib().tb_gp_kinv_apply(self._model.handle, diff.data_ptr(), diff.shape[0], out.data_ptr()))
        return out.cpu().numpy()

    def _prepare_weight_sampler(self):
        n = len(self._model.get_internal_data())

        def sample(b: int):
            w = self._rng.standard_normal((b, self._num_features))
            eps = self._rng.standard_normal((b, n))
            return w, self.canonical_weights(w, eps)

        return sample

    def get_trajectory(self) -> decoupled_trajectory:
        self._weight_sampler = self._prepare_weight_sampler()
        return decoupled_trajectory(self._feature_functions, self._weight_sampler, self._model)

    def resample_trajectory(self, trajectory: decoupled_trajectory) -> decoupled_trajectory:
        if not isinstance(trajectory, decoupled_trajectory):
            raise ValueError("trajectory must be a decoupled_trajectory")
        trajectory.resample()
        return trajectory

    def update_trajectory(self, trajectory: decoupled_trajectory) -> decoupled_trajectory:
        if not isinstance(trajectory, decoupled_trajectory):
            raise ValueError("trajectory must be a decoupled_trajectory")
        self._feature_functions.resample()
        self._weight_sampler = self._prepare_weight_sampler()
        trajectory.update(self._weight_sampler)
        return trajectory
