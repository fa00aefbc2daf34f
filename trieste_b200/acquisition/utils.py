"""``split_acquisition_function`` / ``split_acquisition_function_calls`` / ``select_nth_output`` and the local-model helpers
``copy_to_local_models`` / ``with_local_datasets`` — mirrors trieste/acquisition/utils.py:31-204 — and
``MultivariateNormalCDF`` (acquisition/function/utils.py:29-199).

In the reference these wrappers bound the memory of one TensorFlow evaluation by cutting the leading (candidate) axis into
blocks.  Here the fused kernels already stream any batch through bounded scratch (``run_eval`` chunks at
~1 GB of K* scratch), so the wrappers are not needed for memory; they exist so that callers which wrap their functions or
optimisers keep working, with the reference's splitting rule and error behaviour."""
from __future__ import annotations

import copy
import functools
import math

import numpy as np

from .interface import OBJECTIVE


def _concat(parts):
    if type(parts[0]).__module__.split(".")[0] == "torch":
        import torch

        return torch.cat(parts, dim=0)
    return np.concatenate([np.asarray(p) for p in parts], axis=0)


def split_acquisition_function(fn, split_size: int):
    """utils.py:31-84: call ``fn`` on blocks of at most ``split_size`` ELEMENTS of ``x`` along its first axis and stitch the
    results back together."""
    if split_size <= 0:
        raise ValueError(f"split_size must be positive, got {split_size}")

    @functools.wraps(fn, updated=())
    def wrapper(x):
        x = x if hasattr(x, "shape") else np.asarray(x)
        length = x.shape[0]
        if length == 0:
            return fn(x)
        elements_per_block = int(np.prod(x.shape)) / length
        blocks_per_batch = int(math.ceil(split_size / elements_per_block))
        if length <= blocks_per_batch:
            return fn(x)
        return _concat([fn(x[i : i + blocks_per_batch]) for i in range(0, length, blocks_per_batch)])

    # the fused entry points pass straight through: they never materialise more than one bounded chunk
    for name in ("value_and_gradient", "fused_argmax", "maximize_from"):
        if hasattr(fn, name):
            setattr(wrapper, name, getattr(fn, name))
    return wrapper


def split_acquisition_function_calls(optimizer, split_size: int):
    """utils.py:87-109: an optimiser whose acquisition-function evaluations are split as above."""
    if split_size <= 0:
        raise ValueError(f"split_size must be positive, got {split_size}")

    def split_optimizer(search_space, f):
        af, n = f if isinstance(f, tuple) else (f, 1)
        taf = split_acquisition_function(af, split_size)
        return optimizer(search_space, (taf, n) if isinstance(f, tuple) else taf)

    return split_optimizer


def copy_to_local_models(global_model, num_local_models: int, key=OBJECTIVE):
    """utils.py:146-160: ``num_local_models`` deep copies of ``global_model`` under ``LocalizedTag(key, i)``.  A copy of a
    ``GaussianProcessRegression`` owns its own device handle, data and posterior cache."""
    from ..utils import LocalizedTag

    return {LocalizedTag(key, i): copy.deepcopy(global_model) for i in range(num_local_models)}


def with_local_datasets(datasets, num_local_datasets: int, local_dataset_indices=None):
    """utils.py:163-204: ``datasets`` plus, for every global tag without them, ``num_local_datasets`` local datasets under
    ``LocalizedTag(tag, i)``: the whole global dataset, or its rows ``local_dataset_indices[i]``."""
    from ..data import Dataset
    from ..utils import LocalizedTag

    if local_dataset_indices is not None and len(local_dataset_indices) != num_local_datasets:
        raise ValueError(
            f"local_dataset_indices should have {num_local_datasets} entries, has {len(local_dataset_indices)}"
        )
    updated_datasets = {}
    for tag in datasets:
        updated_datasets[tag] = datasets[tag]
        ltag = LocalizedTag.from_tag(tag)
        if not ltag.is_local:
            for i in range(num_local_datasets):
                target_ltag = LocalizedTag(ltag.global_tag, i)
                if target_ltag not in datasets:
                    if local_dataset_indices is None:
                        updated_datasets[target_ltag] = datasets[tag]
                    else:
                        rows = np.asarray(local_dataset_indices[i], dtype=np.int64)
                        updated_datasets[target_ltag] = Dataset(
                            np.asarray(datasets[tag].query_points)[rows], np.asarray(datasets[tag].observations)[rows]
                        )
    return updated_datasets


def select_nth_output(x, output_dim: int = 0):
    """utils.py:112-123: the ``output_dim``-th output of ``x`` [..., B, L] as the trajectory, shape [..., B]."""
    return x[..., output_dim]


class MultivariateNormalCDF:
    """acquisition/function/utils.py:29-199: the CDF of a multivariate Gaussian by Genz's QMC recursion over
    ``sample_size`` Sobol points (``skip = num_sobol_skip``), evaluated on the device (``tb_mvn_cdf``, fp64; results are
    returned in ``dtype``).  The points are drawn once, on construction."""

    def __init__(self, sample_size: int, dim: int, dtype=np.float64, num_sobol_skip: int = 0):
        if sample_size <= 0:
            raise ValueError(f"sample_size must be positive, got {sample_size}")
        if dim <= 0:
            raise ValueError(f"dim must be positive, got {dim}")
        from ..sampler import sobol_points

        self._S = int(sample_size)
        self._Q = int(dim)
        self._dtype = np.dtype(dtype)
        self._num_sobol_skip = int(num_sobol_skip)
        # [Q-1, S] column-contiguous; column j of the Sobol sequence is the same in every dimension
        self._w = np.ascontiguousarray(sobol_points(self._S, self._Q - 1, self._num_sobol_skip).T)

    def __call__(self, x, mean, cov, jitter: float = 1e-6):
        """x, mean [B, Q], cov [B, Q, Q] -> [B]."""
        from .. import _lib

        x, px = _lib.as_contiguous(x)
        mean, pm = _lib.as_contiguous(mean)
        cov, pc = _lib.as_contiguous(cov)
        B = x.shape[0]
        if B <= 0:
            raise ValueError("MultivariateNormalCDF needs at least one row")
        Q = self._Q
        if tuple(x.shape) != (B, Q) or tuple(mean.shape) != (B, Q) or tuple(cov.shape) != (B, Q, Q):
            raise ValueError(f"expected x, mean [B, {Q}] and cov [B, {Q}, {Q}], got {tuple(x.shape)}, "
                             f"{tuple(mean.shape)}, {tuple(cov.shape)}")
        device = (x.device.index or 0) if _lib.is_torch(x) and x.is_cuda else 0
        out, po = _lib.empty_like_kind(x, (B,))
        _lib.check(_lib.lib().tb_mvn_cdf(device, px, pm, pc, B, Q, self._w.ctypes.data if Q > 1 else None, self._S,
                                         float(jitter), po))
        if isinstance(out, np.ndarray):
            return out.astype(self._dtype)
        import torch

        return out.to(torch.float32 if self._dtype == np.float32 else torch.float64)
