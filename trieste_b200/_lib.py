"""ctypes binding of the C-ABI in ``include/trieste_b200.h``.

The product path has NO CPU fallback: if the CUDA extension is missing or no H100 is visible the
calls below raise.  (The library itself loads on a CPU-only box so that the symbol table can be
checked by the ``-m "not gpu"`` tests.)
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libtrieste_b200.so")

TB_F64, TB_F32 = 0, 1
KERNEL_IDS = {"rbf": 0, "matern12": 1, "matern32": 2, "matern52": 3}
ACQ_EI, ACQ_LOG_EI, ACQ_NEG_LCB, ACQ_LCB, ACQ_PBT, ACQ_AEI, ACQ_MES = 0, 1, 2, 3, 4, 5, 6
ACQ_GIBBON_QUALITY, ACQ_GIBBON_REPULSION, ACQ_GIBBON = 7, 8, 9
ACQ_FEASIBILITY_BICHON, ACQ_FEASIBILITY_RANJAN, ACQ_BALD, ACQ_PREDICTIVE_VARIANCE = 10, 11, 12, 13
ACQ_PENALIZED = 0x100  # OR-ed into the acquisition kind: multiply by the handle's local penalty
PEN_SOFT, PEN_HARD = 1, 2

_lib: Optional[C.CDLL] = None

# name -> (restype, argtypes); mirrors include/trieste_b200.h one to one
_vp, _i64, _i32, _f64 = C.c_void_p, C.c_int64, C.c_int, C.c_double
SIGNATURES = {
    "tb_last_error": (C.c_char_p, []),
    "tb_version": (C.c_char_p, []),
    "tb_device_count": (_i32, [C.POINTER(_i32)]),
    "tb_gp_create": (_i32, [C.POINTER(_vp), _i32, _i32]),
    "tb_gp_destroy": (_i32, [_vp]),
    "tb_gp_set_data": (_i32, [_vp, _vp, _vp, _i64, _i32]),
    "tb_gp_set_hyper": (_i32, [_vp, _i32, _f64, C.POINTER(_f64), _i32, _f64, _f64]),
    "tb_gp_update_posterior_cache": (_i32, [_vp]),
    "tb_gp_append_data": (_i32, [_vp, _vp, _vp, _i64]),
    "tb_gp_get_cholesky": (_i32, [_vp, _vp]),
    "tb_gp_predict": (_i32, [_vp, _vp, _i64, _vp, _vp]),
    "tb_gp_predict_joint": (_i32, [_vp, _vp, _i64, _i32, _vp, _vp]),
    "tb_acq_eval": (_i32, [_vp, _i32, _f64, _vp, _i64, _vp, _vp]),
    "tb_acq_argmax": (_i32, [_vp, _i32, _f64, _vp, _i64, _vp, _vp, C.POINTER(_i64)]),
    "tb_acq_set_min_value_samples": (_i32, [_vp, C.POINTER(_f64), _i32]),
    "tb_acq_set_penalization": (_i32, [_vp, _i32, _vp, _i32, _vp, _vp]),
    "tb_acq_set_gibbon_repulsion": (_i32, [_vp, _vp, _i32, _f64]),
    "tb_acq_set_feasibility": (_i32, [_vp, _f64]),
    "tb_gp_mean_gradient": (_i32, [_vp, _vp, _i64, _vp, _vp]),
    "tb_acq_maximize": (_i32, [_vp, _i32, _f64, _vp, _vp, _vp, _i64, _i32, _i32, _i32, _f64, _f64, _vp, _vp, _vp, _vp]),
    "tb_acq_batch_mc_ei": (_i32, [_vp, _vp, _i64, _i32, _vp, _i32, _f64, _f64, _vp]),
    "tb_acq_batch_mc_ei_grad": (_i32, [_vp, _vp, _i64, _i32, _vp, _i32, _f64, _f64, _vp, _vp]),
    "tb_acq_batch_ei": (_i32, [_vp, _vp, _i64, _i32, _vp, _i32, _f64, _vp]),
    "tb_acq_batch_ei_grad": (_i32, [_vp, _vp, _i64, _i32, _vp, _i32, _f64, _vp, _vp]),
    "tb_acq_predictive_variance": (_i32, [_vp, _vp, _i64, _i32, _f64, _vp, _vp]),
    "tb_mvn_cdf": (_i32, [_i32, _vp, _vp, _vp, _i64, _i32, _vp, _i32, _f64, _vp]),
    "tb_gp_covariance_between_points": (_i32, [_vp, _vp, _i64, _vp, _i64, _vp]),
    "tb_gp_sample_joint": (_i32, [_vp, _vp, _i64, _vp, _i32, _f64, _vp]),
    "tb_gp_reparam_sample": (_i32, [_vp, _vp, _i64, _i32, _vp, _i32, _f64, _vp]),
    "tb_topk": (_i32, [_i32, _i32, _vp, _i64, _i32, _vp, C.POINTER(_i64)]),
    "tb_rff_create": (_i32, [C.POINTER(_vp), _i32]),
    "tb_rff_destroy": (_i32, [_vp]),
    "tb_rff_set": (_i32, [_vp, C.POINTER(_f64), C.POINTER(_f64), _i32, _i32, C.POINTER(_f64), _f64, _f64]),
    "tb_rff_set_theta": (_i32, [_vp, C.POINTER(_f64), _i32]),
    "tb_rff_eval": (_i32, [_vp, _vp, _i64, _vp, C.POINTER(_f64), C.POINTER(_i64)]),
    "tb_rff_set_canonical": (_i32, [_vp, _i32, C.POINTER(_f64), _i64, _vp, _i32]),
    "tb_rff_eval_paired": (_i32, [_vp, _vp, _i64, _i32, _vp, _vp]),
    "tb_rff_maximize": (_i32, [_vp, _vp, _vp, _vp, _i64, _i32, _i32, _i32, _f64, _f64, _vp, _vp, _vp, _vp]),
    "tb_rff_maximize_boxes": (_i32, [_vp, _vp, _vp, _i32, _vp, _i64, _i32, _i32, _i32, _f64, _f64, _vp, _vp, _vp, _vp]),
    "tb_acq_maximize_models": (_i32, [_vp, _vp, _vp, _i32, _vp, _vp, _vp, _i64, _i32, _i32, _i32, _f64, _f64, _vp, _vp, _vp, _vp]),
    "tb_rff_maximize_models": (_i32, [_vp, _i32, _vp, _vp, _vp, _i64, _i32, _i32, _i32, _f64, _f64, _vp, _vp, _vp, _vp]),
    "tb_ehvi_create": (_i32, [C.POINTER(_vp), C.POINTER(_vp), _i32]),
    "tb_ehvi_destroy": (_i32, [_vp]),
    "tb_ehvi_set_cells": (_i32, [_vp, _vp, _vp, _i64]),
    "tb_ehvi_set_penalty": (_i32, [_vp, _vp, _vp, _i32]),
    "tb_ehvi_eval": (_i32, [_vp, _vp, _i64, _vp, _vp]),
    "tb_ehvi_argmax": (_i32, [_vp, _vp, _i64, _vp, _vp, C.POINTER(_i64)]),
    "tb_ehvi_maximize": (_i32, [_vp, _vp, _vp, _vp, _i64, _i32, _i32, _i32, _f64, _f64, _vp, _vp, _vp, _vp]),
    "tb_reduce_create": (_i32, [C.POINTER(_vp), C.POINTER(_vp), _i32]),
    "tb_reduce_destroy": (_i32, [_vp]),
    "tb_reduce_set_terms": (_i32, [_vp, _i32, _i32, _vp, _vp, _vp, _vp]),
    "tb_reduce_eval": (_i32, [_vp, _vp, _i64, _vp, _vp]),
    "tb_reduce_argmax": (_i32, [_vp, _vp, _i64, _vp, _vp, C.POINTER(_i64)]),
    "tb_reduce_maximize": (_i32, [_vp, _vp, _vp, _vp, _i64, _i32, _i32, _i32, _f64, _f64, _vp, _vp, _vp, _vp]),
    "tb_gp_kinv_apply": (_i32, [_vp, _vp, _i32, _vp]),
    "tb_launch_count": (_i64, []),
    "tb_launch_count_reset": (None, []),
    "tb_gp_set_engine": (_i32, [_vp, _i32]),
    "tb_gp_engine_info": (_i32, [_vp, C.POINTER(_i32), C.POINTER(_f64)]),
    "tb_gp_mean_bounds": (_i32, [_vp, _vp, _i64, _vp, _vp]),
    "tb_gp_profile": (_i32, [_vp, _i32]),
    "tb_gp_stream": (_i32, [_vp, C.POINTER(_vp)]),
    "tb_gp_profile_read": (_i32, [_vp, C.POINTER(_f64), C.POINTER(_i64), C.POINTER(_f64)]),
}


class NativeLibraryError(RuntimeError):
    """The CUDA extension is missing or unusable (there is no CPU fallback)."""


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise NativeLibraryError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(trieste_b200 has no CPU fallback)"
            )
        try:
            handle = C.CDLL(LIB_PATH)
        except OSError as e:  # pragma: no cover
            raise NativeLibraryError(f"cannot load {LIB_PATH}: {e}") from e
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def last_error() -> str:
    return lib().tb_last_error().decode("utf-8", "replace")


# enum tb_status (include/trieste_b200.h)
TB_OK, TB_ERR_INVALID, TB_ERR_RUNTIME, TB_ERR_NUMERIC = 0, 1, 2, 3


def check(status: int, exc=ValueError) -> None:
    """Non-zero status -> Python exception carrying the C side's message, chosen by the status CODE: invalid arguments
    and failed factorisations raise ``exc`` (ValueError: the reference raises ValueError / InvalidArgumentError for the
    same conditions), CUDA / library failures raise NativeLibraryError (there is nothing to fall back to)."""
    if status == TB_OK:
        return
    msg = last_error()
    if status == TB_ERR_RUNTIME:
        raise NativeLibraryError(msg)
    raise exc(msg)


def sync_torch_stream(x) -> None:
    """Order the library's (non-blocking) stream after torch's current stream.  The ABI reads device pointers on the
    handle's own stream, so everything torch has queued on its stream — the producer of a tensor passed in, or a
    pending reader of a caching-allocator block about to be handed out as an output — must have finished first.  The
    ABI returns only after its stream has drained, so nothing is needed on the way out."""
    import torch

    torch.cuda.current_stream(x.device).synchronize()


def device_count() -> int:
    n = _i32(0)
    if lib().tb_device_count(C.byref(n)) != 0:
        return 0
    return n.value


def require_gpu() -> None:
    if device_count() <= 0:
        raise NativeLibraryError(
            "no CUDA device visible: trieste_b200 runs only on an H100 (sm_90a); there is no CPU fallback"
        )


# ---- array plumbing: numpy (host) or torch.cuda tensors (device) cross the ABI as raw pointers ----
def is_torch(x) -> bool:
    return type(x).__module__.split(".")[0] == "torch"


def as_contiguous(x, dtype=np.float64):
    """Return (array_like, pointer) in ``dtype`` (np.float64 / np.float32).  numpy in -> numpy
    C-contiguous; torch.cuda in -> contiguous device tensor (zero-copy when already conforming)."""
    if is_torch(x):
        import torch

        tdt = torch.float64 if dtype == np.float64 else torch.float32
        t = x.detach()
        if t.dtype != tdt:
            t = t.to(tdt)
        t = t.contiguous()
        if t.is_cuda:
            sync_torch_stream(t)
        return t, t.data_ptr()
    a = np.ascontiguousarray(np.asarray(x, dtype=dtype))
    return a, a.ctypes.data


def as_f64_contiguous(x):
    return as_contiguous(x, np.float64)


def empty_like_kind(ref, shape, dtype=np.float64):
    """Allocate an output of the same kind (numpy / torch device) as ``ref``."""
    if is_torch(ref):
        import torch

        tdt = {np.float64: torch.float64, np.float32: torch.float32, np.int64: torch.int64}[dtype]
        t = torch.empty(shape, dtype=tdt, device=ref.device)
        if t.is_cuda:
            sync_torch_stream(t)
        return t, t.data_ptr()
    a = np.empty(shape, dtype=dtype)
    return a, a.ctypes.data
