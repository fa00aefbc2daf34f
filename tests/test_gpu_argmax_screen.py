"""Screened fused argmax of EI / log-EI (tb_api.cu, argmax_screened) against the unscreened chunk loop: the same index and
the bit-identical value, on every engine mode and data shape the screen touches.  TB_ARGMAX_SCREEN=1 forces the screen
(small M too), =0 turns it off."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest
import torch

from oracle import gp_oracle as o
from tests.util import candidates, model_pair

pytestmark = pytest.mark.gpu

HEADLINE_CHUNK = 50_688  # candidates per chunk of the 15-product engine at N = 4096, D = 10 (264 tiles of 192)


def _argmax(fn, X, mode, monkeypatch):
    monkeypatch.setenv("TB_ARGMAX_SCREEN", str(mode))
    return fn.fused_argmax(X)


def _same(fn, X, monkeypatch):
    """Screened and unscreened argmax agree bit for bit; returns the pair."""
    i0, v0 = _argmax(fn, X, 0, monkeypatch)
    i1, v1 = _argmax(fn, X, 1, monkeypatch)
    assert i1 == i0
    assert np.float64(v1).tobytes() == np.float64(v0).tobytes(), (v1, v0)
    return i0, v0


def _ei(nm, om, log=False):
    from trieste_b200 import Dataset
    from trieste_b200.acquisition import ExpectedImprovement, LogExpectedImprovement

    b = LogExpectedImprovement() if log else ExpectedImprovement()
    return b.prepare_acquisition_function(nm, Dataset(om.X, om.y))


def _dev(X, dtype=torch.float64):
    return torch.as_tensor(np.ascontiguousarray(X), dtype=dtype, device="cuda")


def _gemm_flops(nm, fn, X, mode, monkeypatch):
    from trieste_b200 import _lib

    lib, h = _lib.lib(), nm.handle
    lib.tb_gp_profile(h, 1)
    res = _argmax(fn, X, mode, monkeypatch)
    ms, n, fl = C.c_double(), C.c_int64(), C.c_double()
    lib.tb_gp_profile_read(h, C.byref(ms), C.byref(n), C.byref(fl))
    lib.tb_gp_profile(h, 0)
    return res, fl.value, n.value


@pytest.fixture(scope="module")
def headline():
    om, nm = model_pair(o.ackley, 4096, 10)
    return om, nm, _ei(nm, om)


def test_headline_multi_chunk_partial_last(headline, monkeypatch):
    om, nm, fn = headline
    M = 3 * HEADLINE_CHUNK + 1000
    X = _dev(candidates(M, 10))
    _same(fn, X, monkeypatch)


def test_headline_screen_engages(headline, monkeypatch):
    om, nm, fn = headline
    M = 3 * HEADLINE_CHUNK + 1000
    X = _dev(candidates(M, 10, seed=4))
    N2 = 4096.0**2
    (i0, v0), fl0, n0 = _gemm_flops(nm, fn, X, 0, monkeypatch)
    (i1, v1), fl1, n1 = _gemm_flops(nm, fn, X, 1, monkeypatch)
    assert (i1, v1) == (i0, v0)
    # unscreened: one GEMM per chunk over McPad candidates
    assert n0 == 4
    assert fl0 == (3 * HEADLINE_CHUNK + 1152) * N2
    # screened: the probe and the survivors only
    assert n1 >= 2
    assert fl1 < 0.05 * M * N2


def test_small_m_ksplit_and_group_bump(monkeypatch):
    om, nm = model_pair(o.hartmann_6, 1024, 6)
    fn = _ei(nm, om)
    for M in (3000, 1, 193):
        _same(fn, _dev(candidates(M, 6, seed=M)), monkeypatch)


def test_branin_n20(monkeypatch):
    om, nm = model_pair(o.branin, 20, 2)
    fn = _ei(nm, om)
    _same(fn, _dev(candidates(20000, 2)), monkeypatch)


@pytest.mark.parametrize("kind", ["rbf", "matern12"])
def test_kernels(kind, monkeypatch):
    om, nm = model_pair(o.hartmann_6, 512, 6, kind=kind)
    fn = _ei(nm, om)
    _same(fn, _dev(candidates(40000, 6)), monkeypatch)


def test_fp32_handle(monkeypatch):
    import trieste_b200 as tb
    from trieste_b200.acquisition import ExpectedImprovement

    om = o.synthetic_model(o.hartmann_6, 1024, 6)
    X32, y32 = om.X.astype(np.float32), om.y.astype(np.float32)
    nm = tb.GaussianProcessRegression(tb.GPRSpec((X32, y32), tb.Matern52(om.variance, om.lengthscales), tb.Constant(om.mean_const), om.noise))
    fn = ExpectedImprovement().prepare_acquisition_function(nm, tb.Dataset(X32, y32))
    _same(fn, _dev(candidates(30000, 6), torch.float32), monkeypatch)


def test_int8x21_engine(monkeypatch):
    om, nm = model_pair(o.hartmann_6, 1024, 6, engine="int8x21")
    fn = _ei(nm, om)
    _same(fn, _dev(candidates(30000, 6)), monkeypatch)
    assert nm.engine_info()[0] == 21


def test_log_ei(headline, monkeypatch):
    om, nm, _ = headline
    fn = _ei(nm, om, log=True)
    _same(fn, _dev(candidates(HEADLINE_CHUNK + 777, 10, seed=2)), monkeypatch)


def test_duplicates_first_index_wins(monkeypatch):
    om, nm = model_pair(o.hartmann_6, 1024, 6)
    fn = _ei(nm, om)
    X = candidates(30000, 6, seed=5)
    i, _ = _argmax(fn, _dev(X), 0, monkeypatch)
    j = i // 2
    X[j] = X[i]
    X[-1] = X[i]
    X[(i + j) // 2 + 1] = X[i]
    k, _ = _same(fn, _dev(X), monkeypatch)
    assert k == j


def test_nan_coordinates(monkeypatch):
    om, nm = model_pair(o.hartmann_6, 1024, 6)
    fn = _ei(nm, om)
    X = candidates(30000, 6, seed=6)
    X[::7, 3] = np.nan
    X[0] = np.nan
    _same(fn, _dev(X), monkeypatch)
    Xn = np.full((5000, 6), np.nan)
    for mode in (0, 1):
        i, v = _argmax(fn, _dev(Xn), mode, monkeypatch)
        assert i == 0 and np.isnan(v)


def test_adversarial_falls_back(headline, monkeypatch):
    """eta far above every mean: ub - tau is below the margin for every candidate, nothing is pruned, and the call runs
    the unscreened loop after the mean pass and the probe."""
    from trieste_b200.acquisition.function import expected_improvement

    om, nm, _ = headline
    fn = expected_improvement(nm, 1e8)
    M = HEADLINE_CHUNK + 5000
    X = _dev(candidates(M, 10, seed=3))
    N2 = 4096.0**2
    (i0, v0), fl0, _ = _gemm_flops(nm, fn, X, 0, monkeypatch)
    (i1, v1), fl1, _ = _gemm_flops(nm, fn, X, 1, monkeypatch)
    assert i1 == i0 and np.float64(v1).tobytes() == np.float64(v0).tobytes()
    assert fl1 == fl0 + 192 * N2  # the full loop plus the probe's one tile
