"""The fp32 bound pass of the screened EI / log-EI argmax (prescreen.cuh, tb_api.cu argmax_screened): screened against
unscreened (TB_ARGMAX_SCREEN=1 / 0) with the same index and the byte-identical value on the shapes where the survivors'
exact means must come from a launch with their chunk's k-split, and the bound itself: every posterior mean lies inside the
interval tb_gp_mean_bounds returns, with the error far below the bound."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from oracle import gp_oracle as o
from tests.util import candidates, model_pair

pytestmark = pytest.mark.gpu

HEADLINE_CHUNK = 50_688  # candidates per chunk of the 15-product engine at N = 4096, D = 10


def _ei(nm, om, log=False):
    from trieste_b200 import Dataset
    from trieste_b200.acquisition import ExpectedImprovement, LogExpectedImprovement

    b = LogExpectedImprovement() if log else ExpectedImprovement()
    return b.prepare_acquisition_function(nm, Dataset(om.X, om.y))


def _dev(X, dtype=torch.float64):
    return torch.as_tensor(np.ascontiguousarray(X), dtype=dtype, device="cuda")


def _same(fn, X, monkeypatch):
    monkeypatch.setenv("TB_ARGMAX_SCREEN", "0")
    i0, v0 = fn.fused_argmax(X)
    monkeypatch.setenv("TB_ARGMAX_SCREEN", "1")
    i1, v1 = fn.fused_argmax(X)
    assert i1 == i0
    assert np.float64(v1).tobytes() == np.float64(v0).tobytes(), (v1, v0)
    return i0, v0


def _bounds(nm, X):
    from trieste_b200 import _lib

    X = np.ascontiguousarray(X, dtype=np.float64)
    M = X.shape[0]
    lo, hi = np.empty(M), np.empty(M)
    _lib.check(_lib.lib().tb_gp_mean_bounds(nm.handle, X.ctypes.data, M, lo.ctypes.data, hi.ctypes.data))
    return lo, hi


def _check_bounds(nm, X):
    """every predict mean inside [lo, hi]; returns max |mu - mid| / half-width (must be far below 1)"""
    lo, hi = _bounds(nm, X)
    mu = np.asarray(nm.predict(X)[0], dtype=np.float64).reshape(-1)
    assert np.all(np.isfinite(lo)) and np.all(np.isfinite(hi))
    assert np.all((lo <= mu) & (mu <= hi)), np.max(np.maximum(lo - mu, mu - hi))
    mid, half = 0.5 * (lo + hi), 0.5 * (hi - lo)
    return float(np.max(np.abs(mu - mid) / half))


@pytest.fixture(scope="module")
def headline():
    om, nm = model_pair(o.ackley, 4096, 10)
    return om, nm, _ei(nm, om)


def test_headline_last_chunk_ksplit(headline, monkeypatch):
    om, nm, fn = headline
    _same(fn, _dev(candidates(3 * HEADLINE_CHUNK + 1000, 10, seed=11)), monkeypatch)


def test_headline_log_ei(headline, monkeypatch):
    om, nm, _ = headline
    _same(_ei(nm, om, log=True), _dev(candidates(2 * HEADLINE_CHUNK + 300, 10, seed=12)), monkeypatch)


def test_small_m(monkeypatch):
    om, nm = model_pair(o.hartmann_6, 1024, 6)
    fn = _ei(nm, om)
    for M in (1, 2, 193, 5000):
        _same(fn, _dev(candidates(M, 6, seed=20 + M)), monkeypatch)


@pytest.mark.parametrize("kind", ["rbf", "matern12", "matern32"])
def test_kernel_kinds(kind, monkeypatch):
    om, nm = model_pair(o.hartmann_6, 512, 6, kind=kind)
    _same(_ei(nm, om), _dev(candidates(40000, 6, seed=13)), monkeypatch)


def test_branin_n20(monkeypatch):
    om, nm = model_pair(o.branin, 20, 2)
    _same(_ei(nm, om), _dev(candidates(20000, 2, seed=14)), monkeypatch)


def test_fp32_handle(monkeypatch):
    import trieste_b200 as tb
    from trieste_b200.acquisition import ExpectedImprovement

    om = o.synthetic_model(o.hartmann_6, 1024, 6)
    X32, y32 = om.X.astype(np.float32), om.y.astype(np.float32)
    nm = tb.GaussianProcessRegression(tb.GPRSpec((X32, y32), tb.Matern52(om.variance, om.lengthscales), tb.Constant(om.mean_const), om.noise))
    fn = ExpectedImprovement().prepare_acquisition_function(nm, tb.Dataset(X32, y32))
    _same(fn, _dev(candidates(30000, 6, seed=15), torch.float32), monkeypatch)


def test_int8x21_engine(monkeypatch):
    om, nm = model_pair(o.hartmann_6, 1024, 6, engine="int8x21")
    _same(_ei(nm, om), _dev(candidates(30000, 6, seed=16)), monkeypatch)
    assert nm.engine_info()[0] == 21


def test_non_finite_and_huge_coordinates(monkeypatch):
    """NaN, +-inf and 1e30 coordinates (the fp32 norms overflow): their bounds are not trusted and they survive"""
    om, nm = model_pair(o.hartmann_6, 1024, 6)
    fn = _ei(nm, om)
    X = candidates(30000, 6, seed=17)
    X[5::11, 2] = np.nan
    X[7::13, 0] = np.inf
    X[9::17, 4] = -np.inf
    X[3::19, 1] = 1e30
    X[4::23, 5] = -1e30
    _same(fn, _dev(X), monkeypatch)
    lo, hi = _bounds(nm, X[:200])
    bad = ~np.all(np.isfinite(X[:200]) & (np.abs(X[:200]) < 1e20), axis=1)
    assert np.all(np.isnan(lo[bad]) & np.isnan(hi[bad]))


def test_duplicates_first_index_wins(monkeypatch):
    om, nm = model_pair(o.hartmann_6, 1024, 6)
    fn = _ei(nm, om)
    X = candidates(30000, 6, seed=18)
    monkeypatch.setenv("TB_ARGMAX_SCREEN", "0")
    i, _ = fn.fused_argmax(_dev(X))
    j = i // 3
    X[j] = X[i]
    X[-1] = X[i]
    k, _ = _same(fn, _dev(X), monkeypatch)
    assert k == j


def test_bounds_headline(headline):
    om, nm, _ = headline
    ratio = _check_bounds(nm, candidates(200_000, 10, seed=19))
    print(f"headline: max |mu - mu~| / E = {ratio:.3g}")
    assert ratio < 0.25


@pytest.mark.parametrize("kind", ["rbf", "matern12", "matern32", "matern52"])
def test_bounds_kernel_kinds(kind):
    om, nm = model_pair(o.hartmann_6, 512, 6, kind=kind)
    ratio = _check_bounds(nm, candidates(50_000, 6, seed=21))
    print(f"{kind}: max |mu - mu~| / E = {ratio:.3g}")
    assert ratio < 0.25
