"""The tensor-core bound pass of the smooth kernels (prescreen.cuh, tc_mean_bounds_kernel): distances from fp16 hi/lo
splits on the tensor cores, training columns sorted by the sign of alpha into whole n8 slices, kernel values on MUFU.
Every posterior mean must lie inside [lo, hi] from tb_gp_mean_bounds wherever the bound is finite, at every supported padded
dimension and on the inputs that stress the fp16 splits (tiny coordinates with subnormal lo parts, candidates far outside the
box, coordinates beyond the fp16 range, which must get NaN bounds); and the screened argmax stays the unscreened one, bit for
bit, on each case.  At short lengthscales, where the tensor-core bound would not be trusted on the training box, the CUDA-core
pass takes over: in-box bounds stay finite and the screen keeps pruning."""
from __future__ import annotations

import numpy as np
import pytest

from oracle import gp_oracle as o
from tests.test_gpu_argmax_prescreen import _bounds, _dev, _ei, _same
from tests.test_gpu_argmax_screen import _gemm_flops
from tests.util import candidates, model_pair, native_from_oracle

pytestmark = pytest.mark.gpu

KINDS = ["rbf", "matern32", "matern52"]


def _contained(nm, X, finite=True):
    """every predict mean inside [lo, hi] where the bound is finite; returns (lo, hi, max |mu - mid| / half-width)"""
    lo, hi = _bounds(nm, X)
    mu = np.asarray(nm.predict(X)[0], dtype=np.float64).reshape(-1)
    ok = np.isfinite(lo) & np.isfinite(hi)
    if finite:
        assert np.all(ok)
    assert np.all(np.isnan(lo[~ok]) & np.isnan(hi[~ok]))
    assert np.all((lo[ok] <= mu[ok]) & (mu[ok] <= hi[ok])), np.max(np.maximum(lo - mu, mu - hi)[ok])
    w = ok & (hi > lo)  # far from the data E can vanish next to the mean: lo == mu == hi
    ratio = float(np.max(np.abs(mu[w] - 0.5 * (lo[w] + hi[w])) / (0.5 * (hi[w] - lo[w])))) if w.any() else 0.0
    return lo, hi, ratio


def _centre(om):
    """the input-space point the bound pass maps to x' = 0: the midpoint of the training rows' bounding box"""
    return 0.5 * (om.X.min(0) + om.X.max(0))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("D", [2, 4, 6, 8, 10, 12, 16, 20, 24, 32])
def test_bounds_every_dp(kind, D, monkeypatch):
    om, nm = model_pair(o.ackley, 300, D, kind=kind)
    X = candidates(20_000, D, seed=30 + D)
    _, _, ratio = _contained(nm, X)
    assert ratio < 0.25
    _same(_ei(nm, om), _dev(X), monkeypatch)


@pytest.mark.parametrize("kind", KINDS)
def test_tiny_coordinates(kind, monkeypatch):
    """x' near 0: fp16 hi parts subnormal or zero, lo parts subnormal"""
    om, nm = model_pair(o.hartmann_6, 512, 6, kind=kind)
    rng = np.random.default_rng(31)
    c = _centre(om)
    scale = np.repeat([0.0, 1e-9, 1e-7, 1e-5, 1e-3], 2000)[:, None]
    X = c + scale * rng.standard_normal((scale.shape[0], 6))
    _contained(nm, X)
    _same(_ei(nm, om), _dev(X), monkeypatch)


@pytest.mark.parametrize("kind", KINDS)
def test_far_outside_box(kind, monkeypatch):
    """|x'| from a few lengthscales out to just below the fp16 limit (2^14 per coordinate): the expansion form cancels
    most there; bounds are contained where finite, finite out to moderate distances, NaN where not trusted"""
    om, nm = model_pair(o.hartmann_6, 512, 6, kind=kind)
    rng = np.random.default_rng(32)
    u = rng.standard_normal((6000, 6))
    u /= np.abs(u).max(1, keepdims=True)
    ls = np.asarray(om.lengthscales, dtype=np.float64)
    # the largest coordinate of x' = (x / l - c) * pre, pre <= sqrt(5) log2(e) < 3.3, stays below 2^14
    r = np.geomspace(1.0, 16000.0 / 3.3, u.shape[0])[:, None]
    X = _centre(om) + r * u * ls
    lo, _, _ = _contained(nm, X, finite=False)
    assert np.all(np.isfinite(lo[r[:, 0] < 2.0]))
    _same(_ei(nm, om), _dev(X), monkeypatch)


@pytest.mark.parametrize("kind", KINDS)
def test_beyond_fp16_range(kind, monkeypatch):
    """a coordinate with |x'| past the fp16 range: NaN bounds (not trusted), and the candidate survives the screen"""
    om, nm = model_pair(o.hartmann_6, 512, 6, kind=kind)
    X = candidates(20_000, 6, seed=33)
    ls = np.asarray(om.lengthscales, dtype=np.float64)
    bad = np.arange(3, X.shape[0], 97)
    X[bad, 1] = _centre(om)[1] + np.where(bad % 2 == 0, 1.0, -1.0) * 1e5 * ls[1]
    lo, hi, _ = _contained(nm, X, finite=False)
    assert np.all(np.isnan(lo[bad]) & np.isnan(hi[bad]))
    good = np.setdiff1d(np.arange(X.shape[0]), bad)
    assert np.all(np.isfinite(lo[good]))
    _same(_ei(nm, om), _dev(X), monkeypatch)


def _signed_alpha_model(kind, N, D, npos, seed):
    """a model whose alpha = (K + noise I)^-1 (y - m) has exactly npos positive entries (the first npos)"""
    rng = np.random.default_rng(seed)
    X = rng.uniform(size=(N, D))
    ls, var, nz, mc = np.full(D, 0.2 * np.sqrt(D)), 1.3, 1e-2, 0.7
    a = rng.uniform(0.5, 1.5, N) * np.where(np.arange(N) < npos, 1.0, -1.0)
    K = o.kernel_matrix(kind, X, X, var, ls) + nz * np.eye(N)
    om = o.build_model(kind, X, (mc + K @ a)[:, None], var, ls, nz, mc)
    alpha = np.linalg.solve(K, om.y[:, 0] - mc)
    assert np.sum(alpha > 0) == npos
    return om, native_from_oracle(om)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("N,npos", [(300, 300), (301, 45), (83, 37), (129, 1)])
def test_alpha_sign_classes(kind, N, npos, monkeypatch):
    """all-positive alpha, and sign classes that are not whole slices or stages"""
    om, nm = _signed_alpha_model(kind, N, 6, npos, seed=34 + N)
    X = candidates(20_000, 6, seed=35)
    _, _, ratio = _contained(nm, X)
    assert ratio < 0.25
    _same(_ei(nm, om), _dev(X), monkeypatch)


@pytest.mark.parametrize("N", [3, 7, 129, 257])
def test_n_not_whole_stages(N, monkeypatch):
    om, nm = model_pair(o.hartmann_6, N, 6)
    X = candidates(20_000, 6, seed=36)
    _contained(nm, X)
    _same(_ei(nm, om), _dev(X), monkeypatch)


def test_fp32_handle_bounds(monkeypatch):
    import torch

    import trieste_b200 as tb
    from trieste_b200.acquisition import ExpectedImprovement

    om = o.synthetic_model(o.hartmann_6, 1024, 6)
    X32, y32 = om.X.astype(np.float32), om.y.astype(np.float32)
    nm = tb.GaussianProcessRegression(tb.GPRSpec((X32, y32), tb.Matern52(om.variance, om.lengthscales), tb.Constant(om.mean_const), om.noise))
    X = candidates(20_000, 6, seed=37)
    _, _, ratio = _contained(nm, X)
    assert ratio < 0.25
    fn = ExpectedImprovement().prepare_acquisition_function(nm, tb.Dataset(X32, y32))
    _same(fn, _dev(X, torch.float32), monkeypatch)


def _short_model(kind, N, D, ls, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.uniform(size=(N, D))
    y = o.ackley(X)
    var = float(np.var(y))
    om = o.build_model(kind, X, y, var, np.full(D, ls), var / 100.0, float(np.mean(y)))
    return om, native_from_oracle(om)


@pytest.mark.parametrize("kind", ["rbf", "matern52"])
@pytest.mark.parametrize("D,ls", [(10, 0.1), (10, 0.17), (6, 0.07)])
def test_short_lengthscale_bounds_trusted(kind, D, ls, monkeypatch):
    """pre-scaled norms of several hundred to thousands on the unit box: every in-box candidate keeps a finite, contained bound"""
    om, nm = _short_model(kind, 2048, D, ls)
    X = candidates(20_000, D, seed=38)
    _contained(nm, X)
    _same(_ei(nm, om), _dev(X), monkeypatch)


@pytest.mark.parametrize("kind", ["rbf", "matern52"])
def test_short_lengthscale_still_prunes(kind, monkeypatch):
    """|x'|^2 up to ~4000 (D = 2, lengthscale 0.05): the screen prunes instead of falling back to the unscreened loop"""
    om, nm = _short_model(kind, 1024, 2, 0.05)
    fn = _ei(nm, om)
    X = _dev(candidates(200_000, 2, seed=39))
    (i0, v0), fl0, _ = _gemm_flops(nm, fn, X, 0, monkeypatch)
    (i1, v1), fl1, _ = _gemm_flops(nm, fn, X, 1, monkeypatch)
    assert i1 == i0 and np.float64(v1).tobytes() == np.float64(v0).tobytes()
    assert fl1 < 0.25 * fl0, (fl1, fl0)
