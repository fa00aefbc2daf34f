"""The screened argmax's rounds of few candidate tiles (tb_api.cu, eval_chunk with gathered candidates): the wide K*
generation (kernel values over many k-split CTAs, the source chunk's mean chain replayed) and the split-K variance GEMM
(int32 level accumulators summed across units, the row-block groups' epilogue in serpentine order) must give what the
unscreened chunk loop gives, bit for bit.

To make many candidates survive without flattening the acquisition, `n` candidates are replaced by copies of the unscreened
winner moved by ~1e-9: their values differ from the winner's by far less than the screen's margin (2^-20 |tau|), so they all
survive, and at the model's own eta the winner's value still depends on every bit of its mean and variance."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from oracle import gp_oracle as o
from tests.test_gpu_argmax_screen import HEADLINE_CHUNK, _argmax, _dev, _ei, _gemm_flops, _same
from tests.util import candidates, model_pair

pytestmark = pytest.mark.gpu


def _near_copies(fn, X, n, monkeypatch, n_last=0, last_from=None, dtype=torch.float64, seed=0):
    """X with n candidates replaced by copies of its unscreened winner moved by ~1e-9; n_last of them in [last_from, M)"""
    i, _ = _argmax(fn, _dev(X, dtype), 0, monkeypatch)
    rng = np.random.default_rng(seed)
    M = X.shape[0]
    cut = M if last_from is None else last_from
    pos = rng.choice(cut, size=n - n_last, replace=False)
    if n_last:
        pos = np.concatenate([pos, last_from + rng.choice(M - last_from, size=n_last, replace=False)])
    X = X.copy()
    X[pos] = X[i] + 1e-9 * rng.standard_normal((len(pos), X.shape[1]))
    return X


@pytest.fixture(scope="module")
def headline():
    om, nm = model_pair(o.ackley, 4096, 10)
    return om, nm, _ei(nm, om)


@pytest.mark.parametrize("n", [700, 3000])
def test_headline_many_tiles(headline, n, monkeypatch):
    """survivors over several tiles in both k-split groups (whole chunks, and the last partial one): ~700 take the wide K*
    and the split GEMM in several tiles, ~3000 are enough tiles for the row-block groups to fill the GPU"""
    om, nm, fn = headline
    M = 3 * HEADLINE_CHUNK + 1000
    X = _dev(_near_copies(fn, candidates(M, 10, seed=7), n, monkeypatch, n_last=50, last_from=3 * HEADLINE_CHUNK))
    _same(fn, X, monkeypatch)
    _, fl, launches = _gemm_flops(nm, fn, X, 1, monkeypatch)
    tiles = fl / 4096.0**2 / 192
    assert launches >= 3 and tiles >= 2 + (n - 50) // 192 and tiles < M / 4 / 192, (launches, tiles)


@pytest.mark.parametrize("M", [193, 3000])
def test_ksplit_source_chunk(M, monkeypatch):
    """N = 1024: a chunk of 193 or 3000 candidates is split over the training rows (ksplit > 1); its survivors fill one
    tile or four"""
    om, nm = model_pair(o.hartmann_6, 1024, 6)
    fn = _ei(nm, om)
    _same(fn, _dev(_near_copies(fn, candidates(M, 6, seed=M), M // 5, monkeypatch)), monkeypatch)


@pytest.mark.parametrize("D", [2, 6, 10, 12, 20, 32])
@pytest.mark.parametrize("kind", ["rbf", "matern12", "matern32", "matern52"])
def test_kernels_and_dimensions(kind, D, monkeypatch):
    om, nm = model_pair(o.ackley, 1024, D, kind=kind)
    fn = _ei(nm, om)
    _same(fn, _dev(_near_copies(fn, candidates(40000, D, seed=D), 300, monkeypatch)), monkeypatch)


def test_fp32_handle(monkeypatch):
    import trieste_b200 as tb
    from trieste_b200.acquisition import ExpectedImprovement

    om = o.synthetic_model(o.hartmann_6, 1024, 6)
    X32, y32 = om.X.astype(np.float32), om.y.astype(np.float32)
    nm = tb.GaussianProcessRegression(tb.GPRSpec((X32, y32), tb.Matern52(om.variance, om.lengthscales), tb.Constant(om.mean_const), om.noise))
    fn = ExpectedImprovement().prepare_acquisition_function(nm, tb.Dataset(X32, y32))
    X = _near_copies(fn, candidates(30000, 6, seed=11).astype(np.float32), 300, monkeypatch, dtype=torch.float32)
    _same(fn, _dev(X, torch.float32), monkeypatch)


def test_int8x21_engine(monkeypatch):
    om, nm = model_pair(o.hartmann_6, 1024, 6, engine="int8x21")
    fn = _ei(nm, om)
    _same(fn, _dev(_near_copies(fn, candidates(30000, 6, seed=12), 300, monkeypatch)), monkeypatch)
    assert nm.engine_info()[0] == 21
