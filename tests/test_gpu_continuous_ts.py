"""Continuous Thompson sampling on the GPU: the paired trajectory kernel (tb_rff_eval_paired) against the per-column
tb_rff_eval path bit for bit, its gradients against tests/cts_oracle.py and finite differences, the device L-BFGS of the
trajectories (tb_rff_maximize) against the host implementation of the same algorithm and SciPy on the oracle trajectory, and
both builders end to end (acquisition/function/continuous_thompson_sampling.py)."""
import ctypes as C

import numpy as np
import pytest

from oracle import gp_oracle as o
from tests import cts_oracle as cts
from tests.util import model_pair

pytestmark = pytest.mark.gpu

KINDS = ["rbf", "matern12", "matern32", "matern52"]


def _trajectory(nm, decoupled: bool, F: int, B: int, D: int, seed=0):
    from trieste_b200.sampler import DecoupledTrajectorySampler, RandomFourierFeatureTrajectorySampler

    cls = DecoupledTrajectorySampler if decoupled else RandomFourierFeatureTrajectorySampler
    s = cls(nm, F, seed=seed)
    traj = s.get_trajectory()
    traj(np.zeros((1, B, D)))  # fixes the batch size, draws the weights
    return s, traj


def _per_column(traj, X):
    """The per-column path: tb_rff_eval of column b under all B trajectories, keep column b."""
    from trieste_b200 import _lib

    M, B, D = X.shape
    out = np.empty((M, B))
    for b in range(B):
        col = np.ascontiguousarray(X[:, b, :])
        o_ = np.empty((M, B))
        _lib.check(_lib.lib().tb_rff_eval(traj._h, col.ctypes.data, M, o_.ctypes.data, None, None))
        out[:, b] = o_[:, b]
    return out


def _paired(traj, X, grad=False):
    from trieste_b200 import _lib

    M, B, D = X.shape
    X = np.ascontiguousarray(X)
    out = np.empty((M, B))
    g = np.empty((M, B, D)) if grad else None
    _lib.check(_lib.lib().tb_rff_eval_paired(traj._h, X.ctypes.data, M, B, out.ctypes.data, None if g is None else g.ctypes.data))
    return out, g


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("decoupled", [False, True])
@pytest.mark.parametrize("D", [1, 6, 32])
def test_paired_values_equal_the_per_column_path_bit_for_bit(kind, decoupled, D):
    om, nm = model_pair(o.ackley, 60, D, kind=kind)
    M = 1000  # not a multiple of the 256-thread block
    for B, F in ((1, 300), (3, 700), (8, 300), (37, 128)):  # F = 700: two feature chunks of shared memory
        _, traj = _trajectory(nm, decoupled, F, B, D, seed=B)
        X = np.random.default_rng(B).uniform(-0.2, 1.2, size=(M, B, D))
        ref = _per_column(traj, X)
        got, _ = _paired(traj, X)
        np.testing.assert_array_equal(got, ref)
        np.testing.assert_array_equal(traj(X)[..., 0], ref)  # __call__ of B > 1 runs the paired kernel
        vg, _ = _paired(traj, X, grad=True)
        np.testing.assert_array_equal(vg, ref)  # the gradient variant's values are the same


def test_paired_call_launches_do_not_grow_with_the_batch_size():
    from trieste_b200 import _lib

    om, nm = model_pair(o.hartmann_6, 100, 6)
    counts = []
    for B in (3, 37):
        _, traj = _trajectory(nm, True, 256, B, 6)
        X = np.random.default_rng(0).uniform(size=(2000, B, 6))
        _lib.lib().tb_launch_count_reset()
        traj(X)
        counts.append(_lib.lib().tb_launch_count())
    assert counts[0] == counts[1] == 1, counts


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("decoupled", [False, True])
def test_paired_gradients_match_the_oracle_and_finite_differences(kind, decoupled):
    om, nm = model_pair(o.hartmann_6, 120, 6, kind=kind)
    B, F = 5, 400
    s, traj = _trajectory(nm, decoupled, F, B, 6, seed=3)
    W, b = s._feature_functions.W, s._feature_functions.b
    X = np.random.default_rng(9).uniform(size=(300, B, 6))
    vals, grads = traj.value_and_gradient(X)
    assert vals.shape == (300, B, 1) and grads.shape == (300, B, 6)
    if decoupled:
        ov, og = cts.decoupled_value_and_gradient(om, X, W, b, traj._weights_sample, traj._canonical_weights)
    else:
        ov, og = cts.rff_value_and_gradient(X, W, b, traj._weights_sample, om.variance, om.lengthscales, om.mean_const)
    scale = np.abs(og).max()
    np.testing.assert_allclose(vals[..., 0], ov, rtol=1e-9, atol=1e-9 * np.abs(ov).max())
    np.testing.assert_allclose(grads, og, rtol=1e-9, atol=1e-9 * scale)
    h = 1e-7  # Matern-12 features have Cauchy-distributed frequencies: a wider step is dominated by truncation error
    fd = np.empty_like(X)
    for d in range(6):
        e = np.zeros(6)
        e[d] = h
        fd[..., d] = (traj(X + e)[..., 0] - traj(X - e)[..., 0]) / (2 * h)
    np.testing.assert_allclose(grads, fd, rtol=1e-5, atol=1e-6 * scale)


def test_device_lbfgs_of_trajectories_matches_host_and_scipy(monkeypatch):
    from trieste_b200.acquisition import ParallelContinuousThompsonSampling
    from trieste_b200.acquisition.optimizer import _perform_parallel_continuous_optimization

    om, nm = model_pair(o.hartmann_6, 200, 6)
    fn = ParallelContinuousThompsonSampling().prepare_acquisition_function(nm)
    R, B = 8, 4
    starts = np.random.default_rng(2).uniform(size=(R, B, 6))
    fn(starts)  # fixes B
    lower, upper = np.zeros(6), np.ones(6)
    ok, val, x, nfev = fn.maximize_from(starts, lower, upper)
    assert ok.shape == (R, B) and x.shape == (R, B, 6) and (x >= 0).all() and (x <= 1).all()
    assert ok.mean() > 0.9 and nfev.min() >= 1
    np.testing.assert_allclose(val, fn(x), rtol=1e-12, atol=1e-12 * np.abs(val).max())
    assert np.all(val >= fn(starts) - 1e-9 * np.abs(val).max())
    _, g = fn.value_and_gradient(x)
    pg = x - np.clip(x + g, lower, upper)
    assert np.abs(pg[ok]).max() < 1e-3 * max(1.0, np.abs(val).max())
    # the host implementation of the same algorithm, same starts
    monkeypatch.setenv("TB_LBFGS", "host")
    s2, f2, x2, n2 = _perform_parallel_continuous_optimization(fn, lower, upper, starts, {})
    monkeypatch.delenv("TB_LBFGS")
    scale = np.abs(f2).max()
    both = ok & s2
    assert (np.abs(val - f2) <= 1e-4 * scale)[both].mean() > 0.85
    np.testing.assert_allclose(val.max(axis=0), f2.max(axis=0), rtol=0, atol=1e-4 * scale)
    # SciPy's L-BFGS-B on the oracle trajectory b from the same starts: the device's best is no worse
    W, bb = fn._feature_functions.W, fn._feature_functions.b
    w, v = fn._weights_sample, fn._canonical_weights
    for b in range(B):
        def neg_traj(xq, b=b):
            f_, g_ = cts.decoupled_value_and_gradient(om, xq[:, None, :], W, bb, w[b:b + 1], v[b:b + 1])
            return -f_[:, 0], -g_[:, 0, :]

        _, sf, _, _ = o.scipy_lbfgsb_multistart(neg_traj, starts[:, b, :], lower, upper)
        assert val[:, b].max() >= sf.max() - 1e-6 * max(1.0, abs(sf.max())), (b, val[:, b].max(), sf.max())


def _gpr(objective, D, n, seed):
    import trieste_b200 as tb

    space = tb.Box([0.0] * D, [1.0] * D)
    X = space.sample(n, seed=seed)
    ds = tb.Dataset(X, objective(X))
    return space, ds, tb.GaussianProcessRegression(tb.build_gpr(ds, space, likelihood_variance=1e-5))


@pytest.mark.parametrize("objective,D", [(o.branin, 2), (o.hartmann_6, 6)])
def test_parallel_builder_end_to_end(objective, D):
    from trieste_b200.acquisition import ParallelContinuousThompsonSampling
    from trieste_b200.rule import EfficientGlobalOptimization

    B = 10
    space, ds, model = _gpr(objective, D, 20, seed=1)
    rule = EfficientGlobalOptimization(ParallelContinuousThompsonSampling(), num_query_points=B)
    pts = rule.acquire_single(space, model, ds)
    assert pts.shape == (B, D) and space.contains(pts).all()
    fn = rule.acquisition_function
    assert type(fn).__name__ == "NegatedTrajectory"
    val, g = fn.value_and_gradient(pts[None])  # point b under its own trajectory b
    pg = pts[None] - np.clip(pts[None] + g, space.lower, space.upper)
    assert np.abs(pg).max() <= 1e-3 * max(1.0, np.abs(val).max()), np.abs(pg).max()
    fmin, _ = fn.argmin_over(space.sample(20000, seed=7))  # each trajectory's minimum over random points
    f_at = -val[0]
    assert np.all(f_at <= fmin + 1e-6 * max(1.0, np.abs(fmin).max())), (f_at, fmin)
    X2 = np.concatenate([ds.query_points, pts])
    import trieste_b200 as tb

    ds2 = tb.Dataset(X2, objective(X2))
    model.update(ds2)
    pts2 = rule.acquire_single(space, model, ds2)
    assert rule.acquisition_function is fn and pts2.shape == (B, D) and space.contains(pts2).all()


def test_greedy_builder_resamples_at_each_step_and_returns_the_batch():
    from trieste_b200.acquisition import GreedyContinuousThompsonSampling
    from trieste_b200.rule import EfficientGlobalOptimization

    space, ds, model = _gpr(o.branin, 2, 20, seed=2)
    builder = GreedyContinuousThompsonSampling()
    fn = builder.prepare_acquisition_function(model, ds)
    fn(np.zeros((1, 1, 2)))
    theta0 = np.array(fn._weights_sample, copy=True)
    same = builder.update_acquisition_function(fn, model, ds, pending_points=np.zeros((1, 2)), new_optimization_step=False)
    assert same is fn and not np.array_equal(fn._weights_sample, theta0)
    rule = EfficientGlobalOptimization(GreedyContinuousThompsonSampling(), num_query_points=5)
    pts = rule.acquire_single(space, model, ds)
    assert pts.shape == (5, 2) and space.contains(pts).all()
    assert len(np.unique(pts, axis=0)) == 5  # a new trajectory at each greedy step


@pytest.mark.parametrize("greedy", [False, True])
def test_seeded_bo_loop_runs_with_each_builder(greedy):
    from trieste_b200.acquisition import GreedyContinuousThompsonSampling, ParallelContinuousThompsonSampling
    from trieste_b200.bayesian_optimizer import BayesianOptimizer
    from trieste_b200.rule import EfficientGlobalOptimization

    np.random.seed(0)
    space, ds, model = _gpr(o.branin, 2, 10, seed=3)
    builder = GreedyContinuousThompsonSampling() if greedy else ParallelContinuousThompsonSampling()
    rule = EfficientGlobalOptimization(builder, num_query_points=4)
    result = BayesianOptimizer(o.branin, space).optimize(5, ds, model, rule)
    assert result.error is None, result.error
    final = result.try_get_final_dataset()
    assert len(final) == 10 + 5 * 4 and all(h.shape == (4, 2) for h in result.history)
    assert space.contains(final.query_points).all()


def test_abi_argument_checks():
    from trieste_b200 import _lib

    om, nm = model_pair(o.hartmann_6, 50, 6)
    _, traj = _trajectory(nm, True, 64, 3, 6)
    X = np.zeros((4, 3, 6))
    out = np.empty((4, 3))
    L = _lib.lib()
    assert L.tb_rff_eval_paired(traj._h, X.ctypes.data, 4, 2, out.ctypes.data, None) == _lib.TB_ERR_INVALID  # B != nb
    assert L.tb_rff_eval_paired(traj._h, None, 4, 3, out.ctypes.data, None) == _lib.TB_ERR_INVALID
    lo, up = np.zeros(6), np.ones(6)
    xo, fo = np.empty((1, 3, 6)), np.empty((1, 3))
    so, no = np.empty((1, 3), np.int32), np.empty((1, 3), np.int64)
    args = lambda R, maxcor: (traj._h, lo.ctypes.data, up.ctypes.data, X.ctypes.data, R, maxcor, 10, 5, 1e-5, 1e-9,  # noqa: E731
                              xo.ctypes.data, fo.ctypes.data, so.ctypes.data, no.ctypes.data)
    assert L.tb_rff_maximize(*args(1, 0)) == _lib.TB_ERR_INVALID
    assert L.tb_rff_maximize(*args(1, 17)) == _lib.TB_ERR_INVALID
    assert L.tb_rff_maximize(*args(1 << 30, 10)) == _lib.TB_ERR_INVALID  # R * nb >= 2^31
    assert L.tb_rff_maximize(None, lo.ctypes.data, up.ctypes.data, X.ctypes.data, 1, 10, 10, 5, 1e-5, 1e-9, xo.ctypes.data,
                             fo.ctypes.data, so.ctypes.data, no.ctypes.data) == _lib.TB_ERR_INVALID
    h = C.c_void_p()
    _lib.check(L.tb_rff_create(C.byref(h), 0))
    try:
        W = np.zeros((4, 6))
        bias, ls = np.zeros(4), np.ones(6)
        dp = C.POINTER(C.c_double)
        _lib.check(L.tb_rff_set(h, W.ctypes.data_as(dp), bias.ctypes.data_as(dp), 4, 6, ls.ctypes.data_as(dp), 1.0, 0.0))
        assert L.tb_rff_eval_paired(h, X.ctypes.data, 4, 3, out.ctypes.data, None) == _lib.TB_ERR_INVALID  # theta not set
    finally:
        L.tb_rff_destroy(h)
