"""CPU checks of continuous Thompson sampling (acquisition/function/continuous_thompson_sampling.py): the NumPy restatement
of the trajectory gradients in tests/cts_oracle.py against central finite differences of the oracle trajectories, the sin
bound of fastmath.cuh's sincos_fast on the host build, and the builders' host logic as the reference's own tests state it
(tests/unit/acquisition/function/test_continuous_thompson_sampling.py), on stand-in trajectories (no device calls)."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import gp_oracle as o
from tests import cts_oracle as cts

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = ["rbf", "matern12", "matern32", "matern52"]


def _central_difference(f, X, h=1e-6):
    """f: [M, B, D] -> [M, B]; returns [M, B, D]."""
    g = np.empty_like(X)
    for d in range(X.shape[-1]):
        e = np.zeros(X.shape[-1])
        e[d] = h
        g[..., d] = (f(X + e) - f(X - e)) / (2.0 * h)
    return g


@pytest.mark.parametrize("kind", KINDS)
def test_rff_trajectory_gradient_matches_finite_differences(kind):
    rng = np.random.default_rng(11)
    D, F, B = 3, 64, 4
    W, b = o.rff_draw(kind, F, D, rng)
    theta = rng.standard_normal((B, F))
    ls, var, mc = np.array([0.3, 0.5, 0.8]), 1.7, 0.25
    X = rng.uniform(size=(9, B, D))
    vals, grads = cts.rff_value_and_gradient(X, W, b, theta, var, ls, mc)
    ref = lambda x: o.rff_trajectory(x, W, b, theta, var, ls, mc)[..., 0]  # noqa: E731
    np.testing.assert_allclose(vals, ref(X), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(grads, _central_difference(ref, X), rtol=1e-6, atol=1e-6 * np.abs(grads).max())


@pytest.mark.parametrize("kind", KINDS)
def test_decoupled_trajectory_gradient_matches_finite_differences(kind):
    om = o.synthetic_model(o.branin, 25, 2, kind=kind, seed=4)
    rng = np.random.default_rng(5)
    F, B = 32, 3
    W, b = o.rff_draw(kind, F, 2, rng)
    w = rng.standard_normal((B, F))
    v = o.decoupled_weights(om, W, b, w, rng.standard_normal((B, 25)))
    X = rng.uniform(size=(7, B, 2))
    vals, grads = cts.decoupled_value_and_gradient(om, X, W, b, w, v)
    ref = lambda x: o.decoupled_trajectory(om, x, W, b, w, v)[..., 0]  # noqa: E731
    np.testing.assert_allclose(vals, ref(X), rtol=1e-11, atol=1e-11 * np.abs(vals).max())
    np.testing.assert_allclose(grads, _central_difference(ref, X), rtol=1e-5, atol=1e-6 * np.abs(grads).max())


def test_matern12_canonical_gradient_is_zero_at_a_training_point():
    """r2 is clamped at 1e-36 (mean_grad_kernel's convention): a coincident training point contributes nothing."""
    om = o.synthetic_model(o.branin, 6, 2, kind="matern12", seed=2)
    W, b = np.zeros((1, 2)), np.zeros(1)
    v = np.zeros((1, 6))
    v[0, 0] = 1.0
    _, g = cts.decoupled_value_and_gradient(om, om.X[:1][:, None, :], W, b, np.zeros((1, 1)), v)
    assert np.all(g == 0.0)


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")
def test_sincos_fast_error_bound_on_the_host(tmp_path):
    exe = str(tmp_path / "sincos_check")
    subprocess.run(["g++", "-O2", "-x", "c++", "-DFM_ITERS=2000000", "-o", exe, os.path.join(ROOT, "tools", "sincos_check.cu")],
                   check=True, capture_output=True)
    res = subprocess.run([exe], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr  # the harness exits non-zero above 1e-13 or on any cos mismatch
    worst = float(res.stdout.split("sincos_fast: max ABS err ")[1].split()[0])
    assert worst < 6e-16  # the bound cos_fast meets
    assert "cos differs from cos_fast at 0 of" in res.stdout


# ---- builders (continuous_thompson_sampling.py) on stand-in trajectories ----------------------------------------------
class _Trajectory:
    """[N, B, D] -> [N, B, 1]; counts its updates and resamples."""

    def __init__(self):
        self.updates = self.resamples = 0
        self.shift = 0.0

    def __call__(self, x):
        return np.sum(np.asarray(x) ** 2, axis=-1, keepdims=True) + self.shift

    def update(self):
        self.updates += 1

    def resample(self):
        self.resamples += 1
        self.shift += 1.0


class _Sampler:
    def __init__(self, in_place=True):
        self.in_place = in_place

    def get_trajectory(self):
        return _Trajectory()

    def update_trajectory(self, trajectory):
        if not isinstance(trajectory, _Trajectory):
            raise ValueError("trajectory must be a _Trajectory")
        if not self.in_place:  # the reference test's DumbTrajectorySampler
            return self.get_trajectory()
        trajectory.update()
        return trajectory

    def resample_trajectory(self, trajectory):
        if not isinstance(trajectory, _Trajectory):
            raise ValueError("trajectory must be a _Trajectory")
        trajectory.resample()
        return trajectory


class _Model:
    def __init__(self, in_place=True):
        self.in_place = in_place

    def trajectory_sampler(self):
        return _Sampler(self.in_place)


def test_builders_raise_for_a_model_without_trajectory_sampler():
    from trieste_b200.acquisition import GreedyContinuousThompsonSampling, ParallelContinuousThompsonSampling

    for builder in (GreedyContinuousThompsonSampling(), ParallelContinuousThompsonSampling()):
        with pytest.raises(ValueError, match="only supports models with a trajectory_sampler"):
            builder.prepare_acquisition_function(object())


@pytest.mark.parametrize("in_place", [True, False])
def test_parallel_builder_builds_negated_trajectory_and_rejects_a_foreign_function(in_place):
    from trieste_b200.acquisition import ParallelContinuousThompsonSampling

    builder = ParallelContinuousThompsonSampling()
    model = _Model(in_place)
    fn = builder.prepare_acquisition_function(model)
    assert type(fn).__name__ == "NegatedTrajectory" and isinstance(fn, _Trajectory)
    new = builder.update_acquisition_function(fn, model)
    assert type(new).__name__ == "NegatedTrajectory"
    assert (new is fn) == in_place
    with pytest.raises(ValueError, match="Wrong trajectory function passed into update_acquisition_function"):
        builder.update_acquisition_function(lambda x: x, model)
    if not in_place:
        with pytest.raises(ValueError, match="Wrong trajectory function"):
            builder.update_acquisition_function(fn, model)  # the superseded function


@pytest.mark.parametrize("in_place", [True, False])
def test_greedy_builder_updates_on_new_steps_and_resamples_within_a_batch(in_place):
    from trieste_b200.acquisition import GreedyContinuousThompsonSampling

    builder = GreedyContinuousThompsonSampling()
    model = _Model(in_place)
    fn = builder.prepare_acquisition_function(model)
    assert type(fn).__name__ == "NegatedTrajectory"
    same = builder.update_acquisition_function(fn, model, new_optimization_step=False)
    assert same is fn and fn.resamples == 1
    new = builder.update_acquisition_function(fn, model, new_optimization_step=True)
    assert type(new).__name__ == "NegatedTrajectory"
    assert (new is fn) == in_place
    if in_place:
        assert fn.updates == 1
    with pytest.raises(ValueError):
        builder.update_acquisition_function(lambda x: x, model)


def test_negation_is_exactly_minus_one_times_and_keeps_methods():
    from trieste_b200.acquisition import ParallelContinuousThompsonSampling, negate_trajectory_function

    fn = ParallelContinuousThompsonSampling().prepare_acquisition_function(_Model())
    x = np.linspace(-10, 10, 100).reshape(10, 5, 2)
    evals = fn(x)
    assert evals.shape == (10, 5)
    np.testing.assert_array_equal(evals, -1.0 * _Trajectory()(x)[..., 0])
    neg = negate_trajectory_function(fn)  # negated again, without an output selection
    np.testing.assert_array_equal(evals, -1.0 * neg(x))
    assert hasattr(neg, "update") and hasattr(neg, "resample")
    plain = negate_trajectory_function(lambda z: np.asarray(z)[..., :1] * 2.0)
    np.testing.assert_array_equal(plain(x), -1.0 * x[..., :1] * 2.0)


def test_select_nth_output():
    from trieste_b200.acquisition import select_nth_output

    x = np.arange(24.0).reshape(2, 3, 4)
    np.testing.assert_array_equal(select_nth_output(x), x[..., 0])
    np.testing.assert_array_equal(select_nth_output(x, 2), x[..., 2])


class _DeviceTrajectory(_Trajectory):
    """Offers the trajectory methods the negated object builds on: value_and_gradient and minimize_from."""

    def value_and_gradient(self, x):
        x = np.asarray(x)
        return _Trajectory.__call__(self, x), 2.0 * x

    def minimize_from(self, starts, lower, upper, **options):
        x = np.clip(np.zeros_like(starts), lower, upper)
        R, B, _ = starts.shape
        self.options = options
        return np.ones((R, B), bool), _Trajectory.__call__(self, x)[..., 0], x, np.full((R, B), 3)


def test_gradient_and_device_paths_only_with_the_default_output_selection():
    from trieste_b200.acquisition import negate_trajectory_function, select_nth_output

    x = np.random.default_rng(0).uniform(0.5, 1.0, size=(6, 3, 2))
    fn = negate_trajectory_function(_DeviceTrajectory(), select_nth_output)
    v, g = fn.value_and_gradient(x)
    np.testing.assert_array_equal(v, -1.0 * np.sum(x**2, axis=-1))
    np.testing.assert_array_equal(g, -2.0 * x)
    ok, f, xs, nfev = fn.maximize_from(x, np.full(2, 0.25), np.ones(2), maxcor=5)
    assert ok.shape == (6, 3) and xs.shape == (6, 3, 2) and fn.options == {"maxcor": 5}
    np.testing.assert_array_equal(f, np.full((6, 3), -0.125))
    ok1, f1, xs1, n1 = fn.maximize_from(x[:, 0, :], np.full(2, 0.25), np.ones(2))  # [P, D] starts for B = 1
    assert ok1.shape == (6,) and f1.shape == (6,) and xs1.shape == (6, 2) and n1.shape == (6,)
    custom = negate_trajectory_function(_DeviceTrajectory(), lambda y: y[..., 0] * 1.0)
    for name in ("value_and_gradient", "maximize_from", "fused_argmax"):
        assert not hasattr(custom, name)
    np.testing.assert_array_equal(custom(x), -1.0 * np.sum(x**2, axis=-1))


def test_trajectory_rejects_a_changed_batch_size():
    """sampler.py:920-927: the first call fixes B; another batch size raises before anything reaches the device."""
    from trieste_b200.acquisition import negate_trajectory_function, select_nth_output
    from trieste_b200.sampler import feature_decomposition_trajectory

    traj = feature_decomposition_trajectory.__new__(feature_decomposition_trajectory)
    traj._h, traj._initialized, traj._batch_size = None, True, 5
    fn = negate_trajectory_function(traj, select_nth_output)
    for call in (fn, fn.value_and_gradient, lambda x: fn.maximize_from(x, 0.0, 1.0)):
        with pytest.raises(ValueError, match="only supports batch sizes of 5"):
            call(np.linspace(-10, 10, 100).reshape(5, 10, 2))
