"""CPU checks of local penalisation (greedy_batch.py:54-388): the NumPy restatement in tests/lp_oracle.py against known
answers and finite differences, and the builder protocol on an oracle-backed model (no device calls)."""
import numpy as np
import pytest

from oracle import gp_oracle as o
from tests import lp_oracle as lp


def _state(seed=0, P=3, D=2):
    rng = np.random.default_rng(seed)
    pending = rng.uniform(size=(P, D))
    radius = rng.uniform(0.05, 0.3, size=P)
    scale = rng.uniform(0.02, 0.2, size=P)
    return pending, radius, scale


def test_soft_penalty_is_one_half_at_the_radius():
    pending, radius, scale = _state(P=1)
    direction = np.array([0.6, 0.8])
    x = pending + radius[0] * direction
    np.testing.assert_allclose(lp.penalty(lp.SOFT, x, pending, radius, scale), [0.5], rtol=1e-14)


def test_hard_penalty_is_zero_at_a_pending_point_and_tends_to_one_far_away():
    pending, radius, scale = _state(P=4)
    assert np.all(lp.penalty(lp.HARD, pending, pending, radius, scale) == 0.0)
    far = pending[:1] + 1e4
    assert lp.penalty(lp.HARD, far, pending, radius, scale)[0] == pytest.approx(1.0, abs=1e-12)
    # a negative radius + scale: ratio in (-1, 0) makes the base of the 1/5 power negative -> NaN, as in the reference
    x = pending[:1] + np.array([[0.01, 0.0]])
    assert np.isnan(lp.penalty(lp.HARD, x, pending[:1], np.array([-0.5]), np.array([0.1])))[0]


def test_penalised_value_is_exp_of_log_base_plus_log_penalty():
    """greedy_batch.py:265-269 as restated by the reference's own test (test_greedy_batch.py:122-157)."""
    om = o.synthetic_model(o.branin, 20, 2, seed=3)
    xs = np.stack(np.meshgrid(np.linspace(0, 1, 11), np.linspace(0, 1, 11), indexing="ij"), axis=-1).reshape(-1, 2)
    L, eta = lp.lipschitz_and_eta(om, np.concatenate([om.X, xs]))
    pending = np.zeros((2, 2))
    radius, scale = lp.penalizer_state(om, pending, L, eta)
    mean, var = o.predict(om, xs)
    base = o.expected_improvement(mean, var, o.ei_eta(om))[:, 0]
    for kind in (lp.SOFT, lp.HARD):
        pen = lp.penalty(kind, xs, pending, radius, scale)
        got = lp.penalized(base, pen)
        with np.errstate(divide="ignore"):
            np.testing.assert_array_equal(got, np.exp(np.log(base) + np.log(pen)))
        np.testing.assert_allclose(got, base * pen, rtol=1e-13, atol=1e-300)
    assert np.isnan(lp.penalized(np.array([-1e-3]), np.array([0.5])))[0]


@pytest.mark.parametrize("kind", [lp.SOFT, lp.HARD])
def test_penalty_and_penalised_ei_gradients_against_finite_differences(kind):
    om = o.synthetic_model(o.branin, 30, 2, seed=1)
    L, eta = lp.lipschitz_and_eta(om, np.concatenate([om.X, np.random.default_rng(0).uniform(size=(100, 2))]))
    pending = np.random.default_rng(2).uniform(size=(3, 2))
    radius, scale = lp.penalizer_state(om, pending, L, eta)
    x = np.random.default_rng(4).uniform(size=(40, 2))
    pen, gpen = lp.penalty_gradient(kind, x, pending, radius, scale)
    ei_eta = o.ei_eta(om)
    val, grad = lp.penalized_ei_value_and_gradient(om, x, ei_eta, kind, pending, radius, scale)
    h = 1e-6
    for d in range(2):
        e = np.zeros(2)
        e[d] = h
        fd_pen = (lp.penalty(kind, x + e, pending, radius, scale) - lp.penalty(kind, x - e, pending, radius, scale)) / (2 * h)
        np.testing.assert_allclose(gpen[:, d], fd_pen, rtol=1e-5, atol=1e-8)
        vp, _ = lp.penalized_ei_value_and_gradient(om, x + e, ei_eta, kind, pending, radius, scale)
        vm, _ = lp.penalized_ei_value_and_gradient(om, x - e, ei_eta, kind, pending, radius, scale)
        np.testing.assert_allclose(grad[:, d], (vp - vm) / (2 * h), rtol=1e-4, atol=1e-7 * np.abs(grad).max())
    # at a pending point: the hard penalty and its gradient are 0, the soft one finite
    p0, g0 = lp.penalty_gradient(kind, pending[:1], pending, radius, scale)
    assert np.all(np.isfinite(g0))
    if kind == lp.HARD:
        assert p0[0] == 0.0 and np.all(g0 == 0.0)


def test_flat_model_falls_back_to_lipschitz_constant_ten():
    X = np.random.default_rng(0).uniform(size=(10, 2))
    om = o.build_model("matern52", X, np.full((10, 1), 3.0), 1.0, [0.3, 0.3], 1e-3, 3.0)  # y == mean: alpha = 0
    L, eta = lp.lipschitz_and_eta(om, np.concatenate([X, np.random.default_rng(1).uniform(size=(50, 2))]))
    assert L == 10.0 and eta == pytest.approx(3.0)


# ---- the builder protocol on a model whose predictions come from the oracle (nothing runs on a device) ----
def _oracle_backed(om):
    import trieste_b200 as tb

    class OracleBacked(tb.GaussianProcessRegression):
        def __init__(self):  # no native handle
            self._h = None
            self._dtype = np.float64
            self._spec = tb.GPRSpec((om.X, om.y), tb.Matern52(om.variance, om.lengthscales), tb.Constant(om.mean_const), om.noise)

        def predict(self, x):
            return o.predict(om, np.asarray(x))

        def mean_gradient(self, x):
            x = np.asarray(x)
            return o.predict(om, x)[0], o.posterior_gradients(om, x)[0]

    return OracleBacked()


def test_two_stage_eta_identity_on_update_and_errors():
    import trieste_b200 as tb
    from trieste_b200.acquisition import (ExpectedImprovement, LocalPenalization, LogExpectedImprovement,
                                          NegativeLowerConfidenceBound, PenalizedAcquisition, expected_improvement,
                                          soft_local_penalizer)

    om = o.synthetic_model(o.branin, 15, 2, seed=6)  # a data set whose mean is lowest away from the data
    model = _oracle_backed(om)
    ds = tb.Dataset(om.X, om.y)
    space = lp.seeded_space([0.0, 0.0], [1.0, 1.0], seed=7)
    builder = LocalPenalization(space, num_samples=200)
    fn = builder.prepare_acquisition_function(model, ds)
    L, eta = lp.lipschitz_and_eta(om, np.concatenate([om.X, space.drawn[0]]))
    assert type(fn) is expected_improvement
    assert builder.lipschitz_constant == pytest.approx(L, rel=1e-12) and builder.eta == pytest.approx(eta, rel=1e-12)
    assert fn.eta == pytest.approx(eta, rel=1e-12)  # first step: the LP eta (samples and data), greedy_batch.py:237-241
    assert eta < o.ei_eta(om)
    pending = np.array([[0.2, 0.3]])
    pen_fn = builder.update_acquisition_function(fn, model, ds, pending_points=pending, new_optimization_step=False)
    assert isinstance(pen_fn, PenalizedAcquisition) and isinstance(pen_fn._penalization, soft_local_penalizer)
    radius, scale = lp.penalizer_state(om, pending, L, eta)
    np.testing.assert_allclose(pen_fn._penalization.radius, radius, rtol=1e-12)
    np.testing.assert_allclose(pen_fn._penalization.scale, scale, rtol=1e-12)
    again = builder.update_acquisition_function(pen_fn, model, ds, pending_points=np.array([[0.2, 0.3], [0.9, 0.1]]),
                                                new_optimization_step=False)
    assert again is pen_fn and pen_fn._penalization.pending_points.shape == (2, 2)
    # a new optimisation step: the base builder's own update resets eta to min mean over the data (:231-236)
    base = builder.update_acquisition_function(pen_fn, model, ds, pending_points=None, new_optimization_step=True)
    assert base is fn and fn.eta == pytest.approx(o.ei_eta(om), rel=1e-12)
    L2, eta2 = lp.lipschitz_and_eta(om, np.concatenate([om.X, space.drawn[1]]))
    assert builder.lipschitz_constant == pytest.approx(L2, rel=1e-12) and builder.eta == pytest.approx(eta2, rel=1e-12)
    assert builder.update_acquisition_function(base, model, ds, pending_points=pending, new_optimization_step=False) is pen_fn
    # errors
    with pytest.raises(ValueError):
        LocalPenalization(space, num_samples=0)
    with pytest.raises(ValueError):
        LocalPenalization(space, num_samples=-5)
    with pytest.raises(ValueError):
        LocalPenalization(space).prepare_acquisition_function(model, None)
    with pytest.raises(ValueError):
        LocalPenalization(space).prepare_acquisition_function(model, tb.Dataset(np.zeros((0, 2)), np.zeros((0, 1))))
    for bad in (np.array([0.0, 0.1]), np.zeros((1, 2, 2))):
        with pytest.raises(ValueError):
            LocalPenalization(space).prepare_acquisition_function(model, ds, bad)
    with pytest.raises(ValueError, match="ExpectedImprovement and MinValueEntropySearch"):
        LocalPenalization(space, base_acquisition_function_builder=LogExpectedImprovement())
    with pytest.raises(ValueError, match="ExpectedImprovement and MinValueEntropySearch"):
        LocalPenalization(space, base_acquisition_function_builder=NegativeLowerConfidenceBound())
    with pytest.raises(ValueError, match="soft_local_penalizer or hard_local_penalizer"):
        LocalPenalization(space, penalizer=lambda model, pending, L, eta: None)
    assert type(LocalPenalization(space, base_acquisition_function_builder=ExpectedImprovement())) is LocalPenalization
