"""Rank-m append of the posterior cache (tb_gp_append_data; SURVEY.md §8f-1) against the oracle's from-scratch cache
(interface.py:108-112) on the grown data set, and against the library's own full refactorisation."""
import numpy as np
import pytest

from oracle import gp_oracle as o
from tests.util import candidates, native_from_oracle

pytestmark = pytest.mark.gpu


def _grown(objective, N0, m, D, kind="matern52", dtype=np.float64):
    full = o.synthetic_model(objective, N0 + m, D, kind=kind, dtype=dtype)
    head = o.build_model(kind, full.X[:N0], full.y[:N0], full.variance, full.lengthscales, full.noise, full.mean_const)
    return head, full


@pytest.mark.parametrize("engine", ["int8", "int8x21", "fp64"])
@pytest.mark.parametrize("N0,m", [(1, 1), (127, 1), (127, 2), (128, 1), (300, 5), (250, 64), (1000, 8)])
def test_append_matches_from_scratch_cache(N0, m, engine):
    import trieste_b200 as tb

    head, full = _grown(o.hartmann_6, N0, m, 6)
    nm = native_from_oracle(head)
    nm.set_engine(engine)
    nm.update(tb.Dataset(full.X, full.y))
    assert nm.last_update_appended
    L = nm.get_cholesky()
    np.testing.assert_allclose(L, full.L, rtol=0, atol=1e-9 * np.sqrt(full.variance))
    Xq = np.concatenate([candidates(700, 6), full.X[-m:]])
    mean, var = nm.predict(Xq)
    omean, ovar = o.predict(full, Xq)
    np.testing.assert_allclose(mean, omean, rtol=1e-9, atol=1e-9 * np.sqrt(full.variance))
    np.testing.assert_allclose(var, ovar, rtol=0, atol=1e-9 * full.variance)
    assert nm.get_internal_data().query_points.shape[0] == N0 + m


def test_repeated_single_appends_track_the_oracle_and_gradients_follow():
    import trieste_b200 as tb
    from trieste_b200.acquisition import expected_improvement

    head, full = _grown(o.ackley, 120, 20, 4)
    nm = native_from_oracle(head)
    for k in range(1, 21):  # twenty BO steps of one new point each, crossing the 128-row block boundary
        nm.update(tb.Dataset(full.X[: 120 + k], full.y[: 120 + k]))
        assert nm.last_update_appended
    np.testing.assert_allclose(nm.get_cholesky(), full.L, rtol=0, atol=1e-9 * np.sqrt(full.variance))
    Xq = candidates(300, 4)
    eta = o.ei_eta(full)
    fn = expected_improvement(nm, eta)
    val, grad = fn.value_and_gradient(Xq[:, None, :])
    oval, ograd = o.ei_gradient(full, Xq, eta)
    np.testing.assert_allclose(val.reshape(-1), oval.reshape(-1), rtol=1e-6, atol=1e-15)
    np.testing.assert_allclose(grad.reshape(-1, 4), ograd, rtol=1e-6, atol=1e-12)
    mj, cj = nm.predict_joint(Xq.reshape(60, 5, 4))
    omj, ocj = o.predict_joint(full, Xq.reshape(60, 5, 4))
    np.testing.assert_allclose(cj, ocj, rtol=0, atol=1e-9 * full.variance)


@pytest.mark.parametrize("engine", ["int8", "int8x21", "fp64"])
def test_gradients_between_appends_use_the_rank_m_update_of_the_inverse(engine):
    """A BO loop with a gradient-based optimiser asks for gradients after EVERY append: the dense K^-1 behind the int8
    engine's gradient GEMM is grown by rank m with the factor (O(m N^2)) instead of being rebuilt (O(N^3))."""
    import trieste_b200 as tb
    from trieste_b200.acquisition import expected_improvement

    head, full = _grown(o.hartmann_6, 250, 12, 6)
    nm = native_from_oracle(head)
    nm.set_engine(engine)
    Xq = candidates(200, 6)
    for k in (0, 1, 4, 12):  # gradients first (builds K^-1), then appends of 1, 3 and 8 rows with gradients in between
        if k:
            nm.update(tb.Dataset(full.X[: 250 + k], full.y[: 250 + k]))
            assert nm.last_update_appended
        ref = o.build_model(full.kind, full.X[: 250 + k], full.y[: 250 + k], full.variance, full.lengthscales, full.noise, full.mean_const)
        eta = o.ei_eta(ref)
        val, grad = expected_improvement(nm, eta).value_and_gradient(Xq[:, None, :])
        oval, ograd = o.ei_gradient(ref, Xq, eta)
        np.testing.assert_allclose(val.reshape(-1), oval.reshape(-1), rtol=1e-6, atol=1e-15)
        np.testing.assert_allclose(grad.reshape(-1, 6), ograd, rtol=1e-6, atol=1e-12)


def test_engine_toggles_between_appends_keep_every_result_bit_for_bit():
    """Every operand derived from the posterior cache records the cache generation it was built from.  A handle that toggles
    between the int8 engines around appends gives bit for bit what handles that never toggle give."""
    import trieste_b200 as tb
    from trieste_b200.acquisition import expected_improvement

    head, full = _grown(o.hartmann_6, 250, 9, 6)
    eta = o.ei_eta(head)
    Xq = candidates(300, 6)

    def run(nm):
        val, grad = expected_improvement(nm, eta).value_and_gradient(Xq[:, None, :])
        return np.concatenate([a.reshape(-1) for a in (val, grad, *nm.predict(Xq))])

    toggled, single, full21 = (native_from_oracle(head) for _ in range(3))
    full21.set_engine("int8x21")
    first = run(toggled)
    toggled.set_engine("int8x21")
    np.testing.assert_array_equal(run(toggled), run(full21))
    toggled.set_engine("int8")
    np.testing.assert_array_equal(run(toggled), first)
    for n in (251, 255, 259):  # appends of 1, 4 and 4 rows
        for nm in (toggled, single, full21):
            nm.update(tb.Dataset(full.X[:n], full.y[:n]))
            assert nm.last_update_appended
        ref = run(single)
        np.testing.assert_array_equal(run(toggled), ref)
        toggled.set_engine("int8x21")
        np.testing.assert_array_equal(run(toggled), run(full21))
        toggled.set_engine("int8")
        np.testing.assert_array_equal(run(toggled), ref)


def test_update_falls_back_to_a_full_refresh_when_it_is_not_an_append():
    import trieste_b200 as tb

    head, full = _grown(o.branin, 60, 70, 2)
    nm = native_from_oracle(head)
    nm.update(tb.Dataset(full.X, full.y))  # 70 new rows > 64: full refactorisation
    assert not nm.last_update_appended
    np.testing.assert_allclose(nm.get_cholesky(), full.L, rtol=0, atol=1e-9 * np.sqrt(full.variance))
    perm = np.random.default_rng(0).permutation(130)
    nm.update(tb.Dataset(full.X[perm], full.y[perm]))  # same size, different rows
    assert not nm.last_update_appended
    shuffled = o.build_model(full.kind, full.X[perm], full.y[perm], full.variance, full.lengthscales, full.noise, full.mean_const)
    np.testing.assert_allclose(nm.get_cholesky(), shuffled.L, rtol=0, atol=1e-9 * np.sqrt(full.variance))
    nm.update(tb.Dataset(full.X[perm][:40], full.y[perm][:40]))  # shrinking data set
    assert not nm.last_update_appended
    mean, _ = nm.predict(full.X[:5])
    small = o.build_model(full.kind, full.X[perm][:40], full.y[perm][:40], full.variance, full.lengthscales, full.noise, full.mean_const)
    np.testing.assert_allclose(mean, o.predict(small, full.X[:5])[0], rtol=1e-9)


def test_append_after_hyperparameter_change_and_argument_errors():
    import ctypes as C

    import trieste_b200 as tb
    from trieste_b200 import _lib

    head, full = _grown(o.hartmann_6, 200, 3, 6)
    nm = native_from_oracle(head)
    nm.set_hyperparameters(kernel=tb.Matern52(full.variance * 2.0, full.lengthscales * 1.5))
    nm.update(tb.Dataset(full.X, full.y))  # cache was rebuilt with the new kernel, so the append is legal
    assert nm.last_update_appended
    ref = o.build_model("matern52", full.X, full.y, full.variance * 2.0, full.lengthscales * 1.5, full.noise, full.mean_const)
    np.testing.assert_allclose(nm.get_cholesky(), ref.L, rtol=0, atol=1e-9 * np.sqrt(ref.variance))
    x = np.zeros((65, 6))
    y = np.zeros(65)
    with pytest.raises(ValueError):
        _lib.check(_lib.lib().tb_gp_append_data(nm.handle, x.ctypes.data, y.ctypes.data, 65))
    with pytest.raises(ValueError):
        _lib.check(_lib.lib().tb_gp_append_data(nm.handle, x.ctypes.data, y.ctypes.data, 0))
    # a stale cache (hyper-parameters pushed, cache not refreshed) must be refused
    ls = np.ascontiguousarray(full.lengthscales)
    _lib.check(_lib.lib().tb_gp_set_hyper(nm.handle, 3, 1.0, ls.ctypes.data_as(C.POINTER(C.c_double)), 6, 0.1, 0.0))
    with pytest.raises(ValueError):
        _lib.check(_lib.lib().tb_gp_append_data(nm.handle, x.ctypes.data, y.ctypes.data, 1))


def test_append_in_single_precision_models():
    import trieste_b200 as tb

    head, full = _grown(o.hartmann_6, 400, 4, 6, dtype=np.float32)
    nm = native_from_oracle(head)
    assert nm.dtype == np.float32
    nm.update(tb.Dataset(full.X, full.y))
    assert nm.last_update_appended
    Xq = candidates(500, 6).astype(np.float32)
    mean, var = nm.predict(Xq)
    assert mean.dtype == np.float32
    full64 = o.build_model(full.kind, full.X.astype(np.float64), full.y.astype(np.float64), full.variance, full.lengthscales.astype(np.float64), full.noise, full.mean_const)
    omean, ovar = o.predict(full64, Xq.astype(np.float64))
    np.testing.assert_allclose(mean, omean, rtol=1e-4, atol=1e-4 * np.sqrt(full.variance))
    np.testing.assert_allclose(var, ovar, rtol=0, atol=1e-4 * full.variance)


@pytest.mark.parametrize("n2", [1, 3, 40])
def test_conditional_predictions_equal_a_model_updated_with_the_additional_data(n2):
    # models.py:355-525 (reference test: test_gpflow_models_conditional_predict, tests/unit/models/gpflow/test_models.py):
    # the exact update formulas must reproduce the posterior of a model that has seen the additional data
    import trieste_b200 as tb

    head, full = _grown(o.hartmann_6, 150, n2, 6)
    nm = native_from_oracle(head)
    Xq = candidates(257, 6)
    add = tb.Dataset(full.X[150:], full.y[150:])
    mean, var = nm.conditional_predict_f(Xq, add)
    omean, ovar = o.predict_f(full, Xq)
    assert mean.shape == (257, 1) and var.shape == (257, 1)
    np.testing.assert_allclose(mean, omean, rtol=1e-8, atol=1e-8 * np.sqrt(full.variance))
    np.testing.assert_allclose(var, ovar, rtol=0, atol=1e-8 * full.variance)
    my, vy = nm.conditional_predict_y(Xq, add)
    np.testing.assert_allclose(vy, ovar + full.noise, rtol=0, atol=1e-8 * full.variance)
    mj, cj = nm.conditional_predict_joint(Xq[:50], add)
    _, ocov = o.predict_f(full, Xq[:50], full_cov=True)
    assert mj.shape == (50, 1) and cj.shape == (1, 50, 50)
    np.testing.assert_allclose(cj[0], ocov, rtol=0, atol=1e-8 * full.variance)
    np.testing.assert_allclose(mj, omean[:50], rtol=1e-8, atol=1e-8 * np.sqrt(full.variance))
    # leading dimensions: two different fantasised observation sets at the same points
    Xa = np.stack([full.X[150:], full.X[150:]])
    Ya = np.stack([full.y[150:], full.y[150:] + 1.0])
    m2, v2 = nm.conditional_predict_f(Xq, tb.Dataset(Xa, Ya))
    assert m2.shape == (2, 257, 1) and v2.shape == (2, 257, 1)
    np.testing.assert_allclose(m2[0], mean, rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(v2[1], var, rtol=1e-8, atol=1e-10)  # the variance does not depend on the observations
    assert not np.allclose(m2[1], mean)
    with pytest.raises(ValueError):
        nm.conditional_predict_f(Xq[None], add)  # query points must be [M, D]
    # the model itself is untouched
    np.testing.assert_allclose(nm.predict(Xq)[0], o.predict(head, Xq)[0], rtol=1e-9)
