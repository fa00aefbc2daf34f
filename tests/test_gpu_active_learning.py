"""GPU: the active-learning acquisitions (trieste/acquisition/function/active_learning.py) against the NumPy restatement in
tests/al_oracle.py — the feasibility criteria (delta = 1, 2), BALD and the predictive variance: values and gradients on every
engine, fp32 handles, the fused argmax, the device L-BFGS against SciPy, handle isolation of alpha, q-batches of the
predictive variance through the joint chain, one EfficientGlobalOptimization acquire over space ** 4, and a short BO loop.

Tolerances.  Values: rtol 1e-9 plus the engine's stated variance error (ENGINE_VAR_EPS sigma_f^2, as in
tests/test_gpu_gibbon.py) times |d value / d var| at each point.  Gradients: 1e-6 of each point's largest component plus
1e-9 of the largest over the set (the V = K^-1 k* digit GEMM errs far below that)."""
import numpy as np
import pytest

from oracle import gp_oracle as o
from tests import al_oracle as al
from tests.util import candidates, model_pair

pytestmark = pytest.mark.gpu

ENGINE_VAR_EPS = {"int8": 1e-9, "int8x21": 1e-9, "fp64": 1e-12}  # stated |delta var| / sigma_f^2 per engine
KINDS = ["bichon", "ranjan", "bald", "pv"]


def _threshold(om):
    return float(np.median(om.y))


def _function(kind, nm, om, alpha=1.0):
    from trieste_b200.acquisition import bayesian_active_learning_by_disagreement, bichon_ranjan_criterion, predictive_variance

    if kind == "bichon":
        return bichon_ranjan_criterion(nm, _threshold(om), alpha, 1)
    if kind == "ranjan":
        return bichon_ranjan_criterion(nm, _threshold(om), alpha, 2)
    if kind == "bald":
        return bayesian_active_learning_by_disagreement(nm, 1e-6)
    return predictive_variance(nm, 1e-6)


def _oracle(kind, om, X, alpha=1.0):
    """(value [M, 1], grad [M, D], |d value / d var| [M, 1]) of the kind at X"""
    if kind in ("bichon", "ranjan"):
        args = (al.feasibility, al.feasibility_partials, _threshold(om), alpha, 1 if kind == "bichon" else 2)
    elif kind == "bald":
        args = (al.bald, al.bald_partials, 1e-6)
    else:
        args = (al.predictive_variance_single, al.predictive_variance_single_partials, 1e-6)
    value, grad = al.single_query(om, X, *args)
    mean, var = o.predict(om, X)
    _, dv = args[1](mean, var, *args[2:])
    return value, grad, np.abs(dv)


def _query_set(om, M=3000):
    """random candidates (far from most data), the training inputs, and points whose mean is near the threshold"""
    X = candidates(M, om.X.shape[1], seed=2)
    mean, _ = o.predict(om, X)
    near = X[np.argsort(np.abs(mean[:, 0] - _threshold(om)))[:200]]
    far = np.clip(candidates(100, om.X.shape[1], seed=3) * 3.0 - 1.0, -1.0, 2.0)
    return np.concatenate([X, om.X[:100], near, far])


def _assert_values(got, ref, dv, om, engine):
    err = np.abs(got - ref)
    assert np.all(err <= 1e-9 * np.abs(ref) + 1e-14 + 2.0 * ENGINE_VAR_EPS[engine] * om.variance * dv), err.max()


def _assert_gradients(got, ref):
    scale = np.abs(ref).max(axis=1, keepdims=True)
    err = np.abs(got - ref)
    assert np.all(err <= 1e-6 * scale + 1e-9 * np.abs(ref).max()), (err.max(), int(np.argmax(err.max(axis=1))))


# ---- 1. values and gradients on every engine ------------------------------------------------------------------------------
@pytest.mark.parametrize("engine", ["int8", "int8x21", "fp64"])
@pytest.mark.parametrize("kind", KINDS)
def test_values_and_gradients_match_oracle(kind, engine):
    om, nm = model_pair(o.hartmann_6, 300, 6, engine=engine)
    X = _query_set(om)
    fn = _function(kind, nm, om)
    ref, gref, dv = _oracle(kind, om, X)
    got = fn(X[:, None, :])
    assert got.shape == (X.shape[0], 1)
    _assert_values(got, ref, dv, om, engine)
    val, grad = fn.value_and_gradient(X[:, None, :])
    assert grad.shape == (X.shape[0], 1, 6)
    _assert_values(val, ref, dv, om, engine)
    _assert_gradients(grad[:, 0, :], gref)


@pytest.mark.parametrize("kind", KINDS)
def test_clipped_variance_has_zero_variance_gradient(kind):
    """a model with posterior variances below the 1e-12 clip near its data: d/dvar is 0 there, as the oracle's"""
    small = lambda x: 1e-4 * o.hartmann_6(x)
    om0 = o.synthetic_model(small, 300, 6)
    om, nm = model_pair(small, 300, 6, noise=1e-7 * om0.variance, engine="fp64")
    rng = np.random.default_rng(8)
    u = rng.standard_normal((8, 6))
    X = om.X[:8] + 1e-3 * u / np.linalg.norm(u, axis=1, keepdims=True)
    assert np.all(o.predict_f(om, X)[1] < 1e-12)
    fn = _function(kind, nm, om)
    ref, gref, _ = _oracle(kind, om, X)
    val, grad = fn.value_and_gradient(X[:, None, :])
    np.testing.assert_allclose(val, ref, rtol=1e-9, atol=1e-14)
    assert np.all(np.isfinite(grad))
    scale = np.abs(o.posterior_gradients(om, X)[0]).max()  # d mean / dx: the size of a gradient the mean partial carries
    np.testing.assert_allclose(grad[:, 0, :], gref, rtol=1e-6, atol=1e-9 * scale)


# ---- 2. fp32 handles ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_fp32_handles(kind):
    import trieste_b200 as tb

    om = o.synthetic_model(o.hartmann_6, 300, 6)
    X32, y32 = om.X.astype(np.float32), om.y.astype(np.float32)
    om32 = o.build_model(om.kind, X32.astype(np.float64), y32.astype(np.float64), om.variance, om.lengthscales, om.noise, om.mean_const)
    nm = tb.GaussianProcessRegression(tb.GPRSpec((X32, y32), tb.Matern52(om.variance, om.lengthscales), tb.Constant(om.mean_const), om.noise))
    X = candidates(3000, 6).astype(np.float32)
    fn = _function(kind, nm, om32)
    ref, gref, dv = _oracle(kind, om32, X.astype(np.float64))
    val, grad = fn.value_and_gradient(X[:, None, :])
    assert val.dtype == np.float32 and grad.dtype == np.float32
    # the stated fp32 variance tolerance 1e-4 sigma_f^2, carried through d value / d var, plus the mean's 1e-4 sigma_f
    _, _, dm = _oracle_mean_partial(kind, om32, X.astype(np.float64))
    atol = 1e-4 * om.variance * dv + 1e-4 * np.sqrt(om.variance) * dm + 1e-6
    assert np.all(np.abs(val - ref) <= 1e-4 * np.abs(ref) + atol)
    err = np.abs(grad[:, 0, :].astype(np.float64) - gref)
    assert np.all(err <= 1e-3 * np.abs(gref).max(axis=1, keepdims=True) + 1e-4 * np.abs(gref).max()), err.max()
    idx, best = fn.fused_argmax(X)
    assert ref[idx, 0] >= ref.max() - 1e-4 * max(1.0, abs(ref.max()))


def _oracle_mean_partial(kind, om, X):
    mean, var = o.predict(om, X)
    if kind in ("bichon", "ranjan"):
        dm, _ = al.feasibility_partials(mean, var, _threshold(om), 1.0, 1 if kind == "bichon" else 2)
    elif kind == "bald":
        dm, _ = al.bald_partials(mean, var, 1e-6)
    else:
        dm = np.zeros_like(mean)
    return mean, var, np.abs(dm)


# ---- 3. fused argmax across chunks ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_fused_argmax_across_chunks(kind):
    om, nm = model_pair(o.hartmann_6, 300, 6, engine="fp64")
    X = np.concatenate([candidates(300_000, 6, seed=5), _query_set(om, 100)])  # more than one chunk of candidates
    fn = _function(kind, nm, om)
    idx, best = fn.fused_argmax(X)
    mean, var = o.predict_batched(om, X)
    if kind in ("bichon", "ranjan"):
        ref = al.feasibility(mean, var, _threshold(om), 1.0, 1 if kind == "bichon" else 2)
    elif kind == "bald":
        ref = al.bald(mean, var, 1e-6)
    else:
        ref = al.predictive_variance_single(mean, var, 1e-6)
    tol = 1e-9 * abs(ref.max()) + 1e-10 * np.sqrt(om.variance)
    assert ref[idx, 0] >= ref.max() - tol, (idx, ref[idx, 0], ref.max())
    assert abs(best - ref[idx, 0]) <= tol


# ---- 4. device L-BFGS against SciPy L-BFGS-B on the oracle -----------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_device_optimiser_against_scipy_lbfgsb_on_the_oracle(kind):
    om, nm = model_pair(o.hartmann_6, 300, 6)
    fn = _function(kind, nm, om)
    lower, upper = np.zeros(6), np.ones(6)
    x0 = candidates(64, 6, seed=11)

    def oracle_vg(x):
        v, g, _ = _oracle(kind, om, x)
        return v[:, 0], g

    ok_d, f_d, x_d, _ = fn.maximize_from(x0, lower, upper)
    ok_s, f_s, _, _ = o.scipy_lbfgsb_multistart(oracle_vg, x0, lower, upper)
    scale = max(1.0, np.abs(f_s).max())
    assert f_d.max() >= f_s.max() - 1e-6 * scale, (f_d.max(), f_s.max())
    fo, _ = oracle_vg(x_d)
    np.testing.assert_allclose(f_d, fo, rtol=1e-6, atol=1e-7 * scale)
    assert ok_d.mean() >= 0.9
    assert np.median(f_d) >= np.median(f_s) - 0.02 * scale


# ---- 5. handle isolation --------------------------------------------------------------------------------------------------
def test_two_alphas_and_ei_on_one_model_do_not_interfere():
    from trieste_b200.acquisition import bichon_ranjan_criterion, expected_improvement

    om, nm = model_pair(o.hartmann_6, 300, 6, engine="fp64")
    X = _query_set(om, 500)
    T = _threshold(om)
    f1 = bichon_ranjan_criterion(nm, T, 0.5, 1)
    f2 = bichon_ranjan_criterion(nm, T, 2.0, 2)
    ei = expected_improvement(nm, o.ei_eta(om))
    mean, var = o.predict(om, X)
    r1, r2 = al.feasibility(mean, var, T, 0.5, 1), al.feasibility(mean, var, T, 2.0, 2)
    rei = o.expected_improvement(mean, var, o.ei_eta(om))
    for _ in range(2):
        for fn, ref in ((f1, r1), (ei, rei), (f2, r2), (f1, r1), (f2, r2)):
            np.testing.assert_allclose(fn(X[:, None, :]), ref, rtol=1e-9, atol=1e-12)
        i1, _ = f1.fused_argmax(X)
        i2, _ = f2.fused_argmax(X)
        assert r1[i1, 0] >= r1.max() - 1e-9 * abs(r1.max()) and r2[i2, 0] >= r2.max() - 1e-9 * abs(r2.max())


def test_native_argument_errors():
    import ctypes as C

    from trieste_b200 import _lib

    om, nm = model_pair(o.hartmann_6, 50, 6)
    lib = _lib.lib()
    for bad in (0.0, -1.0, float("inf"), float("nan")):
        assert lib.tb_acq_set_feasibility(nm.handle, bad) == _lib.TB_ERR_INVALID
    X = np.ascontiguousarray(candidates(4, 6))
    out = np.empty(4)
    best, idx = C.c_double(), C.c_int64()
    assert lib.tb_acq_argmax(nm.handle, _lib.ACQ_BALD, 0.0, X.ctypes.data, 4, None, C.byref(best), C.byref(idx)) == _lib.TB_ERR_INVALID
    assert "Jitter must be positive" in _lib.last_error()
    assert lib.tb_acq_eval(nm.handle, 14, 0.0, X.ctypes.data, 4, out.ctypes.data, None) == _lib.TB_ERR_INVALID
    Xb = np.ascontiguousarray(candidates(33 * 2, 6).reshape(2, 33, 6))
    assert lib.tb_acq_predictive_variance(nm.handle, Xb.ctypes.data, 2, 33, 1e-6, out.ctypes.data, None) == _lib.TB_ERR_INVALID
    # a jitter below minus the prior variance leaves a negative first pivot: the Cholesky error
    Xr = np.ascontiguousarray(candidates(2, 6, seed=6)[None])
    assert lib.tb_acq_predictive_variance(nm.handle, Xr.ctypes.data, 1, 2, -10.0 * om.variance, out.ctypes.data, None) == _lib.TB_ERR_NUMERIC
    assert "Cholesky decomposition was not successful" in _lib.last_error()


# ---- 6. q-batches of the predictive variance ------------------------------------------------------------------------------
@pytest.mark.parametrize("engine", ["int8", "fp64"])
@pytest.mark.parametrize("q", [2, 4, 8, 32])
def test_batch_predictive_variance_values_and_gradients(q, engine):
    from trieste_b200.acquisition import predictive_variance

    om, nm = model_pair(o.hartmann_6, 300, 6, engine=engine)
    B = 300_000 // q + 7  # more than one chunk of whole batches (at most 2112 tiles of 128 candidates per chunk)
    Xb = candidates(B * q, 6, seed=q).reshape(B, q, 6)
    fn = predictive_variance(nm, 1e-6)
    got = fn(Xb)
    val, grad = fn.value_and_gradient(Xb)
    np.testing.assert_array_equal(val, got)
    pick = np.unique(np.concatenate([np.arange(4), np.linspace(0, B - 1, 12).astype(int)]))
    ref = al.predictive_variance(om, Xb[pick], 1e-6)[:, 0]
    for i, b in enumerate(pick):
        v, g = al.predictive_variance_gradient(om, Xb[b], 1e-6)
        assert v == pytest.approx(ref[i], rel=1e-12)
        # det(M) moves by det(M) tr(M^-1 dM): an error eps in each entry of cov changes it by at most det(M) sum |M^-1| eps
        _, cov = o.predict_joint(om, Xb[b][None])
        Minv = np.linalg.inv(al.pv_matrix(cov[0, 0], 1e-6))
        tol = 1e-9 * abs(v) + 4.0 * ENGINE_VAR_EPS[engine] * om.variance * abs(v) * np.abs(Minv).sum()
        assert abs(got[b, 0] - v) <= tol, (b, got[b, 0], v)
        scale = np.abs(g).max()
        err = np.abs(grad[b] - g)
        assert np.all(err <= 1e-6 * scale + 1e-6 * tol), (b, err.max(), scale)


def test_q1_batch_matches_the_single_query_kind():
    from trieste_b200 import _lib
    from trieste_b200.acquisition import predictive_variance

    om, nm = model_pair(o.hartmann_6, 300, 6, engine="fp64")
    X = candidates(2000, 6, seed=4)
    fn = predictive_variance(nm, 1e-6)
    single, gsingle = fn.value_and_gradient(X[:, None, :])
    out, grad = np.empty(2000), np.empty((2000, 1, 6))
    Xc = np.ascontiguousarray(X[:, None, :])
    _lib.check(_lib.lib().tb_acq_predictive_variance(nm.handle, Xc.ctypes.data, 2000, 1, 1e-6, out.ctypes.data, grad.ctypes.data))
    np.testing.assert_allclose(out, single[:, 0], rtol=1e-13)
    np.testing.assert_allclose(grad, gsingle, rtol=1e-9, atol=1e-12 * np.abs(gsingle).max())


def test_ego_joint_batch_beats_its_initial_batches():
    import trieste_b200 as tb
    from trieste_b200.acquisition import PredictiveVariance
    from trieste_b200.acquisition.optimizer import generate_continuous_optimizer
    from trieste_b200.rule import EfficientGlobalOptimization

    om, nm = model_pair(o.hartmann_6, 300, 6)
    space = tb.Box([0.0] * 6, [1.0] * 6)
    opt = generate_continuous_optimizer(num_initial_samples=2000, num_optimization_runs=8)
    rule = EfficientGlobalOptimization(PredictiveVariance(), optimizer=opt, num_query_points=4)
    pts = rule.acquire_single(space, nm, tb.Dataset(om.X, om.y))
    assert pts.shape == (4, 6) and np.all((pts >= 0.0) & (pts <= 1.0))
    assert opt.last_stats["spo_improvement_on_initial_samples"]() >= 0.0
    fn = rule.acquisition_function
    np.testing.assert_allclose(fn(pts[None]), al.predictive_variance(om, pts[None], 1e-6), rtol=1e-6)


# ---- 7. a short BO loop ---------------------------------------------------------------------------------------------------
def test_expected_feasibility_bo_loop_on_branin_runs_through_the_device_route(monkeypatch):
    import trieste_b200 as tb
    from trieste_b200.acquisition import ExpectedFeasibility
    from trieste_b200.acquisition import active_learning as a
    from trieste_b200.bayesian_optimizer import BayesianOptimizer
    from trieste_b200.rule import EfficientGlobalOptimization

    calls = {"maximize_from": 0}
    orig = a.bichon_ranjan_criterion.maximize_from

    def counted(self, *args, **kw):
        calls["maximize_from"] += 1
        return orig(self, *args, **kw)

    monkeypatch.setattr(a.bichon_ranjan_criterion, "maximize_from", counted)
    space = tb.Box([0.0, 0.0], [1.0, 1.0])
    X0 = space.sample(8, seed=0)
    ds = tb.Dataset(X0, o.branin(X0))
    model = tb.GaussianProcessRegression(tb.build_gpr(ds, space, likelihood_variance=1e-7))
    threshold = 20.0
    rule = EfficientGlobalOptimization(ExpectedFeasibility(threshold, delta=2))
    result = BayesianOptimizer(o.branin, space).optimize(6, ds, model, rule)
    final = result.try_get_final_dataset()
    assert len(final) == 14 and len(result.history) == 6
    assert calls["maximize_from"] == 6
    new = np.asarray(final.observations)[8:, 0]
    assert np.all(np.isfinite(new))
