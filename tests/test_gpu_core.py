"""GPU parity: predict / EI / log-EI / LCB / argmax through the C-ABI vs the oracle.

Stated fp64 tolerances (SURVEY.md §8c): mean rtol 1e-9 (+ atol 1e-9 sigma_f), variance
atol 1e-9 * sigma_f^2, EI rtol 1e-6 where EI > 1e-12 else atol 1e-15."""
import numpy as np
import pytest

from oracle import gp_oracle as o
from tests.util import candidates, model_pair

pytestmark = pytest.mark.gpu


def _check_predict(om, nm, Xq):
    mean, var = nm.predict(Xq)
    omean, ovar = o.predict_batched(om, Xq)
    assert mean.shape == omean.shape == (Xq.shape[0], 1) and var.shape == ovar.shape
    sf = np.sqrt(om.variance)
    # Matern12 = exp(-r) is not differentiable at r = 0: GPflow's expansion-form r^2 leaves O(1e-16)
    # noise on the diagonal of K(X,X), which sqrt() turns into an O(1e-8) relative perturbation of k(x,x)
    # (then amplified by cond(K)).  The reference's own result is only defined to ~1e-6 there; the CUDA
    # path uses the exact difference form.  All smooth kernels are held to the 1e-9 bar.
    tol = 1e-5 if om.kind == "matern12" else 1e-9
    np.testing.assert_allclose(mean, omean, rtol=tol, atol=tol * sf)
    np.testing.assert_allclose(var, ovar, rtol=0, atol=tol * om.variance)
    assert var.min() >= 1e-12
    return mean, var, omean, ovar


@pytest.mark.parametrize("engine", ["int8", "int8x21", "fp64"])
@pytest.mark.parametrize("kind", ["matern52", "rbf", "matern32", "matern12"])
@pytest.mark.parametrize("N,D", [(5, 2), (20, 2), (127, 3), (128, 6), (129, 6), (300, 6), (1024, 6)])
def test_predict_matches_oracle(kind, N, D, engine):
    obj = o.branin if D == 2 else (o.hartmann_6 if D == 6 else o.ackley)
    om, nm = model_pair(obj, N, D, kind=kind, engine=engine)
    _check_predict(om, nm, candidates(777, D))


def test_predict_at_training_points_and_clip():
    # near-noiseless model queried at its own training inputs: variance collapses and must clip to 1e-12
    om, nm = model_pair(o.branin, 20, 2, noise=1e-7)
    mean, var, omean, ovar = _check_predict(om, nm, om.X.copy())
    assert var.min() >= 1e-12


def test_predict_leading_dims_and_empty():
    om, nm = model_pair(o.hartmann_6, 64, 6)
    X = candidates(60, 6).reshape(3, 4, 5, 6)
    mean, var = nm.predict(X)
    omean, ovar = o.predict(om, X.reshape(-1, 6))
    assert mean.shape == (3, 4, 5, 1)
    np.testing.assert_allclose(mean.reshape(-1, 1), omean, rtol=1e-9, atol=1e-9)
    m0, v0 = nm.predict(np.zeros((0, 6)))
    assert m0.shape == (0, 1) and v0.shape == (0, 1)
    with pytest.raises(ValueError):
        nm.predict(np.zeros((4, 5)))


def test_config2_slice_n1024_large_batch():
    # C2 shape (Hartmann6, N=1024) on a 200k slice: several chunks, G=1 path
    om, nm = model_pair(o.hartmann_6, 1024, 6)
    Xq = candidates(200_000, 6)
    mean, var = nm.predict(Xq)
    idx = np.random.default_rng(3).choice(Xq.shape[0], 4096, replace=False)
    omean, ovar = o.predict(om, Xq[idx])
    np.testing.assert_allclose(mean[idx], omean, rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(var[idx], ovar, rtol=0, atol=1e-9 * om.variance)


@pytest.mark.parametrize("engine", ["int8", "int8x21", "fp64"])
def test_headline_n4096_d10(engine):
    om, nm = model_pair(o.ackley, 4096, 10, engine=engine)
    Xq = candidates(3000, 10)
    _check_predict(om, nm, Xq)


@pytest.mark.parametrize("N,D", [(20, 2), (300, 6), (1024, 6)])
def test_expected_improvement_and_argmax(N, D):
    from trieste_b200 import Dataset
    from trieste_b200.acquisition import ExpectedImprovement, LogExpectedImprovement

    obj = o.branin if D == 2 else o.hartmann_6
    om, nm = model_pair(obj, N, D)
    Xq = candidates(5000, D)
    ds = Dataset(om.X, om.y)
    fn = ExpectedImprovement().prepare_acquisition_function(nm, ds)
    eta = o.ei_eta(om)
    assert abs(fn.eta - eta) <= 1e-9 * max(1.0, abs(eta))
    ei = fn(Xq[:, None, :])
    omean, ovar = o.predict(om, Xq)
    oei = o.expected_improvement(omean, ovar, eta)
    assert ei.shape == (5000, 1)
    big = oei > 1e-12
    np.testing.assert_allclose(ei[big], oei[big], rtol=1e-6)
    np.testing.assert_allclose(ei[~big], oei[~big], rtol=0, atol=1e-15)
    idx, best = fn.fused_argmax(Xq)
    assert idx == int(np.argmax(ei[:, 0]))
    assert best == ei[idx, 0]
    # log-EI (ours): equals log of the oracle EI wherever that is representable
    lfn = LogExpectedImprovement().prepare_acquisition_function(nm, ds)
    lei = lfn(Xq[:, None, :])
    ok = oei > 1e-300
    np.testing.assert_allclose(lei[ok], np.log(oei[ok]), rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(lei, o.log_expected_improvement(omean, ovar, eta), rtol=1e-6, atol=1e-6)
    assert np.all(np.isfinite(lei))
    with pytest.raises(ValueError):
        fn(Xq[:10].reshape(5, 2, D))  # batch size 2 is rejected (function.py:216-219)


def test_update_returns_same_function_object():
    from trieste_b200 import Dataset
    from trieste_b200.acquisition import ExpectedImprovement

    om, nm = model_pair(o.branin, 20, 2)
    b = ExpectedImprovement()
    fn = b.prepare_acquisition_function(nm, Dataset(om.X, om.y))
    fn2 = b.update_acquisition_function(fn, nm, Dataset(om.X, om.y))
    assert fn2 is fn
    with pytest.raises(ValueError):
        b.prepare_acquisition_function(nm, Dataset(np.zeros((0, 2)), np.zeros((0, 1))))


def test_lower_confidence_bound_closed_form():
    # reference known answer (tests/unit/acquisition/function/test_function.py:786-790 restated):
    # LCB = mean - beta sqrt(var), negated by the builder
    from trieste_b200.acquisition import NegativeLowerConfidenceBound, lower_confidence_bound

    om, nm = model_pair(o.hartmann_6, 200, 6)
    Xq = candidates(2000, 6)
    omean, ovar = o.predict(om, Xq)
    for beta in [0.0, 1.96, 3.0]:
        lcb = lower_confidence_bound(nm, beta)(Xq[:, None, :])
        np.testing.assert_allclose(lcb, o.lower_confidence_bound(omean, ovar, beta), rtol=1e-9, atol=1e-9)
        neg = NegativeLowerConfidenceBound(beta).prepare_acquisition_function(nm)(Xq[:, None, :])
        np.testing.assert_allclose(neg, -lcb, rtol=0, atol=0)
    with pytest.raises(ValueError):
        lower_confidence_bound(nm, -1.0)


def test_update_refreshes_cache():
    from trieste_b200 import Dataset

    om, nm = model_pair(o.hartmann_6, 100, 6)
    rng = np.random.default_rng(9)
    Xn = rng.uniform(size=(37, 6))
    X2 = np.concatenate([om.X, Xn])
    y2 = np.concatenate([om.y, o.hartmann_6(Xn)])
    nm.update(Dataset(X2, y2))
    om2 = o.build_model(om.kind, X2, y2, om.variance, om.lengthscales, om.noise, om.mean_const)
    _check_predict(om2, nm, candidates(500, 6))
    L = nm.get_cholesky()
    np.testing.assert_allclose(L, om2.L, rtol=1e-10, atol=1e-12)


def test_device_resident_torch_io():
    import torch

    om, nm = model_pair(o.hartmann_6, 256, 6)
    Xq = candidates(4096, 6)
    xt = torch.from_numpy(Xq).cuda()
    mean, var = nm.predict(xt)
    assert mean.is_cuda and mean.shape == (4096, 1)
    omean, ovar = o.predict(om, Xq)
    np.testing.assert_allclose(mean.cpu().numpy(), omean, rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(var.cpu().numpy(), ovar, rtol=0, atol=1e-9 * om.variance)


def test_probability_of_improvement_and_feasibility():
    from trieste_b200 import Dataset
    from trieste_b200.acquisition import ProbabilityOfFeasibility, ProbabilityOfImprovement

    om, nm = model_pair(o.hartmann_6, 200, 6)
    Xq = candidates(3000, 6)
    omean, ovar = o.predict(om, Xq)
    ds = Dataset(om.X, om.y)
    b = ProbabilityOfImprovement()
    fn = b.prepare_acquisition_function(nm, ds)
    np.testing.assert_allclose(fn(Xq[:, None, :]), o.probability_below_threshold(omean, ovar, o.ei_eta(om)), rtol=1e-7, atol=1e-15)
    assert b.update_acquisition_function(fn, nm, ds) is fn
    pof = ProbabilityOfFeasibility(-0.5).prepare_acquisition_function(nm)
    ref = o.probability_below_threshold(omean, ovar, -0.5)
    val, grad = pof.value_and_gradient(Xq[:100, None, :])
    np.testing.assert_allclose(val, ref[:100], rtol=1e-7, atol=1e-15)
    h = 1e-6
    e = np.zeros(6)
    e[2] = h
    fd = (pof((Xq[:100] + e)[:, None, :]) - pof((Xq[:100] - e)[:, None, :])) / (2 * h)
    np.testing.assert_allclose(grad[:, 0, 2], fd[:, 0], rtol=2e-4, atol=1e-6 * np.abs(grad).max())


@pytest.mark.parametrize("N,D,noise", [(5, 2, None), (128, 6, None), (129, 6, None), (300, 6, None), (1024, 6, None), (700, 2, 0.05)])
def test_handwritten_factorisation_matches_cusolver_and_oracle(N, D, noise, monkeypatch):
    # posterior-cache precompute (interface.py:89-112): hand-written blocked Cholesky / Linv / alpha (factor.cuh, default)
    # against the cuSOLVER + cuBLAS cross-check path and the oracle's LAPACK factor
    obj = o.branin if D == 2 else o.hartmann_6
    om, nm = model_pair(obj, N, D, noise=noise)
    monkeypatch.setenv("TB_FACTOR", "cusolver")
    from tests.util import native_from_oracle

    ref = native_from_oracle(om)
    monkeypatch.delenv("TB_FACTOR")
    L, Lr = nm.get_cholesky(), ref.get_cholesky()
    scale = np.abs(om.L).max()
    # ill-conditioned case (cond(K) ~ 4e7): the entries of L are only determined to ~cond * eps by ANY factorisation
    ltol = 1e-9 if noise is None else 1e-5
    np.testing.assert_allclose(L, om.L, rtol=ltol, atol=ltol * 1e-2 * scale)
    np.testing.assert_allclose(L, Lr, rtol=ltol, atol=ltol * 1e-2 * scale)
    Xq = candidates(400, D)
    m1, v1 = nm.predict(Xq)
    m2, v2 = ref.predict(Xq)
    tol = 1e-9 if noise is None else 1e-7  # Branin: Var(y) ~ 2.5e3, so noise 0.05 means cond(K) ~ 4e7: both factorisations are only that accurate
    np.testing.assert_allclose(m1, m2, rtol=tol, atol=tol * np.sqrt(om.variance))
    np.testing.assert_allclose(v1, v2, rtol=0, atol=tol * om.variance)
    # gradient path builds K^-1 from the hand-written Linv (kinv_kernel) vs cuSOLVER potri
    from trieste_b200.acquisition import lower_confidence_bound

    g1 = lower_confidence_bound(nm, 1.96).value_and_gradient(Xq[:64, None, :])[1]
    g2 = lower_confidence_bound(ref, 1.96).value_and_gradient(Xq[:64, None, :])[1]
    gtol = 1e-6 if noise is None else 1e-3  # K^-1 itself carries cond(K) * eps ~ 1e-8..1e-7 in the ill-conditioned case
    np.testing.assert_allclose(g1, g2, rtol=gtol, atol=gtol * 1e-2 * np.abs(g2).max())


def test_not_positive_definite_is_reported():
    import trieste_b200 as tb

    X = np.array([[0.1, 0.2], [0.1, 0.2], [0.7, 0.3]])  # duplicate point, (almost) no noise -> singular K
    spec = tb.GPRSpec((X, np.zeros((3, 1))), tb.SquaredExponential(1.0, [0.3, 0.3]), tb.Constant(0.0), 1e-300)
    with pytest.raises(ValueError, match="Cholesky decomposition was not successful"):
        tb.GaussianProcessRegression(spec)


@pytest.mark.parametrize("engine", ["int8", "fp64"])
@pytest.mark.parametrize("D", [1, 7, 19, 32])
def test_input_dimension_extremes(D, engine):
    # every padded-dimension instantiation (DP = 2 .. 32), odd D included
    om, nm = model_pair(o.ackley, 200, D, engine=engine)
    Xq = candidates(513, D)
    _check_predict(om, nm, Xq)
    with pytest.raises(ValueError):
        import trieste_b200 as tb

        tb.GaussianProcessRegression(tb.GPRSpec((np.zeros((4, 33)), np.zeros((4, 1))), tb.Matern52(1.0, np.ones(33)), tb.Constant(0.0), 0.1))


def test_single_candidate_and_single_training_point():
    from trieste_b200.acquisition import expected_improvement

    om, nm = model_pair(o.branin, 1, 2)
    _check_predict(om, nm, candidates(3, 2))
    om, nm = model_pair(o.hartmann_6, 50, 6)
    x1 = candidates(1, 6)
    mean, var = nm.predict(x1)
    omean, ovar = o.predict(om, x1)
    np.testing.assert_allclose(mean, omean, rtol=1e-9, atol=1e-9)
    idx, best = expected_improvement(nm, o.ei_eta(om)).fused_argmax(x1)
    assert idx == 0 and best == o.expected_improvement(omean, ovar, o.ei_eta(om))[0, 0] or abs(best - o.expected_improvement(omean, ovar, o.ei_eta(om))[0, 0]) < 1e-12


def test_engine_reports_the_handle_default_until_set_engine(monkeypatch):
    monkeypatch.setenv("TB_ENGINE", "fp64")  # not a knob of the library: it must not change what is reported
    om, nm = model_pair(o.branin, 20, 2)
    assert nm.engine == "int8" and nm.engine_info()[0] > 0
    nm.set_engine("fp64")
    assert nm.engine == "fp64" and nm.engine_info()[0] == 0


def test_large_model_falls_back_to_fp64_engine():
    # the int8 engine's int32 accumulators are exact up to N = 16384; beyond that the native fp64 engine takes over
    om, nm = model_pair(o.hartmann_6, 16500, 6)
    assert nm.engine == "int8"  # requested engine; the library falls back transparently
    Xq = candidates(256, 6)
    mean, var = nm.predict(Xq)
    omean, ovar = o.predict(om, Xq)
    np.testing.assert_allclose(mean, omean, rtol=1e-8, atol=1e-8 * np.sqrt(om.variance))
    np.testing.assert_allclose(var, ovar, rtol=0, atol=1e-8 * om.variance)


@pytest.mark.parametrize("engine", ["int8", "fp64"])
@pytest.mark.parametrize("noise", [None, 1e-4, 0.5])
def test_augmented_expected_improvement_matches_oracle(noise, engine):
    # function.py:283-325; the builder's eta is the EI builder's (function.py:256-257)
    import trieste_b200 as tb
    from trieste_b200.acquisition import AugmentedExpectedImprovement, augmented_expected_improvement

    om, nm = model_pair(o.hartmann_6, 300, 6, noise=noise, engine=engine)
    Xq = candidates(2000, 6)
    builder = AugmentedExpectedImprovement()
    fn = builder.prepare_acquisition_function(nm, tb.Dataset(om.X, om.y))
    assert isinstance(fn, augmented_expected_improvement)
    eta = o.ei_eta(om)
    np.testing.assert_allclose(fn.eta, eta, rtol=1e-9)
    omean, ovar = o.predict(om, Xq)
    ref = o.augmented_expected_improvement(omean, ovar, eta, om.noise)
    got = fn(Xq[:, None, :])
    np.testing.assert_allclose(got, ref, rtol=1e-6, atol=1e-15)
    idx, best = fn.fused_argmax(Xq)
    assert idx == int(np.argmax(ref[:, 0])) or abs(best - ref.max()) <= 1e-6 * abs(ref.max())
    assert builder.update_acquisition_function(fn, nm, tb.Dataset(om.X, om.y)) is fn
    with pytest.raises(ValueError):
        fn(candidates(6, 6).reshape(3, 2, 6))  # batch size must be one (function.py:313-316)
    # gradient of the augmented tail
    val, grad = fn.value_and_gradient(Xq[:200, None, :])
    oval, ograd = o.aei_gradient(om, Xq[:200], eta)
    np.testing.assert_allclose(val, oval, rtol=1e-6, atol=1e-15)
    np.testing.assert_allclose(grad[:, 0, :], ograd, rtol=1e-6, atol=1e-9 * np.abs(ograd).max())
