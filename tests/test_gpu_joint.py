"""GPU parity: predict_joint, BatchReparametrizationSampler, BatchMonteCarloExpectedImprovement (C3)."""
import numpy as np
import pytest

from oracle import gp_oracle as o
from tests.util import candidates, model_pair

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("engine", ["int8", "fp64"])
@pytest.mark.parametrize("N,D,q", [(20, 2, 1), (20, 2, 3), (300, 6, 8), (300, 6, 5), (128, 6, 16), (300, 10, 11)])
def test_predict_joint_matches_oracle(N, D, q, engine):
    obj = o.branin if D == 2 else (o.hartmann_6 if D == 6 else o.ackley)
    om, nm = model_pair(obj, N, D, engine=engine)
    X = candidates(37 * q, D).reshape(37, q, D)
    mean, cov = nm.predict_joint(X)
    omean, ocov = o.predict_joint(om, X)
    assert mean.shape == (37, q, 1) and cov.shape == (37, 1, q, q)
    np.testing.assert_allclose(mean, omean, rtol=1e-9, atol=1e-9 * np.sqrt(om.variance))
    np.testing.assert_allclose(cov, ocov, rtol=0, atol=1e-9 * om.variance)
    # diagonal agrees with the marginal predict (clip included)
    _, var = nm.predict(X.reshape(-1, D))
    np.testing.assert_allclose(np.diagonal(cov[:, 0], axis1=-2, axis2=-1).reshape(-1, 1), var, rtol=0, atol=1e-10 * om.variance)


def test_predict_joint_leading_dims():
    om, nm = model_pair(o.hartmann_6, 64, 6)
    X = candidates(2 * 3 * 4, 6).reshape(2, 3, 4, 6)
    mean, cov = nm.predict_joint(X)
    assert mean.shape == (2, 3, 4, 1) and cov.shape == (2, 3, 1, 4, 4)
    omean, ocov = o.predict_joint(om, X)
    np.testing.assert_allclose(cov, ocov, rtol=0, atol=1e-9 * om.variance)


@pytest.mark.parametrize("q,S", [(1, 64), (4, 100), (8, 512)])
def test_reparam_sampler_matches_oracle(q, S):
    om, nm = model_pair(o.hartmann_6, 200, 6)
    X = candidates(21 * q, 6).reshape(21, q, 6)
    sampler = nm.reparam_sampler(S)
    eps = np.random.default_rng(3).standard_normal((q, S))
    sampler.set_eps(eps)
    samples = sampler.sample(X, jitter=1e-6)
    assert samples.shape == (21, S, q, 1)
    omean, ocov = o.predict_joint(om, X)
    osamples = o.batch_reparam_sample(omean, ocov, eps[None], 1e-6)
    np.testing.assert_allclose(samples, osamples, rtol=1e-7, atol=1e-7 * np.sqrt(om.variance))
    # repeatability + fixed batch size (sampler.py:329-352)
    np.testing.assert_array_equal(sampler.sample(X), samples)
    with pytest.raises(ValueError):
        sampler.sample(candidates(3 * (q + 1), 6).reshape(3, q + 1, 6))


def test_reparam_sampler_moments():
    # reference test restated (tests/unit/models/gpflow/test_sampler.py:297-326): sample mean / cov
    # match predict_joint within rtol 0.02 / 0.04 (here: absolute tolerances scaled by the prior variance)
    om, nm = model_pair(o.hartmann_6, 100, 6)
    X = candidates(3, 6).reshape(1, 3, 6)
    sampler = nm.reparam_sampler(20000)
    s = sampler.sample(X)[0, :, :, 0]
    mean, cov = nm.predict_joint(X)
    np.testing.assert_allclose(s.mean(0), mean[0, :, 0], atol=0.02 * np.sqrt(om.variance))
    np.testing.assert_allclose(np.cov(s.T), cov[0, 0] + 1e-6 * np.eye(3), atol=0.04 * om.variance)


@pytest.mark.parametrize("engine", ["int8", "fp64"])
@pytest.mark.parametrize("N,D,q,S", [(300, 6, 8, 512), (300, 6, 3, 100), (1024, 10, 8, 512)])
def test_batch_monte_carlo_expected_improvement(N, D, q, S, engine):
    from trieste_b200 import Dataset
    from trieste_b200.acquisition import BatchMonteCarloExpectedImprovement

    obj = o.hartmann_6 if D == 6 else o.ackley
    om, nm = model_pair(obj, N, D, engine=engine)
    builder = BatchMonteCarloExpectedImprovement(S, jitter=1e-6)
    fn = builder.prepare_acquisition_function(nm, Dataset(om.X, om.y))
    eps = np.random.default_rng(3).standard_normal((q, S))
    fn._sampler.set_eps(eps)
    X = candidates(257 * q, D).reshape(257, q, D)
    out = fn(X)
    ref = o.batch_monte_carlo_expected_improvement(om, X, eps[None], o.ei_eta(om), 1e-6)
    assert out.shape == (257, 1)
    np.testing.assert_allclose(out, ref, rtol=1e-6, atol=1e-12)
    fn2 = builder.update_acquisition_function(fn, nm, Dataset(om.X, om.y))
    assert fn2 is fn


def test_qei_q1_reproduces_ei():
    # reference known answer (test_function.py:1359-1371): qEI at q=1 ~ EI within rtol 0.06
    from trieste_b200 import Dataset
    from trieste_b200.acquisition import BatchMonteCarloExpectedImprovement, ExpectedImprovement

    om, nm = model_pair(o.branin, 20, 2)
    ds = Dataset(om.X, om.y)
    X = candidates(200, 2)
    ei = ExpectedImprovement().prepare_acquisition_function(nm, ds)(X[:, None, :])
    qfn = BatchMonteCarloExpectedImprovement(100000).prepare_acquisition_function(nm, ds)
    # all candidates share the same base samples (sampler.py:255-257), so their MC errors are correlated:
    # standardise the draw to remove its first/second-moment error
    eps = np.random.default_rng(0).standard_normal((1, 100000))
    qfn._sampler.set_eps((eps - eps.mean()) / eps.std())
    qei = qfn(X[:, None, :])
    big = ei[:, 0] > 0.05 * ei.max()  # MC noise dominates where improvement events are rare
    np.testing.assert_allclose(qei[big], ei[big], rtol=0.06)


def test_builder_argument_checks():
    from trieste_b200.acquisition import BatchMonteCarloExpectedImprovement

    with pytest.raises(ValueError):
        BatchMonteCarloExpectedImprovement(0)
    with pytest.raises(ValueError):
        BatchMonteCarloExpectedImprovement(10, jitter=-1.0)


def test_predict_joint_max_batch_size_and_argument_checks():
    om, nm = model_pair(o.hartmann_6, 150, 6)
    X = candidates(5 * 32, 6).reshape(5, 32, 6)
    mean, cov = nm.predict_joint(X)
    omean, ocov = o.predict_joint(om, X)
    np.testing.assert_allclose(cov, ocov, rtol=0, atol=1e-9 * om.variance)
    with pytest.raises(ValueError):
        nm.predict_joint(candidates(33 * 2, 6).reshape(2, 33, 6))  # q > 32 is not supported
    with pytest.raises(ValueError):
        nm.predict_joint(candidates(6, 6)[0])  # rank < 2
    m0, c0 = nm.predict_joint(np.zeros((0, 4, 6)))
    assert m0.shape == (0, 4, 1) and c0.shape == (0, 1, 4, 4)


def test_monte_carlo_expected_improvement_single_point():
    # function.py:782-920 (reference test: MC-EI close to EI, test_function.py:651-672)
    from trieste_b200 import Dataset
    from trieste_b200.acquisition import ExpectedImprovement, MonteCarloExpectedImprovement, monte_carlo_expected_improvement

    om, nm = model_pair(o.branin, 20, 2)
    ds = Dataset(om.X, om.y)
    S = 20000
    builder = MonteCarloExpectedImprovement(S)
    fn = builder.prepare_acquisition_function(nm, ds)
    assert isinstance(fn, monte_carlo_expected_improvement)
    eps = fn._sampler._get_eps(1).copy()  # [1, S], fixed until reset
    # eta = min over the data of the sample mean (function.py:838-846), reproduced from the oracle's joint q = 1 samples
    m1, c1 = o.predict_joint(om, om.X[:, None, :])
    samples = o.batch_reparam_sample(m1, c1, eps[None], 1e-6)  # [N, S, 1, 1]
    eta_ref = samples.mean(axis=-3).min()
    np.testing.assert_allclose(fn._eta, eta_ref, rtol=1e-8)
    X = candidates(300, 2)
    ref = o.batch_monte_carlo_expected_improvement(om, X[:, None, :], eps[None], fn._eta, 1e-6)
    np.testing.assert_allclose(fn(X[:, None, :]), ref, rtol=1e-6, atol=1e-12)
    ei = ExpectedImprovement().prepare_acquisition_function(nm, ds)(X[:, None, :])
    big = ei[:, 0] > 0.2 * ei.max()
    np.testing.assert_allclose(fn(X[:, None, :])[big], ei[big], rtol=0.1)
    with pytest.raises(ValueError):
        fn(candidates(8, 2).reshape(2, 2, 2))  # batch size one only (function.py:911-914)
    assert builder.update_acquisition_function(fn, nm, ds) is fn
    assert not np.array_equal(fn._sampler._get_eps(1), eps)  # update resets the sampler (function.py:866)
    with pytest.raises(ValueError):
        MonteCarloExpectedImprovement(0)


@pytest.mark.parametrize("engine", ["int8", "int8x21", "fp64"])
@pytest.mark.parametrize("kind", ["rbf", "matern32", "matern52"])
@pytest.mark.parametrize("N,D,q,S", [(200, 6, 4, 64), (300, 6, 8, 512), (150, 3, 1, 32), (260, 10, 11, 100)])
def test_batch_mc_ei_value_and_gradient_matches_oracle(N, D, q, S, kind, engine):
    # reverse pass of function.py:1181-1186 (what the reference gets from TF autodiff) against the oracle's analytic
    # restatement (itself pinned by finite differences, tests/test_oracle.py)
    from trieste_b200 import Dataset
    from trieste_b200.acquisition import BatchMonteCarloExpectedImprovement

    obj = o.hartmann_6 if D == 6 else o.ackley
    om, nm = model_pair(obj, N, D, kind=kind, engine=engine)
    fn = BatchMonteCarloExpectedImprovement(S, jitter=1e-6).prepare_acquisition_function(nm, Dataset(om.X, om.y))
    eps = np.random.default_rng(3).standard_normal((q, S))
    fn._sampler.set_eps(eps)
    fn._eta = float(np.median(om.y))  # plenty of active samples
    nb = 37
    X = candidates(nb * q, D).reshape(nb, q, D)
    val, grad = fn.value_and_gradient(X)
    assert val.shape == (nb, 1) and grad.shape == (nb, q, D)
    np.testing.assert_allclose(val, fn(X), rtol=1e-9, atol=1e-13)
    for b in range(0, nb, 6):
        oval, ograd = o.batch_mc_ei_gradient(om, X[b], eps, fn._eta, 1e-6)
        np.testing.assert_allclose(val[b, 0], oval, rtol=1e-6, atol=1e-12)
        np.testing.assert_allclose(grad[b], ograd, rtol=1e-5, atol=1e-7 * max(np.abs(ograd).max(), 1e-30))


def test_batch_mc_ei_gradient_drives_the_joint_optimizer():
    # batchify_joint + continuous optimiser over space ** q (optimizer.py:897-936): ends at a point no worse than the
    # best random q-batch and the starts it refined
    import trieste_b200 as tb
    from trieste_b200.acquisition import BatchMonteCarloExpectedImprovement
    from trieste_b200.acquisition.optimizer import batchify_joint, generate_continuous_optimizer

    om, nm = model_pair(o.hartmann_6, 150, 6)
    ds = tb.Dataset(om.X, om.y)
    fn = BatchMonteCarloExpectedImprovement(256).prepare_acquisition_function(nm, ds)
    space = tb.Box([0.0] * 6, [1.0] * 6)
    opt = batchify_joint(generate_continuous_optimizer(num_initial_samples=400, num_optimization_runs=6,
                                                       optimizer_args={"maxiter": 60}), 3)
    pts = opt(space, fn)
    assert pts.shape == (3, 6) and space.contains(pts).all()
    rnd = space.sample(400 * 3, seed=2).reshape(400, 3, 6)
    assert fn(pts[None])[0, 0] >= fn(rnd).max() - 1e-12
    # leading dimensions and argument errors
    v, g = fn.value_and_gradient(rnd[:6].reshape(2, 3, 3, 6))
    assert v.shape == (2, 3, 1) and g.shape == (2, 3, 3, 6)
    nm.set_engine("fp64")  # the native fp64 engine computes the same reverse pass
    v64, g64 = fn.value_and_gradient(rnd[:6].reshape(2, 3, 3, 6))
    nm.set_engine("int8")
    np.testing.assert_allclose(v64, v, rtol=1e-8, atol=1e-13)
    np.testing.assert_allclose(g64, g, rtol=1e-6, atol=1e-9 * np.abs(g).max())


def test_independent_reparametrization_sampler_matches_its_definition():
    # sampler.py:82-164: mean + sqrt(var + jitter) * eps, eps [S, 1] fixed until reset
    from trieste_b200.sampler import IndependentReparametrizationSampler

    om, nm = model_pair(o.hartmann_6, 120, 6)
    s = IndependentReparametrizationSampler(50, nm, seed=1)
    X = candidates(40, 6)
    out = s.sample(X[:, None, :], jitter=1e-6)
    assert out.shape == (40, 50, 1, 1)
    eps = np.random.default_rng(1).standard_normal((50, 1))
    mean, var = o.predict(om, X)
    ref = mean[:, None, :, None] + np.sqrt(var + 1e-6)[:, None, :, None] * eps[None, :, :, None]
    np.testing.assert_allclose(out, ref, rtol=1e-8, atol=1e-9 * np.sqrt(om.variance))
    np.testing.assert_array_equal(out, s.sample(X[:, None, :], jitter=1e-6))  # same draws until reset
    s.reset_sampler()
    assert not np.array_equal(out, s.sample(X[:, None, :], jitter=1e-6))
    with pytest.raises(ValueError):
        s.sample(X.reshape(20, 2, 6))
    with pytest.raises(ValueError):
        IndependentReparametrizationSampler(0, nm)


@pytest.mark.parametrize("engine", ["int8", "fp64"])
@pytest.mark.parametrize("M", [33, 128, 300, 1000])
def test_large_joint_samples_follow_the_oracle_posterior(M, engine):
    # model.sample over more than 32 points (interface.py:135-138 -> predict_f_samples): the device path must reproduce
    # mean + chol(cov + 1e-6 I) z for the z it drew
    om, nm = model_pair(o.hartmann_6, 200, 6, engine=engine)
    X = candidates(M, 6)
    S = 7
    out = nm.sample(X, S, seed=11)
    assert out.shape == (S, M, 1)
    z = np.random.default_rng(11).standard_normal((S, M))
    mean, cov = o.predict_joint(om, X)
    L = np.linalg.cholesky(cov[0] + 1e-6 * np.eye(M))
    ref = mean[None, :, 0] + z @ L.T
    np.testing.assert_allclose(out[..., 0], ref, rtol=0, atol=1e-6 * np.sqrt(om.variance))
    with pytest.raises(ValueError):
        nm.sample(X, 0)


def test_exact_thompson_sampler_and_rule_default():
    # acquisition/sampler.py:85-123 and rule.py:938-943
    import trieste_b200 as tb
    from trieste_b200.acquisition import MinValueEntropySearch
    from trieste_b200.acquisition.sampler import ExactThompsonSampler, GumbelSampler
    from trieste_b200.rule import DiscreteThompsonSampling

    om, nm = model_pair(o.hartmann_6, 100, 6)
    at = candidates(500, 6)
    pts = ExactThompsonSampler().sample(nm, 5, at, seed=0)
    assert pts.shape == (5, 6) and all(any(np.array_equal(p, a) for a in at) for p in pts)
    mins = ExactThompsonSampler(sample_min_value=True).sample(nm, 5, at, seed=0)
    assert mins.shape == (5, 1)
    # same seed -> the minimum values belong to the minimisers drawn above
    samples = nm.sample(at, 5, seed=0)[..., 0]
    np.testing.assert_array_equal(mins[:, 0], samples.min(axis=1))
    np.testing.assert_array_equal(pts, at[samples.argmin(axis=1)])
    # sample minima are below the posterior-mean minimum on average (they include the posterior spread)
    assert mins.mean() < o.predict(om, at)[0].min() + 1e-9
    rule = DiscreteThompsonSampling(400, 3)
    q = rule.acquire_single(tb.Box([0.0] * 6, [1.0] * 6), nm, tb.Dataset(om.X, om.y))
    assert q.shape == (3, 6)
    with pytest.raises(ValueError):
        DiscreteThompsonSampling(400, 3, thompson_sampler=GumbelSampler(True))
    # the reference's default min-value sampler for MES now works too
    builder = MinValueEntropySearch(tb.Box([0.0] * 6, [1.0] * 6), 4, 300, min_value_sampler=ExactThompsonSampler(True))
    fn = builder.prepare_acquisition_function(nm, tb.Dataset(om.X, om.y))
    assert fn.samples.shape == (4, 1) and np.isfinite(fn(at[:, None, :])).all()


@pytest.mark.parametrize("engine", ["int8", "fp64"])
@pytest.mark.parametrize("kind", ["rbf", "matern32", "matern52"])
def test_covariance_between_points_matches_oracle(kind, engine):
    # models.py:188-254 (reference test: tests/unit/models/gpflow/test_models.py:282-305)
    om, nm = model_pair(o.hartmann_6, 300, 6, kind=kind, engine=engine)
    rng = np.random.default_rng(0)
    X1 = rng.uniform(size=(3, 50, 6))
    X2 = np.concatenate([rng.uniform(size=(200, 6)), X1[0, :5]])  # shared points: the exact posterior variance on them
    cov = nm.covariance_between_points(X1, X2)
    ref = o.covariance_between_points(om, X1, X2)
    assert cov.shape == (3, 1, 50, 205)
    np.testing.assert_allclose(cov, ref, rtol=0, atol=1e-9 * om.variance)
    one = nm.covariance_between_points(X1[0, :1], X2[:1])
    assert one.shape == (1, 1, 1)
    np.testing.assert_allclose(one, ref[0, :, :1, :1], rtol=0, atol=1e-9 * om.variance)
    with pytest.raises(ValueError):
        nm.covariance_between_points(X1, X2[None])  # query_points_2 must have rank two
    with pytest.raises(ValueError):
        nm.covariance_between_points(X1[..., :5], X2)  # wrong input dimension
