"""CPU: pins the oracle (oracle/gp_oracle.py) against (i) the committed scikit-learn fixtures and
(ii) restatements of the reference's own model-independent known-answer tests (SURVEY.md §8c)."""
import glob
import math
import os

import numpy as np
import pytest

from oracle import gp_oracle as o

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "gpr_sklearn_*.npz")))


def _load(path):
    z = np.load(path)
    if "X" in z.files:
        X, y = z["X"], z["y"]
    else:  # the benchmark-size fixtures store the generator instead of the data
        gen = o.synthetic_model(getattr(o, str(z["generator"])), int(z["N"]), int(z["D"]), kind=str(z["kind"]), seed=int(z["seed"]))
        X, y = gen.X, gen.y
    om = o.build_model(str(z["kind"]), X, y, float(z["variance"]), z["lengthscales"], float(z["noise"]), float(z["mean_const"]))
    return z, om


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[12:-4] for p in GOLDEN])
def test_oracle_matches_sklearn_fixture(path):
    z, om = _load(path)
    mean, var = o.predict_f(om, z["Xq"])
    # Matern12 = exp(-r): scikit-learn's r (cdist) and the oracle's GPflow-style expansion r^2 differ by O(1e-16) on the
    # diagonal of K(X, X), which sqrt() turns into O(1e-8); every smooth kernel is pinned at 1e-9
    tol = 1e-5 if om.kind == "matern12" else 1e-9
    np.testing.assert_allclose(mean[:, 0], z["mean"], rtol=tol, atol=tol * math.sqrt(om.variance))
    np.testing.assert_allclose(var[:, 0], z["var"], rtol=0, atol=tol * om.variance)
    _, cov = o.predict_f(om, z["Xq"][:16], full_cov=True)
    np.testing.assert_allclose(cov, z["cov"][:16, :16], rtol=0, atol=tol * om.variance)


def test_golden_fixtures_present():
    assert len(GOLDEN) >= 7


def test_predict_clips_variance_and_joint_matches_marginal():
    om = o.synthetic_model(o.branin, 20, 2, noise=1e-7)
    mean, var = o.predict(om, om.X)
    assert var.min() >= 1e-12
    X = np.random.default_rng(1).uniform(size=(5, 3, 2))
    jm, jc = o.predict_joint(om, X)
    mm, mv = o.predict(om, X.reshape(-1, 2))
    assert jm.shape == (5, 3, 1) and jc.shape == (5, 1, 3, 3)
    np.testing.assert_allclose(jm.reshape(-1, 1), mm, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(np.diagonal(jc[:, 0], axis1=-2, axis2=-1).reshape(-1, 1), mv, rtol=0, atol=1e-10 * om.variance)


def test_lcb_closed_form():
    # tests/unit/acquisition/function/test_function.py:786-790: with mean = sum x^2 and var = 1, LCB = x^2 - beta
    x = np.linspace(-3, 3, 13)[:, None]
    mean, var = (x**2).sum(-1, keepdims=True), np.ones((13, 1))
    np.testing.assert_allclose(o.lower_confidence_bound(mean, var, 1.96), x**2 - 1.96, rtol=1e-12)
    with pytest.raises(ValueError):
        o.lower_confidence_bound(mean, var, -1.0)


@pytest.mark.parametrize("variance_scale", [0.1, 1.0, 10.0, 100.0])
@pytest.mark.parametrize("best", [0.0, 1.0, -2.0])
def test_expected_improvement_vs_monte_carlo(variance_scale, best):
    # test_function.py:290-332 restated: analytic EI vs a Monte-Carlo estimate, rtol 0.01
    rng = np.random.default_rng(0)
    mean = np.linspace(-1.5, 1.5, 7)[:, None]
    var = np.full_like(mean, variance_scale)
    ei = o.expected_improvement(mean, var, best)
    samples = mean + np.sqrt(var) * rng.standard_normal((7, 400_000))
    mc = np.maximum(best - samples, 0.0).mean(-1, keepdims=True)
    np.testing.assert_allclose(ei, mc, rtol=0.02, atol=2e-3 * math.sqrt(variance_scale))


def test_log_ei_matches_log_of_ei_and_stays_finite():
    mean = np.linspace(-3, 40, 200)[:, None]
    var = np.full_like(mean, 0.5)
    ei = o.expected_improvement(mean, var, 0.0)
    lei = o.log_expected_improvement(mean, var, 0.0)
    ok = ei[:, 0] > 1e-300
    np.testing.assert_allclose(lei[ok], np.log(ei[ok]), rtol=1e-7, atol=1e-7)
    assert np.all(np.isfinite(lei)) and np.all(np.diff(lei[:, 0]) < 0)


def test_ei_eta_is_min_posterior_mean_and_gradient_fd():
    om = o.synthetic_model(o.hartmann_6, 60, 6)
    eta = o.ei_eta(om)
    assert eta == o.predict(om, om.X)[0].min()
    Xq = np.random.default_rng(2).uniform(size=(4, 6))
    _, g = o.ei_gradient(om, Xq, eta)
    h = 1e-6
    for d in range(6):
        e = np.zeros(6)
        e[d] = h
        fd = (o.expected_improvement(*o.predict(om, Xq + e), eta) - o.expected_improvement(*o.predict(om, Xq - e), eta)) / (2 * h)
        np.testing.assert_allclose(g[:, d], fd[:, 0], rtol=1e-4, atol=1e-9 * np.abs(g).max())


@pytest.mark.parametrize(
    "kind,D,exact",
    [(k, D, False) for k in o.KERNEL_KINDS for D in (1, 6, 13)] + [("matern12", D, True) for D in (1, 6, 13)],
    ids=lambda v: ("exact_L" if v else "oracle_L") if isinstance(v, bool) else str(v),
)
def test_posterior_gradients_match_central_differences(kind, D, exact):
    # the GPU gradient tests hold the kernels to posterior_gradients at 1e-9 of the scale; this pins both of its terms,
    # dmean and dvar, for every kernel, to central differences of predict.  exact: with the difference-form Cholesky the
    # Matern-12 GPU tests compare against (tests/util.py)
    from tests.util import with_exact_cholesky

    om = o.synthetic_model(o.ackley, 64, D, kind=kind)
    if exact:
        om = with_exact_cholesky(om)
    Xq = np.random.default_rng(3).uniform(size=(8, D))
    dmean, dvar = o.posterior_gradients(om, Xq)
    h = 1e-6
    for d in range(D):
        e = np.zeros(D)
        e[d] = h
        mp, vp = o.predict(om, Xq + e)
        mm, vm = o.predict(om, Xq - e)
        np.testing.assert_allclose(dmean[:, d], (mp - mm)[:, 0] / (2 * h), rtol=1e-5, atol=1e-7 * np.abs(dmean).max())
        np.testing.assert_allclose(dvar[:, d], (vp - vm)[:, 0] / (2 * h), rtol=1e-5, atol=1e-7 * np.abs(dvar).max())


def test_qei_q1_matches_ei_and_mvn_samples():
    # test_function.py:1359-1394 restated
    om = o.synthetic_model(o.branin, 20, 2)
    eta = o.ei_eta(om)
    X = np.random.default_rng(1).uniform(size=(30, 1, 2))
    eps = np.random.default_rng(3).standard_normal((1, 1, 50_000))
    qei = o.batch_monte_carlo_expected_improvement(om, X, eps, eta)
    ei = o.expected_improvement(*o.predict(om, X[:, 0]), eta)
    big = ei[:, 0] > 0.05 * ei.max()  # MC noise dominates where improvement events are rare
    np.testing.assert_allclose(qei[big], ei[big], rtol=0.06)
    # q = 3 against direct multivariate-normal sampling
    Xb = np.random.default_rng(4).uniform(size=(1, 3, 2))
    mean, cov = o.predict_joint(om, Xb)
    mvn = np.random.default_rng(5).multivariate_normal(mean[0, :, 0], cov[0, 0], size=200_000)
    direct = np.maximum(eta - mvn.min(-1), 0).mean()
    eps3 = np.random.default_rng(6).standard_normal((1, 3, 200_000))
    np.testing.assert_allclose(o.batch_monte_carlo_expected_improvement(om, Xb, eps3, eta)[0, 0], direct, rtol=0.05, atol=1e-4)


def test_rff_design_equals_gram_and_moments():
    # tests/unit/models/gpflow/test_sampler.py:530-542 (design == gram, rtol 0.02) and
    # test_models.py:638-681 (trajectory moments vs predict)
    om = o.synthetic_model(o.hartmann_6, 100, 6, kind="rbf")
    rng = np.random.default_rng(0)
    W, b = o.rff_draw("rbf", 100, 6, rng)
    # force both routes on the same features: n = 100, F = 100 -> gram; drop one data point -> design
    mg, cg = o.rff_theta_posterior(om, W, b)
    om2 = o.build_model(om.kind, np.concatenate([om.X, om.X[:1] + 1e-3]), np.concatenate([om.y, om.y[:1]]), om.variance,
                        om.lengthscales, om.noise, om.mean_const)
    md, cd = o.rff_theta_posterior(om2, W, b)  # F < n: design space
    assert np.abs(mg - md).max() < 0.05 * np.abs(mg).max() + 0.05
    # moments, in the reference test's own setting: 1-D, x = 0..4, y = 3x + noise, Matern32(1, 1), 1000 features
    x = np.arange(5.0).reshape(-1, 1)
    y = 3.0 * x + 0.1 * rng.standard_normal((5, 1))
    for noise_var in [1e-5, 1e-1]:
        m1 = o.build_model("matern32", x, y, 1.0, np.ones(1), noise_var, 0.0)
        W2, b2 = o.rff_draw("matern32", 1000, 1, rng)
        tm, tc = o.rff_theta_posterior(m1, W2, b2)
        thetas = tm + rng.standard_normal((400, 1000)) @ tc.T
        xp = np.array([[1.0], [2.0], [3.0], [1.5], [2.5], [3.5]])
        f = o.rff_trajectory(np.repeat(xp[:, None, :], 400, 1), W2, b2, thetas, 1.0, np.ones(1), 0.0)[:, :, 0]
        mean, var = o.predict(m1, xp)
        np.testing.assert_allclose(f.mean(1) + 1.0, mean[:, 0] + 1.0, rtol=0.1)
        np.testing.assert_allclose(f.var(1)[3:], var[3:, 0], rtol=0.5, atol=1e-3)


def test_topk_and_argmax_semantics():
    v = np.array([1.0, 3.0, 3.0, -1.0, 3.0, 2.0])
    assert o.argmax_first(v) == 1
    tv, ti = o.top_k(v, 4)
    np.testing.assert_array_equal(ti, [1, 2, 4, 5])
    np.testing.assert_array_equal(tv, [3.0, 3.0, 3.0, 2.0])


def test_objectives_known_minima():
    # trieste/objectives/single_objectives.py minimiser tables
    np.testing.assert_allclose(o.hartmann_6(np.array([[0.20169, 0.150011, 0.476874, 0.275332, 0.311652, 0.6573]])), [[-3.32237]], atol=1e-5)
    np.testing.assert_allclose(o.ackley(np.full((1, 5), 0.5)), [[0.0]], atol=1e-12)
    np.testing.assert_allclose(o.branin(np.array([[0.5427728, 0.1516667]])), [[0.397887]], atol=1e-5)


def test_decoupled_sampler_moments():
    # DecoupledTrajectorySampler restatement: trajectory moments reproduce the exact posterior
    # (tests/unit/models/gpflow/test_models.py:638-681 with use_decoupled_sampler=True)
    om = o.synthetic_model(o.hartmann_6, 60, 6, kind="rbf")
    rng = np.random.default_rng(0)
    W, b = o.rff_draw("rbf", 3000, 6, rng)
    S = 400
    pw, eps = rng.standard_normal((S, 3000)), rng.standard_normal((S, 60))
    v = o.decoupled_weights(om, W, b, pw, eps)
    Xq = rng.uniform(size=(10, 6))
    f = o.decoupled_trajectory(om, np.repeat(Xq[:, None, :], S, 1), W, b, pw, v)[:, :, 0]
    mean, var = o.predict(om, Xq)
    np.testing.assert_allclose(f.mean(1), mean[:, 0], atol=0.15 * math.sqrt(om.variance))
    np.testing.assert_allclose(f.var(1), var[:, 0], rtol=0.5, atol=0.02 * om.variance)


def test_augmented_ei_bounds_and_gradient():
    # function.py:318-325: AEI = EI * (1 - tau / sqrt(tau^2 + s^2)) in (0, EI), -> EI as the noise vanishes
    m = o.synthetic_model(o.hartmann_6, 40, 6)
    Xq = np.random.default_rng(1).uniform(size=(30, 6))
    mean, var = o.predict(m, Xq)
    eta = o.ei_eta(m)
    ei = o.expected_improvement(mean, var, eta)
    aei = o.augmented_expected_improvement(mean, var, eta, m.noise)
    assert np.all(aei < ei) and np.all(aei >= 0)
    np.testing.assert_allclose(o.augmented_expected_improvement(mean, var, eta, 1e-30), ei, rtol=1e-12)
    val, grad = o.aei_gradient(m, Xq, eta)
    np.testing.assert_allclose(val, aei, rtol=1e-12)
    h = 1e-6
    for d in range(6):
        e = np.zeros(6)
        e[d] = h
        fd = []
        for sgn in (1, -1):
            mu, v = o.predict(m, Xq + sgn * e)
            fd.append(o.augmented_expected_improvement(mu, v, eta, m.noise))
        np.testing.assert_allclose(grad[:, d], ((fd[0] - fd[1]) / (2 * h))[:, 0], rtol=1e-4, atol=1e-8 * np.abs(grad).max())


def test_min_value_entropy_search_restatement():
    # entropy.py:193-213 against the closed form for gamma >> 0 / gamma << 0 and direct quadrature-free identities
    from scipy.stats import norm

    mean = np.array([[0.0], [1.0], [-2.0]])
    var = np.array([[1.0], [0.25], [4.0]])
    samples = np.array([[-1.5], [-0.3], [-4.0]])
    got = o.min_value_entropy_search(mean, var, samples)
    gam = (samples.reshape(1, -1) - mean) / np.sqrt(var)
    ref = (-gam * norm.pdf(gam) / (2 * norm.cdf(-gam)) - np.log(norm.cdf(-gam))).mean(1, keepdims=True)
    np.testing.assert_allclose(got, ref, rtol=1e-12)
    assert np.all(got >= 0)  # information gain
    # far tail: finite where the naive form underflows (cdf(-40) == 0)
    far = o.min_value_entropy_search(np.array([[0.0]]), np.array([[1.0]]), np.array([[40.0]]))
    assert np.isfinite(far).all() and far[0, 0] > 0
    # entropy.py:47,201-204: sd clipped from below
    tiny = o.min_value_entropy_search(np.array([[0.0]]), np.array([[1e-30]]), np.array([[-1e-9]]))
    np.testing.assert_allclose(tiny, o.min_value_entropy_search(np.array([[0.0]]), np.array([[1e-16]]), np.array([[-1e-9]])))


def test_gumbel_sampler_restatement_matches_empirical_minimum_quartiles():
    # acquisition/sampler.py:186-204: the fitted Gumbel reproduces the quartiles of the min over independent normals
    rng = np.random.default_rng(0)
    mu = rng.normal(size=50)
    sd = rng.uniform(0.2, 1.0, size=50)
    a, b = o.gumbel_fit(mu, sd)
    draws = (mu + sd * rng.standard_normal((200_000, 50))).min(axis=1)
    q1, q2 = np.quantile(draws, [0.25, 0.75])
    g = o.gumbel_samples(a, b, np.array([0.25, 0.75]))[:, 0]
    np.testing.assert_allclose(g, [q1, q2], atol=0.01)
    assert b > 0


@pytest.mark.parametrize("kind", ["rbf", "matern32", "matern52"])
def test_batch_mc_ei_gradient_restatement_matches_finite_differences(kind):
    # the reverse pass of function.py:1181-1186 (arg-min routing, Cholesky reverse mode) against central differences
    m = o.synthetic_model(o.hartmann_6, 40, 6, kind=kind)
    rng = np.random.default_rng(1)
    q, S = 4, 96
    eps = rng.standard_normal((q, S))
    Xb = rng.uniform(size=(q, 6))
    eta = float(np.median(m.y))
    val, g = o.batch_mc_ei_gradient(m, Xb, eps, eta)
    np.testing.assert_allclose(val, o.batch_monte_carlo_expected_improvement(m, Xb[None], eps[None], eta)[0, 0], rtol=1e-12)
    h = 1e-6
    fd = np.zeros_like(g)
    for j in range(q):
        for d in range(6):
            Xp, Xm = Xb.copy(), Xb.copy()
            Xp[j, d] += h
            Xm[j, d] -= h
            fd[j, d] = (o.batch_monte_carlo_expected_improvement(m, Xp[None], eps[None], eta)[0, 0]
                        - o.batch_monte_carlo_expected_improvement(m, Xm[None], eps[None], eta)[0, 0]) / (2 * h)
    np.testing.assert_allclose(g, fd, rtol=1e-5, atol=1e-7 * np.abs(g).max())


def test_covariance_between_points_restatement_is_consistent_with_predict_joint():
    # reference test_gpflow_models_pairwise_covariance (tests/unit/models/gpflow/test_models.py:282-305): the pairwise
    # covariance of a set with itself equals the off-diagonal blocks of the joint prediction over the union
    m = o.synthetic_model(o.hartmann_6, 50, 6)
    rng = np.random.default_rng(0)
    X1, X2 = rng.uniform(size=(2, 4, 6)), rng.uniform(size=(3, 6))
    cov = o.covariance_between_points(m, X1, X2)
    assert cov.shape == (2, 1, 4, 3)
    for b in range(2):
        _, joint = o.predict_f(m, np.concatenate([X1[b], X2]), full_cov=True)
        np.testing.assert_allclose(cov[b, 0], joint[:4, 4:], rtol=1e-10, atol=1e-12)


# ---- round 2 restatements --------------------------------------------------------------------------------------------
def test_molcb_betas_and_value():
    # function.py:1898-1905: spread = 0.5 + 0.5 b / (B + 1), betas = 5 d Phi^-1(spread); B = 1 -> Phi^-1(0.75)
    np.testing.assert_allclose(o.molcb_betas(1, 2), [5.0 * 2 * 0.6744897501960817], rtol=1e-12)
    b = o.molcb_betas(4, 3)
    assert np.all(np.diff(b) > 0) and b[0] > 0
    om = o.synthetic_model(o.branin, 30, 2)
    X = np.random.default_rng(0).uniform(size=(7, 3, 2))
    out = o.multiple_optimism_lower_confidence_bound(om, X, 2)
    mean, var = o.predict(om, X.reshape(-1, 2))
    np.testing.assert_allclose(out, -mean.reshape(7, 3) + np.sqrt(var.reshape(7, 3)) * o.molcb_betas(3, 2), rtol=1e-13)


def test_conditional_predict_equals_a_model_with_the_data_appended():
    # Chevalier et al. 2014 eqs. 8-10 (models.py:355-425): conditioning on extra data == refitting with them appended
    om = o.synthetic_model(o.hartmann_6, 120, 6)
    rng = np.random.default_rng(1)
    Xq, Xa, ya = rng.uniform(size=(9, 6)), rng.uniform(size=(4, 6)), rng.normal(size=(4, 1))
    m1, v1 = o.conditional_predict_f(om, Xq, Xa, ya)
    om2 = o.build_model(om.kind, np.concatenate([om.X, Xa]), np.concatenate([om.y, ya]), om.variance, om.lengthscales, om.noise, om.mean_const)
    m2, v2 = o.predict_f(om2, Xq)
    np.testing.assert_allclose(m1, m2, rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(v1, v2, rtol=0, atol=1e-12 * om.variance)


def test_log_ei_gradient_restatement_matches_finite_differences_where_ei_underflows():
    om = o.synthetic_model(o.hartmann_6, 100, 6)
    eta = o.ei_eta(om)
    x = np.random.default_rng(0).uniform(size=(6, 6))
    val, g = o.log_ei_gradient(om, x, eta)
    assert np.all(np.isfinite(val)) and np.all(np.isfinite(g)) and val.min() < -20  # plain EI is ~1e-9 or less here
    h = 1e-6
    for d in range(6):
        e = np.zeros(6)
        e[d] = h
        fp = o.log_expected_improvement(*o.predict(om, x + e), eta)
        fm = o.log_expected_improvement(*o.predict(om, x - e), eta)
        np.testing.assert_allclose(g[:, d], ((fp - fm) / (2 * h))[:, 0], rtol=2e-5, atol=1e-4)


def test_scipy_lbfgsb_multistart_known_answers():
    # tests/unit/acquisition/test_optimizer.py:86-168 restated for the optimiser engine: maximiser of a concave quadratic
    # inside the box, and on the boundary when the centre lies outside
    for c, expect in [(np.array([0.3, 0.6]), np.array([0.3, 0.6])), (np.array([1.4, -0.2]), np.array([1.0, 0.0]))]:
        def vg(x, c=c):
            return -np.sum((x - c) ** 2, axis=1), -2.0 * (x - c)

        ok, f, x, nfev = o.scipy_lbfgsb_multistart(vg, np.random.default_rng(0).uniform(size=(5, 2)), 0.0, 1.0)
        assert ok.all() and nfev.min() >= 1
        np.testing.assert_allclose(x, np.broadcast_to(expect, (5, 2)), atol=1e-6)
        np.testing.assert_allclose(f, -np.sum((expect - c) ** 2), atol=1e-10)
