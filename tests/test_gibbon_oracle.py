"""The NumPy restatement of GIBBON (tests/gibbon_oracle.py) against the reference's own known answers, the appended-data
identity of the repulsion term and finite differences.  CPU only."""
import numpy as np
import pytest

from oracle import gp_oracle as o
from tests import gibbon_oracle as gb


def _quadratic_model(noise, n=12, seed=0):
    """An RBF GPR on samples of a quadratic bowl (the reference's tests use a quadratic-mean model)."""
    X = np.random.default_rng(seed).uniform(-1.0, 1.0, size=(n, 2))
    y = np.sum(X * X, axis=1, keepdims=True)
    return o.build_model("rbf", X, y, 1.0, np.array([0.6, 0.8]), noise, 0.5)


def _grid(lo, hi, n):
    r = np.linspace(lo, hi, n)
    return np.stack(np.meshgrid(r, r, indexing="ij"), axis=-1).reshape(-1, 2)


def test_single_sample_quality_term_chooses_as_min_value_entropy_search():
    """test_entropy.py:466-481: with one min-value sample GIBBON's quality term and MES share their argmax."""
    m = _quadratic_model(1e-10)
    xs = _grid(-1.0, 1.0, 11)
    mean, var = o.predict(m, xs)
    for y_star in (-0.3, 0.0, 0.2):
        samples = np.array([[y_star]])
        assert o.argmax_first(gb.quality_term(mean, var, samples, m.noise)[:, 0]) == o.argmax_first(
            o.min_value_entropy_search(mean, var, samples)[:, 0])


@pytest.mark.parametrize("rescaled", [True, False])
@pytest.mark.parametrize("noise", [0.1, 1e-10])
def test_batch_gibbon_is_the_quality_term_plus_the_joint_log_determinant(rescaled, noise):
    """test_entropy.py:484-527: GIBBON = quality + w/2 (logdet(A + noise I) - log A00 - logdet(B + noise I)) with A the
    joint covariance of [x; P] and A00 its noisy candidate entry."""
    m = _quadratic_model(noise)
    xs = _grid(0.0, 1.0, 4)
    pending = np.array([[0.11, 0.51], [0.21, 0.31], [0.41, 0.91]])
    samples = np.array([[-0.1], [0.1]])
    got = gb.gibbon(m, xs, samples, pending, rescaled)
    mean, var = o.predict(m, xs)
    quality = gb.quality_term(mean, var, samples, noise)
    _, Bp = o.predict_joint(m, pending)
    Bn = Bp[0] + noise * np.eye(3)
    w = (1.0 / 3) ** 2 if rescaled else 1.0
    for i in range(xs.shape[0]):
        _, A = o.predict_joint(m, np.concatenate([xs[i:i + 1], pending]))
        A = A[0] + noise * np.eye(4)
        rep = np.linalg.slogdet(A)[1] - np.log(A[0, 0]) - np.linalg.slogdet(Bn)[1]
        np.testing.assert_allclose(got[i], quality[i] + 0.5 * w * rep, rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("kind", ["matern52", "rbf"])
@pytest.mark.parametrize("m_pending", [1, 7])
def test_repulsion_is_the_noisy_variance_ratio_of_the_model_conditioned_on_the_pending_points(kind, m_pending):
    m = o.synthetic_model(o.hartmann_6, 200, 6, kind=kind)
    rng = np.random.default_rng(5)
    pending = rng.uniform(size=(m_pending, 6))
    x = np.concatenate([rng.uniform(size=(300, 6)), pending, m.X[:5]])
    for rescaled in (True, False):
        np.testing.assert_allclose(gb.repulsion_term(m, x, pending, rescaled), gb.augmented_repulsion(m, x, pending, rescaled),
                                   rtol=1e-7, atol=1e-10)


def _central_differences(f, x, h=1e-6):
    g = np.zeros_like(x)
    for d in range(x.shape[1]):
        e = np.zeros(x.shape[1])
        e[d] = h
        g[:, d] = (f(x + e)[:, 0] - f(x - e)[:, 0]) / (2 * h)
    return g


@pytest.mark.parametrize("kind", ["matern52", "rbf", "matern32"])
def test_analytic_gradients_match_central_differences(kind):
    m = o.synthetic_model(o.hartmann_6, 150, 6, kind=kind)
    rng = np.random.default_rng(7)
    pending = rng.uniform(size=(4, 6))
    x = np.concatenate([rng.uniform(size=(40, 6)), pending + 0.01])
    samples = m.y.min() + np.array([[-0.2], [-0.05], [0.1]]) * np.sqrt(m.variance)
    qv, qg = gb.quality_value_and_gradient(m, x, samples)
    np.testing.assert_allclose(qv, gb.quality_term(*o.predict(m, x), samples, m.noise), rtol=1e-12)
    fd = _central_differences(lambda z: gb.quality_term(*o.predict(m, z), samples, m.noise), x)
    np.testing.assert_allclose(qg, fd, rtol=1e-5, atol=1e-7 * np.abs(fd).max())
    rv, rg = gb.repulsion_value_and_gradient(m, x, pending)
    np.testing.assert_allclose(rv, gb.repulsion_term(m, x, pending), rtol=1e-10, atol=1e-14)
    fd = _central_differences(lambda z: gb.repulsion_term(m, z, pending), x)
    np.testing.assert_allclose(rg, fd, rtol=1e-5, atol=1e-7 * np.abs(fd).max())
    v, g = gb.gibbon_value_and_gradient(m, x, samples, pending, rescaled=False)
    np.testing.assert_allclose(g, gb.quality_value_and_gradient(m, x, samples)[1]
                               + gb.repulsion_value_and_gradient(m, x, pending, False)[1], rtol=1e-12)


def test_quality_term_over_the_gamma_range_stays_finite_and_non_negative():
    """gamma from -40 to 8: r (gamma - r) -> -1 cancels for large gamma in the reference's own formula; the term stays a
    finite, non-negative information gain there."""
    mean = np.zeros((1, 1))
    var = np.ones((1, 1))
    gammas = np.linspace(-40.0, 8.0, 481).reshape(-1, 1)
    q = np.concatenate([gb.quality_term(mean, var, g.reshape(1, 1), 0.01) for g in gammas])
    assert np.all(np.isfinite(q)) and np.all(q >= -1e-12)
