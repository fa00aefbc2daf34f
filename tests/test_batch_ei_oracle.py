"""The NumPy restatement of BatchExpectedImprovement (tests/bei_oracle.py) against SciPy's multivariate-normal CDF, the
batch Monte-Carlo EI oracle, finite differences and the Sobol column identity; the builder's argument errors and
protocol conformance of the new classes.  CPU only."""
import inspect
import json
import os

import numpy as np
import pytest
from scipy.stats import multivariate_normal

from oracle import gp_oracle as o
from tests import bei_oracle as bo

HERE = os.path.dirname(os.path.abspath(__file__))


def _sobol(S, dim, skip=12345):
    from trieste_b200.sampler import sobol_points

    return sobol_points(S, dim, skip)


def _quadratic_model(N, D, seed):
    """The reference's check (test_function.py:1214-1252) uses a quadratic objective under an RBF GP on the unit cube.
    Few points and a short lengthscale keep the EI values well above the Monte-Carlo noise of the comparison."""
    X = np.random.default_rng(seed).uniform(size=(N, D))
    y = np.sum(X * X, axis=1, keepdims=True)
    return o.build_model("rbf", X, y, 1.0, np.full(D, 0.2), 1e-6, 0.0)


@pytest.mark.parametrize("Q", [1, 2, 3, 4, 5, 6])
def test_genz_cdf_matches_scipy(Q):
    rng = np.random.default_rng(Q)
    B = 5
    A = rng.standard_normal((B, Q, Q))
    cov = A @ np.transpose(A, (0, 2, 1)) + 0.5 * np.eye(Q)
    mean = rng.standard_normal((B, Q))
    x = mean + rng.standard_normal((B, Q))
    S = 4096
    got = bo.mvn_cdf(x, mean, cov, _sobol(S, max(Q - 1, 1)))
    ref = np.array([multivariate_normal(mean[b], cov[b] + 1e-6 * np.eye(Q)).cdf(x[b]) for b in range(B)])
    # Q = 1 is exact (one Phi); above, the QMC error of 4096 Sobol points plus SciPy's own 1e-5 allowance
    np.testing.assert_allclose(got, ref, rtol=0, atol=1e-12 if Q == 1 else 2e-3)


@pytest.mark.parametrize("q", [2, 3, 5])
def test_batch_ei_reproduces_monte_carlo_ei(q):
    # the reference's criterion: rtol 2e-2 against batch MC-EI with 1e5 samples (test_function.py:1214-1252)
    om = _quadratic_model(4, 2, seed=q)
    eta = float(o.predict(om, om.X)[0].min())
    X = np.random.default_rng(10 + q).uniform(size=(4, q, 2))
    got = bo.batch_expected_improvement_at(om, X, eta, _sobol(2000, q - 1))
    eps = np.random.default_rng(20 + q).standard_normal((1, q, 100_000))
    mc = o.batch_monte_carlo_expected_improvement(om, X, eps, eta)[:, 0]
    np.testing.assert_allclose(got, mc, rtol=2e-2)


@pytest.mark.parametrize("q", [2, 3, 4])
def test_reverse_pass_matches_finite_differences(q):
    om = o.synthetic_model(o.hartmann_6, 60, 6, kind="matern52", seed=q)
    eta = float(np.median(om.y))
    Xb = np.random.default_rng(q).uniform(size=(q, 6))
    w = _sobol(64, q - 1)
    value, grad = bo.bei_gradient(om, Xb, eta, w)
    np.testing.assert_allclose(value, bo.batch_expected_improvement_at(om, Xb[None], eta, w)[0], rtol=1e-12)
    h = 1e-6
    fd = np.zeros_like(grad)
    for j in range(q):
        for d in range(6):
            Xp, Xm = Xb.copy(), Xb.copy()
            Xp[j, d] += h
            Xm[j, d] -= h
            fd[j, d] = (bo.batch_expected_improvement_at(om, Xp[None], eta, w)[0]
                        - bo.batch_expected_improvement_at(om, Xm[None], eta, w)[0]) / (2 * h)
    np.testing.assert_allclose(grad, fd, rtol=1e-4, atol=1e-6 * np.abs(fd).max())


@pytest.mark.parametrize("q", [2, 4, 5])
def test_sobol_columns_are_the_same_in_every_dimension(q):
    # one w [S, q-1] serves the dimension-q CDFs (columns :q-1) and the dimension-(q-1) CDFs (columns :q-2)
    for skip in (0, 12_346):
        wide = _sobol(257, q, skip)
        np.testing.assert_array_equal(_sobol(257, q - 1, skip), wide[:, : q - 1])
        assert not np.any(np.all(wide == 0.0, axis=1))  # never the origin


def test_builder_argument_errors():
    from trieste_b200.acquisition import BatchExpectedImprovement, MultivariateNormalCDF

    for bad in (0, -3):
        with pytest.raises(ValueError):
            BatchExpectedImprovement(bad)
    with pytest.raises(ValueError):
        BatchExpectedImprovement(10, jitter=-1e-9)
    assert repr(BatchExpectedImprovement(100, jitter=1e-5)) == "BatchExpectedImprovement(100, jitter=1e-05)"
    for S, dim in ((0, 2), (5, 0)):
        with pytest.raises(ValueError):
            MultivariateNormalCDF(S, dim, np.float64)


def test_new_classes_follow_the_reference_protocols():
    # the pattern of test_protocol_conformance.py for the builder and its function class
    from trieste_b200.acquisition import function as f

    fixture = json.load(open(os.path.join(HERE, "golden", "reference_protocols.json")))
    protocols = {name: spec for classes in fixture.values() for name, spec in classes.items()}

    def methods(name):
        spec, out = protocols[name], {}
        for b in spec["bases"]:
            if b in protocols:
                out.update(methods(b))
        out.update(spec["methods"])
        return out

    for cls, proto in ((f.BatchExpectedImprovement, "SingleModelAcquisitionBuilder"),
                       (f.batch_expected_improvement, "AcquisitionFunctionClass")):
        for mname, m in methods(proto).items():
            assert hasattr(cls, mname), f"{cls.__name__} lacks {proto}.{mname}"
            if m["property"]:
                assert isinstance(inspect.getattr_static(cls, mname), property)
                continue
            params = [p for p in inspect.signature(getattr(cls, mname)).parameters.values() if p.name != "self"]
            positional = [p for p in params if p.kind in (p.POSITIONAL_ONLY, p.POSITIONAL_OR_KEYWORD)]
            assert [p.name for p in positional][: len(m["args"])] == m["args"], (cls.__name__, mname)
            for extra in positional[len(m["args"]):]:
                assert extra.default is not inspect.Parameter.empty, (cls.__name__, mname, extra.name)
            for name in m["with_default"]:
                assert next(p for p in positional if p.name == name).default is not inspect.Parameter.empty
