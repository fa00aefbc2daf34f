"""CPU: the active-learning oracle (tests/al_oracle.py) against central differences, the reference's jitter-on-every-entry
quirk of the predictive variance, and the builders' argument checks, reprs, update rule and protocol conformance."""
import inspect
import json
import os

import numpy as np
import pytest

from oracle import gp_oracle as o
from tests import al_oracle as al

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def om():
    return o.synthetic_model(o.hartmann_6, 120, 6)


def _fd(f, x, h):
    return (f(x + h) - f(x - h)) / (2 * h)


TAILS = {
    "bichon": (al.feasibility, al.feasibility_partials, (0.1, 1.0, 1)),
    "bichon_alpha": (al.feasibility, al.feasibility_partials, (-0.4, 0.35, 1)),
    "ranjan": (al.feasibility, al.feasibility_partials, (0.1, 1.0, 2)),
    "ranjan_alpha": (al.feasibility, al.feasibility_partials, (-0.4, 2.5, 2)),
    "bald": (al.bald, al.bald_partials, (1e-6,)),
    "bald_big_jitter": (al.bald, al.bald_partials, (0.05,)),
    "pv": (al.predictive_variance_single, al.predictive_variance_single_partials, (1e-6,)),
}


@pytest.mark.parametrize("name", list(TAILS))
def test_tail_partials_match_central_differences(name):
    value, partials, args = TAILS[name]
    rng = np.random.default_rng(3)
    mean = rng.normal(size=200)
    var = np.exp(rng.uniform(-4, 1, size=200))
    dm, dv = partials(mean, var, *args)
    h = 1e-6
    np.testing.assert_allclose(dm, _fd(lambda m: value(m, var, *args), mean, h), rtol=1e-6, atol=1e-8)
    hv = 1e-6 * var
    np.testing.assert_allclose(dv, (value(mean, var + hv, *args) - value(mean, var - hv, *args)) / (2 * hv), rtol=1e-6, atol=1e-8)


def test_bald_variance_partial_is_zero_below_the_jitter():
    mean = np.array([0.3, -1.0, 2.0])
    var = np.array([1e-8, 0.04, 0.2])
    dm, dv = al.bald_partials(mean, var, 0.05)
    assert dv[0] == 0.0 and dv[1] == 0.0 and dv[2] != 0.0
    assert np.all(dm != 0.0)
    # constant in var below the jitter
    assert al.bald(mean[:1], var[:1], 0.05) == al.bald(mean[:1], var[:1] * 3, 0.05)


def test_clipped_variance_has_zero_variance_partial():
    mean, var = np.array([0.1, 0.2]), np.array([1e-12, 0.5])
    clipped = np.array([True, False])
    for partials, args in ((al.feasibility_partials, (0.0, 1.0, 1)), (al.feasibility_partials, (0.0, 1.0, 2)),
                           (al.bald_partials, (1e-13,)), (al.predictive_variance_single_partials, (1e-6,))):
        _, dv = partials(mean, var, *args, clipped=clipped)
        assert dv[0] == 0.0 and dv[1] != 0.0


@pytest.mark.parametrize("name", ["bichon", "ranjan", "bald", "pv"])
def test_single_query_gradients_match_central_differences(om, name):
    value, partials, args = TAILS[name]
    if name in ("bichon", "ranjan"):
        args = (float(np.median(om.y)), 1.0, args[2])
    X = o.synthetic_model(o.hartmann_6, 12, 6, seed=5).X
    _, g = al.single_query(om, X, value, partials, *args)
    h = 1e-6
    for d in range(6):
        e = np.zeros(6)
        e[d] = h

        def f(x):
            m, v = o.predict(om, x)
            return value(m, v, *args)[:, 0]

        np.testing.assert_allclose(g[:, d], (f(X + e) - f(X - e)) / (2 * h), rtol=1e-5, atol=1e-7 * np.abs(g).max())


@pytest.mark.parametrize("q", [1, 2, 5, 8])
def test_batch_predictive_variance_gradient_matches_central_differences(om, q):
    rng = np.random.default_rng(q)
    Xb = rng.uniform(size=(q, 6))
    jitter = 1e-6
    val, g = al.predictive_variance_gradient(om, Xb, jitter)
    assert val == pytest.approx(al.predictive_variance(om, Xb[None], jitter)[0, 0], rel=1e-12)
    h = 1e-6
    fd = np.zeros_like(Xb)
    for j in range(q):
        for d in range(6):
            e = np.zeros_like(Xb)
            e[j, d] = h
            fd[j, d] = (al.predictive_variance(om, (Xb + e)[None], jitter) - al.predictive_variance(om, (Xb - e)[None], jitter))[0, 0] / (2 * h)
    np.testing.assert_allclose(g, fd, rtol=1e-5, atol=1e-6 * np.abs(fd).max())
    if q == 1:  # the q = 1 batch is var + jitter, and its gradient that of the single-query kind
        v1, g1 = al.single_query(om, Xb, al.predictive_variance_single, al.predictive_variance_single_partials, jitter)
        assert val == pytest.approx(v1[0, 0], rel=1e-12)
        np.testing.assert_allclose(g, g1, rtol=1e-9, atol=1e-12 * np.abs(g1).max())


def test_predictive_variance_adds_the_jitter_to_every_entry(om):
    """tf.linalg.logdet(covariance + jitter) broadcasts the scalar: M = cov + j 1 1^T, not cov + j I"""
    Xb = np.random.default_rng(7).uniform(size=(3, 4, 6))
    jitter = 0.05 * om.variance
    got = al.predictive_variance(om, Xb, jitter)[:, 0]
    _, cov = o.predict_joint(om, Xb)
    sign, ld = np.linalg.slogdet(cov[:, 0] + jitter * np.ones((4, 4)))
    assert np.all(sign > 0)
    np.testing.assert_allclose(got, np.exp(ld), rtol=1e-10)
    _, ld_eye = np.linalg.slogdet(cov[:, 0] + jitter * np.eye(4))
    assert np.all(np.abs(got / np.exp(ld_eye) - 1.0) > 1e-3)


# ---- builders -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("threshold", [[1.0], np.ones(2), [[0.0]]])
def test_expected_feasibility_raises_for_non_scalar_threshold(threshold):
    from trieste_b200.acquisition import ExpectedFeasibility

    with pytest.raises(ValueError):
        ExpectedFeasibility(threshold)


@pytest.mark.parametrize("alpha", [0.0, -1.0, -0.1])
def test_expected_feasibility_raises_for_non_positive_alpha(alpha):
    from trieste_b200.acquisition import ExpectedFeasibility

    with pytest.raises(ValueError):
        ExpectedFeasibility(0.0, alpha)


@pytest.mark.parametrize("alpha", [np.inf, np.nan, [1.0]])
def test_expected_feasibility_raises_for_non_finite_or_non_scalar_alpha(alpha):
    from trieste_b200.acquisition import ExpectedFeasibility

    with pytest.raises(ValueError):
        ExpectedFeasibility(0.0, alpha)


@pytest.mark.parametrize("delta", [-1, 0, 1.5, 3])
def test_expected_feasibility_raises_for_invalid_delta(delta):
    from trieste_b200.acquisition import ExpectedFeasibility

    with pytest.raises(ValueError):
        ExpectedFeasibility(0.0, 1.0, delta)


@pytest.mark.parametrize("jitter", [0.0, -1e-6])
def test_bald_raises_for_non_positive_jitter_when_the_function_is_built(jitter):
    from trieste_b200.acquisition import BayesianActiveLearningByDisagreement, bayesian_active_learning_by_disagreement

    builder = BayesianActiveLearningByDisagreement(jitter)  # the builder accepts it, as in the reference
    with pytest.raises(ValueError, match="Jitter must be positive"):
        builder.prepare_acquisition_function(object())
    with pytest.raises(ValueError, match="Jitter must be positive"):
        bayesian_active_learning_by_disagreement(object(), jitter)


def test_builders_reject_models_that_are_not_native():
    from trieste_b200.acquisition import BayesianActiveLearningByDisagreement, ExpectedFeasibility, PredictiveVariance

    for builder in (PredictiveVariance(), ExpectedFeasibility(0.0), ExpectedFeasibility(0.0, 2.0, 2),
                    BayesianActiveLearningByDisagreement()):
        with pytest.raises(ValueError, match="GaussianProcessRegression"):
            builder.prepare_acquisition_function(object())


def test_reprs_follow_the_reference():
    from trieste_b200.acquisition import BayesianActiveLearningByDisagreement, ExpectedFeasibility, PredictiveVariance

    assert repr(PredictiveVariance()) == "PredictiveVariance(jitter=1e-06)"
    assert repr(PredictiveVariance(0.5)) == "PredictiveVariance(jitter=0.5)"
    assert repr(ExpectedFeasibility(1.5)) == "ExpectedFeasibility(threshold=1.5, alpha=1, delta=1)"
    assert repr(ExpectedFeasibility(0, 0.5, 2)) == "ExpectedFeasibility(threshold=0, alpha=0.5, delta=2)"
    assert repr(BayesianActiveLearningByDisagreement()) == "BayesianActiveLearningByDisagreement(jitter=1e-06)"


def test_update_returns_the_same_function():
    from trieste_b200.acquisition import BayesianActiveLearningByDisagreement, ExpectedFeasibility, PredictiveVariance

    sentinel = object()
    for builder in (PredictiveVariance(), ExpectedFeasibility(0.0), BayesianActiveLearningByDisagreement()):
        assert builder.update_acquisition_function(sentinel, None) is sentinel


def test_new_symbols_are_exported_and_bound():
    import trieste_b200.acquisition as acq
    from trieste_b200 import _lib

    for name in ("PredictiveVariance", "predictive_variance", "ExpectedFeasibility", "bichon_ranjan_criterion",
                 "BayesianActiveLearningByDisagreement", "bayesian_active_learning_by_disagreement"):
        assert hasattr(acq, name), name
    assert (_lib.ACQ_FEASIBILITY_BICHON, _lib.ACQ_FEASIBILITY_RANJAN, _lib.ACQ_BALD, _lib.ACQ_PREDICTIVE_VARIANCE) == (10, 11, 12, 13)
    assert "tb_acq_set_feasibility" in _lib.SIGNATURES and "tb_acq_predictive_variance" in _lib.SIGNATURES


# ---- protocol conformance against the reference's extracted protocols ------------------------------------------------------
FIXTURE = json.load(open(os.path.join(HERE, "golden", "reference_protocols.json")))
PROTOCOLS = {name: spec for classes in FIXTURE.values() for name, spec in classes.items()}


def _methods(protocol):
    spec = PROTOCOLS[protocol]
    out = {}
    for b in spec["bases"]:
        if b in PROTOCOLS:
            out.update(_methods(b))
    out.update(spec["methods"])
    return out


def _conformance_cases():
    from trieste_b200.acquisition import active_learning as a

    pairs = [(c, "SingleModelAcquisitionBuilder") for c in (a.PredictiveVariance, a.ExpectedFeasibility,
                                                             a.BayesianActiveLearningByDisagreement)]
    pairs += [(c, "AcquisitionFunctionClass") for c in (a.predictive_variance, a.bichon_ranjan_criterion,
                                                         a.bayesian_active_learning_by_disagreement)]
    for cls, p in pairs:
        for mname, m in _methods(p).items():
            yield pytest.param(cls, p, mname, m, id=f"{cls.__name__}-{p}.{mname}")


@pytest.mark.parametrize("cls,protocol,mname,m", list(_conformance_cases()))
def test_active_learning_classes_offer_the_reference_protocol_methods(cls, protocol, mname, m):
    assert hasattr(cls, mname), f"{cls.__name__} lacks {protocol}.{mname}"
    params = [p for p in inspect.signature(getattr(cls, mname)).parameters.values() if p.name != "self"]
    positional = [p.name for p in params if p.kind in (p.POSITIONAL_ONLY, p.POSITIONAL_OR_KEYWORD)]
    assert positional[: len(m["args"])] == m["args"], (cls.__name__, mname, positional, m["args"])
