"""HIPPO on the host (CPU): the NumPy restatement tests/hippo_oracle.py against central differences and the reference's
log form, the reference's penaliser cases (trieste tests/unit/acquisition/multi_objective/test_function.py:852-906) on a
NumPy quadratic-mean model, and the builder's argument, dataset and protocol checks, all before any device call."""
import inspect
import json
import os

import numpy as np
import pytest

from tests import ehvi_oracle as eo
from tests import hippo_oracle as ho
from trieste_b200.acquisition.multi_objective import (Pareto, get_reference_point,
                                                      prepare_default_non_dominated_partition_bounds)

HERE = os.path.dirname(os.path.abspath(__file__))


class _Quadratic:
    """the reference's QuadraticMeanAndRBFKernel: mean sum(x^2), variance 1 (one output)"""

    def predict(self, x):
        x = np.asarray(x, dtype=np.float64)
        return np.sum(x * x, axis=-1, keepdims=True), np.ones(x.shape[:-1] + (1,))


class _TwoOutputs:
    """two outputs with x-dependent means and fixed variances, to check __call__ against the oracle"""

    def predict(self, x):
        x = np.asarray(x, dtype=np.float64)
        mean = np.stack([np.sum(x * x, axis=-1), np.sin(x[..., 0]) + x[..., -1]], axis=-1)
        return mean, np.broadcast_to([0.3, 2.0], mean.shape).copy()


def _cells(L, seed):
    """the partition of a random front: six points up to four objectives, four from five on (hundreds to thousands of
    cells)"""
    rng = np.random.default_rng(seed)
    front = Pareto(rng.uniform(0.0, 1.0, size=(6 if L <= 4 else 4, L))).front
    return prepare_default_non_dominated_partition_bounds(get_reference_point(front), front)


def _moments(M, L, seed):
    rng = np.random.default_rng(seed)
    return rng.uniform(-0.5, 1.5, size=(M, L)), rng.uniform(0.01, 0.5, size=(M, L))


@pytest.mark.parametrize("L, P", [(2, 1), (2, 4), (3, 3), (4, 7), (5, 2), (6, 5), (7, 1), (8, 9)])
def test_penalty_partials_match_central_differences(L, P):
    mean, _ = _moments(60, L, L + P)
    pmean, pvar = _moments(P, L, 100 + P)
    mean[0] = pmean[0] + 1e-3 * np.arange(1, L + 1)  # near a pending point, not at it
    dpen = ho.penalty_partials(mean, pmean, pvar)
    h = 1e-7
    for l in range(L):
        e = np.zeros(L)
        e[l] = h
        fd = (ho.penalty(mean + e, pmean, pvar) - ho.penalty(mean - e, pmean, pvar)) / (2 * h)
        np.testing.assert_allclose(dpen[:, l], fd, rtol=1e-6, atol=1e-9)
    assert ho.penalty(mean[:1], pmean, pvar)[0] > 0


@pytest.mark.parametrize("L, P", [(2, 1), (3, 2), (4, 5), (5, 3), (6, 1), (7, 2), (8, 4)])
def test_penalised_partials_match_central_differences(L, P):
    lower, upper = _cells(L, L)
    mean, var = _moments(50, L, 3 + L)
    pmean, pvar = _moments(P, L, 40 + P)
    dmu, dvar = ho.partials(mean, var, lower, upper, pmean, pvar)
    for l in range(L):
        e = np.zeros(L)
        e[l] = 1.0
        h = 1e-6
        fd_mu = (ho.value(mean + h * e, var, lower, upper, pmean, pvar)
                 - ho.value(mean - h * e, var, lower, upper, pmean, pvar)) / (2 * h)
        hv = 1e-6 * var[:, l:l + 1] * e
        fd_var = (ho.value(mean, var + hv, lower, upper, pmean, pvar)
                  - ho.value(mean, var - hv, lower, upper, pmean, pvar)) / (2 * hv[:, l])
        np.testing.assert_allclose(dmu[:, l], fd_mu, rtol=1e-6, atol=1e-9)
        np.testing.assert_allclose(dvar[:, l], fd_var, rtol=1e-5, atol=1e-8)


def test_penalised_gradient_in_x_matches_central_differences():
    from oracle import gp_oracle as o

    oms = [o.synthetic_model(o.hartmann_6, 60, 6, seed=0),
           o.synthetic_model(lambda x: o.random_fourier_objective(x, seed=3), 60, 6, seed=1)]
    Y = np.concatenate([om.y.reshape(-1, 1) for om in oms], axis=1)
    front = Pareto(Y).front
    lower, upper = prepare_default_non_dominated_partition_bounds(get_reference_point(front), front)
    rng = np.random.default_rng(5)
    P = rng.uniform(0, 1, size=(3, 6))
    pm, pv = zip(*(o.predict(om, P) for om in oms))
    pmean, pvar = np.concatenate(pm, axis=1), np.concatenate(pv, axis=1)
    X = rng.uniform(0, 1, size=(20, 6))

    def val(Xq):
        mean, var = zip(*(o.predict(om, Xq) for om in oms))
        return ho.value(np.concatenate(mean, axis=1), np.concatenate(var, axis=1), lower, upper, pmean, pvar)

    grad = ho.gradient(oms, X, lower, upper, pmean, pvar, o.predict, o.posterior_gradients)
    h = 1e-6
    for j in range(6):
        e = np.zeros(6)
        e[j] = h
        fd = (val(X + e) - val(X - e)) / (2 * h)
        np.testing.assert_allclose(grad[:, j], fd, rtol=1e-5, atol=1e-8 * np.abs(grad).max())


def test_penalty_is_zero_at_pending_points_and_tends_to_one():
    from trieste_b200.acquisition import hippo_penalizer

    pending = np.array([[0.0, 1.0], [2.0, 3.0], [3.0, 4.0]])
    hp = hippo_penalizer(_Quadratic(), pending)
    for p in pending:
        assert hp(p[None, None, :])[0, 0] == 0.0
    far = hp(np.array([[[100.0, 100.0]]]))[0, 0]
    assert 0.99 < far < 1.0
    assert np.all(np.diff(hp(np.array([[[10.0, 10.0]], [[30.0, 30.0]], [[100.0, 100.0]]]))[:, 0]) > 0)
    # the oracle's restatement agrees, and the penalty ignores the candidate's variances
    pmean, pvar = _Quadratic().predict(pending)
    x = np.random.default_rng(0).uniform(-3, 3, size=(40, 1, 2))
    mean = _Quadratic().predict(x[:, 0])[0]
    np.testing.assert_allclose(hp(x)[:, 0], ho.penalty(mean, pmean, pvar), rtol=1e-14)
    assert np.all(ho.penalty(pmean, pmean, pvar) == 0.0)


def test_penaliser_call_matches_the_oracle_with_several_outputs():
    from trieste_b200.acquisition import hippo_penalizer

    model = _TwoOutputs()
    rng = np.random.default_rng(3)
    pending = rng.uniform(-1, 1, size=(5, 3))
    hp = hippo_penalizer(model, pending)
    np.testing.assert_array_equal(hp._pending_points, pending)
    x = rng.uniform(-1, 1, size=(30, 1, 3))
    pmean, pvar = model.predict(pending)
    out = hp(x)
    assert out.shape == (30, 1)
    np.testing.assert_allclose(out[:, 0], ho.penalty(model.predict(x[:, 0])[0], pmean, pvar), rtol=1e-14)
    hp.update(pending[:2])
    np.testing.assert_allclose(hp(x)[:, 0], ho.penalty(model.predict(x[:, 0])[0], pmean[:2], pvar[:2]), rtol=1e-14)


@pytest.mark.parametrize("L", [2, 3, 5, 8])
def test_product_agrees_with_the_reference_log_form(L):
    lower, upper = _cells(L, 9)
    mean, var = _moments(200, L, 2)
    pmean, pvar = _moments(4, L, 8)
    e = eo.ehvi(mean, var, lower, upper)
    pen = ho.penalty(mean, pmean, pvar)
    assert np.all(e > 0) and np.all(pen > 0)
    logform = np.exp(np.log(e) + np.log(pen))
    prod = ho.value(mean, var, lower, upper, pmean, pvar)
    assert np.all(np.abs(prod - logform) <= 8 * np.spacing(np.abs(logform)))


@pytest.mark.parametrize("at", [np.zeros((2, 1)), np.zeros((1, 2, 1))])
def test_penaliser_rejects_batches_of_points(at):
    from trieste_b200.acquisition import hippo_penalizer

    hp = hippo_penalizer(_Quadratic(), np.zeros((1, 2)))
    with pytest.raises(ValueError):
        hp(at)


def test_penaliser_rejects_empty_pending_points():
    from trieste_b200.acquisition import hippo_penalizer

    with pytest.raises(ValueError):
        hippo_penalizer(_Quadratic(), None)
    with pytest.raises(ValueError):
        hippo_penalizer(_Quadratic(), np.zeros((0, 2)))
    hp = hippo_penalizer(_Quadratic(), np.zeros((1, 2)))
    with pytest.raises(ValueError):
        hp.update(None)
    with pytest.raises(ValueError):
        hp.update(np.zeros((0, 2)))
    with pytest.raises(ValueError, match="rank 2"):
        hp.update(np.zeros((2, 1, 2)))


def test_builder_argument_and_dataset_errors_without_a_device():
    from trieste_b200 import Dataset
    from trieste_b200.acquisition import HIPPO, ExpectedHypervolumeImprovement, ExpectedImprovement, Fantasizer

    with pytest.raises(ValueError, match="ExpectedHypervolumeImprovement"):
        HIPPO(base_acquisition_function_builder=ExpectedImprovement())
    with pytest.raises(ValueError, match="ExpectedHypervolumeImprovement"):
        HIPPO(base_acquisition_function_builder=Fantasizer())
    with pytest.raises(ValueError, match="ExpectedHypervolumeImprovement"):
        HIPPO(base_acquisition_function_builder=object())
    HIPPO("NA", ExpectedHypervolumeImprovement().using("NA"))
    models = {"NA": _Quadratic()}
    empty = {"NA": Dataset(np.zeros((0, 2)), np.zeros((0, 3)))}
    hippo = HIPPO("NA")
    for datasets in (None, {}, {"NA": None}, empty):
        with pytest.raises(ValueError, match="populated"):
            hippo.prepare_acquisition_function(models, datasets)
        with pytest.raises(ValueError, match="populated"):
            hippo.update_acquisition_function(None, models, datasets)
    data = {"NA": Dataset(np.zeros((3, 2)), np.ones((3, 3)))}
    with pytest.raises(ValueError, match="prepare_acquisition_function must be called"):
        hippo.update_acquisition_function(None, models, data)
    with pytest.raises(ValueError, match="ModelStack"):  # the base function's own check, before any device call
        hippo.prepare_acquisition_function({"NA": _TwoOutputs()}, {"NA": Dataset(np.zeros((3, 3)), np.ones((3, 2)))})
    assert repr(HIPPO()).startswith("HIPPO('OBJECTIVE', ExpectedHypervolumeImprovement(get_reference_point) using tag")


def test_builder_follows_the_greedy_builder_protocol():
    from trieste_b200.acquisition import HIPPO, GreedyAcquisitionFunctionBuilder
    from trieste_b200.acquisition.interface import OBJECTIVE

    assert issubclass(HIPPO, GreedyAcquisitionFunctionBuilder)
    fixture = json.load(open(os.path.join(HERE, "golden", "reference_protocols.json")))
    protocol = fixture["acquisition/interface.py"]["GreedyAcquisitionFunctionBuilder"]["methods"]
    for name, m in protocol.items():
        params = [p for p in inspect.signature(getattr(HIPPO, name)).parameters.values() if p.name != "self"]
        assert [p.name for p in params] == m["args"]
        for p in params:
            assert (p.default is not inspect.Parameter.empty) == (p.name in m["with_default"]), (name, p.name)
    init = [p for p in inspect.signature(HIPPO.__init__).parameters.values() if p.name != "self"]
    assert [(p.name, p.default) for p in init] == [("objective_tag", OBJECTIVE), ("base_acquisition_function_builder", None)]
    assert inspect.signature(HIPPO.update_acquisition_function).parameters["new_optimization_step"].default is True
