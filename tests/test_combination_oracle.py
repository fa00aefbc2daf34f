"""CPU tests of the acquisition reducers: the reference's unit tests of trieste/acquisition/combination.py restated with
static NumPy builders, the composed route's gradients against central differences (a product with an exactly zero
factor, MakePositive), and the NumPy oracle of the fused reductions (tests/reduce_oracle.py) against central
differences."""
import numpy as np
import pytest

from oracle import gp_oracle as o
from tests import reduce_oracle as ro
from trieste_b200.acquisition import MakePositive, Product, Reducer, SingleModelAcquisitionBuilder, Sum
from trieste_b200.acquisition.combination import Map, composed_acquisition, differentiable_composed_acquisition
from trieste_b200.acquisition.interface import AcquisitionFunctionBuilder

TAG = ""
MODELS = {TAG: None}


class _Static(AcquisitionFunctionBuilder):
    def __init__(self, f):
        self._f = f

    def prepare_acquisition_function(self, models, datasets=None):
        return self._f

    def update_acquisition_function(self, function, models, datasets=None):
        return lambda x: function(x) + 1


def _xs(seed=0):
    return np.random.default_rng(seed).uniform(-1.0, 1.0, size=(3, 5, 1))


def test_reducer_raises_for_no_builders():
    class UseFirst(Reducer):
        def _reduce(self, inputs):
            return inputs[0]

    with pytest.raises(ValueError, match="At least one acquisition builder expected"):
        UseFirst()


def test_reducer_repr_builders():
    class Dummy(Reducer):
        def _reduce(self, inputs):
            raise AssertionError

    class Builder(AcquisitionFunctionBuilder):
        def __init__(self, name):
            self._name = name

        def __repr__(self):
            return f"Builder({self._name!r})"

        def prepare_acquisition_function(self, models, datasets=None):
            raise AssertionError

    assert repr(Dummy(Builder("foo"))) == "Dummy(Builder('foo'))"
    assert repr(Dummy(Builder("foo"), Builder("bar"))) == "Dummy(Builder('foo'), Builder('bar'))"


def test_reducer_reduce():
    class Mean(Reducer):
        def _reduce(self, inputs):
            return np.mean(inputs, axis=0)

    acq = Mean(_Static(lambda x: -2.0 * x), _Static(lambda x: 3.0 * x)).prepare_acquisition_function(MODELS)
    xs = _xs()
    np.testing.assert_allclose(acq(xs), 0.5 * xs)
    assert not hasattr(acq, "value_and_gradient")  # a custom _reduce gives values only


def test_sum():
    acq = Sum(_Static(lambda x: x), _Static(lambda x: x**2), _Static(lambda x: x**3)).prepare_acquisition_function(MODELS)
    xs = _xs()
    np.testing.assert_allclose(acq(xs), xs + xs**2 + xs**3)


def test_product():
    acq = Product(_Static(lambda x: x + 1), _Static(lambda x: x + 2)).prepare_acquisition_function(MODELS)
    xs = _xs()
    np.testing.assert_allclose(acq(xs), (xs + 1) * (xs + 2))


def test_reducer_calls_update():
    prod = Product(_Static(lambda x: x + 1), _Static(lambda x: x + 2))
    acq = prod.prepare_acquisition_function(MODELS)
    acq = prod.update_acquisition_function(acq, MODELS)
    xs = _xs()
    np.testing.assert_allclose(acq(xs), (xs + 2) * (xs + 3))


@pytest.mark.parametrize("reducer_class", [Sum, Product])
def test_sum_and_product_for_single_builder(reducer_class):
    acq = reducer_class(_Static(lambda x: x**2)).prepare_acquisition_function(MODELS)
    xs = _xs()
    np.testing.assert_allclose(acq(xs), xs**2)


def test_map():
    red = Map(lambda x: x + 1, _Static(lambda x: x + 2))
    acq = red.prepare_acquisition_function(MODELS)
    xs = _xs()
    np.testing.assert_allclose(acq(xs), xs + 3)
    assert isinstance(acq, composed_acquisition) and not hasattr(acq, "value_and_gradient")


def test_reducers_exported():
    import trieste_b200.acquisition as acq
    from trieste_b200.acquisition import combination

    for name in ("Sum", "Product", "Reducer", "MakePositive"):
        assert hasattr(acq, name)
    assert combination.Map is Map


def test_a_subclass_with_its_own_reduce_gives_values_only():
    class Doubled(Sum):
        def _reduce(self, inputs):
            return 2 * super()._reduce(inputs)

    acq = Doubled(_Static(_Quadratic(1.0)), _Static(_Quadratic(2.0))).prepare_acquisition_function(MODELS)
    x = _xs()
    np.testing.assert_allclose(acq(x), 2 * (_Quadratic(1.0)(x) + _Quadratic(2.0)(x)))
    assert not hasattr(acq, "value_and_gradient")


# ---- the composed route's gradients
class _Quadratic:
    """f(x) = c - |x - 0.1 c|^2 over [..., 1, D] -> [..., 1], with value_and_gradient"""

    def __init__(self, c):
        self.c = c

    def __call__(self, x):
        return self.c - np.sum((x - 0.1 * self.c) ** 2, axis=-1)

    def value_and_gradient(self, x):
        return self(x), -2 * (x - 0.1 * self.c)


class _Linear:
    """f(x) = x_0 (exactly zero at x_0 = 0)"""

    def __call__(self, x):
        return x[..., 0].copy()

    def value_and_gradient(self, x):
        g = np.zeros_like(x)
        g[..., 0] = 1.0
        return self(x), g


def _central(fn, x, h=1e-6):
    g = np.zeros_like(x)
    for d in range(x.shape[-1]):
        e = np.zeros_like(x)
        e[..., d] = h
        g[..., d] = (np.asarray(fn(x + e)) - np.asarray(fn(x - e)))[..., 0][..., None] / (2 * h)
    return g


@pytest.mark.parametrize("reducer_class", [Sum, Product])
def test_composed_gradient_matches_central_differences(reducer_class):
    acq = reducer_class(*[_Static(_Quadratic(c)) for c in (1.0, 2.0, 3.0)]).prepare_acquisition_function(MODELS)
    assert isinstance(acq, differentiable_composed_acquisition)
    x = np.random.default_rng(3).uniform(size=(7, 1, 4))
    v, g = acq.value_and_gradient(x)
    np.testing.assert_allclose(v, acq(x), rtol=1e-14)
    np.testing.assert_allclose(g, _central(acq, x), rtol=1e-6, atol=1e-8)


def test_composed_product_with_an_exactly_zero_factor_has_a_finite_gradient():
    acq = Product(_Static(_Linear()), _Static(_Quadratic(2.0)), _Static(_Quadratic(1.0))).prepare_acquisition_function(MODELS)
    x = np.random.default_rng(4).uniform(size=(5, 1, 3))
    x[:, 0, 0] = 0.0
    v, g = acq.value_and_gradient(x)
    assert np.all(v == 0.0) and np.all(np.isfinite(g))
    np.testing.assert_allclose(g, _central(acq, x), rtol=1e-6, atol=1e-8)


class _StaticSingle(SingleModelAcquisitionBuilder):
    def __init__(self, f):
        self._f = f

    def prepare_acquisition_function(self, model, dataset=None):
        return self._f

    def update_acquisition_function(self, function, model, dataset=None):
        return function


def test_make_positive_values_gradient_and_update():
    base = _Quadratic(1.0)
    builder = MakePositive(_StaticSingle(base))
    assert repr(builder).startswith("MakePositive(")
    acq = builder.prepare_acquisition_function(None)
    x = np.random.default_rng(5).uniform(-2, 2, size=(6, 1, 3))
    np.testing.assert_allclose(acq(x), np.log(1 + np.exp(base(x))), rtol=1e-14)
    v, g = acq.value_and_gradient(x)
    np.testing.assert_allclose(g, _central(acq, x), rtol=1e-6, atol=1e-8)
    assert builder.update_acquisition_function(acq, None) is acq  # the base builder updated in place
    assert np.all(acq(x) > 0)


def test_make_positive_update_rebuilds_for_a_new_base_function():
    class Fresh(_StaticSingle):
        def update_acquisition_function(self, function, model, dataset=None):
            return _Quadratic(3.0)

    builder = MakePositive(Fresh(_Quadratic(1.0)))
    acq = builder.prepare_acquisition_function(None)
    new = builder.update_acquisition_function(acq, None)
    assert new is not acq
    x = np.random.default_rng(6).uniform(size=(4, 1, 2))
    np.testing.assert_allclose(new(x), np.log(1 + np.exp(_Quadratic(3.0)(x))))


def test_deepcopy_of_a_prepared_reducer_holds_no_function():
    import copy

    red = Sum(_Static(_Quadratic(1.0)))
    red.prepare_acquisition_function(MODELS)
    cp = copy.deepcopy(red)
    assert cp._function is None and not hasattr(cp, "functions") and cp.acquisitions[0] is not red.acquisitions[0]


# ---- the oracle of the fused reductions
KINDS = [("ei", dict(param=0.3)), ("log_ei", dict(param=-0.2)), ("pbt", dict(param=0.1)), ("lcb", dict(param=1.5)),
         ("neg_lcb", dict(param=2.0)), ("aei", dict(param=0.2)), ("mes", dict(samples=np.array([[-0.5], [0.1], [0.4]]))),
         ("bichon", dict(param=0.2, alpha=1.3)), ("ranjan", dict(param=-0.1, alpha=0.7)), ("bald", dict(param=1e-6)),
         ("pv", dict(param=1e-6))]


@pytest.mark.parametrize("kind,kw", KINDS, ids=[k for k, _ in KINDS])
def test_oracle_kind_partials_match_central_differences(kind, kw):
    rng = np.random.default_rng(7)
    mean = rng.normal(size=(9, 1)) * 0.5
    var = rng.uniform(0.05, 1.0, size=(9, 1))
    v, dm, dv = ro.kind_value_partials(kind, mean, var, noise=0.01, **kw)
    h = 1e-6
    fm = lambda m: ro.kind_value_partials(kind, m, var, noise=0.01, **kw)[0]  # noqa: E731
    fv = lambda s: ro.kind_value_partials(kind, mean, s, noise=0.01, **kw)[0]  # noqa: E731
    np.testing.assert_allclose(dm, (fm(mean + h) - fm(mean - h)) / (2 * h), rtol=1e-5, atol=1e-8)
    np.testing.assert_allclose(dv, (fv(var + h) - fv(var - h)) / (2 * h), rtol=1e-5, atol=1e-8)


@pytest.mark.parametrize("op", ["sum", "product", "softplus"])
def test_oracle_reduction_gradient_matches_central_differences(op):
    om1 = o.synthetic_model(o.hartmann_6, 40, 6, seed=0)
    om2 = o.synthetic_model(lambda x: o.random_fourier_objective(x, seed=3), 30, 6, seed=1)
    terms = [("ei", om1, dict(param=o.ei_eta(om1))), ("pbt", om2, dict(param=0.0)), ("bichon", om2, dict(param=0.1, alpha=1.0)),
             ("neg_lcb", om1, dict(param=1.0))]
    if op == "softplus":
        terms = terms[:1]
    X = np.random.default_rng(8).uniform(size=(6, 6))
    v, g, dvar = ro.reduction(op, terms, X)
    assert set(dvar) == {id(t[1]) for t in terms}
    h = 1e-6
    for d in range(6):
        e = np.zeros_like(X)
        e[:, d] = h
        fd = (ro.reduction(op, terms, X + e)[0] - ro.reduction(op, terms, X - e)[0]) / (2 * h)
        np.testing.assert_allclose(g[:, d : d + 1], fd, rtol=1e-5, atol=1e-8)
