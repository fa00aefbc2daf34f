"""Acquisition reducers on the device (csrc/reduce.cuh, tb_reduce_*) against the NumPy oracle in tests/reduce_oracle.py:
values and gradients of sums and products over several GPs on every engine and on fp32 handles, every fused kind as a
term, the fused route against the composed route, shared handles, members of different sizes over several chunks, the
fused argmax with ties and NaN, the device L-BFGS against SciPy, member state, the C-ABI errors and a constrained BO loop.

Tolerances.  Each member's variance carries its engine's stated error eps sigma_f^2 (fp64 1e-12, int8 engines 1e-9),
which reaches the reduced value through d value / d var_m; the allowance is that product from the oracle, summed over
the members, times 10 (as for EHVI)."""
import ctypes as C

import numpy as np
import pytest

from oracle import gp_oracle as o
from tests import reduce_oracle as ro
from tests.test_gpu_fp32 import _assert_fp32_gradient, _pair32
from tests.util import candidates, model_pair

pytestmark = pytest.mark.gpu

ENGINE_VAR_EPS = {"int8": 1e-9, "int8x21": 1e-9, "fp64": 1e-12}


def _obj(seed):
    return lambda x: o.random_fourier_objective(x, seed=seed)


def _pairs(engine, Ns=(300, 200, 250), D=6):
    objs = [o.hartmann_6, _obj(3), _obj(5)]
    return [model_pair(objs[i], N, D, seed=i, engine=engine) for i, N in enumerate(Ns)]


def _fn(kind, nm, **kw):
    """the native single-query function of a kind, and the oracle kwargs of the same term"""
    from trieste_b200.acquisition import (augmented_expected_improvement, bayesian_active_learning_by_disagreement,
                                          bichon_ranjan_criterion, expected_improvement, log_expected_improvement,
                                          lower_confidence_bound, min_value_entropy_search, predictive_variance,
                                          probability_below_threshold)
    from trieste_b200.acquisition.function import _lcb

    p = kw.get("param", 0.0)
    if kind == "ei":
        return expected_improvement(nm, p)
    if kind == "log_ei":
        return log_expected_improvement(nm, p)
    if kind == "aei":
        return augmented_expected_improvement(nm, p)
    if kind == "pbt":
        return probability_below_threshold(nm, p)
    if kind == "lcb":
        return lower_confidence_bound(nm, p)
    if kind == "neg_lcb":
        return _lcb(nm, p, negate=True)
    if kind == "mes":
        return min_value_entropy_search(nm, kw["samples"])
    if kind in ("bichon", "ranjan"):
        return bichon_ranjan_criterion(nm, p, kw["alpha"], 1 if kind == "bichon" else 2)
    if kind == "bald":
        return bayesian_active_learning_by_disagreement(nm, p)
    if kind == "pv":
        return predictive_variance(nm, p)
    raise ValueError(kind)


def _reduced(op, fns):
    from trieste_b200.acquisition.combination import REDUCE_PRODUCT, REDUCE_SOFTPLUS, REDUCE_SUM, reduced_acquisition

    return reduced_acquisition({"sum": REDUCE_SUM, "product": REDUCE_PRODUCT, "softplus": REDUCE_SOFTPLUS}[op], fns)


def _allowance(dvar, pairs_engines, ref):
    tol = 1e-12 * np.abs(ref) + 1e-13
    for om, eng in pairs_engines:
        if id(om) in dvar:
            tol = tol + 10.0 * ENGINE_VAR_EPS[eng] * om.variance * dvar[id(om)]
    return tol


def _check(op, terms, X, engine):
    """terms: (kind, (om, nm), kw) -> checks values and gradients of the fused reduction against the oracle"""
    fn = _reduced(op, [_fn(k, nm, **kw) for k, (om, nm), kw in terms])
    oterms = [(k, om, kw) for k, (om, nm), kw in terms]
    ref, rg, dvar = ro.reduction(op, oterms, X)
    got = fn(X[:, None, :])
    ok = np.abs(got - ref) <= _allowance(dvar, {id(om): (om, engine) for _, (om, _), _ in terms}.values(), ref)
    assert ok.all(), (op, np.abs(got - ref).max())
    vals, grad = fn.value_and_gradient(X[:400, None, :])
    np.testing.assert_array_equal(vals, fn(X[:400, None, :]))
    scale = np.abs(rg[:400]).max(axis=1, keepdims=True)
    live = scale[:, 0] > 1e-8 * np.abs(rg).max()
    err = np.abs(grad[:400, 0, :] - rg[:400]) / np.maximum(scale, 1e-300)
    assert err[live].max() < 1e-6, (op, err[live].max())
    return fn


@pytest.mark.parametrize("engine", ["fp64", "int8", "int8x21"])
@pytest.mark.parametrize("case", ["ei_x_pof", "ei_plus_pof", "pof_x_pof"])
def test_values_and_gradients_against_oracle(engine, case):
    (o0, n0), (o1, n1), (o2, n2) = _pairs(engine)
    X = np.concatenate([candidates(5000, 6, seed=2), o0.X[:10], o1.X[:10]])
    eta = o.ei_eta(o0)
    if case == "ei_x_pof":
        _check("product", [("ei", (o0, n0), dict(param=eta)), ("pbt", (o1, n1), dict(param=0.0))], X, engine)
    elif case == "ei_plus_pof":
        _check("sum", [("ei", (o0, n0), dict(param=eta)), ("pbt", (o1, n1), dict(param=0.0))], X, engine)
    else:
        _check("product", [("pbt", (o1, n1), dict(param=0.0)), ("pbt", (o2, n2), dict(param=0.2))], X, engine)


def test_fp32_handles():
    o0, n0 = _pair32(o.hartmann_6, 300, 6)
    o1, n1 = _pair32(_obj(3), 200, 6)
    X = candidates(3000, 6, seed=4).astype(np.float32)
    X64 = X.astype(np.float64)
    eta = o.ei_eta(o0)
    fn = _reduced("product", [_fn("ei", n0, param=eta), _fn("pbt", n1, param=0.0)])
    ref, rg, _ = ro.reduction("product", [("ei", o0, dict(param=eta)), ("pbt", o1, dict(param=0.0))], X64)
    got = fn(X[:, None, :])
    assert got.dtype == np.float32
    np.testing.assert_allclose(got.astype(np.float64), ref, rtol=1e-4, atol=1e-4 * np.abs(ref).max())
    vals, grad = fn.value_and_gradient(X[:300, None, :])
    assert grad.dtype == np.float32
    live = np.abs(rg[:300]).max(axis=1) > 1e-3 * np.abs(rg[:300]).max()
    _assert_fp32_gradient(grad[:300, 0, :][live], rg[:300][live])


KIND_KW = [("ei", dict(param=-0.5)), ("log_ei", dict(param=-0.5)), ("pbt", dict(param=0.1)), ("lcb", dict(param=1.5)),
           ("neg_lcb", dict(param=2.0)), ("aei", dict(param=-0.4)), ("mes", dict(samples=np.array([[-1.5], [-1.0], [-0.8]]))),
           ("bichon", dict(param=0.2, alpha=1.3)), ("ranjan", dict(param=-0.1, alpha=0.7)), ("bald", dict(param=1e-6)),
           ("pv", dict(param=1e-6))]


@pytest.mark.parametrize("op", ["sum", "product"])
@pytest.mark.parametrize("kind,kw", KIND_KW, ids=[k for k, _ in KIND_KW])
def test_every_kind_as_a_term(op, kind, kw):
    (o0, n0), (o1, n1), _ = _pairs("fp64")
    X = candidates(2000, 6, seed=5)
    _check(op, [(kind, (o0, n0), kw), ("pbt", (o1, n1), dict(param=0.3))], X, "fp64")


def test_make_positive_over_a_fused_function():
    from trieste_b200.acquisition import MakePositive, NegativeLowerConfidenceBound
    from trieste_b200.acquisition.combination import reduced_acquisition

    (o0, n0), _, _ = _pairs("fp64")
    fn = MakePositive(NegativeLowerConfidenceBound(2.0)).prepare_acquisition_function(n0)
    assert isinstance(fn, reduced_acquisition)
    X = candidates(2000, 6, seed=6)
    ref, rg, _ = ro.reduction("softplus", [("neg_lcb", o0, dict(param=2.0))], X)
    np.testing.assert_allclose(fn(X[:, None, :]), ref, rtol=1e-11)
    _, grad = fn.value_and_gradient(X[:, None, :])
    np.testing.assert_allclose(grad[:, 0, :], rg, rtol=1e-7, atol=1e-9 * np.abs(rg).max())


class _Plain:
    """a child as a plain callable with value_and_gradient: forces the composed route"""

    def __init__(self, f):
        self.f = f

    def __call__(self, x):
        return self.f(x)

    def value_and_gradient(self, x):
        return self.f.value_and_gradient(x)


@pytest.mark.parametrize("op", ["sum", "product"])
def test_fused_agrees_with_composed(op):
    from trieste_b200.acquisition.combination import Product, Sum, differentiable_composed_acquisition, reduce_functions

    (o0, n0), (o1, n1), (o2, n2) = _pairs("int8")
    fns = [_fn("ei", n0, param=o.ei_eta(o0)), _fn("pbt", n1, param=0.0), _fn("bichon", n2, param=0.1, alpha=1.2),
           _fn("neg_lcb", n0, param=1.0)]
    cls = Sum if op == "sum" else Product
    fused = _reduced(op, fns)
    red = cls(object())
    composed = reduce_functions(red._op, red._reduce, [_Plain(fns[0])] + fns[1:])
    assert isinstance(composed, differentiable_composed_acquisition)
    X = candidates(3000, 6, seed=7)[:, None, :]
    v1, g1 = fused.value_and_gradient(X)
    v2, g2 = composed.value_and_gradient(X)
    np.testing.assert_allclose(v1, v2, rtol=1e-13, atol=1e-15)
    np.testing.assert_allclose(g1, g2, rtol=1e-12, atol=1e-14 * np.abs(g2).max())
    np.testing.assert_allclose(fused(X), composed(X), rtol=1e-13, atol=1e-15)


def test_shared_handles_run_one_member_step():
    from trieste_b200 import _lib

    (o0, n0), _, _ = _pairs("fp64")
    X = candidates(1000, 6, seed=8)[:, None, :]
    one = _reduced("sum", [_fn("ei", n0, param=o.ei_eta(o0))])
    two = _reduced("sum", [_fn("ei", n0, param=o.ei_eta(o0)), _fn("neg_lcb", n0, param=1.0)])
    counts = []
    for fn in (one, two):
        fn(X)  # warm
        _lib.lib().tb_launch_count_reset()
        fn(X)
        counts.append(_lib.lib().tb_launch_count())
    assert counts[0] == counts[1] and counts[0] > 0
    ref, _, _ = ro.reduction("sum", [("ei", o0, dict(param=o.ei_eta(o0))), ("neg_lcb", o0, dict(param=1.0))], X[:, 0, :])
    np.testing.assert_allclose(two(X), ref, rtol=1e-10, atol=1e-12)
    # two feasibility terms with different alpha on one model: the values of two separate functions
    f1, f2 = _fn("bichon", n0, param=0.2, alpha=0.5), _fn("bichon", n0, param=0.2, alpha=2.0)
    both = _reduced("sum", [f1, f2])
    np.testing.assert_allclose(both(X), f1(X) + f2(X), rtol=1e-13, atol=1e-15)


def test_range_of_members_chunks_ties_and_nan():
    D = 6
    specs = [(o.hartmann_6, 50, "rbf", 1e-3, "fp64"), (_obj(3), 300, "matern32", 1e-5, "int8"),
             (_obj(5), 2000, "matern52", None, "int8x21")]
    pairs = [model_pair(f, N, D, kind=k, seed=i, noise=nz, engine=e) for i, (f, N, k, nz, e) in enumerate(specs)]
    (o0, n0), (o1, n1), (o2, n2) = pairs
    fns = [_fn("ei", n0, param=o.ei_eta(o0)), _fn("pbt", n1, param=0.0), _fn("pbt", n2, param=0.2)]
    fn = _reduced("product", fns)
    X = candidates(300000, D, seed=9)
    X[1000] = X[250000]  # a tie: the lower index wins
    X[5] = np.nan  # NaN never wins
    vals = fn(X[:, None, :])[:, 0]
    assert np.isnan(vals[5])
    finite = np.where(np.isnan(vals), -np.inf, vals)
    idx, best = fn.fused_argmax(X)
    assert idx == int(np.argmax(finite)) and best == finite[idx]
    Xt = X.copy()
    Xt[123456] = X[idx]  # a later copy of the winner: the first stays
    assert fn.fused_argmax(Xt)[0] == idx
    Xw = Xt.copy()
    Xw[100] = X[idx]
    assert fn.fused_argmax(Xw)[0] == 100
    sub = X[np.r_[0:4, 6:2000]]
    ref, _, dvar = ro.reduction("product", [("ei", o0, dict(param=o.ei_eta(o0))), ("pbt", o1, dict(param=0.0)),
                                            ("pbt", o2, dict(param=0.2))], sub)
    got = fn(sub[:, None, :])
    tol = _allowance(dvar, [(om, spec[4]) for (om, _), spec in zip(pairs, specs)], ref)
    assert np.all(np.abs(got - ref) <= tol)


def test_maximize_from_matches_scipy():
    (o0, n0), (o1, n1) = [model_pair(_obj(3 + 2 * i), N, 4, seed=i) for i, N in enumerate((120, 150))]
    eta = o.ei_eta(o0)
    fn = _reduced("product", [_fn("ei", n0, param=eta), _fn("pbt", n1, param=0.0)])
    terms = [("ei", o0, dict(param=eta)), ("pbt", o1, dict(param=0.0))]

    def vg(x):
        v, g, _ = ro.reduction("product", terms, x)
        return v[:, 0], g

    starts = np.random.default_rng(10).uniform(size=(8, 4))
    ok, f, x, _ = fn.maximize_from(starts, 0.0, 1.0)
    ok_s, f_s, x_s, _ = o.scipy_lbfgsb_multistart(vg, starts, 0.0, 1.0)
    np.testing.assert_allclose(f, f_s, rtol=1e-6, atol=1e-10)
    assert ok.all()


def test_member_state_is_unchanged_and_in_place_updates_are_seen():
    (o0, n0), (o1, n1), _ = _pairs("fp64")
    X = candidates(1500, 6, seed=11)
    ei = _fn("ei", n0, param=o.ei_eta(o0))
    pof = _fn("pbt", n1, param=0.0)
    m0, v0 = n0.predict(X)
    e0 = ei(X[:, None, :])
    fn = _reduced("product", [ei, pof])
    first = fn(X[:, None, :])
    m1, v1 = n0.predict(X)
    np.testing.assert_array_equal(m0, m1)
    np.testing.assert_array_equal(v0, v1)
    np.testing.assert_array_equal(e0, ei(X[:, None, :]))
    ei.update(o.ei_eta(o0) - 0.3)  # the child updated in place: the next call sees it
    second = fn(X[:, None, :])
    ref, _, _ = ro.reduction("product", [("ei", o0, dict(param=o.ei_eta(o0) - 0.3)), ("pbt", o1, dict(param=0.0))], X)
    assert not np.allclose(first, second)
    np.testing.assert_allclose(second, ref, rtol=1e-10, atol=1e-13)


def test_c_abi_errors_before_any_launch():
    from trieste_b200 import _lib

    lib = _lib.lib()
    (o0, n0), (o1, n1), _ = _pairs("fp64")
    n32 = _pair32(o.hartmann_6, 50, 6)[1]
    n4 = model_pair(_obj(3), 50, 4)[1]
    n5 = model_pair(o.hartmann_6, 40, 6, seed=5)[1]  # no min-value samples

    def create(models):
        h = C.c_void_p()
        arr = (C.c_void_p * max(1, len(models)))(*[m.handle.value for m in models])
        return lib.tb_reduce_create(C.byref(h), arr, len(models)), h

    def invalid(status):
        assert status == _lib.TB_ERR_INVALID, _lib.last_error()

    lib.tb_launch_count_reset()
    invalid(lib.tb_reduce_create(None, None, 1))
    invalid(create([])[0])
    invalid(create([n0] * 9)[0])
    invalid(create([n0, n0])[0])
    invalid(create([n0, n32])[0])
    invalid(create([n0, n4])[0])
    st, h = create([n0, n1])
    assert st == 0
    ints = lambda *v: np.array(v, dtype=np.int32)  # noqa: E731
    dbl = lambda *v: np.array(v, dtype=np.float64)  # noqa: E731

    def terms(op, member, acq, param, alpha=None):
        a = alpha.ctypes.data if alpha is not None else None
        return lib.tb_reduce_set_terms(h, op, len(member), member.ctypes.data, acq.ctypes.data, param.ctypes.data, a)

    X = candidates(100, 6)
    out = np.empty(100)
    invalid(lib.tb_reduce_eval(h, X.ctypes.data, 100, out.ctypes.data, None))  # terms not set
    invalid(lib.tb_reduce_set_terms(h, 0, 1, None, None, None, None))
    invalid(terms(7, ints(0), ints(0), dbl(0.0)))  # unknown op
    invalid(terms(2, ints(0, 1), ints(0, 4), dbl(0.0, 0.0)))  # softplus over two terms
    invalid(lib.tb_reduce_set_terms(h, 0, 9, ints(*[0] * 9).ctypes.data, ints(*[0] * 9).ctypes.data, dbl(*[0] * 9).ctypes.data, None))
    invalid(terms(0, ints(2), ints(0), dbl(0.0)))  # member index out of range
    invalid(terms(0, ints(-1), ints(0), dbl(0.0)))
    for bad in (_lib.ACQ_GIBBON_QUALITY, _lib.ACQ_GIBBON, _lib.ACQ_EI | _lib.ACQ_PENALIZED, 99, -1):
        invalid(terms(0, ints(0), ints(bad), dbl(0.0)))
    invalid(terms(0, ints(0), ints(_lib.ACQ_FEASIBILITY_BICHON), dbl(0.0), dbl(0.0)))  # alpha <= 0
    invalid(terms(0, ints(0), ints(_lib.ACQ_FEASIBILITY_BICHON), dbl(0.0)))  # no alpha
    invalid(terms(0, ints(0), ints(_lib.ACQ_NEG_LCB), dbl(-1.0)))
    # MES without samples on a fresh model
    st, h5 = create([n5])
    assert st == 0
    assert lib.tb_reduce_set_terms(h5, 0, 1, ints(0).ctypes.data, ints(_lib.ACQ_MES).ctypes.data, dbl(0.0).ctypes.data, None) == 0
    invalid(lib.tb_reduce_eval(h5, X.ctypes.data, 100, out.ctypes.data, None))
    lib.tb_reduce_destroy(h5)
    assert lib.tb_launch_count() == 0
    assert terms(1, ints(0, 1), ints(_lib.ACQ_EI, _lib.ACQ_PBT), dbl(0.0, 0.0)) == 0
    assert lib.tb_reduce_eval(h, X.ctypes.data, 100, out.ctypes.data, None) == 0
    assert lib.tb_launch_count() > 0
    lib.tb_reduce_destroy(h)


def _constrained_setup():
    import trieste_b200 as tb

    D = 2
    space = tb.Box([0.0] * D, [1.0] * D)
    X0 = space.sample(12, seed=0)
    f = lambda x: o.branin(x)  # noqa: E731
    c1 = lambda x: o.random_fourier_objective(x, seed=3)  # noqa: E731
    c2 = lambda x: o.random_fourier_objective(x, seed=5)  # noqa: E731

    def observer(x):
        return {"OBJECTIVE": tb.Dataset(x, f(x)), "C1": tb.Dataset(x, c1(x)), "C2": tb.Dataset(x, c2(x))}

    datasets = observer(X0)
    models = {t: tb.GaussianProcessRegression(tb.build_gpr(ds, space, likelihood_variance=1e-5)) for t, ds in datasets.items()}
    return tb, space, observer, datasets, models


def test_bo_loop_with_a_product_of_ei_and_two_constraints():
    from trieste_b200.acquisition import ExpectedImprovement, Product, ProbabilityOfFeasibility
    from trieste_b200.acquisition.combination import reduced_acquisition
    from trieste_b200.acquisition.interface import AcquisitionFunctionBuilder
    from trieste_b200.bayesian_optimizer import BayesianOptimizer
    from trieste_b200.rule import EfficientGlobalOptimization

    tb, space, observer, datasets, models = _constrained_setup()
    t1, t2 = 0.0, 0.2

    def builder():
        return Product(ExpectedImprovement().using("OBJECTIVE"), ProbabilityOfFeasibility(t1).using("C1"),
                       ProbabilityOfFeasibility(t2).using("C2"))

    class PlainEI(AcquisitionFunctionBuilder):  # the composed route: one child as a plain callable
        def __init__(self):
            self._b = ExpectedImprovement().using("OBJECTIVE")

        def prepare_acquisition_function(self, models, datasets=None):
            return _Plain(self._b.prepare_acquisition_function(models, datasets))

        def update_acquisition_function(self, function, models, datasets=None):
            return _Plain(self._b.prepare_acquisition_function(models, datasets))

    # the first step from the same seeds and starts: the fused route's device L-BFGS and the composed route's host
    # L-BFGS reach points of equal value
    fused_rule = EfficientGlobalOptimization(builder())
    composed_rule = EfficientGlobalOptimization(Product(PlainEI(), ProbabilityOfFeasibility(t1).using("C1"),
                                                        ProbabilityOfFeasibility(t2).using("C2")))
    space._rng = np.random.default_rng(42)
    xf = fused_rule.acquire(space, models, datasets)
    assert isinstance(fused_rule._acquisition_function, reduced_acquisition)
    space._rng = np.random.default_rng(42)
    xc = composed_rule.acquire(space, models, datasets)
    assert not isinstance(composed_rule._acquisition_function, reduced_acquisition)
    fn = fused_rule._acquisition_function
    vf, vc = float(fn(xf[:, None, :])[0, 0]), float(fn(xc[:, None, :])[0, 0])
    assert abs(vf - vc) <= 1e-6 * max(abs(vf), abs(vc)), (vf, vc, xf, xc)
    # ten steps of the loop on the mapping observer
    result = BayesianOptimizer(observer, space).optimize(10, datasets, models, EfficientGlobalOptimization(builder()))
    assert result.error is None, result.error
    assert len(result.history) == 10
    final = result.try_get_final_datasets()
    assert all(len(ds) == 22 for ds in final.values())
