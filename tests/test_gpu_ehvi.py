"""Expected hypervolume improvement on the device (csrc/ehvi.cuh, tb_ehvi_*) against the NumPy oracle in
tests/ehvi_oracle.py: kernel arithmetic on the stack's own predict outputs, end to end against oracle posteriors on every
engine and a mixed-engine stack, gradients, the fused argmax over several chunks, the device L-BFGS against SciPy, member
handles left untouched, the launch count, the C-ABI errors and a BO loop on VLMOP2.

Tolerances.  The members' variances carry the engine's stated error eps sigma_f^2 (fp64 1e-12, int8 engines 1e-9), which
reaches EHVI through d EHVI / d var_l; the allowance is that product from the oracle, summed over objectives, times 10."""
import ctypes as C

import numpy as np
import pytest

from oracle import gp_oracle as o
from tests import ehvi_oracle as eo
from tests.util import candidates, model_pair

pytestmark = pytest.mark.gpu

ENGINE_VAR_EPS = {"int8": 1e-9, "int8x21": 1e-9, "fp64": 1e-12}
OBJECTIVES = [
    o.hartmann_6,
    lambda x: o.ackley(x).reshape(-1, 1),
    lambda x: o.random_fourier_objective(x, seed=3),
    lambda x: o.random_fourier_objective(x, seed=5),
    lambda x: o.random_fourier_objective(x, seed=7),
    lambda x: o.random_fourier_objective(x, seed=11),
    lambda x: o.random_fourier_objective(x, seed=13),
    lambda x: o.random_fourier_objective(x, seed=17),
]


def _stack(engines, N=300, D=6):
    import trieste_b200 as tb

    pairs = [model_pair(OBJECTIVES[l], N, D, seed=0, engine=e) for l, e in enumerate(engines)]
    oms, nms = [p[0] for p in pairs], [p[1] for p in pairs]
    return oms, nms, tb.TrainableModelStack(*[(m, 1) for m in nms])


def _cells(oms):
    from trieste_b200.acquisition.multi_objective import (Pareto, get_reference_point,
                                                          prepare_default_non_dominated_partition_bounds)

    # a front of tens to hundreds of cells; from five objectives on the cell count grows steeply with the front, so four
    # points give a few hundred to a few thousand
    Y = np.concatenate([om.y.reshape(-1, 1) for om in oms], axis=1)[:40 if len(oms) <= 4 else 4]
    front = Pareto(Y).front
    return prepare_default_non_dominated_partition_bounds(get_reference_point(front), front)


def _oracle_moments(oms, X):
    means, vars_ = zip(*(o.predict(om, X) for om in oms))
    return np.concatenate(means, axis=1), np.concatenate(vars_, axis=1)


def _allowance(oms, engines, mean, var, lower, upper):
    _, dvar = eo.ehvi_partials(mean, var, lower, upper)
    eps = np.array([ENGINE_VAR_EPS[e] * om.variance for e, om in zip(engines, oms)])
    return 1e-14 + 10.0 * np.abs(dvar) @ eps


MIXED8 = ["int8", "fp64", "int8x21"] * 2 + ["int8", "fp64"]
CASES = [["int8"] * 2, ["int8x21"] * 2, ["fp64"] * 2, ["int8"] * 3, ["int8x21"] * 3, ["fp64"] * 3, ["int8"] * 4,
         ["fp64"] * 4, ["int8", "fp64", "int8x21"], ["int8"] * 5, ["fp64"] * 6, ["int8x21"] * 7, ["int8"] * 8, ["fp64"] * 8,
         MIXED8]
# one stack per objective count from five to eight, for the paths that run every kernel instantiation
WIDE = [["int8"] * 5, ["fp64"] * 6, ["int8x21"] * 7, MIXED8]


@pytest.mark.parametrize("engines", CASES, ids=["-".join(c) for c in CASES])
def test_values_match_oracle(engines):
    from trieste_b200.acquisition import expected_hv_improvement

    oms, nms, stack = _stack(engines)
    lower, upper = _cells(oms)
    X = np.concatenate([candidates(3000, 6), oms[0].X[:20]])
    fn = expected_hv_improvement(stack, (lower, upper))
    got = fn(X[:, None, :])
    assert got.shape == (X.shape[0], 1)
    got = got[:, 0]
    # kernel arithmetic: the oracle EHVI on the stack's own predict outputs
    m_n, v_n = stack.predict(X)
    ref_own = eo.ehvi(m_n, v_n, lower, upper)
    np.testing.assert_allclose(got, ref_own, rtol=1e-10, atol=1e-13 * np.abs(ref_own).max())
    # end to end: oracle posteriors and the engines' stated variance error
    mean, var = _oracle_moments(oms, X)
    ref = eo.ehvi(mean, var, lower, upper)
    assert np.all(np.abs(got - ref) <= 1e-9 * np.abs(ref) + _allowance(oms, engines, mean, var, lower, upper))
    assert np.any(ref > 0)


@pytest.mark.parametrize("engines", [["int8"] * 2, ["fp64"] * 3, ["int8x21"] * 4, ["int8", "fp64", "int8x21"]] + WIDE,
                         ids=lambda c: "-".join(c))
def test_gradient_matches_oracle(engines):
    from trieste_b200.acquisition import expected_hv_improvement

    oms, nms, stack = _stack(engines)
    lower, upper = _cells(oms)
    X = candidates(300, 6, seed=4)
    fn = expected_hv_improvement(stack, (lower, upper))
    vals, grad = fn.value_and_gradient(X[:, None, :])
    assert vals.shape == (300, 1) and grad.shape == (300, 1, 6)
    np.testing.assert_array_equal(vals, fn(X[:, None, :]))
    ref = eo.ehvi_gradient(oms, X, lower, upper, o.predict, o.posterior_gradients)
    scale = np.abs(ref).max()
    np.testing.assert_allclose(grad[:, 0, :], ref, rtol=1e-6, atol=1e-7 * scale)


@pytest.mark.parametrize("engines", [["int8"] * 2, ["fp64"] * 3, ["int8"] * 5, MIXED8], ids=lambda c: "-".join(c))
@pytest.mark.parametrize("device_arrays", [False, True])
def test_fused_argmax_is_first_max_of_values(engines, device_arrays):
    from trieste_b200.acquisition import expected_hv_improvement

    oms, nms, stack = _stack(engines)
    lower, upper = _cells(oms)
    M = (1 << 20) + 17
    X = candidates(M, 6, seed=9)
    fn = expected_hv_improvement(stack, (lower, upper))
    first = o.argmax_first(fn(X[:, None, :])[:, 0])
    # a copy of the true maximiser M/2 candidates away, so in another chunk when the call has at least four (each full chunk
    # then holds fewer than M/3): a tie across chunks, which the lower index wins
    assert _kernel_count(lambda: fn.fused_argmax(X), "ehvi_kernel") >= 4
    copy = (first + M // 2) % M
    X[copy] = X[first]
    if device_arrays:
        import torch

        X = torch.from_numpy(X).cuda()
    vals = fn(X[:, None, :])
    idx, best = fn.fused_argmax(X)
    vals = vals.cpu().numpy()[:, 0] if device_arrays else vals[:, 0]
    assert vals[copy] == vals[first]
    assert idx == o.argmax_first(vals) == min(first, copy)
    assert best == vals[idx]


@pytest.mark.parametrize("engines", [["int8"] * 2, ["fp64"] * 3, ["int8"] * 5, MIXED8], ids=lambda c: "-".join(c))
def test_device_lbfgs_reaches_scipy_values(engines):
    from trieste_b200.acquisition import expected_hv_improvement

    oms, nms, stack = _stack(engines)
    lower, upper = _cells(oms)
    fn = expected_hv_improvement(stack, (lower, upper))
    starts = candidates(12, 6, seed=21)
    ok, f, x, nfev = fn.maximize_from(starts, 0.0, 1.0)

    def vg(xq):
        mean, var = _oracle_moments(oms, xq)
        return eo.ehvi(mean, var, lower, upper), eo.ehvi_gradient(oms, xq, lower, upper, o.predict, o.posterior_gradients)

    ok_s, f_s, x_s, _ = o.scipy_lbfgsb_multistart(vg, starts, 0.0, 1.0)
    assert np.all((x >= 0.0) & (x <= 1.0))
    np.testing.assert_allclose(f, fn(x[:, None, :])[:, 0], rtol=1e-12)
    both = ok & ok_s & (np.abs(x - x_s).max(axis=1) < 1e-3)
    assert both.sum() >= 3
    np.testing.assert_allclose(f[both], f_s[both], rtol=1e-5, atol=1e-9 * np.abs(f_s).max())
    assert f.max() >= f_s.max() - 1e-5 * abs(f_s.max())


def test_member_handles_untouched():
    from trieste_b200 import _lib
    from trieste_b200.acquisition import expected_hv_improvement

    oms, nms, stack = _stack(["int8", "fp64", "int8x21"])
    lower, upper = _cells(oms)
    X = candidates(5000, 6, seed=2)

    def own():
        out = []
        for nm in nms:
            m, v = nm.predict(X)
            ei = np.empty(X.shape[0])
            _lib.check(_lib.lib().tb_acq_eval(nm.handle, _lib.ACQ_EI, 0.1, X.ctypes.data, X.shape[0], ei.ctypes.data, None))
            out += [m, v, ei]
        return out

    before = own()
    fn = expected_hv_improvement(stack, (lower, upper))
    fn(X[:, None, :])
    fn.value_and_gradient(X[:100, None, :])
    fn.fused_argmax(X)
    for a, b in zip(before, own()):
        np.testing.assert_array_equal(a, b)


def test_launch_budget_of_the_argmax():
    from trieste_b200 import _lib
    from trieste_b200.acquisition import expected_hv_improvement

    oms, nms, stack = _stack(["int8"] * 3)
    lower, upper = _cells(oms)
    X = candidates((1 << 20) + 17, 6, seed=3)
    fn = expected_hv_improvement(stack, (lower, upper))
    lib = _lib.lib()
    fn.fused_argmax(X)  # lazy builds happen once
    for nm in nms:
        nm.predict(X[:10])

    def count(f):
        c0 = lib.tb_launch_count()
        f()
        return lib.tb_launch_count() - c0

    n = count(lambda: fn.fused_argmax(X))
    members = [count(lambda nm=nm: nm.predict(X)) for nm in nms]
    chunks = _kernel_count(lambda: fn.fused_argmax(X), "ehvi_kernel")
    tails = [_kernel_count(lambda nm=nm: nm.predict(X), "tail_kernel") for nm in nms]
    assert chunks >= 2 and tails == [chunks] * len(nms)  # one chunk plan for the stack and for each member alone
    # each member's predict: its K* and variance launches plus one tail per chunk; the EHVI argmax: the same K* and variance
    # launches, one EHVI kernel and one fold per chunk, and a constant
    assert n <= sum(members) - sum(tails) + 2 * chunks + 4, (n, members, chunks)


def _kernel_count(f, name):
    """launches of kernels whose name contains ``name`` during f(), from the CUDA activity trace"""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        f()
    return sum(e.count for e in prof.key_averages() if name in e.key)


def test_abi_errors():
    import trieste_b200 as tb
    from trieste_b200 import _lib
    from trieste_b200.acquisition import expected_hv_improvement

    lib = _lib.lib()
    oms, nms, stack = _stack(["int8"] * 3)
    hs = [m.handle.value for m in nms]

    def create(handles):
        h = C.c_void_p()
        arr = (C.c_void_p * len(handles))(*handles)
        return lib.tb_ehvi_create(C.byref(h), arr, len(handles)), h

    assert create(hs[:1])[0] == _lib.TB_ERR_INVALID
    assert create(hs * 3)[0] == _lib.TB_ERR_INVALID  # L = 9, and duplicates
    assert create([hs[0], hs[0]])[0] == _lib.TB_ERR_INVALID
    assert create([hs[0], None])[0] == _lib.TB_ERR_INVALID
    assert lib.tb_ehvi_create(None, None, 2) == _lib.TB_ERR_INVALID
    om5, nm5 = model_pair(o.ackley, 100, 5)
    assert create([hs[0], nm5.handle.value])[0] == _lib.TB_ERR_INVALID  # input dimension
    om32 = o.synthetic_model(OBJECTIVES[1], 100, 6, dtype=np.float32)
    from tests.util import native_from_oracle

    nm32 = native_from_oracle(om32)
    assert create([hs[0], nm32.handle.value])[0] == _lib.TB_ERR_INVALID  # dtype
    status, h = create(hs[:2])
    assert status == 0
    X = candidates(10, 6)
    out = np.empty(10)
    assert lib.tb_ehvi_eval(h, X.ctypes.data, 10, out.ctypes.data, None) == _lib.TB_ERR_INVALID  # cells not set
    lo, up = np.zeros((1, 2)), np.ones((1, 2))
    assert lib.tb_ehvi_set_cells(h, lo.ctypes.data, up.ctypes.data, 0) == _lib.TB_ERR_INVALID
    assert lib.tb_ehvi_set_cells(h, None, up.ctypes.data, 1) == _lib.TB_ERR_INVALID
    assert lib.tb_ehvi_set_cells(h, lo.ctypes.data, up.ctypes.data, 1) == 0
    assert lib.tb_ehvi_eval(h, None, 10, out.ctypes.data, None) == _lib.TB_ERR_INVALID
    best, idx = C.c_double(), C.c_int64()
    assert lib.tb_ehvi_argmax(h, X.ctypes.data, 0, None, C.byref(best), C.byref(idx)) == _lib.TB_ERR_INVALID
    assert lib.tb_ehvi_maximize(h, None, None, None, 0, 10, 10, 10, 1e-5, 1e-9, None, None, None, None) == _lib.TB_ERR_INVALID
    # a member whose posterior cache is not built
    raw = C.c_void_p()
    _lib.check(lib.tb_gp_create(C.byref(raw), 0, _lib.TB_F64))
    om = oms[0]
    y = np.ascontiguousarray(om.y[:, 0])
    _lib.check(lib.tb_gp_set_data(raw, om.X.ctypes.data, y.ctypes.data, om.X.shape[0], 6))
    ls = np.ascontiguousarray(om.lengthscales)
    _lib.check(lib.tb_gp_set_hyper(raw, _lib.KERNEL_IDS["matern52"], om.variance, ls.ctypes.data_as(C.POINTER(C.c_double)), 6,
                                   om.noise, om.mean_const))
    status, h2 = create([hs[0], raw.value])
    assert status == 0
    assert lib.tb_ehvi_set_cells(h2, lo.ctypes.data, up.ctypes.data, 1) == 0
    assert lib.tb_ehvi_eval(h2, X.ctypes.data, 10, out.ctypes.data, None) == _lib.TB_ERR_INVALID
    assert "posterior cache" in _lib.last_error()
    lib.tb_ehvi_destroy(h2)
    lib.tb_ehvi_destroy(h)
    lib.tb_gp_destroy(raw)
    # the Python layer: non-native or multi-output members, and batch sizes other than one
    with pytest.raises(ValueError):
        expected_hv_improvement(tb.ModelStack((nms[0], 1), (nms[1], 2)), (lo, up))
    with pytest.raises(ValueError):
        expected_hv_improvement(tb.ModelStack((nms[0], 1), (nms[0], 1)), (lo, up))
    fn = expected_hv_improvement(tb.ModelStack((nms[0], 1), (nms[1], 1)), (lo, up))
    with pytest.raises(ValueError, match="batch sizes of one"):
        fn(X[:4].reshape(2, 2, 6))


def test_bo_loop_on_vlmop2_follows_the_oracle():
    import trieste_b200 as tb
    from trieste_b200.acquisition import ExpectedHypervolumeImprovement
    from trieste_b200.acquisition.multi_objective import (Pareto, get_reference_point,
                                                          prepare_default_non_dominated_partition_bounds)
    from trieste_b200.acquisition.optimizer import _get_max_discrete_points
    from trieste_b200.bayesian_optimizer import BayesianOptimizer
    from trieste_b200.objectives import vlmop2, vlmop2_pareto_optimal_points
    from trieste_b200.rule import EfficientGlobalOptimization

    D = 2
    space = tb.Box([-2.0] * D, [2.0] * D)
    X0 = space.sample(10, seed=0)
    Y0 = vlmop2(X0, D)
    specs = [tb.build_gpr(tb.Dataset(X0, Y0[:, l:l + 1]), space, likelihood_variance=1e-7) for l in range(2)]
    members = [tb.GaussianProcessRegression(s) for s in specs]
    stack = tb.TrainableModelStack(*[(m, 1) for m in members])
    steps = {"n": 0, "checked": 0}

    def optimizer(search_space, fn):
        cand = search_space.sample(2000, seed=500 + steps["n"])
        steps["n"] += 1
        picked = _get_max_discrete_points(cand[:, None, :], fn)
        # the oracle on the members' current data and the same hyper-parameters
        oms = []
        for m, s in zip(members, specs):
            d = m.get_internal_data()
            k = s.kernel
            oms.append(o.build_model("matern52", np.asarray(d.query_points), np.asarray(d.observations), k.variance,
                                     np.asarray(k.lengthscales, dtype=np.float64), s.noise_variance, s.mean_function.c))
        Xd = np.asarray(members[0].get_internal_data().query_points)
        mean_d, _ = _oracle_moments(oms, Xd)
        ref_pt = get_reference_point(mean_d)
        front = Pareto(mean_d).front
        front = front[np.all(front <= ref_pt, axis=-1)]
        lower, upper = prepare_default_non_dominated_partition_bounds(ref_pt, front)
        mean, var = _oracle_moments(oms, cand)
        vals = eo.ehvi(mean, var, lower, upper)
        top = np.sort(vals)[-2:]
        if top[1] - top[0] > 1e-6 * max(abs(top[1]), 1e-12):
            np.testing.assert_array_equal(picked, cand[o.argmax_first(vals)][None])
            steps["checked"] += 1
        return picked

    rule = EfficientGlobalOptimization(ExpectedHypervolumeImprovement(), optimizer=optimizer)
    result = BayesianOptimizer(lambda x: vlmop2(x, D), space).optimize(10, tb.Dataset(X0, Y0), stack, rule)
    final = np.asarray(result.try_get_final_dataset().observations)
    assert steps["n"] == 10 and steps["checked"] >= 5
    ideal = vlmop2_pareto_optimal_points(200, D)
    ref_pt = np.array([1.2, 1.2])
    hv_ideal = Pareto(ideal).hypervolume_indicator(ref_pt)
    gap0 = hv_ideal - Pareto(Y0).hypervolume_indicator(ref_pt)
    gap = hv_ideal - Pareto(final).hypervolume_indicator(ref_pt)
    assert gap < gap0
