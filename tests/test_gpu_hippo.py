"""HIPPO's penalised EHVI on the device (csrc/ehvi.cuh with the penalty, tb_ehvi_set_penalty) against the NumPy oracle in
tests/hippo_oracle.py: values on the stack's own predict outputs and end to end on every engine and a mixed stack, with P
pending points from one to more than a shared-memory tile; gradients; the reference's identities; a base function, a
penalised function and a second EHVI on the same members not disturbing one another; the fused argmax over several
chunks; the device L-BFGS against SciPy; the launch budget; the C-ABI errors; and the greedy loop on VLMOP2.

Tolerances are the EHVI tests' (tests/test_gpu_ehvi.py): the engines' stated variance error reaches the value through
d value / d var, and a mean error of 1e-10 sigma_f through d value / d mean, which now includes the penalty's."""
import ctypes as C

import numpy as np
import pytest

from oracle import gp_oracle as o
from tests import ehvi_oracle as eo
from tests import hippo_oracle as ho
from tests.test_gpu_ehvi import ENGINE_VAR_EPS, MIXED8, WIDE, _cells, _kernel_count, _oracle_moments, _stack
from tests.util import candidates

pytestmark = pytest.mark.gpu

CASES = [["int8"] * 2, ["int8x21"] * 2, ["fp64"] * 2, ["int8"] * 3, ["int8x21"] * 3, ["fp64"] * 3, ["int8"] * 4,
         ["fp64"] * 4, ["int8", "fp64", "int8x21"]]
TILE = 64  # pending points per shared-memory tile of the kernel
# five to eight objectives, with one pending point and with more than a tile of them
WIDE_CASES = [(e, P) for e in WIDE + [["int8"] * 8] for P in (1, TILE + 6)]


def _penalised(stack, lower, upper, P, seed=7):
    from trieste_b200.acquisition import expected_hv_improvement, hippo_penalized_ehvi, hippo_penalizer

    base = expected_hv_improvement(stack, (lower, upper))
    hp = hippo_penalizer(stack, candidates(P, 6, seed=seed))
    return base, hp, hippo_penalized_ehvi(base, hp)


def _allowance(oms, engines, mean, var, lower, upper, pmean, pvar):
    dmu, dvar = ho.partials(mean, var, lower, upper, pmean, pvar)
    veps = np.array([ENGINE_VAR_EPS[e] * om.variance for e, om in zip(engines, oms)])
    meps = np.array([1e-10 * np.sqrt(om.variance) for om in oms])
    return 1e-14 + 10.0 * (np.abs(dvar) @ veps + np.abs(dmu) @ meps)


@pytest.mark.parametrize("engines, P", [(e, P) for P in (1, 4, TILE + 6) for e in CASES] + WIDE_CASES,
                         ids=[f"{'-'.join(e)}-{P}" for P in (1, 4, TILE + 6) for e in CASES] +
                             [f"{'-'.join(e)}-{P}" for e, P in WIDE_CASES])
def test_values_match_oracle(engines, P):
    oms, nms, stack = _stack(engines)
    lower, upper = _cells(oms)
    base, hp, fn = _penalised(stack, lower, upper, P)
    X = np.concatenate([candidates(3000, 6), oms[0].X[:20], hp._pending_points[:3] + 1e-3])
    got = fn(X[:, None, :])
    assert got.shape == (X.shape[0], 1)
    got = got[:, 0]
    pmean, pvar = hp._pending_means, hp._pending_vars
    # kernel arithmetic: the oracle on the stack's own predict outputs
    m_n, v_n = stack.predict(X)
    ref_own = ho.value(m_n, v_n, lower, upper, pmean, pvar)
    np.testing.assert_allclose(got, ref_own, rtol=1e-10, atol=1e-13 * np.abs(ref_own).max())
    # end to end: oracle posteriors at the candidates, the engines' stated errors
    mean, var = _oracle_moments(oms, X)
    ref = ho.value(mean, var, lower, upper, pmean, pvar)
    assert np.all(np.abs(got - ref) <= 1e-9 * np.abs(ref) + _allowance(oms, engines, mean, var, lower, upper, pmean, pvar))
    assert np.any(ref > 0)
    assert np.all(got <= base(X[:, None, :])[:, 0])  # the penalty is at most 1


GRAD_CASES = [(e, P) for e in [["int8"] * 2, ["fp64"] * 3, ["int8x21"] * 4, ["int8", "fp64", "int8x21"]]
              for P in (1, 5, TILE + 6)] + WIDE_CASES


@pytest.mark.parametrize("engines, P", GRAD_CASES, ids=[f"{P}-{'-'.join(e)}" for e, P in GRAD_CASES])
def test_gradient_matches_oracle(engines, P):
    oms, nms, stack = _stack(engines)
    lower, upper = _cells(oms)
    base, hp, fn = _penalised(stack, lower, upper, P)
    X = np.concatenate([candidates(300, 6, seed=4), hp._pending_points[:1]])
    vals, grad = fn.value_and_gradient(X[:, None, :])
    assert vals.shape == (301, 1) and grad.shape == (301, 1, 6)
    np.testing.assert_array_equal(vals, fn(X[:, None, :]))
    assert vals[-1, 0] == 0.0 and np.all(np.isfinite(grad))  # at a pending point: 0, with a finite gradient
    ref = ho.gradient(oms, X[:-1], lower, upper, hp._pending_means, hp._pending_vars, o.predict, o.posterior_gradients)
    scale = np.abs(ref).max()
    np.testing.assert_allclose(grad[:-1, 0, :], ref, rtol=1e-6, atol=1e-7 * scale)


def _data(oms):
    import trieste_b200 as tb

    return tb.Dataset(oms[0].X, np.concatenate([om.y.reshape(-1, 1) for om in oms], axis=1))


@pytest.mark.parametrize("engines", [["int8"] * 2, ["int8x21"] * 2, ["fp64"] * 3, ["int8", "fp64", "int8x21"]],
                         ids=lambda c: "-".join(c))
def test_reference_identities(engines):
    from trieste_b200.acquisition import (HIPPO, ExpectedHypervolumeImprovement, expected_hv_improvement,
                                          hippo_penalized_ehvi)
    from trieste_b200.acquisition.interface import OBJECTIVE

    oms, nms, stack = _stack(engines)
    models, datasets = {OBJECTIVE: stack}, {OBJECTIVE: _data(oms)}
    X = candidates(2000, 6, seed=3)
    plain = ExpectedHypervolumeImprovement().prepare_acquisition_function(stack, datasets[OBJECTIVE])(X[:, None, :])
    for pending in (None, np.zeros((0, 6))):
        hippo = HIPPO()
        fn = hippo.prepare_acquisition_function(models, datasets, pending)
        assert type(fn) is expected_hv_improvement
        np.testing.assert_array_equal(fn(X[:, None, :]), plain)
    hippo = HIPPO()
    base = hippo.prepare_acquisition_function(models, datasets)
    pending = X[:1]
    pen = hippo.update_acquisition_function(base, models, datasets, pending, new_optimization_step=False)
    assert type(pen) is hippo_penalized_ehvi and pen._base is base
    v = pen(X[:, None, :])[:, 0]
    assert v[0] == 0.0 and np.all(v <= plain[:, 0]) and np.any(v > 0)
    # the same penalised object across greedy steps and BO steps, the base updated in place
    pending = X[:3]
    assert hippo.update_acquisition_function(pen, models, datasets, pending, new_optimization_step=False) is pen
    assert np.all(pen(pending[:, None, :]) == 0.0)
    assert hippo.update_acquisition_function(pen, models, datasets, X[:2], new_optimization_step=True) is pen
    assert hippo._base_acquisition_function is base
    np.testing.assert_array_equal(hippo.update_acquisition_function(pen, models, datasets, None, False)(X[:, None, :]), plain)
    assert hippo.update_acquisition_function(pen, models, datasets) is base
    with pytest.raises(ValueError, match="rank 2"):
        hippo.update_acquisition_function(pen, models, datasets, X[:2, None, :], new_optimization_step=False)
    # the host penaliser agrees with the kernel's penalty on the same stack
    pen_host = hippo._penalization(X[:50, None, :])[:, 0]
    np.testing.assert_allclose(pen(X[:50, None, :])[:, 0], plain[:50, 0] * pen_host, rtol=1e-12, atol=0)


def test_shared_state_is_never_seen_by_another_function():
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
    base, hp, pen = _penalised(stack, lower, upper, 5)
    other = expected_hv_improvement(stack, (lower[::-1], upper[::-1]))
    calls = {
        "base": lambda: base(X[:, None, :]),
        "pen": lambda: pen(X[:, None, :]),
        "other": lambda: other(X[:, None, :]),
        "pen_vg": lambda: pen.value_and_gradient(X[:200, None, :]),
        "base_vg": lambda: base.value_and_gradient(X[:200, None, :]),
        "pen_argmax": lambda: pen.fused_argmax(X),
        "base_argmax": lambda: base.fused_argmax(X),
        "pen_max": lambda: pen.maximize_from(X[:3], 0.0, 1.0, maxiter=20),
        "base_max": lambda: base.maximize_from(X[:3], 0.0, 1.0, maxiter=20),
    }
    alone = {}
    for k, f in calls.items():  # each first on a fresh pair of functions
        b2, _, p2 = _penalised(stack, lower, upper, 5)
        alone[k] = {"base": lambda: b2(X[:, None, :]), "pen": lambda: p2(X[:, None, :]), "other": calls["other"],
                    "pen_vg": lambda: p2.value_and_gradient(X[:200, None, :]),
                    "base_vg": lambda: b2.value_and_gradient(X[:200, None, :]),
                    "pen_argmax": lambda: p2.fused_argmax(X), "base_argmax": lambda: b2.fused_argmax(X),
                    "pen_max": lambda: p2.maximize_from(X[:3], 0.0, 1.0, maxiter=20),
                    "base_max": lambda: b2.maximize_from(X[:3], 0.0, 1.0, maxiter=20)}[k]()
    order = ["pen", "base", "other", "pen_vg", "base_argmax", "pen_argmax", "base_vg", "pen", "pen_max", "base", "other",
             "base_max", "pen_argmax", "base"]
    def parts(r):
        return [np.asarray(a) for a in r] if isinstance(r, tuple) else [np.asarray(r)]

    for k in order:
        got = parts(calls[k]())
        assert len(got) == len(parts(alone[k]))
        for a, b in zip(got, parts(alone[k])):
            np.testing.assert_array_equal(a, b, err_msg=k)
    assert not np.array_equal(calls["pen"](), calls["base"]())
    for a, b in zip(before, own()):
        np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("engines", [["int8"] * 2, ["fp64"] * 3], ids=lambda c: "-".join(c))
@pytest.mark.parametrize("device_arrays", [False, True])
def test_fused_argmax_is_first_max_of_values(engines, device_arrays):
    oms, nms, stack = _stack(engines)
    lower, upper = _cells(oms)
    # at least five chunks on both stacks (the fp64 members' chunk is 2112 tiles of 128 candidates, 270,336): a kernel count
    # read from the activity trace may miss a record in a long process, so the check below keeps one chunk in hand and takes
    # the larger of two traces
    M = (3 << 19) + 17
    X = candidates(M, 6, seed=9)
    base, hp, fn = _penalised(stack, lower, upper, 4)
    first = o.argmax_first(fn(X[:, None, :])[:, 0])
    assert max(_kernel_count(lambda: fn.fused_argmax(X), "ehvi_kernel") for _ in range(2)) >= 4
    copy = (first + M // 2) % M  # in another chunk: a tie across chunks, which the lower index wins
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


@pytest.mark.parametrize("engines", [["int8"] * 2, ["fp64"] * 3], ids=lambda c: "-".join(c))
def test_device_lbfgs_reaches_scipy_values(engines):
    oms, nms, stack = _stack(engines)
    lower, upper = _cells(oms)
    base, hp, fn = _penalised(stack, lower, upper, 3)
    pmean, pvar = hp._pending_means, hp._pending_vars
    starts = candidates(12, 6, seed=21)
    ok, f, x, nfev = fn.maximize_from(starts, 0.0, 1.0)

    def vg(xq):
        mean, var = _oracle_moments(oms, xq)
        return (ho.value(mean, var, lower, upper, pmean, pvar),
                ho.gradient(oms, xq, lower, upper, pmean, pvar, o.predict, o.posterior_gradients))

    ok_s, f_s, x_s, _ = o.scipy_lbfgsb_multistart(vg, starts, 0.0, 1.0)
    assert np.all((x >= 0.0) & (x <= 1.0))
    np.testing.assert_allclose(f, fn(x[:, None, :])[:, 0], rtol=1e-12)
    both = ok & ok_s & (np.abs(x - x_s).max(axis=1) < 1e-3)
    assert both.sum() >= 3
    np.testing.assert_allclose(f[both], f_s[both], rtol=1e-5, atol=1e-9 * np.abs(f_s).max())
    assert f.max() >= f_s.max() - 1e-5 * abs(f_s.max())


def test_launch_budget_and_unchanged_push():
    from torch.profiler import ProfilerActivity, profile

    from trieste_b200 import _lib

    oms, nms, stack = _stack(["int8"] * 3)
    lower, upper = _cells(oms)
    X = candidates((1 << 20) + 17, 6, seed=3)
    base, hp, fn = _penalised(stack, lower, upper, TILE + 6)
    lib = _lib.lib()
    for f in (fn, base):  # lazy builds happen once
        f.fused_argmax(X)
        f.value_and_gradient(X[:5000, None, :])

    def count(f):
        c0 = lib.tb_launch_count()
        f()
        return lib.tb_launch_count() - c0

    assert count(lambda: fn.fused_argmax(X)) == count(lambda: base.fused_argmax(X))
    assert count(lambda: fn.value_and_gradient(X[:5000, None, :])) == count(lambda: base.value_and_gradient(X[:5000, None, :]))

    def copies(f):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            f()
        return sum(e.count for e in prof.key_averages() if "memcpy" in e.key.lower())

    Xs = X[:1000, None, :]
    assert copies(lambda: fn(Xs)) >= 1  # the trace sees copies: a host-array call stages its input and output
    fn._before_call()
    # the state the handle already holds: no copy, no launch
    assert copies(fn._before_call) == 0 and count(fn._before_call) == 0
    # a new state reaches the device: the next call after an update is the new penalised function
    hp.update(candidates(3, 6, seed=30))
    m_n, v_n = stack.predict(Xs[:, 0])
    np.testing.assert_allclose(fn(Xs)[:, 0], ho.value(m_n, v_n, lower, upper, hp._pending_means, hp._pending_vars),
                               rtol=1e-10, atol=1e-13 * np.abs(base(Xs)).max())


def test_abi_errors():
    import torch

    from trieste_b200 import _lib

    lib = _lib.lib()
    oms, nms, stack = _stack(["int8"] * 2)
    lower, upper = _cells(oms)
    base, hp, fn = _penalised(stack, lower, upper, 3)
    h = base._h
    mean, var = hp._pending_means.copy(), hp._pending_vars.copy()
    INVALID = _lib.TB_ERR_INVALID
    assert lib.tb_ehvi_set_penalty(None, mean.ctypes.data, var.ctypes.data, 3) == INVALID
    assert lib.tb_ehvi_set_penalty(h, mean.ctypes.data, var.ctypes.data, -1) == INVALID
    assert lib.tb_ehvi_set_penalty(h, None, var.ctypes.data, 3) == INVALID
    assert lib.tb_ehvi_set_penalty(h, mean.ctypes.data, None, 3) == INVALID
    for bad in (-1e-3, np.nan):
        v = var.copy()
        v[1, 1] = bad
        assert lib.tb_ehvi_set_penalty(h, mean.ctypes.data, v.ctypes.data, 3) == INVALID
        assert "variance" in _lib.last_error()
    assert lib.tb_ehvi_set_penalty(h, None, None, 0) == 0
    X = candidates(500, 6, seed=8)
    out = np.empty(500)
    _lib.check(lib.tb_ehvi_eval(h, X.ctypes.data, 500, out.ctypes.data, None))
    np.testing.assert_array_equal(out, base(X[:, None, :])[:, 0])  # P = 0: no penalty
    # device arrays give the host arrays' result
    dm, dv = torch.from_numpy(mean).cuda(), torch.from_numpy(var).cuda()
    assert lib.tb_ehvi_set_penalty(h, dm.data_ptr(), dv.data_ptr(), 3) == 0
    _lib.check(lib.tb_ehvi_eval(h, X.ctypes.data, 500, out.ctypes.data, None))
    np.testing.assert_array_equal(out, fn(X[:, None, :])[:, 0])
    # the Python layer
    from trieste_b200.acquisition import hippo_penalized_ehvi, hippo_penalizer

    with pytest.raises(ValueError, match="expected_hv_improvement"):
        hippo_penalized_ehvi(object(), hp)
    with pytest.raises(ValueError, match="hippo_penalizer"):
        hippo_penalized_ehvi(base, object())
    with pytest.raises(ValueError, match="batch sizes of one"):
        fn(X[:4].reshape(2, 2, 6))
    one = hippo_penalizer(nms[0], X[:2])  # one output against a stack of two
    with pytest.raises(ValueError, match="outputs"):
        hippo_penalized_ehvi(base, one)(X[:4, None, :])


def _vlmop2_setup(n0=10):
    import trieste_b200 as tb
    from trieste_b200.objectives import vlmop2

    D = 2
    space = tb.Box([-2.0] * D, [2.0] * D)
    X0 = space.sample(n0, seed=0)
    Y0 = vlmop2(X0, D)
    specs = [tb.build_gpr(tb.Dataset(X0, Y0[:, l:l + 1]), space, likelihood_variance=1e-7) for l in range(2)]
    members = [tb.GaussianProcessRegression(s) for s in specs]
    return space, X0, Y0, specs, members, tb.TrainableModelStack(*[(m, 1) for m in members])


def test_greedy_loop_picks_the_oracle_points_step_by_step():
    import trieste_b200 as tb
    from trieste_b200.acquisition import HIPPO, hippo_penalized_ehvi
    from trieste_b200.acquisition.multi_objective import (Pareto, get_reference_point,
                                                          prepare_default_non_dominated_partition_bounds)
    from trieste_b200.acquisition.optimizer import _get_max_discrete_points
    from trieste_b200.bayesian_optimizer import BayesianOptimizer
    from trieste_b200.objectives import vlmop2
    from trieste_b200.rule import EfficientGlobalOptimization

    D = 2
    space, X0, Y0, specs, members, stack = _vlmop2_setup()
    steps = {"n": 0, "checked": 0, "penalised": 0}

    def optimizer(search_space, fn):
        cand = search_space.sample(2000, seed=500 + steps["n"])
        steps["n"] += 1
        picked = _get_max_discrete_points(cand[:, None, :], fn)
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
        if isinstance(fn, hippo_penalized_ehvi):
            steps["penalised"] += 1
            pmean, pvar = _oracle_moments(oms, fn._penalization._pending_points)
            vals = ho.value(mean, var, lower, upper, pmean, pvar)
        else:
            vals = eo.ehvi(mean, var, lower, upper)
        top = np.sort(vals)[-2:]
        if top[1] - top[0] > 1e-6 * max(abs(top[1]), 1e-12):
            np.testing.assert_array_equal(picked, cand[o.argmax_first(vals)][None])
            steps["checked"] += 1
        return picked

    rule = EfficientGlobalOptimization(HIPPO(), optimizer=optimizer, num_query_points=4)
    BayesianOptimizer(lambda x: vlmop2(x, D), space).optimize(3, tb.Dataset(X0, Y0), stack, rule)
    assert steps["n"] == 12 and steps["penalised"] == 9 and steps["checked"] >= 8


def test_bo_loop_on_vlmop2_with_the_continuous_optimiser():
    import trieste_b200 as tb
    from trieste_b200.acquisition import HIPPO
    from trieste_b200.acquisition.multi_objective import Pareto
    from trieste_b200.bayesian_optimizer import BayesianOptimizer
    from trieste_b200.objectives import vlmop2, vlmop2_pareto_optimal_points
    from trieste_b200.rule import EfficientGlobalOptimization

    D = 2
    space, X0, Y0, specs, members, stack = _vlmop2_setup()
    rule = EfficientGlobalOptimization(HIPPO(), num_query_points=4)
    result = BayesianOptimizer(lambda x: vlmop2(x, D), space).optimize(5, tb.Dataset(X0, Y0), stack, rule)
    data = result.try_get_final_dataset()
    Xf, final = np.asarray(data.query_points), np.asarray(data.observations)
    assert Xf.shape == (10 + 5 * 4, D)
    for b in range(5):
        batch = Xf[10 + 4 * b: 14 + 4 * b]
        assert len({tuple(r) for r in batch}) == 4, batch
        assert np.min([np.abs(batch[i] - batch[j]).max() for i in range(4) for j in range(i)]) > 1e-6, batch
    ideal = vlmop2_pareto_optimal_points(200, D)
    ref_pt = np.array([1.2, 1.2])
    hv_ideal = Pareto(ideal).hypervolume_indicator(ref_pt)
    gap0 = hv_ideal - Pareto(Y0).hypervolume_indicator(ref_pt)
    gap = hv_ideal - Pareto(final).hypervolume_indicator(ref_pt)
    assert gap < gap0
