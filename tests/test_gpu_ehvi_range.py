"""Expected hypervolume improvement and HIPPO over the range the device path accepts, beyond the equal-member stacks of
tests/test_gpu_ehvi.py and tests/test_gpu_hippo.py: stacks whose members differ in size, kernel, noise and engine, over
several chunks with a partial last one; fp32 stacks; and the kernel's and driver's edges set through hand-made cells (cell
counts at the tile boundaries, clipped lower bounds, zero-width cells, clipped variances, exact zeros, the argmax across
256-candidate blocks and NaN candidates).

Tolerances are those of tests/test_gpu_ehvi.py (rtol 1e-10 on the stack's own predict outputs, the engines' stated
variance error end to end, gradients at rtol 1e-6 and 1e-7 of their scale).  fp32 stacks: the members' stated fp32 errors,
1e-4 sigma_f^2 in variance and 1e-4 sigma_f in mean, reach a value through its partials (times 10), and gradients are held to
1e-4 of each candidate's gradient scale."""
import numpy as np
import pytest

from oracle import gp_oracle as o
from tests import ehvi_oracle as eo
from tests import hippo_oracle as ho
from tests.test_gpu_ehvi import OBJECTIVES, _allowance, _cells, _kernel_count, _oracle_moments, _stack
from tests.test_gpu_fp32 import _assert_fp32_gradient, _pair32
from tests.util import candidates, model_pair, with_exact_cholesky

pytestmark = pytest.mark.gpu

TILE = 64  # cells per shared-memory tile of the kernel


def _fn(stack, lower, upper):
    from trieste_b200.acquisition import expected_hv_improvement

    return expected_hv_improvement(stack, (lower, upper))


def _penalised(base, stack, pending):
    from trieste_b200.acquisition import hippo_penalized_ehvi, hippo_penalizer

    hp = hippo_penalizer(stack, pending)
    return hp, hippo_penalized_ehvi(base, hp)


# ---- a. members of different sizes, kernels, noise and engines, over several chunks ----
# (N, kernel, noise as a fraction of the kernel variance, engine): below one 128-row block, across blocks, the headline size
UNEQUAL = [(37, "matern12", 1e-2, "int8"), (300, "rbf", 1e-4, "int8x21"), (1500, "matern32", 1e-3, "fp64"),
           (4096, "matern52", 1e-2, "int8")]


@pytest.fixture(scope="module")
def unequal():
    import trieste_b200 as tb

    oms, nms = [], []
    for l, (N, kind, nz, engine) in enumerate(UNEQUAL):
        om0 = o.synthetic_model(OBJECTIVES[l], N, 6, kind=kind)
        om, nm = model_pair(OBJECTIVES[l], N, 6, kind=kind, noise=nz * om0.variance, engine=engine)
        # Matern-12 end to end against the difference-form Gram, as the library builds it
        oms.append(with_exact_cholesky(om) if kind == "matern12" else om)
        nms.append(nm)
    stack = tb.TrainableModelStack(*[(m, 1) for m in nms])
    # the members share their first 37 inputs (one seed), so those rows give a front in objective space (123 cells)
    from trieste_b200.acquisition.multi_objective import (Pareto, get_reference_point,
                                                          prepare_default_non_dominated_partition_bounds)

    front = Pareto(np.concatenate([om.y[:12].reshape(-1, 1) for om in oms], axis=1)).front
    lower, upper = prepare_default_non_dominated_partition_bounds(get_reference_point(front), front)
    return oms, nms, stack, lower, upper


def test_unequal_members_values_argmax_and_penalty_over_chunks(unequal):
    oms, nms, stack, lower, upper = unequal
    engines = [u[3] for u in UNEQUAL]
    fn = _fn(stack, lower, upper)
    M = 160_001  # odd: the last chunk is partial whatever the (tile-aligned) chunk size
    X = candidates(M, 6, seed=31)
    assert _kernel_count(lambda: fn(X[:, None, :]), "ehvi_kernel") >= 3
    got = fn(X[:, None, :])[:, 0]
    # every value: the oracle on the stack's own predict outputs
    m_n, v_n = stack.predict(X)
    ref_own = eo.ehvi(m_n, v_n, lower, upper)
    np.testing.assert_allclose(got, ref_own, rtol=1e-10, atol=1e-13 * np.abs(ref_own).max())
    assert np.any(ref_own > 0)
    # a sample end to end, the chunk ends included
    idx = np.unique(np.concatenate([np.arange(50), np.arange(M - 50, M),
                                    np.random.default_rng(0).choice(M, 400, replace=False)]))
    mean, var = _oracle_moments(oms, X[idx])
    ref = eo.ehvi(mean, var, lower, upper)
    assert np.all(np.abs(got[idx] - ref) <= 1e-9 * np.abs(ref) + _allowance(oms, engines, mean, var, lower, upper))
    # the fused argmax: the first max of the values, over the same chunks
    i, best = fn.fused_argmax(X)
    assert i == o.argmax_first(got) and best == got[i]
    # HIPPO on the same stack and chunks
    hp, pen = _penalised(fn, stack, candidates(TILE + 6, 6, seed=32))
    pv = pen(X[:, None, :])[:, 0]
    ref_pen = ref_own * ho.penalty(m_n, hp._pending_means, hp._pending_vars)  # ho.value, without evaluating EHVI again
    np.testing.assert_allclose(pv, ref_pen, rtol=1e-10, atol=1e-13 * np.abs(ref_own).max())
    i, best = pen.fused_argmax(X)
    assert i == o.argmax_first(pv) and best == pv[i]


@pytest.mark.parametrize("penalised", [False, True])
def test_unequal_members_gradients_over_chunks(unequal, penalised):
    oms, nms, stack, lower, upper = unequal
    fn = _fn(stack, lower, upper)
    pending = candidates(5, 6, seed=33)
    if penalised:
        hp, fn = _penalised(fn, stack, pending)
    M = 110_001
    X = candidates(M, 6, seed=34)
    assert _kernel_count(lambda: fn.value_and_gradient(X[:, None, :]), "ehvi_kernel") >= 3
    vals, grad = fn.value_and_gradient(X[:, None, :])
    assert vals.shape == (M, 1) and grad.shape == (M, 1, 6)
    # the values plan and the gradient plan may group the variance sums differently: rounding only
    np.testing.assert_allclose(vals[:, 0], fn(X[:, None, :])[:, 0], rtol=1e-10, atol=1e-13 * np.abs(vals).max())
    assert np.all(np.isfinite(grad))
    idx = np.unique(np.concatenate([np.arange(40), np.arange(M - 40, M),
                                    np.random.default_rng(1).choice(M, 240, replace=False)]))
    if penalised:
        pm, pv = _oracle_moments(oms, pending)
        ref = ho.gradient(oms, X[idx], lower, upper, pm, pv, o.predict, o.posterior_gradients)
    else:
        ref = eo.ehvi_gradient(oms, X[idx], lower, upper, o.predict, o.posterior_gradients)
    np.testing.assert_allclose(grad[idx, 0, :], ref, rtol=1e-6, atol=1e-7 * np.abs(ref).max())


# ---- b. fp32 stacks ----
FP32_VAR_EPS, FP32_MEAN_EPS = 1e-4, 1e-4


def _stack32(L, engine):
    import trieste_b200 as tb

    pairs = [_pair32(OBJECTIVES[l], 300, 6) for l in range(L)]
    oms, nms = [p[0] for p in pairs], [p[1] for p in pairs]
    if engine is not None:
        for nm in nms:
            nm.set_engine(engine)
    return oms, nms, tb.TrainableModelStack(*[(m, 1) for m in nms])


def _allowance32(oms, dmu, dvar, ref):
    veps = np.array([FP32_VAR_EPS * om.variance for om in oms])
    meps = np.array([FP32_MEAN_EPS * np.sqrt(om.variance) for om in oms])
    return 1e-7 * np.abs(ref) + 1e-12 + 10.0 * (np.abs(dvar) @ veps + np.abs(dmu) @ meps)


@pytest.mark.parametrize("engine", [None, "fp64"], ids=["default", "fp64"])
@pytest.mark.parametrize("L", [2, 3])
def test_fp32_stack(L, engine):
    import torch

    oms, nms, stack = _stack32(L, engine)
    assert all(nm.dtype == np.float32 for nm in nms)
    lower, upper = _cells(oms)
    fn = _fn(stack, lower, upper)
    X = np.concatenate([candidates(3000, 6), oms[0].X[:20]]).astype(np.float32)
    X64 = X.astype(np.float64)
    got = fn(X[:, None, :])
    assert got.dtype == np.float32 and got.shape == (X.shape[0], 1)
    got = got[:, 0].astype(np.float64)
    mean, var = _oracle_moments(oms, X64)
    ref = eo.ehvi(mean, var, lower, upper)
    dmu, dvar = eo.ehvi_partials(mean, var, lower, upper)
    assert np.all(np.abs(got - ref) <= _allowance32(oms, dmu, dvar, ref))
    assert np.any(ref > 0)
    # gradient: 1e-4 of each candidate's gradient scale, where there is one
    vals, grad = fn.value_and_gradient(X[:300, None, :])
    assert vals.dtype == np.float32 and grad.dtype == np.float32
    rg = eo.ehvi_gradient(oms, X64[:300], lower, upper, o.predict, o.posterior_gradients)
    live = np.abs(rg).max(axis=1) > 1e-3 * np.abs(rg).max()
    assert live.sum() >= 50
    _assert_fp32_gradient(grad[:300, 0, :][live], rg[live])
    # the fused argmax writes its best value as a float: the returned value at the winner
    idx, best = fn.fused_argmax(X)
    v32 = fn(X[:, None, :])[:, 0]
    assert v32[idx] == v32.max() and best == float(v32[idx])
    # torch device tensors in and out
    xt = torch.from_numpy(X).cuda()
    out = fn(xt[:, None, :])
    assert out.is_cuda and out.dtype == torch.float32
    np.testing.assert_array_equal(out.cpu().numpy()[:, 0], v32)
    assert fn.fused_argmax(xt) == (idx, best)
    # the device L-BFGS: its values are the function's, and it reaches the oracle's SciPy optimum
    starts = candidates(8, 6, seed=21)
    ok, f, x, _ = fn.maximize_from(starts, 0.0, 1.0)
    assert np.all((x >= 0.0) & (x <= 1.0))
    np.testing.assert_allclose(f, fn(x.astype(np.float32)[:, None, :])[:, 0], rtol=1e-5, atol=1e-6 * np.abs(f).max())

    def vg(xq):
        m, v = _oracle_moments(oms, xq)
        return eo.ehvi(m, v, lower, upper), eo.ehvi_gradient(oms, xq, lower, upper, o.predict, o.posterior_gradients)

    _, f_s, _, _ = o.scipy_lbfgsb_multistart(vg, starts, 0.0, 1.0)
    assert f.max() >= f_s.max() - 1e-3 * abs(f_s.max())
    # HIPPO: values end to end, and the value at a pending point
    pending = candidates(4, 6, seed=40).astype(np.float32)
    hp, pen = _penalised(fn, stack, pending)
    pv = pen(X[:, None, :])
    assert pv.dtype == np.float32
    pm, pvar = _oracle_moments(oms, pending.astype(np.float64))
    ref_pen = ho.value(mean, var, lower, upper, pm, pvar)
    dmu, dvar = ho.partials(mean, var, lower, upper, pm, pvar)
    assert np.all(np.abs(pv[:, 0] - ref_pen) <= _allowance32(oms, dmu, dvar, ref_pen))
    # The pending means were rounded to fp32 by predict, and the kernel compares them with the fp64 means it computes, so
    # the distance d at a pending point is at most that rounding over the standard deviations, and the value at most
    # EHVI (2/pi) d: small, not exactly the reference's 0 (DESIGN a25).
    at = pen(pending[:, None, :])[:, 0].astype(np.float64)
    e_at = fn(pending[:, None, :])[:, 0].astype(np.float64)
    rel = np.abs(hp._pending_means) * 2.0 ** -23 / np.sqrt(hp._pending_vars)
    bound = e_at * (2.0 / np.pi) * np.sqrt(np.sum(rel * rel, axis=1)) * 1.01 + 1e-30
    assert np.all(at >= 0.0) and np.all(at <= bound), (at, bound)


# ---- c. kernel and driver edges through hand-made cells ----
@pytest.fixture(scope="module")
def pair():
    """a two-objective and a three-objective stack on the default engine"""
    return {L: _stack(["int8"] * L) for L in (2, 3)}


def _random_cells(m_n, K, seed):
    """K boxes spread over the candidates' means: some below them, some across, some above"""
    rng = np.random.default_rng(seed)
    lo, hi = m_n.min(0), m_n.max(0)
    span = hi - lo
    lower = lo - 0.3 * span + rng.uniform(size=(K, m_n.shape[1])) * 1.2 * span
    upper = lower + rng.uniform(0.05, 0.5, size=(K, m_n.shape[1])) * span
    return lower, upper


@pytest.mark.parametrize("K", [1, TILE - 1, TILE, TILE + 1, 2 * TILE + 1])
@pytest.mark.parametrize("L", [2, 3])
def test_cell_counts_at_tile_boundaries(pair, L, K):
    oms, nms, stack = pair[L]
    X = candidates(700, 6, seed=5)
    m_n, v_n = stack.predict(X)
    if K == 1:  # the single cell of an empty front
        from trieste_b200.acquisition.multi_objective import prepare_default_non_dominated_partition_bounds

        lower, upper = prepare_default_non_dominated_partition_bounds(m_n.max(0))
    else:
        lower, upper = _random_cells(m_n, K, seed=K)
    assert lower.shape == (K, L)
    fn = _fn(stack, np.zeros((1, L)), np.ones((1, L)))
    fn.update((lower, upper))
    vals, grad = fn.value_and_gradient(X[:, None, :])
    ref_own = eo.ehvi(m_n, v_n, lower, upper)
    np.testing.assert_allclose(vals[:, 0], ref_own, rtol=1e-10, atol=1e-13 * np.abs(ref_own).max())
    np.testing.assert_array_equal(fn(X[:, None, :]), vals)
    ref = eo.ehvi_gradient(oms, X, lower, upper, o.predict, o.posterior_gradients)
    np.testing.assert_allclose(grad[:, 0, :], ref, rtol=1e-6, atol=1e-7 * np.abs(ref).max())
    assert np.any(ref_own > 0)


@pytest.mark.parametrize("penalised", [False, True])
def test_clipped_lower_bounds_and_zero_width_cells(pair, penalised):
    oms, nms, stack = pair[3]
    X = candidates(600, 6, seed=6)
    m_n, v_n = stack.predict(X)
    lower, upper = _random_cells(m_n, 40, seed=6)
    fn = _fn(stack, lower, upper)
    if penalised:
        _, fn = _penalised(fn, stack, candidates(3, 6, seed=7))
    runs = []
    for b in (-1e10, -1e12, -np.inf):  # all clip to the same b = 1e10 in the negated coordinates
        lo = lower.copy()
        lo[::3, 0] = b
        lo[1::5, 2] = b
        lo[7] = b
        fn_base = fn._base if penalised else fn
        fn_base.update((lo, upper))
        runs.append(fn.value_and_gradient(X[:, None, :]))
    for v, g in runs[1:]:
        np.testing.assert_array_equal(v, runs[0][0])
        np.testing.assert_array_equal(g, runs[0][1])
    lo = lower.copy()
    lo[::3, 0] = -1e10
    lo[1::5, 2] = -1e10
    lo[7] = -1e10
    if penalised:
        ref = ho.value(m_n, v_n, lo, upper, fn._penalization._pending_means, fn._penalization._pending_vars)
    else:
        ref = eo.ehvi(m_n, v_n, lo, upper)
    assert np.all(np.isfinite(runs[0][0])) and np.all(np.isfinite(runs[0][1]))
    np.testing.assert_allclose(runs[0][0][:, 0], ref, rtol=1e-10, atol=1e-13 * np.abs(ref).max())
    # zero-width cells add exact zeros, to the value and to the gradient
    zl, zu = lo[:6].copy(), upper[:6].copy()
    zu[np.arange(6), np.arange(6) % 3] = zl[np.arange(6), np.arange(6) % 3]
    both_lo = np.concatenate([zl[:3], lo, zl[3:]])
    both_up = np.concatenate([zu[:3], upper, zu[3:]])
    (fn._base if penalised else fn).update((both_lo, both_up))
    v, g = fn.value_and_gradient(X[:, None, :])
    np.testing.assert_array_equal(v, runs[0][0])
    np.testing.assert_array_equal(g, runs[0][1])


def test_clipped_variances_and_exact_zeros():
    """Candidates near the training points of a member whose posterior variance there is below the 1e-12 clip: its
    d/dvar is 0, as the oracle's with var_clipped, and the gradient stays finite.  A cell edge at each such candidate's
    mean makes d EHVI / d s large there, so a kernel that kept it would be far off.  Then cells far below every candidate's
    means in objective space: EHVI and its gradient exactly 0."""
    import trieste_b200 as tb

    # a member with kernel variance ~1e-9 and noise 1e-7 of it: posterior variances of ~1e-16 at its data
    small = lambda x: 1e-4 * o.hartmann_6(x)
    om0 = o.synthetic_model(small, 300, 6)
    om_a, nm_a = model_pair(small, 300, 6, noise=1e-7 * om0.variance, engine="fp64")
    om_b, nm_b = model_pair(OBJECTIVES[2], 300, 6, engine="fp64")
    oms, stack = [om_a, om_b], tb.TrainableModelStack((nm_a, 1), (nm_b, 1))
    rng = np.random.default_rng(8)
    u = rng.standard_normal((8, 6))
    X = om_a.X[:8] + 1e-3 * u / np.linalg.norm(u, axis=1, keepdims=True)
    raw = o.predict_f(om_a, X)[1][:, 0]
    assert np.all(raw < 1e-12)
    m_n, v_n = stack.predict(X)
    assert np.all(v_n[:, 0] == 1e-12)
    # one cell per candidate, its upper edge in objective 0 at that candidate's mean
    lower = np.stack([m_n[:, 0] - 0.5, np.full(8, m_n[:, 1].min() - 1.0)], axis=1)
    upper = np.stack([m_n[:, 0], np.full(8, m_n[:, 1].max() + 1.0)], axis=1)
    fn = _fn(stack, lower, upper)
    vals, grad = fn.value_and_gradient(X[:, None, :])
    assert np.all(np.isfinite(grad))
    mean, var = _oracle_moments(oms, X)
    clipped = np.stack([o.predict_f(om, X)[1][:, 0] < 1e-12 for om in oms], axis=1)
    dmu, dvar = eo.ehvi_partials(mean, var, lower, upper, var_clipped=clipped)
    ref = np.zeros_like(X)
    for l, om in enumerate(oms):
        gm, gv = o.posterior_gradients(om, X)
        ref += dmu[:, l:l + 1] * gm + dvar[:, l:l + 1] * gv
    # what keeping d/dvar at the clipped member would add
    kept = eo.ehvi_partials(mean, var, lower, upper)[1][:, :1] * o.posterior_gradients(om_a, X)[1]
    assert np.all(np.abs(kept).max(axis=1) > 1e-4 * np.abs(ref).max(axis=1))
    np.testing.assert_allclose(grad[:, 0, :], ref, rtol=1e-6, atol=1e-7 * np.abs(ref).max())
    # far below every candidate's means: exact zeros, with and without the penalty
    Xz = np.concatenate([candidates(500, 6, seed=9), X])
    mz, _ = stack.predict(Xz)
    sd = np.sqrt([om.variance for om in oms])
    up = mz.min(0) - 50.0 * sd - rng.uniform(0.0, 1.0, size=(30, 2)) * sd
    fn.update((up - sd, up))
    _, pen = _penalised(fn, stack, candidates(2, 6, seed=10))
    for f in (fn, pen):
        v, g = f.value_and_gradient(Xz[:, None, :])
        assert np.all(v == 0.0) and np.all(g == 0.0)


@pytest.mark.parametrize("M", [1, 255, 256, 257, 513])
@pytest.mark.parametrize("penalised", [False, True])
def test_argmax_across_blocks(pair, M, penalised):
    oms, nms, stack = pair[2]
    fn = _fn(stack, *_cells(oms))
    if penalised:
        _, fn = _penalised(fn, stack, candidates(4, 6, seed=11))
    X = candidates(M, 6, seed=12 + M)
    vals = fn(X[:, None, :])[:, 0]
    j = o.argmax_first(vals)
    X[[j, M - 1]] = X[[M - 1, j]]  # the maximiser in the last (partial) block
    vals = fn(X[:, None, :])[:, 0]
    assert vals.max() > 0 and np.sum(vals == vals.max()) == 1
    assert fn.fused_argmax(X) == (M - 1, vals[M - 1])
    if M > 1:  # a tie with an earlier block (with the same block for M <= 256): the lower index wins
        t = max(0, M - 1 - 256)
        X[t] = X[M - 1]
        vals = fn(X[:, None, :])[:, 0]
        assert vals[t] == vals[M - 1]
        assert fn.fused_argmax(X) == (t, vals[t])


@pytest.mark.parametrize("penalised", [False, True])
def test_nan_candidates(pair, penalised):
    oms, nms, stack = pair[3]
    fn = _fn(stack, *_cells(oms))
    if penalised:
        _, fn = _penalised(fn, stack, candidates(4, 6, seed=13))
    X = candidates(1000, 6, seed=14)
    clean = fn(X[:, None, :])[:, 0]
    Xn = X.copy()
    Xn[::7, 3] = np.nan
    Xn[0] = np.nan
    j = o.argmax_first(clean)
    Xn[j + 1 if j + 1 < 1000 else j - 1] = np.nan
    bad = np.isnan(Xn).any(axis=1)
    vals = fn(Xn[:, None, :])[:, 0]
    assert np.all(np.isnan(vals[bad]))
    np.testing.assert_array_equal(vals[~bad], clean[~bad])
    win = int(np.flatnonzero(~bad)[np.argmax(clean[~bad])])
    assert fn.fused_argmax(Xn) == (win, clean[win])
    # NaN in every candidate: index 0 and a NaN value
    i, v = fn.fused_argmax(np.full((600, 6), np.nan))
    assert i == 0 and np.isnan(v)
