"""LocalPenalization (greedy_batch.py:54-388) on the device against the NumPy restatement in tests/lp_oracle.py: the mean
gradient, penalised values / gradients / argmax on every engine, handle isolation, the builder, device L-BFGS and the
greedy BO loop."""
import numpy as np
import pytest

from oracle import gp_oracle as o
from tests import lp_oracle as lp
from tests.util import candidates, model_pair

pytestmark = pytest.mark.gpu

KINDS = {lp.SOFT: "soft_local_penalizer", lp.HARD: "hard_local_penalizer"}


def _penalizer_cls(kind):
    from trieste_b200 import acquisition as acq

    return getattr(acq, KINDS[kind])


def _lp_state(om, P, seed=3):
    """Lipschitz constant and eta over 500 samples plus the data, P pending points and their radius / scale (oracle)."""
    L, eta = lp.lipschitz_and_eta(om, np.concatenate([om.X, candidates(500, om.X.shape[1], seed=seed)]))
    pending = candidates(P, om.X.shape[1], seed=seed + 1)
    radius, scale = lp.penalizer_state(om, pending, L, eta)
    return L, eta, pending, radius, scale


def _query_set(pending, radius, M=3000, seed=1):
    """Random candidates, the pending points themselves and points at distance radius_j from them."""
    D = pending.shape[1]
    u = np.random.default_rng(seed + 10).normal(size=pending.shape)
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    ring = pending + np.abs(radius)[:, None] * u
    return np.concatenate([candidates(M, D, seed=seed), pending, ring])


def _check_values(got, ref, rtol, base_atol=None):
    """rtol above 1e-12, atol 1e-15 below.  base_atol [M]: an absolute allowance per value instead, for a base whose own
    small values carry absolute rather than relative error (MES: the oracle test's atol 1e-12, times the penalty)."""
    got, ref = np.asarray(got, dtype=np.float64).reshape(-1), np.asarray(ref, dtype=np.float64).reshape(-1)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    ok = ~np.isnan(ref)
    if base_atol is not None:
        err = np.abs(got[ok] - ref[ok])
        bound = rtol * np.abs(ref[ok]) + base_atol[ok] + 1e-15
        assert np.all(err <= bound), (err - bound).max()
        return
    big = ok & (np.abs(ref) >= 1e-12)
    np.testing.assert_allclose(got[big], ref[big], rtol=rtol, atol=0)
    small = ok & ~big
    np.testing.assert_allclose(got[small], ref[small], rtol=0, atol=1e-15)


def test_mean_gradient_matches_oracle_in_one_launch():
    from trieste_b200 import _lib

    om, nm = model_pair(o.hartmann_6, 300, 6)
    X = candidates(4000, 6, seed=2)
    _lib.lib().tb_launch_count_reset()
    c0 = _lib.lib().tb_launch_count()
    mean, grad = nm.mean_gradient(X)
    assert _lib.lib().tb_launch_count() - c0 == 1
    omean, _ = o.predict(om, X)
    odmean, _ = o.posterior_gradients(om, X)
    assert mean.shape == (4000, 1) and grad.shape == (4000, 6)
    np.testing.assert_allclose(mean, omean, rtol=1e-9, atol=1e-12 * np.abs(omean).max())
    np.testing.assert_allclose(grad, odmean, rtol=1e-8, atol=1e-11 * np.abs(odmean).max())
    # leading dimensions and the training points themselves
    m2, g2 = nm.mean_gradient(om.X[:10].reshape(2, 5, 6))
    assert m2.shape == (2, 5, 1) and g2.shape == (2, 5, 6)
    np.testing.assert_allclose(g2.reshape(10, 6), o.posterior_gradients(om, om.X[:10])[0], rtol=1e-8,
                               atol=1e-11 * np.abs(odmean).max())


@pytest.mark.parametrize("engine", ["int8", "int8x21", "fp64"])
@pytest.mark.parametrize("P", [1, 7, 200])
@pytest.mark.parametrize("base", ["ei", "mes"])
@pytest.mark.parametrize("kind", [lp.SOFT, lp.HARD])
def test_penalised_values_match_oracle(kind, base, P, engine):
    from trieste_b200.acquisition import PenalizedAcquisition, expected_improvement, min_value_entropy_search

    om, nm = model_pair(o.hartmann_6, 300, 6, engine=engine)
    L, eta, pending, radius, scale = _lp_state(om, P)
    Xq = _query_set(pending, radius)
    omean, ovar = o.predict(om, Xq)
    if base == "ei":
        ei_eta = o.ei_eta(om)
        fn_base = expected_improvement(nm, ei_eta)
        ref_base = o.expected_improvement(omean, ovar, ei_eta)[:, 0]
    else:
        samples = om.y.min() + np.array([[-0.1], [-0.5], [0.05]]) * np.sqrt(om.variance)
        fn_base = min_value_entropy_search(nm, samples)
        ref_base = o.min_value_entropy_search(omean, ovar, samples)[:, 0]
    pen = _penalizer_cls(kind)(nm, pending, L, eta)
    np.testing.assert_allclose(pen.radius, radius, rtol=1e-8, atol=1e-12 * np.abs(radius).max())
    np.testing.assert_allclose(pen.scale, scale, rtol=1e-6)
    fn = PenalizedAcquisition(fn_base, pen)
    pen_ref = lp.penalty(kind, Xq, pending, radius, scale)
    ref = lp.penalized(ref_base, pen_ref)
    got = fn(Xq[:, None, :])
    assert got.shape == (Xq.shape[0], 1)
    _check_values(got, ref, 1e-6, None if base == "ei" else 1e-12 * np.nan_to_num(pen_ref))
    if kind == lp.HARD:
        assert np.all(got[3000:3000 + P] == 0.0)  # at the pending points themselves
    idx, best = fn.fused_argmax(Xq)
    assert idx == o.argmax_first(np.where(np.isnan(ref), -np.inf, ref))
    assert best == pytest.approx(np.nanmax(ref), rel=1e-6)


def test_penalised_values_single_precision_model():
    import trieste_b200 as tb
    from trieste_b200.acquisition import PenalizedAcquisition, expected_improvement, soft_local_penalizer

    om = o.synthetic_model(o.hartmann_6, 300, 6, dtype=np.float32)
    nm = tb.GaussianProcessRegression(tb.GPRSpec((om.X, om.y), tb.Matern52(om.variance, om.lengthscales),
                                                 tb.Constant(om.mean_const), om.noise))
    assert nm.dtype == np.float32
    om64 = o.build_model("matern52", om.X.astype(np.float64), om.y.astype(np.float64), om.variance, om.lengthscales,
                         om.noise, om.mean_const)
    L, eta, pending, radius, scale = _lp_state(om64, 7)
    ei_eta = o.ei_eta(om64)
    fn = PenalizedAcquisition(expected_improvement(nm, ei_eta), soft_local_penalizer(nm, pending, L, eta))
    Xq = _query_set(pending, radius).astype(np.float32)
    omean, ovar = o.predict(om64, Xq.astype(np.float64))
    ref = lp.penalized(o.expected_improvement(omean, ovar, ei_eta)[:, 0], lp.penalty(lp.SOFT, Xq.astype(np.float64), pending,
                                                                                        radius, scale))
    got = np.asarray(fn(Xq[:, None, :]), dtype=np.float64)[:, 0]
    big = ref > 1e-6 * ref.max()
    np.testing.assert_allclose(got[big], ref[big], rtol=1e-4)


@pytest.mark.parametrize("engine", ["int8", "fp64"])
@pytest.mark.parametrize("kind", [lp.SOFT, lp.HARD])
def test_penalised_gradients_match_oracle(kind, engine):
    from trieste_b200.acquisition import PenalizedAcquisition, expected_improvement

    om, nm = model_pair(o.hartmann_6, 300, 6, engine=engine)
    L, eta, pending, radius, scale = _lp_state(om, 7)
    Xq = _query_set(pending, radius, M=300)
    ei_eta = o.ei_eta(om)
    fn = PenalizedAcquisition(expected_improvement(nm, ei_eta), _penalizer_cls(kind)(nm, pending, L, eta))
    val, grad = fn.value_and_gradient(Xq[:, None, :])
    rval, rgrad = lp.penalized_ei_value_and_gradient(om, Xq, ei_eta, kind, pending, radius, scale)
    assert grad.shape == (Xq.shape[0], 1, 6)
    assert np.all(np.isfinite(grad))  # also at the pending points and on the radius spheres
    _check_values(val, rval, 1e-6)
    np.testing.assert_allclose(grad[:, 0, :], rgrad, rtol=1e-6, atol=1e-9 * np.abs(rgrad).max())
    # device candidates: the same numbers
    import torch

    xt = torch.as_tensor(Xq[:, None, :], device="cuda")
    vt, gt = fn.value_and_gradient(xt)
    np.testing.assert_array_equal(vt.cpu().numpy(), val)
    np.testing.assert_array_equal(gt.cpu().numpy(), grad)


def test_penalised_calls_leave_other_functions_on_the_model_untouched():
    from trieste_b200 import _lib
    from trieste_b200.acquisition import (PenalizedAcquisition, expected_improvement, hard_local_penalizer,
                                          min_value_entropy_search)

    om, nm = model_pair(o.hartmann_6, 300, 6)
    L, eta, pending, radius, scale = _lp_state(om, 7)
    Xq = _query_set(pending, radius, M=5000)
    ei = expected_improvement(nm, o.ei_eta(om))
    a = ei(Xq[:, None, :])
    ia = ei.fused_argmax(Xq)
    ga = ei.value_and_gradient(Xq[:200, None, :])[1]
    mes = min_value_entropy_search(nm, np.array([[om.y.min() - 0.3]]))
    pen_mes = PenalizedAcquisition(min_value_entropy_search(nm, np.array([[om.y.min() - 1.0]])),
                                   hard_local_penalizer(nm, pending, L, eta))
    pen_ei = PenalizedAcquisition(ei, hard_local_penalizer(nm, pending[:3], L, eta))
    m0 = mes(Xq[:, None, :])
    for fn in (pen_mes, pen_ei):
        fn(Xq[:, None, :])
        fn.fused_argmax(Xq)
        fn.value_and_gradient(Xq[:50, None, :])
    np.testing.assert_array_equal(ei(Xq[:, None, :]), a)
    assert ei.fused_argmax(Xq) == ia
    np.testing.assert_array_equal(ei.value_and_gradient(Xq[:200, None, :])[1], ga)
    np.testing.assert_array_equal(mes(Xq[:, None, :]), m0)
    # the ABI: a penalised call needs a penalty; the flag is stripped before the kind check
    import ctypes as C

    _, fresh = model_pair(o.hartmann_6, 50, 6)
    out = np.empty(4)
    x = np.ascontiguousarray(Xq[:4])
    with pytest.raises(ValueError, match="tb_acq_set_penalization"):
        _lib.check(_lib.lib().tb_acq_eval(fresh.handle, _lib.ACQ_EI | _lib.ACQ_PENALIZED, 0.0, x.ctypes.data, 4, out.ctypes.data,
                                          None))
    with pytest.raises(ValueError):
        _lib.check(_lib.lib().tb_acq_eval(fresh.handle, 7 | _lib.ACQ_PENALIZED, 0.0, x.ctypes.data, 4, out.ctypes.data, None))
    with pytest.raises(ValueError):
        _lib.check(_lib.lib().tb_acq_set_penalization(fresh.handle, 3, x.ctypes.data, 1, out.ctypes.data, out.ctypes.data))
    best, idx = C.c_double(), C.c_int64()
    with pytest.raises(ValueError):
        _lib.check(_lib.lib().tb_acq_argmax(fresh.handle, _lib.ACQ_EI | _lib.ACQ_PENALIZED, 0.0, x.ctypes.data, 4, None,
                                            C.byref(best), C.byref(idx)))


def test_builder_estimates_identity_and_errors():
    import trieste_b200 as tb
    from trieste_b200.acquisition import LocalPenalization, MinValueEntropySearch, PenalizedAcquisition

    om, nm = model_pair(o.hartmann_6, 300, 6)
    ds = tb.Dataset(om.X, om.y)
    space = lp.seeded_space([0.0] * 6, [1.0] * 6, seed=11)
    builder = LocalPenalization(space)
    fn = builder.prepare_acquisition_function(nm, ds)
    L, eta = lp.lipschitz_and_eta(om, np.concatenate([om.X, space.drawn[0]]))
    assert len(space.drawn[0]) == 500
    assert builder.lipschitz_constant == pytest.approx(L, rel=1e-8)
    assert builder.eta == pytest.approx(eta, rel=1e-9, abs=1e-12)
    pending = candidates(2, 6, seed=4)
    pfn = builder.update_acquisition_function(fn, nm, ds, pending_points=pending[:1], new_optimization_step=False)
    assert isinstance(pfn, PenalizedAcquisition)
    assert builder.update_acquisition_function(pfn, nm, ds, pending_points=pending, new_optimization_step=False) is pfn
    with pytest.raises(ValueError):
        pfn(candidates(6, 6).reshape(3, 2, 6))  # batch size one only
    with pytest.raises(ValueError):
        builder.update_acquisition_function(pfn, nm, ds, pending_points=pending[None], new_optimization_step=False)
    with pytest.raises(ValueError):
        builder.update_acquisition_function(pfn, nm, tb.Dataset(np.zeros((0, 6)), np.zeros((0, 1))), pending_points=pending)
    with pytest.raises(ValueError):
        LocalPenalization(space, num_samples=0)
    # MES base, hard penaliser: prepared through its own builder
    mb = LocalPenalization(space, num_samples=100, penalizer=_penalizer_cls(lp.HARD),
                           base_acquisition_function_builder=MinValueEntropySearch(space, num_samples=3, grid_size=200, seed=0))
    mfn = mb.prepare_acquisition_function(nm, ds)
    pm = mb.update_acquisition_function(mfn, nm, ds, pending_points=pending, new_optimization_step=False)
    Xq = candidates(500, 6, seed=9)
    omean, ovar = o.predict(om, Xq)
    pen_ref = lp.penalty(lp.HARD, Xq, pending, pm._penalization.radius, pm._penalization.scale)
    ref = lp.penalized(o.min_value_entropy_search(omean, ovar, mfn.samples)[:, 0], pen_ref)
    _check_values(pm(Xq[:, None, :]), ref, 1e-6, 1e-12 * np.nan_to_num(pen_ref))


def test_device_lbfgs_on_the_penalised_function_against_scipy():
    from trieste_b200.acquisition import PenalizedAcquisition, expected_improvement, soft_local_penalizer

    om, nm = model_pair(o.hartmann_6, 300, 6)
    L, eta, pending, radius, scale = _lp_state(om, 3)
    ei_eta = o.ei_eta(om)
    fn = PenalizedAcquisition(expected_improvement(nm, ei_eta), soft_local_penalizer(nm, pending, L, eta))
    lower, upper = np.zeros(6), np.ones(6)
    x0 = candidates(64, 6, seed=11)

    def oracle_vg(x):
        return lp.penalized_ei_value_and_gradient(om, x, ei_eta, lp.SOFT, pending, radius, scale)

    ok_d, f_d, x_d, n_d = fn.maximize_from(x0, lower, upper)
    ok_s, f_s, x_s, n_s = o.scipy_lbfgsb_multistart(oracle_vg, x0, lower, upper)
    scale_ = max(1.0, np.abs(f_s).max())
    assert f_d.max() >= f_s.max() - 1e-6 * scale_, (f_d.max(), f_s.max())
    fo, _ = oracle_vg(x_d)
    np.testing.assert_allclose(f_d, fo, rtol=1e-6, atol=1e-7 * scale_)


def _branin_setup(seed=0):
    import trieste_b200 as tb

    X = np.random.default_rng(seed).uniform(size=(5, 2))
    ds = tb.Dataset(X, o.branin(X))
    space = lp.seeded_space([0.0, 0.0], [1.0, 1.0], seed=100)
    spec = tb.build_gpr(ds, space, likelihood_variance=1e-3)  # the reference's LP integration case
    return ds, space, spec


def test_greedy_loop_picks_the_oracle_points_step_by_step():
    import trieste_b200 as tb
    from trieste_b200.acquisition import LocalPenalization
    from trieste_b200.acquisition.interface import OBJECTIVE
    from trieste_b200.rule import EfficientGlobalOptimization

    ds, space, spec = _branin_setup()
    k = spec.kernel
    nm = tb.GaussianProcessRegression(spec)
    cand_sets = [np.random.default_rng(1000 + s).uniform(size=(5000, 2)) for s in range(10)]
    chosen = []

    def random_search(space_, fn):  # a seeded 5000-point random search per step
        pts = cand_sets[len(chosen) // 3]
        idx, _ = fn.fused_argmax(pts)
        chosen.append(idx)
        return pts[idx:idx + 1]

    rule = EfficientGlobalOptimization(LocalPenalization(space), optimizer=random_search, num_query_points=3)
    X, Y = np.asarray(ds.query_points), np.asarray(ds.observations)
    for step in range(10):
        pts = rule.acquire(space, {OBJECTIVE: nm}, {OBJECTIVE: tb.Dataset(X, Y)})
        assert pts.shape == (3, 2)
        # the oracle's step: L, eta over this step's samples and the data; EI's eta is the LP eta on the first step only
        om = o.build_model("matern52", X, Y, k.variance, k.lengthscales, spec.noise_variance, spec.mean_function.c)
        L, eta = lp.lipschitz_and_eta(om, np.concatenate([X, space.drawn[step]]))
        ei_eta = eta if step == 0 else o.ei_eta(om)
        cands = cand_sets[step]
        mean, var = o.predict(om, cands)
        base = o.expected_improvement(mean, var, ei_eta)[:, 0]
        picks = [o.argmax_first(base)]
        for _ in range(2):
            pending = cands[picks]
            radius, scale = lp.penalizer_state(om, pending, L, eta)
            v = lp.penalized(base, lp.penalty(lp.SOFT, cands, pending, radius, scale))
            picks.append(o.argmax_first(np.where(np.isnan(v), -np.inf, v)))
        assert chosen[-3:] == picks, (step, chosen[-3:], picks)
        X = np.concatenate([X, pts])
        Y = np.concatenate([Y, o.branin(pts)])
        nm.update(tb.Dataset(X, Y))


def test_greedy_loop_with_the_default_optimiser_improves_with_distinct_batches():
    import trieste_b200 as tb
    from trieste_b200.acquisition import LocalPenalization
    from trieste_b200.acquisition.interface import OBJECTIVE
    from trieste_b200.rule import EfficientGlobalOptimization

    ds, space, spec = _branin_setup(seed=3)
    nm = tb.GaussianProcessRegression(spec)
    rule = EfficientGlobalOptimization(LocalPenalization(space), num_query_points=3)
    X, Y = np.asarray(ds.query_points), np.asarray(ds.observations)
    y0 = Y.min()
    for _ in range(15):
        pts = rule.acquire(space, {OBJECTIVE: nm}, {OBJECTIVE: tb.Dataset(X, Y)})
        assert pts.shape == (3, 2) and space.contains(pts).all()
        assert len({tuple(p) for p in np.round(pts, 12)}) == 3
        X = np.concatenate([X, pts])
        Y = np.concatenate([Y, o.branin(pts)])
        nm.update(tb.Dataset(X, Y))
    assert Y.min() < y0
