"""GIBBON (entropy.py:236-618) on the device against the NumPy restatement in tests/gibbon_oracle.py: quality, repulsion
and summed values on every engine, gradients, argmax, device L-BFGS, an independent cross-check through an appended
handle, handle isolation, model updates, launch counts, the C-ABI errors, the builder and the greedy BO loop.

Tolerances.  V_det = yvar - |u|^2 cancels: near a pending point it is about noise plus small terms, so an absolute variance
error eps becomes a repulsion error of about w eps / (2 noise).  The int8 engines state eps ~ 1e-9 sigma_f^2; the synthetic
models here have noise = Var(y) / 100 = sigma_f^2 / 100, so that is ~5e-8 w.  The quality term sees the same error through
rho^2 = var / (var + noise): ~eps / noise.  The cross term itself is computed in fp64 on every engine."""
import ctypes as C

import numpy as np
import pytest

from oracle import gp_oracle as o
from tests import gibbon_oracle as gb
from tests.util import candidates, model_pair, native_from_oracle

pytestmark = pytest.mark.gpu

ENGINE_VAR_EPS = {"int8": 1e-9, "int8x21": 1e-9, "fp64": 1e-12}  # stated |delta var| / sigma_f^2 per engine


def _atol(om, engine, w=1.0):
    """absolute allowance of a GIBBON value: quality ~ eps / noise, repulsion ~ w eps / (2 noise), with a factor 10 margin"""
    r = ENGINE_VAR_EPS[engine] * om.variance / om.noise
    return 1e-12 + 10.0 * r * (1.0 + 0.5 * w)


def _samples(om, S, seed=0):
    rng = np.random.default_rng(seed)
    s = om.y.min() - np.abs(rng.normal(size=(S, 1))) * np.sqrt(om.variance)
    if S > 1:
        s[1, 0] = om.y.max()  # gamma > 0 for most candidates
    return s


def _query_set(om, pending, M=3000, seed=1):
    """random candidates, the pending points themselves and training points"""
    return np.concatenate([candidates(M, om.X.shape[1], seed=seed), pending, om.X[:20]])


@pytest.mark.parametrize("engine", ["int8", "int8x21", "fp64"])
@pytest.mark.parametrize("kind", ["matern52", "rbf"])
@pytest.mark.parametrize("S", [1, 5])
def test_quality_term_values_match_oracle(S, kind, engine):
    from trieste_b200.acquisition import gibbon_quality_term

    om, nm = model_pair(o.hartmann_6, 300, 6, kind=kind, engine=engine)
    samples = _samples(om, S)
    Xq = np.concatenate([candidates(3000, 6), om.X[:20]])
    fn = gibbon_quality_term(nm, samples)
    mean, var = o.predict(om, Xq)
    ref = gb.quality_term(mean, var, samples, om.noise)
    got = fn(Xq[:, None, :])
    assert got.shape == (Xq.shape[0], 1)
    np.testing.assert_allclose(got, ref, rtol=1e-6, atol=_atol(om, engine))
    idx, best = fn.fused_argmax(Xq)
    assert idx == o.argmax_first(got[:, 0]) and best == got[idx, 0]


@pytest.mark.parametrize("engine", ["int8", "fp64"])
@pytest.mark.parametrize("m", [1, 7, 100])
@pytest.mark.parametrize("rescaled", [True, False])
def test_repulsion_and_sum_values_match_oracle(rescaled, m, engine):
    from trieste_b200.acquisition import GibbonAcquisition, gibbon_quality_term, gibbon_repulsion_term

    om, nm = model_pair(o.hartmann_6, 300, 6, engine=engine)
    pending = candidates(m, 6, seed=40 + m)
    Xq = _query_set(om, pending)
    samples = _samples(om, 3)
    rep = gibbon_repulsion_term(nm, pending, rescaled_repulsion=rescaled)
    w = gb.repulsion_weight(m, rescaled)
    assert rep.weight == w
    ref_rep = gb.repulsion_term(om, Xq, pending, rescaled)
    got_rep = rep(Xq[:, None, :])
    np.testing.assert_allclose(got_rep, ref_rep, rtol=1e-6, atol=_atol(om, engine, w))
    fn = GibbonAcquisition(gibbon_quality_term(nm, samples), rep)
    ref = gb.gibbon(om, Xq, samples, pending, rescaled)
    got = fn(Xq[:, None, :])
    np.testing.assert_allclose(got, ref, rtol=1e-6, atol=_atol(om, engine, w))
    # argmax: the first max of the values this build evaluates
    idx, best = fn.fused_argmax(Xq)
    assert idx == o.argmax_first(got[:, 0]) and best == got[idx, 0]
    assert abs(ref[idx, 0] - ref.max()) <= 1e-6 * abs(ref.max()) + _atol(om, engine, w)


def test_gibbon_values_single_precision_model():
    import trieste_b200 as tb
    from trieste_b200.acquisition import GibbonAcquisition, gibbon_quality_term, gibbon_repulsion_term

    om = o.synthetic_model(o.hartmann_6, 300, 6, dtype=np.float32)
    nm = tb.GaussianProcessRegression(tb.GPRSpec((om.X, om.y), tb.Matern52(om.variance, om.lengthscales),
                                                 tb.Constant(om.mean_const), om.noise))
    assert nm.dtype == np.float32
    om64 = o.build_model("matern52", om.X.astype(np.float64), om.y.astype(np.float64), om.variance, om.lengthscales,
                         om.noise, om.mean_const)
    pending = candidates(7, 6, seed=3)
    samples = _samples(om64, 3)
    fn = GibbonAcquisition(gibbon_quality_term(nm, samples), gibbon_repulsion_term(nm, pending))
    Xq = np.concatenate([candidates(3000, 6), pending]).astype(np.float32)
    ref = gb.gibbon(om64, Xq.astype(np.float64), samples, pending)[:, 0]
    got = np.asarray(fn(Xq[:, None, :]), dtype=np.float64)[:, 0]
    np.testing.assert_allclose(got, ref, rtol=1e-4, atol=1e-4 * np.abs(ref).max())


@pytest.mark.parametrize("engine", ["int8", "int8x21", "fp64"])
@pytest.mark.parametrize("acq", ["quality", "repulsion", "gibbon"])
def test_gradients_match_oracle(acq, engine):
    import torch
    from trieste_b200.acquisition import GibbonAcquisition, gibbon_quality_term, gibbon_repulsion_term

    om, nm = model_pair(o.hartmann_6, 300, 6, engine=engine)
    pending = candidates(7, 6, seed=5)
    samples = _samples(om, 3)
    Xq = np.concatenate([candidates(200, 6, seed=6), pending, om.X[:10]])
    q, r = gibbon_quality_term(nm, samples), gibbon_repulsion_term(nm, pending, rescaled_repulsion=False)
    fn = {"quality": q, "repulsion": r, "gibbon": GibbonAcquisition(q, r)}[acq]
    if acq == "quality":
        rval, rgrad = gb.quality_value_and_gradient(om, Xq, samples)
    elif acq == "repulsion":
        rval, rgrad = gb.repulsion_value_and_gradient(om, Xq, pending, False)
    else:
        rval, rgrad = gb.gibbon_value_and_gradient(om, Xq, samples, pending, False)
    val, grad = fn.value_and_gradient(Xq[:, None, :])
    assert grad.shape == (Xq.shape[0], 1, 6) and np.all(np.isfinite(grad))
    np.testing.assert_allclose(val, rval, rtol=1e-6, atol=_atol(om, engine))
    scale = np.abs(rgrad).max()
    np.testing.assert_allclose(grad[:, 0, :], rgrad, rtol=1e-5, atol=1e-6 * scale + 10 * _atol(om, engine))
    # device candidates: the same numbers
    vt, gt = fn.value_and_gradient(torch.as_tensor(Xq[:, None, :], device="cuda"))
    np.testing.assert_array_equal(vt.cpu().numpy(), val)
    np.testing.assert_array_equal(gt.cpu().numpy(), grad)


def test_device_lbfgs_on_gibbon_against_scipy():
    from trieste_b200.acquisition import GibbonAcquisition, gibbon_quality_term, gibbon_repulsion_term

    om, nm = model_pair(o.hartmann_6, 300, 6)
    pending = candidates(3, 6, seed=8)
    samples = _samples(om, 3)
    fn = GibbonAcquisition(gibbon_quality_term(nm, samples), gibbon_repulsion_term(nm, pending))
    lower, upper = np.zeros(6), np.ones(6)
    x0 = candidates(64, 6, seed=11)

    def oracle_vg(x):
        v, g = gb.gibbon_value_and_gradient(om, x, samples, pending)
        return v[:, 0], g

    ok_d, f_d, x_d, n_d = fn.maximize_from(x0, lower, upper)
    ok_s, f_s, x_s, n_s = o.scipy_lbfgsb_multistart(oracle_vg, x0, lower, upper)
    scale = max(1.0, np.abs(f_s).max())
    assert f_d.max() >= f_s.max() - 1e-6 * scale, (f_d.max(), f_s.max())
    np.testing.assert_allclose(f_d, oracle_vg(x_d)[0], rtol=1e-6, atol=1e-7 * scale)


@pytest.mark.parametrize("m", [1, 7])
def test_repulsion_equals_the_variance_ratio_of_an_appended_handle(m):
    """independent of the oracle: w/2 log((noise + var_aug) / (noise + var)) with var_aug from a second handle whose data
    are extended by the pending points through tb_gp_append_data"""
    import trieste_b200 as tb
    from trieste_b200.acquisition import gibbon_repulsion_term

    om, nm = model_pair(o.hartmann_6, 300, 6, engine="fp64")
    aug = native_from_oracle(om)
    aug.set_engine("fp64")
    pending = candidates(m, 6, seed=21)
    aug.update(tb.Dataset(np.concatenate([om.X, pending]), np.concatenate([om.y, np.zeros((m, 1))])))
    assert aug.last_update_appended
    Xq = np.concatenate([candidates(2000, 6, seed=22), pending, om.X[:10]])
    _, var = nm.predict(Xq)
    _, var_aug = aug.predict(Xq)
    ref = gb.repulsion_weight(m, True) * 0.5 * np.log((om.noise + var_aug) / (om.noise + var))
    got = gibbon_repulsion_term(nm, pending)(Xq[:, None, :])
    np.testing.assert_allclose(got, ref, rtol=1e-6, atol=1e-9)


def test_gibbon_calls_leave_other_functions_on_the_model_untouched():
    from trieste_b200.acquisition import (GibbonAcquisition, PenalizedAcquisition, expected_improvement, gibbon_quality_term,
                                          gibbon_repulsion_term, min_value_entropy_search, soft_local_penalizer)

    om, nm = model_pair(o.hartmann_6, 300, 6)
    Xq = candidates(5000, 6, seed=2)
    ei = expected_improvement(nm, o.ei_eta(om))
    mes = min_value_entropy_search(nm, np.array([[om.y.min() - 0.3]]))
    pending = candidates(3, 6, seed=3)
    lp = PenalizedAcquisition(expected_improvement(nm, o.ei_eta(om)), soft_local_penalizer(nm, pending, 5.0, o.ei_eta(om)))
    before = [(f(Xq[:, None, :]), f.fused_argmax(Xq), f.value_and_gradient(Xq[:100, None, :])[1]) for f in (ei, mes, lp)]
    g = GibbonAcquisition(gibbon_quality_term(nm, np.array([[om.y.min() - 1.0]])), gibbon_repulsion_term(nm, pending[:2]))
    g(Xq[:, None, :])
    g.fused_argmax(Xq)
    g.value_and_gradient(Xq[:50, None, :])
    after = [(f(Xq[:, None, :]), f.fused_argmax(Xq), f.value_and_gradient(Xq[:100, None, :])[1]) for f in (ei, mes, lp)]
    for (a0, i0, g0), (a1, i1, g1) in zip(before, after):
        np.testing.assert_array_equal(a0, a1)
        assert i0 == i1
        np.testing.assert_array_equal(g0, g1)


@pytest.mark.parametrize("path", ["append", "refactorise"])
def test_the_same_acquisition_object_follows_model_updates(path):
    import trieste_b200 as tb
    from trieste_b200.acquisition import GibbonAcquisition, gibbon_quality_term, gibbon_repulsion_term

    om, nm = model_pair(o.hartmann_6, 300, 6, engine="fp64")
    pending = candidates(5, 6, seed=31)
    samples = _samples(om, 3)
    fn = GibbonAcquisition(gibbon_quality_term(nm, samples), gibbon_repulsion_term(nm, pending))
    Xq = np.concatenate([candidates(1000, 6, seed=32), pending])
    np.testing.assert_allclose(fn(Xq[:, None, :]), gb.gibbon(om, Xq, samples, pending), rtol=1e-6, atol=1e-10)
    rng = np.random.default_rng(33)
    if path == "append":
        Xn = np.concatenate([om.X, rng.uniform(size=(4, 6))])
    else:
        Xn = rng.uniform(size=(280, 6))
    yn = o.hartmann_6(Xn)
    nm.update(tb.Dataset(Xn, yn))
    assert nm.last_update_appended == (path == "append")
    nm.optimize(tb.Dataset(Xn, yn))
    om2 = o.build_model("matern52", Xn, yn, om.variance, om.lengthscales, om.noise, om.mean_const)
    np.testing.assert_allclose(fn(Xq[:, None, :]), gb.gibbon(om2, Xq, samples, pending), rtol=1e-6, atol=1e-10)


def test_repeated_calls_launch_a_fixed_number_of_kernels_beyond_mes():
    from trieste_b200 import _lib
    from trieste_b200.acquisition import (GibbonAcquisition, gibbon_quality_term, gibbon_repulsion_term,
                                          min_value_entropy_search)

    om, nm = model_pair(o.hartmann_6, 300, 6)
    Xq = candidates(5000, 6, seed=4)
    Xg = Xq[:64, None, :]
    samples = _samples(om, 3)
    lib = _lib.lib()

    def launches(f):
        f()  # warm: lazily built state (digit tiles, K^-1, GIBBON's W and L_B^-1) is built here
        c0 = lib.tb_launch_count()
        f()
        return lib.tb_launch_count() - c0

    mes = min_value_entropy_search(nm, samples)
    base_v, base_a, base_g = (launches(lambda: mes(Xq[:, None, :])), launches(lambda: mes.fused_argmax(Xq)),
                              launches(lambda: mes.value_and_gradient(Xg)))
    q = gibbon_quality_term(nm, samples)
    assert launches(lambda: q(Xq[:, None, :])) == base_v
    for m in (1, 40):
        fn = GibbonAcquisition(q, gibbon_repulsion_term(nm, candidates(m, 6, seed=m)))
        assert launches(lambda: fn(Xq[:, None, :])) == base_v + 1  # one cross-term launch per chunk
        assert launches(lambda: fn.fused_argmax(Xq)) == base_a + 1
        assert launches(lambda: fn.value_and_gradient(Xg)) == base_g + 2  # cross term + its gradient


def test_abi_errors():
    from trieste_b200 import _lib

    om, nm = model_pair(o.hartmann_6, 50, 6)
    lib = _lib.lib()
    x = np.ascontiguousarray(candidates(4, 6))
    out = np.empty(4)
    pend = np.ascontiguousarray(candidates(2, 6, seed=9))

    def ev(acq):
        _lib.check(lib.tb_acq_eval(nm.handle, acq, 0.0, x.ctypes.data, 4, out.ctypes.data, None))

    with pytest.raises(ValueError, match="tb_acq_set_gibbon_repulsion"):
        ev(_lib.ACQ_GIBBON_REPULSION)
    with pytest.raises(ValueError, match="tb_acq_set_min_value_samples"):
        ev(_lib.ACQ_GIBBON_QUALITY)
    s = np.array([om.y.min() - 0.2])
    _lib.check(lib.tb_acq_set_min_value_samples(nm.handle, s.ctypes.data_as(C.POINTER(C.c_double)), 1))
    ev(_lib.ACQ_GIBBON_QUALITY)
    with pytest.raises(ValueError, match="tb_acq_set_gibbon_repulsion"):
        ev(_lib.ACQ_GIBBON)
    for acq in (_lib.ACQ_GIBBON_QUALITY, _lib.ACQ_GIBBON_REPULSION, _lib.ACQ_GIBBON):
        with pytest.raises(ValueError, match="PENALIZED"):
            ev(acq | _lib.ACQ_PENALIZED)
    with pytest.raises(ValueError):
        ev(10)
    for m in (0, -1):
        with pytest.raises(ValueError):
            _lib.check(lib.tb_acq_set_gibbon_repulsion(nm.handle, pend.ctypes.data, m, 1.0))
    _lib.check(lib.tb_acq_set_gibbon_repulsion(nm.handle, pend.ctypes.data, 2, 0.25))
    ev(_lib.ACQ_GIBBON)
    k = nm.get_kernel()
    ls = np.ascontiguousarray(np.asarray(k.lengthscales, dtype=np.float64).reshape(-1))
    _lib.check(lib.tb_gp_set_hyper(nm.handle, 3, float(k.variance), ls.ctypes.data_as(C.POINTER(C.c_double)), ls.size, om.noise,
                                   float(nm.get_mean_function().c)))
    with pytest.raises(ValueError):
        ev(_lib.ACQ_GIBBON)  # the cache is stale after the hyper-parameters changed: the old W and L_B are never used
    _lib.check(lib.tb_gp_update_posterior_cache(nm.handle))
    ev(_lib.ACQ_GIBBON)
    # B + noise I that cannot be factorised (a NaN pending point): TB_ERR_NUMERIC, and the failed set is not kept
    bad = pend.copy()
    bad[1, 0] = np.nan
    with pytest.raises(ValueError, match="Cholesky"):
        _lib.check(lib.tb_acq_set_gibbon_repulsion(nm.handle, bad.ctypes.data, 2, 0.25))
    with pytest.raises(ValueError, match="tb_acq_set_gibbon_repulsion"):
        ev(_lib.ACQ_GIBBON)


def test_builder_protocol_identity_and_errors():
    import trieste_b200 as tb
    from trieste_b200.acquisition import GIBBON, GibbonAcquisition, gibbon_quality_term
    from trieste_b200.acquisition.sampler import ExactThompsonSampler, GumbelSampler
    from tests import lp_oracle as lpo

    om, nm = model_pair(o.hartmann_6, 200, 6)
    ds = tb.Dataset(om.X, om.y)
    space = lpo.seeded_space([0.0] * 6, [1.0] * 6, seed=3)
    b = GIBBON(space, num_samples=3, grid_size=100, seed=0)
    q = b.prepare_acquisition_function(nm, ds)
    assert type(q) is gibbon_quality_term and q.samples.shape == (3, 1)
    assert b.update_acquisition_function(q, nm, ds) is q  # new samples, same object
    pending = candidates(2, 6, seed=1)
    g = b.update_acquisition_function(q, nm, ds, pending_points=pending[:1], new_optimization_step=False)
    assert isinstance(g, GibbonAcquisition)
    assert b.update_acquisition_function(g, nm, ds, pending_points=pending, new_optimization_step=False) is g
    assert g._diversity_term.pending_points.shape == (2, 6) and g._diversity_term.weight == 0.25
    assert b.update_acquisition_function(g, nm, ds, pending_points=None, new_optimization_step=False) is q
    assert b.prepare_acquisition_function(nm, ds, pending_points=pending) is g
    Xq = candidates(300, 6, seed=2)
    mean, var = o.predict(om, Xq)
    np.testing.assert_allclose(g(Xq[:, None, :]), gb.gibbon(om, Xq, q.samples, pending), rtol=1e-6, atol=1e-8)
    with pytest.raises(ValueError):
        g(candidates(6, 6).reshape(3, 2, 6))  # batch size one only
    with pytest.raises(ValueError):
        b.update_acquisition_function(g, nm, ds, pending_points=pending[None], new_optimization_step=False)
    with pytest.raises(ValueError):
        b.prepare_acquisition_function(nm, tb.Dataset(np.zeros((0, 6)), np.zeros((0, 1))))
    with pytest.raises(ValueError):
        b.prepare_acquisition_function(object(), ds)
    for kw in ({"num_samples": 0}, {"grid_size": 0}, {"min_value_sampler": ExactThompsonSampler(sample_min_value=False)}):
        with pytest.raises(ValueError):
            GIBBON(space, **kw)
    GIBBON(space, min_value_sampler=GumbelSampler(sample_min_value=True))
    with pytest.raises(ValueError):
        gibbon_quality_term(nm, np.zeros(3))
    b2 = GIBBON(space, num_samples=3, grid_size=100, rescaled_repulsion=False, seed=0)
    g2 = b2.prepare_acquisition_function(nm, ds, pending_points=pending)
    assert isinstance(g2, GibbonAcquisition) and g2._diversity_term.weight == 1.0


def _branin_setup(seed=0):
    import trieste_b200 as tb
    from tests import lp_oracle as lpo

    X = np.random.default_rng(seed).uniform(size=(5, 2))
    ds = tb.Dataset(X, o.branin(X))
    space = lpo.seeded_space([0.0, 0.0], [1.0, 1.0], seed=100)
    spec = tb.build_gpr(ds, space, likelihood_variance=1e-3)
    return ds, space, spec


def test_greedy_loop_picks_the_oracle_points_step_by_step():
    import trieste_b200 as tb
    from trieste_b200.acquisition import GIBBON
    from trieste_b200.acquisition.interface import OBJECTIVE
    from trieste_b200.rule import EfficientGlobalOptimization

    ds, space, spec = _branin_setup()
    k = spec.kernel
    nm = tb.GaussianProcessRegression(spec)
    nm.set_engine("fp64")
    cand_sets = [np.random.default_rng(2000 + s).uniform(size=(5000, 2)) for s in range(6)]
    chosen = []

    def random_search(space_, fn):
        pts = cand_sets[len(chosen) // 3]
        idx, _ = fn.fused_argmax(pts)
        chosen.append(idx)
        return pts[idx:idx + 1]

    builder = GIBBON(space, num_samples=5, grid_size=200, seed=7)
    rule = EfficientGlobalOptimization(builder, optimizer=random_search, num_query_points=3)
    X, Y = np.asarray(ds.query_points), np.asarray(ds.observations)
    for step in range(6):
        pts = rule.acquire(space, {OBJECTIVE: nm}, {OBJECTIVE: tb.Dataset(X, Y)})
        assert pts.shape == (3, 2)
        om = o.build_model("matern52", X, Y, k.variance, k.lengthscales, spec.noise_variance, spec.mean_function.c)
        samples = builder._min_value_samples
        cands = cand_sets[step]
        mean, var = o.predict(om, cands)
        picks = [o.argmax_first(gb.quality_term(mean, var, samples, om.noise)[:, 0])]
        for _ in range(2):
            v = gb.gibbon(om, cands, samples, cands[picks])[:, 0]
            picks.append(o.argmax_first(np.where(np.isnan(v), -np.inf, v)))
        assert chosen[-3:] == picks, (step, chosen[-3:], picks)
        X = np.concatenate([X, pts])
        Y = np.concatenate([Y, o.branin(pts)])
        nm.update(tb.Dataset(X, Y))


def test_greedy_loop_with_the_default_optimiser_returns_distinct_batches():
    import trieste_b200 as tb
    from trieste_b200.acquisition import GIBBON
    from trieste_b200.acquisition.interface import OBJECTIVE
    from trieste_b200.rule import EfficientGlobalOptimization

    ds, space, spec = _branin_setup(seed=3)
    nm = tb.GaussianProcessRegression(spec)
    rule = EfficientGlobalOptimization(GIBBON(space, seed=1), num_query_points=4)
    X, Y = np.asarray(ds.query_points), np.asarray(ds.observations)
    for _ in range(4):
        pts = rule.acquire(space, {OBJECTIVE: nm}, {OBJECTIVE: tb.Dataset(X, Y)})
        assert pts.shape == (4, 2) and space.contains(pts).all()
        assert len({tuple(p) for p in np.round(pts, 9)}) == 4
        X = np.concatenate([X, pts])
        Y = np.concatenate([Y, o.branin(pts)])
        nm.update(tb.Dataset(X, Y))
