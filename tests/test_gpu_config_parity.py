"""GPU parity at the sizes BASELINE.json names (round-1 verdict, item 1): the CUDA path against the oracle at
C3 (N=4096, D=10, q=8, S=512), C4 (F=2048, D=6, 1e6 candidates), C5 (N=8192, D=20, fp32 I/O), the int8 engine at its
N=16384 limit, EI gradients on the native fp64 engine — and the device optimiser against the REFERENCE's optimiser engine
(SciPy L-BFGS-B on the oracle's value+gradient, trieste/acquisition/optimizer.py:700-745) from identical starts."""
import numpy as np
import pytest

from oracle import gp_oracle as o
from tests.util import candidates, model_pair, native_from_oracle

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def headline_pair():
    return model_pair(o.ackley, 4096, 10)


# ---- C3: Ackley-10, N=4096, BatchMonteCarloExpectedImprovement q=8, S=512 ---------------------------------------------
def test_c3_batch_mc_ei_value_and_gradient_at_config_size(headline_pair):
    from trieste_b200 import Dataset
    from trieste_b200.acquisition import BatchMonteCarloExpectedImprovement

    om, nm = headline_pair
    q, S, D = 8, 512, 10
    fn = BatchMonteCarloExpectedImprovement(S).prepare_acquisition_function(nm, Dataset(om.X, om.y))
    eps = np.random.default_rng(3).standard_normal((q, S))
    fn._sampler.set_eps(eps)
    # batches around the best observations (where the improvement is not identically zero) mixed with uniform ones
    rng = np.random.default_rng(1)
    best = om.X[np.argsort(om.y[:, 0])[:16]]
    near = np.clip(best[rng.integers(0, 16, size=(192, q))] + 0.01 * rng.standard_normal((192, q, D)), 0, 1)
    Xb = np.concatenate([near, rng.uniform(size=(64, q, D))])
    val = fn(Xb)
    ref = o.batch_monte_carlo_expected_improvement(om, Xb, eps[None], fn._eta, 1e-6)
    assert val.shape == (256, 1) and np.count_nonzero(ref > 1e-8) >= 32, np.count_nonzero(ref > 1e-8)
    np.testing.assert_allclose(val, ref, rtol=1e-6, atol=1e-10)
    v16, g16 = fn.value_and_gradient(Xb[:16])
    pairs = [o.batch_mc_ei_gradient(om, Xb[i], eps, fn._eta, 1e-6) for i in range(16)]  # the oracle takes one batch at a time
    rv, rg = np.array([p[0] for p in pairs]), np.stack([p[1] for p in pairs])
    np.testing.assert_allclose(v16[:, 0], rv, rtol=1e-6, atol=1e-10)
    np.testing.assert_allclose(g16, rg, rtol=1e-5, atol=1e-8 * max(1.0, np.abs(rg).max()))


# ---- C4: Hartmann6, RFF F=2048, Thompson argmin over 1e6 candidates -----------------------------------------------------
def test_c4_rff_trajectory_values_and_exact_argmin_at_config_size():
    from trieste_b200.sampler import RandomFourierFeatureTrajectorySampler

    om, nm = model_pair(o.hartmann_6, 1024, 6)
    F = 2048
    sampler = RandomFourierFeatureTrajectorySampler(nm, F, seed=0)
    W, b = o.rff_draw("matern52", F, 6, np.random.default_rng(4))
    sampler._feature_functions.set_weights(W, b)
    traj = sampler.get_trajectory()
    Xq = candidates(1_000_000, 6)
    mv, mi = traj.argmin_over(Xq)  # fused evaluation + argmin: no value leaves the device
    theta = traj._weights_sample  # [1, F]
    # values on a 1e5 sample at the trajectory tolerance
    idx = np.random.default_rng(7).choice(Xq.shape[0], 100_000, replace=False)
    out = traj(Xq[idx][:, None, :])
    ref = o.rff_trajectory(Xq[idx][:, None, :], W, b, theta, om.variance, om.lengthscales, om.mean_const)
    np.testing.assert_allclose(out, ref, rtol=1e-9, atol=1e-9 * np.sqrt(om.variance))
    # exact argmin over all 1e6 candidates (the oracle evaluates every candidate, chunked)
    full = o.rff_trajectory(Xq[:, None, :], W, b, theta, om.variance, om.lengthscales, om.mean_const)[:, 0, 0]
    j = int(np.argmin(full))
    assert int(mi[0]) == j, (int(mi[0]), j, full[int(mi[0])] - full[j])
    assert abs(mv[0] - full[j]) <= 1e-9 * max(1.0, abs(full[j]))


# ---- C5: Synthetic-20D, N=8192, fp32 I/O, log-EI value + gradient --------------------------------------------------------
def test_c5_fp32_log_ei_value_and_gradient_at_config_size():
    import trieste_b200 as tb
    from trieste_b200.acquisition import log_expected_improvement

    N, D = 8192, 20
    om = o.synthetic_model(o.random_fourier_objective, N, D)
    X32, y32 = om.X.astype(np.float32), om.y.astype(np.float32)
    om32 = o.build_model(om.kind, X32.astype(np.float64), y32.astype(np.float64), om.variance, om.lengthscales, om.noise, om.mean_const)
    nm = tb.GaussianProcessRegression(tb.GPRSpec((X32, y32), tb.Matern52(om.variance, om.lengthscales), tb.Constant(om.mean_const), om.noise))
    assert nm.dtype == np.float32 and nm.engine_info()[0] in (6, 15, 10)
    Xq = candidates(2048, D).astype(np.float32)
    mean, var = nm.predict(Xq)
    omean, ovar = o.predict_batched(om32, Xq.astype(np.float64))
    np.testing.assert_allclose(mean, omean, rtol=1e-4, atol=1e-4 * np.sqrt(om.variance))
    np.testing.assert_allclose(var, ovar, rtol=0, atol=1e-4 * om.variance)
    eta = o.ei_eta(om32)
    fn = log_expected_improvement(nm, eta)
    # more than 2048 candidates in one call: the one-warp-per-candidate gradient assembly the multi-start optimiser runs
    Xg = np.concatenate([Xq, candidates(452, D, seed=2).astype(np.float32)])
    val, grad = fn.value_and_gradient(Xg[:, None, :])
    assert val.dtype == np.float32 and grad.dtype == np.float32 and grad.shape == (2500, 1, D)
    sub = np.concatenate([np.arange(0, 2500, 25), np.arange(2500 - 28, 2500)])
    rv, rg = o.log_ei_gradient(om32, Xg[sub].astype(np.float64), eta)
    np.testing.assert_allclose(val[sub], rv, rtol=2e-4, atol=2e-4)
    err = np.abs(grad[sub, 0, :].astype(np.float64) - rg) / np.abs(rg).max(axis=1, keepdims=True)
    assert err.max() < 1e-4, (err.max(), int(sub[np.argmax(err.max(axis=1))]))


# ---- the int8 engine at its accumulator limit --------------------------------------------------------------------------
@pytest.mark.timeout(900)
def test_int8_engine_at_n16384():
    om, nm = model_pair(o.ackley, 16384, 10)
    Xq = candidates(600, 10)
    omean, ovar = o.predict_batched(om, Xq)
    sf = np.sqrt(om.variance)
    for engine in ("int8", "int8x21"):
        nm.set_engine(engine)
        assert nm.engine_info()[0] in (15, 21)
        mean, var = nm.predict(Xq)
        np.testing.assert_allclose(mean, omean, rtol=1e-9, atol=1e-9 * sf)
        np.testing.assert_allclose(var, ovar, rtol=0, atol=1e-9 * om.variance)


# ---- EI / LCB gradients on both engines --------------------------------------------------------------------------------
@pytest.mark.parametrize("engine", ["int8", "fp64"])
def test_ei_gradient_matches_oracle_on_both_engines(engine):
    from trieste_b200.acquisition import expected_improvement

    om, nm = model_pair(o.hartmann_6, 1024, 6, engine=engine)
    eta = o.ei_eta(om)
    fn = expected_improvement(nm, eta)
    best = om.X[np.argsort(om.y[:, 0])[:32]]
    Xq = np.clip(best[np.random.default_rng(0).integers(0, 32, 400)] + 0.05 * np.random.default_rng(1).standard_normal((400, 6)), 0, 1)
    val, grad = fn.value_and_gradient(Xq[:, None, :])
    ei, gei = o.ei_gradient(om, Xq, eta)
    np.testing.assert_allclose(val, ei, rtol=1e-6, atol=1e-14)
    np.testing.assert_allclose(grad[:, 0, :], gei, rtol=1e-6, atol=1e-9 * max(1.0, np.abs(gei).max()))


# ---- the device optimiser against SciPy L-BFGS-B (the reference's engine) from identical starts ---------------------------
@pytest.mark.parametrize("which", ["neg_lcb", "log_ei"])
def test_device_optimiser_against_scipy_lbfgsb_on_the_oracle(which):
    from trieste_b200.acquisition import log_expected_improvement
    from trieste_b200.acquisition.function import _lcb

    om, nm = model_pair(o.hartmann_6, 300, 6)
    eta = o.ei_eta(om)
    lower, upper = np.zeros(6), np.ones(6)
    x0 = candidates(64, 6, seed=11)
    if which == "neg_lcb":
        fn = _lcb(nm, 1.96, negate=True)

        def oracle_vg(x):  # -(mean - beta sqrt(var)) and its gradient from the oracle's posterior gradients
            mean, var = o.predict(om, x)
            dmean, dvar = o.posterior_gradients(om, x)
            sd = np.sqrt(var[:, 0])
            return -mean[:, 0] + 1.96 * sd, -dmean + 1.96 * dvar / (2.0 * sd[:, None])
    else:
        fn = log_expected_improvement(nm, eta)

        def oracle_vg(x):
            val, g = o.log_ei_gradient(om, x, eta)
            return val[:, 0], g

    ok_d, f_d, x_d, n_d = fn.maximize_from(x0, lower, upper)
    ok_s, f_s, x_s, n_s = o.scipy_lbfgsb_multistart(oracle_vg, x0, lower, upper)
    scale = max(1.0, np.abs(f_s).max())
    # (i) the best run of the device optimiser is at least as good as SciPy's best run
    assert f_d.max() >= f_s.max() - 1e-6 * scale, (f_d.max(), f_s.max())
    # (ii) the values the device reports are the oracle's values at the points it returns
    fo, _ = oracle_vg(x_d)
    np.testing.assert_allclose(f_d, fo, rtol=1e-6, atol=1e-7 * scale)
    # (iii) start by start.  The two engines are different algorithms (projected L-BFGS + Armijo backtracking here,
    # L-BFGS-B with Cauchy point + More-Thuente search in SciPy), so from one start they may settle in different local
    # optima of a multi-modal function; what is held is that both converge, that the device run is not systematically the
    # worse of the two, and — for the uni-modal-per-basin LCB — that they agree in >= 90 % of the starts.
    both = ok_d & ok_s
    agree = np.abs(f_d - f_s) <= 1e-4 * scale
    device_better = f_d > f_s + 1e-4 * scale
    scipy_better = f_s > f_d + 1e-4 * scale
    stats = {"which": which, "starts": int(x0.shape[0]), "both_converged": float(both.mean()), "agree": float(agree[both].mean()),
             "device_better": float(device_better[both].mean()), "scipy_better": float(scipy_better[both].mean()),
             "best_device": float(f_d.max()), "best_scipy": float(f_s.max()), "median_device": float(np.median(f_d)),
             "median_scipy": float(np.median(f_s)), "nfev_device_mean": float(n_d.mean()), "nfev_scipy_mean": float(n_s.mean())}
    import json
    import os

    out_dir = os.environ.get("TB_TEST_RECORD_DIR")  # optional: keep the comparison statistics as a JSON record
    if out_dir and os.path.isdir(out_dir):
        json.dump(stats, open(os.path.join(out_dir, f"optimizer_vs_scipy_{which}.json"), "w"))
    assert both.mean() >= 0.9, stats
    assert stats["scipy_better"] <= stats["device_better"] + 0.15, stats  # not systematically the worse engine
    assert stats["median_device"] >= stats["median_scipy"] - 0.02 * scale, stats
    if which == "neg_lcb":
        assert agree[both].mean() >= 0.9, stats


# ---- multiple-optimism LCB (vectorised) ---------------------------------------------------------------------------------
def test_multiple_optimism_lcb_matches_oracle_and_drives_batchify_vectorize():
    import trieste_b200 as tb
    from trieste_b200.acquisition import MultipleOptimismNegativeLowerConfidenceBound
    from trieste_b200.acquisition.optimizer import generate_continuous_optimizer
    from trieste_b200.rule import EfficientGlobalOptimization

    om, nm = model_pair(o.hartmann_6, 300, 6)
    space = tb.Box([0.0] * 6, [1.0] * 6)
    ds = tb.Dataset(om.X, om.y)
    builder = MultipleOptimismNegativeLowerConfidenceBound(space)
    fn = builder.prepare_acquisition_function(nm, ds)
    Xb = candidates(500 * 4, 6).reshape(500, 4, 6)
    out = fn(Xb)
    ref = o.multiple_optimism_lower_confidence_bound(om, Xb, 6)
    assert out.shape == (500, 4)
    np.testing.assert_allclose(fn.betas, o.molcb_betas(4, 6), rtol=1e-12)
    np.testing.assert_allclose(out, ref, rtol=1e-8, atol=1e-9)
    assert builder.update_acquisition_function(fn, nm, ds) is fn
    with pytest.raises(ValueError):
        fn(Xb[:, :3])  # the batch size is fixed by the first call (function.py:1886-1893)
    # gradient: central differences of the oracle restatement
    v, g = fn.value_and_gradient(Xb[:20])
    h = 1e-6
    for d in range(6):
        e = np.zeros(6)
        e[d] = h
        fd = (o.multiple_optimism_lower_confidence_bound(om, Xb[:20] + e, 6) - o.multiple_optimism_lower_confidence_bound(om, Xb[:20] - e, 6)) / (2 * h)
        np.testing.assert_allclose(g[..., d], fd, rtol=1e-4, atol=1e-5)
    # EGO with a vectorised builder optimises the q columns independently (rule.py:291-295)
    rule = EfficientGlobalOptimization(MultipleOptimismNegativeLowerConfidenceBound(space),
                                       generate_continuous_optimizer(2000, 8), num_query_points=3)
    pts = rule.acquire_single(space, nm, ds)
    assert pts.shape == (3, 6) and space.contains(pts).all()
    vals = rule.acquisition_function(pts[None])[0]
    rnd = space.sample(2000, seed=3)
    col = rule.acquisition_function(np.repeat(rnd[:, None, :], 3, axis=1))
    assert np.all(vals >= col.max(axis=0) - 1e-6 * np.abs(col).max())


# ---- Fantasizer --------------------------------------------------------------------------------------------------------
def test_fantasizer_kriging_believer_matches_the_conditional_posterior():
    import trieste_b200 as tb
    from trieste_b200.acquisition import ExpectedImprovement, Fantasizer
    from trieste_b200.acquisition.interface import OBJECTIVE
    from trieste_b200.acquisition.optimizer import generate_continuous_optimizer
    from trieste_b200.rule import EfficientGlobalOptimization

    om, nm = model_pair(o.hartmann_6, 300, 6)
    space = tb.Box([0.0] * 6, [1.0] * 6)
    ds = tb.Dataset(om.X, om.y)
    models, datasets = {OBJECTIVE: nm}, {OBJECTIVE: ds}
    builder = Fantasizer(ExpectedImprovement())
    base = builder.prepare_acquisition_function(models, datasets)
    Xq = candidates(400, 6)
    omean, ovar = o.predict(om, Xq)
    np.testing.assert_allclose(base(Xq[:, None, :]), o.expected_improvement(omean, ovar, o.ei_eta(om)), rtol=1e-6, atol=1e-14)
    # two pending points: kriging believer = posterior mean of the base model as observations
    pending = candidates(2, 6, seed=9)
    fant = builder.update_acquisition_function(base, models, datasets, pending_points=pending, new_optimization_step=False)
    y_kb, _ = o.predict(om, pending)
    cmean, cvar = o.conditional_predict_f(om, Xq, pending, y_kb)
    fmodel = builder._fantasized_models[OBJECTIVE]
    mean, var = fmodel.predict(Xq)
    np.testing.assert_allclose(mean, cmean, rtol=1e-8, atol=1e-9 * np.sqrt(om.variance))
    np.testing.assert_allclose(var, np.maximum(cvar, 1e-12), rtol=0, atol=1e-9 * om.variance)
    # eta of the fantasised EI: min of the conditional mean over data + pending points (function.py:133-149 on the joined data)
    Xall = np.concatenate([om.X, pending])
    eta_f = float(np.min(o.conditional_predict_f(om, Xall, pending, y_kb)[0]))
    assert abs(fant.eta - eta_f) <= 1e-8 * max(1.0, abs(eta_f))
    np.testing.assert_allclose(fant(Xq[:, None, :]), o.expected_improvement(cmean, np.maximum(cvar, 1e-12), eta_f), rtol=1e-5, atol=1e-13)
    # a third pending point extends the cache by a rank-1 append, same function object
    pending3 = np.concatenate([pending, candidates(1, 6, seed=10)])
    fant2 = builder.update_acquisition_function(fant, models, datasets, pending_points=pending3, new_optimization_step=False)
    assert fant2 is fant and fmodel.last_update_appended
    y3, _ = o.predict(om, pending3)
    cmean3, cvar3 = o.conditional_predict_f(om, Xq, pending3, y3)
    mean3, var3 = fmodel.predict(Xq)
    np.testing.assert_allclose(mean3, cmean3, rtol=1e-8, atol=1e-9 * np.sqrt(om.variance))
    np.testing.assert_allclose(var3, np.maximum(cvar3, 1e-12), rtol=0, atol=1e-9 * om.variance)
    # the variance collapses at the pending points, so greedy EGO spreads the batch
    rule = EfficientGlobalOptimization(Fantasizer(), generate_continuous_optimizer(2000, 8), num_query_points=3)
    pts = rule.acquire(space, models, datasets)
    assert pts.shape == (3, 6) and space.contains(pts).all()
    d = np.linalg.norm(pts[:, None, :] - pts[None, :, :], axis=-1)
    assert d[np.triu_indices(3, 1)].min() > 1e-3
    with pytest.raises(ValueError):
        Fantasizer(fantasize_method="mean")
    with pytest.raises(NotImplementedError):
        Fantasizer().prepare_acquisition_function({OBJECTIVE: object()}, datasets)


# ---- torch tensors produced on torch's stream are ordered before the library's stream (round-1 advisor finding) ----------
def test_device_tensor_inputs_need_no_manual_synchronisation():
    import torch

    om, nm = model_pair(o.hartmann_6, 300, 6)
    base = torch.rand(1_500_000, 6, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    for rep in range(3):
        # a long chain of elementwise work queued on torch's stream right before the call
        x = base
        for _ in range(20):
            x = torch.sin(x * 1.000001) * 0.5 + 0.5
        m_dev, v_dev = nm.predict(x)  # no torch.cuda.synchronize() in between
        xh = x.cpu().numpy()
        idx = np.random.default_rng(rep).choice(xh.shape[0], 2000, replace=False)
        omean, ovar = o.predict(om, xh[idx])
        np.testing.assert_allclose(m_dev.cpu().numpy()[idx], omean, rtol=1e-9, atol=1e-9)
        np.testing.assert_allclose(v_dev.cpu().numpy()[idx], ovar, rtol=0, atol=1e-9 * om.variance)
