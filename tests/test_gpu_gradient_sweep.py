"""GPU: the derivative kernels against the oracle at every (kernel kind, padded dimension) pair, on every engine and in both
layouts of the gradient assembly; gradients across chunks at the headline size; GIBBON's cross and gradient kernels across
the register tile of pending points; and the Matern-12 instantiations of the joint paths.

Each derivative kernel is a template on the kernel kind and the padded input dimension DP, one unrolled instantiation per
pair, so each pair is compared separately.  ``grad_kernel`` runs one CTA per candidate for chunks of at most 2048
candidates and one warp per candidate above that; a call with 2,500 candidates at N = 256 is one chunk of the second kind,
and its first 300 candidates in a call of their own run the first.

Tolerances are the stated fp64 gradient ones (rtol 1e-6, atol 1e-9 of the largest reference component; the mean gradient
rtol 1e-8) for every kernel.  Matern-12 = exp(-r) is held to them against an oracle whose Cholesky factor comes from the
difference-form Gram (``tests/util.py``): the oracle's expansion-form r^2 leaves O(1e-16) on the diagonal of K(X, X), which
sqrt() turns into an O(1e-8) error of the reference itself.  The library's Gram has an exact diagonal.

The exceptions are the variance term of the int8 engines on the dense low-dimensional models of the sweep, listed case by
case in INT8_V_ATOL.  These engines form V = K^-1 k* in fixed point, so the error of V is relative to sum |K^-1| |k*| rather
than to |V|, and the LCB gradient divides d var by 2 sd.  With 256 points in D <= 10, cond(K + noise I) is up to 1e4 and sd
falls to 0.016 sigma_f.  Every other case keeps the 1e-9 bar on every engine: the mean gradient, the alpha term (beta = 0),
every fp64-engine gradient, and every int8 case not in the table.  The two layouts agree to 1e-12 of the scale everywhere."""
import numpy as np
import pytest

from oracle import gp_oracle as o
from tests import gibbon_oracle as gb
from tests.test_gpu_gibbon import _atol, _samples
from tests.util import candidates, exact_square_dist, model_pair, native_from_oracle, with_exact_cholesky

pytestmark = pytest.mark.gpu

KINDS = ("rbf", "matern12", "matern32", "matern52")
DIMS = (1, 3, 6, 7, 10, 11, 13, 19, 23, 32)  # DP = 2, 4, 6, 8, 10, 12, 16, 20, 24, 32: every padded dimension once
ENGINES = ("int8", "int8x21", "fp64")
N_SWEEP = 256
M_WARP = 2500  # > 2048 in one chunk: one warp per candidate
M_CTA = 300  # one CTA per candidate
BETAS = (1.0, 100.0)
# (engine, kind, D, beta): atol of the LCB gradient, as a fraction of its scale, where the int8 engines' V term exceeds
# 1e-9 (module docstring).  In the comments: the largest error beyond rtol 1e-6 over both layouts, measured on one H100
# 80GB HBM3.  The 21-product engine gains 15-40x over the single pass here, not the 256x of one more digit, because the
# error is dominated by the conditioning of K^-1.
INT8_V_ATOL = {
    ("int8", "rbf", 1, 1.0): 5e-7,  # 1.8e-7
    ("int8", "rbf", 1, 100.0): 1e-5,  # 4.0e-6
    ("int8", "rbf", 3, 1.0): 4e-8,  # 1.2e-8
    ("int8", "rbf", 3, 100.0): 1e-6,  # 3.1e-7
    ("int8", "rbf", 6, 100.0): 4e-8,  # 1.5e-8
    ("int8", "rbf", 7, 100.0): 1.5e-8,  # 4.8e-9
    ("int8", "rbf", 10, 100.0): 4e-9,  # 1.2e-9
    ("int8", "matern32", 1, 1.0): 5e-8,  # 1.7e-8
    ("int8", "matern32", 1, 100.0): 7e-7,  # 2.2e-7
    ("int8", "matern32", 3, 100.0): 8e-9,  # 2.5e-9
    ("int8", "matern52", 1, 1.0): 1.2e-7,  # 3.9e-8
    ("int8", "matern52", 1, 100.0): 3e-6,  # 1.0e-6
    ("int8", "matern52", 3, 100.0): 8e-8,  # 2.7e-8
    ("int8x21", "rbf", 1, 1.0): 1.2e-8,  # 4.2e-9
    ("int8x21", "rbf", 1, 100.0): 8e-7,  # 2.6e-7
    ("int8x21", "rbf", 3, 100.0): 4.5e-8,  # 1.5e-8
    ("int8x21", "matern32", 1, 100.0): 2.5e-8,  # 7.5e-9
    ("int8x21", "matern52", 1, 100.0): 2e-7,  # 6.1e-8
}
# the headline model (N = 4096, D = 10, Matern-52, beta = 1) on the single-pass engine: 1.7e-9, on the 21-product one 3e-11
HEADLINE_INT8_ATOL = 5e-9


def _reference_model(om):
    return with_exact_cholesky(om) if om.kind == "matern12" else om


def _oracle_rows(om, X, slab=250):
    """(mean, var, dmean, dvar) of the oracle at X, posterior_gradients in slabs (its temporary is [M, N, D])"""
    parts = []
    for s in range(0, X.shape[0], slab):
        mean, var = o.predict(om, X[s : s + slab])
        dmean, dvar = o.posterior_gradients(om, X[s : s + slab])
        parts.append((mean[:, 0], var[:, 0], dmean, dvar))
    return tuple(np.concatenate(p) for p in zip(*parts))


def _lcb_reference(mean, var, dmean, dvar, beta):
    sd = np.sqrt(var)
    return mean - beta * sd, dmean - beta * dvar / (2.0 * sd[:, None])


def _assert_grad(got, ref, what, rtol=1e-6, atol=1e-9):
    np.testing.assert_allclose(got, ref, rtol=rtol, atol=atol * np.abs(ref).max(), err_msg=what)


def _v_atol(engine, kind, D, beta):
    return INT8_V_ATOL.get((engine, kind, D, beta), 1e-9)


_SWEEP = {}


def _sweep_reference(kind, D):
    """built once per (kind, D) and shared by the three engines"""
    if (kind, D) not in _SWEEP:
        om = o.synthetic_model(o.ackley, N_SWEEP, D, kind=kind)
        X = candidates(M_WARP, D, seed=100 + D)
        _SWEEP[(kind, D)] = (om, X, _oracle_rows(_reference_model(om), X))
    return _SWEEP[(kind, D)]


# ---- 1. every (kind, DP) pair on every engine, both grad_kernel layouts and mean_grad_kernel ------------------------------
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("D", DIMS, ids=[f"D{d}" for d in DIMS])
@pytest.mark.parametrize("kind", KINDS)
def test_gradients_match_oracle_for_every_kind_and_padded_dimension(kind, D, engine):
    from trieste_b200.acquisition import lower_confidence_bound

    om, X, (mean, var, dmean, dvar) = _sweep_reference(kind, D)
    nm = native_from_oracle(om)
    nm.set_engine(engine)
    sf = np.sqrt(om.variance)
    # mean_grad_kernel (no variance, no GEMM)
    m_mg, g_mg = nm.mean_gradient(X)
    np.testing.assert_allclose(m_mg[:, 0], mean, rtol=1e-9, atol=1e-9 * sf, err_msg="mean_gradient: mean")
    _assert_grad(g_mg, dmean, "mean_gradient: gradient", rtol=1e-8)
    for beta in (0.0,) + BETAS:
        fn = lower_confidence_bound(nm, beta)
        ref_val, ref_grad = _lcb_reference(mean, var, dmean, dvar, beta)
        v_warp, g_warp = fn.value_and_gradient(X[:, None, :])
        v_cta, g_cta = fn.value_and_gradient(X[:M_CTA, None, :])
        assert g_warp.shape == (M_WARP, 1, D) and g_cta.shape == (M_CTA, 1, D)
        if beta == 0.0:  # the alpha term of grad_kernel alone
            np.testing.assert_allclose(v_warp[:, 0], mean, rtol=1e-9, atol=1e-9 * sf, err_msg="LCB(0) value")
        atol = _v_atol(engine, kind, D, beta)
        _assert_grad(g_warp[:, 0], ref_grad, f"beta={beta}: one warp per candidate", atol=atol)
        _assert_grad(g_cta[:, 0], ref_grad[:M_CTA], f"beta={beta}: one CTA per candidate", atol=atol)
        # the two layouts differ only in the order of the per-candidate sums
        scale = np.abs(ref_grad).max()
        np.testing.assert_allclose(g_cta[:, 0], g_warp[:M_CTA, 0], rtol=0, atol=1e-12 * scale,
                                   err_msg=f"beta={beta}: layouts disagree")


# ---- 2. one call across several chunks at the headline size ------------------------------------------------------------
@pytest.fixture(scope="module")
def headline():
    om = o.synthetic_model(o.ackley, 4096, 10)
    X = candidates(80_001, 10, seed=5)
    idx = np.unique(np.concatenate([np.arange(128), np.arange(0, X.shape[0], 61), np.arange(X.shape[0] - 128, X.shape[0])]))
    return om, X, idx, _oracle_rows(om, X[idx])


@pytest.mark.parametrize("engine", ENGINES)
def test_gradients_across_chunks_match_oracle(headline, engine):
    import torch

    from trieste_b200 import _lib
    from trieste_b200.acquisition import lower_confidence_bound

    om, X, idx, (mean, var, dmean, dvar) = headline
    nm = native_from_oracle(om)
    nm.set_engine(engine)
    fn = lower_confidence_bound(nm, 1.0)
    lib = _lib.lib()
    fn.value_and_gradient(X[:1000, None, :])  # lazy builds
    c0 = lib.tb_launch_count()
    fn.value_and_gradient(X[:1000, None, :])
    one = lib.tb_launch_count() - c0
    c0 = lib.tb_launch_count()
    val, grad = fn.value_and_gradient(X[:, None, :])
    assert lib.tb_launch_count() - c0 > one  # more than one chunk, the last one partial
    ref_val, ref_grad = _lcb_reference(mean, var, dmean, dvar, 1.0)
    np.testing.assert_allclose(val[idx, 0], ref_val, rtol=1e-6, atol=1e-9 * np.abs(ref_val).max())
    _assert_grad(grad[idx, 0], ref_grad, f"{engine}: sampled candidates", atol=HEADLINE_INT8_ATOL if engine == "int8" else 1e-9)
    # the same call on a torch CUDA tensor: the same numbers
    vt, gt = fn.value_and_gradient(torch.as_tensor(X[:, None, :], device="cuda"))
    np.testing.assert_array_equal(vt.cpu().numpy(), val)
    np.testing.assert_array_equal(gt.cpu().numpy(), grad)


# ---- 4. GIBBON across the register tile of pending points --------------------------------------------------------------
# The tolerances of test_gpu_gibbon.py, on the default engine.  One exception: the quality term at large |gamma|.  Both it
# and tests/gibbon_oracle.py evaluate h = r (gamma - r) with r = phi(gamma) / Phi(-gamma) ~ gamma, and that difference
# cancels.  At D = 1 the posterior sd falls to 0.016 sigma_f, so |gamma| reaches 300.  There the summed GIBBON gradient
# differs from the oracle by up to 6.5e-5 of its scale, on the fp64 engine as on the int8 one (one H100 80GB HBM3).  The
# smallest |gamma| seen among those candidates is 70.  So candidates whose largest |gamma| over the samples exceeds
# GIBBON_CANCEL_GAMMA are held at GIBBON_CANCEL_ATOL of the scale, and every other candidate at the stated bar.  The
# repulsion term does not have this form and is held at the stated bar everywhere.
GIBBON_CANCEL_GAMMA = 50.0
GIBBON_CANCEL_ATOL = 2e-4


@pytest.mark.parametrize("m", [7, 17])  # 17 crosses GIB_TILE = 16
@pytest.mark.parametrize("D", [1, 7, 13, 32])
@pytest.mark.parametrize("kind", KINDS)
def test_gibbon_gradients_match_oracle(kind, D, m, monkeypatch):
    from trieste_b200.acquisition import GibbonAcquisition, gibbon_quality_term, gibbon_repulsion_term

    om, nm = model_pair(o.ackley, N_SWEEP, D, kind=kind)
    if kind == "matern12":  # the oracle's K(P, P) and K(X, X) with exact diagonals, as the library's
        monkeypatch.setattr(o, "scaled_square_dist", exact_square_dist)
        om = with_exact_cholesky(om)
    pending = candidates(m, D, seed=40 + m)
    samples = _samples(om, 3)
    Xq = candidates(300, D, seed=6)
    r = gibbon_repulsion_term(nm, pending, rescaled_repulsion=False)
    fn = GibbonAcquisition(gibbon_quality_term(nm, samples), r)
    mean, var = o.predict(om, Xq)
    gamma = np.abs((samples.reshape(1, -1) - mean) / np.sqrt(var)).max(axis=1)
    cases = {
        "repulsion": (r, gb.repulsion_value_and_gradient(om, Xq, pending, False), np.zeros(len(Xq), bool)),
        "gibbon": (fn, gb.gibbon_value_and_gradient(om, Xq, samples, pending, False), gamma > GIBBON_CANCEL_GAMMA),
    }
    for name, (f, (rval, rgrad), cancels) in cases.items():
        val, grad = f.value_and_gradient(Xq[:, None, :])
        np.testing.assert_allclose(val, rval, rtol=1e-6, atol=_atol(om, "int8"), err_msg=name)
        scale = np.abs(rgrad).max()
        atol = np.where(cancels, GIBBON_CANCEL_ATOL, 1e-6)[:, None] * scale + 10 * _atol(om, "int8")
        err = np.abs(grad[:, 0, :] - rgrad) - 1e-5 * np.abs(rgrad)
        assert np.all(err <= atol), (name, int(np.sum((err > atol).any(axis=1))), float((err / scale).max()))


# ---- qEI and the covariance between points for Matern-12 ---------------------------------------------------------------
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("N,D,q,S", [(200, 6, 4, 64), (260, 10, 11, 100)])
def test_matern12_batch_mc_ei_value_and_gradient_matches_oracle(N, D, q, S, engine, monkeypatch):
    from trieste_b200 import Dataset
    from trieste_b200.acquisition import BatchMonteCarloExpectedImprovement

    monkeypatch.setattr(o, "scaled_square_dist", exact_square_dist)  # K(Xq, Xq) of predict_joint with an exact diagonal
    om, nm = model_pair(o.hartmann_6 if D == 6 else o.ackley, N, D, kind="matern12", engine=engine)
    om = with_exact_cholesky(om)
    fn = BatchMonteCarloExpectedImprovement(S, jitter=1e-6).prepare_acquisition_function(nm, Dataset(om.X, om.y))
    eps = np.random.default_rng(3).standard_normal((q, S))
    fn._sampler.set_eps(eps)
    fn._eta = float(np.median(om.y))  # plenty of active samples
    nb = 37
    X = candidates(nb * q, D).reshape(nb, q, D)
    val, grad = fn.value_and_gradient(X)
    np.testing.assert_allclose(val, fn(X), rtol=1e-9, atol=1e-13)
    for b in range(0, nb, 6):
        oval, ograd = o.batch_mc_ei_gradient(om, X[b], eps, fn._eta, 1e-6)
        np.testing.assert_allclose(val[b, 0], oval, rtol=1e-6, atol=1e-12)
        np.testing.assert_allclose(grad[b], ograd, rtol=1e-5, atol=1e-7 * max(np.abs(ograd).max(), 1e-30))


@pytest.mark.parametrize("engine", ["int8", "fp64"])
def test_matern12_covariance_between_points_matches_oracle(engine, monkeypatch):
    monkeypatch.setattr(o, "scaled_square_dist", exact_square_dist)  # K(X1, X2) is exact where the two sets share points
    om, nm = model_pair(o.hartmann_6, 300, 6, kind="matern12", engine=engine)
    om = with_exact_cholesky(om)
    rng = np.random.default_rng(0)
    X1 = rng.uniform(size=(3, 50, 6))
    X2 = np.concatenate([rng.uniform(size=(200, 6)), X1[0, :5]])
    cov = nm.covariance_between_points(X1, X2)
    ref = o.covariance_between_points(om, X1, X2)
    assert cov.shape == (3, 1, 50, 205)
    np.testing.assert_allclose(cov, ref, rtol=0, atol=1e-9 * om.variance)
