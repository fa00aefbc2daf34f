"""GPU: fp32 models (TB_F32 handles; BASELINE config 5 is fp32).  fp32 arrays cross the boundary in both
directions with no silent fp64 arrays at the API (tests/integration/test_bayesian_optimization.py:641-658);
stated fp32 tolerances (SURVEY.md §8c): mean rtol 1e-4, variance atol 1e-4 sigma_f^2."""
import numpy as np
import pytest

from oracle import gp_oracle as o
from tests.util import candidates

pytestmark = pytest.mark.gpu


def _pair32(obj, N, D):
    import trieste_b200 as tb

    om = o.synthetic_model(obj, N, D)
    X32, y32 = om.X.astype(np.float32), om.y.astype(np.float32)
    # the oracle sees exactly the fp32-rounded data, in fp64 arithmetic
    om32 = o.build_model(om.kind, X32.astype(np.float64), y32.astype(np.float64), om.variance, om.lengthscales, om.noise, om.mean_const)
    nm = tb.GaussianProcessRegression(tb.GPRSpec((X32, y32), tb.Matern52(om.variance, om.lengthscales), tb.Constant(om.mean_const), om.noise))
    return om32, nm


def _assert_fp32_gradient(grad, ref):
    """the stated fp32 tolerance, 1e-4 of each candidate's gradient scale (its largest component)"""
    err = np.abs(grad.astype(np.float64) - ref) / np.abs(ref).max(axis=1, keepdims=True)
    assert err.max() < 1e-4, (err.max(), int(np.argmax(err.max(axis=1))))


@pytest.mark.parametrize("N,D", [(300, 6), (1024, 20)])
def test_fp32_predict_and_log_ei(N, D):
    from trieste_b200.acquisition import log_expected_improvement

    om, nm = _pair32(o.hartmann_6 if D == 6 else o.random_fourier_objective, N, D)
    assert nm.dtype == np.float32
    Xq = candidates(3000, D).astype(np.float32)
    mean, var = nm.predict(Xq)
    assert mean.dtype == np.float32 and var.dtype == np.float32
    omean, ovar = o.predict(om, Xq.astype(np.float64))
    np.testing.assert_allclose(mean, omean, rtol=1e-4, atol=1e-4 * np.sqrt(om.variance))
    np.testing.assert_allclose(var, ovar, rtol=0, atol=1e-4 * om.variance)
    eta = o.ei_eta(om)
    fn = log_expected_improvement(nm, eta)
    val, grad = fn.value_and_gradient(Xq[:, None, :])
    assert val.dtype == np.float32 and grad.dtype == np.float32 and grad.shape == (3000, 1, D)
    ref = o.log_expected_improvement(omean, ovar, eta)
    np.testing.assert_allclose(val, ref, rtol=1e-4, atol=1e-4)
    # 3000 candidates in one chunk: one warp per candidate in the gradient assembly
    _, rg = o.log_ei_gradient(om, Xq.astype(np.float64), eta)
    _assert_fp32_gradient(grad[:, 0, :], rg)
    idx, best = fn.fused_argmax(Xq)
    assert idx == int(np.argmax(ref[:, 0])) or abs(ref[idx, 0] - ref.max()) < 1e-4


def test_fp32_joint_and_qei_and_torch_io():
    import torch

    from trieste_b200 import Dataset
    from trieste_b200.acquisition import BatchMonteCarloExpectedImprovement

    om, nm = _pair32(o.hartmann_6, 200, 6)
    X = candidates(64 * 4, 6).reshape(64, 4, 6).astype(np.float32)
    mean, cov = nm.predict_joint(X)
    assert cov.dtype == np.float32
    omean, ocov = o.predict_joint(om, X.astype(np.float64))
    np.testing.assert_allclose(cov, ocov, rtol=0, atol=1e-4 * om.variance)
    fn = BatchMonteCarloExpectedImprovement(128).prepare_acquisition_function(nm, Dataset(om.X.astype(np.float32), om.y.astype(np.float32)))
    eps = np.random.default_rng(0).standard_normal((4, 128)).astype(np.float32)
    fn._sampler.set_eps(eps)
    out = fn(X)
    ref = o.batch_monte_carlo_expected_improvement(om, X.astype(np.float64), eps.astype(np.float64)[None], fn._eta, 1e-6)
    np.testing.assert_allclose(out, ref, rtol=2e-3, atol=1e-5)
    xt = torch.from_numpy(X.reshape(-1, 6)).cuda()
    m2, v2 = nm.predict(xt)
    assert m2.dtype == torch.float32 and m2.is_cuda
    np.testing.assert_allclose(m2.cpu().numpy(), mean.reshape(-1, 1), rtol=1e-6, atol=1e-6)
