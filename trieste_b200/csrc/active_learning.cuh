// The q-batch predictive variance of active learning (predictive_variance, active_learning.py:98-108):
//   value = exp(logdet(cov + jitter)) = exp(2 sum_i log diag chol(M)),  M = cov + jitter 1 1^T
// The reference adds the scalar jitter to EVERY entry of the covariance (a broadcast, not jitter I); kept as it is.
#pragma once
#include "kernels_extra.cuh"

namespace tb {

// One warp per batch, after joint_kernel has left the batch's covariance in cov_in [nb][q][q].  GRAD: the reverse pass in
// qei_backward_kernel's contract: c_mu = 0, c_var = 1 and Sigma_bar = d value / d cov = det(M) M^-1, where M^-1 comes from
// warp_cholesky_backward with the adjoint of the factor's diagonal of logdet = 2 sum log C_ii, i.e. G = diag(2 / C_ii).
// qei_mix_kernel, grad_kernel and qei_cross_kernel then assemble d value / d Xc.  Shared memory per warp: q^2 doubles,
// 3 q^2 with GRAD.  A pivot that is not positive sets *err_flag (TB_ERR_NUMERIC).
constexpr int PV_WARPS = 4;

__host__ __device__ constexpr int pv_warp_doubles(int q, bool grad) { return (grad ? 3 : 1) * q * q; }

template <bool GRAD>
__global__ void __launch_bounds__(PV_WARPS * 32, 1)
pv_kernel(const double* __restrict__ cov_in, int64_t nb, int q, double jitter, double* __restrict__ out_val,
          double* __restrict__ cmu, double* __restrict__ cvar, double* __restrict__ sbar, int* __restrict__ err_flag) {
  extern __shared__ __align__(16) unsigned char pvsm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qq = q * q;
  double* Cs = reinterpret_cast<double*>(pvsm) + (size_t)warp * pv_warp_doubles(q, GRAD);
  const int64_t b = (int64_t)blockIdx.x * PV_WARPS + warp;
  if (b >= nb) return;
  for (int e = lane; e < qq; e += 32) Cs[e] = cov_in[b * qq + e] + jitter;
  __syncwarp();
  if (!warp_cholesky(Cs, q, lane)) {
    if (lane == 0) atomicExch(err_flag, 1);
    return;
  }
  double ld = 0.0;  // tf.linalg.logdet: 2 reduce_sum(log(diag(chol)))
  for (int i = 0; i < q; ++i) ld += log(Cs[i * q + i]);
  const double det = exp(2.0 * ld);
  if (lane == 0) out_val[b] = det;
  if (!GRAD) return;
  double* Gs = Cs + qq;
  double* Ts = Gs + qq;
  for (int e = lane; e < qq; e += 32) {
    const int r = e / q, c = e % q;
    Gs[e] = r == c ? 2.0 / Cs[e] : 0.0;
  }
  __syncwarp();
  warp_cholesky_backward(Cs, Gs, Ts, q, lane);  // Gs = M^-1
  const int64_t t0 = b * q;
  for (int e = lane; e < q; e += 32) {
    cmu[t0 + e] = 0.0;
    cvar[t0 + e] = 1.0;
  }
  for (int e = lane; e < qq; e += 32) sbar[b * qq + e] = det * Gs[e];
}

}  // namespace tb
