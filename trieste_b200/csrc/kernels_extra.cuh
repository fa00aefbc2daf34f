// Kernels beyond the marginal predict + acquisition path:
//   - predict_joint / BatchReparametrizationSampler / MC-qEI  (per-batch Gram on the DMMA pipe)
//   - d acquisition / d x*                                    (second triangular GEMM with Linv^T)
//   - random-Fourier-feature trajectories + Thompson argmin
//   - top-k (bitonic sort of (value, index) pairs)
#pragma once
#include "gp_handle.cuh"
#include "kernels_f64.cuh"

namespace tb {

// one CTA per (row-block K, n-panel nc >= 8K) of the upper triangle: LinvT[k, n] = Linv[n, k]
__global__ void pack_upper_panels_kernel(const double* __restrict__ Linv, int64_t N, int NB, int nkB,
                                         double* __restrict__ P) {
  const int K = blockIdx.y, nc = blockIdx.x;
  if (nc < K * (BM / BK) || nc >= nkB) return;
  const int64_t base = (int64_t)K * nkB - rowblock_panel_offset(K - 1) - (int64_t)K * (BM / BK);
  double* dst = P + (base + nc) * PANEL;
  for (int e = threadIdx.x; e < PANEL; e += blockDim.x) {
    int kk = e % BK, r = e / BK;  // kk fastest: source Linv[n + k*N] with n = 16 nc + kk contiguous
    int64_t k = (int64_t)K * BM + r, n = (int64_t)nc * BK + kk;
    double v = (n < N && k < N && n >= k) ? Linv[n + k * N] : 0.0;
    dst[panel_elem_index(r, kk)] = v;
  }
}

// ------------------------------------------------------------------------------------------------
// K2: joint posterior of q-batches.  One warp per batch:
//   Gram G = A_b^T A_b on the DMMA pipe (A_b = the batch's q columns of A = Linv K*, plain layout),
//   cov = K(x_b, x_b) - G (diagonal clipped >= 1e-12, interface.py:130-132), then by mode
//   JOINT_PREDICT : write mean [q], cov [q,q]
//   JOINT_SAMPLE  : chol(cov + jitter I) (sampler.py:277-278), samples = mean + chol eps   [S,q]
//   JOINT_QEI     : mean_s max(eta - min_q sample, 0)                      (function.py:1183-1186)
// ------------------------------------------------------------------------------------------------
enum { JOINT_PREDICT = 0, JOINT_SAMPLE = 1, JOINT_QEI = 2 };
constexpr int JOINT_WARPS = 4;

template <int KIND, int QT>
__global__ void __launch_bounds__(JOINT_WARPS * 32)
joint_kernel(const double* __restrict__ Aplain, int64_t lda, int Nrows,  // [cands][lda]
             const double* __restrict__ mean_in,                         // [cands]
             const double* __restrict__ Xc, const double* __restrict__ inv_ls, int D,  // raw [cands][D]
             int64_t nb, int q, double variance, int mode, const double* __restrict__ eps, int S,
             double eta, double jitter, double* __restrict__ out_mean, double* __restrict__ out_cov,
             double* __restrict__ out_samples, double* __restrict__ out_qei, int* __restrict__ err_flag) {
  extern __shared__ __align__(16) unsigned char jsm[];
  const int QP = QT * 8;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double* cov_s = reinterpret_cast<double*>(jsm) + (size_t)warp * (QP * QP + QP * D + QP);
  double* x_s = cov_s + QP * QP;   // [q][D] scaled coordinates
  double* mu_s = x_s + QP * D;     // [q]
  const int64_t b = (int64_t)blockIdx.x * JOINT_WARPS + warp;
  if (b >= nb) return;
  const int64_t t0 = b * q;

  // ---- Gram on the DMMA pipe: a-fragment == b-fragment for the diagonal tiles ----
  double acc[QT][QT][2];
#pragma unroll
  for (int i = 0; i < QT; ++i)
#pragma unroll
    for (int j = 0; j < QT; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
  const int cl = lane >> 2, kq = lane & 3;
  const double* colp[QT];
  bool colv[QT];
#pragma unroll
  for (int i = 0; i < QT; ++i) {
    colv[i] = (i * 8 + cl) < q;
    colp[i] = Aplain + (t0 + (colv[i] ? i * 8 + cl : 0)) * lda + kq;
  }
  for (int k0 = 0; k0 < Nrows; k0 += 8) {
    double f0[QT], f1[QT];
#pragma unroll
    for (int i = 0; i < QT; ++i) {
      f0[i] = colv[i] ? colp[i][k0] : 0.0;
      f1[i] = colv[i] ? colp[i][k0 + 4] : 0.0;
    }
#pragma unroll
    for (int i = 0; i < QT; ++i)
#pragma unroll
      for (int j = 0; j < QT; ++j) dmma_m8n8k4(acc[i][j][0], acc[i][j][1], f0[i], f0[j]);
#pragma unroll
    for (int i = 0; i < QT; ++i)
#pragma unroll
      for (int j = 0; j < QT; ++j) dmma_m8n8k4(acc[i][j][0], acc[i][j][1], f1[i], f1[j]);
  }

  // ---- stage the batch's scaled coordinates and means ----
  for (int e = lane; e < q * D; e += 32) x_s[e] = Xc[t0 * D + e] * inv_ls[e % D];
  for (int e = lane; e < q; e += 32) mu_s[e] = mean_in[t0 + e];
  __syncwarp();

  // ---- cov = K(x,x) - G ----
#pragma unroll
  for (int i = 0; i < QT; ++i)
#pragma unroll
    for (int j = 0; j < QT; ++j)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int r = i * 8 + cl, cc = j * 8 + kq * 2 + c;
        if (r < q && cc < q) {
          double v;
          if (r == cc) {
            v = fmax(variance - acc[i][j][c], 1e-12);
          } else {
            double r2 = 0.0;
            for (int d = 0; d < D; ++d) {
              double df = x_s[r * D + d] - x_s[cc * D + d];
              r2 = fma(df, df, r2);
            }
            v = kernel_from_r2<KIND>(r2, variance) - acc[i][j][c];
          }
          cov_s[r * QP + cc] = v;
        }
      }
  __syncwarp();

  if (mode == JOINT_PREDICT) {
    for (int e = lane; e < q; e += 32) out_mean[t0 + e] = mu_s[e];
    for (int e = lane; e < q * q; e += 32) out_cov[b * q * q + e] = cov_s[(e / q) * QP + (e % q)];
    return;
  }

  // ---- in-place Cholesky of cov + jitter I (lower), lane i owns row i ----
  bool bad = false;
  for (int j = 0; j < q; ++j) {
    double djj = 0.0;
    if (lane == 0) {
      double s = cov_s[j * QP + j] + jitter;
      for (int k = 0; k < j; ++k) s = fma(-cov_s[j * QP + k], cov_s[j * QP + k], s);
      djj = sqrt(s);
      cov_s[j * QP + j] = djj;
    }
    djj = __shfl_sync(0xffffffffu, djj, 0);
    if (!(djj > 0.0)) bad = true;
    __syncwarp();
    for (int i = j + 1 + lane; i < q; i += 32) {
      double s = cov_s[i * QP + j];
      for (int k = 0; k < j; ++k) s = fma(-cov_s[i * QP + k], cov_s[j * QP + k], s);
      cov_s[i * QP + j] = s / djj;
    }
    __syncwarp();
  }
  if (bad && lane == 0) atomicExch(err_flag, 1);

  // ---- samples: lanes stride over the S base samples ----
  double accq = 0.0;
  for (int s = lane; s < S; s += 32) {
    double mn = DBL_MAX;
    for (int i = 0; i < q; ++i) {
      double f = mu_s[i];
      for (int k = 0; k <= i; ++k) f = fma(cov_s[i * QP + k], __ldg(eps + (int64_t)k * S + s), f);
      if (mode == JOINT_SAMPLE) out_samples[(b * S + s) * q + i] = f;
      mn = fmin(mn, f);
    }
    accq += fmax(eta - mn, 0.0);
  }
  if (mode == JOINT_QEI) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) accq += __shfl_xor_sync(0xffffffffu, accq, o);
    if (lane == 0) out_qei[b] = accq / (double)S;
  }
}

// In-place Cholesky (lower) of the n x n row-major matrix A by one warp, as in joint_kernel: lane 0 takes the pivot, the
// lanes split the column below it.  The strict upper triangle is left as it was and never read back.  False when a
// pivot is not positive (the result is then meaningless).
__device__ __forceinline__ bool warp_cholesky(double* A, int n, int lane) {
  bool bad = false;
  for (int j = 0; j < n; ++j) {
    double djj = 0.0;
    if (lane == 0) {
      double sdiag = A[j * n + j];
      for (int k = 0; k < j; ++k) sdiag = fma(-A[j * n + k], A[j * n + k], sdiag);
      djj = sqrt(sdiag);
      A[j * n + j] = djj;
    }
    djj = __shfl_sync(0xffffffffu, djj, 0);
    if (!(djj > 0.0)) bad = true;
    __syncwarp();
    for (int i = j + 1 + lane; i < n; i += 32) {
      double v = A[i * n + j];
      for (int k = 0; k < j; ++k) v = fma(-A[i * n + k], A[j * n + k], v);
      A[i * n + j] = v / djj;
    }
    __syncwarp();
  }
  return !bad;
}

// Cholesky reverse mode (Murray 2016, tf.linalg.cholesky's gradient) by one warp: C the lower factor, G the adjoint of
// its lower triangle on entry and the symmetric adjoint of the factorised matrix, C^-T sym(Phi(C^T G)) C^-1, on exit
// (Phi = lower triangle with the diagonal halved).  T is n x n scratch.
__device__ __forceinline__ void warp_cholesky_backward(const double* C, double* G, double* T, int n, int lane) {
  const int nn = n * n;
  // P = Phi(C^T G) (lower, diagonal halved) -> T
  for (int e = lane; e < nn; e += 32) {
    const int a = e / n, c = e % n;
    double v = 0.0;
    if (a >= c) {
      for (int i = a; i < n; ++i) v = fma(C[i * n + a], G[i * n + c], v);
      if (a == c) v *= 0.5;
    }
    T[e] = v;
  }
  __syncwarp();
  // M = (P + P^T) / 2 (symmetric) -> G
  for (int e = lane; e < nn; e += 32) {
    const int a = e / n, c = e % n;
    G[e] = (a == c) ? T[e] : 0.5 * (a > c ? T[a * n + c] : T[c * n + a]);
  }
  __syncwarp();
  // T1 = C^-T M: back substitution of C^T T1 = M, lane = column -> T
  for (int c = lane; c < n; c += 32) {
    for (int a = n - 1; a >= 0; --a) {
      double v = G[a * n + c];
      for (int i = a + 1; i < n; ++i) v = fma(-C[i * n + a], T[i * n + c], v);
      T[a * n + c] = v / C[a * n + a];
    }
  }
  __syncwarp();
  // result = T1 C^-1: row r solves C^T x = T1[r][:]^T, lane = row -> G
  for (int r = lane; r < n; r += 32) {
    for (int a = n - 1; a >= 0; --a) {
      double v = T[r * n + a];
      for (int i = a + 1; i < n; ++i) v = fma(-C[i * n + a], G[r * n + i], v);
      G[r * n + a] = v / C[a * n + a];
    }
  }
  __syncwarp();
}

// ------------------------------------------------------------------------------------------------
// K2g: reverse pass of the batch Monte-Carlo EI of one q-batch (function.py:1181-1186 through sampler.py:262-287), i.e.
// what TensorFlow's autodiff produces for  mean_s max(eta - min_j (mu + C eps_s)_j, 0),  C = chol(cov + jitter I):
//   G_mu[j]   = -(1/S) #{s active, argmin = j}            G_C[j][k] = -(1/S) sum_{s active, argmin = j} eps[k][s]  (k <= j)
//   Sigma_bar = C^-T sym(Phi(C^T G_C)) C^-1               (Cholesky reverse mode, Murray 2016; Phi = tril, diagonal halved)
// One warp per batch; outputs the value, c_mu = G_mu (and c_var = 1) for the gradient assembly, and Sigma_bar [q,q].
// Shared memory per warp: 3 q^2 + 2 q doubles.
// ------------------------------------------------------------------------------------------------
constexpr int QEIG_WARPS = 4;

__global__ void __launch_bounds__(QEIG_WARPS * 32)
qei_backward_kernel(const double* __restrict__ mean_in, const double* __restrict__ cov_in, int64_t nb, int q,
                    const double* __restrict__ eps, int S, double eta, double jitter, double* __restrict__ out_val,
                    double* __restrict__ cmu, double* __restrict__ cvar, double* __restrict__ sbar, int* __restrict__ err_flag) {
  extern __shared__ __align__(16) unsigned char qsm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qq = q * q;
  double* Cs = reinterpret_cast<double*>(qsm) + (size_t)warp * (3 * qq + 2 * q);
  double* Gs = Cs + qq;
  double* Ts = Gs + qq;
  double* mu = Ts + qq;
  double* gmu = mu + q;
  const int64_t b = (int64_t)blockIdx.x * QEIG_WARPS + warp;
  if (b >= nb) return;
  const int64_t t0 = b * q;
  for (int e = lane; e < qq; e += 32) {
    Cs[e] = cov_in[b * qq + e] + ((e / q == e % q) ? jitter : 0.0);
    Gs[e] = 0.0;
  }
  for (int e = lane; e < q; e += 32) {
    mu[e] = mean_in[t0 + e];
    gmu[e] = 0.0;
  }
  __syncwarp();
  if (!warp_cholesky(Cs, q, lane)) {
    if (lane == 0) atomicExch(err_flag, 1);
    return;
  }
  // forward over the base samples; the active arg-min entries feed G_mu / G_C
  const double invS = 1.0 / (double)S;
  double acc = 0.0;
  for (int s = lane; s < S; s += 32) {
    double mn = DBL_MAX;
    int arg = 0;
    for (int i = 0; i < q; ++i) {
      double f = mu[i];
      for (int k = 0; k <= i; ++k) f = fma(Cs[i * q + k], __ldg(eps + (int64_t)k * S + s), f);
      if (f < mn) {  // first minimum wins (tf.reduce_min / argmin)
        mn = f;
        arg = i;
      }
    }
    const double imp = eta - mn;
    if (imp > 0.0) {
      acc += imp;
      atomicAdd(&gmu[arg], -invS);
      for (int k = 0; k <= arg; ++k) atomicAdd(&Gs[arg * q + k], -invS * __ldg(eps + (int64_t)k * S + s));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  __syncwarp();
  warp_cholesky_backward(Cs, Gs, Ts, q, lane);
  if (lane == 0) out_val[b] = acc * invS;
  for (int e = lane; e < q; e += 32) {
    cmu[t0 + e] = gmu[e];
    cvar[t0 + e] = 1.0;
  }
  for (int e = lane; e < qq; e += 32) sbar[b * qq + e] = Gs[e];
}

// V~[j][n] = sum_k Sigma_bar[b][j][k] V[k][n] inside every batch, in place (V plain [point][ldv]); grid (nb, ceil(N/256)):
// the batch index rides on grid.x (no 65535 limit)
__global__ void __launch_bounds__(256)
qei_mix_kernel(double* __restrict__ V, int64_t ldv, int N, int q, const double* __restrict__ sbar) {
  __shared__ double sb[32 * 32];
  const int64_t b = blockIdx.x;
  for (int e = threadIdx.x; e < q * q; e += blockDim.x) sb[e] = sbar[b * q * q + e];
  __syncthreads();
  const int n = blockIdx.y * blockDim.x + threadIdx.x;
  if (n >= N) return;
  double v[32];
  double* base = V + b * q * ldv + n;
  for (int k = 0; k < q; ++k) v[k] = base[(int64_t)k * ldv];
  for (int j = 0; j < q; ++j) {
    double acc = 0.0;
    for (int k = 0; k < q; ++k) acc = fma(sb[j * q + k], v[k], acc);
    base[(int64_t)j * ldv] = acc;
  }
}

// grad[t][d] += 2 sum_{k != j} Sigma_bar[b][j][k] dk(x_j, x_k)/dx_j,d (the K(x_b, x_b) term of the joint covariance);
// one thread per query point
template <int KIND>
__global__ void __launch_bounds__(128)
qei_cross_kernel(const double* __restrict__ Xc, const double* __restrict__ inv_ls, int D, int64_t npts, int q,
                 const double* __restrict__ sbar, double variance, double* __restrict__ grad) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= npts) return;
  const int64_t b = t / q;
  const int j = (int)(t % q);
  double g[32];
  for (int d = 0; d < D; ++d) g[d] = 0.0;
  for (int k = 0; k < q; ++k) {
    if (k == j) continue;
    double r2 = 0.0;
    for (int d = 0; d < D; ++d) {
      const double df = (Xc[t * D + d] - Xc[(b * q + k) * D + d]) * inv_ls[d];
      r2 = fma(df, df, r2);
    }
    const double w = 4.0 * sbar[b * q * q + j * q + k] * kernel_dr2<KIND>(r2, variance);
    for (int d = 0; d < D; ++d) g[d] = fma(w, (Xc[t * D + d] - Xc[(b * q + k) * D + d]) * inv_ls[d] * inv_ls[d], g[d]);
  }
  for (int d = 0; d < D; ++d) grad[t * D + d] += g[d];
}

// ------------------------------------------------------------------------------------------------
// K1g: gradient assembly.  grad[t][d] = sum_k dk/dr2(k,t) * 2 (x~_t,d - x~_k,d) / l_d *
//                                       (c_mu[t] alpha[k] - 2 c_var[t] V[k,t])
//   with V = K^-1 k* = Linv^T (Linv k*) (plain layout [t][ldv]).  WPC warps per candidate: 1 (one warp walks all N training
//   rows) or 8 (the CTA's warps take interleaved 32-row slices and are summed in warp order through shared memory — small
//   batches, e.g. the late rounds of the multi-start optimiser, where one warp per candidate leaves most SMs idle).
// ------------------------------------------------------------------------------------------------
template <int KIND, int DP, int WPC>
__global__ void __launch_bounds__(256)
grad_kernel(const double* __restrict__ Xs, const double* __restrict__ alpha, const double* __restrict__ Xc,
            const double* __restrict__ inv_ls, int N, int D, int64_t Mc, const double* __restrict__ Vplain,
            int64_t ldv, const double* __restrict__ cmu, const double* __restrict__ cvar, double variance,
            const __grid_constant__ fm::Consts fc, double* __restrict__ grad) {
  static_assert(WPC == 1 || WPC == 8, "one warp or one CTA per candidate");
  __shared__ double exp_tab[64];  // 2^(j/64) for the branch-free exp of fastmath.cuh
  __shared__ double red[WPC == 8 ? 8 * DP : 1];
  if (threadIdx.x < 64) exp_tab[threadIdx.x] = fm::EXP2_TABLE_DEV[threadIdx.x];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t t = WPC == 8 ? (int64_t)blockIdx.x : (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
  if (t >= Mc) return;  // WPC == 8: the whole CTA returns together
  double xc[DP], g[DP];
#pragma unroll
  for (int d = 0; d < DP; ++d) {
    xc[d] = (d < D) ? Xc[t * D + d] * inv_ls[d] : 0.0;
    g[d] = 0.0;
  }
  const double cm = cmu[t], cv = -2.0 * cvar[t];
  const double* v = Vplain + t * ldv;
  for (int k = (WPC == 8 ? warp * 32 : 0) + lane; k < N; k += 32 * WPC) {
    const double* xr = Xs + (int64_t)k * DP;
    double diff[DP], r2 = 0.0;
#pragma unroll
    for (int d = 0; d < DP; d += 2) {
      double2 xv = __ldg(reinterpret_cast<const double2*>(xr + d));
      diff[d] = xc[d] - xv.x;
      diff[d + 1] = xc[d + 1] - xv.y;
      r2 = fma(diff[d], diff[d], r2);
      r2 = fma(diff[d + 1], diff[d + 1], r2);
    }
    const double w = 2.0 * kernel_dr2_fast<KIND>(r2, variance, exp_tab, fc) * fma(cm, __ldg(alpha + k), cv * v[k]);
#pragma unroll
    for (int d = 0; d < DP; ++d) g[d] = fma(w, diff[d], g[d]);
  }
#pragma unroll
  for (int d = 0; d < DP; ++d) {
    double s = g[d];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (WPC == 8) {
      if (lane == 0) red[warp * DP + d] = s;
    } else if (lane == 0 && d < D) {
      grad[t * D + d] = s * inv_ls[d];
    }
  }
  if (WPC == 8) {
    __syncthreads();
    if (threadIdx.x < D) {
      double s = 0.0;
#pragma unroll
      for (int w = 0; w < 8; ++w) s += red[w * DP + threadIdx.x];
      grad[t * D + threadIdx.x] = s * inv_ls[threadIdx.x];
    }
  }
}

// ------------------------------------------------------------------------------------------------
// K1h: posterior mean and its gradient, no variance.  mean[t] = sum_k k(x_t, x_k) alpha[k] + m,
//   grad[t][d] = sum_k dk/dr2(k,t) * 2 (x~_t,d - x~_k,d) / l_d * alpha[k].  One warp per point walks all N training rows
//   (the single pass over Xs and alpha of grad_kernel<..., 1>, without V).
// ------------------------------------------------------------------------------------------------
template <int KIND, int DP>
__global__ void __launch_bounds__(256, 1)  // minimum of one CTA per SM: lets ptxas keep every DP in registers
mean_grad_kernel(const double* __restrict__ Xs, const double* __restrict__ alpha, const double* __restrict__ Xc,
                 const double* __restrict__ inv_ls, int N, int D, int64_t M, double variance, double mean_const,
                 double* __restrict__ mean, double* __restrict__ grad) {
  const int lane = threadIdx.x & 31;
  const int64_t t = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (t >= M) return;
  double xc[DP], g[DP];
#pragma unroll
  for (int d = 0; d < DP; ++d) {
    xc[d] = (d < D) ? Xc[t * D + d] * inv_ls[d] : 0.0;
    g[d] = 0.0;
  }
  double macc = 0.0;
  for (int k = lane; k < N; k += 32) {
    const double* xr = Xs + (int64_t)k * DP;
    double diff[DP], r2 = 0.0;
#pragma unroll
    for (int d = 0; d < DP; d += 2) {
      double2 xv = __ldg(reinterpret_cast<const double2*>(xr + d));
      diff[d] = xc[d] - xv.x;
      diff[d + 1] = xc[d + 1] - xv.y;
      r2 = fma(diff[d], diff[d], r2);
      r2 = fma(diff[d + 1], diff[d + 1], r2);
    }
    const double a = __ldg(alpha + k);
    macc = fma(kernel_from_r2<KIND>(r2, variance), a, macc);
    const double w = 2.0 * kernel_dr2<KIND>(r2, variance) * a;
#pragma unroll
    for (int d = 0; d < DP; ++d) g[d] = fma(w, diff[d], g[d]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) macc += __shfl_xor_sync(0xffffffffu, macc, o);
  if (lane == 0) mean[t] = macc + mean_const;
#pragma unroll
  for (int d = 0; d < DP; ++d) {
    double s = g[d];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0 && d < D) grad[t * D + d] = s * inv_ls[d];
  }
}

// ------------------------------------------------------------------------------------------------
// K1i: GIBBON's cross term (entropy.py:580-618).  For the m pending points P (scaled coordinates Ps [m][DP]):
//   c_j(x) = k(x, p_j) - sum_n k(x, x_n) W_nj,  W = K^-1 k(X, P)          (covariance_between_points, unclipped)
//   u = L_B^-1 c(x),  |u|^2,  L_B = chol(B + noise I)
// computed as u_i = sum_{j<=i} Linv_B[i][j] k(x, p_j) - sum_n k(x, x_n) What[n][i], What = W L_B^-T (built once per pending
// set and posterior cache).  One thread per candidate; the pending set is walked in register tiles of GIB_TILE rows of u, each
// one pass over the training rows (warp-uniform loads of Xs and What rows: broadcast through L1), so m has no upper bound.
// U (nullable, [mp][Mc]): u itself, for the gradient.
// ------------------------------------------------------------------------------------------------
constexpr int GIB_TILE = 16;

template <int KIND, int DP>
__global__ void __launch_bounds__(128, 4)  // up to 128 registers: every DP keeps xc and the tile of u in registers
gibbon_cross_kernel(const double* __restrict__ Xs, const double* __restrict__ What, const double* __restrict__ Ps,
                    const double* __restrict__ LBinv, const double* __restrict__ Xc, const double* __restrict__ inv_ls, int N,
                    int D, int m, int mp, int64_t Mc, double variance, const __grid_constant__ fm::Consts fc,
                    double* __restrict__ uu_out, double* __restrict__ U) {
  __shared__ double exp_tab[64];  // 2^(j/64) for the branch-free exp of fastmath.cuh (as the K* generation kernels)
  if (threadIdx.x < 64) exp_tab[threadIdx.x] = fm::EXP2_TABLE_DEV[threadIdx.x];
  __syncthreads();
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= Mc) return;
  double xc[DP];
#pragma unroll
  for (int d = 0; d < DP; ++d) xc[d] = (d < D) ? Xc[t * D + d] * inv_ls[d] : 0.0;
  double uu = 0.0;
  for (int i0 = 0; i0 < mp; i0 += GIB_TILE) {
    double acc[GIB_TILE];
#pragma unroll
    for (int i = 0; i < GIB_TILE; ++i) acc[i] = 0.0;
    const int jend = min(m, i0 + GIB_TILE);  // Linv_B is lower triangular
    for (int j = 0; j < jend; ++j) {
      const double* pr = Ps + (int64_t)j * DP;
      double r2 = 0.0;
#pragma unroll
      for (int d = 0; d < DP; d += 2) {
        const double2 pv = __ldg(reinterpret_cast<const double2*>(pr + d));
        const double a = xc[d] - pv.x, b = xc[d + 1] - pv.y;
        r2 = fma(a, a, r2);
        r2 = fma(b, b, r2);
      }
      const double kj = kernel_from_r2_fast<KIND>(r2, variance, exp_tab, fc);
      const double* lr = LBinv + (int64_t)i0 * m + j;
#pragma unroll
      for (int i = 0; i < GIB_TILE; ++i) acc[i] = fma(__ldg(lr + (int64_t)i * m), kj, acc[i]);
    }
    for (int n = 0; n < N; ++n) {
      const double* xr = Xs + (int64_t)n * DP;
      double r2 = 0.0;
#pragma unroll
      for (int d = 0; d < DP; d += 2) {
        const double2 xv = __ldg(reinterpret_cast<const double2*>(xr + d));
        const double a = xc[d] - xv.x, b = xc[d + 1] - xv.y;
        r2 = fma(a, a, r2);
        r2 = fma(b, b, r2);
      }
      const double kn = -kernel_from_r2_fast<KIND>(r2, variance, exp_tab, fc);
      const double* wr = What + (int64_t)n * mp + i0;
#pragma unroll
      for (int i = 0; i < GIB_TILE; i += 2) {
        const double2 w = __ldg(reinterpret_cast<const double2*>(wr + i));
        acc[i] = fma(kn, w.x, acc[i]);
        acc[i + 1] = fma(kn, w.y, acc[i + 1]);
      }
    }
#pragma unroll
    for (int i = 0; i < GIB_TILE; ++i) {
      uu = fma(acc[i], acc[i], uu);
      if (U) U[(int64_t)(i0 + i) * Mc + t] = acc[i];
    }
  }
  uu_out[t] = uu;
}

// grad[t] += coef[t] (sum_j s_j dk(x, p_j)/dx - sum_n (What u)_n dk(x, x_n)/dx),  s = L_B^-T u,  coef = -w / V_det:
// the |u|^2 part of the repulsion gradient, d|u|^2/dx = 2 u^T du/dx.  One warp per candidate, one pass over the training rows.
template <int KIND, int DP>
__global__ void __launch_bounds__(256, 1)
gibbon_grad_kernel(const double* __restrict__ Xs, const double* __restrict__ What, const double* __restrict__ Ps,
                   const double* __restrict__ LBinv, const double* __restrict__ Xc, const double* __restrict__ inv_ls, int N,
                   int D, int m, int mp, int64_t Mc, double variance, const double* __restrict__ U,
                   const double* __restrict__ coef, double* __restrict__ grad) {
  const int lane = threadIdx.x & 31;
  const int64_t t = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (t >= Mc) return;
  double xc[DP], g[DP];
#pragma unroll
  for (int d = 0; d < DP; ++d) {
    xc[d] = (d < D) ? Xc[t * D + d] * inv_ls[d] : 0.0;
    g[d] = 0.0;
  }
  const double* u = U + t;  // u_i = u[i * Mc]
  for (int k = lane; k < N; k += 32) {
    const double* xr = Xs + (int64_t)k * DP;
    double diff[DP], r2 = 0.0;
#pragma unroll
    for (int d = 0; d < DP; d += 2) {
      const double2 xv = __ldg(reinterpret_cast<const double2*>(xr + d));
      diff[d] = xc[d] - xv.x;
      diff[d + 1] = xc[d + 1] - xv.y;
      r2 = fma(diff[d], diff[d], r2);
      r2 = fma(diff[d + 1], diff[d + 1], r2);
    }
    const double* wr = What + (int64_t)k * mp;
    double wu = 0.0;
    for (int i = 0; i < m; ++i) wu = fma(__ldg(wr + i), u[(int64_t)i * Mc], wu);
    const double w = -2.0 * kernel_dr2<KIND>(r2, variance) * wu;
#pragma unroll
    for (int d = 0; d < DP; ++d) g[d] = fma(w, diff[d], g[d]);
  }
  for (int j = lane; j < m; j += 32) {
    double s = 0.0;
    for (int i = j; i < m; ++i) s = fma(__ldg(LBinv + (int64_t)i * m + j), u[(int64_t)i * Mc], s);
    const double* pr = Ps + (int64_t)j * DP;
    double diff[DP], r2 = 0.0;
#pragma unroll
    for (int d = 0; d < DP; ++d) {
      diff[d] = xc[d] - __ldg(pr + d);
      r2 = fma(diff[d], diff[d], r2);
    }
    const double w = 2.0 * kernel_dr2<KIND>(r2, variance) * s;
#pragma unroll
    for (int d = 0; d < DP; ++d) g[d] = fma(w, diff[d], g[d]);
  }
  const double c = coef[t];
#pragma unroll
  for (int d = 0; d < DP; ++d) {
    double s = g[d];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0 && d < D) grad[t * D + d] = fma(c, s * inv_ls[d], grad[t * D + d]);
  }
}

// k(X, P) as m columns of length N (Kxp[j * N + n])
template <int KIND>
__global__ void __launch_bounds__(128)
gibbon_kxp_kernel(const double* __restrict__ Xs, const double* __restrict__ Ps, int N, int DP, double variance,
                  double* __restrict__ Kxp) {
  const int n = blockIdx.x * 128 + threadIdx.x;
  const int j = blockIdx.y;
  if (n >= N) return;
  double r2 = 0.0;
  for (int d = 0; d < DP; ++d) {
    const double df = Xs[(int64_t)n * DP + d] - Ps[(int64_t)j * DP + d];
    r2 = fma(df, df, r2);
  }
  Kxp[(int64_t)j * N + n] = kernel_from_r2<KIND>(r2, variance);
}

// B = k(P, P) - Y^T Y, Y = Linv k(X, P) (columns of length N): the posterior covariance of the pending points; one block per entry
template <int KIND>
__global__ void __launch_bounds__(256)
gibbon_pcov_kernel(const double* __restrict__ Ps, const double* __restrict__ Y, int N, int DP, int m, double variance,
                   double* __restrict__ B) {
  const int i = blockIdx.x, j = blockIdx.y;
  const double* yi = Y + (int64_t)i * N;
  const double* yj = Y + (int64_t)j * N;
  double acc = 0.0;
  for (int n = threadIdx.x; n < N; n += blockDim.x) acc = fma(yi[n], yj[n], acc);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  __shared__ double red[8];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w];
    double r2 = 0.0;
    for (int d = 0; d < DP; ++d) {
      const double df = Ps[(int64_t)i * DP + d] - Ps[(int64_t)j * DP + d];
      r2 = fma(df, df, r2);
    }
    B[(int64_t)i * m + j] = kernel_from_r2<KIND>(r2, variance) - s;
  }
}

// What[n][i] = sum_{j<=i} W[j][n] Linv_B[i][j] for i < m, 0 for m <= i < mp  (W columns of length N)
__global__ void __launch_bounds__(128)
gibbon_what_kernel(const double* __restrict__ W, const double* __restrict__ LBinv, int N, int m, int mp,
                   double* __restrict__ What) {
  const int n = blockIdx.x * 128 + threadIdx.x;
  const int i = blockIdx.y;
  if (n >= N) return;
  double acc = 0.0;
  if (i < m)
    for (int j = 0; j <= i; ++j) acc = fma(W[(int64_t)j * N + n], LBinv[(int64_t)i * m + j], acc);
  What[(int64_t)n * mp + i] = acc;
}

// per-candidate partial derivatives of the acquisition w.r.t. (mean, var) from the tail inputs
__global__ void __launch_bounds__(256)
acq_partials_kernel(const double* __restrict__ partial, int G, int64_t McPad, const double* __restrict__ mean,
                    int64_t Mc, double variance, int acq, double param, double aux, const double* __restrict__ samp, int nsamp,
                    double* __restrict__ cmu,
                    double* __restrict__ cvar, const double* __restrict__ gib_uu = nullptr, double gib_w = 0.0,
                    double* __restrict__ gib_coef = nullptr) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= Mc) return;
  const double raw = chunk_raw_variance(partial, G, McPad, t, variance);
  const bool clipped = raw < 1e-12;
  double dm, dv;
  if (acq == TB_ACQ_MES) {
    mes_partials(samp, nsamp, mean[t], fmax(raw, 1e-12), clipped, dm, dv);
  } else if (active_learning_kind(acq)) {
    active_learning_partials(acq, param, aux, mean[t], fmax(raw, 1e-12), clipped, dm, dv);
  } else if (gibbon_kind(acq)) {
    const double var = fmax(raw, 1e-12);
    dm = 0.0;
    dv = 0.0;
    if (acq != TB_ACQ_GIBBON_REPULSION) gibbon_quality_partials(samp, nsamp, mean[t], var, aux, clipped, dm, dv);
    if (acq != TB_ACQ_GIBBON_QUALITY) {
      // repulsion w/2 (log V_det - log yvar), V_det = yvar - |u|^2: its var part enters through cvar; the |u|^2 part is
      // -w / V_det times d|u|^2/dx / 2, added by gibbon_grad_kernel
      const double yvar = var + aux, vdet = yvar - gib_uu[t];
      if (!clipped) dv += gib_w * 0.5 * (1.0 / vdet - 1.0 / yvar);
      gib_coef[t] = -gib_w / vdet;
    }
  } else {
    acq_partials(acq, param, aux, mean[t], fmax(raw, 1e-12), clipped, dm, dv);
  }
  cmu[t] = dm;
  cvar[t] = dv;
}

// ------------------------------------------------------------------------------------------------
// K3: RFF trajectory evaluation  f_b(x) = sum_f theta[b,f] * sqrt(2 var / F) cos(W_f . x/l + b_f) + m
//   (sampler.py:901-936; gpflux RandomFourierFeaturesCosine).  One thread per candidate, features
//   streamed through shared memory in chunks; fused per-trajectory argmin (acquisition/sampler.py:269).
// ------------------------------------------------------------------------------------------------
constexpr int RFF_THREADS = 256;
constexpr int RFF_FCHUNK = 512;

template <int DP, int NBT>
__global__ void __launch_bounds__(RFF_THREADS)
rff_eval_kernel(const double* __restrict__ Wp,     // [F][DP] (zero padded)
                const double* __restrict__ bias,   // [F]
                const double* __restrict__ theta,  // [nb][F]
                const double* __restrict__ Xc, const double* __restrict__ inv_ls, int D, int F, int nb,
                int b0, int64_t M, int64_t idx0, double scale, double mean_const, const double* __restrict__ addend,
                const __grid_constant__ fm::TrigConsts tc, double* __restrict__ out, double* __restrict__ blk_best,
                int64_t* __restrict__ blk_idx) {
  extern __shared__ __align__(16) unsigned char rsm[];
  double* sW = reinterpret_cast<double*>(rsm);   // [RFF_FCHUNK][DP]
  double* sb = sW + RFF_FCHUNK * DP;             // [RFF_FCHUNK]
  double* sth = sb + RFF_FCHUNK;                 // [NBT][RFF_FCHUNK]
  const int64_t t = (int64_t)blockIdx.x * RFF_THREADS + threadIdx.x;
  const bool valid = t < M;
  double x[DP];
#pragma unroll
  for (int d = 0; d < DP; ++d) x[d] = (valid && d < D) ? Xc[t * D + d] * inv_ls[d] : 0.0;
  double acc[NBT];
#pragma unroll
  for (int b = 0; b < NBT; ++b) acc[b] = 0.0;
  for (int f0 = 0; f0 < F; f0 += RFF_FCHUNK) {
    const int fc = min(RFF_FCHUNK, F - f0);
    __syncthreads();
    for (int e = threadIdx.x; e < fc * DP; e += RFF_THREADS) sW[e] = Wp[(int64_t)f0 * DP + e];
    for (int e = threadIdx.x; e < fc; e += RFF_THREADS) sb[e] = bias[f0 + e];
    for (int e = threadIdx.x; e < fc * NBT; e += RFF_THREADS) {
      int b = e / fc, f = e % fc;
      sth[b * RFF_FCHUNK + f] = (b0 + b < nb) ? theta[(int64_t)(b0 + b) * F + f0 + f] : 0.0;
    }
    __syncthreads();
    for (int f = 0; f < fc; ++f) {
      double a = sb[f];
#pragma unroll
      for (int d = 0; d < DP; d += 2) {
        double2 w = *reinterpret_cast<const double2*>(sW + f * DP + d);
        a = fma(w.x, x[d], a);
        a = fma(w.y, x[d + 1], a);
      }
      const double c = fm::cos_fast(a, tc);  // branch-free, constants from the constant bank (fastmath.cuh)
#pragma unroll
      for (int b = 0; b < NBT; ++b) acc[b] = fma(sth[b * RFF_FCHUNK + f], c, acc[b]);
    }
  }
  __shared__ double sv[RFF_THREADS / 32];
  __shared__ int64_t si[RFF_THREADS / 32];
#pragma unroll
  for (int b = 0; b < NBT; ++b) {
    if (b0 + b >= nb) break;
    double v = fma(acc[b], scale, mean_const);
    if (valid && addend) v += addend[t * nb + b0 + b];  // canonical (pathwise-update) part of a decoupled trajectory
    if (valid && out) out[t * nb + b0 + b] = v;
    if (blk_best) {
      double bv = valid ? -v : -DBL_MAX;  // argmin == first-max of the negated trajectory
      int64_t bi = valid ? idx0 + t : INT64_MAX;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        double v2 = __shfl_xor_sync(0xffffffffu, bv, o);
        int64_t i2 = __shfl_xor_sync(0xffffffffu, bi, o);
        best_merge(bv, bi, v2, i2);
      }
      __syncthreads();
      if ((threadIdx.x & 31) == 0) {
        sv[threadIdx.x >> 5] = bv;
        si[threadIdx.x >> 5] = bi;
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        for (int w = 1; w < RFF_THREADS / 32; ++w) best_merge(bv, bi, sv[w], si[w]);
        blk_best[(int64_t)(b0 + b) * gridDim.x + blockIdx.x] = bv;
        blk_idx[(int64_t)(b0 + b) * gridDim.x + blockIdx.x] = bi;
      }
    }
  }
}

// canonical part of a decoupled trajectory (sampler.py:809-855): out[t][b] = sum_j v[b][j] k(x_t, x_j).
// One thread per candidate; the training rows and weights are warp-uniform loads.
template <int KIND, int DP, int NBT>
__global__ void __launch_bounds__(256)
kdot_kernel(const double* __restrict__ Xs, const double* __restrict__ V, int64_t ldv, const double* __restrict__ Xc,
            const double* __restrict__ inv_ls, int N, int D, int nb, int b0, int64_t M, double variance,
            const __grid_constant__ fm::Consts fc, double* __restrict__ out) {
  __shared__ double exp_tab[64];
  if (threadIdx.x < 64) exp_tab[threadIdx.x] = fm::EXP2_TABLE_DEV[threadIdx.x];
  __syncthreads();
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool valid = t < M;
  double x[DP], acc[NBT];
#pragma unroll
  for (int d = 0; d < DP; ++d) x[d] = (valid && d < D) ? Xc[t * D + d] * inv_ls[d] : 0.0;
#pragma unroll
  for (int b = 0; b < NBT; ++b) acc[b] = 0.0;
  for (int k = 0; k < N; ++k) {
    const double* xr = Xs + (int64_t)k * DP;
    double r2 = 0.0;
#pragma unroll
    for (int d = 0; d < DP; d += 2) {
      const double2 xv = __ldg(reinterpret_cast<const double2*>(xr + d));
      const double d0 = x[d] - xv.x, d1 = x[d + 1] - xv.y;
      r2 = fma(d0, d0, r2);
      r2 = fma(d1, d1, r2);
    }
    const double kv = kernel_from_r2_fast<KIND>(r2, variance, exp_tab, fc);
#pragma unroll
    for (int b = 0; b < NBT; ++b)
      if (b0 + b < nb) acc[b] = fma(kv, __ldg(V + (int64_t)(b0 + b) * ldv + k), acc[b]);
  }
  if (valid) {
#pragma unroll
    for (int b = 0; b < NBT; ++b)
      if (b0 + b < nb) out[t * nb + b0 + b] = acc[b];
  }
}

// K3b: paired trajectory evaluation: point t under its own trajectory b(t) = (pidx ? pidx[t] : idx0 + t) % nb only, times sgn (+-1,
// exact), with the gradient when GRAD.  pidx carries the compacted problem indices of the device L-BFGS, idx0 + t the flat (m, b)
// index of an [M, B, D] input.  The value repeats rff_eval_kernel's feature order and fma sequence over the DP padded pairs, cos_fast,
// fma(acc, scale, mean), then adds kdot_kernel's canonical sum over j in ascending order, so it is bit for bit the per-column value.
//   grad_d = (-scale sum_f theta_bf sin(a_f) W_fd + sum_j v_bj 2 k'(r2_j) (x~_d - x~_jd)) / l_d
// Matern-12 at a coincident training point: r2 is clamped at 1e-36 as in mean_grad_kernel, and its zero difference makes the
// contribution zero.  One thread per point; W and the bias stream through shared memory, theta_b and v_b are per-lane loads (rows
// of arbitrary trajectories: L1 / L2 hits).  N = 0 (no canonical part): Xs and V are not read.
template <int KIND, int DP, bool GRAD>
__global__ void __launch_bounds__(RFF_THREADS, 1)  // minimum of one CTA per SM: without it ptxas spills at small DP
rff_paired_kernel(const double* __restrict__ Wp, const double* __restrict__ bias, const double* __restrict__ theta,
                  const double* __restrict__ Xs, const double* __restrict__ V, const double* __restrict__ Xc,
                  const double* __restrict__ inv_ls, int D, int F, int N, int nb, int64_t M, int64_t idx0,
                  const int* __restrict__ pidx, double scale, double mean_const, double variance, double sgn,
                  const __grid_constant__ fm::TrigConsts tc, const __grid_constant__ fm::Consts fc, double* __restrict__ out,
                  double* __restrict__ grad) {
  extern __shared__ __align__(16) unsigned char rsm[];
  double* sW = reinterpret_cast<double*>(rsm);  // [RFF_FCHUNK][DP]
  double* sb = sW + RFF_FCHUNK * DP;            // [RFF_FCHUNK]
  __shared__ double exp_tab[64];
  if (threadIdx.x < 64) exp_tab[threadIdx.x] = fm::EXP2_TABLE_DEV[threadIdx.x];
  const int64_t t = (int64_t)blockIdx.x * RFF_THREADS + threadIdx.x;
  const bool valid = t < M;
  const int b = valid ? (int)((pidx ? (int64_t)pidx[t] : idx0 + t) % nb) : 0;
  const double* th = theta + (int64_t)b * F;
  double x[DP], g[GRAD ? DP : 1];
#pragma unroll
  for (int d = 0; d < DP; ++d) x[d] = (valid && d < D) ? Xc[t * D + d] * inv_ls[d] : 0.0;
#pragma unroll
  for (int d = 0; d < (GRAD ? DP : 1); ++d) g[d] = 0.0;
  double acc = 0.0;
  for (int f0 = 0; f0 < F; f0 += RFF_FCHUNK) {
    const int fcn = min(RFF_FCHUNK, F - f0);
    __syncthreads();
    for (int e = threadIdx.x; e < fcn * DP; e += RFF_THREADS) sW[e] = Wp[(int64_t)f0 * DP + e];
    for (int e = threadIdx.x; e < fcn; e += RFF_THREADS) sb[e] = bias[f0 + e];
    __syncthreads();
    for (int f = 0; f < fcn; ++f) {
      double a = sb[f];
#pragma unroll
      for (int d = 0; d < DP; d += 2) {
        double2 w = *reinterpret_cast<const double2*>(sW + f * DP + d);
        a = fma(w.x, x[d], a);
        a = fma(w.y, x[d + 1], a);
      }
      const double tf = __ldg(th + f0 + f);
      if constexpr (GRAD) {
        double s;
        acc = fma(tf, fm::sincos_fast(a, tc, s), acc);
        const double ts = tf * s;
#pragma unroll
        for (int d = 0; d < DP; d += 2) {
          double2 w = *reinterpret_cast<const double2*>(sW + f * DP + d);
          g[d] = fma(ts, w.x, g[d]);
          g[d + 1] = fma(ts, w.y, g[d + 1]);
        }
      } else {
        acc = fma(tf, fm::cos_fast(a, tc), acc);
      }
    }
  }
  if (!valid) return;
  double v = fma(acc, scale, mean_const);
  if constexpr (GRAD) {
#pragma unroll
    for (int d = 0; d < DP; ++d) g[d] *= -scale;
  }
  if (N > 0) {
    const double* vb = V + (int64_t)b * N;
    double cacc = 0.0;
    for (int k = 0; k < N; ++k) {
      const double* xr = Xs + (int64_t)k * DP;
      double r2 = 0.0;
#pragma unroll
      for (int d = 0; d < DP; d += 2) {
        const double2 xv = __ldg(reinterpret_cast<const double2*>(xr + d));
        const double d0 = x[d] - xv.x, d1 = x[d + 1] - xv.y;
        r2 = fma(d0, d0, r2);
        r2 = fma(d1, d1, r2);
      }
      const double vk = __ldg(vb + k);
      cacc = fma(kernel_from_r2_fast<KIND>(r2, variance, exp_tab, fc), vk, cacc);
      if constexpr (GRAD) {
        const double w = 2.0 * kernel_dr2_fast<KIND>(r2, variance, exp_tab, fc) * vk;
#pragma unroll
        for (int d = 0; d < DP; d += 2) {
          const double2 xv = __ldg(reinterpret_cast<const double2*>(xr + d));
          g[d] = fma(w, x[d] - xv.x, g[d]);
          g[d + 1] = fma(w, x[d + 1] - xv.y, g[d + 1]);
        }
      }
    }
    v += cacc;
  }
  out[t] = sgn * v;
  if constexpr (GRAD) {
#pragma unroll
    for (int d = 0; d < DP; ++d)
      if (d < D) grad[t * D + d] = sgn * g[d] * inv_ls[d];
  }
}

// fold block winners per trajectory (grid.x = nb)
__global__ void __launch_bounds__(256)
rff_fold_kernel(const double* __restrict__ blk_best, const int64_t* __restrict__ blk_idx, int nblk,
                double* __restrict__ run_best, int64_t* __restrict__ run_idx) {
  const int b = blockIdx.x;
  double bv = -DBL_MAX;
  int64_t bi = INT64_MAX;
  for (int i = threadIdx.x; i < nblk; i += blockDim.x)
    best_merge(bv, bi, blk_best[(int64_t)b * nblk + i], blk_idx[(int64_t)b * nblk + i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    double v2 = __shfl_xor_sync(0xffffffffu, bv, o);
    int64_t i2 = __shfl_xor_sync(0xffffffffu, bi, o);
    best_merge(bv, bi, v2, i2);
  }
  __shared__ double sv[8];
  __shared__ int64_t si[8];
  if ((threadIdx.x & 31) == 0) {
    sv[threadIdx.x >> 5] = bv;
    si[threadIdx.x >> 5] = bi;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w) best_merge(bv, bi, sv[w], si[w]);
    double rv = run_best[b];
    int64_t ri = run_idx[b];
    best_merge(rv, ri, bv, bi);
    run_best[b] = rv;
    run_idx[b] = ri;
  }
}

// ------------------------------------------------------------------------------------------------
// K4: top-k by bitonic sort of (value, index) pairs, order = (value descending, index ascending)
//   = tf.math.top_k as used by generate_initial_points (optimizer.py:321-335).
// ------------------------------------------------------------------------------------------------
struct VI {
  double v;
  int64_t i;
};
__device__ __forceinline__ bool vi_before(const VI& a, const VI& b) {  // a sorts before b
  return a.v > b.v || (a.v == b.v && a.i < b.i);
}
constexpr int BIT_TILE = 2048;  // elements sorted per CTA in shared memory (1024 threads)

__global__ void topk_init_kernel(const double* __restrict__ vals, int64_t M, int64_t P, VI* __restrict__ a) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  VI e;
  if (i < M) {
    double v = vals[i];
    e.v = (v == v) ? v : -DBL_MAX;  // NaN sorts last
    e.i = i;
  } else {
    e.v = -DBL_MAX;
    e.i = INT64_MAX;
  }
  a[i] = e;
}
// all (k, j) stages with k <= BIT_TILE for a fresh array, or the j < BIT_TILE tail of a larger k
__global__ void __launch_bounds__(1024)
bitonic_local_kernel(VI* __restrict__ a, int64_t kstart, int64_t kend) {
  __shared__ VI s[BIT_TILE];
  const int64_t base = (int64_t)blockIdx.x * BIT_TILE;
  for (int e = threadIdx.x; e < BIT_TILE; e += 1024) s[e] = a[base + e];
  __syncthreads();
  for (int64_t k = kstart; k <= kend; k <<= 1) {
    for (int64_t j = (k > BIT_TILE ? BIT_TILE : k) >> 1; j > 0; j >>= 1) {
      for (int e = threadIdx.x; e < BIT_TILE / 2; e += 1024) {
        int lo = (int)((e / j) * 2 * j + (e % j));
        int hi = lo + (int)j;
        bool up = (((base + lo) & k) == 0);  // ascending-in-order block
        VI x = s[lo], y = s[hi];
        bool swap = up ? vi_before(y, x) : vi_before(x, y);
        if (swap) {
          s[lo] = y;
          s[hi] = x;
        }
      }
      __syncthreads();
    }
  }
  for (int e = threadIdx.x; e < BIT_TILE; e += 1024) a[base + e] = s[e];
}
__global__ void bitonic_global_kernel(VI* __restrict__ a, int64_t P, int64_t k, int64_t j) {
  int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= P / 2) return;
  int64_t lo = (e / j) * 2 * j + (e % j), hi = lo + j;
  bool up = ((lo & k) == 0);
  VI x = a[lo], y = a[hi];
  bool swap = up ? vi_before(y, x) : vi_before(x, y);
  if (swap) {
    a[lo] = y;
    a[hi] = x;
  }
}
__global__ void topk_emit_kernel(const VI* __restrict__ a, int k, double* __restrict__ tv, int64_t* __restrict__ ti) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < k) {
    tv[i] = a[i].v;
    ti[i] = a[i].i;
  }
}

}  // namespace tb
