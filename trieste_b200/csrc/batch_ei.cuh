// Batch expected improvement of Chevalier & Ginsbourger (trieste 4.2.1 acquisition/function/function.py:1281-1805) with
// its multivariate-normal CDFs by Genz's QMC recursion (acquisition/function/utils.py:29-199), and the reverse pass.
//
// For one q-batch in the maximisation form (mu = -mean, T = -eta, C = cov + 1e-6 I):
//   Sigma^(k)[a][b] = C_ab [a!=k][b!=k] - C_ak [a!=k] - C_kb [b!=k] + C_kk           (function.py:1413-1424)
//   d^(k)_j         = b^(k)_j - m^(k)_j = mu_k - mu_j (j != k),  mu_k - T (j == k)     (:1343-1352, :1480)
//   p_k             = Phi_q(d^(k); Sigma^(k))                                           (:1476-1490)
//   c^(k,i)_j       = d_j - d_i Sigma_ij / Sigma_ii                      (j != i)       (:1520-1532)
//   R^(k,i)_uv      = Sigma_uv - Sigma_iu Sigma_iv / Sigma_ii            (u, v != i)    (:1554-1587)
//   ei = sum_k (mu_k - T) p_k + sum_{k,i} Sigma^(k)_ik N(d_i; 0, Sigma^(k)_ii) Phi_{q-1}(c^(k,i); R^(k,i))   (:1724-1743)
// Every CDF factorises its matrix + 1e-6 I (the CDF's default jitter, utils.py:114, 143-144).  The q + q^2 CDFs of a batch
// are its "units": unit u < q is p_u, unit u >= q is (k, i) = ((u - q) / q, (u - q) % q).  One CTA per batch; its warps
// take the units round-robin, build the unit's matrix from the q x q covariance in shared memory, factorise it once and
// spread the S Sobol samples over the lanes.  Nothing of size q^3 or q^4 reaches global memory.
//
// Determinism: every lane sums its own samples in a fixed order and a xor-shuffle tree combines the lanes; unit values
// are summed in unit order; in the reverse pass every adjoint entry has one owning lane (no atomics).
#pragma once
#include "kernels_extra.cuh"

namespace tb {

constexpr double GENZ_CLAMP = 1e-6;    // utils.py:177: y = Phi^-1(1e-6 + (1 - 2e-6) w e)
constexpr double GENZ_PIVOT = 1e-12;   // utils.py:168, 183: added to every pivot of the factor
constexpr double BEI_JITTER = 1e-6;    // function.py:1776-1783 and the CDF's jitter (utils.py:114); hard-coded there too
constexpr int BEI_MAX_WARPS = 4;

__device__ __forceinline__ double std_normal_pdf(double z) { return 0.3989422804014327 * exp(-0.5 * z * z); }

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Genz's estimate of P(X <= b), X ~ N(0, L L^T): L the lower factor (n x n, row-major) and b [n] in shared memory, w
// [n-1][S] the Sobol points column-contiguous (column j is the same sequence in every dimension, so one array serves
// the dimension-q and the dimension-(q-1) CDFs).  ys [n][32] is per-lane scratch.  The mean over the S samples is
// returned on every lane.
__device__ double genz_cdf_warp(const double* L, const double* b, int n, const double* __restrict__ w, int S, double* ys,
                                int lane) {
  const double e0 = normcdf(b[0] / (L[0] + GENZ_PIVOT));
  double acc = 0.0;
  for (int s = lane; s < S; s += 32) {
    double e = e0, f = e0;
    for (int i = 1; i < n; ++i) {
      const double y = normcdfinv(GENZ_CLAMP + (1.0 - 2.0 * GENZ_CLAMP) * __ldg(w + (int64_t)(i - 1) * S + s) * e);
      ys[(i - 1) * 32 + lane] = y;
      double t = 0.0;
      for (int k = 0; k < i; ++k) t = fma(L[i * n + k], ys[k * 32 + lane], t);
      e = normcdf((b[i] - t) / (L[i * n + i] + GENZ_PIVOT));
      f *= e;
    }
    acc += f;
  }
  return warp_sum(acc) / (double)S;
}

// Reverse of genz_cdf_warp for the seed gbar on its result (what TensorFlow differentiates through the recursion).  On
// exit Lb holds the adjoint of the lower triangle of L and bb the adjoint of b.  Per lane and sample the forward values
// are kept in st = [z | e | y | prefix | ybar], each [n][32]; df/de_i is prefix_i * suffix_i (never f / e_i: e_i can be
// 0).  The sums over samples are taken per round of 32 samples, each adjoint entry by one lane in lane order.  Returns
// the forward value, bit-identical to genz_cdf_warp's.
__device__ double genz_cdf_backward_warp(const double* L, const double* b, int n, const double* __restrict__ w, int S,
                                         double gbar, double* Lb, double* bb, double* st, int lane) {
  double* zs = st;             // z_i, then zbar_i after the reverse sweep
  double* es = zs + n * 32;    // e_i, then zbar_i z_i
  double* ys = es + n * 32;    // y_i (i < n - 1)
  double* ps = ys + n * 32;    // prod_{j<i} e_j
  double* yb = ps + n * 32;    // ybar_i
  for (int e = lane; e < n * n; e += 32) Lb[e] = 0.0;
  for (int i = lane; i < n; i += 32) bb[i] = 0.0;
  const double e0 = normcdf(b[0] / (L[0] + GENZ_PIVOT));
  const double seed = gbar / (double)S;
  double acc = 0.0;
  for (int s0 = 0; s0 < S; s0 += 32) {
    const int s = s0 + lane;
    const bool act = s < S;
    // forward, as genz_cdf_warp
    if (act) {
      double e = e0, f = e0;
      zs[lane] = b[0] / (L[0] + GENZ_PIVOT);
      es[lane] = e0;
      ps[lane] = 1.0;
      for (int i = 1; i < n; ++i) {
        const double y = normcdfinv(GENZ_CLAMP + (1.0 - 2.0 * GENZ_CLAMP) * __ldg(w + (int64_t)(i - 1) * S + s) * e);
        ys[(i - 1) * 32 + lane] = y;
        double t = 0.0;
        for (int k = 0; k < i; ++k) t = fma(L[i * n + k], ys[k * 32 + lane], t);
        const double z = (b[i] - t) / (L[i * n + i] + GENZ_PIVOT);
        e = normcdf(z);
        zs[i * 32 + lane] = z;
        es[i * 32 + lane] = e;
        ps[i * 32 + lane] = f;
        f *= e;
      }
      acc += f;
      // reverse
      for (int i = 0; i < n; ++i) yb[i * 32 + lane] = 0.0;
      double suf = 1.0;
      for (int i = n - 1; i >= 0; --i) {
        double eb = seed * ps[i * 32 + lane] * suf;
        if (i < n - 1) {
          const double y = ys[i * 32 + lane];
          eb = fma(yb[i * 32 + lane] * (1.0 - 2.0 * GENZ_CLAMP), __ldg(w + (int64_t)i * S + s) / std_normal_pdf(y), eb);
        }
        suf *= es[i * 32 + lane];
        const double z = zs[i * 32 + lane];
        const double zb = eb * std_normal_pdf(z);
        zs[i * 32 + lane] = zb;
        es[i * 32 + lane] = zb * z;
        const double r = zb / (L[i * n + i] + GENZ_PIVOT);
        for (int k = 0; k < i; ++k) yb[k * 32 + lane] = fma(-r, L[i * n + k], yb[k * 32 + lane]);
      }
    } else {
      for (int i = 0; i < n; ++i) zs[i * 32 + lane] = es[i * 32 + lane] = ys[i * 32 + lane] = 0.0;
    }
    __syncwarp();
    // sums over this round's samples: Lb[i][k] += sum zbar_i y_k (k < i), Lb[i][i] += sum zbar_i z_i, bb[i] += sum zbar_i
    for (int e = lane; e < n * n; e += 32) {
      const int i = e / n, k = e % n;
      if (k > i) continue;
      double v = 0.0;
      if (k == i) {
        for (int l = 0; l < 32; ++l) v += es[i * 32 + l];  // already zbar_i z_i
      } else {
        for (int l = 0; l < 32; ++l) v = fma(zs[i * 32 + l], ys[k * 32 + l], v);
      }
      Lb[e] += v;
    }
    for (int i = lane; i < n; i += 32) {
      double v = 0.0;
      for (int l = 0; l < 32; ++l) v += zs[i * 32 + l];
      bb[i] += v;
    }
    __syncwarp();
  }
  // z_i = (b_i - sum_k L_ik y_k) / (L_ii + 1e-12): dz/db_i = 1/l, dz/dL_ik = -y_k/l, dz/dL_ii = -z/l
  for (int e = lane; e < n * n; e += 32) {
    const int i = e / n, k = e % n;
    Lb[e] = (k <= i) ? -Lb[e] / (L[i * n + i] + GENZ_PIVOT) : 0.0;
  }
  for (int i = lane; i < n; i += 32) bb[i] /= (L[i * n + i] + GENZ_PIVOT);
  __syncwarp();
  return warp_sum(acc) / (double)S;
}

// ---- one batch's units ---------------------------------------------------------------------------------------------
__device__ __forceinline__ double bei_sigma(const double* C, int q, int k, int a, int b) {
  return (((a != k && b != k) ? C[a * q + b] : 0.0) - (a != k ? C[a * q + k] : 0.0) - (b != k ? C[k * q + b] : 0.0)) +
         C[k * q + k];
}
__device__ __forceinline__ double bei_diff(const double* mu, double T, int k, int j) {
  return j == k ? -T + mu[k] : -(mu[j] - mu[k]);
}

// Writes the unit's matrix (+ the CDF jitter) into M and its limits into bv; returns its dimension.
__device__ int bei_unit_setup(const double* C, const double* mu, double T, int q, int u, double* M, double* bv, int lane) {
  if (u < q) {
    const int k = u;
    for (int e = lane; e < q * q; e += 32) {
      const int a = e / q, c = e % q;
      M[e] = bei_sigma(C, q, k, a, c) + (a == c ? BEI_JITTER : 0.0);
    }
    for (int j = lane; j < q; j += 32) bv[j] = bei_diff(mu, T, k, j);
    __syncwarp();
    return q;
  }
  const int k = (u - q) / q, i = (u - q) % q, n = q - 1;
  const double sii = bei_sigma(C, q, k, i, i), di = bei_diff(mu, T, k, i);
  for (int e = lane; e < n * n; e += 32) {
    const int a = e / n, c = e % n;
    const int ua = a + (a >= i), uc = c + (c >= i);
    M[e] = bei_sigma(C, q, k, ua, uc) - bei_sigma(C, q, k, i, ua) * bei_sigma(C, q, k, i, uc) / sii +
           (a == c ? BEI_JITTER : 0.0);
  }
  for (int j = lane; j < n; j += 32) {
    const int uj = j + (j >= i);
    bv[j] = bei_diff(mu, T, k, uj) - di * (bei_sigma(C, q, k, i, uj) / sii);
  }
  __syncwarp();
  return n;
}

// The unit's term of ei given its CDF value g; for the (k, i) units also the Gaussian density factor.
__device__ __forceinline__ double bei_pdf(const double* C, const double* mu, double T, int q, int k, int i) {
  const double sii = bei_sigma(C, q, k, i, i), sd = sqrt(sii);
  return std_normal_pdf(bei_diff(mu, T, k, i) / sd) / sd;
}
__device__ __forceinline__ double bei_unit_term(const double* C, const double* mu, double T, int q, int u, double g) {
  if (u < q) return (mu[u] - T) * g;
  const int k = (u - q) / q, i = (u - q) % q;
  return bei_sigma(C, q, k, i, k) * bei_pdf(C, mu, T, q, k, i) * g;
}

// Stage one batch in the maximisation form: C = cov + 1e-6 I, mu = -mean.
__device__ __forceinline__ void bei_stage(const double* __restrict__ mean_in, const double* __restrict__ cov_in, int64_t b,
                                          int q, double* C, double* mu) {
  for (int e = threadIdx.x; e < q * q; e += blockDim.x) C[e] = cov_in[b * q * q + e] + ((e / q == e % q) ? BEI_JITTER : 0.0);
  for (int e = threadIdx.x; e < q; e += blockDim.x) mu[e] = -mean_in[b * q + e];
  __syncthreads();
}

// Shared memory of bei_kernel: CTA part C [q^2] | mu [q] | unit terms [q + q^2], then per warp M [q^2] | bv [q] | ys [32 q].
__host__ __device__ constexpr size_t bei_cta_doubles(int q) { return (size_t)q * q + q + q + (size_t)q * q; }
__host__ __device__ constexpr size_t bei_warp_doubles(int q) { return (size_t)q * q + q + 32 * (size_t)q; }

// K2b: batch EI of nb q-batches from their joint posterior (mean [nb,q], cov [nb,q,q], device) -> value [nb].
// eta is the minimisation threshold.  A unit whose matrix cannot be factorised sets err_flag.
__global__ void __launch_bounds__(BEI_MAX_WARPS * 32)
bei_kernel(const double* __restrict__ mean_in, const double* __restrict__ cov_in, int q, const double* __restrict__ w, int S,
           double eta, double* __restrict__ out_val, int* __restrict__ err_flag) {
  extern __shared__ __align__(16) unsigned char bsm[];
  const int64_t b = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  double* C = reinterpret_cast<double*>(bsm);
  double* mu = C + q * q;
  double* terms = mu + q;
  double* M = terms + q + q * q + (size_t)warp * bei_warp_doubles(q);
  double* bv = M + q * q;
  double* ys = bv + q;
  const double T = -eta;
  bei_stage(mean_in, cov_in, b, q, C, mu);
  for (int u = warp; u < q + q * q; u += nw) {
    const int n = bei_unit_setup(C, mu, T, q, u, M, bv, lane);
    double g = 0.0;
    if (warp_cholesky(M, n, lane)) {
      g = genz_cdf_warp(M, bv, n, w, S, ys, lane);
    } else if (lane == 0) {
      atomicExch(err_flag, 1);
    }
    if (lane == 0) terms[u] = bei_unit_term(C, mu, T, q, u, g);
    __syncwarp();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double v = 0.0;
    for (int u = 0; u < q + q * q; ++u) v += terms[u];
    out_val[b] = v;
  }
}

// Shared memory of bei_backward_kernel: CTA part as bei_kernel plus per-warp adjoint accumulators, then per warp
// L, Lb, T [n^2] | bv, bb [q] | st [5][32 q] | Sb [q^2] | db, rs, cs [q] | covbar [q^2] | mubar [q].
__host__ __device__ constexpr size_t bei_back_warp_doubles(int q) {
  return 3 * (size_t)q * q + 2 * q + 5 * 32 * (size_t)q + (size_t)q * q + 3 * q + (size_t)q * q + q;
}

// K2bg: reverse pass of bei_kernel — the contract of qei_backward_kernel: value, c_mu = d ei / d mean, c_var = 1 and
// Sigma_bar = sym(d ei / d cov) [q,q], from which qei_mix_kernel, grad_kernel and qei_cross_kernel assemble d ei / d x.
__global__ void __launch_bounds__(BEI_MAX_WARPS * 32)
bei_backward_kernel(const double* __restrict__ mean_in, const double* __restrict__ cov_in, int q, const double* __restrict__ w,
                    int S, double eta, double* __restrict__ out_val, double* __restrict__ cmu, double* __restrict__ cvar,
                    double* __restrict__ sbar, int* __restrict__ err_flag) {
  extern __shared__ __align__(16) unsigned char bsm[];
  const int64_t b = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const int qq = q * q;
  double* C = reinterpret_cast<double*>(bsm);
  double* mu = C + qq;
  double* terms = mu + q;
  double* base = terms + q + qq;
  double* L = base + (size_t)warp * bei_back_warp_doubles(q);
  double* Lb = L + qq;
  double* Ts = Lb + qq;
  double* bv = Ts + qq;
  double* bb = bv + q;
  double* st = bb + q;
  double* Sb = st + 5 * 32 * q;
  double* db = Sb + qq;
  double* rs = db + q;
  double* cs = rs + q;
  double* covb = cs + q;
  double* mub = covb + qq;
  const double T = -eta;
  bei_stage(mean_in, cov_in, b, q, C, mu);
  for (int e = lane; e < qq; e += 32) covb[e] = 0.0;
  for (int e = lane; e < q; e += 32) mub[e] = 0.0;
  __syncwarp();
  bool bad = false;
  for (int u = warp; u < q + qq; u += nw) {
    const int k = u < q ? u : (u - q) / q, i = u < q ? -1 : (u - q) % q;
    const int n = bei_unit_setup(C, mu, T, q, u, L, bv, lane);
    if (!warp_cholesky(L, n, lane)) {
      bad = true;
      if (lane == 0) terms[u] = 0.0;
      continue;
    }
    // seed of the CDF: d ei / d g
    double gbar, pdf = 0.0, sik = 0.0;
    if (u < q) {
      gbar = mu[k] - T;
    } else {
      pdf = bei_pdf(C, mu, T, q, k, i);
      sik = bei_sigma(C, q, k, i, k);
      gbar = sik * pdf;
    }
    const double g = genz_cdf_backward_warp(L, bv, n, w, S, gbar, Lb, bb, st, lane);
    if (lane == 0) terms[u] = bei_unit_term(C, mu, T, q, u, g);
    warp_cholesky_backward(L, Lb, Ts, n, lane);  // Lb: adjoint of the unit's matrix (symmetric)
    // adjoints of Sigma^(k) (Sb) and d^(k) (db)
    for (int e = lane; e < qq; e += 32) Sb[e] = 0.0;
    for (int e = lane; e < q; e += 32) db[e] = 0.0;
    __syncwarp();
    if (u < q) {
      for (int e = lane; e < qq; e += 32) Sb[e] = Lb[e];
      for (int e = lane; e < q; e += 32) db[e] = bb[e];
      if (lane == 0) mub[k] += g;
    } else {
      const double sii = bei_sigma(C, q, k, i, i), di = bei_diff(mu, T, k, i);
      // R_uv = S_uv - S_iu S_iv / S_ii and c_j = d_j - d_i S_ij / S_ii over u, v, j != i; lane = compressed index
      for (int a = lane; a < n; a += 32) {
        const int ua = a + (a >= i);
        const double sia = bei_sigma(C, q, k, i, ua);
        double rs_a = 0.0;
        for (int c = 0; c < n; ++c) {
          const int uc = c + (c >= i);
          Sb[ua * q + uc] = Lb[a * n + c];
          rs_a = fma(Lb[a * n + c], bei_sigma(C, q, k, i, uc), rs_a);
        }
        db[ua] = bb[a];
        // row i of Sigma^(k): from R (both factors, Lb symmetric) and from c
        Sb[i * q + ua] = -2.0 * rs_a / sii - bb[a] * di / sii;
        rs[a] = rs_a * sia;               // for d/dS_ii of R
        cs[a] = bb[a] * sia;              // for d/dS_ii and d/dd_i of c
      }
      __syncwarp();
      if (lane == 0) {
        double r2 = 0.0, c1 = 0.0;
        for (int a = 0; a < n; ++a) {
          r2 += rs[a];
          c1 += cs[a];
        }
        // the term's own factors: Sigma^(k)_ik * pdf * g, pdf = N(d_i; 0, S_ii)
        const double pb = sik * g;
        Sb[i * q + i] = r2 / (sii * sii) + c1 * di / (sii * sii) + pb * pdf * (0.5 * di * di / (sii * sii) - 0.5 / sii);
        db[i] = -c1 / sii - pb * pdf * di / sii;
        Sb[i * q + k] += pdf * g;
      }
    }
    __syncwarp();
    // fold Sigma^(k) and d^(k) into the batch's covariance and mean adjoints (mu = -mean; the sign is applied at the end)
    for (int a = lane; a < q; a += 32) {
      double r = 0.0, c = 0.0;
      for (int j = 0; j < q; ++j) {
        r += Sb[a * q + j];
        c += Sb[j * q + a];
      }
      rs[a] = r;
      cs[a] = c;
    }
    __syncwarp();
    double tot = 0.0;
    for (int a = 0; a < q; ++a) tot += rs[a];
    for (int e = lane; e < qq; e += 32) {
      const int a = e / q, c = e % q;
      double v = (a != k && c != k) ? Sb[e] : 0.0;
      if (c == k && a != k) v -= rs[a];
      if (a == k && c != k) v -= cs[c];
      if (a == k && c == k) v += tot;
      covb[e] += v;
    }
    if (lane == 0) {
      double sd = 0.0;
      for (int j = 0; j < q; ++j) {
        sd += db[j];
        if (j != k) mub[j] -= db[j];
      }
      mub[k] += sd;
    }
    __syncwarp();
  }
  if (bad && lane == 0) atomicExch(err_flag, 1);
  __syncthreads();
  const int64_t t0 = b * q;
  if (threadIdx.x == 0) {
    double v = 0.0;
    for (int u = 0; u < q + qq; ++u) v += terms[u];
    out_val[b] = v;
  }
  const size_t stride = bei_back_warp_doubles(q);
  const size_t off_covb = 3 * (size_t)qq + 2 * q + 5 * 32 * (size_t)q + qq + 3 * q;
  for (int e = threadIdx.x; e < qq; e += blockDim.x) {
    const int a = e / q, c = e % q;
    double g = 0.0;
    for (int v = 0; v < nw; ++v) {
      const double* cb = base + v * stride + off_covb;
      g += 0.5 * (cb[a * q + c] + cb[c * q + a]);
    }
    sbar[b * qq + e] = g;
  }
  for (int j = threadIdx.x; j < q; j += blockDim.x) {
    double g = 0.0;
    for (int v = 0; v < nw; ++v) g += base[v * stride + off_covb + qq + j];
    cmu[t0 + j] = -g;
    cvar[t0 + j] = 1.0;
  }
}

// Standalone CDFs (MultivariateNormalCDF.__call__, utils.py:109-199): one warp per row, P(X <= x) for
// X ~ N(mean, cov + jitter I).  Per warp: M [Q^2] | b [Q] | ys [32 Q].
__global__ void __launch_bounds__(BEI_MAX_WARPS * 32)
mvn_cdf_kernel(const double* __restrict__ x, const double* __restrict__ mean, const double* __restrict__ cov, int64_t nb, int Q,
               const double* __restrict__ w, int S, double jitter, double* __restrict__ out, int* __restrict__ err_flag) {
  extern __shared__ __align__(16) unsigned char msm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * BEI_MAX_WARPS + warp;
  if (r >= nb) return;
  double* M = reinterpret_cast<double*>(msm) + (size_t)warp * bei_warp_doubles(Q);
  double* bv = M + Q * Q;
  double* ys = bv + Q;
  for (int e = lane; e < Q * Q; e += 32) M[e] = cov[r * Q * Q + e] + ((e / Q == e % Q) ? jitter : 0.0);
  for (int j = lane; j < Q; j += 32) bv[j] = x[r * Q + j] - mean[r * Q + j];
  __syncwarp();
  if (!warp_cholesky(M, Q, lane)) {
    if (lane == 0) atomicExch(err_flag, 1);
    return;
  }
  const double g = genz_cdf_warp(M, bv, Q, w, S, ys, lane);
  if (lane == 0) out[r] = g;
}

}  // namespace tb
