// Expected hypervolume improvement over L independent GP posteriors (trieste acquisition/function/multi_objective.py:145-250;
// Yang et al. 2019, eqs. 44-45), one thread per candidate.
//
// The non-dominated region is given as K cells [lower_k, upper_k] in the objectives' minimisation orientation.  In the
// negated (maximisation) coordinates of the reference, for cell k and objective l:
//   a = -upper_kl,  b = min(-lower_kl, 1e10),  m = -mean_l,  s = sqrt(var_l),  z_c = (c - m) / s,  Q(z) = 1 - Phi(z)
//   Psi(a, c) = s phi(z_c) + (m - a) Q(z_c),   nu = (b - a) Q(z_b),   g_kl = max(Psi(a, a) - Psi(a, b), 0) + nu
// The reference sums prod_l over the 2^L picks of (psi difference, nu) per objective; that sum is prod_l g_kl, so
//   EHVI = sum_k prod_l g_kl,
// O(K L) per candidate.  Cells stream through shared memory in tiles and are summed in index order (deterministic).
//
// Gradient (written to each member's sMisc as d/dmean [mc] then d/dvar [mc], the contract of grad_kernel):
//   dPsi(a,c)/dm = phi(z_c) (c - a) / s + Q(z_c),   dPsi(a,c)/ds = phi(z_c) (1 + z_c (c - a) / s)
//   dnu/dm = (b - a) phi(z_b) / s,                  dnu/ds = (b - a) phi(z_b) z_b / s
// d prod_l g_kl / d g_kl is the product of the other factors (prefix x suffix, no division: g may be 0).  The clipped
// branch of max(., 0) passes no gradient; at equality the gradient goes to the difference, as tf.maximum sends it to its
// first argument when x >= y.  dm/dmean = -1, ds/dvar = 1 / (2 s), and 0 where the variance is clipped.
//
// With PEN, HIPPO's penalty (trieste multi_objective.py:664-758) multiplies the value: for pending points p with stack
// moments (mu_pl, sigma_pl) and the candidate's member means mean_l,
//   d_p = sqrt(sum_l ((mean_l - mu_pl) / sigma_pl)^2),   w_p = (2/pi) atan(d_p),   pen = prod_p w_p,
// the pending points streamed through the cell tiles' shared memory after the cells.  pen and G_l = d pen / d mean_l are
// built in one pass in index order, G_l <- G_l w_p + pen w'_p dd_p/dmean_l and then pen <- pen w_p, with
// w'_p = (2/pi) / (1 + d_p^2) and dd_p/dmean_l = (mean_l - mu_pl) / (sigma_pl^2 d_p), taken as 0 at d_p = 0: no division
// by a factor that may be 0.  Then d/dmean_l = pen dEHVI/dmean_l + EHVI G_l and d/dvar_l = pen dEHVI/dvar_l.
#pragma once
#include "batch_ei.cuh"

namespace tb {

constexpr int EHVI_LMAX = MEMBERS_MAX;
constexpr int EHVI_TILE = 64;  // cells per shared-memory tile
constexpr double EHVI_CLIP = 1e10;  // multi_objective.py:215
constexpr double HIPPO_WARP = 0.63661977236758134308;  // 2 / pi, multi_objective.py:755

// HIPPO's penalty state: the pending points' stack moments, P >= 1 when a PEN kernel reads it
struct EhviPenalty {
  const double* mean;  // [P][L]
  const double* sd;    // [P][L], sqrt of the stack's variances
  int P;
};

// g(a, b) of one cell and objective, and with GRAD its derivatives in m and s
template <bool GRAD>
__device__ __forceinline__ double ehvi_factor(double a, double b, double m, double s, double& dm, double& ds) {
  const double za = (a - m) / s, zb = (b - m) / s;
  const double pa = std_normal_pdf(za), pb = std_normal_pdf(zb);
  const double qa = 1.0 - ndtr_tfp(za), qb = 1.0 - ndtr_tfp(zb);
  const double psi_aa = s * pa + (m - a) * qa;
  const double psi_ab = s * pb + (m - a) * qb;
  const double nu = (b - a) * qb;
  const double diff = psi_aa - psi_ab;
  if (GRAD) {
    const double w = b - a;
    dm = w * pb / s;  // nu
    ds = w * pb * zb / s;
    if (diff >= 0.0) {
      dm += qa - (pb * w / s + qb);
      ds += pa - pb * (1.0 + zb * w / s);
    }
  }
  return fmax(diff, 0.0) + nu;
}

// cells: lower [K][L] then upper [K][L].  Candidate t's value to out_vals[t] (nullable); with blk_best the block's first-max
// (NaN never wins) of (value, idx0 + t).  pen is read only with PEN.
template <int L, bool GRAD, bool PEN>
__global__ void __launch_bounds__(256)
ehvi_kernel(const ChunkMembers mb, const EhviPenalty pen, const double* __restrict__ cells, int64_t K, int64_t Mc, int64_t idx0,
            double* __restrict__ out_vals, double* __restrict__ blk_best, int64_t* __restrict__ blk_idx) {
  __shared__ double sa[EHVI_TILE * L], sb[EHVI_TILE * L];
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = t < Mc;
  double m[L], s[L], am[L], as[L];
  bool clipped[L];
#pragma unroll
  for (int l = 0; l < L; ++l) {
    const double raw = live ? chunk_raw_variance(mb.partial[l], mb.G[l], mb.McPad[l], t, mb.variance[l]) : 1.0;
    clipped[l] = raw < 1e-12;
    s[l] = sqrt(fmax(raw, 1e-12));
    m[l] = live ? -mb.mean[l][t] : 0.0;
    am[l] = 0.0;
    as[l] = 0.0;
  }
  const double* lower = cells;
  const double* upper = cells + K * L;
  double val = 0.0;
  for (int64_t k0 = 0; k0 < K; k0 += EHVI_TILE) {  // every thread walks the tiles (barriers)
    const int nk = K - k0 < EHVI_TILE ? (int)(K - k0) : EHVI_TILE;
    __syncthreads();
    for (int i = threadIdx.x; i < nk * L; i += blockDim.x) {
      sa[i] = -upper[k0 * L + i];
      sb[i] = fmin(-lower[k0 * L + i], EHVI_CLIP);
    }
    __syncthreads();
    if (!live) continue;
    for (int k = 0; k < nk; ++k) {
      double g[L], gm[L], gs[L], pre[L];
      double p = 1.0;
#pragma unroll
      for (int l = 0; l < L; ++l) {
        g[l] = ehvi_factor<GRAD>(sa[k * L + l], sb[k * L + l], m[l], s[l], gm[l], gs[l]);
        pre[l] = p;
        p *= g[l];
      }
      val += p;
      if (GRAD) {
        double suf = 1.0;
#pragma unroll
        for (int l = L - 1; l >= 0; --l) {
          const double c = pre[l] * suf;
          am[l] = fma(c, gm[l], am[l]);
          as[l] = fma(c, gs[l], as[l]);
          suf *= g[l];
        }
      }
    }
  }
  double pv = 1.0, G[L];  // penalty and its partials in the member means
  if (PEN) {
#pragma unroll
    for (int l = 0; l < L; ++l) G[l] = 0.0;
    for (int p0 = 0; p0 < pen.P; p0 += EHVI_TILE) {
      const int np = pen.P - p0 < EHVI_TILE ? pen.P - p0 : EHVI_TILE;
      __syncthreads();
      for (int i = threadIdx.x; i < np * L; i += blockDim.x) {
        sa[i] = pen.mean[(int64_t)p0 * L + i];
        sb[i] = pen.sd[(int64_t)p0 * L + i];
      }
      __syncthreads();
      if (!live) continue;
      for (int p = 0; p < np; ++p) {
        double r[L], d2 = 0.0;
#pragma unroll
        for (int l = 0; l < L; ++l) {
          r[l] = (-m[l] - sa[p * L + l]) / sb[p * L + l];
          d2 = fma(r[l], r[l], d2);
        }
        const double d = sqrt(d2);
        const double w = HIPPO_WARP * atan(d);
        if (GRAD) {
          const double c = d > 0.0 ? pv * (HIPPO_WARP / (1.0 + d2)) / d : 0.0;
#pragma unroll
          for (int l = 0; l < L; ++l) G[l] = fma(G[l], w, c * (r[l] / sb[p * L + l]));
        }
        pv *= w;
      }
    }
  }
  double bv = -INFINITY;
  int64_t bi = INT64_MAX;
  if (live) {
    if (GRAD) {
#pragma unroll
      for (int l = 0; l < L; ++l) {
        const double dvar = clipped[l] ? 0.0 : as[l] / (2.0 * s[l]);
        if (PEN) {
          mb.dmv[l][t] = fma(pv, -am[l], val * G[l]);
          mb.dmv[l][Mc + t] = pv * dvar;
        } else {
          mb.dmv[l][t] = -am[l];
          mb.dmv[l][Mc + t] = dvar;
        }
      }
    }
    if (PEN) val *= pv;
    if (out_vals) out_vals[t] = val;
    if (val == val) {
      bv = val;
      bi = idx0 + t;
    }
  }
  if (blk_best == nullptr) return;
  block_best_store(bv, bi, blk_best, blk_idx);
}

}  // namespace tb
