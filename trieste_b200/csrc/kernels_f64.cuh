// fp64 hot-path kernels: K(X*,X) panel generation, triangular DMMA GEMM, acquisition tail.
//
// Data flow for one chunk of candidates (SURVEY.md §3.2; GPflow GPRPosterior.predict_f called at
// trieste/models/gpflow/interface.py:120):
//   kstar_panels_kernel : Ks = K(X, X*) written in DMMA-fragment-packed panels + mean = Ks^T alpha + m
//   trigemm_kernel      : A = Linv · Ks per (row-block, candidate-tile), epilogue sum_n A^2  (never stores A)
//   tail_kernel         : var = clip(k** - sum A^2), EI / log-EI / LCB, block argmax
#pragma once
#include "common.cuh"
#include "../../include/trieste_b200.h"
#include "kernel_fn.cuh"
#include <cfloat>

namespace tb {

// ------------------------------------------------------------------------------------------------
// K1a: cross-covariance panels.  grid.x = candidate tiles of the chunk; 512 threads = 16 warps,
// warp w owns candidates [8w, 8w+8) of the tile; lane l <-> (candidate l/4, k-within-k4 l%4).
// Every store is one 512-byte contiguous warp write into the packed panel.
// ------------------------------------------------------------------------------------------------
template <int KIND, int DP>
__global__ void __launch_bounds__(512)
kstar_panels_kernel(const double* __restrict__ Xs,      // [nkc*16][DP] training inputs / lengthscale
                    const double* __restrict__ alpha,   // [nkc*16]  K^-1 err (0 beyond N)
                    const double* __restrict__ Xc,      // [M][D] raw candidates
                    const double* __restrict__ inv_ls,  // [DP]
                    int N, int nkc, int D, int64_t M, int64_t cand0, double variance,
                    double mean_const, double* __restrict__ KsP, double* __restrict__ mean_out) {
  const int lane = threadIdx.x & 31, tj = threadIdx.x >> 5;
  const int tl = lane >> 2, kq = lane & 3;
  const int t_local = tj * 8 + tl;
  const int64_t t = cand0 + (int64_t)blockIdx.x * BT + t_local;
  const bool valid = t < M;

  double xc[DP];
#pragma unroll
  for (int d = 0; d < DP; ++d) xc[d] = (valid && d < D) ? Xc[t * D + d] * inv_ls[d] : 0.0;

  double* panel = KsP + (int64_t)blockIdx.x * nkc * PANEL;
  double macc = 0.0;
  for (int kc = 0; kc < nkc; ++kc) {
#pragma unroll
    for (int p = 0; p < 2; ++p) {
      double kv[2];
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        const int k = kc * BK + (2 * p + s) * 4 + kq;
        const double* xr = Xs + (int64_t)k * DP;
        double r2 = 0.0;
#pragma unroll
        for (int d = 0; d < DP; d += 2) {
          double2 v = __ldg(reinterpret_cast<const double2*>(xr + d));
          double d0 = xc[d] - v.x, d1 = xc[d + 1] - v.y;
          r2 = fma(d0, d0, r2);
          r2 = fma(d1, d1, r2);
        }
        double kval = (valid && k < N) ? kernel_from_r2<KIND>(r2, variance) : 0.0;
        macc = fma(kval, __ldg(alpha + k), macc);
        kv[s] = kval;
      }
      reinterpret_cast<double2*>(panel + (int64_t)kc * PANEL)[(tj * 2 + p) * 32 + lane] =
          make_double2(kv[0], kv[1]);
    }
  }
  macc += __shfl_xor_sync(0xffffffffu, macc, 1);
  macc += __shfl_xor_sync(0xffffffffu, macc, 2);
  if (kq == 0) mean_out[(int64_t)blockIdx.x * BT + t_local] = macc + mean_const;
}

// ------------------------------------------------------------------------------------------------
// K1b: triangular DMMA GEMM  C = T · B  with T a packed triangular factor (Linv lower, or Linv^T upper)
//   grid = (candidate tiles, G row-block groups); 8 consumer warps (2 x 4, warp tile 64 rows x 32
//   candidates, 64 fp64 accumulators / thread) + 1 producer warp that streams packed 16 KB panels of
//   T and B with 1-D bulk TMA copies through a 4-stage mbarrier ring.
//   Epilogues (compile-time):
//     EPI_SUMSQ         partial[g][t] = sum over the group's rows n of C[n,t]^2            (variance)
//     EPI_SUMSQ_PACKED  + C stored as B-operand panels [tile][row/16][PANEL]   (feeds the Linv^T GEMM)
//     EPI_PLAIN         C stored plain, candidate-major: Cplain[t][ldc] (n contiguous)    (joint / V)
//     EPI_SUMSQ_PLAIN   both
// ------------------------------------------------------------------------------------------------
constexpr int TG_STAGES = 4;
constexpr int TG_CONSUMER_WARPS = 8;
constexpr int TG_THREADS = (TG_CONSUMER_WARPS + 1) * 32;
constexpr size_t TG_SMEM = (size_t)TG_STAGES * 2 * PANEL * sizeof(double) + 2 * TG_STAGES * 8 + 2 * BT * 8 + 64;

enum { EPI_SUMSQ = 0, EPI_SUMSQ_PACKED = 1, EPI_PLAIN = 2, EPI_SUMSQ_PLAIN = 3 };


// panel range [k0, k1) and storage offset of row-block I
template <bool UPPER>
__device__ __forceinline__ void rowblock_range(int I, int nkB, int& k0, int& k1, int64_t& off) {
  if (!UPPER) {
    k0 = 0;
    k1 = min((I + 1) * (BM / BK), nkB);
    off = rowblock_panel_offset(I);
  } else {
    k0 = I * (BM / BK);
    k1 = nkB;
    off = (int64_t)I * nkB - rowblock_panel_offset(I - 1) - (int64_t)k0;  // so that panel kc sits at off + kc
  }
}
__host__ __device__ inline int64_t upper_panel_count(int NB, int nkB) {
  return (int64_t)NB * nkB - rowblock_panel_offset(NB - 1);
}

template <bool UPPER, int EPI>
__global__ void __launch_bounds__(TG_THREADS, 1)
trigemm_kernel(const double* __restrict__ TP,   // packed triangular panels
               const double* __restrict__ BP,   // [tiles][nkB][PANEL]
               int NB, int nkB, int G, int64_t McPad,
               double* __restrict__ partial,    // [G][McPad]                (SUMSQ variants)
               double* __restrict__ Cpacked,    // [tiles][NB*8][PANEL]      (EPI_SUMSQ_PACKED)
               double* __restrict__ Cplain, int64_t ldc) {  // [McPad][ldc] (PLAIN variants)
  extern __shared__ __align__(128) unsigned char smem_raw[];
  double* sA = reinterpret_cast<double*>(smem_raw);
  double* sB = sA + TG_STAGES * PANEL;
  uint64_t* full = reinterpret_cast<uint64_t*>(sB + TG_STAGES * PANEL);
  uint64_t* empty = full + TG_STAGES;
  double* red = reinterpret_cast<double*>(empty + TG_STAGES);  // [2][BT]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x, g = blockIdx.y;

  if (threadIdx.x == 0) {
    for (int s = 0; s < TG_STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], TG_CONSUMER_WARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();

  const double* bTile = BP + (int64_t)tile * nkB * PANEL;

  if (warp == TG_CONSUMER_WARPS) {
    // ===== producer warp: one elected lane issues the bulk copies =====
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int i = 0;; ++i) {
        const int I = serpentine_rowblock(i, g, G);
        if (I >= NB) break;
        int k0, k1;
        int64_t off;
        rowblock_range<UPPER>(I, nkB, k0, k1, off);
        const double* aRow = TP + off * PANEL;
        for (int kc = k0; kc < k1; ++kc) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_expect_tx(&full[stage], 2 * PANEL * sizeof(double));
          bulk_g2s(sA + stage * PANEL, aRow + (int64_t)kc * PANEL, PANEL * sizeof(double), &full[stage]);
          bulk_g2s(sB + stage * PANEL, bTile + (int64_t)kc * PANEL, PANEL * sizeof(double), &full[stage]);
          if (++stage == TG_STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===== consumer warps =====
  const int wm = warp >> 2, wt = warp & 3;
  double acc[8][4][2];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;
  double colsum[4][2];
#pragma unroll
  for (int j = 0; j < 4; ++j) colsum[j][0] = colsum[j][1] = 0.0;

  int stage = 0;
  uint32_t phase = 0;
  for (int i = 0;; ++i) {
    const int I = serpentine_rowblock(i, g, G);
    if (I >= NB) break;
    int k0, k1;
    int64_t off;
    rowblock_range<UPPER>(I, nkB, k0, k1, off);
    for (int kc = k0; kc < k1; ++kc) {
      mbar_wait(&full[stage], phase);
      const double2* a2 = reinterpret_cast<const double2*>(sA + stage * PANEL);
      const double2* b2 = reinterpret_cast<const double2*>(sB + stage * PANEL);
#pragma unroll
      for (int p = 0; p < 2; ++p) {
        double2 af[8], bf[4];
#pragma unroll
        for (int ii = 0; ii < 8; ++ii) af[ii] = a2[((wm * 8 + ii) * 2 + p) * 32 + lane];
#pragma unroll
        for (int j = 0; j < 4; ++j) bf[j] = b2[((wt * 4 + j) * 2 + p) * 32 + lane];
#pragma unroll
        for (int ii = 0; ii < 8; ++ii)
#pragma unroll
          for (int j = 0; j < 4; ++j) dmma_m8n8k4(acc[ii][j][0], acc[ii][j][1], af[ii].x, bf[j].x);
#pragma unroll
        for (int ii = 0; ii < 8; ++ii)
#pragma unroll
          for (int j = 0; j < 4; ++j) dmma_m8n8k4(acc[ii][j][0], acc[ii][j][1], af[ii].y, bf[j].y);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[stage]);
      if (++stage == TG_STAGES) { stage = 0; phase ^= 1; }
    }
    // ---- row-block epilogue ----
    if (EPI == EPI_SUMSQ_PACKED) {
      // C[n,t] -> B-operand panel of the next GEMM: "k" = n % 16, "row" = t within the tile
      double* cTile = Cpacked + ((int64_t)tile * NB * (BM / BK) + (int64_t)I * (BM / BK)) * PANEL;
#pragma unroll
      for (int ii = 0; ii < 8; ++ii) {
        const int np = wm * 4 + (ii >> 1);  // 16-row panel within the row-block
        double* pn = cTile + (int64_t)np * PANEL;
        const int p = ii & 1, s = lane >> 4, kq = (lane >> 2) & 3;
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int g8 = wt * 4 + j, rr = (lane & 3) * 2 + c;
            pn[(((g8 * 2 + p) * 32 + rr * 4 + kq) << 1) + s] = acc[ii][j][c];
          }
      }
    }
    if (EPI == EPI_PLAIN || EPI == EPI_SUMSQ_PLAIN) {
      const int64_t tbase = (int64_t)tile * BT + wt * 32 + (lane & 3) * 2;
      const int64_t nbase = (int64_t)I * BM + wm * 64 + (lane >> 2);
#pragma unroll
      for (int ii = 0; ii < 8; ++ii)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int c = 0; c < 2; ++c)
            Cplain[(tbase + j * 8 + c) * ldc + nbase + ii * 8] = acc[ii][j][c];
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      double s0 = 0.0, s1 = 0.0;
#pragma unroll
      for (int ii = 0; ii < 8; ++ii) {
        s0 = fma(acc[ii][j][0], acc[ii][j][0], s0);
        s1 = fma(acc[ii][j][1], acc[ii][j][1], s1);
        acc[ii][j][0] = 0.0;
        acc[ii][j][1] = 0.0;
      }
      colsum[j][0] += s0;
      colsum[j][1] += s1;
    }
  }

  if (EPI == EPI_PLAIN) return;
  // reduce over the 8 row-lanes (lane / 4) of the warp, then over the two row-warps
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      double v = colsum[j][c];
      v += __shfl_xor_sync(0xffffffffu, v, 4);
      v += __shfl_xor_sync(0xffffffffu, v, 8);
      v += __shfl_xor_sync(0xffffffffu, v, 16);
      colsum[j][c] = v;
    }
  if (lane < 4) {
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int c = 0; c < 2; ++c) red[wm * BT + wt * 32 + j * 8 + lane * 2 + c] = colsum[j][c];
  }
  asm volatile("bar.sync 1, %0;" ::"n"(TG_CONSUMER_WARPS * 32));
  const int tid = threadIdx.x;
  if (tid < BT) partial[(int64_t)g * McPad + (int64_t)tile * BT + tid] = red[tid] + red[BT + tid];
}

// ------------------------------------------------------------------------------------------------
// acquisition tails (trieste/acquisition/function/function.py:221-223, 415-416; log-EI is ours)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ double ndtr_tfp(double x) {  // tfp special_math._ndtr piecewise form
  const double hs2 = 0.7071067811865476;
  double w = x * hs2, z = fabs(w);
  double y = (z < hs2) ? 1.0 + erf(w) : ((w > 0.0) ? 2.0 - erfc(z) : erfc(z));
  return 0.5 * y;
}
// aux: second parameter of the tail (the likelihood noise variance for AEI; unused otherwise)
__device__ __forceinline__ double acq_value(int acq, double param, double aux, double mean, double var) {
  const double sigma = sqrt(var);
  if (acq == TB_ACQ_LCB) return mean - param * sigma;
  if (acq == TB_ACQ_NEG_LCB) return -(mean - param * sigma);
  const double z = (param - mean) / sigma;
  if (acq == TB_ACQ_PBT) return ndtr_tfp(z);
  if (acq == TB_ACQ_EI || acq == TB_ACQ_AEI) {
    const double pdf_term = sigma * exp(-0.5 * z * z) * 0.3989422804014327;  // variance * N(eta; mean, sigma)
    const double ei = (param - mean) * ndtr_tfp(z) + pdf_term;
    if (acq == TB_ACQ_EI) return ei;
    return ei * (1.0 - sqrt(aux) / sqrt(aux + var));  // function.py:318-325
  }
  // log-EI: log(sigma) + log(phi(z) + z Phi(z))
  double lh;
  if (z > -1.0) {
    lh = log(z * ndtr_tfp(z) + exp(-0.5 * z * z) * 0.3989422804014327);
  } else {
    double t;
    if (z < -1e3) {
      double iz2 = 1.0 / (z * z);
      t = (1.0 - 3.0 * iz2) * iz2;
    } else {
      t = 1.0 + z * 1.2533141373155003 * erfcx(-z * 0.7071067811865476);
    }
    lh = -0.5 * z * z - 0.9189385332046727 + log(t);
  }
  return lh + log(sigma);
}

// d acq / d mean and d acq / d var (for the gradient path); clipped variance has zero gradient
__device__ __forceinline__ void acq_partials(int acq, double param, double aux, double mean, double var,
                                             bool clipped, double& dmu, double& dvar) {
  const double sigma = sqrt(var);
  if (acq == TB_ACQ_LCB || acq == TB_ACQ_NEG_LCB) {
    double sgn = (acq == TB_ACQ_LCB) ? 1.0 : -1.0;
    dmu = sgn;
    dvar = clipped ? 0.0 : -sgn * param / (2.0 * sigma);
    return;
  }
  const double z = (param - mean) / sigma;
  const double pdf = exp(-0.5 * z * z) * 0.3989422804014327;
  const double cdf = ndtr_tfp(z);
  if (acq == TB_ACQ_PBT) {
    dmu = -pdf / sigma;
    dvar = clipped ? 0.0 : -pdf * z / (2.0 * var);
    return;
  }
  if (acq == TB_ACQ_EI) {
    dmu = -cdf;
    dvar = clipped ? 0.0 : pdf / (2.0 * sigma);
    return;
  }
  if (acq == TB_ACQ_AEI) {
    const double ei = (param - mean) * cdf + sigma * pdf;
    const double tv = aux + var;
    const double aug = 1.0 - sqrt(aux) / sqrt(tv);
    dmu = -cdf * aug;
    dvar = clipped ? 0.0 : pdf / (2.0 * sigma) * aug + ei * 0.5 * sqrt(aux) / (tv * sqrt(tv));
    return;
  }
  // log-EI: d/dmu = -Phi/(sigma h), d/dvar = phi/(2 sigma^2 h)... with h = phi + z Phi; use the
  // erfcx ratio R = Phi/phi for stability: Phi/h = R/(1+zR), phi/h = 1/(1+zR)
  double R, one_zR;
  if (z > -1.0) {
    R = cdf / pdf;
    one_zR = 1.0 + z * R;
  } else if (z < -1e3) {
    double iz2 = 1.0 / (z * z);
    one_zR = (1.0 - 3.0 * iz2) * iz2;
    R = (one_zR - 1.0) / z;
  } else {
    R = 1.2533141373155003 * erfcx(-z * 0.7071067811865476);
    one_zR = 1.0 + z * R;
  }
  dmu = -R / (sigma * one_zR);
  dvar = clipped ? 0.0 : 1.0 / (2.0 * var * one_zR);
}

// ---- the kinds with a tail of their own beside acq_value (which the screened EI bound pass also inlines)
__host__ __device__ __forceinline__ bool gibbon_kind(int acq) {
  return acq == TB_ACQ_GIBBON_QUALITY || acq == TB_ACQ_GIBBON_REPULSION || acq == TB_ACQ_GIBBON;
}
__host__ __device__ __forceinline__ bool feasibility_kind(int acq) {
  return acq == TB_ACQ_FEASIBILITY_BICHON || acq == TB_ACQ_FEASIBILITY_RANJAN;
}
__host__ __device__ __forceinline__ bool active_learning_kind(int acq) {
  return feasibility_kind(acq) || acq == TB_ACQ_BALD || acq == TB_ACQ_PREDICTIVE_VARIANCE;
}

// ---- active learning (active_learning.py), values in the reference's operation order:
//   feasibility (:220-245): s = sqrt(var), t = (T - mean)/s, t+- = t +- alpha; param = T, aux = alpha
//     Bichon  G1 = alpha (Phi(t+) - Phi(t-)) - t (2 Phi(t) - Phi(t+) - Phi(t-)) - (2 phi(t) - phi(t+) - phi(t-)),  G1 s
//     Ranjan  G2 = (alpha^2 - 1 - t^2)(Phi(t+) - Phi(t-)) - 2 t (phi(t+) - phi(t-)) + t+ phi(t+) - t- phi(t-),     G2 var
//   BALD (:504-513): v = max(var, j), p = Phi(mean / sqrt(v + 1)), E = sqrt(C2)/sqrt(v + C2) exp(-mean^2 / (2 (v + C2))),
//     C2 = pi log 2 / 2:  -p log(p + j) - (1 - p) log(1 - p + j) - E; param = j
//   predictive variance at q = 1 (:108): var + param
constexpr double BALD_C2 = 1.0887930451518010;  // pi log(2) / 2
__device__ __forceinline__ double npdf(double x) { return exp(-0.5 * x * x) * 0.3989422804014327; }
__device__ __forceinline__ double active_learning_value(int acq, double param, double aux, double mean, double var) {
  if (acq == TB_ACQ_PREDICTIVE_VARIANCE) return var + param;
  if (acq == TB_ACQ_BALD) {
    const double v = fmax(var, param);
    const double p = ndtr_tfp(mean / sqrt(v + 1.0));
    const double ef = (sqrt(BALD_C2) / sqrt(v + BALD_C2)) * exp(-(mean * mean) / (2.0 * (v + BALD_C2)));
    return -p * log(p + param) - (1.0 - p) * log(1.0 - p + param) - ef;
  }
  const double s = sqrt(var), a = aux;
  const double t = (param - mean) / s, tp = t + a, tm = t - a;
  const double cp = ndtr_tfp(tp), cm = ndtr_tfp(tm), pp = npdf(tp), pm = npdf(tm);
  if (acq == TB_ACQ_FEASIBILITY_BICHON)
    return (a * (cp - cm) - t * (2.0 * ndtr_tfp(t) - cp - cm) - (2.0 * npdf(t) - pp - pm)) * s;
  return ((a * a - 1.0 - t * t) * (cp - cm) - 2.0 * t * (pp - pm) + tp * pp - tm * pm) * var;
}
// d/dmean and d/dvar of the above (A = Phi(t+) - Phi(t-), B = phi(t+) - phi(t-)):
//   Bichon  dmean = 2 Phi(t) - Phi(t+) - Phi(t-),  dvar = (alpha A - (2 phi(t) - phi(t+) - phi(t-))) / (2 s)
//   Ranjan  dmean = 2 s (t A + B),                 dvar = G2 + t (t A + B)
//   BALD    h' = -log(p + j) - p/(p + j) + log(1 - p + j) + (1 - p)/(1 - p + j), u = mean / sqrt(v + 1):
//           dmean = h' phi(u) / sqrt(v + 1) + E mean / (v + C2),
//           dvar  = -h' phi(u) u / (2 (v + 1)) - E (mean^2 / (2 (v + C2)^2) - 1 / (2 (v + C2))), 0 where var < j
//   predictive variance: dmean = 0, dvar = 1
// and dvar = 0 where the tail clipped the variance
__device__ __forceinline__ void active_learning_partials(int acq, double param, double aux, double mean, double var,
                                                         bool clipped, double& dmu, double& dvar) {
  if (acq == TB_ACQ_PREDICTIVE_VARIANCE) {
    dmu = 0.0;
    dvar = clipped ? 0.0 : 1.0;
    return;
  }
  if (acq == TB_ACQ_BALD) {
    const double v = fmax(var, param), sv = sqrt(v + 1.0), vc = v + BALD_C2;
    const double u = mean / sv, p = ndtr_tfp(u), fu = npdf(u);
    const double ef = (sqrt(BALD_C2) / sqrt(vc)) * exp(-(mean * mean) / (2.0 * vc));
    const double dh = -log(p + param) - p / (p + param) + log(1.0 - p + param) + (1.0 - p) / (1.0 - p + param);
    dmu = dh * fu / sv + ef * mean / vc;
    dvar = (clipped || var < param) ? 0.0
                                    : -dh * fu * u / (2.0 * (v + 1.0)) - ef * (mean * mean / (2.0 * vc * vc) - 1.0 / (2.0 * vc));
    return;
  }
  const double s = sqrt(var), a = aux;
  const double t = (param - mean) / s, tp = t + a, tm = t - a;
  const double cp = ndtr_tfp(tp), cm = ndtr_tfp(tm), pp = npdf(tp), pm = npdf(tm);
  const double A = cp - cm;
  if (acq == TB_ACQ_FEASIBILITY_BICHON) {
    dmu = 2.0 * ndtr_tfp(t) - cp - cm;
    dvar = clipped ? 0.0 : (a * A - (2.0 * npdf(t) - pp - pm)) / (2.0 * s);
    return;
  }
  const double B = pp - pm, tab = t * A + B;
  const double g2 = (a * a - 1.0 - t * t) * A - 2.0 * t * B + tp * pp - tm * pm;
  dmu = 2.0 * s * tab;
  dvar = clipped ? 0.0 : g2 + t * tab;
}

struct BestPair {
  double v;
  int64_t i;
};
__device__ __forceinline__ void best_merge(double& v, int64_t& i, double v2, int64_t i2) {
  // first-max semantics of tf.math.argmax (optimizer.py:149): larger value wins, ties -> lower index
  if (v2 > v || (v2 == v && i2 < i)) {
    v = v2;
    i = i2;
  }
}

// ---- min-value entropy search (entropy.py:193-213): mean over the S min-value samples of
//   -gamma r / 2 - log Phi(-gamma),  gamma = (y*_s - mean) / sd,  r = phi(gamma) / Phi(-gamma)
// log Phi(x) and r are evaluated through erfcx for x < -1 (no cancellation, no underflow)
__device__ __forceinline__ void mes_terms(double gamma, double& log_cdf_neg, double& ratio) {
  const double x = -gamma;
  if (x > -1.0) {
    const double c = ndtr_tfp(x);
    log_cdf_neg = (x > 8.0) ? -ndtr_tfp(-x) : log(c);
    ratio = exp(-0.5 * x * x) * 0.3989422804014327 / c;
  } else {
    const double e = 0.5 * erfcx(-x * 0.7071067811865476);  // Phi(x) = e * exp(-x^2/2)
    log_cdf_neg = log(e) - 0.5 * x * x;
    ratio = 0.3989422804014327 / e;
  }
}
constexpr double MES_CLAMP_LB = 1e-8;  // entropy.py:47
__device__ __forceinline__ double mes_value(const double* __restrict__ samp, int ns, double mean, double var) {
  const double sd = fmax(sqrt(var), MES_CLAMP_LB);
  double acc = 0.0;
  for (int s = 0; s < ns; ++s) {
    const double gamma = (samp[s] - mean) / sd;
    double lc, r;
    mes_terms(gamma, lc, r);
    acc += -0.5 * gamma * r - lc;
  }
  return acc / (double)ns;
}
// d/dmean and d/dvar of the above: df/dgamma = r/2 - gamma r (r - gamma) / 2, dgamma/dmean = -1/sd,
// dgamma/dvar = -gamma / (2 var)
__device__ __forceinline__ void mes_partials(const double* __restrict__ samp, int ns, double mean, double var, bool clipped,
                                             double& dmu, double& dvar) {
  const double sd = fmax(sqrt(var), MES_CLAMP_LB);
  double am = 0.0, av = 0.0;
  for (int s = 0; s < ns; ++s) {
    const double gamma = (samp[s] - mean) / sd;
    double lc, r;
    mes_terms(gamma, lc, r);
    const double dg = 0.5 * r - 0.5 * gamma * r * (r - gamma);
    am += dg;
    av += dg * gamma;
  }
  dmu = -am / (sd * (double)ns);
  dvar = clipped ? 0.0 : -av / (2.0 * var * (double)ns);
}

// ---- GIBBON (entropy.py:479-500, 580-618)
//   quality   = -1/2 mean_s log(1 + rho2 r_s (gamma_s - r_s)),  rho2 = var / (var + noise), gamma and r as for MES
//   repulsion = w/2 (log(yvar - |u|^2) - log yvar),  yvar = var + noise,  |u|^2 = c(x)^T (B + noise I)^-1 c(x) (cross kernel)
// The quality term is evaluated as the reference writes it: for large gamma r (gamma - r) -> -1 cancels there too.
__device__ __forceinline__ double gibbon_quality_value(const double* __restrict__ samp, int ns, double mean, double var,
                                                       double noise) {
  const double rho2 = var / (var + noise);
  const double sd = fmax(sqrt(var), MES_CLAMP_LB);
  double acc = 0.0;
  for (int s = 0; s < ns; ++s) {
    const double gamma = (samp[s] - mean) / sd;
    double lc, r;
    mes_terms(gamma, lc, r);
    acc += log(1.0 + rho2 * r * (gamma - r));
  }
  return -0.5 * (acc / (double)ns);
}
// d/dmean and d/dvar of the above.  With h = r (gamma - r), r' = r (r - gamma), h' = r' (gamma - r) + r (1 - r'),
// I = 1 + rho2 h:  dq/dgamma = -rho2 h' / (2 I),  dq/drho2 = -h / (2 I),  dgamma/dmean = -1/sd,  dgamma/dvar = -gamma/(2 var),
// drho2/dvar = noise / yvar^2; the variance partial is zero where the variance is clipped
__device__ __forceinline__ void gibbon_quality_partials(const double* __restrict__ samp, int ns, double mean, double var,
                                                        double noise, bool clipped, double& dmu, double& dvar) {
  const double yvar = var + noise;
  const double rho2 = var / yvar;
  const double sd = fmax(sqrt(var), MES_CLAMP_LB);
  double am = 0.0, av = 0.0, ar = 0.0;
  for (int s = 0; s < ns; ++s) {
    const double gamma = (samp[s] - mean) / sd;
    double lc, r;
    mes_terms(gamma, lc, r);
    const double h = r * (gamma - r);
    const double dr = r * (r - gamma);
    const double dh = dr * (gamma - r) + r * (1.0 - dr);
    const double inv = 1.0 / (1.0 + rho2 * h);
    const double dg = -0.5 * rho2 * dh * inv;
    am += dg;
    av += dg * gamma;
    ar += -0.5 * h * inv;
  }
  dmu = -am / (sd * (double)ns);
  dvar = clipped ? 0.0 : (-av / (2.0 * var) + ar * noise / (yvar * yvar)) / (double)ns;
}
__device__ __forceinline__ double gibbon_repulsion_value(double var, double noise, double uu, double w) {
  const double yvar = var + noise;
  return w * (0.5 * (log(yvar - uu) - log(yvar)));
}
// kinds TB_ACQ_GIBBON_QUALITY / _REPULSION / TB_ACQ_GIBBON (repulsion + quality, entropy.py:435-436)
__device__ __forceinline__ double gibbon_value(int acq, const double* __restrict__ samp, int ns, double mean, double var,
                                               double noise, double uu, double w) {
  if (acq == TB_ACQ_GIBBON_QUALITY) return gibbon_quality_value(samp, ns, mean, var, noise);
  const double rep = gibbon_repulsion_value(var, noise, uu, w);
  if (acq == TB_ACQ_GIBBON_REPULSION) return rep;
  return rep + gibbon_quality_value(samp, ns, mean, var, noise);
}

// ---- local penalisation (greedy_batch.py:315-388): the base value times prod_j pen_j(||x - x_j||) over the pending points
//   soft (:315-354): pen_j = Phi((dist - radius_j) / scale_j)
//   hard (:357-388): pen_j = ((dist / (radius_j + scale_j))^-5 + 1)^(-1/5)
// f = pen_j and w = (d log pen_j / d dist) / dist, so that grad log pen_j = w (x - x_j).  At dist = 0 the gradient of the norm is
// undefined and w is taken as 0.  The soft ratio phi/Phi goes through erfcx for z < -1 (mes_terms).
__device__ __forceinline__ void penalty_factor(int kind, double dist, double radius, double scale, double& f, double& w) {
  if (kind == TB_PEN_SOFT) {
    const double z = (dist - radius) / scale;
    f = ndtr_tfp(z);
    double lc, ratio;
    mes_terms(-z, lc, ratio);  // ratio = phi(z) / Phi(z)
    w = dist > 0.0 ? ratio / (scale * dist) : 0.0;
  } else {
    const double u = dist / (radius + scale);
    f = pow(pow(u, -5.0) + 1.0, -0.2);
    // d log f / d dist = 1 / (dist (1 + u^5))
    const double u5 = u * u * u * u * u;
    w = dist > 0.0 ? (1.0 / dist) / (dist * (1.0 + u5)) : 0.0;
  }
}

// the value of one single-query kind at (mean, var), as the plain tail computes it (tail_kernel, reduce_kernel); the
// GIBBON repulsion kinds read |u|^2 of candidate t from gib_uu
__device__ __forceinline__ double kind_value(int acq, double param, double aux, const double* __restrict__ samp, int nsamp,
                                             double mu, double var, const double* __restrict__ gib_uu, int64_t t, double gib_w) {
  return (acq == TB_ACQ_MES) ? mes_value(samp, nsamp, mu, var)
         : gibbon_kind(acq)  ? gibbon_value(acq, samp, nsamp, mu, var, aux, gib_uu ? gib_uu[t] : 0.0, gib_w)
         : active_learning_kind(acq) ? active_learning_value(acq, param, aux, mu, var)
                                     : acq_value(acq, param, aux, mu, var);
}

constexpr int PEN_TILE = 32;  // pending points per shared-memory tile of the penalised tail
constexpr int PEN_DMAX = 32;  // largest input dimension (pick_dp)

struct TailPenalty {
  const double* xc = nullptr;      // [Mc][D] candidates of the chunk (device)
  const double* pend = nullptr;    // [P][D] pending points
  const double* radius = nullptr;  // [P]
  const double* scale = nullptr;   // [P]
  double* grad = nullptr;          // [Mc][D] gradient of the base acquisition, turned into the penalised one in place (nullable)
  int P = 0, D = 0, kind = 0;
  const double* gib_uu = nullptr;  // GIBBON repulsion kinds: |u|^2 [Mc] of the cross kernel, and the repulsion weight
  double gib_w = 0.0;
};

// first-max of the block's (value, index) pairs (blockDim.x <= 256) -> blk_best / blk_idx[blockIdx.x]
__device__ __forceinline__ void block_best_store(double bv, int64_t bi, double* __restrict__ blk_best, int64_t* __restrict__ blk_idx) {
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
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) best_merge(bv, bi, sv[w], si[w]);
    blk_best[blockIdx.x] = bv;
    blk_idx[blockIdx.x] = bi;
  }
}

// the posterior variance of candidate t before clipping: the prior variance less its sums of squares over the G row-block
// groups of the variance GEMM, summed in group order.  Every tail of a chunk (values, partials, EHVI) reads it from here.
__device__ __forceinline__ double chunk_raw_variance(const double* __restrict__ partial, int G, int64_t McPad, int64_t t,
                                                     double variance) {
  double ss = 0.0;
  for (int g = 0; g < G; ++g) ss += partial[(int64_t)g * McPad + t];
  return variance - ss;
}

// the chunk outputs of up to MEMBERS_MAX handles evaluated together (EHVI, reducers), as the combining kernels read them
constexpr int MEMBERS_MAX = 8;
struct ChunkMembers {
  const double* partial[MEMBERS_MAX];  // variance sums of squares over G row-block groups, stride McPad
  const double* mean[MEMBERS_MAX];
  double* dmv[MEMBERS_MAX];  // gradient path: d/dmean [Mc] then d/dvar [Mc] (the member's sMisc); null without a gradient
  int64_t McPad[MEMBERS_MAX];
  int G[MEMBERS_MAX];
  double variance[MEMBERS_MAX];
};

// out[i] = sum_l slices[l][i] in l order (the members' gradient assemblies of one chunk)
__global__ void __launch_bounds__(256)
member_grad_sum_kernel(const double* __restrict__ slices, int L, int64_t n, double* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double acc = slices[i];
  for (int l = 1; l < L; ++l) acc += slices[(int64_t)l * n + i];
  out[i] = acc;
}

// one thread per candidate of the chunk; block-level first-max argmax.  PEN: the value (and the gradient, when
// pen.grad is set) is multiplied by the local penalty before the argmax.  The argmax index of candidate t is idx_map[t]
// when idx_map is set (the compacted survivors of the screened argmax), else idx0 + t.
template <bool PEN>
__global__ void __launch_bounds__(256)
tail_kernel(const double* __restrict__ partial, int G, int64_t McPad, const double* __restrict__ mean,
            int64_t Mc, int64_t idx0, double variance, int acq, double param, double aux,
            const double* __restrict__ samp, int nsamp, double* __restrict__ out_vals, double* __restrict__ out_mean, double* __restrict__ out_var,
            double* __restrict__ blk_best, int64_t* __restrict__ blk_idx, const int64_t* __restrict__ idx_map, const TailPenalty pen) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  double bv = -INFINITY;
  int64_t bi = INT64_MAX;
  double vb = 0.0;  // PEN: the base value of this candidate
  if (t < Mc) {
    double var = fmax(chunk_raw_variance(partial, G, McPad, t, variance), 1e-12);
    double mu = mean[t];
    if (out_mean) out_mean[t] = mu;
    if (out_var) out_var[t] = var;
    if (acq >= 0) {
      double v = kind_value(acq, param, aux, samp, nsamp, mu, var, pen.gib_uu, t, pen.gib_w);
      if (PEN) {
        vb = v;
      } else {
        if (out_vals) out_vals[t] = v;
        if (v == v) { bv = v; bi = idx_map ? idx_map[t] : idx0 + t; }
      }
    }
  }
  if (PEN) {
    __shared__ double sp[PEN_TILE * PEN_DMAX], sr[PEN_TILE], sc[PEN_TILE];
    const bool live = t < Mc && acq >= 0;
    const int D = pen.D;
    double x[PEN_DMAX], g[PEN_DMAX];
#pragma unroll
    for (int d = 0; d < PEN_DMAX; ++d) {
      x[d] = (live && d < D) ? pen.xc[t * D + d] : 0.0;
      g[d] = 0.0;
    }
    double prod = 1.0;
    for (int j0 = 0; j0 < pen.P; j0 += PEN_TILE) {  // every thread of the block walks the tiles (barriers)
      const int nj = min(PEN_TILE, pen.P - j0);
      __syncthreads();
      for (int i = threadIdx.x; i < nj * D; i += blockDim.x) sp[i] = pen.pend[(int64_t)j0 * D + i];
      if (threadIdx.x < nj) {
        sr[threadIdx.x] = pen.radius[j0 + threadIdx.x];
        sc[threadIdx.x] = pen.scale[j0 + threadIdx.x];
      }
      __syncthreads();
      if (!live) continue;
      for (int j = 0; j < nj; ++j) {
        double r2 = 0.0;
#pragma unroll
        for (int d = 0; d < PEN_DMAX; ++d)
          if (d < D) {
            const double df = x[d] - sp[j * D + d];
            r2 = fma(df, df, r2);
          }
        double f, w;
        penalty_factor(pen.kind, sqrt(r2), sr[j], sc[j], f, w);
        prod *= f;
        if (pen.grad) {
#pragma unroll
          for (int d = 0; d < PEN_DMAX; ++d)
            if (d < D) g[d] = fma(w, x[d] - sp[j * D + d], g[d]);
        }
      }
    }
    if (live) {
      // exp(log base + log pen) of the reference (greedy_batch.py:265-268): NaN for a negative base value
      const double v = vb < 0.0 ? NAN : vb * prod;
      if (pen.grad) {
        // product rule pen grad(base) + base pen grad(log pen); where pen = 0 its gradient is taken as 0 (finite limit)
        double* gr = pen.grad + t * D;
#pragma unroll
        for (int d = 0; d < PEN_DMAX; ++d)
          if (d < D) gr[d] = fma(prod, gr[d], prod == 0.0 ? 0.0 : vb * (prod * g[d]));
      }
      if (out_vals) out_vals[t] = v;
      if (v == v) { bv = v; bi = idx_map ? idx_map[t] : idx0 + t; }
    }
  }
  if (blk_best == nullptr) return;
  block_best_store(bv, bi, blk_best, blk_idx);
}

// fold the per-block winners of one chunk into the running best (single block)
__global__ void __launch_bounds__(256)
argmax_fold_kernel(const double* __restrict__ blk_best, const int64_t* __restrict__ blk_idx, int nblk,
                   double* __restrict__ run_best, int64_t* __restrict__ run_idx) {
  double bv = -INFINITY;
  int64_t bi = INT64_MAX;
  for (int i = threadIdx.x; i < nblk; i += blockDim.x) best_merge(bv, bi, blk_best[i], blk_idx[i]);
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
    double rv = *run_best;
    int64_t ri = *run_idx;
    best_merge(rv, ri, bv, bi);
    *run_best = rv;
    *run_idx = ri;
  }
}

// ---- screened argmax of EI / log-EI (tb_api.cu, argmax_screened; prescreen.cuh) ----
// Both grow with the variance at a fixed mean, and the tail's variance fmax(variance - ss, 1e-12) (ss: a sum of squares, >= 0
// or NaN) never exceeds var_ub = fmax(variance, 1e-12).  ub = acq_value(mean, var_ub) therefore bounds the value the tail
// computes for the candidate, up to rounding: a candidate with ub < tau - screen_margin cannot reach tau.  The margin covers
// the rounding of both evaluations.  EI: its absolute error is a few ulp of (eta - mean) Phi(z) + sigma phi(z) <= max(2 EI,
// 0.7 sigma) (z^2 phi(z) <= 0.3 bounds the error carried by z), so 2^-20 |tau| + 2^-36 sigma_ub.  log-EI: the error is a few
// ulp of max(1, z^2) ~ max(1, |value|), so 2^-20 max(1, |tau|).
__device__ __forceinline__ double screen_threshold(int acq, double tau, double var_ub) {
  const double m = acq == TB_ACQ_EI ? fma(0x1p-20, fabs(tau), 0x1p-36 * sqrt(var_ub)) : 0x1p-20 * fmax(1.0, fabs(tau));
  return tau - m;  // tau = -inf: -inf (nothing is pruned); tau = +inf: NaN (nothing is pruned)
}

}  // namespace tb
