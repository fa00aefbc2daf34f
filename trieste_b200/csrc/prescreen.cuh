// Screened argmax of EI / log-EI (tb_api.cu, argmax_screened): the fp32 bound pass and the compaction of its survivors.
//
// The bound pass evaluates the posterior mean of every candidate in fp32 from fp32 mirrors of the posterior (training rows
// centred and pre-scaled, their squared norms, σ_f²·α and |σ_f²·α|; built on the host, gp->pre_*) together with
// S = Σ_j |σ_f² α_j| k_j, and turns them into a rigorous bound E(x) >= |μ(x) - μ̃(x)| on the distance to the mean μ(x) that the
// unscreened call computes in fp64 (DESIGN.md §4d derives E and its constants).  A candidate's screen value is
// ub = acq(μ̃ - E, var_ub): EI and log-EI fall as the mean rises and rise with the variance, so ub bounds its exact value.
#pragma once
#include "kernels_f64.cuh"

namespace tb {
namespace pre {

constexpr int KS = 64;   // training rows per shared-memory stage
constexpr int KH = 32;   // terms per fp32 partial sum; each is added into an fp64 accumulator
constexpr int TH = 256;  // threads per CTA
// candidates per thread: the staged row is read once from shared memory for CPT evaluations
template <int DP> struct Cpt { static constexpr int value = DP <= 12 ? 4 : DP <= 20 ? 2 : 1; };
// one mirrored training row: x'[DP], |x'|^2, a = σ_f² α, |a|, zero padding to whole float4s
template <int DP> struct Row { static constexpr int W = ((DP + 3 + 3) / 4) * 4; };

// constants of the bound (host: prescreen_build in tb_api.cu; DESIGN.md §4d)
struct Bound {
  double rel;       // candidate-independent relative part, times S
  double lin;       // times (|x'|^2 + max|X'|^2) (expansion form) or (|x'| + max|X'|) (Matern12): a bound on the log-error of k
  double lin_max;   // where that log-error bound exceeds this, E is not trusted and the candidate survives
  double abs;       // absolute part (underflow, flush to zero, the tail of the s-proportional term)
  double safety;    // factor on the whole bound
  double x2max;     // max_j |X'_j|^2
  double mean_const;
  double pre;       // x' = (x / l - centre) * pre
};

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rsqrt_approx(float x) {
  float y;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// the kernel value over σ_f² on the pre-scaled squared distance q (pre² = log2(e)/2 for RBF, 3 log2(e)² for Matern32,
// 5 log2(e)² for Matern52: the exp argument is q or sqrt(q) itself; log2(e)² for Matern12, whose q comes from the difference form)
template <int KIND>
__device__ __forceinline__ float kfun(float q) {
  constexpr float LN2 = 0.693147180559945309f, LN2SQ3 = 0.160151031252949358f;  // ln 2, (ln 2)²/3
  if (KIND == TB_RBF) return ex2_approx(-q);
  q = fmaxf(q, 1e-30f);
  const float s = q * rsqrt_approx(q);  // sqrt(q) = s_nat log2(e)
  const float e = ex2_approx(-s);
  if (KIND == TB_MATERN12) return e;
  if (KIND == TB_MATERN32) return fmaf(s, LN2, 1.0f) * e;
  return fmaf(q, LN2SQ3, fmaf(s, LN2, 1.0f)) * e;
}

// One CTA: TH threads x CPT candidates.  acq >= 0: ub[t] = acq(μ̃ - E, var_ub) (NaN when E is not finite or not trusted) and
// the CTA's first-max of acq(μ̃, var_ub) (the probe); acq < 0: lo[t] = μ̃ - E, hi[t] = μ̃ + E (tb_gp_mean_bounds).
template <int KIND, int DP>
__global__ void __launch_bounds__(TH, 2)
mean_bounds_kernel(const float* __restrict__ rows, int nst, const double* __restrict__ Xc, const double* __restrict__ inv_ls,
                   const double* __restrict__ centre, int D, int64_t M, const __grid_constant__ Bound b, int acq, double param,
                   double var_ub, double* __restrict__ out0, double* __restrict__ out1, double* __restrict__ blk_best,
                   int64_t* __restrict__ blk_idx) {
  constexpr int CPT = Cpt<DP>::value, W = Row<DP>::W, CH = KS * W / 4;  // CH: 16-byte chunks per stage
  constexpr bool EXPAND = KIND != TB_MATERN12;
  __shared__ __align__(16) float rs[2][KS * W];
  const int64_t t0 = (int64_t)blockIdx.x * (TH * CPT) + threadIdx.x;
  float xc[CPT][DP], xc2[CPT];
#pragma unroll
  for (int c = 0; c < CPT; ++c) {
    const int64_t t = t0 + (int64_t)c * TH;
    xc2[c] = 0.0f;
#pragma unroll
    for (int d = 0; d < DP; ++d) {
      xc[c][d] = (t < M && d < D) ? (float)((Xc[t * D + d] * inv_ls[d] - centre[d]) * b.pre) : 0.0f;
      xc2[c] = fmaf(xc[c][d], xc[c][d], xc2[c]);
    }
  }
  auto stage_load = [&](int kc, int buf) {
    const float* src = rows + (int64_t)kc * KS * W;
#pragma unroll
    for (int i = 0; i < (CH + TH - 1) / TH; ++i) {
      const int e = i * TH + (int)threadIdx.x;
      if (e < CH) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(&rs[buf][4 * e])), "l"(src + 4 * e) : "memory");
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  double mu_d[CPT], s_d[CPT];
#pragma unroll
  for (int c = 0; c < CPT; ++c) mu_d[c] = s_d[c] = 0.0;
  stage_load(0, 0);
  for (int kc = 0; kc < nst; ++kc) {
    const int buf = kc & 1;
    if (kc + 1 < nst) {
      stage_load(kc + 1, buf ^ 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
#pragma unroll
    for (int h = 0; h < KS / KH; ++h) {
      float mu[CPT], sa[CPT];
#pragma unroll
      for (int c = 0; c < CPT; ++c) mu[c] = sa[c] = 0.0f;
#pragma unroll 4
      for (int j = h * KH; j < (h + 1) * KH; ++j) {
        float xr[W];
#pragma unroll
        for (int i = 0; i < W; i += 4) {
          const float4 v = *reinterpret_cast<const float4*>(&rs[buf][j * W + i]);
          xr[i] = v.x, xr[i + 1] = v.y, xr[i + 2] = v.z, xr[i + 3] = v.w;
        }
#pragma unroll
        for (int c = 0; c < CPT; ++c) {
          float q;
          if (EXPAND) {
            float dot = 0.0f;
#pragma unroll
            for (int d = 0; d < DP; ++d) dot = fmaf(xc[c][d], xr[d], dot);
            q = fmaf(-2.0f, dot, xc2[c] + xr[DP]);
          } else {
            q = 0.0f;
#pragma unroll
            for (int d = 0; d < DP; ++d) {
              const float df = xc[c][d] - xr[d];
              q = fmaf(df, df, q);
            }
          }
          const float f = kfun<KIND>(q);
          mu[c] = fmaf(xr[DP + 1], f, mu[c]);
          sa[c] = fmaf(xr[DP + 2], f, sa[c]);
        }
      }
#pragma unroll
      for (int c = 0; c < CPT; ++c) {
        mu_d[c] += (double)mu[c];
        s_d[c] += (double)sa[c];
      }
    }
    __syncthreads();
  }
  double bv = -INFINITY;
  int64_t bi = INT64_MAX;
#pragma unroll
  for (int c = 0; c < CPT; ++c) {
    const int64_t t = t0 + (int64_t)c * TH;
    if (t >= M) continue;
    const double x2 = (double)xc2[c];
    const double lg = EXPAND ? b.lin * (x2 + b.x2max) : b.lin * (sqrt(x2) + sqrt(b.x2max));
    double e = b.safety * (fma(b.rel + lg, s_d[c], b.abs));
    const double mt = b.mean_const + mu_d[c];
    if (!(lg <= b.lin_max) || !(e <= DBL_MAX)) e = NAN;  // not trusted: NaN bounds, the candidate survives
    if (acq < 0) {
      out0[t] = mt - e;
      out1[t] = mt + e;
    } else {
      out0[t] = acq_value(acq, param, 0.0, mt - e, var_ub);
      const double v = acq_value(acq, param, 0.0, mt, var_ub);
      if (v == v) best_merge(bv, bi, v, t);
    }
  }
  if (acq >= 0) block_best_store(bv, bi, blk_best, blk_idx);
}

// the screen's winner as a one-candidate set (coordinates, global index); if every value was NaN, candidate 0
__global__ void probe_kernel(const double* __restrict__ Xc, int D, const int64_t* __restrict__ probe, double* __restrict__ xsel,
                             int64_t* __restrict__ isel) {
  int64_t p = *probe;
  if (p == INT64_MAX) p = 0;
  for (int d = threadIdx.x; d < D; d += blockDim.x) xsel[d] = Xc[p * D + d];
  if (threadIdx.x == 0) isel[0] = p;
}

// The survivors (ub >= screen_threshold(tau), or ub NaN), written densely as coordinates and global indices in two groups:
// candidates t < split (the whole chunks of the unscreened loop) from slot 0 up, the others (its last chunk) from slot cap - 1
// down; count[0] / count[1] count each group whole, slots outside [0, cap) are not written.  Their order depends on the
// scheduling; the first-max fold over global indices does not.
__global__ void __launch_bounds__(256)
compact_kernel(const double* __restrict__ Xc, const double* __restrict__ ub, int64_t M, int64_t split, int D, double var_ub,
               int acq, const double* __restrict__ run_best, int64_t cap, unsigned long long* __restrict__ count,
               double* __restrict__ xsel, int64_t* __restrict__ isel) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const double thr = screen_threshold(acq, *run_best, var_ub);
  const bool keep = t < M && !(ub[t] < thr);
  const bool back = t >= split;
  const unsigned ball = __ballot_sync(0xffffffffu, keep);
  if (ball == 0u) return;
  const int lane = threadIdx.x & 31;
  const unsigned bb = __ballot_sync(0xffffffffu, keep && back), bf = ball & ~bb;
  unsigned long long base_f = 0, base_b = 0;
  if (lane == 0) {
    if (bf) base_f = atomicAdd(&count[0], (unsigned long long)__popc(bf));
    if (bb) base_b = atomicAdd(&count[1], (unsigned long long)__popc(bb));
  }
  base_f = __shfl_sync(0xffffffffu, base_f, 0);
  base_b = __shfl_sync(0xffffffffu, base_b, 0);
  if (!keep) return;
  const unsigned below = (1u << lane) - 1u;
  const int64_t r = back ? (int64_t)(base_b + (unsigned long long)__popc(bb & below)) : (int64_t)(base_f + (unsigned long long)__popc(bf & below));
  if (r >= cap) return;
  const int64_t pos = back ? cap - 1 - r : r;
  for (int d = 0; d < D; ++d) xsel[pos * D + d] = Xc[t * D + d];
  isel[pos] = t;
}

}  // namespace pre
}  // namespace tb
