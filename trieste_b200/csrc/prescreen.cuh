// Screened argmax of EI / log-EI (tb_api.cu, argmax_screened): the fp32 bound pass and the compaction of its survivors.
//
// The bound pass evaluates the posterior mean of every candidate in fp32 from fp32 mirrors of the posterior (training rows
// centred and pre-scaled, their squared norms, σ_f²·α and |σ_f²·α|; built on the host, gp->pre_*) together with
// S = Σ_j |σ_f² α_j| k_j, and turns them into a rigorous bound E(x) >= |μ(x) - μ̃(x)| on the distance to the mean μ(x) that the
// unscreened call computes in fp64 (DESIGN.md §4d derives E and its constants).  A candidate's screen value is
// ub = acq(μ̃ - E, var_ub): EI and log-EI fall as the mean rises and rise with the variance, so ub bounds its exact value.
// RBF, Matern-32 and Matern-52 take their distances from the tensor cores (tc_mean_bounds_kernel) wherever that pass's bound
// is trusted on the training box; Matern-12, whose difference form has no expansion, and the smooth kernels at norms too large
// for the tensor-core bound run on the CUDA cores (mean_bounds_kernel).
#pragma once
#include <cuda_fp16.h>
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

// Geometry of the tensor-core pass (shared with the host, which lays the training columns out for it).  The product depth is
// 3·DP + 2 (x_hi, x_lo, x_hi, 1, 1 against -2X_hi, -2X_hi, -2X_lo, n_hi, n_lo) in k16 steps; a warp owns tc_mt m16 tiles of
// candidates, so one B fragment serves tc_mt tiles while the A fragments stay in registers; a stage holds tc_slices n8 slices
// of training columns, each 32 lanes x tc_nk x 8 bytes of B fragments followed by the slice's 8 weights |a_j|.
__host__ __device__ constexpr int tc_nk(int dp) { return (3 * dp + 2 + 15) / 16; }
__host__ __device__ constexpr int tc_mt(int dp) { return tc_nk(dp) <= 2 ? 4 : tc_nk(dp) <= 4 ? 2 : 1; }
__host__ __device__ constexpr int tc_slices(int dp) { return tc_nk(dp) <= 2 ? 16 : 8; }
__host__ __device__ constexpr int tc_slice_bytes(int dp) { return 256 * tc_nk(dp) + 32; }
__host__ __device__ constexpr int tc_cands(int dp) { return 16 * tc_mt(dp) * (TH / 32); }  // candidates per CTA

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

// The candidate's outputs from its fp64 sums μ̃ - mean_const and S̃: acq >= 0: ub[t] = acq(μ̃ - E, var_ub) (NaN when E is not
// finite or not trusted) and the first-max of acq(μ̃, var_ub) into (bv, bi) (the probe); acq < 0: lo[t] = μ̃ - E,
// hi[t] = μ̃ + E (tb_gp_mean_bounds).  lg: the distance log-error bound L(x).
__device__ __forceinline__ void bound_out(const Bound& b, int64_t t, double lg, double mu, double s, int acq, double param,
                                          double var_ub, double* __restrict__ out0, double* __restrict__ out1, double& bv,
                                          int64_t& bi) {
  double e = b.safety * (fma(b.rel + lg, s, b.abs));
  const double mt = b.mean_const + mu;
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

// The bound pass on the CUDA cores: Matern-12 (difference form), and the smooth kernels where the tensor-core pass's wider
// distance bound would not be trusted on the training box (prescreen_ensure; expansion form with an FFMA dot product).  One
// CTA: TH threads x CPT candidates; outputs as bound_out.
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
    bound_out(b, t, lg, mu_d[c], s_d[c], acq, param, var_ub, out0, out1, bv, bi);
  }
  if (acq >= 0) block_best_store(bv, bi, blk_best, blk_idx);
}

// D(16x8, f32) = A(16x16, f16, row) * B(16x8, f16, col) + C
__device__ __forceinline__ void mma_f16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// RBF, Matern-32, Matern-52: q = |x'|² + n_j - 2 x'·X'_j from tensor-core products of fp16 hi/lo splits.  A candidate's row
// [x_hi, x_lo, x_hi, 1, 1, 0...] against a training column [-2X_hi, -2X_hi, -2X_lo, n_hi, n_lo, 0...] (prescreen_ensure),
// with |x'|² as the accumulator input, misses only x_lo·X_lo and the splits' residuals (DESIGN.md §4d).  8 warps, each with
// MT m16 tiles of candidates whose A fragments and |x'|² stay in registers for the whole pass; the training columns stream
// through shared memory in stages of SL n8 slices.  The columns are sorted by the sign of a_j = σ_f²α_j and each sign class
// is padded to whole slices (weight 0), so a slice adds |a_j| k_j into one accumulator, P (a > 0, the first npos_sl slices)
// or Q: μ̃ = P - Q, S̃ = P + Q.  Per thread and candidate row, P and Q run in fp32 over one stage (at most 32 terms) and are
// then added into fp64; the quad's four fp64 sums are added in a fixed order at the end.  Outputs as bound_out.
template <int KIND, int DP>
__global__ void __launch_bounds__(TH, 2)
tc_mean_bounds_kernel(const unsigned char* __restrict__ cols, int nsl, int npos_sl, const double* __restrict__ Xc,
                      const double* __restrict__ inv_ls, const double* __restrict__ centre, int D, int64_t M,
                      const __grid_constant__ Bound b, int acq, double param, double var_ub, double* __restrict__ out0,
                      double* __restrict__ out1, double* __restrict__ blk_best, int64_t* __restrict__ blk_idx) {
  constexpr int NK = tc_nk(DP), K = 16 * NK, MT = tc_mt(DP), SL = tc_slices(DP), SLB = tc_slice_bytes(DP);
  constexpr int CB = tc_cands(DP), STB = SL * SLB;
  constexpr int CAND_BYTES = CB * (2 * K + 4), SMEM = CAND_BYTES > 2 * STB ? CAND_BYTES : 2 * STB;
  static_assert(KIND != TB_MATERN12 && STB % 16 == 0 && SMEM <= 48 * 1024, "tc_mean_bounds_kernel geometry");
  // the candidates' fp16 rows and |x'|² first, then (once they sit in registers) the double-buffered stages
  __shared__ __align__(16) unsigned char sm[SMEM];
  const int64_t c0 = (int64_t)blockIdx.x * CB;
  {
    __half* sa = reinterpret_cast<__half*>(sm);
    float* sx2 = reinterpret_cast<float*>(sm + CB * 2 * K);
    for (int c = threadIdx.x; c < CB; c += TH) {
      const int64_t t = c0 + c;
      __half* row = sa + c * K;
      float x2 = 0.0f;
#pragma unroll
      for (int d = 0; d < DP; ++d) {
        const float x = (t < M && d < D) ? (float)((Xc[t * D + d] * inv_ls[d] - centre[d]) * b.pre) : 0.0f;
        x2 = fmaf(x, x, x2);
        const __half hi = __float2half_rn(x);
        row[d] = row[2 * DP + d] = hi;
        row[DP + d] = __float2half_rn(x - __half2float(hi));
      }
      row[3 * DP] = row[3 * DP + 1] = __float2half_rn(1.0f);
#pragma unroll
      for (int k = 3 * DP + 2; k < K; ++k) row[k] = __float2half_rn(0.0f);
      sx2[c] = x2;
    }
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, tg = lane & 3;
  uint32_t af[MT][NK][4];
  float cx[MT][2];
#pragma unroll
  for (int m = 0; m < MT; ++m) {
    const int r = (warp * MT + m) * 16 + g;
    const __half* sa = reinterpret_cast<const __half*>(sm);
#pragma unroll
    for (int kk = 0; kk < NK; ++kk) {
      const __half* p = sa + r * K + kk * 16 + 2 * tg;
      af[m][kk][0] = *reinterpret_cast<const uint32_t*>(p);
      af[m][kk][1] = *reinterpret_cast<const uint32_t*>(p + 8 * K);
      af[m][kk][2] = *reinterpret_cast<const uint32_t*>(p + 8);
      af[m][kk][3] = *reinterpret_cast<const uint32_t*>(p + 8 * K + 8);
    }
    const float* sx2 = reinterpret_cast<const float*>(sm + CB * 2 * K);
    cx[m][0] = sx2[r];
    cx[m][1] = sx2[r + 8];
  }
  __syncthreads();  // the stages overwrite the candidates' rows

  auto stage_load = [&](int kc, int buf) {
    const unsigned char* src = cols + (int64_t)kc * STB;
#pragma unroll
    for (int i = 0; i < (STB / 16 + TH - 1) / TH; ++i) {
      const int e = i * TH + (int)threadIdx.x;
      if (e < STB / 16) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(sm + buf * STB + 16 * e)), "l"(src + 16 * e) : "memory");
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  // one n8 slice: the thread's 4 MT kernel values (rows g, g + 8 of each tile, columns 2 tg, 2 tg + 1) weighted into acc
  auto slice = [&](const unsigned char* sp, float (&acc)[MT][2]) {
    uint32_t bf[NK][2];
    if constexpr (NK % 2 == 0) {
#pragma unroll
      for (int kk = 0; kk < NK; kk += 2) {
        const uint4 v = reinterpret_cast<const uint4*>(sp)[(lane * NK + kk) / 2];
        bf[kk][0] = v.x, bf[kk][1] = v.y, bf[kk + 1][0] = v.z, bf[kk + 1][1] = v.w;
      }
    } else {
#pragma unroll
      for (int kk = 0; kk < NK; ++kk) {
        const uint2 v = reinterpret_cast<const uint2*>(sp)[lane * NK + kk];
        bf[kk][0] = v.x, bf[kk][1] = v.y;
      }
    }
    const float2 w = reinterpret_cast<const float2*>(sp + 256 * NK)[tg];
#pragma unroll
    for (int m = 0; m < MT; ++m) {
      float c[4] = {cx[m][0], cx[m][0], cx[m][1], cx[m][1]};
#pragma unroll
      for (int kk = 0; kk < NK; ++kk) mma_f16(c, af[m][kk], bf[kk][0], bf[kk][1]);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        acc[m][i >> 1] = fmaf(i & 1 ? w.y : w.x, kfun<KIND>(c[i]), acc[m][i >> 1]);
      }
    }
  };

  double pd[MT][2], qd[MT][2];
#pragma unroll
  for (int m = 0; m < MT; ++m) pd[m][0] = pd[m][1] = qd[m][0] = qd[m][1] = 0.0;
  const int nst = (nsl + SL - 1) / SL;
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
    const unsigned char* st = sm + buf * STB;
    const int s0 = kc * SL, pe = min(SL, nsl - s0), bnd = min(max(npos_sl - s0, 0), pe);
    // the stage's P slices, then its Q slices, each through one fp32 partial per row
    auto run = [&](int sa, int sb, double (&dd)[MT][2]) {
      float acc[MT][2];
#pragma unroll
      for (int m = 0; m < MT; ++m) acc[m][0] = acc[m][1] = 0.0f;
#pragma unroll 1  // a slice already holds 4 MT independent evaluations per thread; unrolled, RBF's would spill
      for (int s = sa; s < sb; ++s) slice(st + s * SLB, acc);
#pragma unroll
      for (int m = 0; m < MT; ++m) dd[m][0] += (double)acc[m][0], dd[m][1] += (double)acc[m][1];
    };
    run(0, bnd, pd);
    run(bnd, pe, qd);
    __syncthreads();
  }
  double bv = -INFINITY;
  int64_t bi = INT64_MAX;
#pragma unroll
  for (int m = 0; m < MT; ++m)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      // the quad's sums in a fixed order, the same in all four lanes
      pd[m][h] += __shfl_xor_sync(0xffffffffu, pd[m][h], 1);
      qd[m][h] += __shfl_xor_sync(0xffffffffu, qd[m][h], 1);
      pd[m][h] += __shfl_xor_sync(0xffffffffu, pd[m][h], 2);
      qd[m][h] += __shfl_xor_sync(0xffffffffu, qd[m][h], 2);
      const int64_t t = c0 + (warp * MT + m) * 16 + g + 8 * h;
      if ((2 * m + h) % 4 != tg || t >= M) continue;  // each of the quad's rows is finished by one lane
      const double x2 = (double)cx[m][h];
      // |x'_d| < 2^14 keeps every fp16 operand finite; far larger norms already fail lin_max
      const double lg = x2 < 0x1p28 ? b.lin * (x2 + b.x2max) : NAN;
      bound_out(b, t, lg, pd[m][h] - qd[m][h], pd[m][h] + qd[m][h], acq, param, var_ub, out0, out1, bv, bi);
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
