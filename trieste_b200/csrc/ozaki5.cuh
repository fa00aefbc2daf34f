// The int8 digit engine: centred K* generation and the digit count of a call.
//
// Operands are cut by ozaki.cuh's digit cutters against TIGHT scales (|x̂| <= 0.4975, an arbitrary fp64 scale per row of Linv),
// and K* is CENTRED: K* = h + K̃ with h = σ_f²/2, |K̃| <= h, so the sign bit of the top digit carries information;
// A = Linv·K̃ + h·rowsum(Linv), the second term is a per-row constant added in the epilogue.  With S balanced base-256 digits
// the pairs p + q <= S + 1 are kept, and all S levels r = 2..S+1 are accumulated at once: ONE pass per row-block and column
// chunk, one epilogue.  The host (int8_engines.cu) picks S from an a-priori bound computed from the row scales:
//   * S = 5 (15 products) keeps max |Δvar| at ~1e-10·σ_f² (emulated) on fp64 handles;
//   * fp32 models compute with S = 3 or 4 leading planes of a 4-digit split (6 / 10 products): ~5e-6·σ_f² against the
//     1e-4·σ_f² fp32 bar;
//   * handles the bound refuses (and tb_gp_set_engine(2)) run S = 6 (21 products; fp32 handles compute with its 4 leading
//     planes).
// The K* digit tiles are NT candidates wide (192 for S = 5, 128 otherwise); the GEMM (digit_gemm.cuh) works on them in
// column chunks of 64 candidates (32 for S = 6), whose S levels of int32 accumulators fit the registers of two consumer
// warpgroups.
#pragma once
#include "kernel_fn.cuh"
#include "ozaki.cuh"

namespace tb {
namespace oz5 {

using oz::FILL;
using oz::Geo;
using oz::KST;
using oz::LBO;
using oz::SBO;
using oz::two_pow_8S;

template <int S> __host__ __device__ constexpr double dig_koff() {  // 0x808080808080 / 0x8080808080 / 0x80808080 / 0x808080
  return S == 6 ? 141289400074368.0 : S == 5 ? 551911719040.0 : S == 4 ? 2155905152.0 : 8421504.0;
}

// X2[k] = |Xs[k]|^2 for the rows that exist (Xs is [rows_have][DP], zero padded), 0 beyond
__global__ void row_norms_kernel(const double* __restrict__ Xs, int64_t rows_have, int DP, int64_t rows, double* __restrict__ X2) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= rows) return;
  double s = 0.0;
  if (k < rows_have)
    for (int d = 0; d < DP; ++d) s = fma(Xs[k * DP + d], Xs[k * DP + d], s);
  X2[k] = s;
}

// ------------------------------------------------------------------------------------------------
// centred K* digit tiles + posterior mean.  CTAs of KGEN_WARPS warps; warp (global index wg) owns the 8 candidates
// [8 (wg % (NT/8)), +8) of candidate tile wg / (NT/8); lane l <-> (candidate l % 8, 16-wide k chunk l / 8): every digit
// store of a warp is 512 contiguous bytes.  The training rows of a stage are staged per CTA (they do not depend on the tile).
//   inv_bscale_2p = 2^(8S) / sB,  sB = h / FILL,  h = variance / 2
// A candidate's mean depends on (ksplit = gridDim.y, kc_per) only: the screened argmax (tb_api.cu) reproduces the mean of a
// candidate of an unscreened chunk by launching with that chunk's split.
// KVAL (the screened argmax's gathered tiles): no mean; every kernel value goes to mean_out as kval[ntiles NT][nst 64] instead, so
// that the k-stages can be split far finer than the mean's chain allows, and mean_replay_kernel rebuilds the chain of any split.
// ------------------------------------------------------------------------------------------------
constexpr int KGEN_WARPS = 8;
// S <= 5: 64 registers / 32 warps per SM (80 / 24 for D > 12).  S = 6 spills at 64 and 80 registers: 128, 255 for D > 10,
// and no spills.  KVAL launches are a few CTAs per SM at most: 128 registers, 255 for D > 12; no spills.
template <int KIND, int DP, int S, bool KVAL = false>
__global__ void __launch_bounds__(KGEN_WARPS * 32, KVAL ? (DP <= 12 ? 2 : 1) : S == 6 ? (DP <= 10 ? 2 : 1) : DP <= 12 ? 4 : 3)
kstar_digits_kernel(const double* __restrict__ Xs, const double* __restrict__ X2, const double* __restrict__ alpha,
                    const double* __restrict__ Xc, const double* __restrict__ inv_ls, int N, int nst, int D, int64_t M, double variance,
                    double inv_bscale_2p, double dig_c, double mean_const, const __grid_constant__ fm::Consts fc, int ntiles,
                    int kc_per, int8_t* __restrict__ BS, double* __restrict__ mean_out) {
  constexpr int NT = Geo<S>::NT, BTILE = NT * KST, TH = KGEN_WARPS * 32, WPT = NT / 8;  // WPT: warps per candidate tile
  // No masking of k >= N or of candidates t >= M is needed: training rows beyond N are zero-padded (their kernel values are
  // finite), alpha is zero there and so are all digits of Linv's columns k >= N, so those K* digits never reach a result;
  // padded candidates produce values nobody reads.
  // squared distances: the exact difference form for Matern12 (exp(-r) is not differentiable at r = 0, so the O(1e-16)
  // cancellation noise of the expansion form would show at 1e-8), the expansion |a|^2 + |b|^2 - 2 a.b (GPflow's
  // square_distance; D FMAs instead of 2 D operations per element) for the smooth kernels
  constexpr bool EXPAND = KIND != TB_MATERN12;
  const int lane = threadIdx.x & 31;
  const int64_t wg = (int64_t)blockIdx.x * KGEN_WARPS + (threadIdx.x >> 5);
  const int64_t tile_id = wg / WPT;
  const int w = (int)(wg % WPT);
  const int cl = lane & 7, ch = lane >> 3;
  const int t_local = w * 8 + cl;
  const int64_t t = tile_id * NT + t_local;
  const bool valid = t < M && tile_id < ntiles;  // warps past the last tile still take part in the staging barriers
  double xc[DP];
  double xc2 = 0.0;
#pragma unroll
  for (int d = 0; d < DP; ++d) {
    xc[d] = (valid && d < D) ? Xc[t * D + d] * inv_ls[d] : 0.0;
    xc2 = fma(xc[d], xc[d], xc2);
  }
  int8_t* tile = BS + tile_id * (int64_t)nst * (S * BTILE) + w * SBO + ch * LBO + cl * 16;
  // lanes with different ch read rows 16 apart: 16 rows are a multiple of 128 bytes, i.e. the same banks (ncu: 4-way conflicts
  // on every operand load) — every 16-row block is skewed by 16 bytes
  constexpr int XROW = KST * DP + 2 * (KST / 16), VROW = KST + 2 * (KST / 16);
  __shared__ __align__(16) double xs_s[2][XROW];
  __shared__ __align__(16) double al_s[2][VROW];
  __shared__ __align__(16) double x2_s[2][VROW];
  __shared__ __align__(16) double exp_tab[64];
  if (threadIdx.x < 64) exp_tab[threadIdx.x] = fm::EXP2_TABLE_DEV[threadIdx.x];
  auto stage_load = [&](int kc, int buf) {
    const double* src = Xs + (int64_t)kc * KST * DP;
    constexpr int CH = KST * DP / 2;  // 16-byte chunks of the stage's training rows
#pragma unroll
    for (int i = 0; i < (CH + TH - 1) / TH; ++i) {
      const int e = i * TH + (int)threadIdx.x;
      const int blk = (2 * e) / (16 * DP);  // 16-row block of this chunk (DP is even: a chunk never straddles rows)
      if (e < CH) asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(smem_u32(&xs_s[buf][2 * e + 2 * blk])), "l"(src + 2 * e) : "memory");
    }
    if (threadIdx.x < KST / 2) {
      const int e = threadIdx.x;
      asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(smem_u32(&al_s[buf][2 * e + 2 * (e / 8)])), "l"(alpha + (int64_t)kc * KST + 2 * e)
                   : "memory");
    } else if (EXPAND && threadIdx.x < KST) {
      const int e = threadIdx.x - KST / 2;
      asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(smem_u32(&x2_s[buf][2 * e + 2 * (e / 8)])), "l"(X2 + (int64_t)kc * KST + 2 * e)
                   : "memory");
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  // k-split (small candidate counts: a tile is 1.5 - 2 CTAs, far too few to fill 132 SMs): blockIdx.y takes the stages
  // [kc0, kc1) and writes its share of the mean to mean_out[blockIdx.y][ntiles NT] (summed in fixed order by mean_reduce_kernel)
  const int kc0 = (int)blockIdx.y * kc_per, kc1 = min(nst, kc0 + kc_per);
  stage_load(kc0, 0);
  // digit extraction without a conversion: v = rint(k inv) - c rides in the low mantissa bits of
  //   fma(k, inv, dig_c),  dig_c = 1.5 2^52 + 0x80..80 - c,  c = the INTEGER nearest to h inv (host: the centre actually
  //   subtracted is h_eff = c / inv, and the epilogue's row constant uses the same h_eff, so no bias is introduced);
  // the int8 digits are the low S bytes XOR 0x80 (digit_bytes, folded)
  double macc = 0.0, kprev = 0.0;
  for (int kc = kc0; kc < kc1; ++kc) {
    const int buf = (kc - kc0) & 1;
    if (kc + 1 < kc1) {
      stage_load(kc + 1, buf ^ 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    uint32_t pk[S][4];
#pragma unroll
    for (int p = 0; p < S; ++p) pk[p][0] = pk[p][1] = pk[p][2] = pk[p][3] = 0u;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int kl = ch * 16 + j, kv = kl + 2 * ch;  // kv: index into the skewed per-row vectors
      const double* xr = &xs_s[buf][kl * DP + 2 * ch];
      double r2;
      if (EXPAND) {
        double dot = 0.0;
#pragma unroll
        for (int d = 0; d < DP; d += 2) {
          const double2 v = *reinterpret_cast<const double2*>(xr + d);
          dot = fma(xc[d], v.x, dot);
          dot = fma(xc[d + 1], v.y, dot);
        }
        r2 = fma(-2.0, dot, xc2 + x2_s[buf][kv]);
      } else {
        r2 = 0.0;
#pragma unroll
        for (int d = 0; d < DP; d += 2) {
          const double2 v = *reinterpret_cast<const double2*>(xr + d);
          double d0 = xc[d] - v.x, d1 = xc[d + 1] - v.y;
          r2 = fma(d0, d0, r2);
          r2 = fma(d1, d1, r2);
        }
      }
      const double kval = kernel_from_r2_fast<KIND>(r2, variance, exp_tab, fc);
      if constexpr (KVAL) {  // kval[t][k]: the lane's 16 values of a stage are 128 contiguous bytes
        if (!(j & 1)) {
          kprev = kval;
        } else if (tile_id < ntiles) {
          *reinterpret_cast<double2*>(mean_out + (tile_id * NT + t_local) * (int64_t)nst * KST + (int64_t)kc * KST + kl - 1) =
              make_double2(kprev, kval);
        }
      } else {
        macc = fma(kval, al_s[buf][kv], macc);
      }
      const double tb = fma(kval, inv_bscale_2p, dig_c);
      const uint32_t wl = (uint32_t)__double2loint(tb) ^ 0x80808080u, wh = (uint32_t)__double2hiint(tb) ^ (S == 6 ? 0x8080u : 0x80u);
      oz::scatter_rt<S>(pk, j, wl, wh);
    }
    if (tile_id < ntiles) {
#pragma unroll
      for (int p = 0; p < S; ++p)
        *reinterpret_cast<uint4*>(tile + (int64_t)kc * (S * BTILE) + p * BTILE) = make_uint4(pk[p][0], pk[p][1], pk[p][2], pk[p][3]);
    }
    __syncthreads();
  }
  if constexpr (!KVAL) {
    macc += __shfl_xor_sync(0xffffffffu, macc, 8);
    macc += __shfl_xor_sync(0xffffffffu, macc, 16);
    if (ch == 0 && tile_id < ntiles)
      mean_out[(int64_t)blockIdx.y * ntiles * NT + tile_id * NT + t_local] = gridDim.y == 1 ? macc + mean_const : macc;
  }
}

// mean[t] = mean_const + Σ_s part[s][t] (fixed order: results do not depend on the scheduling of the k-split CTAs)
__global__ void mean_reduce_kernel(const double* __restrict__ part, int ksplit, int64_t stride, double mean_const,
                                   double* __restrict__ mean_out) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= stride) return;
  double s = 0.0;
  for (int i = 0; i < ksplit; ++i) s += part[(int64_t)i * stride + t];
  mean_out[t] = s + mean_const;
}

// The means of kstar_digits_kernel<.., KVAL = false> launched with split (ksplit, kc_per), bit for bit, from the kernel
// values kval[stride][nst 64] of its KVAL launch: per candidate and 16-wide k chunk ch the same fma chain over the stages of
// each split and the same lanes (candidate lane % 8, chunk lane / 8), the same xor-8 / xor-16 shuffle combine, and for
// ksplit > 1 the same fixed-order sum as mean_reduce_kernel.  stride = tiles NT; threads = 4 stride, in whole warps.  The
// chain is latency-bound: small CTAs spread it over many SMs, and each lane loads a stage's values while it sums the last.
constexpr int REPLAY_THREADS = 64;
__global__ void __launch_bounds__(REPLAY_THREADS)
mean_replay_kernel(const double* __restrict__ kval, const double* __restrict__ alpha, int nst, int ksplit, int kc_per, int64_t stride,
                   double mean_const, double* __restrict__ mean_out) {
  const int lane = threadIdx.x & 31, cl = lane & 7, ch = lane >> 3;
  const int64_t t = (((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 8 + cl;
  if (t - cl >= stride) return;  // whole warps leave together
  const double* kt = kval + t * (int64_t)nst * KST + ch * 16;
  double s = 0.0, macc = 0.0;
  const double* at = alpha + ch * 16;
  double2 kv[8], av[8];
  auto load = [&](int kc) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      kv[j] = *reinterpret_cast<const double2*>(kt + kc * KST + 2 * j);
      av[j] = *reinterpret_cast<const double2*>(at + kc * KST + 2 * j);
    }
  };
  load(0);
  for (int sp = 0; sp < ksplit; ++sp) {
    const int kc0 = sp * kc_per, kc1 = min(nst, kc0 + kc_per);
    macc = 0.0;
    for (int kc = kc0; kc < kc1; ++kc) {
      const double2 k2[8] = {kv[0], kv[1], kv[2], kv[3], kv[4], kv[5], kv[6], kv[7]};
      const double2 a2[8] = {av[0], av[1], av[2], av[3], av[4], av[5], av[6], av[7]};
      if (kc + 1 < nst) load(kc + 1);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        macc = fma(k2[j].x, a2[j].x, macc);
        macc = fma(k2[j].y, a2[j].y, macc);
      }
    }
    macc += __shfl_xor_sync(0xffffffffu, macc, 8);
    macc += __shfl_xor_sync(0xffffffffu, macc, 16);
    s += macc;
  }
  if (ch == 0) mean_out[t] = ksplit == 1 ? macc + mean_const : s + mean_const;
}

}  // namespace oz5
}  // namespace tb
