// fp64-accurate triangular GEMM on the INT8 tensor cores (Ozaki error-free splitting), the 6-digit engine.
//
//   A = Linv · K*  is needed to ~2^-46 relative to |row scale|·|K* scale| for the 1e-9·σ_f² variance bar.
//   Each fp64 operand is split into S = 6 balanced base-256 digits (int8 in [-128, 127]) under a power-of-two
//   scale (per row of Linv; one global scale for K*):   x = 2^e · Σ_p d_p · 2^(-8p)   (48 bits kept).
//   Products of digit matrices are EXACT in int32 accumulators, and all pairs with the same p + q = r share one
//   accumulator T_r, so
//        A[n,t] = 2^(e_n + f) · Σ_{r=2..R} 2^(-8r) · T_r[n,t],        R = 7  (21 digit products);
//   |T_r| <= 6 · K · 2^14 < 2^31 for K <= 16384.
//   The GEMM itself is the shared warpgroup-MMA digit GEMM (digit_gemm.cuh) with S = 6 (npass = 2, all 21 products) or,
//   for fp32 models, S = 4 on the 4 leading planes (npass = 1: 10 products, ~2^-28 of the operand scales, orders of
//   magnitude inside the fp32 tolerance).  Operands are pre-packed in the no-swizzle K-major core-matrix layout, so each
//   pipeline stage is a few contiguous 1-D bulk-TMA copies.
#pragma once
#include "common.cuh"
#include "digit_gemm.cuh"
#include "kernel_fn.cuh"
#include <cfloat>

namespace tb {
namespace oz {

constexpr int S = 6;                         // digits per operand
constexpr int TILE = 128 * KST;              // one digit tile: 128 rows x 64 k-bytes = 8 KB
constexpr int DIGIT_BITS = 48;               // v = rint(x / 2^e * 2^48) = Σ d_p 256^(6-p)

// balanced base-256 digits of v (|v| <= 2^46, so the top digit stays below 128): d[0] most significant
__device__ __forceinline__ void digits7(long long v, int d[S]) {
#pragma unroll
  for (int p = S - 1; p >= 0; --p) {
    int lo = (int)(((v + 128) & 255) - 128);
    d[p] = lo;
    v = (v - lo) >> 8;
  }
}

// The same 6 digits without a carry chain: v = Σ d_p 256^(6-p) with d_p in [-128,127]  <=>  the ordinary base-256 digits of
// u = v + Σ 128·256^i are d_p + 128, so the int8 digits are the bytes of (u ^ 0x808080808080); byte 0 = least significant = d_6.
__device__ __forceinline__ void digit_bytes6(long long v, uint32_t& lo, uint32_t& hi) {
  const unsigned long long K = 0x0000808080808080ULL;
  const unsigned long long w = ((unsigned long long)v + K) ^ K;
  lo = (uint32_t)w;
  hi = (uint32_t)(w >> 32);
}
// scatter the six digit bytes of one element into the six digit planes: element index JJ (0..15) within the lane's 16-byte rows
template <int JJ>
__device__ __forceinline__ void scatter_digits(uint32_t (&pk)[S][4], uint32_t lo, uint32_t hi) {
  // plane p (0 = most significant digit d_1) takes byte (5 - p) of w
  pk[0][JJ >> 2] = put_byte<JJ & 3, 1>(pk[0][JJ >> 2], hi);
  pk[1][JJ >> 2] = put_byte<JJ & 3, 0>(pk[1][JJ >> 2], hi);
  pk[2][JJ >> 2] = put_byte<JJ & 3, 3>(pk[2][JJ >> 2], lo);
  pk[3][JJ >> 2] = put_byte<JJ & 3, 2>(pk[3][JJ >> 2], lo);
  pk[4][JJ >> 2] = put_byte<JJ & 3, 1>(pk[4][JJ >> 2], lo);
  pk[5][JJ >> 2] = put_byte<JJ & 3, 0>(pk[5][JJ >> 2], lo);
}

__device__ __forceinline__ void scatter_digits_rt(uint32_t (&pk)[S][4], int jj, uint32_t lo, uint32_t hi) {
  switch (jj) {  // jj is a compile-time constant after unrolling: the switch folds away
    case 0: scatter_digits<0>(pk, lo, hi); break;
    case 1: scatter_digits<1>(pk, lo, hi); break;
    case 2: scatter_digits<2>(pk, lo, hi); break;
    case 3: scatter_digits<3>(pk, lo, hi); break;
    case 4: scatter_digits<4>(pk, lo, hi); break;
    case 5: scatter_digits<5>(pk, lo, hi); break;
    case 6: scatter_digits<6>(pk, lo, hi); break;
    case 7: scatter_digits<7>(pk, lo, hi); break;
    case 8: scatter_digits<8>(pk, lo, hi); break;
    case 9: scatter_digits<9>(pk, lo, hi); break;
    case 10: scatter_digits<10>(pk, lo, hi); break;
    case 11: scatter_digits<11>(pk, lo, hi); break;
    case 12: scatter_digits<12>(pk, lo, hi); break;
    case 13: scatter_digits<13>(pk, lo, hi); break;
    case 14: scatter_digits<14>(pk, lo, hi); break;
    default: scatter_digits<15>(pk, lo, hi); break;
  }
}

// ------------------------------------------------------------------------------------------------
// once per BO step: digit tiles of Linv.  grid = (stage kc, row-block I), 256 threads.
//   rowscale[n] = 2^e_n with 2^e_n > 2 max_k |Linv[n,k]|  (so |x|/2^e < 1/2 and the top digit fits)
// ------------------------------------------------------------------------------------------------
__global__ void linv_rowscale_kernel(const double* __restrict__ Linv, int64_t N, int64_t rows, double* __restrict__ rowscale) {
  const int64_t n = blockIdx.x;
  double mx = 0.0;
  if (n < N)
    for (int64_t k = threadIdx.x; k <= n; k += blockDim.x) mx = fmax(mx, fabs(Linv[n + k * N]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  __shared__ double sm[8];
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) mx = fmax(mx, sm[w]);
    int e = 0;
    if (mx > 0.0) {
      frexp(mx, &e);  // mx = m 2^e, m in [0.5, 1)
      e += 2;         // |x| / 2^e < 1/4
    }
    if (n < rows) rowscale[n] = ldexp(1.0, e);
  }
}

__global__ void linv_digits_kernel(const double* __restrict__ Linv, int64_t N, const double* __restrict__ rowscale,
                                   int8_t* __restrict__ AS) {
  const int I = blockIdx.y, kc = blockIdx.x;
  if (kc >= 2 * (I + 1)) return;
  int8_t* dst = AS + (a_stage_offset(I) + kc) * (int64_t)(S * TILE);
  for (int e = threadIdx.x; e < 128 * KST; e += blockDim.x) {
    const int r = e % 128, kin = e / 128;  // r fastest: column-major source is contiguous in n
    const int64_t n = (int64_t)I * 128 + r, k = (int64_t)kc * KST + kin;
    long long v = 0;
    if (n < N && k <= n) v = __double2ll_rn(Linv[n + k * N] / rowscale[n] * 281474976710656.0);  // 2^48
    int d[S];
    digits7(v, d);
    const int off = (r >> 3) * SBO + (kin >> 4) * LBO + (r & 7) * 16 + (kin & 15);
#pragma unroll
    for (int p = 0; p < S; ++p) dst[p * TILE + off] = (int8_t)d[p];
  }
}

// K^-1 (gradient path): symmetric matrix given by its lower triangle (column-major, cusolver potri); full rows.
__device__ __forceinline__ double sym_at(const double* __restrict__ A, int64_t N, int64_t n, int64_t k) {
  return n >= k ? A[n + k * N] : A[k + n * N];
}
__global__ void sym_rowscale_kernel(const double* __restrict__ A, int64_t N, int64_t rows, double* __restrict__ rowscale) {
  const int64_t n = blockIdx.x;
  double mx = 0.0;
  if (n < N)
    for (int64_t k = threadIdx.x; k < N; k += blockDim.x) mx = fmax(mx, fabs(sym_at(A, N, n, k)));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  __shared__ double sm[8];
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) mx = fmax(mx, sm[w]);
    int e = 0;
    if (mx > 0.0) {
      frexp(mx, &e);
      e += 2;
    }
    if (n < rows) rowscale[n] = ldexp(1.0, e);
  }
}
__global__ void sym_digits_kernel(const double* __restrict__ A, int64_t N, int nst, const double* __restrict__ rowscale,
                                  int8_t* __restrict__ AS) {
  const int I = blockIdx.y, kc = blockIdx.x;
  int8_t* dst = AS + ((int64_t)I * nst + kc) * (int64_t)(S * TILE);
  for (int e = threadIdx.x; e < 128 * KST; e += blockDim.x) {
    const int r = e % 128, kin = e / 128;
    const int64_t n = (int64_t)I * 128 + r, k = (int64_t)kc * KST + kin;
    long long v = 0;
    if (n < N && k < N) v = __double2ll_rn(sym_at(A, N, n, k) / rowscale[n] * 281474976710656.0);
    int d[S];
    digits7(v, d);
    const int off = (r >> 3) * SBO + (kin >> 4) * LBO + (r & 7) * 16 + (kin & 15);
#pragma unroll
    for (int p = 0; p < S; ++p) dst[p * TILE + off] = (int8_t)d[p];
  }
}

// ------------------------------------------------------------------------------------------------
// K* digit tiles + posterior mean.  grid = candidate tiles x (512 / blockDim); warp w (0..15 within a tile) owns candidates
// [8w, 8w+8); lane l <-> (candidate l % 8, 16-wide k chunk l / 8): every digit store of a warp is 512
// contiguous bytes (four adjacent core matrices).  A candidate's mean does not depend on the other candidates of the launch.
// ------------------------------------------------------------------------------------------------
template <int KIND, int DP>
__global__ void __launch_bounds__(512, 2)
kstar_digits_kernel(const double* __restrict__ Xs, const double* __restrict__ alpha, const double* __restrict__ Xc,
                    const double* __restrict__ inv_ls, int N, int nst, int D, int64_t M, double variance,
                    double inv_bscale_2p48, double mean_const, int8_t* __restrict__ BS, double* __restrict__ mean_out) {
  // CTA size is free (any multiple of 32 dividing 512): each warp owns one 8-candidate row group of a tile
  const int lane = threadIdx.x & 31;
  const int wg = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), w = wg & 15, tile_id = wg >> 4;
  const int cl = lane & 7, ch = lane >> 3;
  const int t_local = w * 8 + cl;
  const int64_t t = (int64_t)tile_id * 128 + t_local;
  const bool valid = t < M;
  double xc[DP];
#pragma unroll
  for (int d = 0; d < DP; ++d) xc[d] = (valid && d < D) ? Xc[t * D + d] * inv_ls[d] : 0.0;
  int8_t* tile = BS + (int64_t)tile_id * nst * (S * TILE) + w * SBO + ch * LBO + cl * 16;
  // the 64 training rows (+ alpha) of a stage are staged through shared memory with cp.async, double-buffered: ncu showed the
  // kernel waiting on L1/L2 latency of these warp-broadcast loads (long_scoreboard was the top stall)
  __shared__ __align__(16) double xs_s[2][KST * DP];
  __shared__ __align__(16) double al_s[2][KST];
  auto stage_load = [&](int kc, int buf) {
    const double* src = Xs + (int64_t)kc * KST * DP;
    for (int e = threadIdx.x; e < KST * DP / 2; e += blockDim.x)
      asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(smem_u32(&xs_s[buf][2 * e])), "l"(src + 2 * e) : "memory");
    for (int e = threadIdx.x; e < KST / 2; e += blockDim.x)
      asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(smem_u32(&al_s[buf][2 * e])), "l"(alpha + (int64_t)kc * KST + 2 * e)
                   : "memory");
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  stage_load(0, 0);
  double macc = 0.0;
  for (int kc = 0; kc < nst; ++kc) {
    const int buf = kc & 1;
    if (kc + 1 < nst) {
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
      const int kl = ch * 16 + j, k = kc * KST + kl;
      const double* xr = &xs_s[buf][kl * DP];
      double r2 = 0.0;
#pragma unroll
      for (int d = 0; d < DP; d += 2) {
        const double2 v = *reinterpret_cast<const double2*>(xr + d);
        double d0 = xc[d] - v.x, d1 = xc[d + 1] - v.y;
        r2 = fma(d0, d0, r2);
        r2 = fma(d1, d1, r2);
      }
      const double kval = (valid && k < N) ? kernel_from_r2<KIND>(r2, variance) : 0.0;
      macc = fma(kval, al_s[buf][kl], macc);
      uint32_t wl, wh;
      digit_bytes6(__double2ll_rn(kval * inv_bscale_2p48), wl, wh);
      scatter_digits_rt(pk, j, wl, wh);
    }
#pragma unroll
    for (int p = 0; p < S; ++p)
      *reinterpret_cast<uint4*>(tile + (int64_t)kc * (S * TILE) + p * TILE) = make_uint4(pk[p][0], pk[p][1], pk[p][2], pk[p][3]);
    __syncthreads();  // everyone is done with xs_s[buf] before the next iteration's prefetch overwrites it
  }
  macc += __shfl_xor_sync(0xffffffffu, macc, 8);
  macc += __shfl_xor_sync(0xffffffffu, macc, 16);
  if (ch == 0) mean_out[(int64_t)tile_id * 128 + t_local] = macc + mean_const;
}

// ------------------------------------------------------------------------------------------------
// the GEMM: partial[g][t] = Σ_{rows n of group g} A[n,t]^2 (OZ_SUMSQ) or A itself, fp64, candidate-major [t][lda] (OZ_STORE)
// ------------------------------------------------------------------------------------------------
enum { OZ_SUMSQ = dg::EPI_SUMSQ, OZ_STORE = dg::EPI_STORE };

inline int trigemm_init() {
  TB_TRY((dg::set_smem<6, dg::EPI_SUMSQ, 128>()));
  TB_TRY((dg::set_smem<6, dg::EPI_STORE, 128>()));
  TB_TRY((dg::set_smem<4, dg::EPI_SUMSQ, 128>()));
  TB_TRY((dg::set_smem<4, dg::EPI_STORE, 128>()));
  return 0;
}

// full_rows = 0: lower-triangular left factor (Linv): row-block I spans stages [0, 2(I+1)), packed triangularly.
// full_rows = 1: dense square left factor (K^-1, gradient path): every row-block spans all nst stages, offset I*nst.
template <int EPI>
inline int launch_trigemm(cudaStream_t st, int tiles, const int8_t* AS, const int8_t* BS, const double* rowscale, int NB, int nst, int G,
                          int64_t McPad, double out_scale, int npass, int full_rows, double* partial, double* Aplain, int64_t lda) {
  if (npass == 2)
    return dg::launch<6, EPI, 128>(st, AS, BS, rowscale, nullptr, NB, nst, G, tiles, McPad, out_scale, 0.0, S, S, full_rows, partial,
                                   Aplain, lda);
  return dg::launch<4, EPI, 128>(st, AS, BS, rowscale, nullptr, NB, nst, G, tiles, McPad, out_scale, 0.0, S, S, full_rows, partial,
                                 Aplain, lda);
}

}  // namespace oz
}  // namespace tb
