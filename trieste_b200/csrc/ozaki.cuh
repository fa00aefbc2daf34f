// fp64-accurate GEMMs on the INT8 tensor cores (Ozaki error-free splitting): the digit cutting both int8 engines share, and the
// K* generation of the 21-product engine.
//
//   A = Linv · K*  is needed to ~2^-46 relative to |row scale|·|K* scale| for the 1e-9·σ_f² variance bar.
//   Each fp64 operand is split into S balanced base-256 digits (int8 in [-128, 127]) under a per-row scale:
//        x = scale · Σ_{p=1..S} d_p · 2^(-8p)
//   Products of digit matrices are EXACT in int32 accumulators, and all pairs with the same p + q = r share one
//   accumulator T_r.  The 21-product engine splits into S = 6 digits under power-of-two scales with two spare bits (per row
//   of Linv; one global scale for K*), and keeps every level:
//        A[n,t] = 2^(e_n + f) · Σ_{r=2..R} 2^(-8r) · T_r[n,t],        R = 7  (21 digit products);
//   |T_r| <= 6 · K · 2^14 < 2^31 for K <= 16384.  fp32 models compute with the 4 leading planes (10 products, ~2^-28 of the
//   operand scales, orders of magnitude inside the fp32 tolerance).  The single-pass engine (ozaki5.cuh) cuts 4 or 5 digits
//   under tight scales.  The GEMM itself is the shared warpgroup-MMA digit GEMM (digit_gemm.cuh).  Operands are pre-packed in
//   the no-swizzle K-major core-matrix layout, so each pipeline stage is a few contiguous 1-D bulk-TMA copies.
#pragma once
#include "common.cuh"
#include "digit_gemm.cuh"
#include "kernel_fn.cuh"
#include <cfloat>

namespace tb {
namespace oz {

constexpr int S21 = 6;             // digits per operand of the 21-product engine
constexpr double FILL = 0.4975;    // tight split: |x̂| bound (the largest 5-digit balanced value is 0.49804)

// candidates per K* digit tile of a GEMM that computes with S digits
template <int S> struct Geo;
template <> struct Geo<6> { static constexpr int NT = 128; };
template <> struct Geo<5> { static constexpr int NT = 192; };
template <> struct Geo<4> { static constexpr int NT = 128; };
template <> struct Geo<3> { static constexpr int NT = 128; };

template <int S> __host__ __device__ constexpr double two_pow_8S() {  // 2^48 / 2^40 / 2^32 / 2^24
  return S == 6 ? 281474976710656.0 : S == 5 ? 1099511627776.0 : S == 4 ? 4294967296.0 : 16777216.0;
}

// v = Σ_{p=1..S} d_p 256^(S-p), d_p in [-128,127]: the ordinary base-256 digits of v + Σ 128·256^i are d_p + 128, so the int8
// digits are the bytes of (v + 0x80..80) ^ 0x80..80 (no carry chain); byte 0 = least significant digit d_S
template <int S>
__device__ __forceinline__ void digit_bytes(long long v, uint32_t& lo, uint32_t& hi) {
  constexpr unsigned long long K = S == 6 ? 0x0000808080808080ULL : S == 5 ? 0x0000008080808080ULL : S == 4 ? 0x0000000080808080ULL
                                                                                                              : 0x0000000000808080ULL;
  const unsigned long long w = ((unsigned long long)v + K) ^ K;
  lo = (uint32_t)w;
  hi = (uint32_t)(w >> 32);
}
// element JJ (0..15) of the lane's 16-byte rows: plane p (0 = most significant digit) takes byte S-1-p of the word
template <int S, int JJ>
__device__ __forceinline__ void scatter(uint32_t (&pk)[S][4], uint32_t lo, uint32_t hi) {
#pragma unroll
  for (int p = 0; p < S; ++p) {
    const int b = S - 1 - p;
    if (b == 5) {
      pk[p][JJ >> 2] = put_byte<JJ & 3, 1>(pk[p][JJ >> 2], hi);
    } else if (b == 4) {
      pk[p][JJ >> 2] = put_byte<JJ & 3, 0>(pk[p][JJ >> 2], hi);
    } else if (b == 3) {
      pk[p][JJ >> 2] = put_byte<JJ & 3, 3>(pk[p][JJ >> 2], lo);
    } else if (b == 2) {
      pk[p][JJ >> 2] = put_byte<JJ & 3, 2>(pk[p][JJ >> 2], lo);
    } else if (b == 1) {
      pk[p][JJ >> 2] = put_byte<JJ & 3, 1>(pk[p][JJ >> 2], lo);
    } else {
      pk[p][JJ >> 2] = put_byte<JJ & 3, 0>(pk[p][JJ >> 2], lo);
    }
  }
}
template <int S>
__device__ __forceinline__ void scatter_rt(uint32_t (&pk)[S][4], int jj, uint32_t lo, uint32_t hi) {
  switch (jj) {  // jj is a compile-time constant after unrolling: the switch folds away
    case 0: scatter<S, 0>(pk, lo, hi); break;
    case 1: scatter<S, 1>(pk, lo, hi); break;
    case 2: scatter<S, 2>(pk, lo, hi); break;
    case 3: scatter<S, 3>(pk, lo, hi); break;
    case 4: scatter<S, 4>(pk, lo, hi); break;
    case 5: scatter<S, 5>(pk, lo, hi); break;
    case 6: scatter<S, 6>(pk, lo, hi); break;
    case 7: scatter<S, 7>(pk, lo, hi); break;
    case 8: scatter<S, 8>(pk, lo, hi); break;
    case 9: scatter<S, 9>(pk, lo, hi); break;
    case 10: scatter<S, 10>(pk, lo, hi); break;
    case 11: scatter<S, 11>(pk, lo, hi); break;
    case 12: scatter<S, 12>(pk, lo, hi); break;
    case 13: scatter<S, 13>(pk, lo, hi); break;
    case 14: scatter<S, 14>(pk, lo, hi); break;
    default: scatter<S, 15>(pk, lo, hi); break;
  }
}

// ------------------------------------------------------------------------------------------------
// once per BO step: the left operands of the digit GEMM.  full = 0: lower-triangular Linv (column-major, ld = N; row n has
// the columns k <= n); full = 1: the dense symmetric K^-1 given by its lower triangle (column-major, ld = N), full rows.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ double sym_at(const double* __restrict__ A, int64_t N, int64_t n, int64_t k) {
  return n >= k ? A[n + k * N] : A[k + n * N];
}

// One CTA per row, two scale rules:
//   rowsum == nullptr (21-product split): rowscale[n] = 2^e_n > 2 max_k |A[n,k]|, so |x|/2^e < 1/4 and the top digit fits
//   otherwise (tight split):               rowscale[n] = max_k |A[n,k]| / FILL (1 for empty / padded rows), rowsum[n] = Σ_k A[n,k]
__global__ void rowstats_kernel(const double* __restrict__ A, int64_t N, int64_t rows, int full, double* __restrict__ rowscale,
                                double* __restrict__ rowsum) {
  const int64_t n = blockIdx.x;
  double mx = 0.0, sm = 0.0;
  if (n < N)
    for (int64_t k = threadIdx.x, kend = full ? N : n + 1; k < kend; k += blockDim.x) {
      const double v = sym_at(A, N, n, k);
      mx = fmax(mx, fabs(v));
      sm += v;
    }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    sm += __shfl_xor_sync(0xffffffffu, sm, o);
  }
  __shared__ double smx[8], ssm[8];
  if ((threadIdx.x & 31) == 0) {
    smx[threadIdx.x >> 5] = mx;
    ssm[threadIdx.x >> 5] = sm;
  }
  __syncthreads();
  if (threadIdx.x == 0 && n < rows) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) {
      mx = fmax(mx, smx[w]);
      sm += ssm[w];
    }
    if (rowsum) {
      rowscale[n] = mx > 0.0 ? mx / FILL : 1.0;
      rowsum[n] = sm;
    } else {
      int e = 0;
      if (mx > 0.0) {
        frexp(mx, &e);  // mx = m 2^e, m in [0.5, 1)
        e += 2;
      }
      rowscale[n] = ldexp(1.0, e);
    }
  }
}

// S digit planes of v = rint(A[n,k] / rowscale[n] · 2^(8S)) in the GEMM's stage layout.  full = 0: grid (2 NB, NB), row-block I
// spans stages [0, 2(I+1)), packed triangularly; full = 1: grid (nst, NB), every row-block spans all nst stages.
template <int S>
__global__ void digits_kernel(const double* __restrict__ A, int64_t N, int nst, int full, const double* __restrict__ rowscale,
                              int8_t* __restrict__ AS) {
  const int I = blockIdx.y, kc = blockIdx.x;
  if (!full && kc >= 2 * (I + 1)) return;
  int8_t* dst = AS + ((full ? (int64_t)I * nst : a_stage_offset(I)) + kc) * (int64_t)(S * ATILE);
  for (int e = threadIdx.x; e < 128 * KST; e += blockDim.x) {
    const int r = e % 128, kin = e / 128;  // r fastest: column-major source is contiguous in n
    const int64_t n = (int64_t)I * 128 + r, k = (int64_t)kc * KST + kin;
    long long v = 0;
    if (n < N && (full ? k < N : k <= n)) v = __double2ll_rn(sym_at(A, N, n, k) / rowscale[n] * two_pow_8S<S>());
    uint32_t lo, hi;
    digit_bytes<S>(v, lo, hi);
    const unsigned long long w = ((unsigned long long)hi << 32) | lo;
    const int off = (r >> 3) * SBO + (kin >> 4) * LBO + (r & 7) * 16 + (kin & 15);
#pragma unroll
    for (int p = 0; p < S; ++p) dst[p * ATILE + off] = (int8_t)((w >> (8 * (S - 1 - p))) & 0xff);
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
  int8_t* tile = BS + (int64_t)tile_id * nst * (S21 * ATILE) + w * SBO + ch * LBO + cl * 16;
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
    uint32_t pk[S21][4];
#pragma unroll
    for (int p = 0; p < S21; ++p) pk[p][0] = pk[p][1] = pk[p][2] = pk[p][3] = 0u;
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
      digit_bytes<S21>(__double2ll_rn(kval * inv_bscale_2p48), wl, wh);
      scatter_rt<S21>(pk, j, wl, wh);
    }
#pragma unroll
    for (int p = 0; p < S21; ++p)
      *reinterpret_cast<uint4*>(tile + (int64_t)kc * (S21 * ATILE) + p * ATILE) = make_uint4(pk[p][0], pk[p][1], pk[p][2], pk[p][3]);
    __syncthreads();  // everyone is done with xs_s[buf] before the next iteration's prefetch overwrites it
  }
  macc += __shfl_xor_sync(0xffffffffu, macc, 8);
  macc += __shfl_xor_sync(0xffffffffu, macc, 16);
  if (ch == 0) mean_out[(int64_t)tile_id * 128 + t_local] = macc + mean_const;
}

}  // namespace oz
}  // namespace tb
