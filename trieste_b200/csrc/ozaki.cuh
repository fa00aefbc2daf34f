// fp64-accurate GEMMs on the INT8 tensor cores (Ozaki error-free splitting): the digit cutting of the left operands.
//
//   A = Linv · K*  is needed to ~2^-46 relative to |row scale|·|K* scale| for the 1e-9·σ_f² variance bar.
//   Each fp64 operand is split into S balanced base-256 digits (int8 in [-128, 127]) under a tight per-row scale:
//        x = scale · Σ_{p=1..S} d_p · 2^(-8p),        |x / scale| <= FILL
//   Products of digit matrices are EXACT in int32 accumulators, and all pairs with the same p + q = r share one
//   accumulator T_r; the pairs p + q <= S + 1 are kept (S = 6: 21 products, |T_r| <= 6 · K · 2^14 < 2^31 for K <= 16384).
//   The digit count, the centred K* generation and the error budget are in ozaki5.cuh; the GEMM itself is the shared
//   warpgroup-MMA digit GEMM (digit_gemm.cuh).  Operands are pre-packed in the no-swizzle K-major core-matrix layout, so each
//   pipeline stage is a few contiguous 1-D bulk-TMA copies.
#pragma once
#include "common.cuh"
#include "digit_gemm.cuh"

namespace tb {
namespace oz {

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

// One CTA per row: rowscale[n] = max_k |A[n,k]| / FILL (1 for empty / padded rows), rowsum[n] = Σ_k A[n,k]
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
    rowscale[n] = mx > 0.0 ? mx / FILL : 1.0;
    rowsum[n] = sm;
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

}  // namespace oz
}  // namespace tb
