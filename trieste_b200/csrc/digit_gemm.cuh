// The digit GEMM of the INT8 engine (ozaki.cuh, ozaki5.cuh: 3 - 6 digits), on Hopper warpgroup MMA.
//
// Operands are int8 digit planes pre-packed in the no-swizzle K-major core-matrix layout (8 rows x 16 bytes per core matrix,
// K-adjacent core matrices LBO apart, 8-row groups SBO apart), so one pipeline stage is a handful of contiguous 1-D bulk-TMA
// copies and the wgmma shared-memory descriptors of the right operand are 32-bit adds.  For a row-block of 128 rows of the
// left factor and a column chunk of CN candidates, level r = p + q (2 <= r <= S + 1) accumulates every digit product
// d_p(A) d_q(B) exactly in int32:
//        A[n,t] = rowscale[n]·out_scale · Σ_{r=2..S+1} 2^(-8r) T_r[n,t]  +  half_var·rowsum[n]
// (rowsum = nullptr: no centring term).  The accumulators live in registers: two consumer warpgroups take rows [0, 64) and
// [64, 128) of the row-block, S levels x CN / 2 int32 registers per thread, which is what bounds CN (32 for S = 6, 64 below;
// the producer warpgroup hands its registers to the consumers with setmaxnreg); a candidate tile of NTB columns is worked
// on as NTB / CN chunks.  The left operand is register-sourced: per digit plane each warp loads its 16 rows with ldmatrix
// once and issues that plane's S + 1 - p MMAs against the shared-memory descriptors of the K* planes, so a plane is read
// from shared memory once instead of once per pair.  Each plane's MMAs are one wgmma group; one group stays in flight while
// the next plane is loaded, and a stage is released when the last group that reads it has retired.  One lane of the
// producer warpgroup streams the stages through a STAGES-deep mbarrier ring.  The grid is persistent: work item = (candidate tile, chunk, row-block group g),
// item = (tile·NCH + chunk)·G + g, CTA c takes items c, c + gridDim.x, ... (co-running CTAs share few candidate tiles, so the
// K* digits stay in L2; the serpentine row-block assignment gives every group the same cost).
//   EPI_SUMSQ: partial[g][t] = Σ_{rows n of group g} A[n,t]^2  (variance path)
//   EPI_STORE: A itself, fp64, candidate-major [t][lda]  (joint / gradient paths)
//   EPI_SPLIT: split-K over (tile, chunk, row-block, stage range) units, the int32 levels summed in a scratch, and
//              split_epilogue_kernel runs the EPI_SUMSQ epilogue on the sums (the screened argmax's rounds of few tiles)
// a_planes / b_planes: digit planes STORED per stage of the left / right operand (>= S): a GEMM computing with S digits reads
// the S most significant planes of a wider split.  full_rows = 0: lower-triangular left factor (Linv), row-block I spans
// stages [0, 2(I+1)), packed triangularly; full_rows = 1: dense square left factor, every row-block spans all nst stages.
#pragma once
#include "common.cuh"
#include "kernel_fn.cuh"

namespace tb {
namespace oz {

constexpr int KST = 64;                      // K bytes (= k columns) per pipeline stage
constexpr uint32_t LBO = 128;                // core matrices adjacent in K (no-swizzle K-major layout)
constexpr uint32_t SBO = (KST / 16) * 128;   // 8-row groups
constexpr int ATILE = 128 * KST;             // one digit plane of a 128-row block of the left factor: 8 KB

__host__ __device__ inline int64_t a_stage_offset(int I) {  // stages before row-block I: Σ 2(i+1)
  return (int64_t)I * (I + 1);
}

// insert byte SRC (0..3) of w into byte POS (0..3) of acc: one PRMT
template <int POS, int SRC>
__device__ __forceinline__ uint32_t put_byte(uint32_t acc, uint32_t w) {
  constexpr uint32_t sel = (POS == 0 ? (4u + SRC) : 0u) | ((POS == 1 ? (4u + SRC) : 1u) << 4) | ((POS == 2 ? (4u + SRC) : 2u) << 8) |
                           ((POS == 3 ? (4u + SRC) : 3u) << 12);
  return __byte_perm(acc, w, sel);
}

}  // namespace oz

namespace dg {

using oz::ATILE;
using oz::KST;
using oz::LBO;
using oz::SBO;

constexpr int STAGES = 3;
constexpr int CONSUMER_WARPS = 8;                     // two warpgroups
constexpr int THREADS = CONSUMER_WARPS * 32 + 128;    // + the producer warpgroup (setmaxnreg acts on whole warpgroups)
// per-thread registers after setmaxnreg: 128 · 40 + 256 · 232 = 64512 of the 64K register file, which is also what the
// launch allocates (168 per thread at __launch_bounds__(384, 1))
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;
enum { EPI_SUMSQ = 0, EPI_STORE = 1, EPI_SPLIT = 2 };

__host__ __device__ constexpr int chunk_cols_of(int S) { return S >= 6 ? 32 : 64; }
template <int S> __host__ __device__ constexpr int chunk_cols() { return chunk_cols_of(S); }
template <int S> __host__ __device__ constexpr int stage_bytes() { return S * (ATILE + chunk_cols<S>() * KST); }
template <int S> __host__ __device__ constexpr size_t smem_bytes() {  // stages + barriers + per-warp column sums
  return (size_t)STAGES * stage_bytes<S>() + 256 + (size_t)CONSUMER_WARPS * chunk_cols<S>() * sizeof(double);
}

// Hopper shared-memory matrix descriptor, no swizzle: start >> 4 | LBO >> 4 << 16 | SBO >> 4 << 32 (layout type 0)
__device__ __forceinline__ uint64_t smem_desc(uint32_t saddr) {
  return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)((LBO >> 4) & 0x3FFF) << 16) | ((uint64_t)((SBO >> 4) & 0x3FFF) << 32);
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// The A fragment of one k32 step of an 8-bit wgmma: the warp's 16 rows x 32 bytes as four 8 x 16-byte core matrices
// (register j: rows +8 if j is odd, bytes +16 if j >= 2), each 128 contiguous bytes of the no-swizzle layout.
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&a)[4], uint32_t saddr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(a[0]), "=r"(a[1]), "=r"(a[2]), "=r"(a[3])
               : "r"(saddr)
               : "memory");
}

// D(64 x N, s32) += A(64 x 32, s8) B(N x 32, s8)^T, A from registers, B K-major in shared memory
#define TB_R4(i) "+r"(d[i]), "+r"(d[i + 1]), "+r"(d[i + 2]), "+r"(d[i + 3])
__device__ __forceinline__ void wgmma_s8(uint32_t (&d)[16], const uint32_t (&a)[4], uint64_t db) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %21, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16,%17,%18,%19}, %20, p;\n}\n"
      : TB_R4(0), TB_R4(4), TB_R4(8), TB_R4(12)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(1));
}
__device__ __forceinline__ void wgmma_s8(uint32_t (&d)[32], const uint32_t (&a)[4], uint64_t db) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
      "{%32,%33,%34,%35}, %36, p;\n}\n"
      : TB_R4(0), TB_R4(4), TB_R4(8), TB_R4(12), TB_R4(16), TB_R4(20), TB_R4(24), TB_R4(28)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(1));
}
#undef TB_R4

// keeps the compiler from moving reads / writes of the accumulators across the asynchronous MMAs
template <int S, int NR>
__device__ __forceinline__ void fence_acc(uint32_t (&acc)[S][NR]) {
#pragma unroll
  for (int l = 0; l < S; ++l)
#pragma unroll
    for (int i = 0; i < NR; ++i) asm volatile("" : "+r"(acc[l][i])::"memory");
}

// exact int32 -> fp64 on the ALU + fp64 pipes: bits(2^52 + 2^31 + t) = {0x43300000, t ^ 0x80000000}
__device__ __forceinline__ double int_to_double(uint32_t t) {
  return __hiloint2double(0x43300000, (int)(t ^ 0x80000000u)) - 4503601774854144.0;  // 2^52 + 2^31
}

__host__ __device__ inline int rowblock_stages(int I, int nst, int full_rows) { return full_rows ? nst : min(2 * (I + 1), nst); }

// EPI_SPLIT work units per (candidate tile, chunk): every row-block's stages in ranges of kper, numbered by row-block, then range
__host__ __device__ inline int split_units(int NB, int nst, int full_rows, int kper) {
  int u = 0;
  for (int I = 0; I < NB; ++I) u += (rowblock_stages(I, nst, full_rows) + kper - 1) / kper;
  return u;
}

// The i-th (row-block I, stages [k0, k1)) of work item g of a (tile, chunk); false past the last.  EPI_SUMSQ / EPI_STORE: g is a
// row-block group, whose row-blocks are taken whole in serpentine order; EPI_SPLIT: g is a unit, one range of one row-block.
template <int EPI>
__device__ __forceinline__ bool item_range(int g, int i, int G, int NB, int nst, int full_rows, int kper, int& I, int& k0, int& k1) {
  if constexpr (EPI == EPI_SPLIT) {
    if (i > 0) return false;
    for (I = 0; I < NB; ++I) {
      const int nk = rowblock_stages(I, nst, full_rows), p = (nk + kper - 1) / kper;
      if (g < p) {
        k0 = g * kper;
        k1 = min(nk, k0 + kper);
        return true;
      }
      g -= p;
    }
    return false;
  } else {
    I = serpentine_rowblock(i, g, G);
    k0 = 0;
    k1 = rowblock_stages(I, nst, full_rows);
    return I < NB;
  }
}

// The epilogue of one row-block from its S levels of int32 accumulators in the m64nCN fragment layout of consumer warp `warp`:
// register 4j + e holds row 16 wq + lane/4 (+8 for e >= 2) of warpgroup wg's 64, column 8j + 2 (lane % 4) + (e & 1) of the
// chunk.  EPI_SUMSQ adds the warp's 16 rows of A^2 to colbuf[warp] (row-blocks in the order of the calls); EPI_STORE writes A.
template <int S, int EPI, int NTB>
__device__ __forceinline__ void rowblock_epilogue(const uint32_t (&acc)[S][chunk_cols<S>() / 2], int I, int tile, int c, int warp, int lane,
                                                  const double* __restrict__ rowscale, const double* __restrict__ rowsum,
                                                  double out_scale, double half_var, double (*colbuf)[chunk_cols<S>()],
                                                  double* __restrict__ Aplain, int64_t lda) {
  constexpr int CN = chunk_cols<S>();
  const int wg = warp >> 2, wq = warp & 3;
  const int64_t r0 = (int64_t)I * 128 + wg * 64 + wq * 16 + (lane >> 2), r1 = r0 + 8;
  const double rs0 = rowscale[r0] * out_scale * 0x1p-16, rs1 = rowscale[r1] * out_scale * 0x1p-16;
  const double rc0 = rowsum ? rowsum[r0] * half_var : 0.0, rc1 = rowsum ? rowsum[r1] * half_var : 0.0;
#pragma unroll
  for (int j = 0; j < CN / 8; ++j) {
    double a[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      // Horner over the levels, least significant first: v = ((T_{S+1} 2^-8 + T_S) 2^-8 + ...) + T_2
      double v = int_to_double(acc[S - 1][4 * j + e]);
#pragma unroll
      for (int l = S - 2; l >= 0; --l) v = fma(v, 0x1p-8, int_to_double(acc[l][4 * j + e]));
      a[e] = e < 2 ? fma(v, rs0, rc0) : fma(v, rs1, rc1);
    }
    const int col = 8 * j + 2 * (lane & 3);
    if constexpr (EPI == EPI_STORE) {
      double* dst = Aplain + ((int64_t)tile * NTB + (int64_t)c * CN + col) * lda;
      dst[r0] = a[0];
      dst[lda + r0] = a[1];
      dst[r1] = a[2];
      dst[lda + r1] = a[3];
    } else {
      double s0 = fma(a[0], a[0], a[2] * a[2]), s1 = fma(a[1], a[1], a[3] * a[3]);
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) {
        s0 += __shfl_xor_sync(0xffffffffu, s0, o);
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      }
      if (lane < 4) {  // the warp's 16 rows, accumulated over the item's row-blocks in a fixed order
        colbuf[warp][col] += s0;
        colbuf[warp][col + 1] += s1;
      }
    }
  }
}

// EPI_SUMSQ, after an item's last row-block: dst[col] = Σ_w colbuf[w][col] in warp order, colbuf zeroed.  Threads 0 .. 255
// (the consumer warps) take part.
template <int CN>
__device__ __forceinline__ void colbuf_flush(double (*colbuf)[CN], double* __restrict__ dst) {
  asm volatile("bar.sync 1, %0;" ::"n"(CONSUMER_WARPS * 32) : "memory");
  if (threadIdx.x < CN) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < CONSUMER_WARPS; ++w) {
      s += colbuf[w][threadIdx.x];
      colbuf[w][threadIdx.x] = 0.0;
    }
    dst[threadIdx.x] = s;
  }
  asm volatile("bar.sync 1, %0;" ::"n"(CONSUMER_WARPS * 32) : "memory");
}

// EPI_SPLIT (split-K for a few candidate tiles, whose row-block groups would leave most SMs idle): G units per (tile, chunk),
// each adds its int32 level accumulators to the zeroed acc_out[(tile NCH + chunk) NB + I][S NR][256 consumer threads].
// Integer addition is exact and commutative, so the sums are those one CTA would accumulate; split_epilogue_kernel finishes.
template <int S, int EPI, int NTB>
__global__ void __launch_bounds__(THREADS, 1)
digit_gemm_kernel(const int8_t* __restrict__ AS, const int8_t* __restrict__ BS, const double* __restrict__ rowscale,
                  const double* __restrict__ rowsum, int NB, int nst, int G, int tiles, int64_t McPad, double out_scale,
                  double half_var, int a_planes, int b_planes, int full_rows, double* __restrict__ partial,
                  double* __restrict__ Aplain, int64_t lda, int kper, int* __restrict__ acc_out) {
  constexpr int CN = chunk_cols<S>(), NCH = NTB / CN, BCH = CN * KST, BTILE = NTB * KST, STAGE = stage_bytes<S>(), NR = CN / 2;
  static_assert(NTB % CN == 0, "a candidate tile is a whole number of column chunks");
  extern __shared__ __align__(1024) unsigned char smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)STAGES * STAGE);
  uint64_t* empty = full + STAGES;
  double (*colbuf)[CN] = reinterpret_cast<double (*)[CN]>(smem + (size_t)STAGES * STAGE + 256);  // [consumer warp][column]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nitems = tiles * NCH * G;
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], CONSUMER_WARPS);
    }
    fence_barrier_init();
  }
  for (int i = threadIdx.x; i < CONSUMER_WARPS * CN; i += blockDim.x) colbuf[i / CN][i % CN] = 0.0;
  __syncthreads();

  if (warp >= CONSUMER_WARPS) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == CONSUMER_WARPS && lane == 0) {
      int st = 0;
      uint32_t ph = 0;
      for (int item = blockIdx.x; item < nitems; item += gridDim.x) {
        const int g = item % G, tc = item / G, tile = tc / NCH, c = tc % NCH;
        const int8_t* bTile = BS + (int64_t)tile * nst * ((int64_t)b_planes * BTILE) + (int64_t)c * BCH;
        int I, k0, k1;
        for (int i = 0; item_range<EPI>(g, i, G, NB, nst, full_rows, kper, I, k0, k1); ++i) {
          const int8_t* aRow = AS + (full_rows ? (int64_t)I * nst : oz::a_stage_offset(I)) * ((int64_t)a_planes * ATILE);
          for (int kc = k0; kc < k1; ++kc) {
            mbar_wait(&empty[st], ph ^ 1);
            unsigned char* dst = smem + (size_t)st * STAGE;
            mbar_expect_tx(&full[st], STAGE);
            bulk_g2s(dst, aRow + (int64_t)kc * ((int64_t)a_planes * ATILE), S * ATILE, &full[st]);  // the S leading planes
            const int8_t* b = bTile + (int64_t)kc * ((int64_t)b_planes * BTILE);
#pragma unroll
            for (int p = 0; p < S; ++p) bulk_g2s(dst + S * ATILE + p * BCH, b + (int64_t)p * BTILE, BCH, &full[st]);
            if (++st == STAGES) { st = 0; ph ^= 1; }
          }
        }
      }
    }
    return;
  }

  // ===================== consumer warpgroups: MMA + epilogue =====================
  setmaxnreg_inc<CONSUMER_REGS>();
  const int wg = warp >> 2, wq = warp & 3;
  // ldmatrix row address of this lane: row lane % 8 of core matrix lane / 8 of the warp's 16 rows x 32 bytes (ldmatrix_x4)
  const uint32_t a_lane = (uint32_t)((wg * 8 + wq * 2 + ((lane >> 3) & 1)) * (int)SBO + (lane >> 4) * (int)LBO + (lane & 7) * 16);
  uint32_t acc[S][NR];
  int st = 0;
  uint32_t ph = 0;
  for (int item = blockIdx.x; item < nitems; item += gridDim.x) {
    const int g = item % G, tc = item / G, tile = tc / NCH, c = tc % NCH;
    int I, k0, k1;
    for (int i = 0; item_range<EPI>(g, i, G, NB, nst, full_rows, kper, I, k0, k1); ++i) {
#pragma unroll
      for (int l = 0; l < S; ++l)
#pragma unroll
        for (int j = 0; j < NR; ++j) acc[l][j] = 0u;
      fence_acc(acc);
      int held = -1;  // the previous stage: its last MMA group may still be running
      for (int kc = k0; kc < k1; ++kc) {
        mbar_wait(&full[st], ph);
        const uint32_t base = smem_u32(smem + (size_t)st * STAGE);
        const uint64_t b0 = smem_desc(base + (uint32_t)(S * ATILE));
#pragma unroll
        for (int p = 1; p <= S; ++p) {
          uint32_t a[KST / 32][4];
#pragma unroll
          for (int kk = 0; kk < KST / 32; ++kk) ldmatrix_x4(a[kk], base + a_lane + (uint32_t)((p - 1) * ATILE + kk * 2 * (int)LBO));
          // all groups but the last one have retired: the registers of the group before it can be reused, and at the
          // second plane the previous stage's last group is done, so this warp's reads of that stage are over
          wgmma_wait<1>();
          if (p == 2 && held >= 0) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[held]);
          }
          wgmma_fence();
#pragma unroll
          for (int q = 1; q <= S + 1 - p; ++q)
#pragma unroll
            for (int kk = 0; kk < KST / 32; ++kk) wgmma_s8(acc[p + q - 2], a[kk], b0 + (uint64_t)(((q - 1) * BCH + kk * 2 * (int)LBO) >> 4));
          wgmma_commit();
        }
        held = st;
        if (++st == STAGES) { st = 0; ph ^= 1; }
      }
      wgmma_wait<0>();
      fence_acc(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[held]);
      if constexpr (EPI == EPI_SPLIT) {
        int* dst = acc_out + ((int64_t)tc * NB + I) * (S * NR * CONSUMER_WARPS * 32) + threadIdx.x;
#pragma unroll
        for (int l = 0; l < S; ++l)
#pragma unroll
          for (int j = 0; j < NR; ++j) atomicAdd(dst + (l * NR + j) * (CONSUMER_WARPS * 32), (int)acc[l][j]);
      } else {
        rowblock_epilogue<S, EPI, NTB>(acc, I, tile, c, warp, lane, rowscale, rowsum, out_scale, half_var, colbuf, Aplain, lda);
      }
    }
    if constexpr (EPI == EPI_SUMSQ) colbuf_flush<CN>(colbuf, partial + (int64_t)g * McPad + (int64_t)tile * NTB + (int64_t)c * CN);
  }
}

// The EPI_SUMSQ epilogue of a split-K GEMM (EPI_SPLIT) of `tiles` candidate tiles over G row-block groups: CTA (tile, chunk, g)
// loads the summed accumulators of group g's row-blocks in serpentine order into the same fragment layout, per consumer
// thread, and runs the same epilogue, so partial[g][t] is byte for byte what digit_gemm_kernel<S, EPI_SUMSQ> writes.
template <int S, int NTB>
__global__ void __launch_bounds__(CONSUMER_WARPS * 32, 1)
split_epilogue_kernel(const int* __restrict__ acc_in, const double* __restrict__ rowscale, const double* __restrict__ rowsum, int NB,
                      int G, int64_t McPad, double out_scale, double half_var, double* __restrict__ partial) {
  constexpr int CN = chunk_cols<S>(), NCH = NTB / CN, NR = CN / 2;
  __shared__ double colbuf[CONSUMER_WARPS][CN];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = blockIdx.x % G, tc = blockIdx.x / G, tile = tc / NCH, c = tc % NCH;
  for (int i = threadIdx.x; i < CONSUMER_WARPS * CN; i += blockDim.x) colbuf[i / CN][i % CN] = 0.0;
  __syncthreads();
  for (int i = 0;; ++i) {
    const int I = serpentine_rowblock(i, g, G);
    if (I >= NB) break;
    const int* src = acc_in + ((int64_t)tc * NB + I) * (S * NR * CONSUMER_WARPS * 32) + threadIdx.x;
    uint32_t acc[S][NR];
#pragma unroll
    for (int l = 0; l < S; ++l)
#pragma unroll
      for (int j = 0; j < NR; ++j) acc[l][j] = (uint32_t)src[(l * NR + j) * (CONSUMER_WARPS * 32)];
    rowblock_epilogue<S, EPI_SUMSQ, NTB>(acc, I, tile, c, warp, lane, rowscale, rowsum, out_scale, half_var, colbuf, nullptr, 0);
  }
  colbuf_flush<CN>(colbuf, partial + (int64_t)g * McPad + (int64_t)tile * NTB + (int64_t)c * CN);
}

// ---- host side ----
inline int sm_count(int* n) {
  int dev = 0;
  TB_CUDA(cudaGetDevice(&dev));
  TB_CUDA(cudaDeviceGetAttribute(n, cudaDevAttrMultiProcessorCount, dev));
  return 0;
}

template <int S, int EPI, int NTB>
inline int set_smem() {
  TB_CUDA(cudaFuncSetAttribute(digit_gemm_kernel<S, EPI, NTB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes<S>()));
  return 0;
}

// persistent launch: one CTA per SM, fewer when there are fewer work items
template <int S, int EPI, int NTB>
inline int launch(cudaStream_t st, const int8_t* AS, const int8_t* BS, const double* rowscale, const double* rowsum, int NB, int nst,
                  int G, int tiles, int64_t McPad, double out_scale, double half_var, int a_planes, int b_planes, int full_rows,
                  double* partial, double* Aplain, int64_t lda, int kper = 0, int* acc = nullptr) {
  int sms = 0;
  TB_TRY(sm_count(&sms));
  const int64_t items = (int64_t)tiles * (NTB / chunk_cols<S>()) * G;
  const int grid = (int)std::min<int64_t>(sms, items);
  if (grid <= 0) return 0;
  digit_gemm_kernel<S, EPI, NTB><<<grid, THREADS, smem_bytes<S>(), st>>>(AS, BS, rowscale, rowsum, NB, nst, G, tiles, McPad, out_scale,
                                                                         half_var, a_planes, b_planes, full_rows, partial, Aplain, lda,
                                                                         kper, acc);
  TB_LAUNCHED();
  TB_CUDA(cudaGetLastError());
  return 0;
}

// Split-K for an EPI_SUMSQ GEMM whose tiles * NCH * G work items fill less than one wave of SMs: the stages per unit, the
// fewest (at least 8: each unit adds S * 128 * CN int32 to the scratch) that keep the units within one wave, at most a whole
// row-block.  0: no split.
inline int split_kper(int S, int NTB, int tiles, int G, int NB, int nst, int full_rows) {
  const int nch = NTB / chunk_cols_of(S);
  if ((int64_t)tiles * nch * G >= NUM_SMS) return 0;
  int64_t stages = 0;
  for (int I = 0; I < NB; ++I) stages += rowblock_stages(I, nst, full_rows);
  stages *= (int64_t)tiles * nch;
  int kper = (int)std::min<int64_t>(nst, std::max<int64_t>(8, (stages + NUM_SMS - 1) / NUM_SMS));
  while (kper < nst && (int64_t)tiles * nch * split_units(NB, nst, full_rows, kper) > NUM_SMS) ++kper;
  return kper;
}
template <int S> inline size_t split_acc_bytes(int tiles, int NTB, int NB) {
  return (size_t)tiles * (NTB / chunk_cols<S>()) * NB * S * (chunk_cols<S>() / 2) * (CONSUMER_WARPS * 32) * sizeof(int);
}

// EPI_SUMSQ through the split: zero the accumulator scratch acc (split_acc_bytes), the units, then the epilogue over G groups
template <int S, int NTB>
inline int launch_split(cudaStream_t st, const int8_t* AS, const int8_t* BS, const double* rowscale, const double* rowsum, int NB,
                        int nst, int G, int tiles, int64_t McPad, double out_scale, double half_var, int a_planes, int b_planes,
                        int full_rows, int kper, int* acc, double* partial) {
  TB_CUDA(cudaMemsetAsync(acc, 0, split_acc_bytes<S>(tiles, NTB, NB), st));
  TB_TRY((launch<S, EPI_SPLIT, NTB>(st, AS, BS, rowscale, rowsum, NB, nst, split_units(NB, nst, full_rows, kper), tiles, McPad,
                                    out_scale, half_var, a_planes, b_planes, full_rows, nullptr, nullptr, 0, kper, acc)));
  split_epilogue_kernel<S, NTB><<<tiles * (NTB / chunk_cols<S>()) * G, CONSUMER_WARPS * 32, 0, st>>>(acc, rowscale, rowsum, NB, G, McPad,
                                                                                                   out_scale, half_var, partial);
  TB_LAUNCHED();
  TB_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace dg
}  // namespace tb
