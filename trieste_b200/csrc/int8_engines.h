// The int8 digit engine, host side (int8_engines.cu; kernels in ozaki.cuh and ozaki5.cuh).  tb_api.cu picks the engine of a
// call; int8_select picks the digit count, which every function below runs with.
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include <cstdint>
struct tb_gp;
namespace tb {
int int8_init();  // kernel attributes (once per process)
// The lazy builds a call on the int8 engine needs after a cache refresh, and the digit count it computes with, recorded in
// gp->digits.S: the admitted split's (5 on fp64 handles, 4 on fp32 ones) when the a-priori error estimate admits the handle
// and, with need_v, the V GEMM's own estimate does too; otherwise 6.  need_v: the call also needs V = K^-1 K* (gradients); the
// dense K^-1 in gp->dKinv must then be current.
int int8_select(tb_gp* gp, bool need_v);
int int8_tile_width(const tb_gp* gp);     // candidates per K* digit tile
size_t int8_tile_bytes(const tb_gp* gp);  // K* digit bytes per candidate tile
// k-split of the K* generation: the training rows are split into ksplit ranges of kc_per stages (ksplit = 1: no split).  A
// candidate's mean depends on this pair only, never on the other candidates of the launch.
struct KSplit {
  int ksplit = 1, kc_per = 0;
};
KSplit int8_kstar_split(const tb_gp* gp, int tiles);  // the split a launch over `tiles` candidate tiles uses
// K* digit tiles of mc device candidates into BS, their posterior means into mean.  split == nullptr: int8_kstar_split(gp,
// tiles); otherwise that split (the screened argmax reproduces a chunk's means).  wide: the k-stages spread over many more CTAs
// than `split` has, the same digits and means.
int int8_kstar(tb_gp* gp, const double* Xc_dev, int64_t mc, int tiles, int8_t* BS, double* mean, const KSplit* split = nullptr,
               bool wide = false);
// variance path: partial[g][t] = sum over the rows of group g of A[n,t]^2, A = Linv K*.  kper > 0: split-K in units of kper
// stages (int8_split_kper), the same partial.
int int8_variance(tb_gp* gp, const int8_t* BS, int tiles, int G, int64_t McPad, double* partial, int kper = 0);
// The split-K stages per unit for a variance GEMM over `tiles` tiles and G row-block groups, 0 when its groups fill a wave
int int8_split_kper(const tb_gp* gp, int tiles, int G);
// store path: out[t][lda] = (left K*)[., t], kinv = false: Linv (A of the joint paths), true: dense K^-1 (V of the gradient path)
int int8_store(tb_gp* gp, bool kinv, const int8_t* BS, int tiles, int G, int64_t McPad, double* out, int64_t lda);
// after int8_select: digit products of the variance GEMM, and the a-priori error estimate of the admitted split (0 when it was
// not admitted)
void int8_info(const tb_gp* gp, int* products, double* estimate);
void int8_pin_full(tb_gp* gp, bool full);  // tb_gp_set_engine: 2 pins 6 digits, 1 lets the estimate choose
}  // namespace tb
