// Single-pass digit engine (ozaki5.cuh), host entry points used by tb_api.cu.
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include <cstdint>
struct tb_gp;
namespace tb {
int oz5_init();                              // kernel attributes (once per process)
int oz5_ensure(tb_gp* gp);                   // (re)build row stats + digit tiles after a cache refresh; sets gp->oz5_mode / oz5_planes
int oz5_ensure_kinv(tb_gp* gp);              // tight digit tiles of the dense K^-1 in gp->dKinv (caller keeps it current); sets kinv5_ok
int oz5_tile_width(const tb_gp* gp);         // candidates per tile in the chosen mode
size_t oz5_tile_bytes(const tb_gp* gp);      // K* digit bytes per candidate tile
// k-split of the K* generation: the training rows are split into ksplit ranges of kc_per stages (ksplit = 1: no split).  A
// candidate's mean depends on this pair only, never on the other candidates of the launch.
struct KSplit {
  int ksplit = 1, kc_per = 0;
};
KSplit oz5_kstar_split(const tb_gp* gp, int tiles);  // the split a launch over `tiles` candidate tiles uses
// split == nullptr: oz5_kstar_split(gp, tiles); otherwise that split (the screened argmax reproduces a chunk's means)
int oz5_launch_kstar(tb_gp* gp, cudaStream_t st, const double* Xc_dev, int64_t mc, int tiles, int8_t* BS, double* mean,
                     const KSplit* split = nullptr);
// variance path: partial[g][t] = sum over the rows of group g of A[n,t]^2, A = Linv K*
int oz5_launch_gemm(tb_gp* gp, cudaStream_t st, const int8_t* BS, int tiles, int G, int64_t McPad, double* partial);
// store path: out[t][lda] = (left K*)[., t], left = 0: Linv (A of the joint paths), 1: dense K^-1 (V of the gradient path)
int oz5_launch_gemm_store(tb_gp* gp, cudaStream_t st, int left, const int8_t* BS, int tiles, int G, double* out, int64_t lda);
}  // namespace tb
