// Host side of the single-pass digit engine (ozaki5.cuh): mode selection from an a-priori error bound, digit tiles of Linv,
// launches of the centred K* digit generation and of the digit GEMM.  Called from tb_api.cu (the engine operations).
#include "gp_handle.cuh"
#include "ozaki5.cuh"
#include "oz5_api.h"

namespace tb {

int oz5_init() {
  TB_TRY((dg::set_smem<5, dg::EPI_SUMSQ, oz5::Geo<5>::NT>()));
  TB_TRY((dg::set_smem<5, dg::EPI_STORE, oz5::Geo<5>::NT>()));
  TB_TRY((dg::set_smem<4, dg::EPI_SUMSQ, oz5::Geo<4>::NT>()));
  TB_TRY((dg::set_smem<4, dg::EPI_STORE, oz5::Geo<4>::NT>()));
  TB_TRY((dg::set_smem<3, dg::EPI_SUMSQ, oz5::Geo<3>::NT>()));
  return 0;
}

int oz5_tile_width(const tb_gp* gp) { return gp->oz5_planes == 5 ? oz5::Geo<5>::NT : oz5::Geo<4>::NT; }
size_t oz5_tile_bytes(const tb_gp* gp) {
  return (size_t)gp->nst * (gp->oz5_planes == 5 ? 5 * oz5::btile<5>() : 4 * oz5::btile<4>());
}

// Calibrated a-priori estimate of max |Δvar| / σ_f² when the levels r > S+1 are dropped: per element of A the dropped
// level r = S+2 contributes ~ rowscale·sB·sqrt(6 K)·E[d²]·2^(-8(S+2)) (E[d²] = 256²/12 for uniform balanced digits, K <= N
// terms with independent signs), and Δvar = 2 Σ_n A_n δ_n with Σ A_n² <= σ_f².  The constant (8/5) was calibrated on the
// emulated engine over the benchmark configurations (oracle-side study in DESIGN.md §4c): estimate / measured max = 1.1 .. 5.
static double oz5_estimate(double variance, double max_rowscale, int64_t N, int S) {
  const double sB = 0.5 * variance / oz5::FILL;
  return 1.6 * std::sqrt(variance) * max_rowscale * sB * std::sqrt(6.0 * (double)N) * (65536.0 / 12.0) * std::ldexp(1.0, -8 * (S + 2)) / variance;
}

template <int S>
static int build_digits(tb_gp* gp, cudaStream_t st) {
  const int64_t nstages = oz::a_stage_offset(gp->NB);
  const size_t bytes = (size_t)nstages * S * oz5::ATILE;
  TB_TRY(gp->dAS5.reserve(bytes));
  TB_CUDA(cudaMemsetAsync(gp->dAS5.p, 0, bytes, st));
  oz5::linv_digits_kernel<S><<<dim3(2 * gp->NB, gp->NB), 256, 0, st>>>(gp->dLinv.as<double>(), gp->N, gp->dRowScale5.as<double>(),
                                                                      gp->dAS5.as<int8_t>());
  TB_LAUNCHED();
  TB_CUDA(cudaGetLastError());
  return 0;
}

int oz5_ensure(tb_gp* gp) {
  if (gp->oz5_valid) return 0;
  gp->oz5_mode = 0;
  gp->oz5_planes = 0;
  gp->oz5_est = 0.0;
  if (gp->oz_full || gp->N > 16384) {
    gp->oz5_valid = true;
    return 0;
  }
  cudaStream_t st = gp->stream;
  const int64_t rows = (int64_t)gp->NB * BM;
  gp->nst = (int)((gp->N + oz::KST - 1) / oz::KST);
  {  // squared row norms of the scaled training inputs (expansion-form distances of the K* generation kernel)
    const int64_t xrows = (int64_t)gp->nst * oz::KST;
    TB_TRY(gp->dX2.reserve(sizeof(double) * xrows));
    oz5::row_norms_kernel<<<(unsigned)((xrows + 255) / 256), 256, 0, st>>>(gp->dXs.as<double>(), (int64_t)gp->NB * BM, gp->DP, xrows,
                                                                         gp->dX2.as<double>());
    TB_LAUNCHED();
  }
  TB_TRY(gp->dRowScale5.reserve(sizeof(double) * rows));
  TB_TRY(gp->dRowSum5.reserve(sizeof(double) * rows));
  oz5::linv_rowstats_kernel<<<(unsigned)rows, 256, 0, st>>>(gp->dLinv.as<double>(), gp->N, rows, gp->dRowScale5.as<double>(),
                                                           gp->dRowSum5.as<double>());
  TB_LAUNCHED();
  std::vector<double> h((size_t)gp->N);
  TB_CUDA(cudaMemcpyAsync(h.data(), gp->dRowScale5.p, sizeof(double) * (size_t)gp->N, cudaMemcpyDeviceToHost, st));
  TB_CUDA(cudaStreamSynchronize(st));
  double mx = 0.0;
  for (double v : h) mx = std::max(mx, v);
  // fp64 handles: 5 digits / 15 products if the estimate clears 3e-10 (bar: 1e-9).  fp32 handles (bar: 1e-4): 4 planes are
  // stored; the variance GEMM computes with 3 digits / 6 products if that clears 3e-5, else with all 4 (10 products, one pass);
  // if even 4 digits do not clear it the handle is treated like an fp64 one.  Otherwise: the 6-digit two-pass kernels.
  int mode = 0, planes = 0;
  if (gp->dtype == TB_F32) {
    if (oz5_estimate(gp->variance, mx, gp->N, 3) <= 3e-5) mode = 3, planes = 4;
    else if (oz5_estimate(gp->variance, mx, gp->N, 4) <= 3e-5) mode = 4, planes = 4;
  }
  if (mode == 0 && oz5_estimate(gp->variance, mx, gp->N, 5) <= (gp->dtype == TB_F32 ? 3e-5 : 3e-10)) mode = 5, planes = 5;
  if (planes == 5) TB_TRY(build_digits<5>(gp, st));
  if (planes == 4) TB_TRY(build_digits<4>(gp, st));
  if (mode) gp->oz5_est = oz5_estimate(gp->variance, mx, gp->N, mode);
  gp->oz5_mode = mode;
  gp->oz5_planes = planes;
  gp->kinv5_valid = false;
  gp->oz5_valid = true;
  return 0;
}

// Tight digit tiles of the dense K^-1 (gp->dKinv, lower triangle, ld = N; kept current by ensure_kinv_dense / the rank-m
// growth on append).  The V GEMM has its own admission test: the element error of V = K^-1 k* is
// ~ rowscale(K^-1) sB sqrt(6 N) E[d^2] 2^(-8(S+2)); gradients are held to rtol 1e-6 (fp64) / 1e-3 (fp32) and V enters them
// through sums of ~N terms with |V| ~ 0.1 .. 1, so the element error must stay below ~1e-7 / ~1e-4.
int oz5_ensure_kinv(tb_gp* gp) {
  if (gp->kinv5_valid) return 0;
  gp->kinv5_ok = false;
  if (gp->oz5_planes == 0) {
    gp->kinv5_valid = true;
    return 0;
  }
  cudaStream_t st = gp->stream;
  const int64_t N = gp->N, rows = (int64_t)gp->NB * BM;
  TB_TRY(gp->dKinvScale5.reserve(sizeof(double) * rows));
  TB_TRY(gp->dKinvSum5.reserve(sizeof(double) * rows));
  oz5::sym_rowstats_kernel<<<(unsigned)rows, 256, 0, st>>>(gp->dKinv.as<double>(), N, rows, gp->dKinvScale5.as<double>(),
                                                          gp->dKinvSum5.as<double>());
  TB_LAUNCHED();
  std::vector<double> h((size_t)N);
  TB_CUDA(cudaMemcpyAsync(h.data(), gp->dKinvScale5.p, sizeof(double) * (size_t)N, cudaMemcpyDeviceToHost, st));
  TB_CUDA(cudaStreamSynchronize(st));
  double mx = 0.0;
  for (double v : h) mx = std::max(mx, v);
  const int S = gp->oz5_planes;
  const double sB = 0.5 * gp->variance / oz5::FILL;
  const double eps_v = mx * sB * std::sqrt(6.0 * (double)N) * (65536.0 / 12.0) * std::ldexp(1.0, -8 * (S + 2));
  gp->kinv5_ok = eps_v <= (gp->dtype == TB_F32 ? 1e-4 : 1e-7);
  if (gp->kinv5_ok) {
    const size_t bytes = (size_t)gp->NB * gp->nst * S * oz5::ATILE;
    TB_TRY(gp->dKinvS5.reserve(bytes));
    if (S == 5)
      oz5::sym_digits_kernel<5><<<dim3(gp->nst, gp->NB), 256, 0, st>>>(gp->dKinv.as<double>(), N, gp->nst, gp->dKinvScale5.as<double>(),
                                                                      gp->dKinvS5.as<int8_t>());
    else
      oz5::sym_digits_kernel<4><<<dim3(gp->nst, gp->NB), 256, 0, st>>>(gp->dKinv.as<double>(), N, gp->nst, gp->dKinvScale5.as<double>(),
                                                                      gp->dKinvS5.as<int8_t>());
    TB_LAUNCHED();
    TB_CUDA(cudaStreamSynchronize(st));
    TB_CUDA(cudaGetLastError());
  }
  gp->kinv5_valid = true;
  return 0;
}

// the centre of K* in digit units: the integer nearest to h * inv_b = FILL * 2^(8S); the centre actually subtracted is
// h_eff = centre / inv_b = h * centre / (FILL 2^(8S)), used consistently by the generation kernel and the GEMM epilogue
template <int S>
static double oz5_centre_int() { return std::nearbyint(oz5::FILL * oz5::two_pow_8S<S>()); }
template <int S>
static double oz5_h_eff(double variance) { return 0.5 * variance * oz5_centre_int<S>() / (oz5::FILL * oz5::two_pow_8S<S>()); }

template <int S>
static unsigned kstar_ctas(int tiles) {
  return (unsigned)(((int64_t)tiles * (oz5::Geo<S>::NT / 8) + oz5::KGEN_WARPS - 1) / oz5::KGEN_WARPS);
}

KSplit oz5_kstar_split(const tb_gp* gp, int tiles) {
  const int nst = gp->nst;
  const unsigned ctas = gp->oz5_planes == 5 ? kstar_ctas<5>(tiles) : kstar_ctas<4>(tiles);
  // few tiles (the late rounds of the multi-start optimiser, small predict calls): split the training rows over blockIdx.y so
  // that ~4 CTAs per SM exist; each split covers >= 2 stages
  KSplit s;
  s.kc_per = nst;
  if (ctas < NUM_SMS && nst >= 4) {
    s.ksplit = std::min<int>(nst / 2, (int)((4 * NUM_SMS + ctas - 1) / ctas));
    s.kc_per = (nst + s.ksplit - 1) / s.ksplit;
    s.ksplit = (nst + s.kc_per - 1) / s.kc_per;
  }
  return s;
}

template <int S>
static int launch_kstar_s(tb_gp* gp, cudaStream_t st, const double* Xc_dev, int64_t mc, int tiles, int8_t* BS, double* mean,
                          const KSplit* split) {
  const double* Xs = gp->dXs.as<double>();
  const double* al = gp->dAlpha.as<double>();
  const double* il = gp->dInvLs.as<double>();
  const int N = (int)gp->N, nst = gp->nst, D = gp->D;
  const double var = gp->variance, mc0 = gp->mean_const;
  const double inv_b = oz5::two_pow_8S<S>() * oz5::FILL / (0.5 * var);
  const double dig_c = fm::MAGIC + oz5::dig_koff<S>() - oz5_centre_int<S>();
  const double* X2 = gp->dX2.as<double>();
  constexpr int TH = oz5::KGEN_WARPS * 32;
  const unsigned ctas = kstar_ctas<S>(tiles);
  const KSplit ks = split ? *split : oz5_kstar_split(gp, tiles);
  const int ksplit = ks.ksplit, kc_per = ks.kc_per;
  const int64_t mstride = (int64_t)tiles * oz5::Geo<S>::NT;
  double* mean_dst = mean;
  if (ksplit > 1) {
    TB_TRY(gp->sMeanPart.reserve(sizeof(double) * (size_t)ksplit * mstride));
    mean_dst = gp->sMeanPart.as<double>();
  }
  with_kind_dp(gp->kernel, gp->DP, [&](auto K, auto P) {
    oz5::kstar_digits_kernel<decltype(K)::value, decltype(P)::value, S><<<dim3(ctas, ksplit), TH, 0, st>>>(
        Xs, X2, al, Xc_dev, il, N, nst, D, mc, var, inv_b, dig_c, mc0, fm::Consts(), tiles, kc_per, BS, mean_dst);
  });
  TB_LAUNCHED();
  if (ksplit > 1) {
    oz5::mean_reduce_kernel<<<(unsigned)((mstride + 255) / 256), 256, 0, st>>>(mean_dst, ksplit, mstride, mc0, mean);
    TB_LAUNCHED();
  }
  TB_CUDA(cudaGetLastError());
  return 0;
}

int oz5_launch_kstar(tb_gp* gp, cudaStream_t st, const double* Xc_dev, int64_t mc, int tiles, int8_t* BS, double* mean,
                     const KSplit* split) {
  return gp->oz5_planes == 5 ? launch_kstar_s<5>(gp, st, Xc_dev, mc, tiles, BS, mean, split)
                             : launch_kstar_s<4>(gp, st, Xc_dev, mc, tiles, BS, mean, split);
}

// The K* digits are cut against sB = h / FILL with 2^(8 planes) steps; a GEMM that computes with S < planes leading digits sees
// exactly the same scaled operand (the planes are a prefix of the same balanced expansion), so out_scale and h_eff are those
// of the STORED split.
template <int PL>
static double h_eff_planes(double variance) { return oz5_h_eff<PL>(variance); }

int oz5_launch_gemm(tb_gp* gp, cudaStream_t st, const int8_t* BS, int tiles, int G, int64_t McPad, double* partial) {
  const double sB = 0.5 * gp->variance / oz5::FILL;
  const int pl = gp->oz5_planes;
  const double h = pl == 5 ? h_eff_planes<5>(gp->variance) : h_eff_planes<4>(gp->variance);
#define TB_GEMM(SV)                                                                                                                \
  dg::launch<SV, dg::EPI_SUMSQ, oz5::Geo<SV>::NT>(st, gp->dAS5.as<int8_t>(), BS, gp->dRowScale5.as<double>(), gp->dRowSum5.as<double>(), \
                                                  gp->NB, gp->nst, G, tiles, McPad, sB, h, pl, pl, 0, partial, nullptr, 0)
  if (gp->oz5_mode == 5) TB_TRY(TB_GEMM(5));
  else if (gp->oz5_mode == 4) TB_TRY(TB_GEMM(4));
  else TB_TRY(TB_GEMM(3));
#undef TB_GEMM
  return 0;
}

int oz5_launch_gemm_store(tb_gp* gp, cudaStream_t st, int left, const int8_t* BS, int tiles, int G, double* out, int64_t lda) {
  const double sB = 0.5 * gp->variance / oz5::FILL;
  const int pl = gp->oz5_planes;
  const double h = pl == 5 ? h_eff_planes<5>(gp->variance) : h_eff_planes<4>(gp->variance);
  const int8_t* AS = left ? gp->dKinvS5.as<int8_t>() : gp->dAS5.as<int8_t>();
  const double* rs = left ? gp->dKinvScale5.as<double>() : gp->dRowScale5.as<double>();
  const double* rc = left ? gp->dKinvSum5.as<double>() : gp->dRowSum5.as<double>();
#define TB_GEMM(SV) \
  dg::launch<SV, dg::EPI_STORE, oz5::Geo<SV>::NT>(st, AS, BS, rs, rc, gp->NB, gp->nst, G, tiles, 0, sB, h, pl, pl, left ? 1 : 0, nullptr, out, lda)
  if (pl == 5) TB_TRY(TB_GEMM(5));
  else TB_TRY(TB_GEMM(4));
#undef TB_GEMM
  return 0;
}

}  // namespace tb
