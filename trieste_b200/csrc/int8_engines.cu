// Host side of the int8 digit engine (ozaki5.cuh: 3 - 6 digits under tight scales, centred K*).  Digit operands of Linv and K^-1
// built lazily after each cache refresh, the digit count of a call from a-priori error bounds, launches of the K* digit
// generation and of the digit GEMM.  Called from tb_api.cu, which picks the engine of a call.
#include "gp_handle.cuh"
#include "ozaki5.cuh"
#include "int8_engines.h"

namespace tb {

int int8_init() {  // each digit GEMM instantiation once
  TB_TRY((dg::set_smem<6, dg::EPI_SUMSQ, oz::Geo<6>::NT>()));
  TB_TRY((dg::set_smem<6, dg::EPI_STORE, oz::Geo<6>::NT>()));
  TB_TRY((dg::set_smem<5, dg::EPI_SUMSQ, oz::Geo<5>::NT>()));
  TB_TRY((dg::set_smem<5, dg::EPI_STORE, oz::Geo<5>::NT>()));
  TB_TRY((dg::set_smem<4, dg::EPI_SUMSQ, oz::Geo<4>::NT>()));
  TB_TRY((dg::set_smem<4, dg::EPI_STORE, oz::Geo<4>::NT>()));
  TB_TRY((dg::set_smem<3, dg::EPI_SUMSQ, oz::Geo<3>::NT>()));
  TB_TRY((dg::set_smem<6, dg::EPI_SPLIT, oz::Geo<6>::NT>()));
  TB_TRY((dg::set_smem<5, dg::EPI_SPLIT, oz::Geo<5>::NT>()));
  TB_TRY((dg::set_smem<4, dg::EPI_SPLIT, oz::Geo<4>::NT>()));
  TB_TRY((dg::set_smem<3, dg::EPI_SPLIT, oz::Geo<3>::NT>()));
  return 0;
}

static int nst_of(const tb_gp* gp) { return (int)((gp->N + oz::KST - 1) / oz::KST); }

// The digit planes stored per operand stage are gp->digits.S: 5 (fp64 handles), 4 (fp32 handles, whose variance GEMM may
// compute with the 3 leading planes and whose store-A / V GEMMs use all 4) or 6.  Tiles are 128 wide but for S = 5.
int int8_tile_width(const tb_gp* gp) { return gp->digits.S == 5 ? oz::Geo<5>::NT : oz::Geo<6>::NT; }
size_t int8_tile_bytes(const tb_gp* gp) { return (size_t)nst_of(gp) * gp->digits.S * int8_tile_width(gp) * oz::KST; }

// ---- digit operands ----------------------------------------------------------------------------------------------------

// the left operand: full = 0: Linv; 1: the dense K^-1
static const double* operand_src(const tb_gp* gp, int full) { return (full ? gp->dKinv : gp->dLinv).as<double>(); }

// Row scales and row sums of a left operand into o; its 6-plane cut is stale from then on
static int row_stats(tb_gp* gp, DigitOperand& o, int full) {
  const int64_t rows = (int64_t)gp->NB * BM;
  TB_TRY(o.scale.reserve(sizeof(double) * rows));
  TB_TRY(o.sum.reserve(sizeof(double) * rows));
  oz::rowstats_kernel<<<(unsigned)rows, 256, 0, gp->stream>>>(operand_src(gp, full), gp->N, rows, full, o.scale.as<double>(),
                                                              o.sum.as<double>());
  TB_LAUNCHED();
  o.gen6 = STALE;
  return 0;
}

// the largest row scale of o (the admission estimates): one host round trip
static int max_row_scale(tb_gp* gp, const DigitOperand& o, double* mx) {
  std::vector<double> h((size_t)gp->N);
  TB_CUDA(cudaMemcpyAsync(h.data(), o.scale.p, sizeof(double) * (size_t)gp->N, cudaMemcpyDeviceToHost, gp->stream));
  TB_CUDA(cudaStreamSynchronize(gp->stream));
  *mx = 0.0;
  for (double v : h) *mx = std::max(*mx, v);
  return 0;
}

// `planes` digit planes of a left operand into dst, cut against o's row scales, in the GEMM's stage layout (Linv's triangular
// one is zeroed first)
static int cut_digits(tb_gp* gp, const DigitOperand& o, int full, int planes, DevBuf& dst) {
  const int nst = nst_of(gp);
  const int64_t stages = full ? (int64_t)gp->NB * nst : oz::a_stage_offset(gp->NB);
  const size_t bytes = (size_t)stages * planes * oz::ATILE;
  TB_TRY(dst.reserve(bytes));
  if (!full) TB_CUDA(cudaMemsetAsync(dst.p, 0, bytes, gp->stream));
  const dim3 grid(full ? nst : 2 * gp->NB, gp->NB);
  auto cut = [&](auto kernel) {
    kernel<<<grid, 256, 0, gp->stream>>>(operand_src(gp, full), gp->N, nst, full, o.scale.as<double>(), dst.as<int8_t>());
  };
  if (planes == 6) cut(oz::digits_kernel<6>);
  else if (planes == 5) cut(oz::digits_kernel<5>);
  else cut(oz::digits_kernel<4>);
  TB_LAUNCHED();
  TB_CUDA(cudaGetLastError());
  return 0;
}

// the 6-plane cut of a left operand whose row stats are current
static int cut_six(tb_gp* gp, DigitOperand& o, int full) {
  if (o.gen6 == gp->cache_gen) return 0;
  TB_TRY(cut_digits(gp, o, full, 6, o.digits6));
  o.gen6 = gp->cache_gen;
  return 0;
}

// Calibrated a-priori estimate of max |Δvar| / σ_f² when the levels r > S+1 are dropped: per element of A the dropped
// level r = S+2 contributes ~ rowscale·sB·sqrt(6 K)·E[d²]·2^(-8(S+2)) (E[d²] = 256²/12 for uniform balanced digits, K <= N
// terms with independent signs), and Δvar = 2 Σ_n A_n δ_n with Σ A_n² <= σ_f².  The constant (8/5) was calibrated on the
// emulated engine over the benchmark configurations (oracle-side study in DESIGN.md §4c): estimate / measured max = 1.1 .. 5.
static double single_pass_estimate(double variance, double max_rowscale, int64_t N, int S) {
  const double sB = 0.5 * variance / oz::FILL;
  return 1.6 * std::sqrt(variance) * max_rowscale * sB * std::sqrt(6.0 * (double)N) * (65536.0 / 12.0) * std::ldexp(1.0, -8 * (S + 2)) / variance;
}

// The row stats of Linv, its split at the digit count the estimate admits and the admission (stamped together in linv.gen).  A
// new split makes the K^-1 one stale.
static int admit(tb_gp* gp) {
  DigitState& d = gp->digits;
  if (d.linv.gen == gp->cache_gen) return 0;
  d.mode = 0;
  d.linv.planes = 0;
  d.est = 0.0;
  d.kinv.gen = STALE;
  cudaStream_t st = gp->stream;
  {  // squared row norms of the scaled training inputs (expansion-form distances of the K* generation kernel)
    const int64_t xrows = (int64_t)nst_of(gp) * oz::KST;
    TB_TRY(d.X2.reserve(sizeof(double) * xrows));
    oz5::row_norms_kernel<<<(unsigned)((xrows + 255) / 256), 256, 0, st>>>(gp->dXs.as<double>(), (int64_t)gp->NB * BM, gp->DP, xrows,
                                                                         d.X2.as<double>());
    TB_LAUNCHED();
  }
  TB_TRY(row_stats(gp, d.linv, 0));
  if (d.full) {
    d.linv.gen = gp->cache_gen;
    return 0;
  }
  double mx;
  TB_TRY(max_row_scale(gp, d.linv, &mx));
  // fp64 handles: 5 digits / 15 products if the estimate clears 3e-10 (bar: 1e-9).  fp32 handles (bar: 1e-4): 4 planes are
  // stored; the variance GEMM computes with 3 digits / 6 products if that clears 3e-5, else with all 4 (10 products, one pass);
  // if even 4 digits do not clear it the handle is treated like an fp64 one.  Otherwise: 6 digits.
  int mode = 0, planes = 0;
  if (gp->dtype == TB_F32) {
    if (single_pass_estimate(gp->variance, mx, gp->N, 3) <= 3e-5) mode = 3, planes = 4;
    else if (single_pass_estimate(gp->variance, mx, gp->N, 4) <= 3e-5) mode = 4, planes = 4;
  }
  if (mode == 0 && single_pass_estimate(gp->variance, mx, gp->N, 5) <= (gp->dtype == TB_F32 ? 3e-5 : 3e-10)) mode = 5, planes = 5;
  if (planes) TB_TRY(cut_digits(gp, d.linv, 0, planes, d.linv.digits));
  if (mode) d.est = single_pass_estimate(gp->variance, mx, gp->N, mode);
  d.mode = mode;
  d.linv.planes = planes;
  d.linv.gen = gp->cache_gen;
  return 0;
}

// The row stats of the dense K^-1 (gp->dKinv) and, when Linv's split was admitted, its split at the same digit count with the
// V GEMM's own admission test (kinv.planes = 0: refused): the element error of V = K^-1 k* is
// ~ rowscale(K^-1) sB sqrt(6 N) E[d^2] 2^(-8(S+2)).  The bound (~1e-7 fp64 / ~1e-4 fp32) assumes V enters the gradient through
// sums of ~N terms with |V| ~ 0.1 .. 1.  It does not see the 1/(2 sd) by which LCB / EI scale d var.  So on dense
// low-dimensional models (cond(K + noise I) ~ 1e4, sd ~ 0.02 sigma_f) the variance term of a gradient can miss rtol 1e-6 at
// every digit count.  The measured cases are listed in tests/test_gpu_gradient_sweep.py (INT8_V_ATOL).
static int admit_kinv(tb_gp* gp) {
  DigitState& d = gp->digits;
  if (d.kinv.gen == gp->cache_gen) return 0;
  const int S = d.linv.planes;
  TB_TRY(row_stats(gp, d.kinv, 1));
  d.kinv.planes = 0;
  if (S) {
    double mx;
    TB_TRY(max_row_scale(gp, d.kinv, &mx));
    const double sB = 0.5 * gp->variance / oz::FILL;
    const double eps_v = mx * sB * std::sqrt(6.0 * (double)gp->N) * (65536.0 / 12.0) * std::ldexp(1.0, -8 * (S + 2));
    if (eps_v <= (gp->dtype == TB_F32 ? 1e-4 : 1e-7)) {
      TB_TRY(cut_digits(gp, d.kinv, 1, S, d.kinv.digits));
      d.kinv.planes = S;
    }
  }
  d.kinv.gen = gp->cache_gen;
  return 0;
}

int int8_select(tb_gp* gp, bool need_v) {
  TB_CHECK(gp->N <= 16384, "the int8 engine supports N <= 16384 (int32 accumulator headroom)");
  DigitState& d = gp->digits;
  TB_TRY(admit(gp));
  int S = d.linv.planes;
  if (need_v) {
    TB_TRY(admit_kinv(gp));
    S = d.kinv.planes;
  }
  if (!S) {
    S = 6;
    TB_TRY(cut_six(gp, d.linv, 0));
    if (need_v) TB_TRY(cut_six(gp, d.kinv, 1));
  }
  d.S = S;
  return 0;
}

void int8_pin_full(tb_gp* gp, bool full) {
  if (gp->digits.full != full) gp->digits.linv.gen = STALE;
  gp->digits.full = full;
}

// digits the variance GEMM computes with: the admitted mode; with 6 digits all 6, or the 4 leading planes on fp32 handles
// (10 products, error ~1e-7 σ_f² << the fp32 tolerance)
static int variance_digits(const tb_gp* gp) {
  const DigitState& d = gp->digits;
  return d.S != 6 ? d.mode : gp->dtype == TB_F32 ? 4 : 6;
}

void int8_info(const tb_gp* gp, int* products, double* estimate) {
  const int S = variance_digits(gp);
  *products = S * (S + 1) / 2;
  *estimate = gp->digits.est;
}

// ---- K* digit generation -----------------------------------------------------------------------------------------------

// the centre of K* in digit units, the integer nearest to h * inv_b = FILL * 2^(8 planes); the centre
// actually subtracted is h_eff = centre / inv_b = h * centre / (FILL 2^(8 planes)), used consistently by the generation kernel
// and the GEMM epilogue.  A GEMM that computes with S < planes leading digits sees exactly the same scaled operand (the
// planes are a prefix of the same balanced expansion), so its out_scale and h_eff are those of the STORED split.
static double centre_int(int planes) { return std::nearbyint(oz::FILL * std::ldexp(1.0, 8 * planes)); }
static double h_eff(double variance, int planes) {
  return 0.5 * variance * centre_int(planes) / (oz::FILL * std::ldexp(1.0, 8 * planes));
}

static unsigned kstar_ctas(const tb_gp* gp, int tiles) {
  return (unsigned)(((int64_t)tiles * (int8_tile_width(gp) / 8) + oz5::KGEN_WARPS - 1) / oz5::KGEN_WARPS);
}

KSplit int8_kstar_split(const tb_gp* gp, int tiles) {
  KSplit s;
  const int nst = nst_of(gp);
  const unsigned ctas = kstar_ctas(gp, tiles);
  // few tiles (the late rounds of the multi-start optimiser, small predict calls): split the training rows over blockIdx.y so
  // that ~4 CTAs per SM exist; each split covers >= 2 stages
  s.kc_per = nst;
  if (ctas < NUM_SMS && nst >= 4) {
    s.ksplit = std::min<int>(nst / 2, (int)((4 * NUM_SMS + ctas - 1) / ctas));
    s.kc_per = (nst + s.ksplit - 1) / s.ksplit;
    s.ksplit = (nst + s.kc_per - 1) / s.kc_per;
  }
  return s;
}

template <int S>
static int kstar(tb_gp* gp, const double* Xc_dev, int64_t mc, int tiles, int8_t* BS, double* mean, const KSplit* split, bool wide) {
  const double* Xs = gp->dXs.as<double>();
  const double* al = gp->dAlpha.as<double>();
  const double* il = gp->dInvLs.as<double>();
  const int N = (int)gp->N, nst = nst_of(gp), D = gp->D;
  const double var = gp->variance, mc0 = gp->mean_const;
  const double inv_b = oz::two_pow_8S<S>() * oz::FILL / (0.5 * var);
  const double dig_c = fm::MAGIC + oz5::dig_koff<S>() - centre_int(S);
  const double* X2 = gp->digits.X2.as<double>();
  cudaStream_t st = gp->stream;
  constexpr int TH = oz5::KGEN_WARPS * 32;
  const unsigned ctas = kstar_ctas(gp, tiles);
  const KSplit ks = split ? *split : int8_kstar_split(gp, tiles);
  const int ksplit = ks.ksplit, kc_per = ks.kc_per;
  const int64_t mstride = (int64_t)tiles * oz::Geo<S>::NT;
  if (wide) {
    // the k-stages over ~4 CTAs per SM, the kernel values to gp->sKval, then the means of split ks replayed from them
    const int wsplit = (int)std::min<int64_t>(nst, (4 * NUM_SMS + ctas - 1) / ctas);
    const int wkc = (nst + wsplit - 1) / wsplit;
    TB_TRY(gp->sKval.reserve(sizeof(double) * (size_t)nst * oz::KST * mstride));
    double* kval = gp->sKval.as<double>();
    with_kind_dp(gp->kernel, gp->DP, [&](auto K, auto P) {
      oz5::kstar_digits_kernel<decltype(K)::value, decltype(P)::value, S, true><<<dim3(ctas, (nst + wkc - 1) / wkc), TH, 0, st>>>(
          Xs, X2, al, Xc_dev, il, N, nst, D, mc, var, inv_b, dig_c, mc0, fm::Consts(), tiles, wkc, BS, kval);
    });
    TB_LAUNCHED();
    oz5::mean_replay_kernel<<<(unsigned)(mstride * 4 / oz5::REPLAY_THREADS), oz5::REPLAY_THREADS, 0, st>>>(kval, al, nst, ksplit, kc_per,
                                                                                                        mstride, mc0, mean);
    TB_LAUNCHED();
    TB_CUDA(cudaGetLastError());
    return 0;
  }
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

int int8_kstar(tb_gp* gp, const double* Xc_dev, int64_t mc, int tiles, int8_t* BS, double* mean, const KSplit* split, bool wide) {
  switch (gp->digits.S) {
    case 6: return kstar<6>(gp, Xc_dev, mc, tiles, BS, mean, split, wide);
    case 5: return kstar<5>(gp, Xc_dev, mc, tiles, BS, mean, split, wide);
  }
  return kstar<4>(gp, Xc_dev, mc, tiles, BS, mean, split, wide);
}

int int8_split_kper(const tb_gp* gp, int tiles, int G) {
  return dg::split_kper(variance_digits(gp), int8_tile_width(gp), tiles, G, gp->NB, nst_of(gp), 0);
}

// ---- digit GEMM --------------------------------------------------------------------------------------------------------

// The digit GEMM: `left` (Linv, full_rows = 0, or K^-1, full_rows = 1) times the K* digits BS, both stored with gp->digits.S
// planes, computing with the S leading planes of both on K* tiles of Geo<S>::NT candidates.  The K* scale and centre are
// those of the stored split: the S leading planes are a prefix of the same balanced expansion.
// kper > 0 (EPI_SUMSQ): split-K in units of kper stages (dg::launch_split), the accumulators in gp->sSplitAcc.
template <int EPI>
static int digit_gemm(tb_gp* gp, const DigitOperand& left, int full_rows, int S, const int8_t* BS, int tiles, int G, int64_t McPad,
                      double* partial, double* out, int64_t lda, int kper = 0) {
  const int planes = gp->digits.S;
  const int8_t* AS = (planes == 6 ? left.digits6 : left.digits).as<int8_t>();
  const double out_scale = 0.5 * gp->variance / oz::FILL, h = h_eff(gp->variance, planes);
  auto launch = [&](auto SV) {
    constexpr int s = decltype(SV)::value, NT = oz::Geo<s>::NT;
    if constexpr (EPI == dg::EPI_SUMSQ) {
      if (kper > 0) {
        TB_TRY(gp->sSplitAcc.reserve(dg::split_acc_bytes<s>(tiles, NT, gp->NB)));
        return dg::launch_split<s, NT>(gp->stream, AS, BS, left.scale.as<double>(), left.sum.as<double>(), gp->NB, nst_of(gp), G, tiles,
                                       McPad, out_scale, h, planes, planes, full_rows, kper, gp->sSplitAcc.as<int>(), partial);
      }
    }
    return dg::launch<s, EPI, NT>(gp->stream, AS, BS, left.scale.as<double>(), left.sum.as<double>(), gp->NB, nst_of(gp), G, tiles,
                                  McPad, out_scale, h, planes, planes, full_rows, partial, out, lda);
  };
  switch (S) {
    case 6: return launch(std::integral_constant<int, 6>{});
    case 5: return launch(std::integral_constant<int, 5>{});
    case 4: return launch(std::integral_constant<int, 4>{});
  }
  if constexpr (EPI == dg::EPI_SUMSQ) return launch(std::integral_constant<int, 3>{});  // fp32 handles' variance GEMM only
  return fail("digit GEMM: no store kernel computes with " + std::to_string(S) + " digits", ERR_RUNTIME);
}

int int8_variance(tb_gp* gp, const int8_t* BS, int tiles, int G, int64_t McPad, double* partial, int kper) {
  return digit_gemm<dg::EPI_SUMSQ>(gp, gp->digits.linv, 0, variance_digits(gp), BS, tiles, G, McPad, partial, nullptr, 0, kper);
}

// the store GEMMs compute with every stored plane, but with the 4 leading ones of 6 on fp32 handles
int int8_store(tb_gp* gp, bool kinv, const int8_t* BS, int tiles, int G, int64_t McPad, double* out, int64_t lda) {
  const DigitState& d = gp->digits;
  const int S = d.S == 6 && gp->dtype == TB_F32 ? 4 : d.S;
  return digit_gemm<dg::EPI_STORE>(gp, kinv ? d.kinv : d.linv, kinv, S, BS, tiles, G, McPad, nullptr, out, lda);
}

}  // namespace tb
