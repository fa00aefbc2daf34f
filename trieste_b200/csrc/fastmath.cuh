// Branch-free fp64 exp(-s) and sqrt for the K* generation kernels.
//
// ncu (round 2, kstar_digits_kernel): 148 warp instructions per K* element, of which only ~53 on the fp64 pipe — the rest are
// the uniform-register constant loads (UMOV, 20 %), the slow-path branches (BRA/BSSY/BSYNC, 9 %) and integer glue of the
// library exp() / sqrt() inlined sixteen times per loop body.  The kernels need exp(-s) for s >= 0 (Matern / RBF arguments)
// and sqrt(x) for x >= 5e-36, so the special cases are not needed:
//   exp(-s): n = rint(-s 64 / ln 2) by the 1.5 2^52 magic add, f = -s - n ln2/64 (two-term Cody-Waite, |f| <= ln2/128),
//            e^f by a degree-5 Taylor polynomial (remainder < 3.5e-17 relative), times 2^((n mod 64)/64) from a 64-entry table
//            (correctly rounded, held in shared memory), times 2^(n div 64) by an integer add to the exponent field
//            (clamped at 2^-1020: results below ~1e-307 are returned as ~1e-307).
//   sqrt(x): float rsqrt seed (MUFU.RSQ), one coupled Newton step on (g ~ sqrt x, h ~ 1 / (2 sqrt x)) and a final
//            residual correction: 2 DMUL + 5 DFMA.
// Max relative errors measured by the host harness tools/fastmath_check.cu are quoted in DESIGN.md.
#pragma once
#include <cstdint>
#include <cstring>
#include <cmath>

namespace tb {
namespace fm {

// 2^(j/64), j = 0..63, correctly rounded (generated with 60-digit decimal arithmetic)
#define TB_EXP2_TABLE_VALUES                                                                                          \
  0x1.0000000000000p+0, 0x1.02c9a3e778061p+0, 0x1.059b0d3158574p+0, 0x1.0874518759bc8p+0, 0x1.0b5586cf9890fp+0,      \
      0x1.0e3ec32d3d1a2p+0, 0x1.11301d0125b51p+0, 0x1.1429aaea92de0p+0, 0x1.172b83c7d517bp+0, 0x1.1a35beb6fcb75p+0,  \
      0x1.1d4873168b9aap+0, 0x1.2063b88628cd6p+0, 0x1.2387a6e756238p+0, 0x1.26b4565e27cddp+0, 0x1.29e9df51fdee1p+0,  \
      0x1.2d285a6e4030bp+0, 0x1.306fe0a31b715p+0, 0x1.33c08b26416ffp+0, 0x1.371a7373aa9cbp+0, 0x1.3a7db34e59ff7p+0,  \
      0x1.3dea64c123422p+0, 0x1.4160a21f72e2ap+0, 0x1.44e086061892dp+0, 0x1.486a2b5c13cd0p+0, 0x1.4bfdad5362a27p+0,  \
      0x1.4f9b2769d2ca7p+0, 0x1.5342b569d4f82p+0, 0x1.56f4736b527dap+0, 0x1.5ab07dd485429p+0, 0x1.5e76f15ad2148p+0,  \
      0x1.6247eb03a5585p+0, 0x1.6623882552225p+0, 0x1.6a09e667f3bcdp+0, 0x1.6dfb23c651a2fp+0, 0x1.71f75e8ec5f74p+0,  \
      0x1.75feb564267c9p+0, 0x1.7a11473eb0187p+0, 0x1.7e2f336cf4e62p+0, 0x1.82589994cce13p+0, 0x1.868d99b4492edp+0,  \
      0x1.8ace5422aa0dbp+0, 0x1.8f1ae99157736p+0, 0x1.93737b0cdc5e5p+0, 0x1.97d829fde4e50p+0, 0x1.9c49182a3f090p+0,  \
      0x1.a0c667b5de565p+0, 0x1.a5503b23e255dp+0, 0x1.a9e6b5579fdbfp+0, 0x1.ae89f995ad3adp+0, 0x1.b33a2b84f15fbp+0,  \
      0x1.b7f76f2fb5e47p+0, 0x1.bcc1e904bc1d2p+0, 0x1.c199bdd85529cp+0, 0x1.c67f12e57d14bp+0, 0x1.cb720dcef9069p+0,  \
      0x1.d072d4a07897cp+0, 0x1.d5818dcfba487p+0, 0x1.da9e603db3285p+0, 0x1.dfc97337b9b5fp+0, 0x1.e502ee78b3ff6p+0,  \
      0x1.ea4afa2a490dap+0, 0x1.efa1bee615a27p+0, 0x1.f50765b6e4540p+0, 0x1.fa7c1819e90d8p+0

#ifdef __CUDACC__
__device__ const double EXP2_TABLE_DEV[64] = {TB_EXP2_TABLE_VALUES};
#define TB_FM_HD __host__ __device__ __forceinline__
#else
#define TB_FM_HD inline
#endif
static const double EXP2_TABLE_HOST[64] = {TB_EXP2_TABLE_VALUES};

constexpr double MAGIC = 6755399441055744.0;         // 1.5 * 2^52: x + MAGIC rounds x to the nearest integer (low mantissa bits)
constexpr double L2E64 = 0x1.71547652b82fep+6;      // 64 / ln 2
constexpr double LN2_64_HI = 0x1.62e42fee00000p-7;  // ln 2 / 64, 32 significant bits: n * HI is exact for |n| < 2^20
constexpr double LN2_64_LO = 0x1.a39ef35793c76p-39;

// The constants whose low mantissa word is non-zero cannot be encoded as instruction immediates; as literals the compiler
// re-materialises each of them with two UMOVs at every use (issue slots: the generation kernel is issue bound).  Passed as a
// __grid_constant__ kernel parameter they are read straight from the constant bank as DFMA operands.
struct Consts {
  double l2e64 = L2E64, ln2_hi = LN2_64_HI, ln2_lo = LN2_64_LO;
  double c120 = 1.0 / 120.0, c24 = 1.0 / 24.0, c6 = 1.0 / 6.0, third = 1.0 / 3.0;
};

TB_FM_HD int lo_word(double x) {
#ifdef __CUDA_ARCH__
  return __double2loint(x);
#else
  int64_t b;
  std::memcpy(&b, &x, 8);
  return (int)(uint32_t)b;
#endif
}
TB_FM_HD int hi_word(double x) {
#ifdef __CUDA_ARCH__
  return __double2hiint(x);
#else
  int64_t b;
  std::memcpy(&b, &x, 8);
  return (int)(b >> 32);
#endif
}
TB_FM_HD double with_hi_word(double x, int hi) {
#ifdef __CUDA_ARCH__
  return __hiloint2double(hi, __double2loint(x));
#else
  int64_t b;
  std::memcpy(&b, &x, 8);
  b = (b & 0xffffffffLL) | ((int64_t)hi << 32);
  std::memcpy(&x, &b, 8);
  return x;
#endif
}
// max(x, lo) / min(x, hi) for a NON-NEGATIVE bound by one integer compare on the high words (doubles order like their
// sign-magnitude high words; a negative x has a negative high word).  The low word is kept, so the result may exceed the
// bound by < 2^-20 relative — irrelevant for the clamps below.  No NaN handling (the callers never produce one).
TB_FM_HD double clamp_below(double x, double lo) {
  const int h = hi_word(x), b = hi_word(lo);
  return with_hi_word(x, h > b ? h : b);
}
TB_FM_HD double clamp_above_nonneg(double x, double hi) {  // x >= 0
  const int h = hi_word(x), b = hi_word(hi);
  return with_hi_word(x, h < b ? h : b);
}

// exp(-s), s >= 0; T = the 64-entry table (shared memory on the device)
TB_FM_HD double exp_neg(double s, const double* T, const Consts& c) {
  s = clamp_above_nonneg(s, 1000.0);  // exp(-1000) is below the smallest normal: keeps n inside the exact range of the reduction
  const double t = fma(-s, c.l2e64, MAGIC);
  const int n = lo_word(t);
  const double nf = t - MAGIC;
  double f = fma(nf, -c.ln2_hi, -s);
  f = fma(nf, -c.ln2_lo, f);
  double p = fma(f, c.c120, c.c24);
  p = fma(p, f, c.c6);
  p = fma(p, f, 0.5);
  p = fma(p, f, 1.0);
  p = fma(p, f, 1.0);
  int e = n >> 6;
  e = e < -1020 ? -1020 : e;
  const double r = T[n & 63] * p;
  return with_hi_word(r, hi_word(r) + e * 1048576);  // r * 2^e
}

// sqrt(x) for x in [1e-37, 1e37] (float range of the seed)
TB_FM_HD double sqrt_pos(double x) {
#ifdef __CUDA_ARCH__
  float yf;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(yf) : "f"((float)x));  // one MUFU.RSQ, no denormal fix-up path
  const double y = (double)yf;
#else
  const double y = (double)(1.0f / std::sqrt((float)x));
#endif
  double g = x * y;    // ~ sqrt(x), 22 bits
  double h = 0.5 * y;  // ~ 1 / (2 sqrt x)
  const double r = fma(-g, h, 0.5);
  g = fma(g, r, g);
  h = fma(h, r, h);
  const double d = fma(-g, g, x);
  return fma(d, h, g);
}

// cos(a) for |a| < ~1e6 (the random-Fourier-feature arguments w.x + b): cos(a) = sin(a + pi/2) = (-1)^k sin(r) with
// k = rint(a / pi + 1/2), r = a - (2k - 1) pi/2 in [-pi/2, pi/2] (three-term Cody-Waite, the odd multiple m = 2k - 1 times each
// 33-bit part of pi/2 is exact for |m| < 2^20), sin(r) by its Taylor polynomial through r^19 (remainder < 3e-16; max absolute error
// measured by tools/fastmath_check.cu: 4e-16).  ncu: the library cos() left rff_eval_kernel issue-bound
// (issue 77 %, fp64 pipe 48 %) on its slow-path branches and constant traffic.
struct TrigConsts {
  double inv_pi = 0x1.45f306dc9c883p-2;
  double pio2_hi = 0x1.921fb54400000p+0, pio2_mid = 0x1.0b4611a600000p-34, pio2_lo = 0x1.3198a2e037073p-69;
  double s3 = -0x1.5555555555555p-3, s5 = 0x1.1111111111111p-7, s7 = -0x1.a01a01a01a01ap-13, s9 = 0x1.71de3a556c734p-19;
  double s11 = -0x1.ae64567f544e4p-26, s13 = 0x1.6124613a86d09p-33, s15 = -0x1.ae7f3e733b81fp-41, s17 = 0x1.952c77030ad4ap-49;
  double s19 = -0x1.2f49b46814157p-57;
  // cos(r) Taylor coefficients 1 / (2j)! with signs, j = 2..10 (the r^2 one is -1/2, an immediate)
  double c4 = 0x1.5555555555555p-5, c6 = -0x1.6c16c16c16c17p-10, c8 = 0x1.a01a01a01a01ap-16, c10 = -0x1.27e4fb7789f5cp-22;
  double c12 = 0x1.1eed8eff8d898p-29, c14 = -0x1.93974a8c07c9dp-37, c16 = 0x1.ae7f3e733b81fp-45, c18 = -0x1.6827863b97d97p-53;
  double c20 = 0x1.e542ba4020225p-62;
};

// the shared argument reduction: a = r + (2k - 1) pi/2, r in [-pi/2, pi/2]; returns r, sets k
TB_FM_HD double trig_reduce(double a, const TrigConsts& c, int& k) {
  const double t = fma(a, c.inv_pi, 0.5) + MAGIC;  // low word = k = rint(a / pi + 1/2)  (MAGIC + 0.5 is not representable)
  k = lo_word(t);
  const double m = fma(2.0, t - MAGIC, -1.0);      // 2k - 1 (exact)
  double r = fma(m, -c.pio2_hi, a);
  r = fma(m, -c.pio2_mid, r);
  r = fma(m, -c.pio2_lo, r);
  return r;
}

// cos(a) = (-1)^k sin(r) from the reduced argument
TB_FM_HD double cos_reduced(double r, int k, const TrigConsts& c) {
  const double r2 = r * r;
  double p = fma(c.s19, r2, c.s17);
  p = fma(p, r2, c.s15);
  p = fma(p, r2, c.s13);
  p = fma(p, r2, c.s11);
  p = fma(p, r2, c.s9);
  p = fma(p, r2, c.s7);
  p = fma(p, r2, c.s5);
  p = fma(p, r2, c.s3);
  const double sr = fma(p * r2, r, r);  // sin(r)
  return with_hi_word(sr, hi_word(sr) ^ (k << 31));  // (-1)^k
}

TB_FM_HD double cos_fast(double a, const TrigConsts& c) {
  int k;
  const double r = trig_reduce(a, c, k);
  return cos_reduced(r, k, c);
}

// cos(a), returned bit for bit as cos_fast(a), and sin(a) into s, from one reduction: sin(a) = (-1)^(k+1) cos(r) with cos(r) by its
// Taylor polynomial through r^20 (remainder < 2e-17 on [-pi/2, pi/2]); the absolute error is bounded like cos_fast's
// (tools/sincos_check.cu).
TB_FM_HD double sincos_fast(double a, const TrigConsts& c, double& s) {
  int k;
  const double r = trig_reduce(a, c, k);
  const double r2 = r * r;
  double p = fma(c.c20, r2, c.c18);
  p = fma(p, r2, c.c16);
  p = fma(p, r2, c.c14);
  p = fma(p, r2, c.c12);
  p = fma(p, r2, c.c10);
  p = fma(p, r2, c.c8);
  p = fma(p, r2, c.c6);
  p = fma(p, r2, c.c4);
  p = fma(p, r2, -0.5);
  const double cr = fma(p, r2, 1.0);  // cos(r) >= 0
  s = with_hi_word(cr, hi_word(cr) ^ ((k + 1) << 31));  // (-1)^(k+1)
  return cos_reduced(r, k, c);
}

}  // namespace fm
}  // namespace tb
