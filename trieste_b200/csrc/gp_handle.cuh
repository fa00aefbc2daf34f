// The model handle: device-resident posterior cache + scratch, and its once-per-step precompute.
#pragma once
#include "common.cuh"
#include "../../include/trieste_b200.h"
#include <cublas_v2.h>
#include <cusolverDn.h>
#include <vector>
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <type_traits>
#include <utility>

namespace tb {

// A device allocation that grows on demand and is freed with its owner.  None may have static storage duration: its cudaFree
// would run after the CUDA runtime has been torn down at process exit.
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), cap(o.cap) {
    o.p = nullptr;
    o.cap = 0;
  }
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) {
      release();
      std::swap(p, o.p);
      std::swap(cap, o.cap);
    }
    return *this;
  }
  ~DevBuf() { release(); }
  int reserve(size_t bytes) {
    if (bytes <= cap) return 0;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    TB_CUDA(cudaMalloc(&p, bytes));
    cap = bytes;
    return 0;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
  template <class T>
  T* as() const { return reinterpret_cast<T*>(p); }
};

// State derived from the posterior cache records the cache_gen it was built from (tb_gp::cache_gen); it is current when the
// two are equal.
constexpr uint64_t STALE = ~(uint64_t)0;

// One left operand of the digit GEMM (Linv or the dense K^-1): per-row scales and per-row sums (the centring term), and digit
// planes cut against them in the GEMM's stage layout at two plane counts: the admitted split's (4 or 5) and 6.
struct DigitOperand {
  DevBuf scale, sum, digits, digits6;
  int planes = 0;         // planes of `digits`; 0: the a-priori estimate refused the operand
  uint64_t gen = STALE;   // cache_gen the row stats, the admission and `digits` were built from
  uint64_t gen6 = STALE;  // cache_gen `digits6` was cut from
};

// The int8 engine's state (int8_engines.cu owns it).  Both cuts of Linv and of K^-1 stay alive together, so one handle can run
// values at 5 digits and gradients at 6 when the V estimate refuses 5.
struct DigitState {
  DigitOperand linv, kinv;  // linv.gen also stamps the admission below
  DevBuf X2;                // squared row norms of the scaled training inputs (centred K* generation)
  bool full = false;        // tb_gp_set_engine(2): always 6 digits
  int mode = 0;             // digits the variance GEMM computes with on the admitted split (0: not admitted)
  double est = 0.0;         // a-priori estimate of max |Δvar| / σ_f² in that mode
  int S = 0;                // digit planes of the K* tiles and left operands of the current call (int8_select)
};

inline bool is_device_ptr(const void* p) {
  if (!p) return false;
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

// A caller's array of items of `width` elements each, on the device or on the host.  A device array is read and written in
// place; a host array goes through `scratch` one chunk of items at a time.  Every copy goes on the call's stream `st`, and
// the host waits once, at the end of the call: a copy from pageable memory to the device has consumed its source when it
// returns, a copy from the device to pageable memory returns only once it has completed, and each copy is ordered with the
// kernels on `st`, so stream order protects the scratch that the next chunk reuses.  (Pinned host arrays are read and
// written by the stream alone until that final wait.)
template <class T>
struct Staged {
  T* user;
  int64_t width;
  DevBuf* scratch;
  cudaStream_t st;
  bool dev;
  Staged(T* user, int64_t width, DevBuf& scratch, cudaStream_t st)
      : user(user), width(width), scratch(&scratch), st(st), dev(is_device_ptr(user)) {}
  bool host() const { return user && !dev; }
  int reserve(int64_t n) const { return host() ? scratch->reserve(sizeof(T) * width * n) : 0; }
  // items [c0, c0 + n) of an input, on the device (null for a null array)
  int in(int64_t c0, int64_t n, T** d) const {
    if (!host()) {
      *d = user ? user + c0 * width : nullptr;
      return 0;
    }
    TB_CUDA(cudaMemcpyAsync(scratch->p, user + c0 * width, sizeof(T) * width * n, cudaMemcpyHostToDevice, st));
    *d = scratch->as<T>();
    return 0;
  }
  // where the items of an output from c0 on are written (null for a null array); back() brings a host array's home
  T* out(int64_t c0) const { return host() ? scratch->as<T>() : user ? user + c0 * width : nullptr; }
  int back(int64_t c0, int64_t n) const {
    if (host()) TB_CUDA(cudaMemcpyAsync(user + c0 * width, scratch->p, sizeof(T) * width * n, cudaMemcpyDeviceToHost, st));
    return 0;
  }
};

// supported padded input dimensions of the distance loop (even, so rows load as double2), ascending
template <int... V>
struct DpList {};
using SupportedDp = DpList<2, 4, 6, 8, 10, 12, 16, 20, 24, 32>;

template <int... V>
inline int pick_dp_in(DpList<V...>, int D) {
  for (int o : {V...})
    if (D <= o) return o;
  return -1;
}
inline int pick_dp(int D) { return pick_dp_in(SupportedDp{}, D); }

// f(std::integral_constant<int, DP>) for the supported DP equal to dp; any other value runs the largest
template <int V, int... Rest, class F>
inline decltype(auto) with_dp_in(DpList<V, Rest...>, int dp, F&& f) {
  if constexpr (sizeof...(Rest) == 0) {
    return f(std::integral_constant<int, V>{});
  } else {
    if (dp == V) return f(std::integral_constant<int, V>{});
    return with_dp_in(DpList<Rest...>{}, dp, std::forward<F>(f));
  }
}
template <class F>
inline decltype(auto) with_dp(int dp, F&& f) { return with_dp_in(SupportedDp{}, dp, std::forward<F>(f)); }

// f(std::integral_constant<int, KIND>) for the kernel kind; an unknown kind runs Matern52
template <class F>
inline decltype(auto) with_kind(int kernel, F&& f) {
  switch (kernel) {
    case TB_RBF: return f(std::integral_constant<int, TB_RBF>{});
    case TB_MATERN12: return f(std::integral_constant<int, TB_MATERN12>{});
    case TB_MATERN32: return f(std::integral_constant<int, TB_MATERN32>{});
    default: return f(std::integral_constant<int, TB_MATERN52>{});
  }
}
template <class F>
inline decltype(auto) with_kind_dp(int kernel, int dp, F&& f) {
  return with_kind(kernel, [&](auto K) -> decltype(auto) { return with_dp(dp, [&](auto P) -> decltype(auto) { return f(K, P); }); });
}

}  // namespace tb

struct tb_gp {
  int device = 0;
  int dtype = TB_F64;
  cudaStream_t stream = nullptr;
  cublasHandle_t cublas = nullptr;
  cusolverDnHandle_t cusolver = nullptr;

  // model (host copies of the small things)
  int64_t N = 0;
  int D = 0, DP = 0;
  int kernel = TB_MATERN52;
  double variance = 1.0, noise = 1.0, mean_const = 0.0;
  std::vector<double> ls;  // [D]
  bool have_data = false, have_hyper = false, cache_valid = false;

  // geometry of the packed cache
  int nkc = 0;  // k panels = ceil(N/16)
  int NB = 0;   // row-blocks = ceil(N/128)

  tb::DevBuf dX, dy;            // raw data [N,D], [N]
  tb::DevBuf dXs;               // [nkc*16][DP] scaled, zero padded
  tb::DevBuf dInvLs;            // [DP]
  tb::DevBuf dAlpha;            // [nkc*16]
  tb::DevBuf dL;                // [N,N] column-major lower Cholesky factor
  tb::DevBuf dLinv;             // [N,N] column-major Linv (kept: predict_joint / gradients reuse it)
  tb::DevBuf dLinvP;            // packed lower panels
  tb::DevBuf dLinvTP;           // packed upper panels of Linv^T (lazy; gradient path)
  uint64_t upper_gen = tb::STALE;
  int engine = 1;  // 0 = fp64 DMMA, 1 = int8 tensor cores (default; same stated tolerances, ~3x faster)
  // dense K^-1 (lower triangle, ld = N) of the int8 engine's gradient path: an append grows it by rank m (tb_gp_append_data)
  // instead of rebuilding it in O(N^3)
  tb::DevBuf dKinv, dKinvSpare;
  uint64_t kinv_gen = tb::STALE;
  tb::DigitState digits;       // the int8 engine's digit operands (int8_engines.cu)
  tb::DevBuf sMeanPart;        // per-split mean partials of the k-split K* generation (few candidate tiles)
  tb::DevBuf dWork, dInfo;      // cusolver workspace / info flag
  tb::DevBuf dDinv;             // inverses of the diagonal blocks of L (hand-written factorisation)
  bool factor_own = true;       // false (TB_FACTOR=cusolver): cuSOLVER / cuBLAS cross-check path

  // per-call scratch
  tb::DevBuf sKs, sPartial, sMean, sVals, sVar, sXc, sBlkBest, sBlkIdx, sRun;
  tb::DevBuf sA, sV, sGrad, sMisc;  // A / V panels (joint + gradient paths), misc staging
  tb::DevBuf dXspare, dyspare, dLspare, dLinvSpare;  // ping-pong partners of dX / dy / dL / dLinv (tb_gp_append_data)
  tb::DevBuf dMes;              // min-value samples of TB_ACQ_MES (tb_acq_set_min_value_samples)
  int mesS = 0;
  tb::DevBuf dPen;              // local penalisation (tb_acq_set_penalization): pending [P][D], radius [P], scale [P]
  int penP = 0, penKind = 0, penD = 0;
  // GIBBON repulsion (tb_acq_set_gibbon_repulsion): raw pending points [m][D] and weight, and what is derived from them and
  // the posterior cache: scaled pending points [m][DP], L_B^-1 [mp][m] (zero rows past m), What = K^-1 k(X,P) L_B^-T [N][mp]
  std::vector<double> gibP;
  int gibM = 0, gibMp = 0, gibD = 0;
  double gibW = 0.0;
  double feasAlpha = 0.0;               // alpha of the feasibility kinds (tb_acq_set_feasibility); 0 = not set
  uint64_t cache_gen = 0;               // bumped whenever the posterior cache is (re)built
  uint64_t gib_gen = tb::STALE;         // cache_gen the derived GIBBON state was built for
  tb::DevBuf dGibPs, dGibLinv, dGibWhat;
  tb::DevBuf sGib;                      // per chunk: |u|^2 [mc], -w / V_det [mc], u [mp][mc] (gradient path)
  // screened argmax (tb_api.cu, argmax_screened): the screen bound ub of all M candidates, the survivors' coordinates / global
  // indices, and the bound pass's per-block winners + probe pair + survivor counts
  tb::DevBuf sScrUb, sScrX, sScrIdx, sScrBlk;
  // its rounds of few candidate tiles: the kernel values of the wide K* generation [nst*64][tiles NT], the int32 level
  // accumulators of the split-K variance GEMM
  tb::DevBuf sKval, sSplitAcc;
  // mirrors of the posterior for the bound pass (prescreen.cuh), rebuilt when cache_gen moves: pre_tc (tensor-core pass): its
  // stages of fp16 B fragments and |σ_f² α| (pre_nsl n8 slices, the first pre_npos_sl with α > 0); otherwise (CUDA-core pass)
  // fp32 rows [nst*64][W] of (x', |x'|^2, σ_f² α, |σ_f² α|); the centre [DP] subtracted from scaled inputs, and the constants
  // of the bound
  tb::DevBuf dPreRows, dPreCentre;
  uint64_t pre_gen = tb::STALE;
  bool pre_tc = false;
  int pre_nsl = 0, pre_npos_sl = 0;
  double pre_scale = 1.0, pre_x2max = 0.0, pre_rel = 0.0, pre_lin = 0.0, pre_lin_max = 0.0, pre_abs = 0.0;

  // profiling of the dominant kernel
  bool profile = false;
  double prof_ms = 0.0, prof_flops = 0.0;
  int64_t prof_launches = 0;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> prof_events;
  std::vector<double> prof_event_flops;
};
