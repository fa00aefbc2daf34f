// C-ABI entry points (include/trieste_b200.h).  Host orchestration only: every per-candidate flop
// runs in the kernels of kernels_f64.cuh / kernels_extra.cuh.
#include "gp_handle.cuh"
#include "kernels_extra.cuh"
#include "prescreen.cuh"
#include "batch_ei.cuh"
#include "active_learning.cuh"
#include "ehvi.cuh"
#include "reduce.cuh"
#include "int8_engines.h"
#include <chrono>
#include <memory>
#include "factor.cuh"
#include "lbfgs.cuh"

using namespace tb;
namespace tb {
int kernels_init();
}

// =================================================================================================
// once-per-step precompute kernels (posterior cache; SURVEY.md §8 a3)
// =================================================================================================
namespace tb {

// Xs[k][d] = X[k][d] / l_d, zero padded to [nkc*16][DP]
__global__ void scale_inputs_kernel(const double* __restrict__ X, const double* __restrict__ inv_ls,
                                    int64_t N, int D, int DP, int64_t rows, double* __restrict__ Xs) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * DP) return;
  int64_t k = i / DP;
  int d = (int)(i % DP);
  Xs[i] = (k < N && d < D) ? X[k * D + d] * inv_ls[d] : 0.0;
}

// K(X,X) + noise I, full symmetric, column-major [N,N]
template <int KIND>
__global__ void gram_kernel(const double* __restrict__ Xs, int64_t N, int DP, double variance,
                            double noise, double* __restrict__ K) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t j = blockIdx.y;
  if (i >= N) return;
  double r2 = 0.0;
  for (int d = 0; d < DP; ++d) {
    double df = Xs[i * DP + d] - Xs[j * DP + d];
    r2 = fma(df, df, r2);
  }
  double v = kernel_from_r2<KIND>(r2, variance);
  if (i == j) v = variance + noise;
  K[i + j * N] = v;
}

// ---- rank-m append of training points to an existing cache (tb_gp_append_data; SURVEY.md §8f-1) ----
// W[:, j] (column-major [N, m]) = k(x_i, xnew_j) for every row i of the grown data set; the diagonal entry of the new
// block carries the likelihood noise
template <int KIND>
__global__ void append_cross_kernel(const double* __restrict__ Xs, int DP, int64_t N0, int64_t N, double variance,
                                    double noise, double* __restrict__ W) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t j = blockIdx.y;
  if (i >= N) return;
  double r2 = 0.0;
  for (int d = 0; d < DP; ++d) {
    const double df = Xs[i * DP + d] - Xs[(N0 + j) * DP + d];
    r2 = fma(df, df, r2);
  }
  double v = kernel_from_r2<KIND>(r2, variance);
  if (i == N0 + j) v = variance + noise;
  W[i + j * N] = v;
}

// Y[:, j] = T[0:n, 0:n] X[:, j] for a column-major lower-triangular T with leading dimension ld (one thread per row:
// coalesced along the rows of a column)
__global__ void trmv_lower_cols_kernel(const double* __restrict__ T, int64_t n, int64_t ld, const double* __restrict__ X,
                                       int64_t ldx, double* __restrict__ Y, int64_t ldy) {
  __shared__ double xs[128];
  const int64_t r = (int64_t)blockIdx.x * 128 + threadIdx.x;
  const int64_t j = blockIdx.y;
  const int64_t kend = min(n, ((int64_t)blockIdx.x + 1) * 128);
  double s = 0.0;
  for (int64_t k0 = 0; k0 < kend; k0 += 128) {
    __syncthreads();
    xs[threadIdx.x] = (k0 + threadIdx.x < n) ? X[k0 + threadIdx.x + j * ldx] : 0.0;
    __syncthreads();
    if (r < n) {
      const int64_t kk_end = min((int64_t)128, r - k0 + 1);
      for (int64_t kk = 0; kk < kk_end; ++kk) s = fma(T[r + (k0 + kk) * ld], xs[kk], s);
    }
  }
  if (r < n) Y[r + j * ldy] = s;
}

// U[:, j] = T[0:n, 0:n]^T X[:, j] (one warp per column of T)
__global__ void trmv_lower_t_cols_kernel(const double* __restrict__ T, int64_t n, int64_t ld, const double* __restrict__ X,
                                         int64_t ldx, double* __restrict__ U, int64_t ldu) {
  const int64_t k = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int64_t j = blockIdx.y;
  if (k >= n) return;
  double s = 0.0;
  for (int64_t r = k + lane; r < n; r += 32) s = fma(T[r + k * ld], X[r + j * ldx], s);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) U[k + j * ldu] = s;
}

// S[i + j*m] = C[i][j] - l_i . l_j (Schur complement of the new block; l_i = Y[:, i], C = W[N0:, :])
__global__ void append_schur_kernel(const double* __restrict__ Y, const double* __restrict__ W, int64_t N0, int64_t N, int m,
                                    double* __restrict__ S) {
  __shared__ double red[8];
  const int i = blockIdx.x, j = blockIdx.y;
  double s = 0.0;
  for (int64_t k = threadIdx.x; k < N0; k += blockDim.x) s = fma(Y[k + (int64_t)i * N], Y[k + (int64_t)j * N], s);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
    S[i + j * m] = W[N0 + i + (int64_t)j * N] - t;
  }
}

constexpr int APPEND_MAX = 64;  // larger appends refactorise from scratch

// one CTA of APPEND_MAX threads: L22 = chol(S) in shared memory, R = L22^-1; writes both into the new corner of L / Linv
// and R (row-major [m, m]) to Rout; info = failing leading minor (global index) if S is not positive definite
__global__ void append_chol_kernel(const double* __restrict__ S, int m, int64_t N0, int64_t N, double* __restrict__ L,
                                   double* __restrict__ Linv, double* __restrict__ Rout, int* __restrict__ info) {
  __shared__ double A[APPEND_MAX][APPEND_MAX + 1];
  __shared__ int bad;
  const int t = threadIdx.x;
  if (t == 0) bad = 0;
  for (int j = 0; j < m; ++j)
    if (t < m) A[t][j] = S[t + j * m];
  __syncthreads();
  for (int j = 0; j < m; ++j) {
    if (t == j) {
      const double d = A[j][j];
      if (!(d > 0.0)) {
        if (!bad) bad = (int)(N0 + j + 1);
        A[j][j] = 1.0;
      } else {
        A[j][j] = sqrt(d);
      }
    }
    __syncthreads();
    if (t > j && t < m) A[t][j] /= A[j][j];
    __syncthreads();
    if (t > j && t < m)
      for (int k = j + 1; k <= t; ++k) A[t][k] -= A[t][j] * A[k][j];
    __syncthreads();
  }
  // column t of R: forward substitution of L22 r = e_t
  if (t < m) {
    for (int i = 0; i < m; ++i) {
      double s = (i == t) ? 1.0 : 0.0;
      for (int k = t; k < i; ++k) s -= A[i][k] * Rout[k * m + t];
      Rout[i * m + t] = (i < t) ? 0.0 : s / A[i][i];  // column t is private to this thread
    }
  }
  __syncthreads();
  if (t == 0 && bad) *info = bad;
  if (t < m)
    for (int j = 0; j < m; ++j) {
      L[(N0 + t) + (N0 + j) * N] = (j <= t) ? A[t][j] : 0.0;
      Linv[(N0 + t) + (N0 + j) * N] = (j <= t) ? Rout[t * m + j] : 0.0;
    }
}

// new rows left of the corner: L[N0+i, k] = Y[k, i] (Y = Linv0 B, so L21 = Y^T) and Linv[N0+i, k] = -(R U^T)[i, k] with
// U = Linv0^T Y (Linv21 = -L22^-1 L21 Linv0)
__global__ void append_rows_kernel(const double* __restrict__ Y, const double* __restrict__ U, const double* __restrict__ R,
                                   int m, int64_t N0, int64_t N, double* __restrict__ L, double* __restrict__ Linv) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int i = blockIdx.y;
  if (k >= N0) return;
  double b = 0.0;
  for (int j = 0; j <= i; ++j) b = fma(R[i * m + j], U[k + (int64_t)j * N], b);
  L[(N0 + i) + k * N] = Y[k + (int64_t)i * N];
  Linv[(N0 + i) + k * N] = -b;
}

__global__ void identity_kernel(int64_t N, double* __restrict__ A) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * N) return;
  A[i] = (i % N == i / N) ? 1.0 : 0.0;
}

__global__ void zero_upper_kernel(int64_t N, double* __restrict__ A) {  // column-major: zero i < j
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t j = blockIdx.y;
  if (i < N && i < j) A[i + j * N] = 0.0;
}

__global__ void residual_kernel(const double* __restrict__ y, int64_t N, int64_t rows, double mean_const,
                                double* __restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < rows) out[i] = (i < N) ? y[i] - mean_const : 0.0;
}

// one CTA per (row-block I, k-panel kc) of the lower triangle: Linv (column-major) -> packed panel
__global__ void pack_lower_panels_kernel(const double* __restrict__ Linv, int64_t N, int nkc,
                                         double* __restrict__ P) {
  const int I = blockIdx.y, kc = blockIdx.x;
  const int nk = min((I + 1) * (BM / BK), nkc);
  if (kc >= nk) return;
  double* dst = P + (rowblock_panel_offset(I) + kc) * PANEL;
  for (int e = threadIdx.x; e < PANEL; e += blockDim.x) {
    // iterate in source-friendly order: r fastest (column-major source), scatter into the panel
    int r = e % BM, k = e / BM;
    int64_t n = (int64_t)I * BM + r, kk = (int64_t)kc * BK + k;
    double v = (n < N && kk <= n) ? Linv[n + kk * N] : 0.0;
    dst[panel_elem_index(r, k)] = v;
  }
}

// column-major lower factor -> row-major dense (upper zeroed), for tb_gp_get_cholesky
__global__ void colmajor_lower_to_rowmajor_kernel(const double* __restrict__ A, int64_t N,
                                                  double* __restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t j = blockIdx.y;
  if (i < N) out[i * N + j] = (j <= i) ? A[i + j * N] : 0.0;
}

// =================================================================================================
// dtype bridge.  TB_F32 handles (fp32 models, e.g. BASELINE config 5) take and return float arrays: whole inputs are widened
// to device doubles and outputs narrowed back.  Their posterior cache is fp64.  select_engine runs their candidate GEMMs on
// the int8 engine with fewer digits than an fp64 handle gets: the fewest digits int8_select admits (3 digits / 6 products,
// 4 / 10 or 5 / 15), else the 4 leading planes (10 products) of the 6-digit split.
// Above N = 16384 and on engine 0 they run the fp64 DMMA kernels, as fp64 handles do.
// =================================================================================================
__global__ void widen_kernel(const float* __restrict__ in, int64_t n, double* __restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (double)in[i];
}
__global__ void narrow_kernel(const double* __restrict__ in, int64_t n, float* __restrict__ out) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (float)in[i];
}

// The arrays of one call in the handle's dtype, as device doubles.  TB_F64 handles: the caller's pointers, with no CUDA call.
// TB_F32 handles: one device buffer per staged array, one widen / narrow launch per array, and finish() waits once.
struct DtypeBridge {
  tb_gp* gp;
  bool f32;
  std::vector<DevBuf> allocs;
  struct Pending { double* dev; void* user; int64_t n; };
  std::vector<Pending> outs;
  explicit DtypeBridge(tb_gp* g) : gp(g), f32(g->dtype == TB_F32) {}
  int alloc(void** p, size_t bytes) {
    if (allocs.empty()) TB_CUDA(cudaSetDevice(gp->device));
    allocs.emplace_back();
    TB_TRY(allocs.back().reserve(std::max<size_t>(bytes, 16)));
    *p = allocs.back().p;
    return 0;
  }
  int in(const void* user, int64_t n, const double** out) {  // float (host or device) -> device double
    *out = (const double*)user;
    if (!f32) return 0;
    *out = nullptr;
    if (!user || n == 0) return 0;
    const float* src = (const float*)user;
    if (!is_device_ptr(user)) {
      void* tmp;
      TB_TRY(alloc(&tmp, sizeof(float) * n));
      TB_CUDA(cudaMemcpyAsync(tmp, user, sizeof(float) * n, cudaMemcpyHostToDevice, gp->stream));
      src = (const float*)tmp;
    }
    void* d;
    TB_TRY(alloc(&d, sizeof(double) * n));
    widen_kernel<<<(unsigned)((n + 255) / 256), 256, 0, gp->stream>>>(src, n, (double*)d);
    TB_LAUNCHED();
    *out = (const double*)d;
    return 0;
  }
  int out(void* user, int64_t n, double** dev) {  // device double scratch, narrowed into `user` by finish()
    *dev = (double*)user;
    if (!f32) return 0;
    *dev = nullptr;
    if (!user || n == 0) return 0;
    void* d;
    TB_TRY(alloc(&d, sizeof(double) * n));
    *dev = (double*)d;
    outs.push_back({(double*)d, user, n});
    return 0;
  }
  int finish() {
    if (!f32) return 0;
    for (auto& o : outs) {
      float* dst = (float*)o.user;
      void* tmp = nullptr;
      const bool dev = is_device_ptr(o.user);
      if (!dev) {
        TB_TRY(alloc(&tmp, sizeof(float) * o.n));
        dst = (float*)tmp;
      }
      narrow_kernel<<<(unsigned)((o.n + 255) / 256), 256, 0, gp->stream>>>(o.dev, o.n, dst);
      TB_LAUNCHED();
      if (!dev) TB_CUDA(cudaMemcpyAsync(o.user, tmp, sizeof(float) * o.n, cudaMemcpyDeviceToHost, gp->stream));
    }
    TB_CUDA(cudaStreamSynchronize(gp->stream));
    TB_CUDA(cudaGetLastError());
    return 0;
  }
};

}  // namespace tb

#define TB_CUSOLVER(expr)                                                                          \
  do {                                                                                             \
    cusolverStatus_t _s = (expr);                                                                  \
    if (_s != CUSOLVER_STATUS_SUCCESS) return tb::fail(std::string(#expr) + ": cusolver status " + \
                                                       std::to_string((int)_s), tb::ERR_RUNTIME);  \
  } while (0)
#define TB_CUBLAS(expr)                                                                        \
  do {                                                                                         \
    cublasStatus_t _s = (expr);                                                                \
    if (_s != CUBLAS_STATUS_SUCCESS) return tb::fail(std::string(#expr) + ": cublas status " + \
                                                     std::to_string((int)_s), tb::ERR_RUNTIME);\
  } while (0)

static const char* kVersion = "trieste_b200 0.2 (sm_90a; fp64 DMMA + int8 wgmma digit GEMMs)";

extern "C" {

const char* tb_last_error(void) { return tb::last_error().c_str(); }
const char* tb_version(void) { return kVersion; }
int tb_device_count(int* count) {
  TB_CHECK(count != nullptr, "tb_device_count: null output");
  cudaError_t e = cudaGetDeviceCount(count);
  if (e != cudaSuccess) {
    *count = 0;
    cudaGetLastError();
    return tb::fail(std::string("cudaGetDeviceCount: ") + cudaGetErrorString(e), tb::ERR_RUNTIME);
  }
  return 0;
}
int64_t tb_launch_count(void) { return tb::launch_counter().load(); }
void tb_launch_count_reset(void) { tb::launch_counter().store(0); }

int tb_gp_create(tb_gp** out, int device, int dtype) {
  TB_CHECK(out != nullptr, "tb_gp_create: null output");
  TB_CHECK(dtype == TB_F64 || dtype == TB_F32, "tb_gp_create: dtype must be TB_F64 or TB_F32");
  int n = 0;
  TB_TRY(tb_device_count(&n));
  TB_CHECK_CODE(n > 0, "tb_gp_create: no CUDA device visible (this library has no CPU fallback)", tb::ERR_RUNTIME);
  TB_CHECK(device >= 0 && device < n, "tb_gp_create: device index out of range");
  TB_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  TB_CUDA(cudaGetDeviceProperties(&prop, device));
  TB_CHECK(prop.major == 9 && prop.minor == 0, "tb_gp_create: this library is built for sm_90a (H100) only; found sm_" +
                                 std::to_string(prop.major) + std::to_string(prop.minor));
  tb_gp* gp = new tb_gp();
  gp->device = device;
  gp->dtype = dtype;
  if (const char* e = std::getenv("TB_FACTOR")) gp->factor_own = std::string(e) != "cusolver";
  {
    // the handle's stream at the highest priority: a caller that runs its own work on other streams (tb_gp_stream) gets the
    // candidate GEMMs scheduled first
    int least = 0, greatest = 0;
    TB_CUDA(cudaDeviceGetStreamPriorityRange(&least, &greatest));
    TB_CUDA(cudaStreamCreateWithPriority(&gp->stream, cudaStreamNonBlocking, greatest));
  }
  TB_TRY(tb::kernels_init());
  *out = gp;
  return 0;
}

int tb_gp_destroy(tb_gp* gp) {
  if (!gp) return 0;
  cudaSetDevice(gp->device);
  cudaStreamSynchronize(gp->stream);
  for (auto& ev : gp->prof_events) {
    cudaEventDestroy(ev.first);
    cudaEventDestroy(ev.second);
  }
  if (gp->cusolver) cusolverDnDestroy(gp->cusolver);
  if (gp->cublas) cublasDestroy(gp->cublas);
  if (gp->stream) cudaStreamDestroy(gp->stream);
  delete gp;  // frees the device buffers
  return 0;
}

int tb_gp_set_data(tb_gp* gp, const void* X_in, const void* y_in, int64_t N, int D) {
  TB_CHECK(gp && X_in && y_in, "tb_gp_set_data: null argument");
  TB_CHECK(N > 0, "tb_gp_set_data: dataset must be populated (N > 0)");
  TB_CHECK(D > 0 && tb::pick_dp(D) > 0, "tb_gp_set_data: input dimension must be in [1, 32]");
  TB_CHECK(N <= 65535, "tb_gp_set_data: N > 65535 is not supported");  // grid.y of the per-column kernels
  tb::DtypeBridge br(gp);
  const double *X, *y;
  TB_TRY(br.in(X_in, N * D, &X));
  TB_TRY(br.in(y_in, N, &y));
  TB_CUDA(cudaSetDevice(gp->device));
  gp->N = N;
  gp->D = D;
  gp->DP = tb::pick_dp(D);
  gp->nkc = (int)((N + BK - 1) / BK);
  gp->NB = (int)((N + BM - 1) / BM);
  TB_TRY(gp->dX.reserve(sizeof(double) * N * D));
  TB_TRY(gp->dy.reserve(sizeof(double) * N));
  TB_CUDA(cudaMemcpyAsync(gp->dX.p, X, sizeof(double) * N * D, cudaMemcpyDefault, gp->stream));
  TB_CUDA(cudaMemcpyAsync(gp->dy.p, y, sizeof(double) * N, cudaMemcpyDefault, gp->stream));
  TB_CUDA(cudaStreamSynchronize(gp->stream));
  gp->have_data = true;
  gp->cache_valid = false;
  if ((int)gp->ls.size() != D && gp->ls.size() == 1) gp->ls.assign(D, gp->ls[0]);
  return 0;
}

int tb_gp_set_hyper(tb_gp* gp, int kernel, double variance, const double* lengthscales, int n_ls,
                    double noise_variance, double mean_const) {
  TB_CHECK(gp && lengthscales, "tb_gp_set_hyper: null argument");
  TB_CHECK(kernel >= TB_RBF && kernel <= TB_MATERN52, "tb_gp_set_hyper: unknown kernel kind");
  TB_CHECK(variance > 0.0, "tb_gp_set_hyper: kernel variance must be positive");
  TB_CHECK(noise_variance > 0.0, "tb_gp_set_hyper: likelihood variance must be positive");
  TB_CHECK(n_ls >= 1, "tb_gp_set_hyper: need at least one lengthscale");
  for (int i = 0; i < n_ls; ++i)
    TB_CHECK(lengthscales[i] > 0.0, "tb_gp_set_hyper: lengthscales must be positive");
  TB_CHECK(!gp->have_data || n_ls == 1 || n_ls == gp->D,
           "tb_gp_set_hyper: lengthscales must have 1 or D entries");
  gp->kernel = kernel;
  gp->variance = variance;
  gp->noise = noise_variance;
  gp->mean_const = mean_const;
  gp->ls.assign(lengthscales, lengthscales + n_ls);
  if (gp->have_data && n_ls == 1) gp->ls.assign(gp->D, lengthscales[0]);
  gp->have_hyper = true;
  gp->cache_valid = false;
  return 0;
}

static int scale_inputs(tb_gp* gp) {
  const int D = gp->D, DP = gp->DP;
  const int64_t rows = (int64_t)gp->NB * BM;
  std::vector<double> inv_ls(DP, 0.0);
  for (int d = 0; d < D; ++d) inv_ls[d] = 1.0 / gp->ls[d];
  TB_TRY(gp->dInvLs.reserve(sizeof(double) * DP));
  TB_CUDA(cudaMemcpyAsync(gp->dInvLs.p, inv_ls.data(), sizeof(double) * DP, cudaMemcpyHostToDevice, gp->stream));
  TB_TRY(gp->dXs.reserve(sizeof(double) * rows * DP));
  int64_t tot = rows * DP;
  scale_inputs_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, gp->stream>>>(gp->dX.as<double>(), gp->dInvLs.as<double>(), gp->N, D,
                                                                            DP, rows, gp->dXs.as<double>());
  TB_LAUNCHED();
  return 0;
}

// cuSOLVER / cuBLAS handles exist only for the TB_FACTOR=cusolver cross-check path: created on first use
static int ensure_library_handles(tb_gp* gp) {
  if (gp->cublas && gp->cusolver) return 0;
  if (!gp->cublas) {
    TB_CUBLAS(cublasCreate(&gp->cublas));
    TB_CUBLAS(cublasSetStream(gp->cublas, gp->stream));
  }
  if (!gp->cusolver) {
    TB_CUSOLVER(cusolverDnCreate(&gp->cusolver));
    TB_CUSOLVER(cusolverDnSetStream(gp->cusolver, gp->stream));
  }
  return 0;
}

// alpha = Linv^T (Linv (y - m)) by two triangular mat-vecs on the current Linv
static int alpha_from_linv(tb_gp* gp) {
  const int64_t N = gp->N, rows = (int64_t)gp->NB * BM;
  cudaStream_t st = gp->stream;
  TB_TRY(gp->sMisc.reserve(sizeof(double) * 2 * rows));
  double* err = gp->sMisc.as<double>();
  double* tmp = err + rows;
  residual_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, st>>>(gp->dy.as<double>(), N, rows, gp->mean_const, err);
  TB_LAUNCHED();
  TB_CUDA(cudaMemsetAsync(gp->dAlpha.p, 0, sizeof(double) * rows, st));
  fac::trmv_lower_kernel<<<(unsigned)((N + 7) / 8), 256, 0, st>>>(gp->dLinv.as<double>(), N, err, tmp);
  TB_LAUNCHED();
  fac::trmv_lower_t_kernel<<<(unsigned)((N + 7) / 8), 256, 0, st>>>(gp->dLinv.as<double>(), N, tmp, gp->dAlpha.as<double>());
  TB_LAUNCHED();
  return 0;
}

// Blocked Cholesky (factor.cuh) of the n x n column-major matrix A in place on gp->stream: L in the lower triangle, the
// inverses of L's diagonal 128-blocks in dinv [ceil(n/128)][128][128].  *minor: the first leading minor that is not positive
// definite (1-based), 0 if none.  Waits for the stream.
static int blocked_cholesky(tb_gp* gp, double* A, int64_t n, double* dinv, int* minor) {
  cudaStream_t st = gp->stream;
  TB_TRY(gp->dInfo.reserve(sizeof(int)));
  TB_CUDA(cudaMemsetAsync(gp->dInfo.p, 0, sizeof(int), st));
  const int nbk = (int)((n + fac::FB - 1) / fac::FB);
  const size_t diag_smem = sizeof(double) * fac::FB * (fac::FB + 1);
  for (int jb = 0; jb < nbk; ++jb) {
    const int j0 = jb * fac::FB;
    fac::chol_diag_kernel<<<1, fac::THREADS, diag_smem, st>>>(A, n, j0, dinv, gp->dInfo.as<int>());
    TB_LAUNCHED();
    const int64_t below = n - (int64_t)(j0 + fac::FB);
    if (below > 0) {
      const unsigned t = (unsigned)((below + fac::FB - 1) / fac::FB);
      fac::chol_panel_kernel<<<t, fac::THREADS, fac::GEMM_SMEM, st>>>(A, n, j0, dinv);
      TB_LAUNCHED();
      fac::chol_syrk_kernel<<<dim3(t, t), fac::THREADS, fac::GEMM_SMEM, st>>>(A, n, j0);
      TB_LAUNCHED();
    }
  }
  *minor = 0;
  TB_CUDA(cudaMemcpyAsync(minor, gp->dInfo.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  TB_CUDA(cudaStreamSynchronize(st));
  TB_CUDA(cudaGetLastError());
  return 0;
}

// pack the lower triangle of Linv into DMMA-fragment-ordered panels and move to the next cache generation, which makes every
// derived operand stale.  appended_from > 0: the cache was extended from that many rows by tb_gp_append_data; a dense K^-1 of
// the previous generation is grown by the same rank instead.
static int finish_cache(tb_gp* gp, int64_t appended_from = 0) {
  const int64_t N = gp->N;
  cudaStream_t st = gp->stream;
  int64_t npanels = rowblock_panel_offset(gp->NB);
  TB_TRY(gp->dLinvP.reserve(sizeof(double) * npanels * PANEL));
  TB_CUDA(cudaMemsetAsync(gp->dLinvP.p, 0, sizeof(double) * npanels * PANEL, st));
  dim3 grid((unsigned)std::min<int64_t>(gp->nkc, (int64_t)gp->NB * (BM / BK)), (unsigned)gp->NB);
  pack_lower_panels_kernel<<<grid, 256, 0, st>>>(gp->dLinv.as<double>(), N, gp->nkc, gp->dLinvP.as<double>());
  TB_LAUNCHED();
  TB_CUDA(cudaStreamSynchronize(st));
  TB_CUDA(cudaGetLastError());
  gp->cache_valid = true;
  const bool grow_kinv = appended_from > 0 && gp->kinv_gen == gp->cache_gen;
  ++gp->cache_gen;  // every operand derived from the posterior is rebuilt before its next use
  if (grow_kinv) {
    TB_TRY(gp->dKinvSpare.reserve(sizeof(double) * N * N));
    fac::kinv_grow_kernel<<<dim3((unsigned)((N + 127) / 128), (unsigned)N), 128, 0, st>>>(gp->dKinv.as<double>(), appended_from,
                                                                                       gp->dLinv.as<double>(), N, gp->dKinvSpare.as<double>());
    TB_LAUNCHED();
    TB_CUDA(cudaStreamSynchronize(st));
    TB_CUDA(cudaGetLastError());
    std::swap(gp->dKinv, gp->dKinvSpare);
    gp->kinv_gen = gp->cache_gen;
  }
  return 0;
}

int tb_gp_update_posterior_cache(tb_gp* gp) {
  TB_CHECK(gp, "tb_gp_update_posterior_cache: null handle");
  TB_CHECK(gp->have_data && gp->have_hyper, "tb_gp_update_posterior_cache: set data and hyper-parameters first");
  TB_CHECK((int)gp->ls.size() == gp->D, "tb_gp_update_posterior_cache: lengthscales must have 1 or D entries");
  TB_CUDA(cudaSetDevice(gp->device));
  const int64_t N = gp->N;
  const int D = gp->D, DP = gp->DP;
  const int64_t rows = (int64_t)gp->NB * BM;  // >= nkc*16 and >= nst*64
  cudaStream_t st = gp->stream;

  TB_TRY(scale_inputs(gp));
  TB_TRY(gp->dL.reserve(sizeof(double) * N * N));
  TB_TRY(gp->dLinv.reserve(sizeof(double) * N * N));
  {
    dim3 grid((unsigned)((N + 127) / 128), (unsigned)N);
    double* K = gp->dL.as<double>();
    const double* Xs = gp->dXs.as<double>();
    with_kind(gp->kernel, [&](auto K_) { gram_kernel<decltype(K_)::value><<<grid, 128, 0, st>>>(Xs, N, DP, gp->variance, gp->noise, K); });
    TB_LAUNCHED();
  }
  TB_TRY(gp->dInfo.reserve(sizeof(int)));
  TB_TRY(gp->dAlpha.reserve(sizeof(double) * rows));
  if (gp->factor_own) {
    // ---- hand-written path (factor.cuh): blocked Cholesky, Linv, alpha on the DMMA pipe; no library call ----
    const int nbk = (int)((N + fac::FB - 1) / fac::FB);
    TB_TRY(gp->dDinv.reserve(sizeof(double) * (size_t)nbk * fac::FB * fac::FB));
    double* A = gp->dL.as<double>();
    int info;
    TB_TRY(blocked_cholesky(gp, A, N, gp->dDinv.as<double>(), &info));
    TB_CHECK_CODE(info == 0, "tb_gp_update_posterior_cache: Cholesky decomposition was not successful "
                        "(K + noise*I not positive definite at leading minor " + std::to_string(info) + ")", tb::ERR_NUMERIC);
    {
      dim3 grid((unsigned)((N + 127) / 128), (unsigned)N);
      zero_upper_kernel<<<grid, 128, 0, st>>>(N, A);
      TB_LAUNCHED();
    }
    TB_CUDA(cudaMemsetAsync(gp->dLinv.p, 0, sizeof(double) * N * N, st));
    // Linv by recursive doubling: diagonal 128-blocks first, then block sizes 128, 256, ... (two GEMM launches per level)
    fac::trinv_diag_kernel<<<nbk, 256, 0, st>>>(gp->dLinv.as<double>(), N, gp->dDinv.as<double>());
    TB_LAUNCHED();
    if (nbk > 1) {
      TB_TRY(gp->dKinv.reserve(sizeof(double) * N * N));  // scratch T (the buffer is reused later for K^-1)
      for (int64_t n = fac::FB; n < (int64_t)nbk * fac::FB; n *= 2) {
        const unsigned tiles = (unsigned)(n / fac::FB), pairs = (unsigned)((N + 2 * n - 1) / (2 * n));
        fac::trinv_level_kernel<1><<<dim3(tiles, tiles, pairs), fac::THREADS, fac::GEMM_SMEM, st>>>(A, gp->dLinv.as<double>(),
                                                                                                   gp->dKinv.as<double>(), N, (int)n);
        TB_LAUNCHED();
        fac::trinv_level_kernel<2><<<dim3(tiles, tiles, pairs), fac::THREADS, fac::GEMM_SMEM, st>>>(A, gp->dLinv.as<double>(),
                                                                                                   gp->dKinv.as<double>(), N, (int)n);
        TB_LAUNCHED();
      }
    }
    TB_TRY(alpha_from_linv(gp));
  } else {
    // ---- library path (TB_FACTOR=cusolver): cuSOLVER potrf / potrs + cuBLAS trsm; kept as a cross-check ----
    TB_TRY(ensure_library_handles(gp));
    int lwork = 0;
    TB_CUSOLVER(cusolverDnDpotrf_bufferSize(gp->cusolver, CUBLAS_FILL_MODE_LOWER, (int)N, gp->dL.as<double>(), (int)N, &lwork));
    TB_TRY(gp->dWork.reserve(sizeof(double) * (size_t)std::max(lwork, 1)));
    TB_CUSOLVER(cusolverDnDpotrf(gp->cusolver, CUBLAS_FILL_MODE_LOWER, (int)N, gp->dL.as<double>(), (int)N,
                                 gp->dWork.as<double>(), lwork, gp->dInfo.as<int>()));
    int info = 0;
    TB_CUDA(cudaMemcpyAsync(&info, gp->dInfo.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    TB_CUDA(cudaStreamSynchronize(st));
    TB_CHECK_CODE(info == 0, "tb_gp_update_posterior_cache: Cholesky decomposition was not successful "
                        "(K + noise*I not positive definite at leading minor " + std::to_string(info) + ")", tb::ERR_NUMERIC);
    {
      dim3 grid((unsigned)((N + 127) / 128), (unsigned)N);
      zero_upper_kernel<<<grid, 128, 0, st>>>(N, gp->dL.as<double>());
      TB_LAUNCHED();
    }
    residual_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, st>>>(gp->dy.as<double>(), N, rows, gp->mean_const,
                                                                    gp->dAlpha.as<double>());
    TB_LAUNCHED();
    TB_CUSOLVER(cusolverDnDpotrs(gp->cusolver, CUBLAS_FILL_MODE_LOWER, (int)N, 1, gp->dL.as<double>(), (int)N,
                                 gp->dAlpha.as<double>(), (int)N, gp->dInfo.as<int>()));
    int64_t tot = N * N;
    identity_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(N, gp->dLinv.as<double>());
    TB_LAUNCHED();
    const double one = 1.0;
    TB_CUBLAS(cublasDtrsm(gp->cublas, CUBLAS_SIDE_LEFT, CUBLAS_FILL_MODE_LOWER, CUBLAS_OP_N, CUBLAS_DIAG_NON_UNIT, (int)N,
                          (int)N, &one, gp->dL.as<double>(), (int)N, gp->dLinv.as<double>(), (int)N));
  }
  return finish_cache(gp);
}

// Rank-m append (SURVEY.md §8f-1): the reference refactorises from scratch whenever the data change
// (models.py:171-186 -> interface.py:108-112); one BO step only appends rows, so L, Linv and alpha are extended in
// O(m N^2) instead of O(N^3).  The hyper-parameters must be unchanged since the cache was built.
int tb_gp_append_data(tb_gp* gp, const void* Xnew_in, const void* ynew_in, int64_t m) {
  TB_CHECK(gp && Xnew_in && ynew_in, "tb_gp_append_data: null argument");
  TB_CHECK(gp->cache_valid, "tb_gp_append_data: posterior cache is not built: call tb_gp_update_posterior_cache first");
  TB_CHECK(m > 0 && m <= APPEND_MAX, "tb_gp_append_data: between 1 and " + std::to_string(APPEND_MAX) + " new points per call");
  const int64_t N0 = gp->N, N = N0 + m;
  TB_CHECK(N <= 65535, "tb_gp_append_data: N > 65535 is not supported");
  tb::DtypeBridge br(gp);
  const double *Xnew, *ynew;
  TB_TRY(br.in(Xnew_in, m * gp->D, &Xnew));
  TB_TRY(br.in(ynew_in, m, &ynew));
  TB_CUDA(cudaSetDevice(gp->device));
  cudaStream_t st = gp->stream;
  const int D = gp->D, DP = gp->DP;
  // grow the raw data and the two triangular factors (leading dimension N0 -> N) into the handle's spare buffers, which are
  // sized with slack (next multiple of 256 rows + 256) and ping-pong with the live ones: after the second append of a run
  // no cudaMalloc / cudaFree (both device-synchronising) is left on this path
  const int64_t cap_rows = ((N + 255) / 256) * 256 + 256;
  tb::DevBuf &nX = gp->dXspare, &ny = gp->dyspare, &nL = gp->dLspare, &nLinv = gp->dLinvSpare;
  TB_TRY(nX.reserve(sizeof(double) * cap_rows * D));
  TB_TRY(ny.reserve(sizeof(double) * cap_rows));
  TB_TRY(nL.reserve(sizeof(double) * cap_rows * cap_rows));
  TB_TRY(nLinv.reserve(sizeof(double) * cap_rows * cap_rows));
  TB_CUDA(cudaMemcpyAsync(nX.p, gp->dX.p, sizeof(double) * N0 * D, cudaMemcpyDeviceToDevice, st));
  TB_CUDA(cudaMemcpyAsync(nX.as<double>() + N0 * D, Xnew, sizeof(double) * m * D, cudaMemcpyDefault, st));
  TB_CUDA(cudaMemcpyAsync(ny.p, gp->dy.p, sizeof(double) * N0, cudaMemcpyDeviceToDevice, st));
  TB_CUDA(cudaMemcpyAsync(ny.as<double>() + N0, ynew, sizeof(double) * m, cudaMemcpyDefault, st));
  TB_CUDA(cudaMemsetAsync(nL.p, 0, sizeof(double) * N * N, st));
  TB_CUDA(cudaMemsetAsync(nLinv.p, 0, sizeof(double) * N * N, st));
  TB_CUDA(cudaMemcpy2DAsync(nL.p, sizeof(double) * N, gp->dL.p, sizeof(double) * N0, sizeof(double) * N0, N0,
                            cudaMemcpyDeviceToDevice, st));
  TB_CUDA(cudaMemcpy2DAsync(nLinv.p, sizeof(double) * N, gp->dLinv.p, sizeof(double) * N0, sizeof(double) * N0, N0,
                            cudaMemcpyDeviceToDevice, st));
  TB_CUDA(cudaStreamSynchronize(st));
  std::swap(gp->dX, nX);
  std::swap(gp->dy, ny);
  std::swap(gp->dL, nL);
  std::swap(gp->dLinv, nLinv);
  gp->N = N;
  gp->nkc = (int)((N + BK - 1) / BK);
  gp->NB = (int)((N + BM - 1) / BM);
  gp->cache_valid = false;  // until the append completes
  const int64_t rows = (int64_t)gp->NB * BM;
  TB_TRY(scale_inputs(gp));
  TB_TRY(gp->dAlpha.reserve(sizeof(double) * rows));
  // scratch: W (cross kernel block), Y = Linv0 B, U = Linv0^T Y as [N, m] column-major; S, R as [m, m]
  // sized for the largest append at the spare buffers' row capacity: no reallocation while the capacity lasts
  TB_TRY(gp->sA.reserve(sizeof(double) * (3 * cap_rows * APPEND_MAX + 2 * APPEND_MAX * APPEND_MAX)));
  double* W = gp->sA.as<double>();
  double* Y = W + N * m;
  double* U = Y + N * m;
  double* S = U + N * m;
  double* R = S + m * m;
  TB_TRY(gp->dInfo.reserve(sizeof(int)));
  TB_CUDA(cudaMemsetAsync(gp->dInfo.p, 0, sizeof(int), st));
  {
    dim3 grid((unsigned)((N + 127) / 128), (unsigned)m);
    const double* Xs = gp->dXs.as<double>();
    with_kind(gp->kernel, [&](auto K) {
      append_cross_kernel<decltype(K)::value><<<grid, 128, 0, st>>>(Xs, DP, N0, N, gp->variance, gp->noise, W);
    });
    TB_LAUNCHED();
  }
  double* L = gp->dL.as<double>();
  double* Linv = gp->dLinv.as<double>();
  trmv_lower_cols_kernel<<<dim3((unsigned)((N0 + 127) / 128), (unsigned)m), 128, 0, st>>>(Linv, N0, N, W, N, Y, N);
  TB_LAUNCHED();
  append_schur_kernel<<<dim3((unsigned)m, (unsigned)m), 256, 0, st>>>(Y, W, N0, N, (int)m, S);
  TB_LAUNCHED();
  append_chol_kernel<<<1, APPEND_MAX, 0, st>>>(S, (int)m, N0, N, L, Linv, R, gp->dInfo.as<int>());
  TB_LAUNCHED();
  trmv_lower_t_cols_kernel<<<dim3((unsigned)((N0 + 7) / 8), (unsigned)m), 256, 0, st>>>(Linv, N0, N, Y, N, U, N);
  TB_LAUNCHED();
  append_rows_kernel<<<dim3((unsigned)((N0 + 127) / 128), (unsigned)m), 128, 0, st>>>(Y, U, R, (int)m, N0, N, L, Linv);
  TB_LAUNCHED();
  int info = 0;
  TB_CUDA(cudaMemcpyAsync(&info, gp->dInfo.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  TB_CUDA(cudaStreamSynchronize(st));
  TB_CUDA(cudaGetLastError());
  TB_CHECK_CODE(info == 0, "tb_gp_append_data: Cholesky decomposition was not successful "
                      "(K + noise*I not positive definite at leading minor " + std::to_string(info) + ")", tb::ERR_NUMERIC);
  TB_TRY(alpha_from_linv(gp));
  return finish_cache(gp, N0);
}

int tb_gp_get_cholesky(tb_gp* gp, void* L_user) {
  TB_CHECK(gp && L_user, "tb_gp_get_cholesky: null argument");
  TB_CHECK(gp->cache_valid, "tb_gp_get_cholesky: posterior cache is not built");
  const int64_t N = gp->N;
  tb::DtypeBridge br(gp);
  double* L_out;
  TB_TRY(br.out(L_user, N * N, &L_out));
  TB_CUDA(cudaSetDevice(gp->device));
  TB_TRY(gp->sMisc.reserve(sizeof(double) * N * N));
  dim3 grid((unsigned)((N + 127) / 128), (unsigned)N);
  colmajor_lower_to_rowmajor_kernel<<<grid, 128, 0, gp->stream>>>(gp->dL.as<double>(), N, gp->sMisc.as<double>());
  TB_LAUNCHED();
  TB_CUDA(cudaMemcpyAsync(L_out, gp->sMisc.p, sizeof(double) * N * N, cudaMemcpyDefault, gp->stream));
  TB_CUDA(cudaStreamSynchronize(gp->stream));
  return br.finish();
}

}  // extern "C"

// =================================================================================================
// per-candidate path: chunked driver for predict / acquisition / argmax
// =================================================================================================
namespace tb {

struct EvalRequest {
  int acq = -1;  // -1: predict only
  double param = 0.0;
  const double* Xc = nullptr;  // host or device, [M, D]
  int64_t M = 0;
  double* out_vals = nullptr;  // host or device (nullable)
  double* out_mean = nullptr;
  double* out_var = nullptr;
  double* out_grad = nullptr;  // [M, D] (nullable)
  bool want_argmax = false;
  bool pen = false;  // TB_ACQ_PENALIZED: multiply by the handle's local penalty (tb_acq_set_penalization)
  bool sync = true;  // false: run_eval returns with its work queued on the handle's stream (device outputs only, no argmax)
  double best_value = 0.0;
  int64_t best_index = -1;
};

static int launch_kstar(tb_gp* gp, const double* Xc_dev, int64_t mc, int tiles, double* KsP, double* mean) {
  const double* Xs = gp->dXs.as<double>();
  const double* al = gp->dAlpha.as<double>();
  const double* il = gp->dInvLs.as<double>();
  const int N = (int)gp->N, nkc = gp->nkc, D = gp->D;
  const double var = gp->variance, mc0 = gp->mean_const;
  cudaStream_t st = gp->stream;
  with_kind_dp(gp->kernel, gp->DP, [&](auto K, auto P) {
    kstar_panels_kernel<decltype(K)::value, decltype(P)::value><<<tiles, 512, 0, st>>>(Xs, al, Xc_dev, il, N, nkc, D, mc, 0, var, mc0,
                                                                                        KsP, mean);
  });
  TB_LAUNCHED();
  TB_CUDA(cudaGetLastError());
  return 0;
}

// candidates per chunk: bounded by the Ks scratch budget, a whole number of one-CTA-per-SM waves when possible
static int64_t chunk_tiles(const tb_gp* gp) {
  const size_t per_tile = (size_t)gp->nkc * PANEL * sizeof(double);
  const size_t budget = (size_t)1536 << 20;
  int64_t t = (int64_t)(budget / per_tile);
  t = std::max<int64_t>(t, 1);
  if (t >= NUM_SMS) t = (t / NUM_SMS) * NUM_SMS;
  return std::min<int64_t>(t, NUM_SMS * 16);
}

int kernels_init() {
  TB_CUDA(cudaFuncSetAttribute(fac::chol_diag_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(double) * fac::FB * (fac::FB + 1))));
  TB_CUDA(cudaFuncSetAttribute(fac::chol_panel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fac::GEMM_SMEM));
  TB_CUDA(cudaFuncSetAttribute(fac::chol_syrk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fac::GEMM_SMEM));
  TB_CUDA(cudaFuncSetAttribute(fac::trinv_level_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fac::GEMM_SMEM));
  TB_CUDA(cudaFuncSetAttribute(fac::trinv_level_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fac::GEMM_SMEM));
  TB_CUDA(cudaFuncSetAttribute(fac::kinv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fac::GEMM_SMEM));
  TB_TRY(int8_init());
  TB_CUDA(cudaFuncSetAttribute(trigemm_kernel<false, EPI_SUMSQ>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TG_SMEM));
  TB_CUDA(cudaFuncSetAttribute(trigemm_kernel<false, EPI_SUMSQ_PACKED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TG_SMEM));
  TB_CUDA(cudaFuncSetAttribute(trigemm_kernel<false, EPI_PLAIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TG_SMEM));
  TB_CUDA(cudaFuncSetAttribute(trigemm_kernel<true, EPI_PLAIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TG_SMEM));
  return 0;
}

// Linv^T packed upper panels: built lazily, only the gradient path needs them
static int ensure_upper_panels(tb_gp* gp) {
  if (gp->upper_gen == gp->cache_gen) return 0;
  const int nkB = gp->NB * (BM / BK);
  const int64_t np = upper_panel_count(gp->NB, nkB);
  TB_TRY(gp->dLinvTP.reserve(sizeof(double) * np * PANEL));
  dim3 grid((unsigned)nkB, (unsigned)gp->NB);
  pack_upper_panels_kernel<<<grid, 256, 0, gp->stream>>>(gp->dLinv.as<double>(), gp->N, gp->NB, nkB,
                                                         gp->dLinvTP.as<double>());
  TB_LAUNCHED();
  TB_CUDA(cudaGetLastError());
  gp->upper_gen = gp->cache_gen;
  return 0;
}

// gradient assembly of one chunk (grad_kernel): the training-point sums over V = K^-1 K* in gp->sV, with the partials
// d acq / d (mean, var) in gp->sMisc
static int launch_grad(tb_gp* gp, const double* xc, int64_t mc, double* grad_dev) {
  const bool wide = mc <= 2048;  // one CTA (8 warps) per candidate when one warp each would leave SMs idle
  const int blocks = wide ? (int)mc : (int)((mc + 7) / 8);
  const double* Xs = gp->dXs.as<double>();
  const double* al = gp->dAlpha.as<double>();
  const double* il = gp->dInvLs.as<double>();
  const double* V = gp->sV.as<double>();
  const int64_t ldv = (int64_t)gp->NB * BM;
  const double* cmu = gp->sMisc.as<double>();
  const double* cvar = cmu + mc;
  with_kind_dp(gp->kernel, gp->DP, [&](auto K, auto P) {
    constexpr int KIND = decltype(K)::value, DP = decltype(P)::value;
    if (wide)
      grad_kernel<KIND, DP, 8><<<blocks, 256, 0, gp->stream>>>(Xs, al, xc, il, (int)gp->N, gp->D, mc, V, ldv, cmu, cvar, gp->variance,
                                                               fm::Consts(), grad_dev);
    else
      grad_kernel<KIND, DP, 1><<<blocks, 256, 0, gp->stream>>>(Xs, al, xc, il, (int)gp->N, gp->D, mc, V, ldv, cmu, cvar, gp->variance,
                                                               fm::Consts(), grad_dev);
  });
  TB_LAUNCHED();
  TB_CUDA(cudaGetLastError());
  return 0;
}

static inline bool gibbon_repulsion_kind(int acq) { return acq == TB_ACQ_GIBBON_REPULSION || acq == TB_ACQ_GIBBON; }

// the tails' second parameter: the feasibility kinds' alpha (tb_acq_set_feasibility), else the likelihood noise variance
static inline double tail_aux(const tb_gp* gp, int acq) { return feasibility_kind(acq) ? gp->feasAlpha : gp->noise; }

// GIBBON cross term of one chunk (ensure_gibbon has run): |u|^2 into sGib[0, mc); with keep_u also u into sGib[2 mc, ...) for
// gibbon_grad_kernel.  One launch whatever m.
static int launch_gibbon_cross(tb_gp* gp, cudaStream_t st, const double* xc, int64_t mc, bool keep_u) {
  TB_TRY(gp->sGib.reserve(sizeof(double) * (size_t)mc * (2 + (keep_u ? gp->gibMp : 0))));
  double* uu = gp->sGib.as<double>();
  double* U = keep_u ? uu + 2 * mc : nullptr;
  const unsigned blocks = (unsigned)((mc + 127) / 128);
  with_kind_dp(gp->kernel, gp->DP, [&](auto K, auto P) {
    gibbon_cross_kernel<decltype(K)::value, decltype(P)::value><<<blocks, 128, 0, st>>>(
        gp->dXs.as<double>(), gp->dGibWhat.as<double>(), gp->dGibPs.as<double>(), gp->dGibLinv.as<double>(), xc, gp->dInvLs.as<double>(),
        (int)gp->N, gp->D, gp->gibM, gp->gibMp, mc, gp->variance, fm::Consts(), uu, U);
  });
  TB_LAUNCHED();
  TB_CUDA(cudaGetLastError());
  return 0;
}

// the |u|^2 part of the repulsion gradient, added in place to gd (device [mc][D]) after the gradient assembly
static int launch_gibbon_grad(tb_gp* gp, cudaStream_t st, const double* xc, int64_t mc, double* gd) {
  const double* uu = gp->sGib.as<double>();
  const unsigned blocks = (unsigned)((mc + 7) / 8);
  with_kind_dp(gp->kernel, gp->DP, [&](auto K, auto P) {
    gibbon_grad_kernel<decltype(K)::value, decltype(P)::value><<<blocks, 256, 0, st>>>(
        gp->dXs.as<double>(), gp->dGibWhat.as<double>(), gp->dGibPs.as<double>(), gp->dGibLinv.as<double>(), xc, gp->dInvLs.as<double>(),
        (int)gp->N, gp->D, gp->gibM, gp->gibMp, mc, gp->variance, uu + 2 * mc, uu + mc, gd);
  });
  TB_LAUNCHED();
  TB_CUDA(cudaGetLastError());
  return 0;
}

// d acq / d (mean, var) of one chunk into sMisc (cmu [mc], cvar [mc]); the GIBBON repulsion kinds first run the cross term
// of the chunk, whose |u|^2 the partials and the tail read
static int launch_partials(tb_gp* gp, cudaStream_t st, int acq, double param, const double* partial, int G, int64_t McPad,
                           const double* mean, const double* xc, int64_t mc) {
  double* cmu = gp->sMisc.as<double>();
  const bool gib = gibbon_repulsion_kind(acq);
  if (gib) TB_TRY(launch_gibbon_cross(gp, st, xc, mc, true));
  double* g = gib ? gp->sGib.as<double>() : nullptr;
  acq_partials_kernel<<<(unsigned)((mc + 255) / 256), 256, 0, st>>>(partial, G, McPad, mean, mc, gp->variance, acq, param,
                                                                    tail_aux(gp, acq), gp->dMes.as<double>(), gp->mesS, cmu, cmu + mc,
                                                                    g, gp->gibW, g ? g + mc : nullptr);
  TB_LAUNCHED();
  return 0;
}

// The acquisition tail of one chunk.  A penalised request (rq.pen) multiplies the value, and the gradient in gd (device,
// [mc][D], nullable) in place, by the handle's local penalty at the candidates xc (device, [mc][D]); so the tail must run
// after the gradient assembly and before the gradient leaves the device.  Unpenalised requests run the plain tail.  The GIBBON
// repulsion kinds add their term: without a gradient the cross kernel runs here; with one it ran before the partials
// (launch_partials) and its |u|^2 gradient part is added to gd here.
static int launch_tail(tb_gp* gp, cudaStream_t st, const EvalRequest& rq, const double* partial, int G, int64_t McPad,
                       const double* mean, int64_t mc, int64_t c0, double* d_vals, double* d_mean, double* d_var,
                       const double* xc, double* gd, const int64_t* idx_map = nullptr) {
  const int blocks = (int)((mc + 255) / 256);
  double* bb = rq.want_argmax ? gp->sBlkBest.as<double>() : nullptr;
  int64_t* bi = rq.want_argmax ? gp->sBlkIdx.as<int64_t>() : nullptr;
  TailPenalty pen;
  if (gibbon_repulsion_kind(rq.acq)) {
    if (gd)
      TB_TRY(launch_gibbon_grad(gp, st, xc, mc, gd));
    else
      TB_TRY(launch_gibbon_cross(gp, st, xc, mc, false));
    pen.gib_uu = gp->sGib.as<double>();
    pen.gib_w = gp->gibW;
  }
  if (rq.pen) {
    pen.xc = xc;
    pen.pend = gp->dPen.as<double>();
    pen.radius = pen.pend + (int64_t)gp->penP * gp->D;
    pen.scale = pen.radius + gp->penP;
    pen.grad = gd;
    pen.P = gp->penP;
    pen.D = gp->D;
    pen.kind = gp->penKind;
    tail_kernel<true><<<blocks, 256, 0, st>>>(partial, G, McPad, mean, mc, c0, gp->variance, rq.acq, rq.param, tail_aux(gp, rq.acq),
                                              gp->dMes.as<double>(), gp->mesS, d_vals, d_mean, d_var, bb, bi, idx_map, pen);
  } else {
    tail_kernel<false><<<blocks, 256, 0, st>>>(partial, G, McPad, mean, mc, c0, gp->variance, rq.acq, rq.param, tail_aux(gp, rq.acq),
                                               gp->dMes.as<double>(), gp->mesS, d_vals, d_mean, d_var, bb, bi, idx_map, pen);
  }
  TB_LAUNCHED();
  return 0;
}

// The dense K^-1 whose digit tiles the int8 engine's gradient path multiplies with the K* digits (V = K^-1 K*, one dense digit
// GEMM): Linv^T Linv (lower triangle, ld = N), O(N^3) on the DMMA pipe (cuSOLVER potri on the cross-check path), lazily once
// per full cache refresh; appends grow it in O(m N^2) (finish_cache / fac::kinv_grow_kernel)
static int ensure_kinv_dense(tb_gp* gp) {
  const int64_t N = gp->N;
  if (gp->kinv_gen == gp->cache_gen) return 0;
  cudaStream_t st = gp->stream;
  TB_TRY(gp->dKinv.reserve(sizeof(double) * N * N));
  if (gp->factor_own) {
    const unsigned t = (unsigned)((N + fac::FB - 1) / fac::FB);
    fac::kinv_kernel<<<dim3(t, t), fac::THREADS, fac::GEMM_SMEM, st>>>(gp->dLinv.as<double>(), gp->dKinv.as<double>(), N);
    TB_LAUNCHED();
  } else {
    TB_TRY(ensure_library_handles(gp));
    TB_CUDA(cudaMemcpyAsync(gp->dKinv.p, gp->dL.p, sizeof(double) * N * N, cudaMemcpyDeviceToDevice, st));
    int lwork = 0;
    cusolverStatus_t cs = cusolverDnDpotri_bufferSize(gp->cusolver, CUBLAS_FILL_MODE_LOWER, (int)N, gp->dKinv.as<double>(), (int)N, &lwork);
    TB_CHECK_CODE(cs == CUSOLVER_STATUS_SUCCESS, "cusolverDnDpotri_bufferSize failed", tb::ERR_RUNTIME);
    TB_TRY(gp->dWork.reserve(sizeof(double) * (size_t)std::max(lwork, 1)));
    cs = cusolverDnDpotri(gp->cusolver, CUBLAS_FILL_MODE_LOWER, (int)N, gp->dKinv.as<double>(), (int)N, gp->dWork.as<double>(), lwork,
                          gp->dInfo.as<int>());
    TB_CHECK_CODE(cs == CUSOLVER_STATUS_SUCCESS, "cusolverDnDpotri failed", tb::ERR_RUNTIME);
  }
  gp->kinv_gen = gp->cache_gen;
  return 0;
}

// Does this argmax call take the screened path (argmax_screened)?  EI / log-EI, unpenalised, nothing but the winner out, and
// device candidates (the survivors are gathered from them).  TB_ARGMAX_SCREEN=0: never; =1: always (small M too);
// unset: from SCREEN_MIN_M candidates (a conservative bound, not tuned: below it a call takes a few ms at most, and the
// screen's extra launches and host round trip are a larger share of it).
constexpr int64_t SCREEN_MIN_M = 16384;
static bool argmax_screen_wanted(const EvalRequest& rq, bool xc_dev) {
  if (!rq.want_argmax || rq.out_vals || rq.out_mean || rq.out_var || rq.out_grad || rq.pen || !xc_dev) return false;
  if (rq.acq != TB_ACQ_EI && rq.acq != TB_ACQ_LOG_EI) return false;
  if (const char* e = std::getenv("TB_ARGMAX_SCREEN"))
    if (*e) return std::atoi(e) != 0;
  return rq.M >= SCREEN_MIN_M;
}

// The tensor-core pass's training columns (tc_mean_bounds_kernel) from the fp32 mirror rows h (x', n = |x'|^2, a, |a|):
// columns with a > 0 first, then the others, each class padded with zero columns to whole n8 slices; per slice, lane
// (g, tg)'s B fragments of column g (k = 16 kk + 2 tg + {0, 1} and + 8) and then the slice's 8 weights |a|; zero stages up to
// a whole one.  *f16_ok: every |X'_d| < 2^14 and n < 2^15, so the fp16 operands stay finite.
static std::vector<unsigned char> prescreen_tc_columns(const std::vector<float>& h, int64_t N, int DP, int W, int* nsl,
                                                       int* npos_sl, bool* f16_ok) {
  const int NK = pre::tc_nk(DP), K = 16 * NK, SL = pre::tc_slices(DP), SLB = pre::tc_slice_bytes(DP);
  std::vector<int64_t> cls[2];
  for (int64_t j = 0; j < N; ++j) cls[h[(size_t)j * W + DP + 1] > 0.0f ? 0 : 1].push_back(j);
  *npos_sl = (int)((cls[0].size() + 7) / 8);
  *nsl = *npos_sl + (int)((cls[1].size() + 7) / 8);
  std::vector<unsigned char> out((size_t)((*nsl + SL - 1) / SL) * SL * SLB, 0);
  std::vector<__half> col((size_t)K);
  *f16_ok = true;
  auto split = [](float x, __half* lo) {
    const __half hi = __float2half_rn(x);
    *lo = __float2half_rn(x - __half2float(hi));
    return hi;
  };
  for (int c = 0; c < 8 * *nsl; ++c) {
    const int k = c < 8 * *npos_sl ? 0 : 1;
    const int64_t i = k == 0 ? c : c - 8 * *npos_sl;
    if (i >= (int64_t)cls[k].size()) continue;
    const float* r = &h[(size_t)cls[k][i] * W];
    std::fill(col.begin(), col.end(), __float2half_rn(0.0f));
    for (int d = 0; d < DP; ++d) {
      __half lo;
      const __half hi = split(r[d], &lo);
      col[d] = col[DP + d] = __float2half_rn(-2.0f * __half2float(hi));
      col[2 * DP + d] = __float2half_rn(-2.0f * __half2float(lo));
      *f16_ok = *f16_ok && std::fabs(r[d]) < 16384.0f;
    }
    col[3 * DP] = split(r[DP], &col[3 * DP + 1]);
    *f16_ok = *f16_ok && r[DP] < 32768.0f;
    unsigned char* sp = &out[(size_t)(c / 8) * SLB];
    const int g = c % 8;
    for (int tg = 0; tg < 4; ++tg)
      for (int kk = 0; kk < NK; ++kk)
        for (int hf = 0; hf < 2; ++hf) std::memcpy(sp + ((g * 4 + tg) * NK + kk) * 8 + 4 * hf, &col[kk * 16 + 8 * hf + 2 * tg], 4);
    std::memcpy(sp + 256 * NK + 4 * g, &r[DP + 2], 4);
  }
  return out;
}

// Mirrors of the posterior for the bound pass (prescreen.cuh) and the constants of its error bound (DESIGN.md §4d),
// rebuilt on the host whenever the posterior cache moves (cache_gen: refits and appends).  x' = (x / l - centre) * pre: the
// centre is the midpoint of the training rows' bounding box (a shift leaves distances alone and shrinks the norms the
// expansion form cancels), pre folds the kernel's distance scale and log2(e) into the coordinates.
static int prescreen_ensure(tb_gp* gp) {
  if (gp->pre_gen == gp->cache_gen) return 0;
  const int64_t N = gp->N;
  const int D = gp->D, DP = gp->DP;
  const int W = ((DP + 3 + 3) / 4) * 4;
  const int64_t rows = ((N + pre::KS - 1) / pre::KS) * pre::KS;
  cudaStream_t st = gp->stream;
  std::vector<double> xs((size_t)N * DP), al((size_t)N);
  TB_CUDA(cudaMemcpyAsync(xs.data(), gp->dXs.p, sizeof(double) * N * DP, cudaMemcpyDeviceToHost, st));
  TB_CUDA(cudaMemcpyAsync(al.data(), gp->dAlpha.p, sizeof(double) * N, cudaMemcpyDeviceToHost, st));
  TB_CUDA(cudaStreamSynchronize(st));
  const double LOG2E = 1.4426950408889634, LN2 = 0.6931471805599453;
  double pre2, cq;  // pre^2, and |d ln k / dq| in pre-scaled units (expansion-form kernels)
  switch (gp->kernel) {
    case TB_RBF: pre2 = 0.5 * LOG2E, cq = LN2; break;
    case TB_MATERN12: pre2 = LOG2E * LOG2E, cq = 0.0; break;
    case TB_MATERN32: pre2 = 3.0 * LOG2E * LOG2E, cq = 0.5 * LN2 * LN2; break;
    default: pre2 = 5.0 * LOG2E * LOG2E, cq = LN2 * LN2 / 6.0; break;
  }
  const double pre = std::sqrt(pre2);
  std::vector<double> centre((size_t)DP, 0.0), half_width((size_t)DP, 0.0);
  double unc2 = 0.0;  // max_j |x_j / l|^2, uncentred (the fp64 path's own cancellation)
  for (int d = 0; d < D; ++d) {
    double lo = INFINITY, hi = -INFINITY;
    for (int64_t j = 0; j < N; ++j) lo = std::min(lo, xs[j * DP + d]), hi = std::max(hi, xs[j * DP + d]);
    centre[d] = 0.5 * (lo + hi);
    half_width[d] = 0.5 * (hi - lo);
  }
  std::vector<float> h((size_t)rows * W, 0.0f);
  double x2max = 0.0, asum = 0.0, c2 = 0.0, box2 = 0.0;  // box2: |x'|^2 at a corner of the training rows' bounding box
  for (int d = 0; d < D; ++d) {
    c2 += centre[d] * centre[d];
    const double hw = half_width[d] * pre;
    box2 += hw * hw;
  }
  for (int64_t j = 0; j < N; ++j) {
    float* r = &h[(size_t)j * W];
    double n2 = 0.0, u2 = 0.0;
    for (int d = 0; d < D; ++d) {
      r[d] = (float)((xs[j * DP + d] - centre[d]) * pre);
      n2 += (double)r[d] * (double)r[d];
      u2 += xs[j * DP + d] * xs[j * DP + d];
    }
    r[DP] = (float)n2;
    const float a = (float)(gp->variance * al[j]);
    r[DP + 1] = a;
    r[DP + 2] = std::fabs(a);
    x2max = std::max(x2max, (double)r[DP]);
    unc2 = std::max(unc2, u2);
    asum += std::fabs((double)a);
  }
  // the bound (DESIGN.md §4d): E = safety ((rel + lin * norms) S + abs)
  const double u = std::ldexp(1.0, -24), mufu = std::ldexp(1.0, -21);
  const bool expand = gp->kernel != TB_MATERN12;
  // s-proportional part (Matern): the error of sqrt(q) = q rsqrt(q) (and, for Matern12, of the difference form's q) is
  // relative, kappa s on the exp argument; split at s0: kappa (s0 S + T(s0) sum |a|), T(s0) = sup_{s >= s0} s k(s) / σ_f²
  double kappa = 0.0, s0 = 0.0, tail = 0.0;
  if (gp->kernel != TB_RBF) {
    kappa = 1.01 * (mufu + u + (expand ? 0.0 : (2 * DP + 2) * u / 2));
    auto T = [&](double s) {
      const double p = gp->kernel == TB_MATERN12 ? 1.0 : gp->kernel == TB_MATERN32 ? 1.0 + s : 1.0 + s + s * s / 3.0;
      return s * p * std::exp(-s);  // decreasing for s >= 4 in all three
    };
    double best = INFINITY;
    for (double s = 4.0; s <= 48.0; s += 1.0) {
      const double cost = s * 0.01 * asum + T(s) * asum;  // against a typical S of 1 % of sum |a|
      if (cost < best) best = cost, s0 = s;
    }
    tail = T(s0);
  }
  double rel = mufu + 4 * u                                 // ex2, polynomial, product, rounding of a
               + 32 * u / (1 - 32 * u)                      // fp32 partial sums of KH = 32 terms
               + kappa * s0                                 // s-proportional part up to s0
               + (double)(N + 64) * std::ldexp(1.0, -52)    // the fp64 path's own kernel values and sum, the fp64 folds
               + 1e-15;                                     // the clamp q >= 1e-30
  const double lin_max = std::ldexp(1.0, -10);
  double lin;
  std::vector<unsigned char> tc;
  double terms = (double)rows;  // terms each candidate's sums add
  gp->pre_tc = false;
  if (expand) {
    const double l64 = cq * (2 * DP + 10) * std::ldexp(1.0, -52);  // the fp64 path's expansion form on uncentred inputs
    rel += l64 * pre2 * (c2 + unc2);
    // FFMA dot product (mean_bounds_kernel): |dq| <= (2 DP + 10) u (|x'|^2 + max n_j)
    lin = cq * (2 * DP + 10) * u + l64;
    // tensor cores (tc_mean_bounds_kernel): |dq| <= lin_q (|x'|^2 + max n_j) + abs_q
    const double rd = std::sqrt((double)DP);
    const double lin_q = (4 + 1.01 * DP + 1) * u                      // input rounding of x' and X', the fp32 |x'|^2, n_j
                         + 4.01 * std::ldexp(1.0, -22)                // dropped x_lo X_lo and the lo parts' rounding
                         + 1.01 * rd * std::ldexp(1.0, -25)           // subnormal lo parts, via |x| + |X| <= 1 + (x2 + n) / 2
                         + pre::tc_nk(DP) * 2.01 * 24 * std::ldexp(1.0, -23);  // accumulation, per k16 step
    const double abs_q = 1.01 * rd * std::ldexp(1.0, -24) + std::ldexp(1.0, -25);
    const double lin_tc = cq * lin_q + l64;
    // The tensor-core pass's distance bound is ~7x wider.  It runs only where it still trusts, with a factor 2 to spare, every
    // candidate inside the training rows' bounding box (|x'|^2 <= box2); elsewhere (short lengthscales: large pre-scaled norms)
    // the FFMA pass keeps the screen pruning.
    bool f16_ok = false;
    if (1.01 * lin_tc * (box2 + 1.01 * x2max) <= 0.5 * lin_max) {
      tc = prescreen_tc_columns(h, N, DP, W, &gp->pre_nsl, &gp->pre_npos_sl, &f16_ok);
      gp->pre_tc = f16_ok;  // the fp16 operands of every training row are finite
    }
    if (gp->pre_tc) {
      terms = 8.0 * gp->pre_nsl;
      lin = lin_tc;
      rel += cq * abs_q;
    }
  } else {
    lin = LN2 * u;  // Matern12: |dr'| <= u (|x'| + max|X'|) from the input rounding
  }
  gp->pre_rel = 1.01 * rel;
  gp->pre_lin = 1.01 * lin;
  gp->pre_lin_max = lin_max;
  gp->pre_abs = 1.01 * (asum * (2700.0 * std::ldexp(1.0, -126) + kappa * tail) + 2.0 * terms * std::ldexp(1.0, -149));
  gp->pre_scale = pre;
  gp->pre_x2max = 1.01 * x2max;
  const size_t bytes = gp->pre_tc ? tc.size() : sizeof(float) * h.size();
  TB_TRY(gp->dPreRows.reserve(bytes));
  TB_TRY(gp->dPreCentre.reserve(sizeof(double) * DP));
  TB_CUDA(cudaMemcpyAsync(gp->dPreRows.p, gp->pre_tc ? (const void*)tc.data() : (const void*)h.data(), bytes, cudaMemcpyHostToDevice, st));
  TB_CUDA(cudaMemcpyAsync(gp->dPreCentre.p, centre.data(), sizeof(double) * DP, cudaMemcpyHostToDevice, st));
  TB_CUDA(cudaStreamSynchronize(st));
  gp->pre_gen = gp->cache_gen;
  return 0;
}

static int prescreen_blocks(const tb_gp* gp, int64_t M) {
  const int DP = gp->DP;
  const int64_t per = gp->pre_tc ? pre::tc_cands(DP) : (int64_t)pre::TH * (DP <= 12 ? 4 : DP <= 20 ? 2 : 1);
  return (int)((M + per - 1) / per);
}

// the bound pass over M device candidates: acq >= 0: out0 = ub, per-CTA first-max of acq(μ̃) into blk_best / blk_idx;
// acq < 0: out0 / out1 = μ̃ -/+ E
static int launch_mean_bounds(tb_gp* gp, cudaStream_t st, const double* Xc, int64_t M, int acq, double param, double var_ub,
                              double* out0, double* out1, double* blk_best, int64_t* blk_idx) {
  TB_TRY(prescreen_ensure(gp));
  pre::Bound b;
  b.rel = gp->pre_rel;
  b.lin = gp->pre_lin;
  b.lin_max = gp->pre_lin_max;
  b.abs = gp->pre_abs;
  b.safety = 4.0;
  b.x2max = gp->pre_x2max;
  b.mean_const = gp->mean_const;
  b.pre = gp->pre_scale;
  const int D = gp->D;
  const double* il = gp->dInvLs.as<double>();
  const double* cen = gp->dPreCentre.as<double>();
  const unsigned blocks = (unsigned)prescreen_blocks(gp, M);
  with_kind_dp(gp->kernel, gp->DP, [&](auto K, auto P) {
    constexpr int KIND = decltype(K)::value, DP = decltype(P)::value;
    if (!gp->pre_tc) {
      const int nst = (int)((gp->N + pre::KS - 1) / pre::KS);
      pre::mean_bounds_kernel<KIND, DP><<<blocks, pre::TH, 0, st>>>(gp->dPreRows.as<float>(), nst, Xc, il, cen, D, M, b, acq, param,
                                                                    var_ub, out0, out1, blk_best, blk_idx);
    } else if constexpr (KIND != TB_MATERN12) {
      pre::tc_mean_bounds_kernel<KIND, DP><<<blocks, pre::TH, 0, st>>>(gp->dPreRows.as<unsigned char>(), gp->pre_nsl, gp->pre_npos_sl,
                                                                       Xc, il, cen, D, M, b, acq, param, var_ub, out0, out1, blk_best,
                                                                       blk_idx);
    }
  });
  TB_LAUNCHED();
  TB_CUDA(cudaGetLastError());
  return 0;
}

// =================================================================================================
// GEMM engines of the candidate path.  select_engine decides which one a call runs; the operations below hold each
// engine's launches.
// =================================================================================================
enum class Engine {
  F64,   // native fp64 DMMA kernels (kernels_f64.cuh)
  INT8,  // int8 digit engine (ozaki5.cuh, int8_engines.cu): 15 or 21 digit products on fp64 handles, 6, 10 or 15 on fp32 ones
};

// The engine of a call, after the lazy builds it needs.  need_v: the call also needs V = K^-1 K* (gradients).  The int8
// engine's int32 accumulators are exact up to K = N = 16384; larger models and engine 0 run the fp64 kernels.  The int8
// engine's digit count (gp->digits.S) comes from its a-priori error estimates (int8_select).
static int select_engine(tb_gp* gp, bool need_v, Engine* eng) {
  if (!(gp->engine == 1 && gp->N <= 16384)) {
    if (need_v) TB_TRY(ensure_upper_panels(gp));
    *eng = Engine::F64;
    return 0;
  }
  if (need_v) TB_TRY(ensure_kinv_dense(gp));
  TB_TRY(int8_select(gp, need_v));
  *eng = Engine::INT8;
  return 0;
}

// candidates per K* tile, and the K* scratch bytes per tile
static int eng_tile_width(const tb_gp* gp, Engine e) { return e == Engine::F64 ? BT : int8_tile_width(gp); }
static size_t eng_tile_bytes(const tb_gp* gp, Engine e) {
  return e == Engine::F64 ? (size_t)gp->nkc * PANEL * sizeof(double) : int8_tile_bytes(gp);
}

// Row-block groups per candidate tile of the Linv GEMMs.  int8 engine: ~4 row-blocks per CTA amortise the CTA prologue
// while the co-resident CTAs share few enough candidate tiles for the K* digits to stay in L2; small batches get more
// groups (>= 2 items per SM).  fp64 engine: one group from a full wave of tiles on.
static int eng_groups(const tb_gp* gp, Engine e, int tiles) {
  const int fill = (2 * NUM_SMS + tiles - 1) / tiles;
  if (e == Engine::F64) return tiles >= NUM_SMS ? 1 : std::max(1, std::min(fill, gp->NB));
  return std::max(std::max(1, (gp->NB + 3) / 4), std::min(gp->NB, fill));
}

// K* of mc device candidates into gp->sKs (fp64 panels or digit tiles), their posterior means into gp->sMean.
// split: the int8 engine's k-split (nullptr: the one int8_kstar_split gives for this many tiles); wide: int8_kstar's
static int eng_kstar(tb_gp* gp, Engine e, const double* xc, int64_t mc, int tiles, const KSplit* split = nullptr, bool wide = false) {
  double* mean = gp->sMean.as<double>();
  if (e == Engine::F64) return launch_kstar(gp, xc, mc, tiles, gp->sKs.as<double>(), mean);
  return int8_kstar(gp, xc, mc, tiles, gp->sKs.as<int8_t>(), mean, split, wide);
}

// Variance GEMM: sums of squares of A = Linv K* over G row-block groups into gp->sPartial.  fp64 engine with packed_a: A
// also goes to gp->sA as packed panels, the operand of its V GEMM.  kper > 0 (int8 engine): split-K (int8_split_kper).
static int eng_variance(tb_gp* gp, Engine e, int tiles, int G, int64_t McPad, bool packed_a, int kper = 0) {
  cudaStream_t st = gp->stream;
  double* partial = gp->sPartial.as<double>();
  if (e != Engine::F64) return int8_variance(gp, gp->sKs.as<int8_t>(), tiles, G, McPad, partial, kper);
  if (packed_a)
    trigemm_kernel<false, EPI_SUMSQ_PACKED><<<dim3(tiles, G), TG_THREADS, TG_SMEM, st>>>(
        gp->dLinvP.as<double>(), gp->sKs.as<double>(), gp->NB, gp->nkc, G, McPad, partial, gp->sA.as<double>(), nullptr, 0);
  else
    trigemm_kernel<false, EPI_SUMSQ><<<dim3(tiles, G), TG_THREADS, TG_SMEM, st>>>(
        gp->dLinvP.as<double>(), gp->sKs.as<double>(), gp->NB, gp->nkc, G, McPad, partial, nullptr, nullptr, 0);
  TB_LAUNCHED();
  TB_CUDA(cudaGetLastError());
  return 0;
}

// A = Linv K* stored plain into out ([candidate][NB*128])
static int eng_store_a(tb_gp* gp, Engine e, int tiles, int64_t McPad, double* out) {
  const int64_t lda = (int64_t)gp->NB * BM;
  const int G = eng_groups(gp, e, tiles);
  if (e != Engine::F64) return int8_store(gp, false, gp->sKs.as<int8_t>(), tiles, G, McPad, out, lda);
  trigemm_kernel<false, EPI_PLAIN><<<dim3(tiles, G), TG_THREADS, TG_SMEM, gp->stream>>>(gp->dLinvP.as<double>(), gp->sKs.as<double>(),
                                                                                        gp->NB, gp->nkc, G, McPad, nullptr, nullptr, out, lda);
  TB_LAUNCHED();
  TB_CUDA(cudaGetLastError());
  return 0;
}

// V = K^-1 K* stored plain into gp->sV ([candidate][NB*128]).  fp64 engine: Linv^T A over the packed A that eng_variance left
// in gp->sA; int8 engine: the digit tiles of the dense K^-1 times the same K* digits.  With 6 digits the V GEMM has its own
// row-block groups: at most ~8 row-blocks each.
static int eng_store_v(tb_gp* gp, Engine e, int tiles, int64_t McPad) {
  const int64_t ldv = (int64_t)gp->NB * BM;
  double* V = gp->sV.as<double>();
  if (e == Engine::INT8) {
    const int G = gp->digits.S == 6 ? std::max(1, std::min(gp->NB, std::max((gp->NB + 7) / 8, (2 * NUM_SMS + tiles - 1) / tiles)))
                                    : eng_groups(gp, e, tiles);
    return int8_store(gp, true, gp->sKs.as<int8_t>(), tiles, G, McPad, V, ldv);
  }
  const int G = eng_groups(gp, e, tiles);
  trigemm_kernel<true, EPI_PLAIN><<<dim3(tiles, G), TG_THREADS, TG_SMEM, gp->stream>>>(gp->dLinvTP.as<double>(), gp->sA.as<double>(), gp->NB,
                                                                                       gp->NB * (BM / BK), G, McPad, nullptr, nullptr, V, ldv);
  TB_LAUNCHED();
  TB_CUDA(cudaGetLastError());
  return 0;
}

// =================================================================================================
// per-candidate driver
// =================================================================================================

// The running argmax of a call in gp->sRun (best value, then its index).  argmax_begin reserves it, and the tail's per-block
// winners of chunks of up to chunk_cap candidates, and resets it; argmax_fold folds one chunk's winners in; argmax_end reads
// the winner into rq (the caller synchronises).
static int argmax_reset(tb_gp* gp) {
  const double init_v = -INFINITY;  // a candidate worth -inf still beats "nothing seen" through the lower-index tie rule
  const int64_t init_i = INT64_MAX;
  TB_CUDA(cudaMemcpyAsync(gp->sRun.p, &init_v, 8, cudaMemcpyHostToDevice, gp->stream));
  TB_CUDA(cudaMemcpyAsync((char*)gp->sRun.p + 8, &init_i, 8, cudaMemcpyHostToDevice, gp->stream));
  return 0;
}
static int argmax_begin(tb_gp* gp, int64_t chunk_cap) {
  const int tail_blocks_cap = (int)((chunk_cap + 255) / 256);
  TB_TRY(gp->sRun.reserve(16));
  TB_TRY(gp->sBlkBest.reserve(sizeof(double) * tail_blocks_cap));
  TB_TRY(gp->sBlkIdx.reserve(sizeof(int64_t) * tail_blocks_cap));
  return argmax_reset(gp);
}
static int argmax_fold(tb_gp* gp, int64_t n) {  // the tail's per-block winners of n candidates into gp->sRun
  argmax_fold_kernel<<<1, 256, 0, gp->stream>>>(gp->sBlkBest.as<double>(), gp->sBlkIdx.as<int64_t>(), (int)((n + 255) / 256),
                                                gp->sRun.as<double>(), reinterpret_cast<int64_t*>((char*)gp->sRun.p + 8));
  TB_LAUNCHED();
  return 0;
}
static int argmax_end(tb_gp* gp, EvalRequest& rq) {
  TB_CUDA(cudaMemcpyAsync(&rq.best_value, gp->sRun.p, 8, cudaMemcpyDeviceToHost, gp->stream));
  TB_CUDA(cudaMemcpyAsync(&rq.best_index, (char*)gp->sRun.p + 8, 8, cudaMemcpyDeviceToHost, gp->stream));
  return 0;
}

// tb_gp_profile: CUDA events around each variance GEMM, accumulated into the handle's counters by profile_fold once the
// call has synchronised
template <class F>
static int profiled_gemm(tb_gp* gp, double flops, F&& launch) {
  if (!gp->profile) return launch();
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  TB_CUDA(cudaEventCreate(&e0));
  TB_CUDA(cudaEventCreate(&e1));
  TB_CUDA(cudaEventRecord(e0, gp->stream));
  TB_TRY(launch());
  TB_CUDA(cudaEventRecord(e1, gp->stream));
  gp->prof_events.emplace_back(e0, e1);
  gp->prof_event_flops.push_back(flops);
  return 0;
}
static int profile_fold(tb_gp* gp) {
  for (size_t i = 0; i < gp->prof_events.size(); ++i) {
    float ms = 0.f;
    TB_CUDA(cudaEventElapsedTime(&ms, gp->prof_events[i].first, gp->prof_events[i].second));
    gp->prof_ms += ms;
    gp->prof_flops += gp->prof_event_flops[i];
    gp->prof_launches += 1;
    cudaEventDestroy(gp->prof_events[i].first);
    cudaEventDestroy(gp->prof_events[i].second);
  }
  gp->prof_events.clear();
  gp->prof_event_flops.clear();
  return 0;
}

// where one chunk's outputs go (null: not requested)
struct EvalOut {
  double *vals = nullptr, *mean = nullptr, *var = nullptr, *grad = nullptr;
};

// One handle's share of a chunk of n device candidates at xc, on the handle's stream: K* and the means (gp->sKs, gp->sMean),
// the variance sums of squares (gp->sPartial) and, with grad, V = K^-1 K* (gp->sV).  Gfix: the call's row-block groups (0:
// eng_groups of this chunk); *G and *McPad return the groups and the candidates padded to whole tiles, the layout of
// gp->sPartial.  The screened argmax passes the k-split of the chunk its candidates come from, and spread: when they are too
// few tiles for the row-block groups to fill the SMs, the int8 engine spreads them wider (split-K variance GEMM, wide K*
// generation) with the same results.
static int member_step(tb_gp* gp, Engine e, const double* xc, int64_t n, int Gfix, bool grad, int* G, int64_t* McPad,
                       const KSplit* split = nullptr, bool spread = false) {
  const int nt = eng_tile_width(gp, e);
  const int tiles = (int)((n + nt - 1) / nt);
  *G = Gfix ? Gfix : eng_groups(gp, e, tiles);
  *McPad = (int64_t)tiles * nt;
  const int kper = spread && e != Engine::F64 ? int8_split_kper(gp, tiles, *G) : 0;
  TB_TRY(eng_kstar(gp, e, xc, n, tiles, split, kper > 0));
  TB_TRY(profiled_gemm(gp, (double)*McPad * (double)gp->N * (double)gp->N,
                       [&] { return eng_variance(gp, e, tiles, *G, *McPad, grad, kper); }));
  return grad ? eng_store_v(gp, e, tiles, *McPad) : 0;
}

// One chunk of n device candidates at xc: member_step, then with o.grad the partials d acq / d (mean, var) and the gradient
// assembly, then the acquisition tail and the argmax fold.  c0: global index of the first candidate.  The screened argmax's
// gathered candidates pass their global indices in idx_map instead, and the k-split of the chunk they come from.
static int eval_chunk(tb_gp* gp, const EvalRequest& rq, Engine e, const double* xc, int64_t n, int64_t c0, int Gfix, const EvalOut& o,
                      const int64_t* idx_map = nullptr, const KSplit* split = nullptr) {
  cudaStream_t st = gp->stream;
  const double* partial = gp->sPartial.as<double>();
  const double* mean = gp->sMean.as<double>();
  int G;
  int64_t McPad;
  TB_TRY(member_step(gp, e, xc, n, Gfix, o.grad != nullptr, &G, &McPad, split, idx_map != nullptr));
  if (o.grad) {
    TB_TRY(launch_partials(gp, st, rq.acq, rq.param, partial, G, McPad, mean, xc, n));
    TB_TRY(launch_grad(gp, xc, n, o.grad));
  }
  TB_TRY(launch_tail(gp, st, rq, partial, G, McPad, mean, n, c0, o.vals, o.mean, o.var, xc, o.grad, idx_map));
  return rq.want_argmax ? argmax_fold(gp, n) : 0;
}

// Screened argmax of EI / log-EI (argmax_screen_wanted): the variance GEMM runs only for candidates that can still win.
//   1. bound pass (prescreen.cuh): fp32 means with a rigorous error bound E -> ub = acq(μ̃ - E, var_ub) >= the exact value,
//      and the first-max of acq(μ̃, var_ub): the probe
//   2. the probe's exact value tau -> gp->sRun
//   3. compaction of the survivors (ub >= tau - margin, or ub NaN), grouped by the k-split of their unscreened chunk; the host
//      reads their counts (one synchronisation)
//   4. exact values of the survivors (eval_chunk with their chunk's k-split and the call's G), folded on their global indices
// A gathered candidate's digits, its sum of squares over G groups and its mean are what the unscreened call computes for it,
// so its value is too.  More than M / 4 survivors: *done stays false, gp->sRun is reset and the caller runs the unscreened
// chunk loop.
static int argmax_screened(tb_gp* gp, const EvalRequest& rq, Engine e, int64_t chunk_cap, int G, bool* done) {
  *done = false;
  cudaStream_t st = gp->stream;
  const int D = gp->D, nt = eng_tile_width(gp, e);
  const int64_t M = rq.M;
  const int64_t cap = std::max<int64_t>(1, M / 4);
  TB_TRY(prescreen_ensure(gp));  // it picks the bound-pass kernel, and with it the CTA count
  const int sblocks = (int)((M + 255) / 256), bblocks = prescreen_blocks(gp, M);
  TB_TRY(gp->sScrUb.reserve(sizeof(double) * (size_t)M));
  TB_TRY(gp->sScrX.reserve(sizeof(double) * (size_t)cap * D));
  TB_TRY(gp->sScrIdx.reserve(sizeof(int64_t) * (size_t)cap));
  TB_TRY(gp->sScrBlk.reserve(16 * (size_t)bblocks + 32));
  double* ub = gp->sScrUb.as<double>();
  double* xsel = gp->sScrX.as<double>();
  int64_t* isel = gp->sScrIdx.as<int64_t>();
  double* bb = gp->sScrBlk.as<double>();
  int64_t* bi = reinterpret_cast<int64_t*>(bb + bblocks);
  double* probe_v = reinterpret_cast<double*>(bi + bblocks);
  int64_t* probe_i = reinterpret_cast<int64_t*>(probe_v + 1);
  unsigned long long* count = reinterpret_cast<unsigned long long*>(probe_v + 2);
  // the unscreened loop's chunks: whole ones over [0, split), the last over [split, M); only the last can have another k-split
  const int64_t split = ((M - 1) / chunk_cap) * chunk_cap;
  const KSplit ks_full = int8_kstar_split(gp, (int)(chunk_cap / nt)), ks_last = int8_kstar_split(gp, (int)((M - split + nt - 1) / nt));
  const bool same_split = ks_full.ksplit == ks_last.ksplit && ks_full.kc_per == ks_last.kc_per;
  // 1. bound pass
  const double var_ub = std::fmax(gp->variance, 1e-12);
  const double init_v = -INFINITY;
  const int64_t init_i = INT64_MAX;
  TB_CUDA(cudaMemcpyAsync(probe_v, &init_v, 8, cudaMemcpyHostToDevice, st));
  TB_CUDA(cudaMemcpyAsync(probe_i, &init_i, 8, cudaMemcpyHostToDevice, st));
  TB_TRY(launch_mean_bounds(gp, st, rq.Xc, M, rq.acq, rq.param, var_ub, ub, nullptr, bb, bi));
  argmax_fold_kernel<<<1, 256, 0, st>>>(bb, bi, bblocks, probe_v, probe_i);
  TB_LAUNCHED();
  // 2. probe
  pre::probe_kernel<<<1, 32, 0, st>>>(rq.Xc, D, probe_i, xsel, isel);
  TB_LAUNCHED();
  bool probe_last = true;
  if (!same_split) {  // the probe's chunk decides its k-split
    int64_t p = 0;
    TB_CUDA(cudaMemcpyAsync(&p, probe_i, 8, cudaMemcpyDeviceToHost, st));
    TB_CUDA(cudaStreamSynchronize(st));
    probe_last = (p == INT64_MAX ? 0 : p) >= split;
  }
  const EvalOut none;
  TB_TRY(eval_chunk(gp, rq, e, xsel, 1, 0, G, none, isel, probe_last ? &ks_last : &ks_full));
  // 3. compaction
  TB_CUDA(cudaMemsetAsync(count, 0, 16, st));
  pre::compact_kernel<<<sblocks, 256, 0, st>>>(rq.Xc, ub, M, split, D, var_ub, rq.acq, gp->sRun.as<double>(), cap, count, xsel, isel);
  TB_LAUNCHED();
  unsigned long long n[2] = {0, 0};
  TB_CUDA(cudaMemcpyAsync(n, count, 16, cudaMemcpyDeviceToHost, st));
  TB_CUDA(cudaStreamSynchronize(st));
  TB_CUDA(cudaGetLastError());
  if (n[0] + n[1] > (unsigned long long)cap) return argmax_reset(gp);
  // 4. exact evaluation of the survivors: whole-chunk ones in slots [0, n0), last-chunk ones in [cap - n1, cap)
  const int64_t nf = (int64_t)n[0], nb = (int64_t)n[1];
  for (int64_t s0 = 0; s0 < nf; s0 += chunk_cap)
    TB_TRY(eval_chunk(gp, rq, e, xsel + s0 * D, std::min<int64_t>(chunk_cap, nf - s0), 0, G, none, isel + s0, &ks_full));
  for (int64_t s0 = cap - nb; s0 < cap; s0 += chunk_cap)
    TB_TRY(eval_chunk(gp, rq, e, xsel + s0 * D, std::min<int64_t>(chunk_cap, cap - s0), 0, G, none, isel + s0, &ks_last));
  *done = true;
  return 0;
}

// Chunk geometry of a call over the n handles gps with engines eng (one for run_eval, the members for ehvi_run): candidates
// per chunk (chunk_cap, the smallest of the handles' own) and each handle's row-block groups G[l], fixed for the call when
// G[l] > 0, else eng_groups of each chunk.  The screened argmax and the k-split of the int8 engine reproduce these
// chunks, so they must not drift; with one handle chunk_cap is a whole number of its tiles.  A handle's own chunk size:
//   int8 engine, values: K* digit scratch within 1,280 MB, whole pairs of waves (or one wave), at most 8 waves; G of the
//                        first chunk for the whole call
//   int8 engine, gradients below 6 digits: K* digits or V (NB*128 doubles per candidate), whichever is larger, within
//                        1,280 MB, whole waves
//   fp64 engine, and the int8 engine's gradients at 6 digits: chunk_tiles
// A handle whose own chunk size is the common one therefore sums each candidate's variance exactly as its tb_gp_predict does;
// the others agree with it to rounding.
struct ChunkPlan {
  int64_t chunk_cap = 0;
  int G[MEMBERS_MAX] = {};
};
static ChunkPlan plan_chunks(tb_gp* const* gps, const Engine* eng, int n, bool grad, int64_t M) {
  ChunkPlan p;
  const size_t budget = (size_t)1280 << 20;
  for (int l = 0; l < n; ++l) {
    const tb_gp* gp = gps[l];
    const Engine e = eng[l];
    const int nt = eng_tile_width(gp, e);
    int64_t max_tiles;
    if (e != Engine::F64 && !grad) {
      max_tiles = std::max<int64_t>(1, (int64_t)(budget / eng_tile_bytes(gp, e)));
      if (max_tiles >= 2 * NUM_SMS) max_tiles = (max_tiles / (2 * NUM_SMS)) * (2 * NUM_SMS);
      else if (max_tiles >= NUM_SMS) max_tiles = NUM_SMS;
      max_tiles = std::min<int64_t>(max_tiles, 8 * NUM_SMS);
    } else if (e == Engine::INT8 && gp->digits.S != 6) {
      const size_t v_bytes = (size_t)nt * gp->NB * BM * sizeof(double);
      max_tiles = std::max<int64_t>(1, (int64_t)(budget / std::max(eng_tile_bytes(gp, e), v_bytes)));
      if (max_tiles >= NUM_SMS) max_tiles = (max_tiles / NUM_SMS) * NUM_SMS;
    } else {
      max_tiles = chunk_tiles(gp);
    }
    const int64_t cap = std::min<int64_t>(max_tiles * nt, ((M + nt - 1) / nt) * nt);
    p.chunk_cap = l == 0 ? cap : std::min(p.chunk_cap, cap);
  }
  for (int l = 0; l < n; ++l) {
    const int nt = eng_tile_width(gps[l], eng[l]);
    if (eng[l] != Engine::F64 && !grad) p.G[l] = eng_groups(gps[l], eng[l], (int)((p.chunk_cap + nt - 1) / nt));
  }
  return p;
}

// One handle's chunk scratch for chunks of up to chunk_cap candidates (padded to its tiles) on engine e: K*, the variance sums
// of squares over G row-block groups (0: per chunk, at most NB), the means and, with grad, the packed A (fp64 engine), V and
// d acq / d (mean, var)
static int reserve_chunk(tb_gp* gp, Engine e, bool grad, int64_t chunk_cap, int G) {
  const int nt = eng_tile_width(gp, e);
  const int64_t tiles_cap = (chunk_cap + nt - 1) / nt, pad_cap = tiles_cap * nt;
  TB_TRY(gp->sKs.reserve((size_t)tiles_cap * eng_tile_bytes(gp, e)));
  TB_TRY(gp->sPartial.reserve(sizeof(double) * (size_t)(G ? G : gp->NB) * pad_cap));
  TB_TRY(gp->sMean.reserve(sizeof(double) * pad_cap));
  if (grad) {
    if (e == Engine::F64) TB_TRY(gp->sA.reserve((size_t)tiles_cap * gp->NB * (BM / BK) * PANEL * sizeof(double)));  // packed A
    TB_TRY(gp->sV.reserve((size_t)pad_cap * gp->NB * BM * sizeof(double)));
    TB_TRY(gp->sMisc.reserve(sizeof(double) * 2 * pad_cap));
  }
  return 0;
}

// the argument checks of run_eval, made before anything is staged
static int check_eval(const tb_gp* gp, const EvalRequest& rq) {
  TB_CHECK(gp->cache_valid, "posterior cache is not built: call tb_gp_update_posterior_cache first");
  TB_CHECK(rq.M >= 0, "negative candidate count");
  if (rq.want_argmax) TB_CHECK(rq.M > 0, "argmax over an empty candidate set");
  return 0;
}

// The driver behind predict, acquisition values and gradients and the fused argmax: the candidates in chunks (plan_chunks),
// each through eval_chunk, all on the handle's stream, host arrays staged as Staged describes.
static int run_eval(tb_gp* gp, EvalRequest& rq) {
  TB_CUDA(cudaSetDevice(gp->device));
  cudaStream_t st = gp->stream;
  const int D = gp->D;
  const bool grad = rq.out_grad != nullptr;
  if (rq.M == 0) return 0;
  if (grad) TB_CHECK(rq.acq >= 0, "gradients need an acquisition kind");
  Engine e;
  TB_TRY(select_engine(gp, grad, &e));
  const ChunkPlan cp = plan_chunks(&gp, &e, 1, grad, rq.M);
  const int64_t chunk_cap = cp.chunk_cap;
  // a host out_mean is copied from gp->sMean, which the K* step fills anyway
  const Staged<const double> xin(rq.Xc, D, gp->sXc, st);
  const Staged<double> vals(rq.out_vals, 1, gp->sVals, st), mean(rq.out_mean, 1, gp->sMean, st), var(rq.out_var, 1, gp->sVar, st),
      grads(rq.out_grad, D, gp->sGrad, st);
  TB_TRY(reserve_chunk(gp, e, grad, chunk_cap, cp.G[0]));
  TB_TRY(xin.reserve(chunk_cap));
  TB_TRY(vals.reserve(chunk_cap));
  TB_TRY(var.reserve(chunk_cap));
  TB_TRY(grads.reserve(chunk_cap));
  if (rq.want_argmax) TB_TRY(argmax_begin(gp, chunk_cap));

  bool screened = false;
  if (e != Engine::F64 && argmax_screen_wanted(rq, xin.dev)) TB_TRY(argmax_screened(gp, rq, e, chunk_cap, cp.G[0], &screened));
  const int64_t m_loop = screened ? 0 : rq.M;  // the screened path has folded its survivors into gp->sRun already
  for (int64_t c0 = 0; c0 < m_loop; c0 += chunk_cap) {
    const int64_t mc = std::min<int64_t>(chunk_cap, rq.M - c0);
    const double* xc;
    TB_TRY(xin.in(c0, mc, &xc));
    EvalOut o;
    o.vals = vals.out(c0);
    o.mean = mean.host() ? nullptr : mean.out(c0);
    o.var = var.out(c0);
    o.grad = grads.out(c0);
    TB_TRY(eval_chunk(gp, rq, e, xc, mc, c0, cp.G[0], o));
    TB_TRY(grads.back(c0, mc));
    TB_TRY(vals.back(c0, mc));
    TB_TRY(mean.back(c0, mc));
    TB_TRY(var.back(c0, mc));
  }
  if (rq.want_argmax) TB_TRY(argmax_end(gp, rq));
  if (!rq.sync) return 0;  // the caller synchronises, then folds the profile
  TB_CUDA(cudaStreamSynchronize(st));
  TB_CUDA(cudaGetLastError());
  return profile_fold(gp);
}

// posterior mean and its gradient (no variance, no GEMM, no K^-1): one mean_grad_kernel launch per 65,536 points
static int run_mean_grad(tb_gp* gp, const double* Xc, int64_t M, double* mean, double* grad) {
  if (M == 0) return 0;
  TB_CUDA(cudaSetDevice(gp->device));
  cudaStream_t st = gp->stream;
  const int D = gp->D;
  constexpr int64_t CHUNK = 65536;
  const int64_t cap = std::min(M, CHUNK);
  const Staged<const double> xin(Xc, D, gp->sXc, st);
  const Staged<double> means(mean, 1, gp->sMean, st), grads(grad, D, gp->sGrad, st);
  TB_TRY(xin.reserve(cap));
  TB_TRY(means.reserve(cap));
  TB_TRY(grads.reserve(cap));
  const double* Xs = gp->dXs.as<double>();
  const double* al = gp->dAlpha.as<double>();
  const double* il = gp->dInvLs.as<double>();
  for (int64_t c0 = 0; c0 < M; c0 += CHUNK) {
    const int64_t mc = std::min(CHUNK, M - c0);
    const double* xc;
    TB_TRY(xin.in(c0, mc, &xc));
    double* md = means.out(c0);
    double* gd = grads.out(c0);
    const unsigned blocks = (unsigned)((mc + 7) / 8);
    with_kind_dp(gp->kernel, gp->DP, [&](auto K, auto P) {
      mean_grad_kernel<decltype(K)::value, decltype(P)::value><<<blocks, 256, 0, st>>>(Xs, al, xc, il, (int)gp->N, D, mc, gp->variance,
                                                                                       gp->mean_const, md, gd);
    });
    TB_LAUNCHED();
    TB_CUDA(cudaGetLastError());
    TB_TRY(means.back(c0, mc));
    TB_TRY(grads.back(c0, mc));
  }
  TB_CUDA(cudaStreamSynchronize(st));
  TB_CUDA(cudaGetLastError());
  return 0;
}

// GIBBON repulsion state derived from the pending points and the current posterior cache (gibbon_cross_kernel):
//   Kxp = k(X, P), Y = Linv Kxp, W = Linv^T Y = K^-1 k(X, P), B = k(P, P) - Y^T Y with its diagonal clipped at >= 1e-12
//   (predict_joint, interface.py:126-133), L_B = chol(B + noise I) and L_B^-1 on the host (m x m), What = W L_B^-T.
// Rebuilt only when the cache generation moved since the last build: O(N^2 m) once per pending set and posterior.
static int ensure_gibbon(tb_gp* gp) {
  TB_CHECK(gp->cache_valid, "GIBBON repulsion: posterior cache is not built: call tb_gp_update_posterior_cache first");
  if (gp->gib_gen == gp->cache_gen) return 0;
  TB_CUDA(cudaSetDevice(gp->device));
  cudaStream_t st = gp->stream;
  const int m = gp->gibM, D = gp->D, DP = gp->DP;
  const int mp = ((m + GIB_TILE - 1) / GIB_TILE) * GIB_TILE;
  const int N = (int)gp->N;
  std::vector<double> ps((size_t)m * DP, 0.0);
  for (int j = 0; j < m; ++j)
    for (int d = 0; d < D; ++d) ps[(size_t)j * DP + d] = gp->gibP[(size_t)j * D + d] / gp->ls[d];
  TB_TRY(gp->dGibPs.reserve(sizeof(double) * ps.size()));
  TB_CUDA(cudaMemcpyAsync(gp->dGibPs.p, ps.data(), sizeof(double) * ps.size(), cudaMemcpyHostToDevice, st));
  tb::DevBuf work;  // Kxp, Y, W [m][N] and B [m][m]
  TB_TRY(work.reserve(sizeof(double) * (3 * (size_t)m * N + (size_t)m * m)));
  double* Kxp = work.as<double>();
  double* Y = Kxp + (size_t)m * N;
  double* W = Y + (size_t)m * N;
  double* B = W + (size_t)m * N;
  const double* Xs = gp->dXs.as<double>();
  const double* Psd = gp->dGibPs.as<double>();
  const double* Linv = gp->dLinv.as<double>();
  const dim3 cols((unsigned)((N + 127) / 128), (unsigned)m);
  with_kind(gp->kernel, [&](auto K) { gibbon_kxp_kernel<decltype(K)::value><<<cols, 128, 0, st>>>(Xs, Psd, N, DP, gp->variance, Kxp); });
  TB_LAUNCHED();
  trmv_lower_cols_kernel<<<cols, 128, 0, st>>>(Linv, N, N, Kxp, N, Y, N);
  TB_LAUNCHED();
  trmv_lower_t_cols_kernel<<<dim3((unsigned)((N + 7) / 8), (unsigned)m), 256, 0, st>>>(Linv, N, N, Y, N, W, N);
  TB_LAUNCHED();
  const dim3 pairs((unsigned)m, (unsigned)m);
  with_kind(gp->kernel, [&](auto K) { gibbon_pcov_kernel<decltype(K)::value><<<pairs, 256, 0, st>>>(Psd, Y, N, DP, m, gp->variance, B); });
  TB_LAUNCHED();
  std::vector<double> b((size_t)m * m);
  TB_CUDA(cudaMemcpyAsync(b.data(), B, sizeof(double) * b.size(), cudaMemcpyDeviceToHost, st));
  TB_CUDA(cudaStreamSynchronize(st));
  TB_CUDA(cudaGetLastError());
  // L_B = chol(B + noise I) (lower, in place) and its inverse, rows padded to mp with zeros
  for (int i = 0; i < m; ++i) b[(size_t)i * m + i] = std::max(b[(size_t)i * m + i], 1e-12) + gp->noise;
  for (int j = 0; j < m; ++j) {
    double djj = b[(size_t)j * m + j];
    for (int k = 0; k < j; ++k) djj -= b[(size_t)j * m + k] * b[(size_t)j * m + k];
    TB_CHECK_CODE(djj > 0.0 && std::isfinite(djj),
                  "GIBBON repulsion: Cholesky decomposition of the pending points' covariance plus noise was not successful "
                  "(not positive definite at leading minor " + std::to_string(j + 1) + ")", tb::ERR_NUMERIC);
    const double ljj = std::sqrt(djj);
    b[(size_t)j * m + j] = ljj;
    for (int i = j + 1; i < m; ++i) {
      double v = b[(size_t)i * m + j];
      for (int k = 0; k < j; ++k) v -= b[(size_t)i * m + k] * b[(size_t)j * m + k];
      b[(size_t)i * m + j] = v / ljj;
    }
  }
  std::vector<double> li((size_t)mp * m, 0.0);
  for (int c = 0; c < m; ++c) {  // column c of L^-1 by forward substitution
    li[(size_t)c * m + c] = 1.0 / b[(size_t)c * m + c];
    for (int i = c + 1; i < m; ++i) {
      double v = 0.0;
      for (int k = c; k < i; ++k) v -= b[(size_t)i * m + k] * li[(size_t)k * m + c];
      li[(size_t)i * m + c] = v / b[(size_t)i * m + i];
    }
  }
  TB_TRY(gp->dGibLinv.reserve(sizeof(double) * li.size()));
  TB_CUDA(cudaMemcpyAsync(gp->dGibLinv.p, li.data(), sizeof(double) * li.size(), cudaMemcpyHostToDevice, st));
  TB_TRY(gp->dGibWhat.reserve(sizeof(double) * (size_t)N * mp));
  gibbon_what_kernel<<<dim3((unsigned)((N + 127) / 128), (unsigned)mp), 128, 0, st>>>(W, gp->dGibLinv.as<double>(), N, m, mp,
                                                                                    gp->dGibWhat.as<double>());
  TB_LAUNCHED();
  TB_CUDA(cudaStreamSynchronize(st));  // the host vectors and the work buffer go out of scope
  TB_CUDA(cudaGetLastError());
  gp->gibMp = mp;
  gp->gib_gen = gp->cache_gen;
  return 0;
}

}  // namespace tb

extern "C" {

int tb_gp_predict(tb_gp* gp, const void* Xc, int64_t M, void* mean, void* var) {
  TB_CHECK(gp && (M == 0 || (Xc && mean && var)), "tb_gp_predict: null argument");
  tb::EvalRequest rq;
  rq.M = M;
  TB_TRY(tb::check_eval(gp, rq));
  tb::DtypeBridge br(gp);
  TB_TRY(br.in(Xc, M * gp->D, &rq.Xc));
  TB_TRY(br.out(mean, M, &rq.out_mean));
  TB_TRY(br.out(var, M, &rq.out_var));
  TB_TRY(tb::run_eval(gp, rq));
  return br.finish();
}

int tb_gp_mean_gradient(tb_gp* gp, const void* Xc, int64_t M, void* mean, void* grad) {
  TB_CHECK(gp && (M == 0 || (Xc && mean && grad)), "tb_gp_mean_gradient: null argument");
  TB_CHECK(gp->cache_valid, "posterior cache is not built: call tb_gp_update_posterior_cache first");
  TB_CHECK(M >= 0, "negative point count");
  tb::DtypeBridge br(gp);
  const double* xd;
  double *md, *gd;
  TB_TRY(br.in(Xc, M * gp->D, &xd));
  TB_TRY(br.out(mean, M, &md));
  TB_TRY(br.out(grad, M * gp->D, &gd));
  TB_TRY(tb::run_mean_grad(gp, xd, M, md, gd));
  return br.finish();
}

// The acquisition arguments of tb_acq_eval, tb_acq_argmax and tb_acq_maximize, and the handle state their kind reads (the
// local penalty, min-value samples, GIBBON's pending points, whose derived state is brought up to date with the posterior
// cache here).  TB_ACQ_PENALIZED is stripped from acq into pen: every kernel and check below sees the plain kind.
static int check_acq(tb_gp* gp, int& acq, double param, bool& pen, const char* who) {
  pen = (acq & TB_ACQ_PENALIZED) != 0;
  acq &= ~TB_ACQ_PENALIZED;
  TB_CHECK(acq >= TB_ACQ_EI && acq <= TB_ACQ_PREDICTIVE_VARIANCE, std::string(who) + ": unknown acquisition kind");
  TB_CHECK(!(pen && gibbon_kind(acq)),
           std::string(who) + ": the GIBBON kinds do not compose with TB_ACQ_PENALIZED (the repulsion term is their batch term)");
  if (pen)
    TB_CHECK(gp->penP > 0 && gp->penD == gp->D,
             std::string(who) + ": a penalised acquisition needs the local penalty first (tb_acq_set_penalization)");
  if (acq == TB_ACQ_LCB || acq == TB_ACQ_NEG_LCB)
    TB_CHECK(param >= 0.0, "Standard deviation scaling parameter beta must not be negative");
  if (acq == TB_ACQ_MES) TB_CHECK(gp->mesS > 0, "min-value entropy search: set the min-value samples first (tb_acq_set_min_value_samples)");
  if (feasibility_kind(acq))
    TB_CHECK(gp->feasAlpha > 0.0, std::string(who) + ": the feasibility criteria need alpha first (tb_acq_set_feasibility)");
  if (acq == TB_ACQ_BALD) TB_CHECK(param > 0.0, "Jitter must be positive.");
  if (!gibbon_kind(acq)) return 0;
  if (acq != TB_ACQ_GIBBON_REPULSION)
    TB_CHECK(gp->mesS > 0, std::string(who) + ": GIBBON's quality term needs the min-value samples first (tb_acq_set_min_value_samples)");
  if (acq != TB_ACQ_GIBBON_QUALITY) {
    TB_CHECK(gp->gibM > 0 && gp->gibD == gp->D,
             std::string(who) + ": GIBBON's repulsion term needs the pending points first (tb_acq_set_gibbon_repulsion)");
    TB_TRY(tb::ensure_gibbon(gp));
  }
  return 0;
}

// The winner of an argmax as the ABI returns it, best_value in the handle's dtype.  Every value NaN: index 0 and value NaN,
// as tf.math.argmax still returns a valid index (optimizer.py:149).
static void argmax_result(const tb::EvalRequest& rq, int dtype, void* best_value, int64_t* best_index) {
  const bool none = rq.best_index == INT64_MAX;
  const double v = none ? std::nan("") : rq.best_value;
  if (dtype == TB_F32) *(float*)best_value = (float)v;
  else *(double*)best_value = v;
  *best_index = none ? 0 : rq.best_index;
}

// tb_acq_eval, and tb_acq_argmax when best_index is set
static int acq_call(tb_gp* gp, int acq, double param, const void* Xc, int64_t M, void* out, void* grad, void* best_value,
                    int64_t* best_index, const char* who) {
  tb::EvalRequest rq;
  TB_TRY(check_acq(gp, acq, param, rq.pen, who));
  rq.acq = acq;
  rq.param = param;
  rq.M = M;
  rq.want_argmax = best_index != nullptr;
  TB_TRY(tb::check_eval(gp, rq));
  tb::DtypeBridge br(gp);
  TB_TRY(br.in(Xc, M * gp->D, &rq.Xc));
  TB_TRY(br.out(out, M, &rq.out_vals));
  TB_TRY(br.out(grad, M * gp->D, &rq.out_grad));
  TB_TRY(tb::run_eval(gp, rq));
  if (best_index) argmax_result(rq, gp->dtype, best_value, best_index);
  return br.finish();
}

int tb_acq_eval(tb_gp* gp, int acq, double param, const void* Xc, int64_t M, void* out, void* grad) {
  TB_CHECK(gp && (M == 0 || (Xc && out)), "tb_acq_eval: null argument");
  return acq_call(gp, acq, param, Xc, M, out, grad, nullptr, nullptr, "tb_acq_eval");
}

int tb_acq_argmax(tb_gp* gp, int acq, double param, const void* Xc, int64_t M, void* out, void* best_value,
                  int64_t* best_index) {
  TB_CHECK(gp && Xc && best_value && best_index, "tb_acq_argmax: null argument");
  return acq_call(gp, acq, param, Xc, M, out, nullptr, best_value, best_index, "tb_acq_argmax");
}

int tb_acq_set_min_value_samples(tb_gp* gp, const double* samples, int S) {
  TB_CHECK(gp && samples, "tb_acq_set_min_value_samples: null argument");
  TB_CHECK(S > 0, "tb_acq_set_min_value_samples: need at least one sample");
  TB_CUDA(cudaSetDevice(gp->device));
  TB_TRY(gp->dMes.reserve(sizeof(double) * (size_t)S));
  TB_CUDA(cudaMemcpyAsync(gp->dMes.p, samples, sizeof(double) * (size_t)S, cudaMemcpyDefault, gp->stream));
  TB_CUDA(cudaStreamSynchronize(gp->stream));
  gp->mesS = S;
  return 0;
}

int tb_acq_set_penalization(tb_gp* gp, int kind, const double* pending, int P, const double* radius, const double* scale) {
  TB_CHECK(gp && pending && radius && scale, "tb_acq_set_penalization: null argument");
  TB_CHECK(kind == TB_PEN_SOFT || kind == TB_PEN_HARD, "tb_acq_set_penalization: kind must be 1 (soft) or 2 (hard)");
  TB_CHECK(P > 0, "tb_acq_set_penalization: need at least one pending point");
  TB_CHECK(gp->have_data, "tb_acq_set_penalization: the model has no data (input dimension unknown)");
  TB_CUDA(cudaSetDevice(gp->device));
  const size_t PD = (size_t)P * gp->D;
  TB_TRY(gp->dPen.reserve(sizeof(double) * (PD + 2 * (size_t)P)));
  double* d = gp->dPen.as<double>();
  TB_CUDA(cudaMemcpyAsync(d, pending, sizeof(double) * PD, cudaMemcpyDefault, gp->stream));
  TB_CUDA(cudaMemcpyAsync(d + PD, radius, sizeof(double) * (size_t)P, cudaMemcpyDefault, gp->stream));
  TB_CUDA(cudaMemcpyAsync(d + PD + P, scale, sizeof(double) * (size_t)P, cudaMemcpyDefault, gp->stream));
  TB_CUDA(cudaStreamSynchronize(gp->stream));
  gp->penP = P;
  gp->penKind = kind;
  gp->penD = gp->D;
  return 0;
}

int tb_acq_set_gibbon_repulsion(tb_gp* gp, const double* pending, int m, double weight) {
  TB_CHECK(gp && pending, "tb_acq_set_gibbon_repulsion: null argument");
  TB_CHECK(m > 0, "tb_acq_set_gibbon_repulsion: need at least one pending point");
  TB_CHECK(std::isfinite(weight), "tb_acq_set_gibbon_repulsion: the repulsion weight must be finite");
  TB_CHECK(gp->have_data, "tb_acq_set_gibbon_repulsion: the model has no data (input dimension unknown)");
  TB_CHECK(gp->cache_valid, "tb_acq_set_gibbon_repulsion: posterior cache is not built: call tb_gp_update_posterior_cache first");
  TB_CUDA(cudaSetDevice(gp->device));
  std::vector<double> p((size_t)m * gp->D);
  TB_CUDA(cudaMemcpy(p.data(), pending, sizeof(double) * p.size(), cudaMemcpyDefault));
  // the same pending set again (pushed before every launch): the derived state stays if the posterior did not move either
  const bool same = gp->gibM == m && gp->gibD == gp->D && gp->gibP == p;
  gp->gibW = weight;
  if (same && gp->gib_gen == gp->cache_gen) return 0;
  gp->gibP.swap(p);
  gp->gibM = m;
  gp->gibD = gp->D;
  gp->gib_gen = STALE;
  const int rc = tb::ensure_gibbon(gp);
  if (rc) gp->gibM = 0;  // a pending set that cannot be factorised is not kept
  return rc;
}

int tb_acq_set_feasibility(tb_gp* gp, double alpha) {
  TB_CHECK(gp, "tb_acq_set_feasibility: null handle");
  TB_CHECK(std::isfinite(alpha) && alpha > 0.0, "Parameter alpha must be positive.");
  gp->feasAlpha = alpha;
  return 0;
}

int tb_gp_profile(tb_gp* gp, int enable) {
  TB_CHECK(gp, "tb_gp_profile: null handle");
  gp->profile = enable != 0;
  gp->prof_ms = 0.0;
  gp->prof_flops = 0.0;
  gp->prof_launches = 0;
  return 0;
}
int tb_gp_set_engine(tb_gp* gp, int engine) {
  TB_CHECK(gp, "tb_gp_set_engine: null handle");
  TB_CHECK(engine >= 0 && engine <= 2, "tb_gp_set_engine: engine must be 0 (fp64 DMMA), 1 (int8 Ozaki) or 2 (int8, full 21 products)");
  gp->engine = engine == 0 ? 0 : 1;
  tb::int8_pin_full(gp, engine == 2);
  return 0;
}
int tb_gp_engine_info(tb_gp* gp, int* digit_products, double* error_estimate) {
  TB_CHECK(gp, "tb_gp_engine_info: null handle");
  TB_CHECK(gp->cache_valid, "tb_gp_engine_info: posterior cache is not built");
  TB_CUDA(cudaSetDevice(gp->device));
  tb::Engine e;
  TB_TRY(tb::select_engine(gp, false, &e));
  int products = 0;
  double est = 0.0;
  if (e != tb::Engine::F64) tb::int8_info(gp, &products, &est);
  if (digit_products) *digit_products = products;
  if (error_estimate) *error_estimate = est;
  return 0;
}
int tb_gp_mean_bounds(tb_gp* gp, const double* Xc, int64_t M, double* lo, double* hi) {
  TB_CHECK(gp && Xc && lo && hi, "tb_gp_mean_bounds: null argument");
  TB_CHECK(gp->cache_valid, "tb_gp_mean_bounds: posterior cache is not built");
  TB_CHECK(M >= 0, "tb_gp_mean_bounds: negative candidate count");
  if (M == 0) return 0;
  TB_CUDA(cudaSetDevice(gp->device));
  cudaStream_t st = gp->stream;
  TB_TRY(gp->sXc.reserve(sizeof(double) * (size_t)M * gp->D));
  TB_TRY(gp->sMisc.reserve(sizeof(double) * 2 * (size_t)M));
  double* x = gp->sXc.as<double>();
  double* b = gp->sMisc.as<double>();
  TB_CUDA(cudaMemcpyAsync(x, Xc, sizeof(double) * (size_t)M * gp->D, cudaMemcpyDefault, st));
  TB_TRY(tb::launch_mean_bounds(gp, st, x, M, -1, 0.0, 0.0, b, b + M, nullptr, nullptr));
  TB_CUDA(cudaMemcpyAsync(lo, b, sizeof(double) * (size_t)M, cudaMemcpyDefault, st));
  TB_CUDA(cudaMemcpyAsync(hi, b + M, sizeof(double) * (size_t)M, cudaMemcpyDefault, st));
  TB_CUDA(cudaStreamSynchronize(st));
  TB_CUDA(cudaGetLastError());
  return 0;
}
int tb_gp_kinv_apply(tb_gp* gp, const double* B, int nrhs, double* out) {
  TB_CHECK(gp && B && out, "tb_gp_kinv_apply: null argument");
  TB_CHECK(gp->cache_valid, "tb_gp_kinv_apply: posterior cache is not built");
  TB_CHECK(nrhs >= 1, "tb_gp_kinv_apply: need at least one right-hand side");
  TB_CUDA(cudaSetDevice(gp->device));
  const int64_t N = gp->N;
  cudaStream_t st = gp->stream;
  TB_TRY(gp->sMisc.reserve(sizeof(double) * 2 * N * nrhs));
  double* rhs = gp->sMisc.as<double>();
  double* tmp = rhs + N * nrhs;
  TB_CUDA(cudaMemcpyAsync(rhs, B, sizeof(double) * N * nrhs, cudaMemcpyDefault, st));
  // (K + noise I)^-1 B = Linv^T (Linv B) through the cached triangular inverse: two batched triangular mat-vecs
  // (once per trajectory, off the candidate path)
  trmv_lower_cols_kernel<<<dim3((unsigned)((N + 127) / 128), (unsigned)nrhs), 128, 0, st>>>(gp->dLinv.as<double>(), N, N, rhs, N, tmp, N);
  TB_LAUNCHED();
  trmv_lower_t_cols_kernel<<<dim3((unsigned)((N + 7) / 8), (unsigned)nrhs), 256, 0, st>>>(gp->dLinv.as<double>(), N, N, tmp, N, rhs, N);
  TB_LAUNCHED();
  TB_CUDA(cudaMemcpyAsync(out, rhs, sizeof(double) * N * nrhs, cudaMemcpyDefault, st));
  TB_CUDA(cudaStreamSynchronize(st));
  TB_CUDA(cudaGetLastError());
  return 0;
}
int tb_gp_stream(tb_gp* gp, void** stream) {
  TB_CHECK(gp && stream, "tb_gp_stream: null argument");
  *stream = (void*)gp->stream;
  return 0;
}
int tb_gp_profile_read(tb_gp* gp, double* trigemm_ms, int64_t* trigemm_launches, double* flops) {
  TB_CHECK(gp, "tb_gp_profile_read: null handle");
  if (trigemm_ms) *trigemm_ms = gp->prof_ms;
  if (trigemm_launches) *trigemm_launches = gp->prof_launches;
  if (flops) *flops = gp->prof_flops;
  return 0;
}

}  // extern "C"

// =================================================================================================
// q-batches of the joint posterior: predict_joint, reparam samples, MC-qEI and batch EI, values and gradients
// =================================================================================================
namespace tb {

// what a q-batch call makes of each batch's joint posterior (mean [q], cov [q, q])
enum class BatchTail {
  Predict,  // mean and cov
  Samples,  // mean + chol(cov + jitter I) eps, eps [q, S] normal base samples (sampler.py:277-278)
  McEi,     // batch Monte-Carlo EI (function.py:1181-1186) over eps [q, S] normal base samples
  BatchEi,  // batch EI of Chevalier & Ginsbourger (function.py:1747-1805) over the Sobol points w [q-1, S]
  PredVar,  // exp(logdet(cov + jitter 1 1^T)) of active learning's predictive variance (active_learning.py:98-108)
};

struct BatchRequest {
  BatchTail tail;
  bool grad = false;  // also d out_val / d Xc (McEi, BatchEi, PredVar)
  const double* Xc = nullptr;  // [B, q, D]
  int64_t B;
  int q;
  const double* eps = nullptr;  // host or device: eps [q, S], or w [q-1, S] for BatchEi
  int S;
  double eta, jitter;
  double* out_mean = nullptr;     // [B, q]
  double* out_cov = nullptr;      // [B, q, q]
  double* out_samples = nullptr;  // [B, S, q]
  double* out_val = nullptr;      // [B]
  double* out_grad = nullptr;     // [B, q, D]
  BatchRequest(BatchTail tail, int64_t B, int q, int S = 0, double eta = 0.0, double jitter = 0.0)
      : tail(tail), B(B), q(q), S(S), eta(eta), jitter(jitter) {}
};

// joint_kernel over nb batches of the chunk whose A = Linv K* (plain) is in A and whose means are in gp->sMean
template <int KIND>
static int launch_joint(tb_gp* gp, const BatchRequest& rq, int mode, const double* A, const double* xc, int64_t nb,
                        const double* eps_dev, double* om, double* oc, double* os, double* oq, int* err) {
  const int QT = (rq.q + 7) / 8, QP = QT * 8;
  const int blocks = (int)((nb + JOINT_WARPS - 1) / JOINT_WARPS);
  const size_t smem = (size_t)JOINT_WARPS * (QP * QP + QP * gp->D + QP) * sizeof(double);
  const int64_t lda = (int64_t)gp->NB * BM;
  const double* il = gp->dInvLs.as<double>();
#define TB_JOINT(QTV)                                                                                              \
  {                                                                                                                \
    TB_CUDA(cudaFuncSetAttribute(joint_kernel<KIND, QTV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    joint_kernel<KIND, QTV><<<blocks, JOINT_WARPS * 32, smem, gp->stream>>>(A, lda, (int)lda, gp->sMean.as<double>(), xc, il, \
        gp->D, nb, rq.q, gp->variance, mode, eps_dev, rq.S, rq.eta, rq.jitter, om, oc, os, oq, err);              \
  }
  switch (QT) {
    case 1: TB_JOINT(1); break;
    case 2: TB_JOINT(2); break;
    case 3: TB_JOINT(3); break;
    default: TB_JOINT(4); break;
  }
#undef TB_JOINT
  TB_LAUNCHED();
  TB_CUDA(cudaGetLastError());
  return 0;
}

// the argument checks of the q-batch calls other than batch EI (bei_args), made before anything is staged; sampled: the
// call takes base samples
static int check_batch(const tb_gp* gp, int64_t B, int q, bool sampled, int S, const void* eps, double jitter) {
  TB_CHECK(gp->cache_valid, "posterior cache is not built: call tb_gp_update_posterior_cache first");
  TB_CHECK(q >= 1 && q <= 32, "batch size q must be in [1, 32]");
  TB_CHECK(B >= 0, "negative batch count");
  if (sampled) {
    TB_CHECK(S >= 1 && eps, "need S >= 1 base samples");
    TB_CHECK(jitter >= 0.0, "jitter must be non-negative");
  }
  return 0;
}

static int launch_qei_cross(tb_gp* gp, const double* xc, int64_t npts, int q, const double* sbar, double* grad) {
  with_kind(gp->kernel, [&](auto K) {
    qei_cross_kernel<decltype(K)::value><<<(unsigned)((npts + 127) / 128), 128, 0, gp->stream>>>(xc, gp->dInvLs.as<double>(), gp->D, npts,
                                                                                                 q, sbar, gp->variance, grad);
  });
  TB_LAUNCHED();
  TB_CUDA(cudaGetLastError());
  return 0;
}

// Every q-batch call, chunk by chunk of whole batches: K* -> A = Linv K* (stored plain) -> with a gradient, V = K^-1 K*
// -> per-batch mean / cov (joint_kernel, which also computes the Samples tail and the McEi value) -> the other tails:
// bei_kernel for the BatchEi value, pv_kernel for the PredVar value; for a gradient the tail's reverse kernel (value, G_mu,
// Sigma_bar: qei_backward_kernel, bei_backward_kernel or pv_kernel<true>) -> per-batch mix V~ = Sigma_bar V (qei_mix_kernel)
// -> grad_kernel (the training-point sums) -> qei_cross_kernel (the K(x_b, x_b) term).
static int run_batch(tb_gp* gp, const BatchRequest& rq) {
  if (rq.B == 0) return 0;
  TB_CUDA(cudaSetDevice(gp->device));
  cudaStream_t st = gp->stream;
  const int D = gp->D, q = rq.q, S = rq.S;
  const int64_t lda = (int64_t)gp->NB * BM;
  const bool bei = rq.tail == BatchTail::BatchEi, pv = rq.tail == BatchTail::PredVar;
  const int mode = rq.tail == BatchTail::Samples ? JOINT_SAMPLE : rq.tail == BatchTail::McEi && !rq.grad ? JOINT_QEI : JOINT_PREDICT;
  const bool post_dev = bei || pv || rq.grad;  // joint_kernel leaves mean / cov in bmu / bcov for a tail kernel
  Engine e;
  TB_TRY(select_engine(gp, rq.grad, &e));
  const int nt = eng_tile_width(gp, e);  // candidates per tile
  const int64_t nbc_cap = std::min<int64_t>(std::max<int64_t>(1, (chunk_tiles(gp) * BT) / q), rq.B);  // whole batches per chunk
  const int64_t cand_cap = nbc_cap * q;
  const int64_t tiles_cap = (cand_cap + nt - 1) / nt;
  const size_t plain_bytes = (size_t)tiles_cap * nt * lda * sizeof(double);
  // A plain, joint_kernel's operand, is in gp->sA, except on the fp64 engine with a gradient: there gp->sA holds A as the
  // packed panels that the V GEMM reads, and A plain has the call's own buffer baplain
  const bool packed_a = rq.grad && e == Engine::F64;
  tb::DevBuf baplain, beps, bval, bmu, bcov, bsbar;
  TB_TRY(gp->sKs.reserve((size_t)tiles_cap * eng_tile_bytes(gp, e)));
  if (packed_a) {
    TB_TRY(gp->sA.reserve((size_t)tiles_cap * gp->NB * (BM / BK) * PANEL * sizeof(double)));
    TB_TRY(baplain.reserve(plain_bytes));
    TB_TRY(gp->sPartial.reserve(sizeof(double) * (size_t)gp->NB * tiles_cap * BT));
  } else {
    TB_TRY(gp->sA.reserve(plain_bytes));
  }
  double* A = packed_a ? baplain.as<double>() : gp->sA.as<double>();
  TB_TRY(gp->sMean.reserve(sizeof(double) * tiles_cap * nt));
  if (rq.grad) {
    TB_TRY(gp->sV.reserve(plain_bytes));                        // V plain
    TB_TRY(gp->sMisc.reserve(sizeof(double) * 2 * cand_cap));  // c_mu, c_var
    TB_TRY(bsbar.reserve(sizeof(double) * (size_t)nbc_cap * q * q));
  }
  if (post_dev) {
    TB_TRY(bmu.reserve(sizeof(double) * (size_t)cand_cap));
    TB_TRY(bcov.reserve(sizeof(double) * (size_t)nbc_cap * q * q));
  }
  // with a gradient, gp->sMisc holds c_mu / c_var: the base samples and the values of host arrays go to the call's own buffers
  const Staged<const double> xin(rq.Xc, (int64_t)q * D, gp->sXc, st);
  const Staged<const double> eps(rq.eps, (int64_t)(bei ? q - 1 : q) * S, rq.grad ? beps : gp->sMisc, st);
  const Staged<double> mean(rq.out_mean, q, gp->sVals, st), cov(rq.out_cov, (int64_t)q * q, gp->sVar, st);
  const Staged<double> samples(rq.out_samples, (int64_t)S * q, gp->sGrad, st), grad(rq.out_grad, (int64_t)q * D, gp->sGrad, st);
  const Staged<double> val(rq.out_val, 1, rq.grad ? bval : gp->sBlkBest, st);
  const Staged<double>* outs[] = {&mean, &cov, &samples, &val, &grad};
  TB_TRY(xin.reserve(nbc_cap));
  for (auto* o : outs) TB_TRY(o->reserve(nbc_cap));
  const double* eps_dev;  // null for Predict
  TB_TRY(eps.reserve(1));
  TB_TRY(eps.in(0, 1, &eps_dev));
  TB_TRY(gp->sRun.reserve(16));
  int* err = reinterpret_cast<int*>(gp->sRun.p);
  TB_CUDA(cudaMemsetAsync(err, 0, sizeof(int), st));
  // shared memory of the tail kernel, and warps per CTA of the batch EI kernels
  int bei_warps = 0;
  size_t tail_smem = 0;
  if (bei) {
    // as many warps (up to 4) as fit: one per unit CDF in flight, each with its per-sample state in shared memory
    const size_t cta = bei_cta_doubles(q) * sizeof(double);
    const size_t per_warp = (rq.grad ? bei_back_warp_doubles(q) : bei_warp_doubles(q)) * sizeof(double);
    bei_warps = (int)std::min<size_t>(std::min<size_t>(BEI_MAX_WARPS, q + q * q), (227 * 1024 - cta) / per_warp);
    tail_smem = cta + bei_warps * per_warp;
    if (rq.grad)
      TB_CUDA(cudaFuncSetAttribute(bei_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tail_smem));
    else
      TB_CUDA(cudaFuncSetAttribute(bei_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tail_smem));
  } else if (pv) {
    tail_smem = (size_t)PV_WARPS * pv_warp_doubles(q, rq.grad) * sizeof(double);
    if (rq.grad)
      TB_CUDA(cudaFuncSetAttribute(pv_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tail_smem));
    else
      TB_CUDA(cudaFuncSetAttribute(pv_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tail_smem));
  } else if (rq.grad) {
    tail_smem = (size_t)QEIG_WARPS * (3 * q * q + 2 * q) * sizeof(double);
    TB_CUDA(cudaFuncSetAttribute(qei_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tail_smem));
  }

  for (int64_t b0 = 0; b0 < rq.B; b0 += nbc_cap) {
    const int64_t nbc = std::min<int64_t>(nbc_cap, rq.B - b0);
    const int64_t mc = nbc * q;
    const int tiles = (int)((mc + nt - 1) / nt);
    const int64_t McPad = (int64_t)tiles * nt;
    const double* xc;
    TB_TRY(xin.in(b0, nbc, &xc));
    TB_TRY(eng_kstar(gp, e, xc, mc, tiles));
    TB_TRY(eng_store_a(gp, e, tiles, McPad, A));
    if (rq.grad) {
      if (packed_a) TB_TRY(eng_variance(gp, e, tiles, eng_groups(gp, e, tiles), McPad, true));
      TB_TRY(eng_store_v(gp, e, tiles, McPad));
    }
    double* mu = post_dev ? bmu.as<double>() : mean.out(b0);
    double* cv = post_dev ? bcov.as<double>() : cov.out(b0);
    double* dval = val.out(b0);
    TB_TRY(with_kind(gp->kernel, [&](auto K) {
      return launch_joint<decltype(K)::value>(gp, rq, mode, A, xc, nbc, eps_dev, mu, cv, samples.out(b0), post_dev ? nullptr : dval,
                                              err);
    }));
    if (bei && !rq.grad) {
      bei_kernel<<<(unsigned)nbc, bei_warps * 32, tail_smem, st>>>(mu, cv, q, eps_dev, S, rq.eta, dval, err);
      TB_LAUNCHED();
      TB_CUDA(cudaGetLastError());
    }
    if (pv) {
      const unsigned blocks = (unsigned)((nbc + PV_WARPS - 1) / PV_WARPS);
      double* cmu = rq.grad ? gp->sMisc.as<double>() : nullptr;
      if (rq.grad)
        pv_kernel<true><<<blocks, PV_WARPS * 32, tail_smem, st>>>(cv, nbc, q, rq.jitter, dval, cmu, cmu + mc, bsbar.as<double>(), err);
      else
        pv_kernel<false><<<blocks, PV_WARPS * 32, tail_smem, st>>>(cv, nbc, q, rq.jitter, dval, nullptr, nullptr, nullptr, err);
      TB_LAUNCHED();
      TB_CUDA(cudaGetLastError());
    }
    if (rq.grad) {
      double* cmu = gp->sMisc.as<double>();
      if (bei)
        bei_backward_kernel<<<(unsigned)nbc, bei_warps * 32, tail_smem, st>>>(mu, cv, q, eps_dev, S, rq.eta, dval, cmu, cmu + mc,
                                                                              bsbar.as<double>(), err);
      else if (!pv)
        qei_backward_kernel<<<(unsigned)((nbc + QEIG_WARPS - 1) / QEIG_WARPS), QEIG_WARPS * 32, tail_smem, st>>>(
            mu, cv, nbc, q, eps_dev, S, rq.eta, rq.jitter, dval, cmu, cmu + mc, bsbar.as<double>(), err);
      TB_LAUNCHED();
      qei_mix_kernel<<<dim3((unsigned)nbc, (unsigned)((gp->N + 255) / 256)), 256, 0, st>>>(gp->sV.as<double>(), lda, (int)gp->N, q,
                                                                                          bsbar.as<double>());
      TB_LAUNCHED();
      double* gd = grad.out(b0);
      TB_TRY(launch_grad(gp, xc, mc, gd));
      TB_TRY(launch_qei_cross(gp, xc, mc, q, bsbar.as<double>(), gd));
    }
    for (auto* o : outs) TB_TRY(o->back(b0, nbc));
  }
  int herr = 0;
  TB_CUDA(cudaMemcpyAsync(&herr, err, sizeof(int), cudaMemcpyDeviceToHost, st));
  TB_CUDA(cudaStreamSynchronize(st));
  TB_CUDA(cudaGetLastError());
  TB_CHECK_CODE(herr == 0, pv ? "Cholesky decomposition was not successful. The input might not be valid "
                                "(covariance + jitter of a query batch is not positive definite)"
                              : "Cholesky decomposition was not successful. The input might not be valid "
                                "(covariance + jitter*I of a query batch is not positive definite)", tb::ERR_NUMERIC);
  return 0;
}

// A = Linv K(X, Xc) for M device-resident points, stored plain ([point][lda], lda = NB*128) in gp->sA; posterior means in
// gp->sMean.  One launch over all M points (callers bound M).
static int compute_a_plain(tb_gp* gp, const double* xc_dev, int64_t M) {
  Engine e;
  TB_TRY(select_engine(gp, false, &e));
  const int nt = eng_tile_width(gp, e);
  const int tiles = (int)((M + nt - 1) / nt);
  const int64_t McPad = (int64_t)tiles * nt;
  TB_TRY(gp->sKs.reserve((size_t)tiles * eng_tile_bytes(gp, e)));
  TB_TRY(gp->sA.reserve((size_t)McPad * gp->NB * BM * sizeof(double)));
  TB_TRY(gp->sMean.reserve(sizeof(double) * McPad));
  TB_TRY(eng_kstar(gp, e, xc_dev, M, tiles));
  return eng_store_a(gp, e, tiles, McPad, gp->sA.as<double>());
}

// out[i][j] = k(x1_i, x2_j) - sum_k A1[i][k] A2[j][k]: posterior covariance between two point sets, row-major [M1, M2]
// (covariance_between_points_encoded, models/gpflow/models.py:188-254: K12 - Kx1 (K + s^2 I)^-1 Kx2, no clipping)
template <int KIND>
__global__ void __launch_bounds__(fac::THREADS)
cross_cov_kernel(const double* __restrict__ A1, const double* __restrict__ A2, int64_t lda, int Nk, const double* __restrict__ X1,
                 const double* __restrict__ X2, const double* __restrict__ inv_ls, int D, int64_t M1, int64_t M2, double variance,
                 double* __restrict__ out) {
  extern __shared__ __align__(16) double sm[];
  const int64_t r0 = (int64_t)blockIdx.y * fac::FB, c0 = (int64_t)blockIdx.x * fac::FB;
  double acc[8][4][2];
  fac::zero_acc(acc);
  fac::dmma_tile<true, true>([&](int m, int k) { return (r0 + m < M1) ? A1[(r0 + m) * lda + k] : 0.0; },
                             [&](int k, int n) { return (c0 + n < M2) ? A2[(c0 + n) * lda + k] : 0.0; }, 0, Nk, acc, sm);
  fac::for_each_acc(acc, [&](int m, int n, double& v) {
    const int64_t i = r0 + m, j = c0 + n;
    if (i >= M1 || j >= M2) return;
    double r2 = 0.0;
    for (int d = 0; d < D; ++d) {
      const double df = (X1[i * D + d] - X2[j * D + d]) * inv_ls[d];
      r2 = fma(df, df, r2);
    }
    out[i * M2 + j] = kernel_from_r2<KIND>(r2, variance) - v;
  });
}

static int run_cross_cov(tb_gp* gp, const double* X1, int64_t M1, const double* X2, int64_t M2, double* out) {
  TB_CUDA(cudaSetDevice(gp->device));
  cudaStream_t st = gp->stream;
  const int D = gp->D;
  const int64_t lda = (int64_t)gp->NB * BM, M = M1 + M2;
  tb::DevBuf bx, bout;
  TB_TRY(bx.reserve(sizeof(double) * M * D));  // [X1; X2] contiguous on the device
  TB_CUDA(cudaMemcpyAsync(bx.p, X1, sizeof(double) * M1 * D, cudaMemcpyDefault, st));
  TB_CUDA(cudaMemcpyAsync(bx.as<double>() + M1 * D, X2, sizeof(double) * M2 * D, cudaMemcpyDefault, st));
  TB_TRY(compute_a_plain(gp, bx.as<double>(), M));
  const Staged<double> outs(out, M1 * M2, bout, st);
  TB_TRY(outs.reserve(1));
  double* od = outs.out(0);
  const double* A1 = gp->sA.as<double>();
  const double* A2 = A1 + M1 * lda;
  const double* x1 = bx.as<double>();
  const double* x2 = x1 + M1 * D;
  const double* il = gp->dInvLs.as<double>();
  const dim3 grid((unsigned)((M2 + fac::FB - 1) / fac::FB), (unsigned)((M1 + fac::FB - 1) / fac::FB));
  TB_TRY(with_kind(gp->kernel, [&](auto K) {
    constexpr int KIND = decltype(K)::value;
    TB_CUDA(cudaFuncSetAttribute(cross_cov_kernel<KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fac::GEMM_SMEM));
    cross_cov_kernel<KIND><<<grid, fac::THREADS, fac::GEMM_SMEM, st>>>(A1, A2, lda, (int)lda, x1, x2, il, D, M1, M2, gp->variance, od);
    return 0;
  }));
  TB_LAUNCHED();
  TB_TRY(outs.back(0, 1));
  TB_CUDA(cudaStreamSynchronize(st));
  TB_CUDA(cudaGetLastError());
  return 0;
}

// ---- joint samples over a LARGE point set (interface.py:135-138 -> gpflow predict_f_samples; the ExactThompsonSampler's
// model.sample, acquisition/sampler.py:85-123): full posterior covariance, blocked Cholesky, mean + L z ----
// cov[i][j] = k(x_i, x_j) - sum_k A[i][k] A[j][k]  (+ jitter on the clipped diagonal); lower 128-tiles, mirrored
template <int KIND>
__global__ void __launch_bounds__(fac::THREADS)
posterior_cov_kernel(const double* __restrict__ A, int64_t lda, int Nk, const double* __restrict__ Xc,
                     const double* __restrict__ inv_ls, int D, int64_t M, double variance, double jitter,
                     double* __restrict__ cov) {
  extern __shared__ __align__(16) double sm[];
  const int tj = blockIdx.x, ti = blockIdx.y;
  if (ti < tj) return;
  const int64_t r0 = (int64_t)ti * fac::FB, c0 = (int64_t)tj * fac::FB;
  double acc[8][4][2];
  fac::zero_acc(acc);
  fac::dmma_tile<true, true>([&](int m, int k) { return (r0 + m < M) ? A[(r0 + m) * lda + k] : 0.0; },
                             [&](int k, int n) { return (c0 + n < M) ? A[(c0 + n) * lda + k] : 0.0; }, 0, Nk, acc, sm);
  fac::for_each_acc(acc, [&](int m, int n, double& v) {
    const int64_t i = r0 + m, j = c0 + n;
    if (i >= M || j >= M || i < j) return;
    double val;
    if (i == j) {
      val = fmax(variance - v, 1e-12) + jitter;
    } else {
      double r2 = 0.0;
      for (int d = 0; d < D; ++d) {
        const double df = (Xc[i * D + d] - Xc[j * D + d]) * inv_ls[d];
        r2 = fma(df, df, r2);
      }
      val = kernel_from_r2<KIND>(r2, variance) - v;
    }
    cov[i + j * M] = val;
    cov[j + i * M] = val;
  });
}

// out[s][i] += mean[i]
__global__ void add_mean_rows_kernel(double* __restrict__ out, const double* __restrict__ mean, int64_t M, int64_t total) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < total) out[e] += mean[e % M];
}

static int run_sample_joint(tb_gp* gp, const double* Xc, int64_t M, const double* z, int S, double jitter, double* out) {
  TB_CUDA(cudaSetDevice(gp->device));
  cudaStream_t st = gp->stream;
  const int D = gp->D;
  const int64_t lda = (int64_t)gp->NB * BM;
  tb::DevBuf bx, bcov, bz, bout, bdinv;
  const Staged<const double> xin(Xc, D, bx, st);
  const double* xc;
  TB_TRY(xin.reserve(M));
  TB_TRY(xin.in(0, M, &xc));
  TB_TRY(compute_a_plain(gp, xc, M));
  TB_TRY(bcov.reserve(sizeof(double) * M * M));
  {
    const unsigned t = (unsigned)((M + fac::FB - 1) / fac::FB);
    const double* A = gp->sA.as<double>();
    const double* il = gp->dInvLs.as<double>();
    double* cov = bcov.as<double>();
    TB_TRY(with_kind(gp->kernel, [&](auto K) {
      constexpr int KIND = decltype(K)::value;
      TB_CUDA(cudaFuncSetAttribute(posterior_cov_kernel<KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fac::GEMM_SMEM));
      posterior_cov_kernel<KIND><<<dim3(t, t), fac::THREADS, fac::GEMM_SMEM, st>>>(A, lda, (int)lda, xc, il, D, M, gp->variance, jitter, cov);
      return 0;
    }));
    TB_LAUNCHED();
  }
  // blocked Cholesky of the covariance with the cache-build kernels (factor.cuh)
  const int nbk = (int)((M + fac::FB - 1) / fac::FB);
  TB_TRY(bdinv.reserve(sizeof(double) * (size_t)nbk * fac::FB * fac::FB));
  int info;
  TB_TRY(blocked_cholesky(gp, bcov.as<double>(), M, bdinv.as<double>(), &info));
  TB_CHECK_CODE(info == 0, "Cholesky decomposition was not successful. The input might not be valid "
                      "(joint covariance + jitter*I is not positive definite at leading minor " + std::to_string(info) + ")", tb::ERR_NUMERIC);
  // samples = mean + L z
  const Staged<const double> zin(z, (int64_t)S * M, bz, st);
  const double* zd;
  TB_TRY(zin.reserve(1));
  TB_TRY(zin.in(0, 1, &zd));
  const Staged<double> outs(out, (int64_t)S * M, bout, st);
  TB_TRY(outs.reserve(1));
  double* od = outs.out(0);
  trmv_lower_cols_kernel<<<dim3((unsigned)((M + 127) / 128), (unsigned)S), 128, 0, st>>>(bcov.as<double>(), M, M, zd, M, od, M);
  TB_LAUNCHED();
  add_mean_rows_kernel<<<(unsigned)(((int64_t)S * M + 255) / 256), 256, 0, st>>>(od, gp->sMean.as<double>(), M, (int64_t)S * M);
  TB_LAUNCHED();
  TB_TRY(outs.back(0, 1));
  TB_CUDA(cudaStreamSynchronize(st));
  TB_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace tb

extern "C" {

int tb_gp_predict_joint(tb_gp* gp, const void* Xc, int64_t B, int q, void* mean, void* cov) {
  TB_CHECK(gp && (B == 0 || (Xc && mean && cov)), "tb_gp_predict_joint: null argument");
  TB_TRY(tb::check_batch(gp, B, q, false, 0, nullptr, 0.0));
  tb::BatchRequest rq(tb::BatchTail::Predict, B, q);
  tb::DtypeBridge br(gp);
  TB_TRY(br.in(Xc, B * q * gp->D, &rq.Xc));
  TB_TRY(br.out(mean, B * q, &rq.out_mean));
  TB_TRY(br.out(cov, B * q * q, &rq.out_cov));
  TB_TRY(tb::run_batch(gp, rq));
  return br.finish();
}

int tb_acq_batch_mc_ei(tb_gp* gp, const void* Xc, int64_t B, int q, const void* eps, int S, double eta, double jitter,
                       void* out) {
  TB_CHECK(gp && (B == 0 || (Xc && eps && out)), "tb_acq_batch_mc_ei: null argument");
  TB_TRY(tb::check_batch(gp, B, q, true, S, eps, jitter));
  tb::BatchRequest rq(tb::BatchTail::McEi, B, q, S, eta, jitter);
  tb::DtypeBridge br(gp);
  TB_TRY(br.in(Xc, B * q * gp->D, &rq.Xc));
  TB_TRY(br.in(eps, (int64_t)q * S, &rq.eps));
  TB_TRY(br.out(out, B, &rq.out_val));
  TB_TRY(tb::run_batch(gp, rq));
  return br.finish();
}

int tb_gp_reparam_sample(tb_gp* gp, const void* Xc, int64_t B, int q, const void* eps, int S, double jitter, void* samples) {
  TB_CHECK(gp && (B == 0 || (Xc && eps && samples)), "tb_gp_reparam_sample: null argument");
  TB_TRY(tb::check_batch(gp, B, q, true, S, eps, jitter));
  tb::BatchRequest rq(tb::BatchTail::Samples, B, q, S, 0.0, jitter);
  tb::DtypeBridge br(gp);
  TB_TRY(br.in(Xc, B * q * gp->D, &rq.Xc));
  TB_TRY(br.in(eps, (int64_t)q * S, &rq.eps));
  TB_TRY(br.out(samples, B * S * q, &rq.out_samples));
  TB_TRY(tb::run_batch(gp, rq));
  return br.finish();
}

// ---- top-k ---------------------------------------------------------------------------------------
int tb_topk(int device, int dtype, const void* values, int64_t M, int k, void* top_values, int64_t* top_indices) {
  TB_CHECK(dtype == TB_F64, "tb_topk: only TB_F64 is implemented in this build");
  TB_CHECK(values && top_values && top_indices, "tb_topk: null argument");
  TB_CHECK(M >= 1 && k >= 1 && k <= M, "tb_topk: need 1 <= k <= M");
  TB_CUDA(cudaSetDevice(device));
  int64_t P = BIT_TILE;
  while (P < M) P <<= 1;
  tb::DevBuf a, vin, tv, ti;  // legacy default stream (0) throughout
  const tb::Staged<const double> vals((const double*)values, M, vin, 0);
  const tb::Staged<double> tvals((double*)top_values, k, tv, 0);
  const tb::Staged<int64_t> tidx(top_indices, k, ti, 0);
  TB_TRY(a.reserve(sizeof(VI) * P));
  const double* vd;
  TB_TRY(vals.reserve(1));
  TB_TRY(vals.in(0, 1, &vd));
  topk_init_kernel<<<(unsigned)((P + 255) / 256), 256>>>(vd, M, P, a.as<VI>());
  TB_LAUNCHED();
  const unsigned nblk = (unsigned)(P / BIT_TILE);
  bitonic_local_kernel<<<nblk, 1024>>>(a.as<VI>(), 2, BIT_TILE);
  TB_LAUNCHED();
  for (int64_t kk = (int64_t)BIT_TILE * 2; kk <= P; kk <<= 1) {
    for (int64_t j = kk >> 1; j >= BIT_TILE; j >>= 1) {
      bitonic_global_kernel<<<(unsigned)((P / 2 + 255) / 256), 256>>>(a.as<VI>(), P, kk, j);
      TB_LAUNCHED();
    }
    bitonic_local_kernel<<<nblk, 1024>>>(a.as<VI>(), kk, kk);
    TB_LAUNCHED();
  }
  TB_TRY(tvals.reserve(1));
  TB_TRY(tidx.reserve(1));
  topk_emit_kernel<<<(k + 255) / 256, 256>>>(a.as<VI>(), k, tvals.out(0), tidx.out(0));
  TB_LAUNCHED();
  TB_CUDA(cudaGetLastError());
  TB_TRY(tvals.back(0, 1));
  TB_TRY(tidx.back(0, 1));
  TB_CUDA(cudaDeviceSynchronize());
  return 0;
}

}  // extern "C"

// =================================================================================================
// random-Fourier-feature trajectories
// =================================================================================================
struct tb_rff {
  int device = 0;
  cudaStream_t stream = nullptr;
  int F = 0, D = 0, DP = 0, nb = 0;
  double variance = 1.0, mean_const = 0.0;
  tb::DevBuf dW, dB, dTheta, dInvLs, sXc, sOut, sBlkBest, sBlkIdx, sRunV, sRunI;
  // canonical features of a decoupled trajectory: scaled training inputs + per-trajectory weights v [nbc, N]
  tb::DevBuf dXs, dV, sCanon, sGrad;
  int kernel = TB_MATERN52, nbc = 0;
  int64_t N = 0;
};

extern "C" {

int tb_rff_create(tb_rff** out, int device) {
  TB_CHECK(out, "tb_rff_create: null output");
  int n = 0;
  TB_TRY(tb_device_count(&n));
  TB_CHECK_CODE(n > 0, "tb_rff_create: no CUDA device visible (this library has no CPU fallback)", tb::ERR_RUNTIME);
  TB_CHECK(device >= 0 && device < n, "tb_rff_create: device index out of range");
  TB_CUDA(cudaSetDevice(device));
  tb_rff* r = new tb_rff();
  r->device = device;
  TB_CUDA(cudaStreamCreateWithFlags(&r->stream, cudaStreamNonBlocking));
  *out = r;
  return 0;
}

int tb_rff_destroy(tb_rff* r) {
  if (!r) return 0;
  cudaSetDevice(r->device);
  cudaStreamSynchronize(r->stream);
  cudaStreamDestroy(r->stream);
  delete r;  // frees the device buffers
  return 0;
}

int tb_rff_set(tb_rff* r, const double* W, const double* b, int F, int D, const double* lengthscales,
               double variance, double mean_const) {
  TB_CHECK(r && W && b && lengthscales, "tb_rff_set: null argument");
  TB_CHECK(F >= 1, "tb_rff_set: need at least one feature");
  TB_CHECK(D >= 1 && tb::pick_dp(D) > 0, "tb_rff_set: input dimension must be in [1, 32]");
  TB_CHECK(variance > 0.0, "tb_rff_set: kernel variance must be positive");
  TB_CUDA(cudaSetDevice(r->device));
  const int DP = tb::pick_dp(D);
  std::vector<double> Wp((size_t)F * DP, 0.0), il(DP, 0.0);
  for (int f = 0; f < F; ++f)
    for (int d = 0; d < D; ++d) Wp[(size_t)f * DP + d] = W[(size_t)f * D + d];
  for (int d = 0; d < D; ++d) {
    TB_CHECK(lengthscales[d] > 0.0, "tb_rff_set: lengthscales must be positive");
    il[d] = 1.0 / lengthscales[d];
  }
  TB_TRY(r->dW.reserve(sizeof(double) * Wp.size()));
  TB_TRY(r->dB.reserve(sizeof(double) * F));
  TB_TRY(r->dInvLs.reserve(sizeof(double) * DP));
  TB_CUDA(cudaMemcpy(r->dW.p, Wp.data(), sizeof(double) * Wp.size(), cudaMemcpyHostToDevice));
  TB_CUDA(cudaMemcpy(r->dB.p, b, sizeof(double) * F, cudaMemcpyHostToDevice));
  TB_CUDA(cudaMemcpy(r->dInvLs.p, il.data(), sizeof(double) * DP, cudaMemcpyHostToDevice));
  r->F = F;
  r->D = D;
  r->DP = DP;
  r->variance = variance;
  r->mean_const = mean_const;
  r->nb = 0;
  r->nbc = 0;
  r->N = 0;
  return 0;
}

int tb_rff_set_theta(tb_rff* r, const double* theta, int nb) {
  TB_CHECK(r && theta, "tb_rff_set_theta: null argument");
  TB_CHECK(r->F > 0, "tb_rff_set_theta: call tb_rff_set first");
  TB_CHECK(nb >= 1, "tb_rff_set_theta: need at least one trajectory");
  TB_CUDA(cudaSetDevice(r->device));
  TB_TRY(r->dTheta.reserve(sizeof(double) * (size_t)nb * r->F));
  TB_CUDA(cudaMemcpy(r->dTheta.p, theta, sizeof(double) * (size_t)nb * r->F, cudaMemcpyDefault));
  r->nb = nb;
  return 0;
}

}  // extern "C"

namespace tb {
template <int DP>
static int launch_rff(tb_rff* r, int nbt, int blocks, const double* xc, int b0, int64_t mc, int64_t idx0, double scale,
                      const double* addend, double* out, double* bb, int64_t* bi) {
  const size_t smem = sizeof(double) * ((size_t)RFF_FCHUNK * DP + RFF_FCHUNK + (size_t)nbt * RFF_FCHUNK);
#define TB_RFF(NBT)                                                                                              \
  {                                                                                                              \
    TB_CUDA(cudaFuncSetAttribute(rff_eval_kernel<DP, NBT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    rff_eval_kernel<DP, NBT><<<blocks, RFF_THREADS, smem, r->stream>>>(r->dW.as<double>(), r->dB.as<double>(),      \
        r->dTheta.as<double>(), xc, r->dInvLs.as<double>(), r->D, r->F, r->nb, b0, mc, idx0, scale, r->mean_const,  \
        addend, fm::TrigConsts(), out, bb, bi);                                                                          \
  }
  switch (nbt) {
    case 1: TB_RFF(1); break;
    case 2: TB_RFF(2); break;
    case 4: TB_RFF(4); break;
    default: TB_RFF(8); break;
  }
#undef TB_RFF
  TB_LAUNCHED();
  TB_CUDA(cudaGetLastError());
  return 0;
}
}  // namespace tb

namespace tb {
template <int KIND, int DP>
static void launch_kdot_nbt(tb_rff* r, const double* xc, int64_t mc, double* out) {
  const int blocks = (int)((mc + 255) / 256);
  for (int b0 = 0; b0 < r->nbc; b0 += 4) {
    const int rem = r->nbc - b0;
    if (rem >= 3)
      kdot_kernel<KIND, DP, 4><<<blocks, 256, 0, r->stream>>>(r->dXs.as<double>(), r->dV.as<double>(), r->N, xc, r->dInvLs.as<double>(),
                                                            (int)r->N, r->D, r->nbc, b0, mc, r->variance, fm::Consts(), out);
    else if (rem == 2)
      kdot_kernel<KIND, DP, 2><<<blocks, 256, 0, r->stream>>>(r->dXs.as<double>(), r->dV.as<double>(), r->N, xc, r->dInvLs.as<double>(),
                                                            (int)r->N, r->D, r->nbc, b0, mc, r->variance, fm::Consts(), out);
    else
      kdot_kernel<KIND, DP, 1><<<blocks, 256, 0, r->stream>>>(r->dXs.as<double>(), r->dV.as<double>(), r->N, xc, r->dInvLs.as<double>(),
                                                            (int)r->N, r->D, r->nbc, b0, mc, r->variance, fm::Consts(), out);
    TB_LAUNCHED();
  }
}
static int launch_kdot(tb_rff* r, const double* xc, int64_t mc, double* out) {
  with_kind_dp(r->kernel, r->DP, [&](auto K, auto P) { launch_kdot_nbt<decltype(K)::value, decltype(P)::value>(r, xc, mc, out); });
  TB_CUDA(cudaGetLastError());
  return 0;
}
}  // namespace tb

extern "C" {

int tb_rff_set_canonical(tb_rff* r, int kernel, const double* X, int64_t N, const double* v, int nb) {
  TB_CHECK(r, "tb_rff_set_canonical: null handle");
  TB_CHECK(r->F > 0, "tb_rff_set_canonical: call tb_rff_set first");
  if (N == 0) {  // switch the canonical part off
    r->N = 0;
    r->nbc = 0;
    return 0;
  }
  TB_CHECK(X && v, "tb_rff_set_canonical: null argument");
  TB_CHECK(kernel >= TB_RBF && kernel <= TB_MATERN52, "tb_rff_set_canonical: unknown kernel kind");
  TB_CHECK(N > 0 && nb >= 1, "tb_rff_set_canonical: need N >= 1 training points and nb >= 1 trajectories");
  TB_CUDA(cudaSetDevice(r->device));
  const int D = r->D, DP = r->DP;
  std::vector<double> il(DP, 0.0), Xs((size_t)N * DP, 0.0);
  TB_CUDA(cudaMemcpy(il.data(), r->dInvLs.p, sizeof(double) * DP, cudaMemcpyDeviceToHost));
  for (int64_t k = 0; k < N; ++k)
    for (int d = 0; d < D; ++d) Xs[(size_t)k * DP + d] = X[(size_t)k * D + d] * il[d];
  TB_TRY(r->dXs.reserve(sizeof(double) * Xs.size()));
  TB_TRY(r->dV.reserve(sizeof(double) * (size_t)nb * N));
  TB_CUDA(cudaMemcpy(r->dXs.p, Xs.data(), sizeof(double) * Xs.size(), cudaMemcpyHostToDevice));
  TB_CUDA(cudaMemcpy(r->dV.p, v, sizeof(double) * (size_t)nb * N, cudaMemcpyDefault));
  r->kernel = kernel;
  r->N = N;
  r->nbc = nb;
  return 0;
}

}  // extern "C"

extern "C" {

int tb_rff_eval(tb_rff* r, const void* Xc, int64_t M, void* out, double* min_value, int64_t* min_index) {
  TB_CHECK(r && (M == 0 || Xc), "tb_rff_eval: null argument");
  TB_CHECK(r->F > 0 && r->nb > 0, "tb_rff_eval: features and theta must be set first");
  TB_CHECK((min_value == nullptr) == (min_index == nullptr), "tb_rff_eval: min_value and min_index go together");
  TB_CHECK(M > 0 || !min_value, "tb_rff_eval: argmin over an empty candidate set");
  if (M == 0) return 0;
  TB_CUDA(cudaSetDevice(r->device));
  cudaStream_t st = r->stream;
  const int D = r->D, nb = r->nb;
  const double scale = std::sqrt(2.0 * r->variance / (double)r->F);
  const int64_t chunk = std::min<int64_t>(M, (int64_t)1 << 22);
  const int blocks_cap = (int)((chunk + RFF_THREADS - 1) / RFF_THREADS);
  const tb::Staged<const double> xin((const double*)Xc, D, r->sXc, st);
  const tb::Staged<double> outs((double*)out, nb, r->sOut, st);
  TB_TRY(xin.reserve(chunk));
  TB_TRY(outs.reserve(chunk));
  const bool want_min = min_value != nullptr;
  if (want_min) {
    TB_TRY(r->sBlkBest.reserve(sizeof(double) * (size_t)nb * blocks_cap));
    TB_TRY(r->sBlkIdx.reserve(sizeof(int64_t) * (size_t)nb * blocks_cap));
    TB_TRY(r->sRunV.reserve(sizeof(double) * nb));
    TB_TRY(r->sRunI.reserve(sizeof(int64_t) * nb));
    std::vector<double> iv(nb, -DBL_MAX);
    std::vector<int64_t> ii(nb, INT64_MAX);
    TB_CUDA(cudaMemcpyAsync(r->sRunV.p, iv.data(), sizeof(double) * nb, cudaMemcpyHostToDevice, st));
    TB_CUDA(cudaMemcpyAsync(r->sRunI.p, ii.data(), sizeof(int64_t) * nb, cudaMemcpyHostToDevice, st));
    TB_CUDA(cudaStreamSynchronize(st));
  }
  for (int64_t c0 = 0; c0 < M; c0 += chunk) {
    const int64_t mc = std::min<int64_t>(chunk, M - c0);
    const int blocks = (int)((mc + RFF_THREADS - 1) / RFF_THREADS);
    const double* xc;
    TB_TRY(xin.in(c0, mc, &xc));
    double* od = outs.out(c0);
    const double* addend = nullptr;
    if (r->N > 0) {
      TB_CHECK(r->nbc == nb, "tb_rff_eval: canonical weights and theta must have the same number of trajectories");
      TB_TRY(r->sCanon.reserve(sizeof(double) * (size_t)chunk * nb));
      TB_TRY(tb::launch_kdot(r, xc, mc, r->sCanon.as<double>()));
      addend = r->sCanon.as<double>();
    }
    for (int b0 = 0, nbt = 0; b0 < nb; b0 += nbt) {
      const int rem = nb - b0;
      nbt = rem >= 5 ? 8 : rem >= 3 ? 4 : rem;  // trajectories per pass: the cosine of a feature is shared by all of them
      double* bb = want_min ? r->sBlkBest.as<double>() : nullptr;
      int64_t* bi = want_min ? r->sBlkIdx.as<int64_t>() : nullptr;
      TB_TRY(tb::with_dp(r->DP, [&](auto P) { return tb::launch_rff<decltype(P)::value>(r, nbt, blocks, xc, b0, mc, c0, scale, addend, od, bb, bi); }));
    }
    if (want_min) {
      // blk arrays are laid out [nb][blocks of this launch]
      rff_fold_kernel<<<nb, 256, 0, st>>>(r->sBlkBest.as<double>(), r->sBlkIdx.as<int64_t>(), blocks,
                                          r->sRunV.as<double>(), r->sRunI.as<int64_t>());
      TB_LAUNCHED();
    }
    TB_TRY(outs.back(c0, mc));
  }
  if (want_min) {
    std::vector<double> hv(nb);
    TB_CUDA(cudaMemcpyAsync(hv.data(), r->sRunV.p, sizeof(double) * nb, cudaMemcpyDeviceToHost, st));
    TB_CUDA(cudaMemcpyAsync(min_index, r->sRunI.p, sizeof(int64_t) * nb, cudaMemcpyDeviceToHost, st));
    TB_CUDA(cudaStreamSynchronize(st));
    for (int b = 0; b < nb; ++b) min_value[b] = -hv[b];
  }
  TB_CUDA(cudaStreamSynchronize(st));
  TB_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"

namespace tb {
// at most this many points per paired launch (the chunk of tb_rff_eval)
constexpr int64_t RFF_PAIRED_CHUNK = (int64_t)1 << 22;

// M (<= RFF_PAIRED_CHUNK) device points, point t under trajectory (pidx ? pidx[t] : idx0 + t) % nb: sgn * values -> out [M],
// sgn * gradients -> grad [M, D] when grad is not null
static int launch_rff_paired(tb_rff* r, const double* xc, int64_t M, int64_t idx0, const int* pidx, double sgn, double* out,
                             double* grad) {
  const int blocks = (int)((M + RFF_THREADS - 1) / RFF_THREADS);
  const double scale = std::sqrt(2.0 * r->variance / (double)r->F);
  const bool canon = r->N > 0;
  return with_kind_dp(r->kernel, r->DP, [&](auto K, auto P) -> int {
    constexpr int KIND = decltype(K)::value, DP = decltype(P)::value;
    const size_t smem = sizeof(double) * ((size_t)RFF_FCHUNK * DP + RFF_FCHUNK);
    auto launch = [&](auto kern) -> int {
      TB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      kern<<<blocks, RFF_THREADS, smem, r->stream>>>(r->dW.as<double>(), r->dB.as<double>(), r->dTheta.as<double>(),
                                                      canon ? r->dXs.as<double>() : nullptr, canon ? r->dV.as<double>() : nullptr,
                                                      xc, r->dInvLs.as<double>(), r->D, r->F, (int)r->N, r->nb, M, idx0, pidx,
                                                      scale, r->mean_const, r->variance, sgn, fm::TrigConsts(), fm::Consts(),
                                                      out, grad);
      TB_LAUNCHED();
      TB_CUDA(cudaGetLastError());
      return 0;
    };
    return grad ? launch(rff_paired_kernel<KIND, DP, true>) : launch(rff_paired_kernel<KIND, DP, false>);
  });
}

static int check_rff_paired(tb_rff* r, const char* name) {
  TB_CHECK(r->F > 0 && r->nb > 0, std::string(name) + ": features and theta must be set first");
  TB_CHECK(r->N == 0 || r->nbc == r->nb,
           std::string(name) + ": canonical weights and theta must have the same number of trajectories");
  return 0;
}
}  // namespace tb

extern "C" {

int tb_rff_eval_paired(tb_rff* r, const void* Xc, int64_t M, int B, void* out, void* grad) {
  TB_CHECK(r, "tb_rff_eval_paired: null handle");
  TB_CHECK(M >= 0, "tb_rff_eval_paired: negative number of points");
  TB_CHECK(M == 0 || (Xc && out), "tb_rff_eval_paired: null argument");
  TB_TRY(tb::check_rff_paired(r, "tb_rff_eval_paired"));
  TB_CHECK(B == r->nb, "tb_rff_eval_paired: the batch size must equal the number of trajectories");
  if (M == 0) return 0;
  TB_CUDA(cudaSetDevice(r->device));
  cudaStream_t st = r->stream;
  const int D = r->D;
  const int64_t P = M * B;
  const int64_t chunk = std::min<int64_t>(P, tb::RFF_PAIRED_CHUNK);
  const tb::Staged<const double> xin((const double*)Xc, D, r->sXc, st);
  const tb::Staged<double> outs((double*)out, 1, r->sOut, st);
  const tb::Staged<double> grads((double*)grad, D, r->sGrad, st);
  TB_TRY(xin.reserve(chunk));
  TB_TRY(outs.reserve(chunk));
  TB_TRY(grads.reserve(chunk));
  for (int64_t c0 = 0; c0 < P; c0 += chunk) {
    const int64_t mc = std::min<int64_t>(chunk, P - c0);
    const double* xc;
    TB_TRY(xin.in(c0, mc, &xc));
    TB_TRY(tb::launch_rff_paired(r, xc, mc, c0, nullptr, 1.0, outs.out(c0), grads.out(c0)));
    TB_TRY(outs.back(c0, mc));
    TB_TRY(grads.back(c0, mc));
  }
  TB_CUDA(cudaStreamSynchronize(st));
  TB_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"


extern "C" {

// ---- device-side multi-start L-BFGS (SURVEY.md §8f-3; acquisition/optimizer.py:566-745) ----
__global__ void lbfgs_finish_kernel(tb::lb::State s, int64_t P, double* __restrict__ f_out, int32_t* __restrict__ success,
                                    int64_t* __restrict__ nfev) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  f_out[p] = -s.f[p];
  success[p] = s.status[p] == tb::lb::ST_SUCCESS ? 1 : 0;
  nfev[p] = (int64_t)s.nfev[p];
}

}  // extern "C"

namespace tb {
// the arguments of every device maximiser: P starts (and their outputs) and the L-BFGS options
static int check_starts(const std::string& who, int64_t P, const double* starts, const double* x_out, const double* f_out,
                        const int32_t* success, const int64_t* nfev, int maxcor, int maxiter, int maxls, double gtol, double ftol) {
  TB_CHECK(P >= 0 && P < ((int64_t)1 << 31), who + ": number of starts out of range");
  TB_CHECK(P == 0 || (starts && x_out && f_out && success && nfev), who + ": null argument");
  TB_CHECK(maxcor >= 1 && maxcor <= lb::MMAX, who + ": maxcor must be in [1, " + std::to_string(lb::MMAX) + "]");
  TB_CHECK(maxiter >= 1 && maxls >= 1, who + ": maxiter and maxls must be positive");
  TB_CHECK(gtol >= 0.0 && ftol >= 0.0, who + ": tolerances must be non-negative");
  return 0;
}

// The multi-start L-BFGS round loop shared by every device maximiser: P (>= 1) problems in D dimensions on the stream st, problem
// p inside box p % nbox of lower/upper [nbox, D] and in group p % G; each
// round asks eval(xt [n, D], idx [n], n, vals [n], grad [n, D], group_n [G]) for the values and gradients of the function to
// MAXIMISE at the trial points of the n active problems (all device arrays; idx holds their problem indices, ordered by group,
// and the host array group_n the number of them in each group), then runs one step of each.  The device-to-host read of the
// group counts is the round's one host synchronise.
template <class Eval>
static int lbfgs_run(const char* name, cudaStream_t st, int D, const double* lower, const double* upper, int nbox, int G,
                     const double* starts, int64_t P, int maxcor, int maxiter, int maxls, double gtol, double ftol, Eval&& eval, double* x_out,
                     double* f_out, int32_t* success, int64_t* nfev) {
  const int m = maxcor;
  const size_t PD = (size_t)P * D;
  // per-problem state + compact evaluation buffers (freed on return)
  tb::DevBuf bx, bf, bg, bd, bt, bS, bY, brho, bgam, bint, bnfev, btrial, bidx, bxt, bval, bgrad, bbox, bcount, bres;
  TB_TRY(bx.reserve(8 * PD)); TB_TRY(bg.reserve(8 * PD)); TB_TRY(bd.reserve(8 * PD)); TB_TRY(btrial.reserve(8 * PD));
  TB_TRY(bf.reserve(8 * (size_t)P)); TB_TRY(bt.reserve(8 * (size_t)P)); TB_TRY(bgam.reserve(8 * (size_t)P));
  TB_TRY(bS.reserve(8 * PD * m)); TB_TRY(bY.reserve(8 * PD * m)); TB_TRY(brho.reserve(8 * (size_t)P * m));
  TB_TRY(bint.reserve(sizeof(int) * 6 * (size_t)P)); TB_TRY(bnfev.reserve(8 * (size_t)P));
  TB_TRY(bidx.reserve(sizeof(int) * (size_t)P)); TB_TRY(bxt.reserve(8 * PD)); TB_TRY(bval.reserve(8 * (size_t)P));
  TB_TRY(bgrad.reserve(8 * PD)); TB_TRY(bbox.reserve(8 * 2 * (size_t)nbox * D)); TB_TRY(bcount.reserve(sizeof(int) * (size_t)G));
  tb::lb::State s;
  s.x = bx.as<double>(); s.f = bf.as<double>(); s.g = bg.as<double>(); s.d = bd.as<double>(); s.t = bt.as<double>();
  s.S = bS.as<double>(); s.Y = bY.as<double>(); s.rho = brho.as<double>(); s.gam = bgam.as<double>();
  int* ints = bint.as<int>();
  s.npairs = ints; s.head = ints + P; s.ls = ints + 2 * P; s.iters = ints + 3 * P; s.phase = ints + 4 * P; s.status = ints + 5 * P;
  s.nfev = bnfev.as<long long>();
  s.xtrial = btrial.as<double>();
  double* dlo = bbox.as<double>();
  double* dup = dlo + (size_t)nbox * D;
  TB_CUDA(cudaMemcpyAsync(dlo, lower, 8 * (size_t)nbox * D, cudaMemcpyDefault, st));
  TB_CUDA(cudaMemcpyAsync(dup, upper, 8 * (size_t)nbox * D, cudaMemcpyDefault, st));
  TB_CUDA(cudaMemcpyAsync(bxt.p, starts, 8 * PD, cudaMemcpyDefault, st));  // staged through the trial buffer
  TB_CUDA(cudaMemsetAsync(bS.p, 0, 8 * PD * m, st));
  TB_CUDA(cudaMemsetAsync(bY.p, 0, 8 * PD * m, st));
  TB_CUDA(cudaMemsetAsync(brho.p, 0, 8 * (size_t)P * m, st));
  tb::lb::lbfgs_init_kernel<<<(unsigned)((PD + 255) / 256), 256, 0, st>>>(bxt.as<double>(), P, D, dlo, dup, nbox, s);
  TB_LAUNCHED();
  tb::lb::Options o{D, m, maxiter, maxls, nbox, gtol, ftol};
  int n_active = 0;
  std::vector<int> group_n(G, 0);
  auto compact = [&]() -> int {
    tb::lb::lbfgs_compact_kernel<<<1, 1024, 0, st>>>(s.status, P, G, bidx.as<int>(), bcount.as<int>());
    TB_LAUNCHED();
    TB_CUDA(cudaMemcpyAsync(group_n.data(), bcount.p, sizeof(int) * (size_t)G, cudaMemcpyDeviceToHost, st));
    TB_CUDA(cudaStreamSynchronize(st));
    n_active = 0;
    for (int g = 0; g < G; ++g) n_active += group_n[g];
    if (n_active > 0) {
      tb::lb::lbfgs_gather_kernel<<<(unsigned)(((size_t)n_active * D + 255) / 256), 256, 0, st>>>(s.xtrial, bidx.as<int>(), n_active, D,
                                                                                                 bxt.as<double>());
      TB_LAUNCHED();
    }
    return 0;
  };
  TB_TRY(compact());
  // every problem ends after at most maxiter accepted steps of at most maxls trials each
  const int64_t max_rounds = (int64_t)maxiter * (int64_t)maxls + 2;
  const bool trace = std::getenv("TB_LBFGS_TRACE") != nullptr;  // per-round (active starts, milliseconds) on stderr
  std::vector<std::pair<int, double>> trace_rows;
  for (int64_t round = 0; n_active > 0 && round < max_rounds; ++round) {
    const auto t_round = std::chrono::steady_clock::now();
    const int n_round = n_active;
    TB_TRY(eval(bxt.as<double>(), bidx.as<int>(), n_active, bval.as<double>(), bgrad.as<double>(), group_n.data()));
    tb::lb::lbfgs_step_kernel<<<(unsigned)((n_active + 7) / 8), 256, 0, st>>>(s, o, n_active, bidx.as<int>(), bxt.as<double>(),
                                                                             bval.as<double>(), bgrad.as<double>(), dlo, dup);
    TB_LAUNCHED();
    TB_TRY(compact());
    if (trace) trace_rows.emplace_back(n_round, std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_round).count());
  }
  if (trace) {
    double total = 0.0;
    for (auto& r : trace_rows) total += r.second;
    std::fprintf(stderr, "[%s] P=%lld rounds=%zu total=%.2f ms:", name, (long long)P, trace_rows.size(), total);
    for (auto& r : trace_rows) std::fprintf(stderr, " %d:%.2f", r.first, r.second);
    std::fprintf(stderr, "\n");
  }
  TB_TRY(bres.reserve((8 + 4 + 8) * (size_t)P));
  double* rf = bres.as<double>();
  int64_t* rn = reinterpret_cast<int64_t*>(rf + P);
  int32_t* rs = reinterpret_cast<int32_t*>(rn + P);
  lbfgs_finish_kernel<<<(unsigned)((P + 255) / 256), 256, 0, st>>>(s, P, rf, rs, rn);
  TB_LAUNCHED();
  TB_CUDA(cudaMemcpyAsync(x_out, s.x, 8 * PD, cudaMemcpyDefault, st));
  TB_CUDA(cudaMemcpyAsync(f_out, rf, 8 * (size_t)P, cudaMemcpyDefault, st));
  TB_CUDA(cudaMemcpyAsync(nfev, rn, 8 * (size_t)P, cudaMemcpyDefault, st));
  TB_CUDA(cudaMemcpyAsync(success, rs, 4 * (size_t)P, cudaMemcpyDefault, st));
  TB_CUDA(cudaStreamSynchronize(st));
  TB_CUDA(cudaGetLastError());
  return 0;
}
}  // namespace tb

extern "C" {

int tb_acq_maximize(tb_gp* gp, int acq, double param, const double* lower, const double* upper, const double* starts, int64_t P,
                    int maxcor, int maxiter, int maxls, double gtol, double ftol, double* x_out, double* f_out,
                    int32_t* success, int64_t* nfev) {
  TB_CHECK(gp && lower && upper, "tb_acq_maximize: null argument");
  TB_TRY(tb::check_starts("tb_acq_maximize", P, starts, x_out, f_out, success, nfev, maxcor, maxiter, maxls, gtol, ftol));
  TB_CHECK(gp->cache_valid, "posterior cache is not built: call tb_gp_update_posterior_cache first");
  bool pen = false;
  TB_TRY(check_acq(gp, acq, param, pen, "tb_acq_maximize"));
  if (P == 0) return 0;
  TB_CUDA(cudaSetDevice(gp->device));
  auto eval = [&](const double* xt, const int*, int n, double* vals, double* grad, const int*) -> int {
    tb::EvalRequest rq;
    rq.acq = acq;
    rq.pen = pen;
    rq.param = param;
    rq.Xc = xt;
    rq.M = n;
    rq.out_vals = vals;
    rq.out_grad = grad;
    return tb::run_eval(gp, rq);
  };
  return tb::lbfgs_run("tb_acq_maximize", gp->stream, gp->D, lower, upper, 1, 1, starts, P, maxcor, maxiter, maxls, gtol, ftol, eval,
                       x_out, f_out, success, nfev);
}

int tb_rff_maximize_boxes(tb_rff* r, const double* lower, const double* upper, int nbox, const double* starts, int64_t R,
                          int maxcor, int maxiter, int maxls, double gtol, double ftol, double* x_out, double* f_out,
                          int32_t* success, int64_t* nfev) {
  TB_CHECK(r && lower && upper, "tb_rff_maximize: null argument");
  TB_TRY(tb::check_rff_paired(r, "tb_rff_maximize"));
  TB_CHECK(nbox >= 1 && r->nb % nbox == 0, "tb_rff_maximize_boxes: the number of boxes " + std::to_string(nbox) +
                                               " must divide the trajectory batch size " + std::to_string(r->nb));
  const int64_t P = R * r->nb;  // nb >= 1 (check_rff_paired): P < 0 exactly when R < 0
  TB_TRY(tb::check_starts("tb_rff_maximize", P, starts, x_out, f_out, success, nfev, maxcor, maxiter, maxls, gtol, ftol));
  if (P == 0) return 0;
  TB_CUDA(cudaSetDevice(r->device));
  const int D = r->D;
  // problem p = (i, b) of the [R, nb, D] starts runs on trajectory p % nb inside box p % nbox = b % nbox (nbox divides nb); the
  // step kernel maximises, so the values and gradients handed to it are those of -f_b
  auto eval = [&](const double* xt, const int* idx, int n, double* vals, double* grad, const int*) -> int {
    for (int64_t c0 = 0; c0 < n; c0 += tb::RFF_PAIRED_CHUNK) {
      const int64_t mc = std::min<int64_t>(tb::RFF_PAIRED_CHUNK, n - c0);
      TB_TRY(tb::launch_rff_paired(r, xt + c0 * D, mc, 0, idx + c0, -1.0, vals + c0, grad + c0 * D));
    }
    return 0;
  };
  return tb::lbfgs_run("tb_rff_maximize", r->stream, D, lower, upper, nbox, 1, starts, P, maxcor, maxiter, maxls, gtol, ftol, eval,
                       x_out, f_out, success, nfev);
}

int tb_rff_maximize(tb_rff* r, const double* lower, const double* upper, const double* starts, int64_t R, int maxcor,
                    int maxiter, int maxls, double gtol, double ftol, double* x_out, double* f_out, int32_t* success,
                    int64_t* nfev) {
  return tb_rff_maximize_boxes(r, lower, upper, 1, starts, R, maxcor, maxiter, maxls, gtol, ftol, x_out, f_out, success, nfev);
}

}  // extern "C"

namespace tb {
// ordering events that destroy themselves
struct Events {
  std::vector<cudaEvent_t> e;
  Events() = default;
  Events(const Events&) = delete;
  Events& operator=(const Events&) = delete;
  ~Events() {
    for (cudaEvent_t x : e)
      if (x) cudaEventDestroy(x);
  }
  int create(int n) {
    e.assign(n, nullptr);
    for (cudaEvent_t& x : e) TB_CUDA(cudaEventCreateWithFlags(&x, cudaEventDisableTiming));
    return 0;
  }
};

// One evaluation round of a maximiser over S handles (lbfgs_run with G = S): group s, the group_n[s] compacted problems at
// offset o, is queued by run(s, o, group_n[s]) on streams[s].  Every stream waits for st before its group and st waits for it
// after (the ehvi_run pattern), so the groups overlap on the device and the round keeps lbfgs_run's single host synchronise.
// ev holds S + 1 events.
template <class Run>
static int fork_join(cudaStream_t st, const cudaStream_t* streams, int S, const int* group_n, Events& ev, Run&& run) {
  TB_CUDA(cudaEventRecord(ev.e[0], st));
  int64_t o = 0;
  for (int s = 0; s < S; ++s) {
    if (group_n[s] == 0) continue;
    const bool own = streams[s] != st;
    if (own) TB_CUDA(cudaStreamWaitEvent(streams[s], ev.e[0], 0));
    TB_TRY(run(s, o, group_n[s]));
    if (own) {
      TB_CUDA(cudaEventRecord(ev.e[s + 1], streams[s]));
      TB_CUDA(cudaStreamWaitEvent(st, ev.e[s + 1], 0));
    }
    o += group_n[s];
  }
  return 0;
}
}  // namespace tb

extern "C" {

int tb_acq_maximize_models(tb_gp* const* models, const int* acq, const double* param, int S, const double* lower,
                           const double* upper, const double* starts, int64_t R, int maxcor, int maxiter, int maxls, double gtol,
                           double ftol, double* x_out, double* f_out, int32_t* success, int64_t* nfev) {
  const std::string who = "tb_acq_maximize_models";
  TB_CHECK(models && acq && param && lower && upper, who + ": null argument");
  TB_CHECK(S >= 1, who + ": the number of models must be at least 1, got " + std::to_string(S));
  std::vector<int> kind(acq, acq + S);
  std::vector<char> pen(S, 0);
  for (int s = 0; s < S; ++s) {
    tb_gp* gp = models[s];
    TB_CHECK(gp, who + ": null model handle " + std::to_string(s));
    // handle state (min-value samples, local penalty, feasibility alpha) belongs to one function: no handle twice
    for (int j = 0; j < s; ++j) TB_CHECK(models[j] != gp, who + ": the same model handle appears twice");
    TB_CHECK(gp->device == models[0]->device, who + ": the models must be on one device");
    TB_CHECK(gp->dtype == models[0]->dtype, who + ": the models must have one dtype");
    TB_CHECK(gp->D == models[0]->D, who + ": the models must have one input dimension");
    TB_CHECK(gp->cache_valid, who + ": posterior cache of model " + std::to_string(s) +
                                  " is not built: call tb_gp_update_posterior_cache first");
    bool p = false;
    TB_TRY(check_acq(gp, kind[s], param[s], p, who.c_str()));
    pen[s] = p;
  }
  TB_CHECK(R >= 0 && R < ((int64_t)1 << 31) / S, who + ": number of starts out of range");
  const int64_t P = R * S;
  TB_TRY(tb::check_starts(who, P, starts, x_out, f_out, success, nfev, maxcor, maxiter, maxls, gtol, ftol));
  if (P == 0) return 0;
  TB_CUDA(cudaSetDevice(models[0]->device));
  const int D = models[0]->D;
  std::vector<cudaStream_t> streams(S);
  for (int s = 0; s < S; ++s) streams[s] = models[s]->stream;
  tb::Events ev;
  TB_TRY(ev.create(S + 1));
  // problem p = r * S + s: model s, box s, group s; each group's rounds see exactly the points tb_acq_maximize on model s alone
  // would evaluate from the starts [R, s, D]
  auto eval = [&](const double* xt, const int*, int, double* vals, double* grad, const int* group_n) -> int {
    return tb::fork_join(streams[0], streams.data(), S, group_n, ev, [&](int s, int64_t o, int n) -> int {
      tb::EvalRequest rq;
      rq.acq = kind[s];
      rq.pen = pen[s] != 0;
      rq.param = param[s];
      rq.Xc = xt + o * D;
      rq.M = n;
      rq.out_vals = vals + o;
      rq.out_grad = grad + o * D;
      rq.sync = false;
      return tb::run_eval(models[s], rq);
    });
  };
  TB_TRY(tb::lbfgs_run(who.c_str(), streams[0], D, lower, upper, S, S, starts, P, maxcor, maxiter, maxls, gtol, ftol, eval, x_out,
                       f_out, success, nfev));
  for (int s = 0; s < S; ++s) TB_TRY(tb::profile_fold(models[s]));  // lbfgs_run's last synchronise joined every stream
  return 0;
}

int tb_rff_maximize_models(tb_rff* const* r, int S, const double* lower, const double* upper, const double* starts, int64_t R,
                           int maxcor, int maxiter, int maxls, double gtol, double ftol, double* x_out, double* f_out,
                           int32_t* success, int64_t* nfev) {
  const std::string who = "tb_rff_maximize_models";
  TB_CHECK(r && lower && upper, who + ": null argument");
  TB_CHECK(S >= 1, who + ": the number of trajectory handles must be at least 1, got " + std::to_string(S));
  for (int s = 0; s < S; ++s) {
    TB_CHECK(r[s], who + ": null trajectory handle " + std::to_string(s));
    for (int j = 0; j < s; ++j) TB_CHECK(r[j] != r[s], who + ": the same trajectory handle appears twice");
    TB_TRY(tb::check_rff_paired(r[s], who.c_str()));
    TB_CHECK(r[s]->device == r[0]->device, who + ": the trajectory handles must be on one device");
    TB_CHECK(r[s]->D == r[0]->D, who + ": the trajectory handles must have one input dimension");
    TB_CHECK(r[s]->nb == r[0]->nb, who + ": every handle must hold the same number of trajectories, got " +
                                       std::to_string(r[s]->nb) + " and " + std::to_string(r[0]->nb));
  }
  const int k = r[0]->nb, V = k * S;
  TB_CHECK(R >= 0 && R < ((int64_t)1 << 31) / V, who + ": number of starts out of range");
  const int64_t P = R * V;
  TB_TRY(tb::check_starts(who, P, starts, x_out, f_out, success, nfev, maxcor, maxiter, maxls, gtol, ftol));
  if (P == 0) return 0;
  TB_CUDA(cudaSetDevice(r[0]->device));
  const int D = r[0]->D;
  std::vector<cudaStream_t> streams(S);
  for (int s = 0; s < S; ++s) streams[s] = r[s]->stream;
  tb::Events ev;
  TB_TRY(ev.create(S + 1));
  tb::DevBuf btraj;
  TB_TRY(btraj.reserve(sizeof(int) * (size_t)P));
  int* traj = btraj.as<int>();
  // problem p = i * V + v: trajectory v / S of handle v % S, box v % S, group v % S = p % S
  auto eval = [&](const double* xt, const int* idx, int n, double* vals, double* grad, const int* group_n) -> int {
    tb::lb::lbfgs_traj_index_kernel<<<(unsigned)((n + 255) / 256), 256, 0, streams[0]>>>(idx, n, V, S, traj);
    TB_LAUNCHED();
    return tb::fork_join(streams[0], streams.data(), S, group_n, ev, [&](int s, int64_t o, int ns) -> int {
      for (int64_t c0 = 0; c0 < ns; c0 += tb::RFF_PAIRED_CHUNK) {
        const int64_t mc = std::min<int64_t>(tb::RFF_PAIRED_CHUNK, ns - c0);
        TB_TRY(tb::launch_rff_paired(r[s], xt + (o + c0) * D, mc, 0, traj + o + c0, -1.0, vals + o + c0, grad + (o + c0) * D));
      }
      return 0;
    });
  };
  return tb::lbfgs_run(who.c_str(), streams[0], D, lower, upper, S, S, starts, P, maxcor, maxiter, maxls, gtol, ftol, eval, x_out,
                       f_out, success, nfev);
}

int tb_gp_covariance_between_points(tb_gp* gp, const void* X1, int64_t M1, const void* X2, int64_t M2, void* out) {
  TB_CHECK(gp && X1 && X2 && out, "tb_gp_covariance_between_points: null argument");
  TB_CHECK(gp->cache_valid, "posterior cache is not built: call tb_gp_update_posterior_cache first");
  TB_CHECK(M1 >= 1 && M2 >= 1 && M1 + M2 <= 16384, "tb_gp_covariance_between_points: between 1 and 16384 points in total");
  tb::DtypeBridge br(gp);
  const double *x1, *x2;
  double* od;
  TB_TRY(br.in(X1, M1 * gp->D, &x1));
  TB_TRY(br.in(X2, M2 * gp->D, &x2));
  TB_TRY(br.out(out, M1 * M2, &od));
  TB_TRY(tb::run_cross_cov(gp, x1, M1, x2, M2, od));
  return br.finish();
}

int tb_gp_sample_joint(tb_gp* gp, const void* Xc, int64_t M, const double* z, int S, double jitter, void* out) {
  TB_CHECK(gp && Xc && z && out, "tb_gp_sample_joint: null argument");
  TB_CHECK(gp->cache_valid, "posterior cache is not built: call tb_gp_update_posterior_cache first");
  TB_CHECK(M >= 1 && M <= 16384, "tb_gp_sample_joint: between 1 and 16384 points");
  TB_CHECK(S >= 1, "tb_gp_sample_joint: need S >= 1 standard-normal draws per point");
  TB_CHECK(jitter >= 0.0, "jitter must be non-negative");
  tb::DtypeBridge br(gp);
  const double* xd;
  double* od;
  TB_TRY(br.in(Xc, M * gp->D, &xd));
  TB_TRY(br.out(out, (int64_t)S * M, &od));
  TB_TRY(tb::run_sample_joint(gp, xd, M, z, S, jitter, od));
  return br.finish();
}

int tb_acq_batch_mc_ei_grad(tb_gp* gp, const void* Xc, int64_t B, int q, const void* eps, int S, double eta, double jitter,
                            void* out, void* grad) {
  TB_CHECK(gp && (B == 0 || (Xc && eps && out && grad)), "tb_acq_batch_mc_ei_grad: null argument");
  TB_TRY(tb::check_batch(gp, B, q, true, S, eps, jitter));
  tb::BatchRequest rq(tb::BatchTail::McEi, B, q, S, eta, jitter);
  rq.grad = true;
  tb::DtypeBridge br(gp);
  TB_TRY(br.in(Xc, B * q * gp->D, &rq.Xc));
  TB_TRY(br.in(eps, (int64_t)q * S, &rq.eps));
  TB_TRY(br.out(out, B, &rq.out_val));
  TB_TRY(br.out(grad, B * q * gp->D, &rq.out_grad));
  TB_TRY(tb::run_batch(gp, rq));
  return br.finish();
}

int tb_acq_predictive_variance(tb_gp* gp, const void* Xc, int64_t B, int q, double jitter, void* out, void* grad) {
  TB_CHECK(gp && (B == 0 || (Xc && out)), "tb_acq_predictive_variance: null argument");
  TB_TRY(tb::check_batch(gp, B, q, false, 0, nullptr, 0.0));
  tb::BatchRequest rq(tb::BatchTail::PredVar, B, q, 0, 0.0, jitter);
  rq.grad = grad != nullptr;
  tb::DtypeBridge br(gp);
  TB_TRY(br.in(Xc, B * q * gp->D, &rq.Xc));
  TB_TRY(br.out(out, B, &rq.out_val));
  TB_TRY(br.out(grad, B * q * gp->D, &rq.out_grad));
  TB_TRY(tb::run_batch(gp, rq));
  return br.finish();
}

// ---- batch expected improvement (Chevalier & Ginsbourger with Genz CDFs) ----
static int bei_args(tb_gp* gp, const void* Xc, int64_t B, int q, const double* w, int S, const void* out, const void* grad,
                    bool want_grad, const char* fn) {
  TB_CHECK(gp && w && (B == 0 || (Xc && out && (!want_grad || grad))), std::string(fn) + ": null argument");
  TB_CHECK(q >= 2 && q <= 32, std::string(fn) + ": batch size q must be in [2, 32]");
  TB_CHECK(S >= 1, std::string(fn) + ": need S >= 1 Sobol points");
  TB_CHECK(B >= 0, std::string(fn) + ": negative batch count");
  TB_CHECK(gp->cache_valid, "posterior cache is not built: call tb_gp_update_posterior_cache first");
  return 0;
}

int tb_acq_batch_ei(tb_gp* gp, const void* Xc, int64_t B, int q, const double* w, int S, double eta, void* out) {
  TB_TRY(bei_args(gp, Xc, B, q, w, S, out, nullptr, false, "tb_acq_batch_ei"));
  if (B == 0) return 0;
  tb::BatchRequest rq(tb::BatchTail::BatchEi, B, q, S, eta);
  rq.eps = w;
  tb::DtypeBridge br(gp);
  TB_TRY(br.in(Xc, B * q * gp->D, &rq.Xc));
  TB_TRY(br.out(out, B, &rq.out_val));
  TB_TRY(tb::run_batch(gp, rq));
  return br.finish();
}

int tb_acq_batch_ei_grad(tb_gp* gp, const void* Xc, int64_t B, int q, const double* w, int S, double eta, void* out,
                         void* grad) {
  TB_TRY(bei_args(gp, Xc, B, q, w, S, out, grad, true, "tb_acq_batch_ei_grad"));
  if (B == 0) return 0;
  tb::BatchRequest rq(tb::BatchTail::BatchEi, B, q, S, eta);
  rq.grad = true;
  rq.eps = w;
  tb::DtypeBridge br(gp);
  TB_TRY(br.in(Xc, B * q * gp->D, &rq.Xc));
  TB_TRY(br.out(out, B, &rq.out_val));
  TB_TRY(br.out(grad, B * q * gp->D, &rq.out_grad));
  TB_TRY(tb::run_batch(gp, rq));
  return br.finish();
}

int tb_mvn_cdf(int device, const double* x, const double* mean, const double* cov, int64_t B, int Q, const double* w, int S,
               double jitter, double* out) {
  TB_CHECK(B >= 0, "tb_mvn_cdf: negative batch count");
  TB_CHECK(B == 0 || (x && mean && cov && out), "tb_mvn_cdf: null argument");
  TB_CHECK(Q >= 1 && Q <= 32, "tb_mvn_cdf: dimension Q must be in [1, 32]");
  TB_CHECK(Q == 1 || w, "tb_mvn_cdf: Q >= 2 needs the Sobol points w [Q-1, S]");
  TB_CHECK(S >= 1, "tb_mvn_cdf: need S >= 1 Sobol points");
  if (B == 0) return 0;
  TB_CUDA(cudaSetDevice(device));
  tb::DevBuf bx, bm, bc, bw, bo, berr;  // legacy default stream (0) throughout
  auto stage = [](const tb::Staged<const double>& s, const double** dev) -> int {
    TB_TRY(s.reserve(1));
    return s.in(0, 1, dev);
  };
  const double *xd, *md, *cd, *wd;
  TB_TRY(stage({x, (int64_t)B * Q, bx, 0}, &xd));
  TB_TRY(stage({mean, (int64_t)B * Q, bm, 0}, &md));
  TB_TRY(stage({cov, (int64_t)B * Q * Q, bc, 0}, &cd));
  TB_TRY(stage({Q >= 2 ? w : nullptr, (int64_t)(Q - 1) * S, bw, 0}, &wd));
  const tb::Staged<double> outs(out, B, bo, 0);
  TB_TRY(outs.reserve(1));
  double* od = outs.out(0);
  TB_TRY(berr.reserve(sizeof(int)));
  TB_CUDA(cudaMemset(berr.p, 0, sizeof(int)));
  const size_t smem = (size_t)tb::BEI_MAX_WARPS * tb::bei_warp_doubles(Q) * sizeof(double);
  TB_CUDA(cudaFuncSetAttribute(tb::mvn_cdf_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  tb::mvn_cdf_kernel<<<(unsigned)((B + tb::BEI_MAX_WARPS - 1) / tb::BEI_MAX_WARPS), tb::BEI_MAX_WARPS * 32, smem>>>(
      xd, md, cd, B, Q, wd, S, jitter, od, berr.as<int>());
  TB_LAUNCHED();
  TB_CUDA(cudaGetLastError());
  int herr = 0;
  TB_CUDA(cudaMemcpy(&herr, berr.p, sizeof(int), cudaMemcpyDeviceToHost));
  TB_TRY(outs.back(0, 1));
  TB_CUDA(cudaDeviceSynchronize());
  TB_CHECK_CODE(herr == 0, "Cholesky decomposition was not successful. The input might not be valid "
                      "(cov + jitter*I of a row is not positive definite)", tb::ERR_NUMERIC);
  return 0;
}

}  // extern "C"

// =================================================================================================
// several handles per chunk: the members' predict on their own streams, one combining kernel (EHVI, reducers)
// =================================================================================================
namespace tb {

// the borrowed member handles of a function over several GPs, its staging buffers and the events of its chunk loop
struct MemberSet {
  std::vector<tb_gp*> m;  // borrowed, distinct
  int L = 0, D = 0, device = 0, dtype = TB_F64;
  DevBuf sXc, sVals, sGrad, sGradL;  // staged candidates, values, gradient, and the members' gradients [L][mc][D]
  std::vector<cudaEvent_t> ev;       // ev[l] orders member l's stream against the first member's (ev[0]: the other way)
  ~MemberSet() {
    if (!ev.empty()) cudaSetDevice(device);
    for (cudaEvent_t e : ev)
      if (e) cudaEventDestroy(e);
  }
};

// the checks of a create call on the L handles (the caller has checked L's range), then the events
static int members_init(MemberSet* s, tb_gp* const* models, int L, const char* who) {
  const std::string w(who);
  for (int l = 0; l < L; ++l) {
    TB_CHECK(models[l], w + ": null model handle");
    TB_CHECK(models[l]->have_data, w + ": member " + std::to_string(l) + " has no data");
    for (int j = 0; j < l; ++j) TB_CHECK(models[j] != models[l], w + ": the same model handle appears twice");
    TB_CHECK(models[l]->device == models[0]->device, w + ": the members must be on one device");
    TB_CHECK(models[l]->dtype == models[0]->dtype, w + ": the members must have one dtype");
    TB_CHECK(models[l]->D == models[0]->D, w + ": the members must have one input dimension");
  }
  TB_CUDA(cudaSetDevice(models[0]->device));
  s->m.assign(models, models + L);
  s->L = L;
  s->D = models[0]->D;
  s->device = models[0]->device;
  s->dtype = models[0]->dtype;
  s->ev.assign(L, nullptr);
  for (int l = 0; l < L; ++l) {
    if (cudaEventCreateWithFlags(&s->ev[l], cudaEventDisableTiming) != cudaSuccess) {
      cudaGetLastError();
      return fail(w + ": cudaEventCreate failed", ERR_RUNTIME);
    }
  }
  return 0;
}

// what every evaluation needs of the members, checked before anything is staged
static int members_check(const MemberSet* s, const char* who) {
  for (int l = 0; l < s->L; ++l) {
    const tb_gp* gp = s->m[l];
    TB_CHECK(gp->cache_valid, std::string(who) + ": posterior cache of member " + std::to_string(l) +
                                  " is not built: call tb_gp_update_posterior_cache first");
    TB_CHECK(gp->D == s->D, std::string(who) + ": member " + std::to_string(l) + " has input dimension " + std::to_string(gp->D) +
                                ", the stack " + std::to_string(s->D));
  }
  return 0;
}

// The chunk loop over several members (rq.acq unused).  The candidates are staged once, on the first member's stream st;
// each chunk runs every member's member_step on the member's own stream, then combine(mb, mc, c0, vals) on st over all
// members' chunk outputs (it writes the values, each member's d/d(mean, var) with a gradient, and with rq.want_argmax the
// block winners into the first member's sBlkBest / sBlkIdx), then the members' gradient assemblies and their fixed-order
// sum, then the argmax fold.  Events order the member streams against st both ways; the host waits once, at the end.
template <class Combine>
static int members_run(MemberSet* h, EvalRequest& rq, Combine&& combine) {
  TB_CUDA(cudaSetDevice(h->device));
  const int L = h->L, D = h->D;
  tb_gp* g0 = h->m[0];
  cudaStream_t st = g0->stream;
  const bool grad = rq.out_grad != nullptr;
  if (rq.M == 0) return 0;
  Engine eng[MEMBERS_MAX];
  for (int l = 0; l < L; ++l) TB_TRY(select_engine(h->m[l], grad, &eng[l]));
  const ChunkPlan cp = plan_chunks(h->m.data(), eng, L, grad, rq.M);
  const int64_t chunk_cap = cp.chunk_cap;
  for (int l = 0; l < L; ++l) TB_TRY(reserve_chunk(h->m[l], eng[l], grad, chunk_cap, cp.G[l]));
  const Staged<const double> xin(rq.Xc, D, h->sXc, st);
  const Staged<double> vals(rq.out_vals, 1, h->sVals, st), grads(rq.out_grad, D, h->sGrad, st);
  TB_TRY(xin.reserve(chunk_cap));
  TB_TRY(vals.reserve(chunk_cap));
  TB_TRY(grads.reserve(chunk_cap));
  if (grad) TB_TRY(h->sGradL.reserve(sizeof(double) * (size_t)L * chunk_cap * D));
  if (rq.want_argmax) TB_TRY(argmax_begin(g0, chunk_cap));
  // st -> members (ev[0]) and member l -> st (ev[l])
  auto fan_out = [&]() -> int {
    TB_CUDA(cudaEventRecord(h->ev[0], st));
    for (int l = 1; l < L; ++l) TB_CUDA(cudaStreamWaitEvent(h->m[l]->stream, h->ev[0], 0));
    return 0;
  };
  auto join = [&](int l) -> int {
    if (l == 0) return 0;
    TB_CUDA(cudaEventRecord(h->ev[l], h->m[l]->stream));
    TB_CUDA(cudaStreamWaitEvent(st, h->ev[l], 0));
    return 0;
  };
  for (int64_t c0 = 0; c0 < rq.M; c0 += chunk_cap) {
    const int64_t mc = std::min<int64_t>(chunk_cap, rq.M - c0);
    const double* xc;
    TB_TRY(xin.in(c0, mc, &xc));
    TB_TRY(fan_out());
    ChunkMembers mb{};
    for (int l = 0; l < L; ++l) {
      tb_gp* gp = h->m[l];
      TB_TRY(member_step(gp, eng[l], xc, mc, cp.G[l], grad, &mb.G[l], &mb.McPad[l]));
      TB_TRY(join(l));
      mb.partial[l] = gp->sPartial.as<double>();
      mb.mean[l] = gp->sMean.as<double>();
      mb.dmv[l] = grad ? gp->sMisc.as<double>() : nullptr;
      mb.variance[l] = gp->variance;
    }
    TB_TRY(combine(mb, mc, c0, vals.out(c0)));
    if (grad) {
      TB_TRY(fan_out());
      double* gl = h->sGradL.as<double>();
      for (int l = 0; l < L; ++l) {
        TB_TRY(launch_grad(h->m[l], xc, mc, gl + (size_t)l * mc * D));
        TB_TRY(join(l));
      }
      member_grad_sum_kernel<<<(unsigned)((mc * D + 255) / 256), 256, 0, st>>>(gl, L, mc * D, grads.out(c0));
      TB_LAUNCHED();
      TB_CUDA(cudaGetLastError());
    }
    if (rq.want_argmax) TB_TRY(argmax_fold(g0, mc));
    TB_TRY(grads.back(c0, mc));
    TB_TRY(vals.back(c0, mc));
  }
  if (rq.want_argmax) TB_TRY(argmax_end(g0, rq));
  TB_CUDA(cudaStreamSynchronize(st));
  TB_CUDA(cudaGetLastError());
  for (int l = 0; l < L; ++l) TB_TRY(profile_fold(h->m[l]));
  return 0;
}

// a function over several handles as the ABI takes it: eval, and argmax when best_index is set; run(rq) runs the loop
template <class Run>
static int members_call(const MemberSet* h, const void* Xc, int64_t M, void* out, void* grad, void* best_value,
                        int64_t* best_index, Run&& run) {
  EvalRequest rq;
  rq.M = M;
  rq.want_argmax = best_index != nullptr;
  DtypeBridge br(h->m[0]);
  TB_TRY(br.in(Xc, M * h->D, &rq.Xc));
  TB_TRY(br.out(out, M, &rq.out_vals));
  TB_TRY(br.out(grad, M * h->D, &rq.out_grad));
  TB_TRY(run(rq));
  if (best_index) argmax_result(rq, h->dtype, best_value, best_index);
  return br.finish();
}

}  // namespace tb

// =================================================================================================
// expected hypervolume improvement over a stack of L handles (ehvi.cuh)
// =================================================================================================
struct tb_ehvi : tb::MemberSet {  // one member per objective
  int64_t K = 0;          // cells; 0: not set
  tb::DevBuf dCells;      // lower [K][L] then upper [K][L]
  int P = 0;              // HIPPO pending points (tb_ehvi_set_penalty); 0: no penalty
  tb::DevBuf dPen;        // their means [P][L] then standard deviations [P][L]
  std::vector<double> hPen;  // the means and variances [2][P][L] as last set, to recognise an unchanged push
};

namespace tb {

template <int L>
static void launch_ehvi_l(bool grad, const ChunkMembers& mb, const EhviPenalty& pen, const double* cells, int64_t K, int64_t mc,
                          int64_t c0, double* vals, double* bb, int64_t* bi, cudaStream_t st) {
  const unsigned blocks = (unsigned)((mc + 255) / 256);
  if (pen.P > 0) {
    if (grad)
      ehvi_kernel<L, true, true><<<blocks, 256, 0, st>>>(mb, pen, cells, K, mc, c0, vals, bb, bi);
    else
      ehvi_kernel<L, false, true><<<blocks, 256, 0, st>>>(mb, pen, cells, K, mc, c0, vals, bb, bi);
  } else if (grad) {
    ehvi_kernel<L, true, false><<<blocks, 256, 0, st>>>(mb, pen, cells, K, mc, c0, vals, bb, bi);
  } else {
    ehvi_kernel<L, false, false><<<blocks, 256, 0, st>>>(mb, pen, cells, K, mc, c0, vals, bb, bi);
  }
}

static int launch_ehvi(tb_ehvi* h, bool grad, const ChunkMembers& mb, int64_t mc, int64_t c0, double* vals, bool argmax) {
  tb_gp* g0 = h->m[0];
  double* bb = argmax ? g0->sBlkBest.as<double>() : nullptr;
  int64_t* bi = argmax ? g0->sBlkIdx.as<int64_t>() : nullptr;
  const double* cells = h->dCells.as<double>();
  const double* pd = h->P > 0 ? h->dPen.as<double>() : nullptr;
  const EhviPenalty pen{pd, pd ? pd + (size_t)h->P * h->L : nullptr, h->P};
  switch (h->L) {
    case 2: launch_ehvi_l<2>(grad, mb, pen, cells, h->K, mc, c0, vals, bb, bi, g0->stream); break;
    case 3: launch_ehvi_l<3>(grad, mb, pen, cells, h->K, mc, c0, vals, bb, bi, g0->stream); break;
    case 4: launch_ehvi_l<4>(grad, mb, pen, cells, h->K, mc, c0, vals, bb, bi, g0->stream); break;
    case 5: launch_ehvi_l<5>(grad, mb, pen, cells, h->K, mc, c0, vals, bb, bi, g0->stream); break;
    case 6: launch_ehvi_l<6>(grad, mb, pen, cells, h->K, mc, c0, vals, bb, bi, g0->stream); break;
    case 7: launch_ehvi_l<7>(grad, mb, pen, cells, h->K, mc, c0, vals, bb, bi, g0->stream); break;
    default: launch_ehvi_l<8>(grad, mb, pen, cells, h->K, mc, c0, vals, bb, bi, g0->stream); break;
  }
  TB_LAUNCHED();
  TB_CUDA(cudaGetLastError());
  return 0;
}

// what every EHVI evaluation needs of the object and its members, checked before anything is staged
static int ehvi_check(const tb_ehvi* h, const char* who) {
  TB_CHECK(h->K >= 1, std::string(who) + ": the partition cells are not set (tb_ehvi_set_cells)");
  return members_check(h, who);
}

// the EHVI chunk loop: members_run with the EHVI kernel as the combining step
static int ehvi_run(tb_ehvi* h, EvalRequest& rq) {
  const bool grad = rq.out_grad != nullptr;
  return members_run(h, rq, [&](const ChunkMembers& mb, int64_t mc, int64_t c0, double* vals) {
    return launch_ehvi(h, grad, mb, mc, c0, vals, rq.want_argmax);
  });
}

}  // namespace tb

extern "C" {

int tb_ehvi_create(tb_ehvi** out, tb_gp* const* models, int L) {
  TB_CHECK(out && models, "tb_ehvi_create: null argument");
  TB_CHECK(L >= 2 && L <= tb::EHVI_LMAX, "tb_ehvi_create: the number of objectives must be in [2, " +
                                             std::to_string(tb::EHVI_LMAX) + "], got " + std::to_string(L));
  std::unique_ptr<tb_ehvi> h(new tb_ehvi());
  TB_TRY(tb::members_init(h.get(), models, L, "tb_ehvi_create"));
  *out = h.release();
  return 0;
}

int tb_ehvi_destroy(tb_ehvi* h) {
  if (!h) return 0;
  cudaSetDevice(h->device);
  delete h;  // frees the device buffers and the events; the member handles are borrowed
  return 0;
}

int tb_ehvi_set_cells(tb_ehvi* h, const double* lower, const double* upper, int64_t K) {
  TB_CHECK(h && lower && upper, "tb_ehvi_set_cells: null argument");
  TB_CHECK(K >= 1, "tb_ehvi_set_cells: need at least one cell");
  TB_CUDA(cudaSetDevice(h->device));
  const size_t n = (size_t)K * h->L;
  cudaStream_t st = h->m[0]->stream;
  TB_TRY(h->dCells.reserve(sizeof(double) * 2 * n));
  TB_CUDA(cudaMemcpyAsync(h->dCells.p, lower, sizeof(double) * n, cudaMemcpyDefault, st));
  TB_CUDA(cudaMemcpyAsync(h->dCells.as<double>() + n, upper, sizeof(double) * n, cudaMemcpyDefault, st));
  TB_CUDA(cudaStreamSynchronize(st));
  h->K = K;
  return 0;
}

int tb_ehvi_set_penalty(tb_ehvi* h, const double* pending_mean, const double* pending_var, int P) {
  TB_CHECK(h, "tb_ehvi_set_penalty: null handle");
  TB_CHECK(P >= 0, "tb_ehvi_set_penalty: negative number of pending points");
  if (P == 0) {
    h->P = 0;
    h->hPen.clear();
    return 0;
  }
  TB_CHECK(pending_mean && pending_var, "tb_ehvi_set_penalty: null argument");
  const size_t n = (size_t)P * h->L;
  const bool dev = tb::is_device_ptr(pending_mean) || tb::is_device_ptr(pending_var);
  std::vector<double> in;
  const double *mean = pending_mean, *var = pending_var;
  if (dev) {  // device arrays are read back: the variances are checked on the host
    TB_CUDA(cudaSetDevice(h->device));
    in.resize(2 * n);
    TB_CUDA(cudaMemcpy(in.data(), pending_mean, sizeof(double) * n, cudaMemcpyDefault));
    TB_CUDA(cudaMemcpy(in.data() + n, pending_var, sizeof(double) * n, cudaMemcpyDefault));
    mean = in.data();
    var = in.data() + n;
  }
  // the state the object already holds (the penalised function pushes before every launch): no copy, no synchronise
  if (h->P == P && std::equal(mean, mean + n, h->hPen.begin()) && std::equal(var, var + n, h->hPen.begin() + n)) return 0;
  for (size_t i = 0; i < n; ++i)
    TB_CHECK(var[i] >= 0.0, "tb_ehvi_set_penalty: the pending variances must be non-negative, got " + std::to_string(var[i]));
  std::vector<double> held(mean, mean + n);
  held.insert(held.end(), var, var + n);
  std::vector<double> up(mean, mean + n);
  for (size_t i = 0; i < n; ++i) up.push_back(std::sqrt(var[i]));
  TB_CUDA(cudaSetDevice(h->device));
  cudaStream_t st = h->m[0]->stream;
  h->P = 0;  // a failed upload leaves no penalty
  h->hPen.clear();
  TB_TRY(h->dPen.reserve(sizeof(double) * 2 * n));
  TB_CUDA(cudaMemcpyAsync(h->dPen.p, up.data(), sizeof(double) * 2 * n, cudaMemcpyHostToDevice, st));
  TB_CUDA(cudaStreamSynchronize(st));
  h->hPen.swap(held);
  h->P = P;
  return 0;
}

// tb_ehvi_eval, and tb_ehvi_argmax when best_index is set
static int ehvi_call(tb_ehvi* h, const void* Xc, int64_t M, void* out, void* grad, void* best_value, int64_t* best_index,
                     const char* who) {
  TB_TRY(tb::ehvi_check(h, who));
  return tb::members_call(h, Xc, M, out, grad, best_value, best_index, [&](tb::EvalRequest& rq) { return tb::ehvi_run(h, rq); });
}

int tb_ehvi_eval(tb_ehvi* h, const void* Xc, int64_t M, void* out, void* grad) {
  TB_CHECK(h && (M == 0 || (Xc && out)), "tb_ehvi_eval: null argument");
  TB_CHECK(M >= 0, "tb_ehvi_eval: negative candidate count");
  return ehvi_call(h, Xc, M, out, grad, nullptr, nullptr, "tb_ehvi_eval");
}

int tb_ehvi_argmax(tb_ehvi* h, const void* Xc, int64_t M, void* out, void* best_value, int64_t* best_index) {
  TB_CHECK(h && Xc && best_value && best_index, "tb_ehvi_argmax: null argument");
  TB_CHECK(M > 0, "tb_ehvi_argmax: argmax over an empty candidate set");
  return ehvi_call(h, Xc, M, out, nullptr, best_value, best_index, "tb_ehvi_argmax");
}

int tb_ehvi_maximize(tb_ehvi* h, const double* lower, const double* upper, const double* starts, int64_t P, int maxcor,
                     int maxiter, int maxls, double gtol, double ftol, double* x_out, double* f_out, int32_t* success,
                     int64_t* nfev) {
  TB_CHECK(h && lower && upper, "tb_ehvi_maximize: null argument");
  TB_TRY(tb::check_starts("tb_ehvi_maximize", P, starts, x_out, f_out, success, nfev, maxcor, maxiter, maxls, gtol, ftol));
  TB_TRY(tb::ehvi_check(h, "tb_ehvi_maximize"));
  if (P == 0) return 0;
  TB_CUDA(cudaSetDevice(h->device));
  auto eval = [&](const double* xt, const int*, int n, double* vals, double* grad, const int*) -> int {
    tb::EvalRequest rq;
    rq.Xc = xt;
    rq.M = n;
    rq.out_vals = vals;
    rq.out_grad = grad;
    return tb::ehvi_run(h, rq);
  };
  return tb::lbfgs_run("tb_ehvi_maximize", h->m[0]->stream, h->D, lower, upper, 1, 1, starts, P, maxcor, maxiter, maxls, gtol, ftol,
                       eval, x_out, f_out, success, nfev);
}

}  // extern "C"

// =================================================================================================
// reducers over single-query acquisitions of several handles (reduce.cuh)
// =================================================================================================
struct tb_reduce : tb::MemberSet {  // the distinct handles the terms use
  int op = -1;  // tb_reduce_op; -1: the terms are not set
  int T = 0;
  int member[tb::REDUCE_TMAX] = {}, acq[tb::REDUCE_TMAX] = {};
  double param[tb::REDUCE_TMAX] = {}, alpha[tb::REDUCE_TMAX] = {};  // alpha: the feasibility terms' only, else 0
};

namespace tb {

static bool reduce_kind(int acq) {
  return acq == TB_ACQ_EI || acq == TB_ACQ_LOG_EI || acq == TB_ACQ_NEG_LCB || acq == TB_ACQ_LCB || acq == TB_ACQ_PBT ||
         acq == TB_ACQ_AEI || acq == TB_ACQ_MES || active_learning_kind(acq);
}

// what every evaluation needs of the object and its members, checked before anything is staged
static int reduce_check(const tb_reduce* h, const char* who) {
  TB_CHECK(h->op >= 0, std::string(who) + ": the terms are not set (tb_reduce_set_terms)");
  TB_TRY(members_check(h, who));
  for (int k = 0; k < h->T; ++k)
    if (h->acq[k] == TB_ACQ_MES)
      TB_CHECK(h->m[h->member[k]]->mesS > 0, std::string(who) + ": term " + std::to_string(k) +
                                                 " (min-value entropy search) needs its member's min-value samples first "
                                                 "(tb_acq_set_min_value_samples)");
  return 0;
}

template <int OP>
static void launch_reduce_op(bool grad, const ChunkMembers& mb, const ReduceTerms& tm, int L, int64_t mc, int64_t c0,
                             double* vals, double* bb, int64_t* bi, cudaStream_t st) {
  const unsigned blocks = (unsigned)((mc + 255) / 256);
  if (grad)
    reduce_kernel<OP, true><<<blocks, 256, 0, st>>>(mb, tm, L, mc, c0, vals, bb, bi);
  else
    reduce_kernel<OP, false><<<blocks, 256, 0, st>>>(mb, tm, L, mc, c0, vals, bb, bi);
}

// the chunk loop: members_run with reduce_kernel as the combining step
static int reduce_run(tb_reduce* h, EvalRequest& rq) {
  const bool grad = rq.out_grad != nullptr;
  ReduceTerms tm{};
  tm.T = h->T;
  for (int k = 0; k < h->T; ++k) {
    const tb_gp* gp = h->m[h->member[k]];
    tm.member[k] = h->member[k];
    tm.acq[k] = h->acq[k];
    tm.param[k] = h->param[k];
    tm.aux[k] = feasibility_kind(h->acq[k]) ? h->alpha[k] : gp->noise;
    tm.samp[k] = h->acq[k] == TB_ACQ_MES ? gp->dMes.as<double>() : nullptr;
    tm.nsamp[k] = h->acq[k] == TB_ACQ_MES ? gp->mesS : 0;
  }
  return members_run(h, rq, [&](const ChunkMembers& mb, int64_t mc, int64_t c0, double* vals) -> int {
    tb_gp* g0 = h->m[0];
    double* bb = rq.want_argmax ? g0->sBlkBest.as<double>() : nullptr;
    int64_t* bi = rq.want_argmax ? g0->sBlkIdx.as<int64_t>() : nullptr;
    if (h->op == TB_REDUCE_SUM)
      launch_reduce_op<TB_REDUCE_SUM>(grad, mb, tm, h->L, mc, c0, vals, bb, bi, g0->stream);
    else if (h->op == TB_REDUCE_PRODUCT)
      launch_reduce_op<TB_REDUCE_PRODUCT>(grad, mb, tm, h->L, mc, c0, vals, bb, bi, g0->stream);
    else
      launch_reduce_op<TB_REDUCE_SOFTPLUS>(grad, mb, tm, h->L, mc, c0, vals, bb, bi, g0->stream);
    TB_LAUNCHED();
    TB_CUDA(cudaGetLastError());
    return 0;
  });
}

}  // namespace tb

extern "C" {

int tb_reduce_create(tb_reduce** out, tb_gp* const* models, int n) {
  TB_CHECK(out && models, "tb_reduce_create: null argument");
  TB_CHECK(n >= 1 && n <= tb::MEMBERS_MAX, "tb_reduce_create: the number of distinct models must be in [1, " +
                                                std::to_string(tb::MEMBERS_MAX) + "], got " + std::to_string(n));
  std::unique_ptr<tb_reduce> h(new tb_reduce());
  TB_TRY(tb::members_init(h.get(), models, n, "tb_reduce_create"));
  *out = h.release();
  return 0;
}

int tb_reduce_destroy(tb_reduce* h) {
  if (!h) return 0;
  cudaSetDevice(h->device);
  delete h;  // frees the device buffers and the events; the member handles are borrowed
  return 0;
}

int tb_reduce_set_terms(tb_reduce* h, int op, int T, const int* member, const int* acq, const double* param,
                        const double* alpha) {
  TB_CHECK(h && member && acq && param, "tb_reduce_set_terms: null argument");
  TB_CHECK(op == TB_REDUCE_SUM || op == TB_REDUCE_PRODUCT || op == TB_REDUCE_SOFTPLUS,
           "tb_reduce_set_terms: unknown reduction " + std::to_string(op));
  TB_CHECK(T >= 1 && T <= tb::REDUCE_TMAX, "tb_reduce_set_terms: the number of terms must be in [1, " +
                                               std::to_string(tb::REDUCE_TMAX) + "], got " + std::to_string(T));
  TB_CHECK(op != TB_REDUCE_SOFTPLUS || T == 1, "tb_reduce_set_terms: the softplus takes one term, got " + std::to_string(T));
  double al[tb::REDUCE_TMAX] = {};
  for (int k = 0; k < T; ++k) {
    const std::string term = "tb_reduce_set_terms: term " + std::to_string(k);
    TB_CHECK(member[k] >= 0 && member[k] < h->L, term + ": member index " + std::to_string(member[k]) + " is not in [0, " +
                                                     std::to_string(h->L) + ")");
    TB_CHECK(tb::reduce_kind(acq[k]), term + ": kind " + std::to_string(acq[k]) +
                                          " is not one a reduction fuses (GIBBON, penalised and unknown kinds are not)");
    if (acq[k] == TB_ACQ_LCB || acq[k] == TB_ACQ_NEG_LCB)
      TB_CHECK(param[k] >= 0.0, term + ": Standard deviation scaling parameter beta must not be negative");
    if (acq[k] == TB_ACQ_BALD) TB_CHECK(param[k] > 0.0, term + ": Jitter must be positive.");
    if (tb::feasibility_kind(acq[k])) {
      TB_CHECK(alpha, "tb_reduce_set_terms: null alpha with a feasibility term");
      TB_CHECK(alpha[k] > 0.0 && std::isfinite(alpha[k]), term + ": alpha must be positive and finite, got " + std::to_string(alpha[k]));
      al[k] = alpha[k];
    }
  }
  h->op = op;
  h->T = T;
  for (int k = 0; k < T; ++k) {
    h->member[k] = member[k];
    h->acq[k] = acq[k];
    h->param[k] = param[k];
    h->alpha[k] = al[k];
  }
  return 0;
}

int tb_reduce_eval(tb_reduce* h, const void* Xc, int64_t M, void* out, void* grad) {
  TB_CHECK(h && (M == 0 || (Xc && out)), "tb_reduce_eval: null argument");
  TB_CHECK(M >= 0, "tb_reduce_eval: negative candidate count");
  TB_TRY(tb::reduce_check(h, "tb_reduce_eval"));
  return tb::members_call(h, Xc, M, out, grad, nullptr, nullptr, [&](tb::EvalRequest& rq) { return tb::reduce_run(h, rq); });
}

int tb_reduce_argmax(tb_reduce* h, const void* Xc, int64_t M, void* out, void* best_value, int64_t* best_index) {
  TB_CHECK(h && Xc && best_value && best_index, "tb_reduce_argmax: null argument");
  TB_CHECK(M > 0, "tb_reduce_argmax: argmax over an empty candidate set");
  TB_TRY(tb::reduce_check(h, "tb_reduce_argmax"));
  return tb::members_call(h, Xc, M, out, nullptr, best_value, best_index, [&](tb::EvalRequest& rq) { return tb::reduce_run(h, rq); });
}

int tb_reduce_maximize(tb_reduce* h, const double* lower, const double* upper, const double* starts, int64_t P, int maxcor,
                       int maxiter, int maxls, double gtol, double ftol, double* x_out, double* f_out, int32_t* success,
                       int64_t* nfev) {
  TB_CHECK(h && lower && upper, "tb_reduce_maximize: null argument");
  TB_TRY(tb::check_starts("tb_reduce_maximize", P, starts, x_out, f_out, success, nfev, maxcor, maxiter, maxls, gtol, ftol));
  TB_TRY(tb::reduce_check(h, "tb_reduce_maximize"));
  if (P == 0) return 0;
  TB_CUDA(cudaSetDevice(h->device));
  auto eval = [&](const double* xt, const int*, int n, double* vals, double* grad, const int*) -> int {
    tb::EvalRequest rq;
    rq.Xc = xt;
    rq.M = n;
    rq.out_vals = vals;
    rq.out_grad = grad;
    return tb::reduce_run(h, rq);
  };
  return tb::lbfgs_run("tb_reduce_maximize", h->m[0]->stream, h->D, lower, upper, 1, 1, starts, P, maxcor, maxiter, maxls, gtol,
                       ftol, eval, x_out, f_out, success, nfev);
}

}  // extern "C"
