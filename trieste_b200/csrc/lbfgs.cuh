// Device-side multi-start projected L-BFGS (SURVEY.md §8f-3): the replacement of the reference's R greenlets + R SciPy
// L-BFGS-B instances (acquisition/optimizer.py:566-745).  Every start is an independent problem with its own curvature
// history; one warp owns one problem (lane = input dimension, D <= 32), so the two-loop recursion is m warp-reductions.
// The host loop is: batched value+gradient evaluation of the trial points of all ACTIVE problems (the fused GP kernels)
// -> lbfgs_step_kernel (line-search decision, history update, convergence tests, next direction and trial point)
// -> compaction of the active set.  Minimises f = -acquisition inside problem p's box: lower/upper hold nbox boxes [nbox, D]
// and problem p uses box p % nbox (with starts laid out [R, nb, D] and nbox | nb, column b uses box b % nbox).  The box is
// looked up from the original problem index, never from a compacted slot.
#pragma once
#include "common.cuh"

namespace tb {
namespace lb {

constexpr int MMAX = 16;  // largest history length (SciPy's maxcor default is 10)

enum Phase : int { PH_INIT = 0, PH_LINESEARCH = 1 };
enum Status : int { ST_ACTIVE = 0, ST_SUCCESS = 1, ST_FAILED = 2 };

struct State {
  double *x, *f, *g, *d, *t;       // accepted iterate [P,D], [P], [P,D]; search direction [P,D]; current step [P]
  double *S, *Y, *rho, *gam;       // history [P,m,D] x2, [P,m], initial Hessian scaling [P]
  int *npairs, *head, *ls, *iters, *phase, *status;
  long long* nfev;
  double* xtrial;                  // next point to evaluate, by problem [P,D]
};

struct Options {
  int D, m, maxiter, maxls, nbox;
  double gtol, ftol;
};

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double clampd(double v, double lo, double hi) { return fmin(fmax(v, lo), hi); }

// new search direction from the stored pairs (two-loop recursion on the free variables), first trial point of the line
// search; returns false when the projected direction vanishes (first-order point)
__device__ __forceinline__ bool new_direction(const State& s, const Options& o, long long p, int lane, bool in, double x, double g,
                                              double lo, double up) {
  const int m = o.m, D = o.D;
  const bool free_ = in && !((x <= lo && g > 0.0) || (x >= up && g < 0.0));
  double q = free_ ? g : 0.0;
  const int np = min(s.npairs[p], m), head = s.head[p];
  double alpha[MMAX];
  for (int i = 0; i < np; ++i) {  // newest first
    const int slot = (head - 1 - i + 2 * m) % m;
    const double sv = free_ ? s.S[(p * m + slot) * D + lane] : 0.0, yv = free_ ? s.Y[(p * m + slot) * D + lane] : 0.0;
    const double a = s.rho[p * m + slot] * warp_sum(sv * q);
    q -= a * yv;
    alpha[i] = a;
  }
  double r = s.gam[p] * q;
  for (int i = np - 1; i >= 0; --i) {  // oldest first
    const int slot = (head - 1 - i + 2 * m) % m;
    const double sv = free_ ? s.S[(p * m + slot) * D + lane] : 0.0, yv = free_ ? s.Y[(p * m + slot) * D + lane] : 0.0;
    const double beta = s.rho[p * m + slot] * warp_sum(yv * r);
    r += sv * (alpha[i] - beta);
  }
  double d = free_ ? -r : 0.0;
  const double gd = warp_sum(in ? g * d : 0.0);
  if (!(gd < 0.0)) d = free_ ? -g : 0.0;  // not a descent direction: projected steepest descent
  const double nrm = sqrt(warp_sum(d * d));
  if (nrm == 0.0) return false;
  const double t = (s.npairs[p] == 0) ? fmin(1.0, 1.0 / fmax(nrm, 1e-300)) : 1.0;  // SciPy-like conservative first step
  if (in) {
    s.d[p * D + lane] = d;
    s.xtrial[p * D + lane] = clampd(x + t * d, lo, up);
  }
  if (lane == 0) {
    s.t[p] = t;
    s.ls[p] = 0;
  }
  return true;
}

// one warp per active problem: consume the evaluation of its trial point
__global__ void __launch_bounds__(256)
lbfgs_step_kernel(State s, Options o, int n_active, const int* __restrict__ idx, const double* __restrict__ xt,
                  const double* __restrict__ acq_val, const double* __restrict__ acq_grad, const double* __restrict__ lower,
                  const double* __restrict__ upper) {
  const int w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w >= n_active) return;
  const long long p = idx[w];
  const int D = o.D, m = o.m;
  const bool in = lane < D;
  const long long box = (p % o.nbox) * D;
  const double lo = in ? lower[box + lane] : 0.0, up = in ? upper[box + lane] : 0.0;
  const double xn = in ? xt[(long long)w * D + lane] : 0.0;
  const double fn = -acq_val[w];
  const double gn = in ? -acq_grad[(long long)w * D + lane] : 0.0;
  if (lane == 0) s.nfev[p] += 1;
  int status = ST_ACTIVE;
  bool accepted;
  double f_old = 0.0;
  if (s.phase[p] == PH_INIT) {
    accepted = true;
    if (!isfinite(fn)) status = ST_FAILED;
  } else {
    const double x0 = in ? s.x[p * D + lane] : 0.0, g0 = in ? s.g[p * D + lane] : 0.0;
    const double step = xn - x0;
    f_old = s.f[p];
    const double slope = warp_sum(g0 * step);
    accepted = isfinite(fn) && fn <= f_old + 1e-4 * slope;  // Armijo on the projected step
    if (accepted) {
      const double y = gn - g0;
      const double sy = warp_sum(step * y), yy = warp_sum(y * y);
      if (sy > 1e-10 * yy) {
        const int head = s.head[p];
        if (in) {
          s.S[(p * m + head) * D + lane] = step;
          s.Y[(p * m + head) * D + lane] = y;
        }
        if (lane == 0) {
          s.rho[p * m + head] = 1.0 / sy;
          s.gam[p] = sy / yy;
          s.npairs[p] += 1;
          s.head[p] = (head + 1) % m;
        }
      }
      __syncwarp();
    }
  }
  if (accepted && status == ST_ACTIVE) {
    if (in) {
      s.x[p * D + lane] = xn;
      s.g[p * D + lane] = gn;
    }
    if (lane == 0) s.f[p] = fn;
    const double pg = in ? fabs(xn - clampd(xn - gn, lo, up)) : 0.0;
    const bool conv_g = warp_max(pg) <= o.gtol;
    bool conv_f = false;
    int iters = s.iters[p];
    if (s.phase[p] != PH_INIT) {
      conv_f = (f_old - fn) <= o.ftol * fmax(fmax(fabs(f_old), fabs(fn)), 1.0);
      iters += 1;
    }
    __syncwarp();
    if (lane == 0) {
      s.iters[p] = iters;
      s.phase[p] = PH_LINESEARCH;
    }
    if (conv_g || conv_f) {
      status = ST_SUCCESS;
    } else if (iters >= o.maxiter) {
      status = ST_FAILED;
    } else {
      __syncwarp();
      if (!new_direction(s, o, p, lane, in, xn, gn, lo, up)) status = ST_SUCCESS;
    }
  } else if (status == ST_ACTIVE) {
    // rejected trial: halve the step (projected backtracking); a failed line search ends the run unsuccessfully
    const int ls = s.ls[p] + 1;
    const double t = s.t[p] * 0.5;
    __syncwarp();
    if (ls >= o.maxls) {
      status = ST_FAILED;
    } else {
      if (in) s.xtrial[p * D + lane] = clampd(s.x[p * D + lane] + t * s.d[p * D + lane], lo, up);
      if (lane == 0) {
        s.ls[p] = ls;
        s.t[p] = t;
      }
    }
  }
  if (lane == 0) s.status[p] = status;
}

// deterministic compaction of the active problems (single CTA, block scan) + gather of their trial points.  The active problems
// are ordered by group g = p % G, increasing p within a group; count[g] receives the number of active problems of group g (with
// G = 1, count[0] is the number of active problems and idx lists them in increasing order).
__global__ void __launch_bounds__(1024)
lbfgs_compact_kernel(const int* __restrict__ status, long long P, int G, int* __restrict__ idx, int* __restrict__ count) {
  __shared__ int warp_tot[32];
  __shared__ int base;
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  int prev = 0;  // thread 0: active problems of the groups before g
  for (int g = 0; g < G; ++g) {
    const long long nG = (P - g + G - 1) / G;  // problems g, g + G, ...
    for (long long c0 = 0; c0 < nG; c0 += blockDim.x) {
      const long long j = c0 + threadIdx.x, p = g + j * G;
      const int a = (j < nG && status[p] == ST_ACTIVE) ? 1 : 0;
      int v = a;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int n = __shfl_up_sync(0xffffffffu, v, o);
        if ((threadIdx.x & 31) >= o) v += n;
      }
      if ((threadIdx.x & 31) == 31) warp_tot[threadIdx.x >> 5] = v;
      __syncthreads();
      if (threadIdx.x < 32) {
        int t = warp_tot[threadIdx.x];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int n = __shfl_up_sync(0xffffffffu, t, o);
          if (threadIdx.x >= o) t += n;
        }
        warp_tot[threadIdx.x] = t;  // inclusive totals of the warps
      }
      __syncthreads();
      const int before = ((threadIdx.x >> 5) > 0 ? warp_tot[(threadIdx.x >> 5) - 1] : 0) + v - a;
      if (a) idx[base + before] = (int)p;
      __syncthreads();
      if (threadIdx.x == 0) base += warp_tot[31];
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      count[g] = base - prev;
      prev = base;
    }
  }
}

// trajectory of each compacted problem of tb_rff_maximize_models: problem p = i * V + v runs trajectory v / S of its handle
__global__ void lbfgs_traj_index_kernel(const int* __restrict__ idx, int n, int V, int S, int* __restrict__ traj) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n) traj[t] = (idx[t] % V) / S;
}

__global__ void lbfgs_gather_kernel(const double* __restrict__ xtrial, const int* __restrict__ idx, int n_active, int D,
                                    double* __restrict__ xt) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)n_active * D) return;
  const long long i = e / D;
  const int d = (int)(e % D);
  xt[e] = xtrial[(long long)idx[i] * D + d];
}

// starting points clipped into their problems' boxes; all problems active in phase INIT
__global__ void lbfgs_init_kernel(const double* __restrict__ starts, long long P, int D, const double* __restrict__ lower,
                                  const double* __restrict__ upper, int nbox, State s) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= P * D) return;
  const int d = (int)(e % D);
  const long long b = ((e / D) % nbox) * D + d;
  s.xtrial[e] = clampd(starts[e], lower[b], upper[b]);
  s.x[e] = s.xtrial[e];
  s.g[e] = 0.0;
  s.d[e] = 0.0;
  if (d == 0) {
    const long long p = e / D;
    s.f[p] = 0.0;
    s.t[p] = 1.0;
    s.gam[p] = 1.0;
    s.npairs[p] = 0;
    s.head[p] = 0;
    s.ls[p] = 0;
    s.iters[p] = 0;
    s.phase[p] = PH_INIT;
    s.status[p] = ST_ACTIVE;
    s.nfev[p] = 0;
  }
}

}  // namespace lb
}  // namespace tb
