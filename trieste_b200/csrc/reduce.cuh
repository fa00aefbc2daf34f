// Reducers over single-query acquisitions of several GPs (trieste acquisition/combination.py: Sum, Product;
// function/function.py:1914-1990: MakePositive), one thread per candidate of a chunk.
//
// Term k is kind acq[k] with parameter param[k] on member member[k]; its value v_k is what tail_kernel computes for that
// kind on the member's chunk outputs (kind_value, the variance clipped at 1e-12).  The terms combine in term order:
//   sum      v_0 + v_1 + ... + v_{T-1}
//   product  ((v_0 v_1) ...) v_{T-1}
//   softplus log(1 + exp(v_0))  (T = 1, the reference's form)
// Gradient (each member's sMisc, d/dmean [mc] then d/dvar [mc], the layout grad_kernel reads): the partials of term k,
// times c_k = 1 (sum), the product of the other terms' values as prefix x suffix (product: no division, a zero factor
// gives a finite gradient) or sigmoid(v_0) (softplus: 1 / (1 + exp(-v_0)), the finite form of exp(v)/(1 + exp(v))),
// accumulated in term order into the term's member.
#pragma once
#include "kernels_f64.cuh"

namespace tb {

constexpr int REDUCE_TMAX = 8;

// the terms as the kernel reads them; aux[k]: the feasibility kinds' alpha, else the member's noise (tail_aux)
struct ReduceTerms {
  int T;
  int member[REDUCE_TMAX];
  int acq[REDUCE_TMAX];
  double param[REDUCE_TMAX];
  double aux[REDUCE_TMAX];
  const double* samp[REDUCE_TMAX];  // MES: the member's min-value samples
  int nsamp[REDUCE_TMAX];
};

// d value / d (mean, var) of one term: acq_partials_kernel's selection for the kinds a reducer takes
__device__ __forceinline__ void kind_partials(int acq, double param, double aux, const double* __restrict__ samp, int nsamp,
                                              double mu, double var, bool clipped, double& dm, double& dv) {
  if (acq == TB_ACQ_MES)
    mes_partials(samp, nsamp, mu, var, clipped, dm, dv);
  else if (active_learning_kind(acq))
    active_learning_partials(acq, param, aux, mu, var, clipped, dm, dv);
  else
    acq_partials(acq, param, aux, mu, var, clipped, dm, dv);
}

// OP: TB_REDUCE_SUM / _PRODUCT / _SOFTPLUS.  L: the number of members.  Candidate t's value to out_vals[t] (nullable); with
// blk_best the block's first-max (NaN never wins) of (value, idx0 + t).
template <int OP, bool GRAD>
__global__ void __launch_bounds__(256)
reduce_kernel(const ChunkMembers mb, const ReduceTerms tm, int L, int64_t Mc, int64_t idx0, double* __restrict__ out_vals,
              double* __restrict__ blk_best, int64_t* __restrict__ blk_idx) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  double bv = -INFINITY;
  int64_t bi = INT64_MAX;
  if (t < Mc) {
    double v[REDUCE_TMAX], dm[REDUCE_TMAX], dv[REDUCE_TMAX];
#pragma unroll
    for (int k = 0; k < REDUCE_TMAX; ++k) {
      v[k] = OP == TB_REDUCE_PRODUCT ? 1.0 : 0.0;
      dm[k] = 0.0;
      dv[k] = 0.0;
      if (k < tm.T) {
        const int l = tm.member[k];
        const double raw = chunk_raw_variance(mb.partial[l], mb.G[l], mb.McPad[l], t, mb.variance[l]);
        const double var = fmax(raw, 1e-12), mu = mb.mean[l][t];
        v[k] = kind_value(tm.acq[k], tm.param[k], tm.aux[k], tm.samp[k], tm.nsamp[k], mu, var, nullptr, t, 0.0);
        if (GRAD) kind_partials(tm.acq[k], tm.param[k], tm.aux[k], tm.samp[k], tm.nsamp[k], mu, var, raw < 1e-12, dm[k], dv[k]);
      }
    }
    double val;
    if (OP == TB_REDUCE_SOFTPLUS) {
      val = log(1.0 + exp(v[0]));
    } else {
      val = v[0];
#pragma unroll
      for (int k = 1; k < REDUCE_TMAX; ++k)
        if (k < tm.T) val = OP == TB_REDUCE_SUM ? val + v[k] : val * v[k];
    }
    if (GRAD) {
      double c[REDUCE_TMAX];
      if (OP == TB_REDUCE_PRODUCT) {
        double pre = 1.0;
#pragma unroll
        for (int k = 0; k < REDUCE_TMAX; ++k) {
          c[k] = pre;
          pre *= v[k];  // the padding terms are 1
        }
        double suf = 1.0;
#pragma unroll
        for (int k = REDUCE_TMAX - 1; k >= 0; --k) {
          c[k] *= suf;
          suf *= v[k];
        }
      } else {
#pragma unroll
        for (int k = 0; k < REDUCE_TMAX; ++k) c[k] = OP == TB_REDUCE_SOFTPLUS ? 1.0 / (1.0 + exp(-v[0])) : 1.0;
      }
      for (int l = 0; l < L; ++l) {
        double am = 0.0, av = 0.0;
#pragma unroll
        for (int k = 0; k < REDUCE_TMAX; ++k)
          if (k < tm.T && tm.member[k] == l) {
            am = fma(c[k], dm[k], am);
            av = fma(c[k], dv[k], av);
          }
        mb.dmv[l][t] = am;
        mb.dmv[l][Mc + t] = av;
      }
    }
    if (out_vals) out_vals[t] = val;
    if (val == val) {
      bv = val;
      bi = idx0 + t;
    }
  }
  if (blk_best == nullptr) return;
  block_best_store(bv, bi, blk_best, blk_idx);
}

}  // namespace tb
