/*
 * trieste_b200 — C-ABI of the H100-native GP-posterior + acquisition engine.
 *
 * This is the drop-in boundary for the hot path named by BASELINE.json `north_star`
 * (SURVEY.md §8b).  The reference has no FFI: its boundary is a set of Python structural
 * protocols.  Each entry point below cites the reference interface it stands behind
 * (paths relative to the trieste 4.2.1 source tree).  The Python host layer (`trieste_b200/`) binds these
 * with ctypes and mirrors the reference's class/method names on top; INTEGRATION.md shows the
 * binding a trieste maintainer would add.
 *
 * Conventions
 *   - every function returns a tb_status: 0 on success, otherwise the class of the failure (below);
 *     tb_last_error() returns the thread-local message.  The Python layer maps the CODE (not the text) to the
 *     exception the reference raises for the same condition; nothing aborts the process (the BO loop records
 *     exceptions, bayesian_optimizer.py:855-875).
 *   - plain pointers + sizes only.  Every array pointer may be a HOST pointer or a DEVICE pointer
 *     on the handle's GPU (detected with cudaPointerGetAttributes); host buffers are staged
 *     through the handle's stream inside the call.
 *   - row-major, dense; fp64 unless the handle was created with TB_F32.
 *   - one caller per handle, one CUDA stream per handle, synchronous return
 *     (results are immediately `.numpy()`-ed by the reference, optimizer.py:665-666).
 */
#ifndef TRIESTE_B200_H
#define TRIESTE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct tb_gp tb_gp;   /* exact-GPR posterior: owns device copies of X, Linv, alpha, hyper-params */
typedef struct tb_rff tb_rff; /* random-Fourier-feature trajectory: owns W, b, theta */
typedef struct tb_ehvi tb_ehvi; /* expected hypervolume improvement over L borrowed tb_gp handles: owns the partition cells */
typedef struct tb_reduce tb_reduce; /* sum / product / softplus of single-query acquisitions over n borrowed tb_gp handles */

enum tb_status {
  TB_OK = 0,
  TB_ERR_INVALID = 1, /* bad argument / unmet precondition: ValueError (tf.errors.InvalidArgumentError in the reference) */
  TB_ERR_RUNTIME = 2, /* CUDA or library failure, no GPU: RuntimeError (there is no CPU fallback) */
  TB_ERR_NUMERIC = 3  /* a Cholesky factorisation met a non-positive-definite matrix: ValueError, like tf.linalg.cholesky's
                         InvalidArgumentError ("Cholesky decomposition was not successful") */
};
enum tb_dtype { TB_F64 = 0, TB_F32 = 1 };
/* gpflow.kernels.{SquaredExponential,Matern12,Matern32,Matern52}; trieste default Matern52
 * (models/gpflow/builders.py:399) */
enum tb_kernel { TB_RBF = 0, TB_MATERN12 = 1, TB_MATERN32 = 2, TB_MATERN52 = 3 };
enum tb_acq {
  TB_ACQ_EI = 0,      /* expected_improvement.__call__, acquisition/function/function.py:215-223 */
  TB_ACQ_LOG_EI = 1,  /* log of the above; ABSENT in the reference (SURVEY.md §8 a8) */
  TB_ACQ_NEG_LCB = 2, /* NegativeLowerConfidenceBound, function.py:358-359 (−lower_confidence_bound :415-416) */
  TB_ACQ_LCB = 3,     /* lower_confidence_bound, function.py:389-418 */
  TB_ACQ_PBT = 4,     /* probability_below_threshold.__call__, function.py:501-509 (ProbabilityOfImprovement :47-93,
                         ProbabilityOfFeasibility :421-478): Normal(mean, sqrt(var)).cdf(param) */
  TB_ACQ_AEI = 5,     /* augmented_expected_improvement.__call__, function.py:311-325: EI(param = eta) times
                         1 − sqrt(noise)/sqrt(noise + var), noise = the handle's likelihood variance */
  TB_ACQ_MES = 6,     /* min_value_entropy_search.__call__, entropy.py:193-213: mean over the min-value samples set by
                         tb_acq_set_min_value_samples of −γ·φ(γ)/(2Φ(−γ)) − log Φ(−γ), γ = (y* − mean)/sd; param unused */
  TB_ACQ_GIBBON_QUALITY = 7,   /* gibbon_quality_term.__call__, entropy.py:479-500: −½ mean_s log(1 + ρ² r_s (γ_s − r_s)),
                                  ρ² = var/(var + σ²), r = φ(γ)/Φ(−γ), over the tb_acq_set_min_value_samples samples */
  TB_ACQ_GIBBON_REPULSION = 8, /* gibbon_repulsion_term.__call__, entropy.py:580-618: w·½(log(yvar − ‖L_B⁻¹c(x)‖²) − log yvar)
                                  over the pending points set by tb_acq_set_gibbon_repulsion; yvar = var + σ²;
                                  needs no min-value samples */
  TB_ACQ_GIBBON = 9,           /* GibbonAcquisition.__call__, entropy.py:435-436: repulsion + quality */
  TB_ACQ_FEASIBILITY_BICHON = 10, /* bichon_ranjan_criterion(delta = 1), active_learning.py:227-234: G_1 * sqrt(var),
                                     t = (param - mean)/sqrt(var); param = the threshold T, alpha set by tb_acq_set_feasibility */
  TB_ACQ_FEASIBILITY_RANJAN = 11, /* bichon_ranjan_criterion(delta = 2), active_learning.py:235-243: G_2 * var */
  TB_ACQ_BALD = 12,               /* bayesian_active_learning_by_disagreement.__call__, active_learning.py:498-513:
                                     h(Phi(mean / sqrt(v + 1))) - E, v = max(var, param); param = the jitter (> 0) */
  TB_ACQ_PREDICTIVE_VARIANCE = 13 /* predictive_variance at q = 1, active_learning.py:98-108: exp(logdet([[var + param]]))
                                     = var + param; param = the jitter (q > 1: tb_acq_predictive_variance) */
};
/* OR-ed into `acq` of tb_acq_eval / tb_acq_argmax / tb_acq_maximize: the value (and gradient) is multiplied by the local
 * penalty set by tb_acq_set_penalization (PenalizedAcquisition, acquisition/function/greedy_batch.py:250-269). */
#define TB_ACQ_PENALIZED 0x100
/* local penalisers (greedy_batch.py:315-388) */
enum tb_penalizer {
  TB_PEN_SOFT = 1, /* soft_local_penalizer: prod_j Φ((‖x − x_j‖ − radius_j)/scale_j) */
  TB_PEN_HARD = 2  /* hard_local_penalizer: prod_j ((‖x − x_j‖/(radius_j + scale_j))^−5 + 1)^(−1/5) */
};

/* ---- errors / build info ------------------------------------------------------------------ */
const char* tb_last_error(void);
const char* tb_version(void);
int tb_device_count(int* count);

/* ---- model handle ----------------------------------------------------------------------------
 * mirrors GaussianProcessRegression (models/gpflow/models.py:69-186) + GPflowPredictor's posterior
 * cache (models/gpflow/interface.py:89-112). */
int tb_gp_create(tb_gp** out, int device, int dtype);
int tb_gp_destroy(tb_gp* gp);

/* GPR data Variables assign, models.py:171-186 (update_encoded).  X [N,D], y [N] (E = 1). */
int tb_gp_set_data(tb_gp* gp, const void* X, const void* y, int64_t N, int D);

/* kernel / likelihood / mean-function hyper-parameters (gpflow Parameters read through
 * get_kernel / get_observation_noise / get_mean_function, models/interfaces.py:166-225).
 * lengthscales: n_ls = 1 (isotropic) or D (ARD), always double. */
int tb_gp_set_hyper(tb_gp* gp, int kernel, double variance, const double* lengthscales, int n_ls,
                    double noise_variance, double mean_const);

/* update_posterior_cache (interface.py:108-112): err = y − m(X), L = chol(K(X,X) + σ²I) (hand-written blocked
 * Cholesky on the DMMA pipe, once per BO step), then Linv and alpha = K⁻¹err packed for the kernels. */
int tb_gp_update_posterior_cache(tb_gp* gp);

/* Append m (1..64) observations to the data AND extend the cached L, Linv and alpha in O(m N²) — the incremental form of
 * update_encoded (models.py:171-186) followed by update_posterior_cache (interface.py:108-112), which in the reference
 * refactorise from scratch every BO step (SURVEY.md §8f-1).  Requires a valid cache and unchanged hyper-parameters;
 * same error behaviour as tb_gp_update_posterior_cache (on failure the cache is left invalid).  Xnew [m,D], ynew [m]. */
int tb_gp_append_data(tb_gp* gp, const void* Xnew, const void* ynew, int64_t m);

/* copy out the cached Cholesky factor L [N,N] row-major lower (tests / diagnostics). */
int tb_gp_get_cholesky(tb_gp* gp, void* L_out);

/* predict_encoded (interface.py:119-124): Xc [M,D] → mean [M], var [M] (clipped to ≥ 1e-12). */
int tb_gp_predict(tb_gp* gp, const void* Xc, int64_t M, void* mean, void* var);

/* predict_joint_encoded (interface.py:126-133): Xc [B,q,D] → mean [B,q], cov [B,q,q]
 * (diagonal clipped to ≥ 1e-12). */
int tb_gp_predict_joint(tb_gp* gp, const void* Xc, int64_t B, int q, void* mean, void* cov);

/* ---- fused predict + acquisition tail --------------------------------------------------------
 * acq: tb_acq; param = eta (EI / log-EI) or beta (LCB).  Xc [M,D] → out [M].
 * grad (nullable): [M,D] = d out / d Xc (what tfp.math.value_and_gradient returns at
 * acquisition/optimizer.py:621-629). */
int tb_acq_eval(tb_gp* gp, int acq, double param, const void* Xc, int64_t M, void* out, void* grad);

/* generate_random_search_optimizer / _get_max_discrete_points (optimizer.py:124-150, 973-1011):
 * fused evaluation + first-max argmax.  best_value (1 scalar of the handle dtype, host),
 * best_index (host).  out may be NULL (values are then never written to HBM). */
int tb_acq_argmax(tb_gp* gp, int acq, double param, const void* Xc, int64_t M, void* out,
                  void* best_value, int64_t* best_index);

/* min_value_entropy_search.update / __init__ (entropy.py:166-191): the samples of the objective minimum y* are a
 * tf.Variable assigned in place; here they are a device array owned by the handle.  samples [S] (the reference holds them
 * as [S,1]), always double, S ≥ 1.  Required before any TB_ACQ_MES evaluation. */
int tb_acq_set_min_value_samples(tb_gp* gp, const double* samples, int S);

/* local_penalizer.__init__ / update (greedy_batch.py:272-312): the pending points and their exclusion radius
 * (μ(x_j) − η)/L and scale sqrt(var(x_j))/L, held by the handle for calls with TB_ACQ_PENALIZED.  kind: tb_penalizer;
 * pending [P,D], radius [P], scale [P]; always double, host or device pointers, P ≥ 1. */
int tb_acq_set_penalization(tb_gp* gp, int kind, const double* pending, int P, const double* radius, const double* scale);

/* gibbon_repulsion_term.__init__ / update (entropy.py:580-618): the m pending points P and the repulsion weight w
 * ((1/m)² with rescaled_repulsion, else 1), held by the handle for TB_ACQ_GIBBON_REPULSION and TB_ACQ_GIBBON.  From them the
 * handle derives W = K⁻¹k(X, P) and L_B⁻¹, L_B = chol(B + σ²I), B = predict_joint(P) with its diagonal clipped at ≥ 1e-12.
 * They follow the posterior: after tb_gp_update_posterior_cache or tb_gp_append_data they are rebuilt before the next
 * GIBBON launch, and not otherwise.  pending [m,D], always double, host or device pointer, m ≥ 1, needs a valid cache;
 * TB_ERR_NUMERIC if B + σ²I is not positive definite. */
int tb_acq_set_gibbon_repulsion(tb_gp* gp, const double* pending, int m, double weight);

/* ExpectedFeasibility.__init__ (active_learning.py:121-140): the neighbourhood parameter alpha of the two feasibility kinds,
 * held by the handle for every later TB_ACQ_FEASIBILITY_BICHON / _RANJAN launch (which refuse to run before it is set).
 * TB_ERR_INVALID for alpha <= 0 or non-finite alpha; the alpha held before then stays. */
int tb_acq_set_feasibility(tb_gp* gp, double alpha);

/* the posterior mean and its gradient, what LocalPenalization's Lipschitz estimate differentiates
 * (greedy_batch.py:207-217): Xc [M,D] → mean [M] = k(x, X) α + m and grad [M,D] = its derivative in x.  No variance: one
 * kernel launch per 65,536 points, no GEMM.  Handle dtype, host or device pointers. */
int tb_gp_mean_gradient(tb_gp* gp, const void* Xc, int64_t M, void* mean, void* grad);

/* _perform_parallel_continuous_optimization (acquisition/optimizer.py:566-697) with one ScipyOptimizerGreenlet per start
 * (:700-745, L-BFGS-B): here P independent projected L-BFGS runs advance together ON THE DEVICE — one batched fused
 * value+gradient evaluation of all active trial points per round, then one warp per run updates its curvature history,
 * line search and convergence tests (SciPy's option names: maxcor ≤ 16, maxiter, maxls, gtol on the projected gradient,
 * ftol on the relative decrease).  Maximises the acquisition `acq` inside the box.  lower, upper [D]; starts [P,D];
 * x_out [P,D], f_out [P] (maximised values), success [P] (1 = converged), nfev [P].  All arrays double / as declared
 * (the reference's SciPy side is fp64 whatever the model dtype, optimizer.py:635-639), host or device pointers. */
int tb_acq_maximize(tb_gp* gp, int acq, double param, const double* lower, const double* upper, const double* starts,
                    int64_t P, int maxcor, int maxiter, int maxls, double gtol, double ftol, double* x_out, double* f_out,
                    int32_t* success, int64_t* nfev);

/* batch_monte_carlo_expected_improvement.__call__ (function.py:1181-1186) on top of
 * BatchReparametrizationSampler.sample (models/gpflow/sampler.py:208-287):
 * Xc [B,q,D], eps [q,S] (the sampler's fixed base samples, injected) → out [B]. */
int tb_acq_batch_mc_ei(tb_gp* gp, const void* Xc, int64_t B, int q, const void* eps, int S,
                       double eta, double jitter, void* out);

/* The same value together with its gradient w.r.t. the query batches — what tfp.math.value_and_gradient
 * (acquisition/optimizer.py:621-629) differentiates when a batch function is maximised through batchify_joint
 * (:897-936): reduce_min routes to the arg-min sample, maximum(., 0) to the active ones, the Cholesky of the joint
 * covariance by its reverse-mode rule.  out [B], grad [B,q,D]. */
int tb_acq_batch_mc_ei_grad(tb_gp* gp, const void* Xc, int64_t B, int q, const void* eps, int S, double eta,
                            double jitter, void* out, void* grad);

/* batch_expected_improvement.__call__ (function.py:1747-1805): the multi-point EI of Chevalier & Ginsbourger over the
 * joint posterior of each q-batch, with q CDFs of dimension q and q² of dimension q−1 by Genz's QMC recursion
 * (MultivariateNormalCDF, acquisition/function/utils.py:109-199).  Xc [B,q,D] (handle dtype) → out [B] (handle dtype);
 * w [q−1,S] the Sobol points (double, host or device, column j contiguous as in eps: the same points serve both CDF
 * dimensions, column j of a Sobol sequence being the same in every dimension).  eta is the minimisation threshold; the
 * sign flip to the maximisation form (:1797-1803) and the hard-coded 1e-6 jitters (:1776-1783, utils.py:114) are
 * applied inside.  2 ≤ q ≤ 32 (the reference's q = 1 fails inside MultivariateNormalCDF(dim=0)); TB_ERR_INVALID also for
 * S < 1, a null pointer or no posterior cache; TB_ERR_NUMERIC if a matrix cannot be factorised. */
int tb_acq_batch_ei(tb_gp* gp, const void* Xc, int64_t B, int q, const double* w, int S, double eta, void* out);

/* The same value together with its gradient w.r.t. the query batches (what tfp.math.value_and_gradient returns under
 * batchify_joint, optimizer.py:621-629, 897-936): the reverse pass of the Genz recursion, the small Cholesky
 * factorisations and the Σ/c/R construction down to the adjoints of the joint mean and covariance, then the same
 * gradient assembly as tb_acq_batch_mc_ei_grad.  out [B], grad [B,q,D]. */
int tb_acq_batch_ei_grad(tb_gp* gp, const void* Xc, int64_t B, int q, const double* w, int S, double eta, void* out,
                         void* grad);

/* predictive_variance.acquisition (active_learning.py:98-108): exp(logdet(cov + jitter)) of the joint posterior of each
 * q-batch.  As in the reference the scalar jitter is added to EVERY entry of cov (cov + jitter 1 1^T, not cov + jitter I);
 * the log-determinant is 2 sum log diag chol.  Xc [B,q,D] → out [B]; grad (nullable) [B,q,D] = d out / d Xc (the reverse
 * pass with Sigma_bar = det(M) M^-1, M = cov + jitter 1 1^T, assembled as for tb_acq_batch_mc_ei_grad).  Handle dtype,
 * host or device pointers.  1 <= q <= 32 (the reference has no bound); TB_ERR_NUMERIC if M of a batch is not positive
 * definite. */
int tb_acq_predictive_variance(tb_gp* gp, const void* Xc, int64_t B, int q, double jitter, void* out, void* grad);

/* MultivariateNormalCDF.__call__ (acquisition/function/utils.py:109-199): P(X ≤ x) for X ~ N(mean, cov + jitter I) by
 * Genz's recursion over the S Sobol points w [Q−1,S] (column-contiguous; may be null for Q = 1).  x, mean [B,Q],
 * cov [B,Q,Q] → out [B].  fp64 only; host or device pointers.  1 ≤ Q ≤ 32, S ≥ 1; TB_ERR_NUMERIC if cov + jitter I of a
 * row is not positive definite. */
int tb_mvn_cdf(int device, const double* x, const double* mean, const double* cov, int64_t B, int Q, const double* w,
               int S, double jitter, double* out);

/* BatchReparametrizationSampler.sample (sampler.py:208-287): → samples [B,S,q]. */
int tb_gp_reparam_sample(tb_gp* gp, const void* Xc, int64_t B, int q, const void* eps, int S,
                         double jitter, void* samples);

/* model.sample over a large point set (GPflowPredictor.sample, interface.py:135-138 -> gpflow predict_f_samples: joint
 * mean / full covariance, Cholesky of cov + jitter I, mean + L z) — the call behind ExactThompsonSampler
 * (acquisition/sampler.py:85-123).  Xc [M,D] (handle dtype), z [S,M] standard-normal draws (double), out [S,M] (handle
 * dtype).  1 ≤ M ≤ 16384; the covariance is built and factorised on the device (DMMA Gram + the blocked Cholesky of the
 * cache build). */
int tb_gp_sample_joint(tb_gp* gp, const void* Xc, int64_t M, const double* z, int S, double jitter, void* out);

/* covariance_between_points_encoded (models/gpflow/models.py:188-254): posterior covariance between two point sets,
 * K12 − Kx1 (K + σ²I)⁻¹ Kx2, no clipping.  X1 [M1,D], X2 [M2,D], out [M1,M2] row-major (handle dtype); M1 + M2 ≤ 16384.
 * (The reference's leading dimensions of X1 are flattened into M1 by the caller.) */
int tb_gp_covariance_between_points(tb_gp* gp, const void* X1, int64_t M1, const void* X2, int64_t M2, void* out);

/* ---- streaming reductions over candidate scores ----------------------------------------------
 * tf.math.top_k as used by generate_initial_points (optimizer.py:321-335): values [M] →
 * top values [k] (descending, ties → lower index), indices [k].  Host or device pointers. */
int tb_topk(int device, int dtype, const void* values, int64_t M, int k, void* top_values,
            int64_t* top_indices);

/* ---- random-Fourier-feature trajectories -----------------------------------------------------
 * feature_decomposition_trajectory.__call__ (models/gpflow/sampler.py:901-936) with
 * ResampleableRandomFourierFeatureFunctions (:741-806): always fp64 (sampler.py:782). */
int tb_rff_create(tb_rff** out, int device);
int tb_rff_destroy(tb_rff* r);
/* W [F,D], b [F], lengthscales [D], theta [nb,F] (nb trajectories = batch size B). */
int tb_rff_set(tb_rff* r, const double* W, const double* b, int F, int D, const double* lengthscales,
               double variance, double mean_const);
int tb_rff_set_theta(tb_rff* r, const double* theta, int nb);
/* Xc [M,D] evaluated under all nb trajectories → out [M,nb]; ThompsonSamplerFromTrajectory
 * (acquisition/sampler.py:262-271): argmin per trajectory → min_value [nb], min_index [nb]
 * (either may be NULL). */
int tb_rff_eval(tb_rff* r, const void* Xc, int64_t M, void* out, double* min_value,
                int64_t* min_index);
/* DecoupledTrajectorySampler (models/gpflow/sampler.py:594-738) / ResampleableDecoupledFeatureFunctions (:809-855):
 * adds the canonical features  sum_j v[b][j] k(x, X_j)  to trajectory b.  X [N,D] raw training inputs (host),
 * v [nb,N] column layout [trajectory][training point] (host or device).  N = 0 switches the term off. */
int tb_rff_set_canonical(tb_rff* r, int kernel, const double* X, int64_t N, const double* v, int nb);
/* feature_decomposition_trajectory.__call__ for x [M, B, D] (models/gpflow/sampler.py:901-936): point (m, b) under
 * trajectory b only -> out [M, B]; grad (nullable) [M, B, D].  B == nb (and == the canonical weights' nb when set).
 * Values are bit for bit those of tb_rff_eval on column b.  fp64, host or device pointers. */
int tb_rff_eval_paired(tb_rff* r, const void* Xc, int64_t M, int B, void* out, void* grad);
/* tb_acq_maximize's contract for the NEGATED trajectories: starts [R, nb, D], start (i, b) maximises -f_b inside the box;
 * x_out [R, nb, D], f_out [R, nb] (= -f_b at x_out), success, nfev as tb_acq_maximize.  R * nb < 2^31. */
int tb_rff_maximize(tb_rff* r, const double* lower, const double* upper, const double* starts, int64_t R, int maxcor,
                    int maxiter, int maxls, double gtol, double ftol, double* x_out, double* f_out, int32_t* success,
                    int64_t* nfev);
/* tb_rff_maximize with one box per batch column (BatchTrustRegionBox over a TaggedMultiSearchSpace, acquisition/optimizer.py
 * round robin): lower/upper [nbox, D], start (i, b) maximises -f_b inside box b % nbox.  nbox must divide nb (TB_ERR_INVALID
 * otherwise); tb_rff_maximize is this call with nbox = 1. */
int tb_rff_maximize_boxes(tb_rff* r, const double* lower, const double* upper, int nbox, const double* starts, int64_t R,
                          int maxcor, int maxiter, int maxls, double gtol, double ftol, double* x_out, double* f_out,
                          int32_t* success, int64_t* nfev);
/* BatchTrustRegionBox with local models (rule.py:1364-1435: the base rule deep-copied per region, each region's function
 * maximised inside its region by _perform_parallel_continuous_optimization, optimizer.py:566-745), all regions in ONE device
 * L-BFGS: problem p = r * S + s of the starts [R, S, D] maximises acq[s] with param[s] under models[s] inside the box s of
 * lower / upper [S, D].  Each round evaluates every model's active problems on that model's stream, the models side by side,
 * with one host synchronise per round.  Results are bit for bit those of S tb_acq_maximize calls, model s from the starts
 * [R, s, D].  The models share one device, dtype and D, have their posterior caches built, pass tb_acq_maximize's acquisition
 * checks and are distinct handles (their min-value samples, penalty and alpha are their own).  x_out [R, S, D], f_out, success,
 * nfev [R, S] as tb_acq_maximize.  R * S < 2^31. */
int tb_acq_maximize_models(tb_gp* const* models, const int* acq, const double* param, int S, const double* lower,
                           const double* upper, const double* starts, int64_t R, int maxcor, int maxiter, int maxls, double gtol,
                           double ftol, double* x_out, double* f_out, int32_t* success, int64_t* nfev);
/* The same for ParallelContinuousThompsonSampling with local models (rule.py:1364-1435): S trajectory handles of k = nb
 * trajectories each (every r[s]->nb == k), V = k * S columns; start (i, v) of the starts [R, V, D] maximises -f of trajectory
 * v / S of r[v % S] inside box v % S of lower / upper [S, D], the round robin of a TaggedMultiSearchSpace (optimizer.py:859-890).
 * Bit for bit the results of tb_rff_maximize_boxes(r[s], box s) from the starts [R, k, D] of the columns v = j * S + s.
 * x_out [R, V, D], f_out [R, V] (= -f at x_out), success, nfev as tb_rff_maximize.  R * V < 2^31. */
int tb_rff_maximize_models(tb_rff* const* r, int S, const double* lower, const double* upper, const double* starts, int64_t R,
                           int maxcor, int maxiter, int maxls, double gtol, double ftol, double* x_out, double* f_out,
                           int32_t* success, int64_t* nfev);
/* (K(X,X) + noise I)^-1 B = Linv^T (Linv B) through the cached triangular inverse: B, out [nrhs][N] (each right-hand side contiguous);
 * the v-weights of a decoupled trajectory (sampler.py:716, gpflux compute_A_inv_b).  fp64, host or device. */
int tb_gp_kinv_apply(tb_gp* gp, const double* B, int nrhs, double* out);

/* ---- expected hypervolume improvement over a stack of GPs ---------------------------------------
 * expected_hv_improvement (acquisition/function/multi_objective.py:145-250) over L one-output models, one tb_gp per
 * objective: EHVI(x) = sum_k prod_l g_kl(mean_l(x), var_l(x)) over the K cells of the non-dominated partition.
 * tb_ehvi_create borrows the handles (they must outlive the object): 2 <= L <= 8, distinct handles with data, on one
 * device, with one dtype and one input dimension D; TB_ERR_INVALID otherwise. */
int tb_ehvi_create(tb_ehvi** out, tb_gp* const* models, int L);
int tb_ehvi_destroy(tb_ehvi* h);
/* the cells' bounds lower, upper [K, L] (fp64, host or device) as prepare_default_non_dominated_partition_bounds returns
 * them, in the objectives' minimisation orientation; K >= 1. */
int tb_ehvi_set_cells(tb_ehvi* h, const double* lower, const double* upper, int64_t K);
/* HIPPO's penalty (acquisition/function/multi_objective.py:664-758): every later evaluation, argmax and maximisation
 * returns EHVI(x) * prod_p (2/pi) atan(d_p(x)), d_p(x) = sqrt(sum_l ((mean_l(x) - pending_mean[p, l]) / sqrt(pending_var[p, l]))^2),
 * with its gradient.  pending_mean, pending_var [P, L] (fp64, host or device); P = 0 (null pointers allowed) removes the
 * penalty, which a new object does not have.  Setting the state the object already holds copies nothing and does not
 * synchronise (a device array is read back for the comparison).  TB_ERR_INVALID for P < 0, null arrays with P > 0, or a
 * negative or NaN variance; the penalty held before then stays. */
int tb_ehvi_set_penalty(tb_ehvi* h, const double* pending_mean, const double* pending_var, int P);
/* Xc [M, D] -> out [M]; grad (nullable) [M, D].  The members' dtype, host or device pointers.  TB_ERR_INVALID if the cells
 * are not set or a member's posterior cache is not built. */
int tb_ehvi_eval(tb_ehvi* h, const void* Xc, int64_t M, void* out, void* grad);
/* tb_acq_argmax's contract for EHVI: first-max index and value over Xc [M, D]; out [M] nullable. */
int tb_ehvi_argmax(tb_ehvi* h, const void* Xc, int64_t M, void* out, void* best_value, int64_t* best_index);
/* tb_acq_maximize's contract for EHVI: the device multi-start L-BFGS maximising EHVI inside the box [lower, upper] ([D]). */
int tb_ehvi_maximize(tb_ehvi* h, const double* lower, const double* upper, const double* starts, int64_t P, int maxcor,
                     int maxiter, int maxls, double gtol, double ftol, double* x_out, double* f_out, int32_t* success,
                     int64_t* nfev);

/* ---- reducers over single-query acquisitions of several GPs -----------------------------------
 * Sum / Product / MakePositive (acquisition/combination.py, function/function.py:1914-1990) over T terms, each a fused
 * single-query kind on one of n distinct borrowed handles: value = v_0 + ... + v_{T-1}, v_0 * ... * v_{T-1} (in term order,
 * as tf.add_n / tf.reduce_prod over the children) or log(1 + exp(v_0)) (T = 1).  Each distinct handle runs its predict once
 * per chunk, however many terms use it.  tb_reduce_create borrows the handles (they must outlive the object): 1 <= n <= 8,
 * distinct handles with data, on one device, with one dtype and one input dimension D; TB_ERR_INVALID otherwise. */
enum tb_reduce_op { TB_REDUCE_SUM = 0, TB_REDUCE_PRODUCT = 1, TB_REDUCE_SOFTPLUS = 2 };
int tb_reduce_create(tb_reduce** out, tb_gp* const* models, int n);
int tb_reduce_destroy(tb_reduce* h);
/* the terms of every later call: op (tb_reduce_op), 1 <= T <= 8 (T == 1 for the softplus); term t is kind acq[t] with
 * parameter param[t] on handle member[t] (0 <= member[t] < n).  The kinds are EI, log-EI, PBT, NegLCB, LCB, AEI, MES, the
 * two feasibility kinds, BALD and predictive variance; the feasibility kinds take alpha[t] > 0 (finite) as their alpha, the
 * other kinds ignore alpha[t] (alpha may be null when no term is a feasibility kind).  AEI reads its handle's noise, MES
 * its handle's min-value samples (tb_acq_set_min_value_samples) at each call.  Setting the terms the object already holds
 * does nothing.  TB_ERR_INVALID for a bad op, T, member index, kind (GIBBON, penalised and unknown kinds are refused) or
 * parameter; the terms held before then stay. */
int tb_reduce_set_terms(tb_reduce* h, int op, int T, const int* member, const int* acq, const double* param,
                        const double* alpha);
/* Xc [M, D] -> out [M]; grad (nullable) [M, D].  The members' dtype, host or device pointers.  TB_ERR_INVALID, before
 * anything is launched, if the terms are not set, a member's posterior cache is not built, or an MES term's handle has
 * no min-value samples. */
int tb_reduce_eval(tb_reduce* h, const void* Xc, int64_t M, void* out, void* grad);
/* tb_acq_argmax's contract for the reduction: first-max index and value over Xc [M, D] (NaN never wins); out [M] nullable. */
int tb_reduce_argmax(tb_reduce* h, const void* Xc, int64_t M, void* out, void* best_value, int64_t* best_index);
/* tb_acq_maximize's contract for the reduction: the device multi-start L-BFGS inside the box [lower, upper] ([D]). */
int tb_reduce_maximize(tb_reduce* h, const double* lower, const double* upper, const double* starts, int64_t P, int maxcor,
                       int maxiter, int maxls, double gtol, double ftol, double* x_out, double* f_out, int32_t* success,
                       int64_t* nfev);

/* ---- instrumentation (bench / tests) ---------------------------------------------------------
 * kernels launched by this library in this process since the last reset; device time (ms) of the
 * dominant kernel (triangular DMMA GEMM) accumulated with CUDA events on the handle's stream when
 * profiling is enabled. */
int64_t tb_launch_count(void);
void tb_launch_count_reset(void);
/* engine of the variance GEMM: 0 = native fp64 (DMMA), 1 = fp64-accurate emulation on the INT8 tensor cores
 * (Ozaki splitting, wgmma s8; same stated tolerances; N <= 16384, larger models fall back to engine 0), 2 = engine 1
 * with the number of digit products pinned to the full 21 (engine 1 drops to 15 — fp32 handles: 6 — when the a-priori error
 * estimate of the cache allows it; csrc/int8_engines.cu, csrc/ozaki5.cuh).  The
 * engine serves every path: predict / acquisition values, gradients (V = K^-1 k* as a dense digit GEMM) and the joint
 * paths (predict_joint / reparam samples / MC-qEI through the store-A epilogue). */
int tb_gp_set_engine(tb_gp* gp, int engine);
/* what the variance GEMM of this handle runs right now: int8 digit products per k-step (15 or 21; fp32 handles 6 or 10;
 * 0 = native fp64 engine) and, for the reduced modes, the a-priori estimate of max |Δvar| / σ_f² that admitted them.
 * Needs a valid cache.  Either output may be NULL. */
int tb_gp_engine_info(tb_gp* gp, int* digit_products, double* error_estimate);
/* diagnostics of the screened argmax: the fp32 bound pass's interval [lo, hi] for the posterior mean of each of M candidates
 * (Xc: [M, D] fp64; all pointers host or device).  The mean the predict path computes lies inside it; a bound that could not
 * be trusted (non-finite or overflowing coordinates) is [NaN, NaN].  Needs a valid cache. */
int tb_gp_mean_bounds(tb_gp* gp, const double* Xc, int64_t M, double* lo, double* hi);
int tb_gp_profile(tb_gp* gp, int enable);
/* the handle's CUDA stream (cudaStream_t as void*), so callers can record CUDA events on the stream the
 * kernels are launched on (torch.cuda.ExternalStream in bench.py). */
int tb_gp_stream(tb_gp* gp, void** stream);
int tb_gp_profile_read(tb_gp* gp, double* trigemm_ms, int64_t* trigemm_launches, double* flops);

#ifdef __cplusplus
}
#endif
#endif /* TRIESTE_B200_H */
