/* gpk.h — C ABI of libgpk.so: H100-native (sm_90a) GP posterior + acquisition kernels.
 *
 * This is the drop-in boundary for RoBO's hot path (SURVEY.md section 8b).  Every entry
 * point replaces a call the reference makes into george / scipy-LAPACK / scipy.stats from
 *   robo/models/gaussian_process.py          (train / nll / predict)
 *   robo/acquisition_functions/{ei,log_ei,pi,lcb}.py   (compute)
 * The reference is pure Python; its "FFI" for this path is george's Cython bridge, so the
 * binding a RoBO maintainer would add is a ctypes stub (see INTEGRATION.md and
 * robo_b200/_lib.py, which is exactly that stub).
 *
 * Conventions
 *   - plain C: pointers + sizes, no torch / numpy types.  All floating point is IEEE fp64.
 *   - host pointers are caller-owned, C-contiguous, read/written only during the call.
 *   - `*_dev` entry points take device pointers (e.g. torch.Tensor.data_ptr()) and are
 *     asynchronous on the handle's stream.
 *   - every function returns a gpk_status; nothing throws or aborts.  The Python side maps
 *     GPK_NOT_PD -> numpy.linalg.LinAlgError (caught at gaussian_process.py:120,156 and by
 *     the bare except at gaussian_process_mcmc.py:196), GPK_BAD_ARG -> ValueError,
 *     GPK_CUDA_ERROR -> RuntimeError.
 *   - one CUDA stream per handle; calls on one handle are not re-entrant.
 */
#ifndef GPK_H_
#define GPK_H_

#ifdef __cplusplus
extern "C" {
#endif

typedef struct gpk_handle gpk_handle;

typedef enum {
    GPK_OK = 0,
    GPK_NOT_PD = 1,        /* Cholesky pivot <= 0 or NaN: numpy.linalg.LinAlgError in the reference */
    GPK_BAD_ARG = 2,
    GPK_CUDA_ERROR = 3,
    GPK_NOT_FITTED = 4,
    GPK_NOT_APPLICABLE = 5, /* gpk_fit_append: preconditions not met, nothing was changed; do a full fit */
    GPK_EP_FAILED = 6      /* gpk_ep_joint_min: an EP update produced a NaN variance (the reference raises Exception,
                              robo/util/epmgp.py:204-207) */
} gpk_status;

/* stationary radial families, george names (oracle/george_oracle.py) */
typedef enum {
    GPK_MATERN52 = 0,      /* george.kernels.Matern52Kernel   */
    GPK_EXPSQUARED = 1,    /* george.kernels.ExpSquaredKernel */
    GPK_MATERN32 = 2       /* george.kernels.Matern32Kernel   */
} gpk_family;

typedef enum {
    GPK_ACQ_NONE = 0,      /* posterior moments only                              */
    GPK_ACQ_EI = 1,        /* robo/acquisition_functions/ei.py:65-78              */
    GPK_ACQ_LOG_EI = 2,    /* robo/acquisition_functions/log_ei.py:67-122         */
    GPK_ACQ_PI = 3,        /* robo/acquisition_functions/pi.py:58-63              */
    GPK_ACQ_LCB = 4        /* robo/acquisition_functions/lcb.py:62-65             */
} gpk_acq_kind;

/* posterior objectives of gpk_maximize_lbfgs (robo/util/posterior_optimization.py), minimised: */
#define GPK_OBJ_MEAN 5         /* mu(x)                                                */
#define GPK_OBJ_MEAN_STD 6     /* mu(x) + sqrt(v(x))                                   */

#define GPK_MAX_TERMS 64   /* metric entries (input dims x product factors) per kernel */

/* hyper-parameter sampling (gpk_sample_hypers): the factor of one theta lives in one SM's shared memory as a packed fp64
 * lower triangle, which bounds the training points; theta holds at most GPK_HYPER_MAX_DIM entries (noise included) */
#define GPK_HYPER_MAX_N 232
#define GPK_HYPER_MAX_DIM 96
/* the blocked hyper-parameter entry points (gpk_*_blocked): one fp64 matrix per theta in device memory, so the training
 * points are bounded by the chunk's byte budget ("hyper_batch_bytes", default GPK_HYPER_BATCH_BYTES) instead */
#define GPK_HYPER_BLOCKED_MAX_N 8192
#define GPK_HYPER_BATCH_BYTES 4294967296L

/* tasks of the multi-task factor (gpk_set_task_factor): n_tasks (n_tasks + 1) / 2 <= 36 Cholesky entries */
#define GPK_MAX_TASKS 8

/* hyper-priors the device restates (robo/priors/default_priors.py, robo/priors/env_priors.py) */
typedef enum {
    GPK_PRIOR_NONE = 0,
    GPK_PRIOR_DEFAULT = 1,     /* DefaultPrior */
    GPK_PRIOR_ENV = 2,         /* EnvPrior     */
    GPK_PRIOR_MTBO = 3         /* MTBOPrior    */
} gpk_prior_kind;

/* ---- lifetime ---------------------------------------------------------------------- */
int gpk_create(gpk_handle** h, int device);
int gpk_destroy(gpk_handle* h);
const char* gpk_last_error(gpk_handle* h);
const char* gpk_version(void);
/* key in
 *   "chunk"     candidates per scoring pass (multiple of 128); 0 = automatic [default]: the K* buffer is kept near
 *               512 MB (16384 candidates at N = 4096, 65536 at N <= 1024)
 *   "ozaki"     1 = variance contraction on the int8 tensor pipe (wgmma s8, register accumulators) through an
 *               error-free split of L^-1 and K* into 7 balanced base-256 digits each, 28 digit-pair products
 *               (gpk_ozaki.cuh); used while max |L^-1| < 64, N <= 16384 and the kernel has no environment factor
 *               (gpk_set_env_factor) or task factor (gpk_set_task_factor), otherwise the fp64 kernel runs [default;
 *               batches of >= 2048 candidates]; 0 = always fp64 DMMA.  The posterior mean never goes through the digits
 *               (fp64 K* alpha); the covariance builder writes the digits and the mean partials itself, no fp64 K*
 *               in HBM
 *   "ozpersist" 0 = one CTA per tile; 1 = one CTA per SM walks the tile list (by clusters); 3 = automatic [default]:
 *               persistent for N <= 4096, one CTA per tile above (tools/persist_threshold.py, DESIGN.md 9.5)
 *   "ozcluster" 1, 2 or 4 [default 4] = CTAs per cluster of the int8 contraction: they take adjacent candidate blocks of
 *               one row block and share its L^-1 digit slices by TMA multicast, so each CTA reads 1 / CS of them from L2.
 *               Every value gives bit-identical results
 *   "ozgrid"    >= 0: most clusters the persistent walk of the int8 contraction launches; 0 = as many as fit at once
 *               [default].  Tests and diagnostics: with "ozpersist" = 1 and "ozgrid" = 1 one cluster walks every tile in
 *               the L2-grouped, longest-first order.  Results are bit-identical for every value
 *   "depth2"    1 = trailing updates of two consecutive panels in one K = 256 contraction (odd steps; even steps update
 *               only the next-but-one block column); 0 = one K = 128 update per step (bit-identical factor);
 *               2 = automatic [default]: on for N >= 6144, where the trailing updates gate the fit
 *   "diagprof"  1 = the diagonal-block kernel records clock64() stamps per phase (gpk_get_diag_profile)
 *   "overlap"   1 = build K* of chunk i+1 on the side stream while chunk i contracts [default]
 *   "hyper_batch_bytes"  >= 1: device memory one chunk of the blocked hyper-parameter entry points (gpk_*_blocked)
 *               may take for its matrices, (ceil(n / 128) + 2) ceil(n / 128) 131072 bytes per theta and a few kB
 *               [default GPK_HYPER_BATCH_BYTES = 4 GiB: 7 thetas per chunk at n = 8192]; the results do not depend on it
 *   "meanonly"  1 = gpk_predict_mean (and the cost models of gpk_es_cost_multi) run the mean-only builder pass [default];
 *               0 = they take the mean of the full scoring pass, variance contraction included (tools/fabolas_acq_bench.py
 *               compares the two) */
int gpk_set_option(gpk_handle* h, const char* key, long value);
/* run on an existing CUDA stream (cudaStream_t passed as void*); NULL = the handle's own.  The handle's own stream has
 * the highest priority and its side stream (trailing updates, K* look-ahead) the lowest: give an external stream a high
 * priority too, or the single-CTA kernels of the Cholesky chain queue behind the side stream's tiles and the fit gets longer. */
int gpk_set_stream(gpk_handle* h, void* cuda_stream);
int gpk_synchronize(gpk_handle* h);

/* ---- model state ------------------------------------------------------------------- */
/* Training inputs as the reference hands them to george: X already scaled by
 * zero_one_normalization (gaussian_process.py:89-93), y already standardised if
 * normalize_output (:95-101).  X is (n, d) row-major. */
int gpk_set_data(gpk_handle* h, const double* X, const double* y, int n, int d);

/* Test-input scaling fused into the scoring kernels: x <- (x - lower) / (upper - lower)
 * (robo/util/normalization.py:11, applied at gaussian_process.py:276).  NULL disables. */
int gpk_set_input_bounds(gpk_handle* h, const double* lower, const double* upper, int d);

/* Output un-normalisation fused into the scoring kernels (gaussian_process.py:282-284):
 * mu <- mu * y_std + y_mean ; var <- var * y_std^2.  enabled = 0 disables. */
int gpk_set_output_transform(gpk_handle* h, int enabled, double y_mean, double y_std);

/* k(x, x') = exp(log_amp) * prod_g f( sum_{t in g} (x[axis_t] - x'[axis_t])^2 / exp(log_metric_t) )
 * Terms are listed group by group (group[] non-decreasing from 0).  One group over all
 * columns = george's axis-aligned (ARD) kernel; one group per column = the product of 1-D
 * kernels built at robo/fmin/fabolas.py:104-110.  Replaces kernel.set_parameter_vector
 * (gaussian_process.py:110,151). */
int gpk_set_kernel(gpk_handle* h, int family, double log_amp, int n_terms,
                   const int* axis, const int* group, const double* log_metric);

/* Environment factor of Fabolas (robo/fmin/fabolas.py:104-117, BayesianLinearRegressionKernel): multiplies the
 * handle's kernel by
 *     k_env(z, z') = exp(log_a) + exp(log_b) * z * z'
 * on input column `axis` (the coordinate the radial terms see: after the input-bounds scaling; for a FabolasGP the
 * basis-transformed dataset size).  This is a restatement from the Fabolas paper (arXiv:1605.07079: a Bayesian linear
 * regression in the features (1, z) with the prior covariance diag(exp(log_a), exp(log_b))) and the reference's call
 * sites; the george fork that defines the kernel is not public, so it has not been checked against that source.
 * axis = -1 removes the factor; gpk_set_kernel also removes it.  GPK_BAD_ARG for a non-finite parameter or an axis < -1;
 * an axis outside the data's width is refused by gpk_fit / gpk_kernel_matrix / the hyper sampler.  Scoring with the
 * factor always takes the fp64 contraction (the int8 split assumes 0 < k <= amp). */
int gpk_set_env_factor(gpk_handle* h, int axis, double log_a, double log_b);

/* Task factor of multi-task Bayesian optimisation (robo/fmin/mtbo.py:101, :134, george's TaskKernel(ndim, axis,
 * n_tasks)): multiplies the handle's kernel by
 *     K_t[t, t'],   K_t = L L^T,   L lower triangular n_tasks x n_tasks,   L_pq = exp(theta[p (p + 1) / 2 + q])
 * on input column `axis`, theta holding the n_tasks (n_tasks + 1) / 2 entries of L packed row by row (L00, L10, L11,
 * L20, ...).  K_t[a, b] = sum_{q <= min(a, b)} L_aq L_bq in ascending q.  This is a restatement from the paper (Swersky,
 * Snoek, Adams, NIPS 2013: a free-form positive-definite task covariance) and the reference's call sites; the george
 * fork that defines the kernel is not public, so it has not been checked against that source.  A coordinate is a task
 * only when it is an integer in [0, n_tasks): a candidate with any other value gets a NaN factor, and training inputs
 * with one are refused by gpk_fit.  axis = -1 removes the factor; gpk_set_kernel also removes it.  GPK_BAD_ARG for a
 * non-finite theta, n_tasks outside 1..GPK_MAX_TASKS, an axis < -1 or an environment factor already set (and
 * gpk_set_env_factor refuses a task factor); gpk_fit / gpk_kernel_matrix / the hyper sampler refuse an axis outside the
 * data's width, and gpk_fit refuses input bounds (the task column must reach the kernel unscaled).  Scoring with the
 * factor always takes the fp64 contraction (K_t entries may exceed 1). */
int gpk_set_task_factor(gpk_handle* h, int axis, int n_tasks, const double* theta);

/* ---- fit: K build + Cholesky + forward solve + log-det ------------------------------- */
/* Replaces george GP.compute + GP.log_likelihood (gaussian_process.py:119,155,159):
 *   K = k(X, X) + diag_add * I ; K = L L^T ; z = L^-1 (y - mean)
 *   logdet = 2 sum log L_ii ; loglik = -1/2 z^T z - 1/2 logdet - n/2 log(2 pi)
 * diag_add is the value george adds to the diagonal, yerr^2 + 1.25e-12, computed by the host
 * exactly as george does.  Returns GPK_NOT_PD where scipy.linalg.cholesky would raise. */
int gpk_fit(gpk_handle* h, double diag_add, double mean, double* logdet, double* loglik);

/* The same in two halves, for evaluating many hyper-parameter vectors at once: gpk_fit_begin only
 * enqueues the work on the handle's stream and returns; gpk_fit_end waits and returns the
 * results.  With one handle per theta (each on its own stream) the latency-bound Cholesky chains
 * of several thetas overlap on the GPU: this is how GaussianProcessMCMC.loglikelihood
 * (gaussian_process_mcmc.py:168-202) is served for a half-ensemble of emcee walkers per step. */
int gpk_fit_begin(gpk_handle* h, double diag_add, double mean);
int gpk_fit_end(gpk_handle* h, double* logdet, double* loglik);

/* Incremental refit after rows were appended (robo/models/base_model.py:30-45 `update`, and
 * robo/solver/bayesian_optimization.py:161-167 train(do_optimize=False) when hyper-parameters are frozen).
 * X (n x d) and y (n) are the full new training set; its first rows must be the ones of the last fit, the kernel
 * and diag_add unchanged.  Requires a fitted handle whose L^-1 has been built (any predict / acq call) and the new
 * rows to fall into the last 128-row block of the padded layout; otherwise returns GPK_NOT_APPLICABLE without
 * touching the model.  O(N^2): only the last block row of the factor and of its inverse is recomputed. */
int gpk_fit_append(gpk_handle* h, const double* X, const double* y, int n, int d, double diag_add, double mean,
                   double* logdet, double* loglik);

/* ---- posterior + acquisition over a candidate batch -------------------------------- */
/* Replaces george GP.predict + np.diag + clip (gaussian_process.py:276-294):
 * mu[m], var[m] (var clipped to >= DBL_EPSILON).  Xs is (m, d) row-major, raw (un-scaled). */
int gpk_predict(gpk_handle* h, const double* Xs, long m, double* mu, double* var);

/* The predictive mean alone: predict(X)[0], as the cost model of InformationGainPerUnitCost uses it
 * (robo/acquisition_functions/information_gain_per_unit_cost.py:91).  Runs the int8 path's covariance builder with its
 * digit stores compiled out and sums the per-tile shares of K* alpha in the same fixed order, alpha = L^-T z built once
 * per fit: mu is bit-identical to gpk_predict's wherever gpk_predict takes the int8 path (option "ozaki", m >= 2048),
 * and within rounding of its fp64 path elsewhere; no variance work.  Xs (m, d) raw inputs, m >= 1; mu (m).
 * GPK_NOT_FITTED before gpk_fit. */
int gpk_predict_mean(gpk_handle* h, const double* Xs, long m, double* mu);
/* the same on device pointers (d_Xs: m x d, d_mu: m doubles), asynchronous on the handle's stream */
int gpk_predict_mean_dev(gpk_handle* h, const void* d_Xs, long m, void* d_mu);

/* full_cov=True path (gaussian_process.py:280-294): cov is (m, m) row-major, every entry
 * clipped to >= DBL_EPSILON like the reference does. */
int gpk_predict_cov(gpk_handle* h, const double* Xs, long m, double* mu, double* cov);

/* The same without the clip: the raw posterior covariance K** - K* K^-1 K*^T (negative off-diagonal entries kept,
 * output transform applied).  This is what george's GP.sample_conditional draws from at gaussian_process.py:324
 * (sample_functions); only predict() clips (:290-294). */
int gpk_posterior_cov(gpk_handle* h, const double* Xs, long m, double* mu, double* cov);

/* Fused predict -> acquisition -> argmax.  out (m values) may be NULL when only the argmax
 * is wanted.  best_idx follows numpy.argmax (first maximum; NaN counts as maximum) as used at
 * robo/maximizers/random_sampling.py:50.  n_negative counts EI values < 0 (the reference
 * raises ValueError on any, ei.py:86-88).  mu/var may be NULL. */
int gpk_acq(gpk_handle* h, const double* Xs, long m, int acq_kind, double eta, double par,
            double* out, double* mu, double* var,
            double* best_val, long* best_idx, long* n_negative);

/* Device-pointer variant, asynchronous on the handle's stream.  d_Xs: (m, d) fp64 row-major
 * on the device.  d_out/d_mu/d_var (m doubles each) may be NULL.  d_best: 16 bytes
 * {double value; long long index}.  */
int gpk_acq_dev(gpk_handle* h, const void* d_Xs, long m, int acq_kind, double eta, double par,
                void* d_out, void* d_mu, void* d_var, void* d_best);

/* Predictive gradients and acquisition gradients (SURVEY.md section 8f rank 3).  The reference's
 * acquisition functions call model.predictive_gradients when derivative=True (ei.py:80-85, pi.py:65-71,
 * lcb.py:66-69) but none of its models implements it.  Xs: (m, d) raw inputs; mu, var: (m); dmu, dvar:
 * (m, d) = d mu / d x, d var / d x (chain rules of the input scaling and output transform included).
 * acq_kind = GPK_ACQ_NONE, or EI / PI / LCB to also get f (m) and df (m, d) = d acquisition / d x. */
int gpk_predict_grad(gpk_handle* h, const double* Xs, long m, int acq_kind, double eta, double par,
                     double* mu, double* var, double* dmu, double* dvar, double* f, double* df);

/* RandomSampling.maximize with the candidates generated on the device
 * (robo/maximizers/random_sampling.py:38-50; SURVEY.md section 8f rank 2).  Candidate i (global index) is
 *   i < n_uniform : lower + (upper - lower) * U[0,1)^d
 *   otherwise     : clip(incumbent + scale * N(0,1)^d, lower, upper)
 * from Philox4x32-10 keyed by (seed, i, coordinate pair): independent of chunking and of how the range
 * [first, first+count) is split over GPUs.  Returns the best candidate of the range (numpy.argmax
 * tie-breaking), its acquisition value and its GLOBAL index; no candidate or value crosses PCIe. */
int gpk_maximize_random(gpk_handle* h, unsigned long long seed, long first, long count, long n_uniform,
                        const double* lower, const double* upper, const double* incumbent, double scale,
                        int acq_kind, double eta, double par,
                        double* best_x, double* best_val, long* best_idx);
/* the same generator, candidates copied to the host (out: count x d row-major); tests and re-creating
 * the winning point on another rank */
int gpk_generate_candidates(gpk_handle* h, unsigned long long seed, long first, long count, long n_uniform, int d,
                            const double* lower, const double* upper, const double* incumbent, double scale,
                            double* out);

/* Acquisition closed forms on caller-supplied moments (host arrays), evaluated by the same
 * device function as the fused path.  Serves models that are not GPU GPs (e.g. the
 * reference's test/dummy_model.py).  No handle state is used except the device/stream. */
int gpk_acq_moments(gpk_handle* h, const double* mu, const double* var, long m, int acq_kind,
                    double eta, double par, double* out, long* n_negative);

/* Reductions over the n_models hyper-parameter samples of a GP-MCMC model; A, B are
 * (n_models, m) row-major host arrays.
 *   mode 0: out1 = mean_i A_i                      MarginalizationGPMCMC.compute (marginalization.py:115-121)
 *   mode 1: out1 = mean_i A_i, out2 = var_i(A_i) + mean_i(B_i) clipped at DBL_EPSILON
 *                                                  GaussianProcessMCMC.predict (gaussian_process_mcmc.py:235-247) */
int gpk_reduce_models(gpk_handle* h, const double* A, const double* B, int n_models, long m, int mode,
                      double* out1, double* out2);

/* One candidate batch against the n_models fitted handles of a GP-MCMC model (all on one device, same input
 * dimension), reduced over the models ON THE DEVICE: the batch goes H2D once, every model scores it on its own stream
 * (the small launches overlap), and only the reduced vectors come back.  Xs: (m, d) raw host inputs.
 *   mode 0: out1 = mean_i acq_i(x)  with eta[i] the incumbent of model i      MarginalizationGPMCMC.compute
 *           (robo/acquisition_functions/marginalization.py:115-121); best_val/best_idx = numpy.argmax of out1 (may be
 *           NULL); n_negative = EI values < 0 over all models (ei.py:86-88 raises on any)
 *   mode 1: out1 = mean_i mu_i, out2 = var_i(mu_i) + mean_i var_i clipped at DBL_EPSILON   GaussianProcessMCMC.predict
 *           (robo/models/gaussian_process_mcmc.py:235-247); acq_kind / eta / par ignored */
int gpk_acq_multi(gpk_handle* const* models, int n_models, const double* Xs, long m, int mode, int acq_kind,
                  const double* eta, double par, double* out1, double* out2, long* n_negative, double* best_val,
                  long* best_idx);

/* DifferentialEvolution.maximize (robo/maximizers/differential_evolution.py:27-51) on the device: scipy's
 * differential_evolution with strategy 'best1bin' and Latin-hypercube initialisation
 * (scipy/optimize/_differentialevolution.py) minimising the energy -acq(x), x = clip(scaled member, lower, upper),
 * acq = mean over the n_models handles (the value gpk_acq_multi mode 0 returns; one handle: gpk_acq's value), an
 * infinite energy replaced by DBL_MAX as the reference's wrapper does.  Population, trials, energies, selection and the
 * convergence test std(E) <= atol + tol |mean(E)| stay on the device; each generation is one scoring pass of pop rows
 * over all models, and only a 16-byte status record crosses PCIe per generation.
 * Two deviations from the reference:
 *   - updating='deferred' (a whole generation is scored at once) instead of scipy's default 'immediate', which is
 *     serial by construction;
 *   - the random stream is Philox4x32-10 keyed by `seed`, counter (member, generation, word, tag) with a tag disjoint
 *     from gpk_maximize_random's counters (gpk_de.cuh).  The reference never passes an rng to scipy, so its stream
 *     cannot be reproduced anyway.  Results depend on nothing but the arguments: not on chunking or n_models' order of
 *     completion.
 * The order of every rounding step, the sums of mean and std included, is documented in gpk_de.cuh.
 * pop: 5 <= pop <= 2^24 (scipy: max(5, popsize * d)).  maxiter >= 0 generations (0: score the initial population
 * only); 0 <= mut_lo <= mut_hi < 2 (dither F ~ U[mut_lo, mut_hi) per generation); 0 <= recombination <= 1;
 * lower < upper (d each); acq_kind EI ... LCB; eta[n_models]; the handles as for gpk_acq_multi.  Out: best_x (d) =
 * the scaled winner, best_energy = its energy, nit = generations run, nfev = pop * (nit + 1), n_negative = EI values
 * < 0 over all evaluations; population (pop x d unit cube, row-major, slot 0 = winner) and energies (pop) may be NULL. */
int gpk_maximize_de(gpk_handle* const* models, int n_models, unsigned long long seed, long pop, int maxiter,
                    double mut_lo, double mut_hi, double recombination, double tol, double atol,
                    const double* lower, const double* upper, int acq_kind, const double* eta, double par,
                    double* best_x, double* best_energy, int* nit, long* nfev, long* n_negative,
                    double* population, double* energies);

/* epmgp.joint_min(mu, V, with_derivatives=True) (robo/util/epmgp.py:11-250): the EPMGP approximation of p_min, the
 * probability of each of nb points to be the minimum of a Gaussian N(mu, V), on caller operands.  One CTA per point k
 * runs the EP problem of k (at most 50 sweeps, stop when sum |d| < 0.001, float32 epsilon in the message clamps), then
 * joint_min's renormalisation runs on the device (gpk_es.cuh).  2 <= nb <= 64; mu (nb), V (nb x nb row-major).
 * Out: logP (nb) = log p_min; dlogPdMu (nb x nb), dlogPdSigma (nb x nb (nb + 1) / 2: row k is the lower triangle of the
 * symmetrised derivative in row-major order), dlogPdMudMu (nb x nb x nb), sweeps (nb: EP sweeps of problem k); each of
 * these four may be NULL.  Uses its own scratch: a fitted model is left untouched, and no fit is needed.
 * GPK_EP_FAILED when an EP update yields a NaN variance; GPK_NOT_PD when IRSR is not positive definite even with
 * +1e-6 I (numpy.linalg.LinAlgError in the reference). */
int gpk_ep_joint_min(gpk_handle* h, const double* mu, const double* V, int nb, double* logP, double* dlogPdMu,
                     double* dlogPdSigma, double* dlogPdMudMu, int* sweeps);

/* InformationGain.update after the representer points are sampled (robo/acquisition_functions/information_gain.py:
 * 153-167): Mb, Vb = predict(zb, full_cov=True) on the handle (clipped like the reference), EP for p_min
 * (gpk_ep_joint_min), and U = K^-1 K(X, zb) (N x Nb, fp64, from the handle's L^-1) for the cross-covariance of the
 * candidates; everything stays on the device.  zb (nb x d raw inputs), lmb (nb, the log-probabilities of zb under the
 * sampling acquisition: GPK_BAD_ARG "lmb should not be infinite." when one is not finite, :207-211), sn2 = the model's
 * noise, W (np) the quantiles of the hallucinated observations, lower / upper (d) the acquisition's bounds.
 * logP (nb), dlogPdMu, dlogPdSigma, dlogPdMudMu (shapes as gpk_ep_joint_min) may be NULL.  2 <= nb <= 64, np >= 1. */
int gpk_es_update(gpk_handle* h, const double* zb, int nb, const double* lmb, double sn2, const double* W, int np,
                  const double* lower, const double* upper, double* logP, double* dlogPdMu, double* dlogPdSigma,
                  double* dlogPdMudMu);
/* InformationGain.compute (information_gain.py:87-125, 169-203) over m candidates Xs (m x d raw inputs): the
 * predictive variance v from the scoring pass, the covariance sigma to zb, the innovations and the entropy change dH
 * per candidate (gpk_es.cuh).  A candidate outside [lower, upper] gives DBL_EPSILON, NaN or +inf gives -DBL_MAX, -inf is
 * kept.  Each candidate is computed on its own, so the values do not depend on "chunk" or on how a batch is split.
 * GPK_BAD_ARG before gpk_es_update or after the model changed since. */
int gpk_es_compute(gpk_handle* h, const double* Xs, long m, double* out);
/* the same on device pointers (d_Xs: m x d, d_out: m doubles), asynchronous on the handle's stream */
int gpk_es_compute_dev(gpk_handle* h, const void* d_Xs, long m, void* d_out);

/* MarginalizationGPMCMC.compute over InformationGain estimators (robo/acquisition_functions/marginalization.py:115-121)
 * as one call: gpk_es_compute of every objective[i] on Xs (m x d raw inputs), each handle on its own stream, then the
 * mean over the n handles summed in index order (gpk_reduce_models mode 0, also for n = 1).  Bit-identical to the n
 * gpk_es_compute values reduced by gpk_reduce_models.  out (m) and best_val / best_idx (numpy.argmax of out) may be
 * NULL.  GPK_BAD_ARG: n < 1, m < 1, handles on different devices or with different input dimensions, a handle listed
 * twice, a handle without a current gpk_es_update (or changed since). */
int gpk_es_multi(gpk_handle* const* objective, int n, const double* Xs, long m, double* out, double* best_val,
                 long* best_idx);
/* the same on a device batch (d_Xs: m x d), asynchronous on objective[0]'s stream: d_out (m doubles) is required,
 * d_best (16 bytes {double value; long long index}) may be NULL. */
int gpk_es_multi_dev(gpk_handle* const* objective, int n, const void* d_Xs, long m, void* d_out, void* d_best);

/* The sampling-based entropy search, InformationGainMC (robo/acquisition_functions/information_gain_mc.py) with its
 * p_min estimator joint_pmin (robo/util/mc_part.py), on the device (robo_b200/csrc/gpk_esmc.cuh states every rounding
 * step and summation order).  The reference draws F ~ N(0, I) (Nf x Nb) afresh on every joint_pmin call; here F (nb x
 * nf) comes from Philox4x32-10 keyed by `seed` and Box-Muller, and one F serves an update and every candidate until the
 * next update (common random numbers): each value has the reference's marginal law, compute(x) is a deterministic
 * function of x between updates, and no value depends on its position in a batch, on "chunk" or on how a batch is split.
 * The factorisation of V + noise I climbs the reference's jitter ladder float for float (0, 1e-9, 1e-8, ..., 10000.0);
 * a failure at 10000.0 is GPK_NOT_PD (numpy.linalg.LinAlgError, mc_part.py:40-41). */

/* mc_part.joint_pmin(m, V, Nf) (mc_part.py:7-68) on caller operands: m (nb x np row-major; the reference's Mb is np = 1),
 * V (nb x nb, only its lower triangle is read), F drawn from `seed`.  pmin (nb) = count of each point as the column
 * minimum (numpy.argmin: the first index wins a tie) over the nf np columns, divided by nf np and clamped below at
 * 1e-70.  n_jitter (may be NULL): 1 when the factorisation needed jitter (the reference logs it), else 0.  Uses its own
 * scratch; no fit is needed.  1 <= nb <= 64, np >= 1, nf >= 1, nf np < 2^31. */
int gpk_mc_pmin(gpk_handle* h, const double* m, int np, const double* V, int nb, int nf, unsigned long long seed,
                double* pmin, int* n_jitter);
/* The draws F (nb x nf row-major) that `seed` gives gpk_mc_pmin and gpk_esmc_update; F[k][f] depends on (seed, k, f)
 * only.  nb >= 1, nf >= 1. */
int gpk_mc_draws(gpk_handle* h, unsigned long long seed, int nb, int nf, double* F);
/* InformationGainMC.update after the representer points are sampled (information_gain_mc.py:103-121): Mb, Vb =
 * predict(zb, full_cov=True) (clipped like the reference), F from `seed`, pmin = joint_pmin(Mb as (nb, 1), Vb, nf),
 * logP = log(pmin), H = -sum_i exp(logP_i) (logP_i + lmb_i), the scaled zb and U = K^-1 K(X, zb) as gpk_es_update builds
 * them; everything the candidates need stays on the device.  zb (nb x d raw inputs), lmb (nb: GPK_BAD_ARG "lmb should
 * not be infinite." when one is not finite), sn2 the model's noise, W (np) the innovation quantiles.  logP and pmin (nb)
 * may be NULL.  2 <= nb <= 64, np >= 1, nf >= 1, nf np < 2^31.  GPK_NOT_PD as for gpk_mc_pmin.  After it, gpk_es_compute
 * and the other consumers of gpk_es_update are GPK_BAD_ARG until the next gpk_es_update, and the reverse holds for the
 * gpk_esmc_* consumers; gpk_es_moments, gpk_es_dims and gpk_es_get_u serve either update. */
int gpk_esmc_update(gpk_handle* h, const double* zb, int nb, const double* lmb, double sn2, const double* W, int np,
                    int nf, unsigned long long seed, double* logP, double* pmin);
/* InformationGainMC.compute (information_gain_mc.py:67-79, 123-156) over m candidates Xs (m x d raw inputs), one value
 * each: with v the predictive variance (noise included), iv = 1 / (v - sn2), sigma the clipped covariance to zb (as
 * gpk_es_compute), nc_a = sigma_a iv: Mb_new[a][p] = Mb_a + nc_a sqrt(v + 1e-10) W_p, Vb_new[a][b] = Vb[a][b] -
 * nc_a sigma_b, new = joint_pmin(Mb_new, Vb_new, nf) on the update's F, and
 *   value = sum_i new_i (log new_i + lmb_i) + H   (larger is more information; NaN or +inf -> -DBL_MAX).
 * There is no bounds test (the reference has none).  GPK_BAD_ARG before gpk_esmc_update, after the model changed since,
 * or after a gpk_es_update; GPK_NOT_PD when a candidate's factorisation fails at every rung (on the _dev variant that
 * candidate's value is NaN and the status is not read back). */
int gpk_esmc_compute(gpk_handle* h, const double* Xs, long m, double* out);
/* the same on device pointers (d_Xs: m x d, d_out: m doubles), asynchronous on the handle's stream */
int gpk_esmc_compute_dev(gpk_handle* h, const void* d_Xs, long m, void* d_out);
/* MarginalizationGPMCMC.compute over InformationGainMC estimators as one call: gpk_esmc_compute of every objective[i],
 * each handle on its own stream, then the mean over the n handles (gpk_reduce_models mode 0, also for n = 1); bit-identical
 * to the n gpk_esmc_compute values reduced by gpk_reduce_models.  Arguments and errors as for gpk_es_multi, with
 * gpk_esmc_update in place of gpk_es_update, and GPK_NOT_PD as for gpk_esmc_compute. */
int gpk_esmc_multi(gpk_handle* const* objective, int n, const double* Xs, long m, double* out, double* best_val,
                   long* best_idx);
int gpk_esmc_multi_dev(gpk_handle* const* objective, int n, const void* d_Xs, long m, void* d_out, void* d_best);
/* gpk_maximize_de_es over the sampling-based entropy change: -(gpk_esmc_multi's value of the member over objective[0 ..
 * n-1]); n = 1: -(gpk_esmc_compute's value), no reduction.  Arguments and outputs as for gpk_maximize_de_es; GPK_NOT_PD
 * as for gpk_esmc_compute (checked after every generation). */
int gpk_maximize_de_esmc(gpk_handle* const* objective, int n, unsigned long long seed, long pop, int maxiter,
                         double mut_lo, double mut_hi, double recombination, double tol, double atol,
                         const double* lower, const double* upper, double* best_x, double* best_energy, int* nit,
                         long* nfev, double* population, double* energies);
/* Diagnostics of the current gpk_esmc_update: its draws F (nb x nf row-major), and its Mb (nb) and Vb (nb x nb), as a
 * host restatement needs them; GPK_BAD_ARG as for gpk_esmc_compute. */
int gpk_esmc_get_draws(gpk_handle* h, double* F);
int gpk_esmc_get_state(gpk_handle* h, double* Mb, double* Vb);
/* factorisations that needed jitter in the handle's last host-synchronised p_min call (gpk_mc_pmin, gpk_esmc_update,
 * gpk_esmc_compute; for gpk_esmc_multi and gpk_maximize_de_esmc: on objective[0], over all models, a DE run counted
 * from its start) */
int gpk_esmc_last_jitter(gpk_handle* h, long* n_jitter);

/* maps of the last input column of Fabolas models (robo/fmin/fabolas.py:96-102) and MTBO models
 * (robo/models/mtbo_gp.py:12-15) */
typedef enum {
    GPK_BASIS_S = 0,           /* basis(s) = s          (the Fabolas cost model)      */
    GPK_BASIS_ONE_MINUS_S_SQ = 1,  /* basis(s) = (1 - s)^2  (the Fabolas objective model) */
    GPK_BASIS_TASK = 2         /* basis(s) = rint(s)    (MTBO: the task index, half to even as np.rint) */
} gpk_basis;

/* InformationGainPerUnitCost.compute (robo/acquisition_functions/information_gain_per_unit_cost.py:67-106) over n
 * (objective, cost) pairs of Fabolas models, averaged as MarginalizationGPMCMC.compute does (marginalization.py:115-121):
 *   out[c] = mean_i dh_i(x_c) / (exp(mu_i(x_c)) + overhead)
 * Xs (m x d) raw candidates: d - 1 configuration columns and the environment column last.  On the device the batch is
 * mapped as FabolasGP.normalize maps it (fabolas_gp.py:122-126): configuration columns to (x - lower) / (upper - lower),
 * the environment column through the family's basis (basis_objective / basis_cost, gpk_basis), bit-identical to numpy.
 * dh_i is gpk_es_compute of objective[i] on the transformed batch, except that its bounds test sees the RAW candidate
 * against the [lower, upper] given to gpk_es_update (DBL_EPSILON outside, NaN / +inf -> -DBL_MAX); mu_i is
 * gpk_predict_mean of cost[i] on the transformed batch.  -DBL_MAX / c overflows to -inf for c < 1, as in numpy.  The mean
 * over pairs is summed in index order (gpk_reduce_models mode 0); n = 1 returns the ratio itself.  Every handle runs on
 * its own stream; the values do not depend on "chunk", on stream timing or on whether the batch came from the host.
 * lower / upper (n_bounds = d - 1 entries each): the configuration bounds of the models' transform.  out (m) and best_val / best_idx
 * (numpy.argmax of out) may be NULL.  GPK_BAD_ARG: n < 1, m < 1, a basis code out of range, lower >= upper, handles on
 * different devices or with different input dimensions, a handle listed twice (objective and cost lists together), an
 * objective handle without a current gpk_es_update (or changed since). */
int gpk_es_cost_multi(gpk_handle* const* objective, gpk_handle* const* cost, int n, const double* Xs, long m,
                      const double* lower, const double* upper, int n_bounds, int basis_objective, int basis_cost,
                      double overhead,
                      double* out, double* best_val, long* best_idx);
/* the same on a device batch (d_Xs: m x d), asynchronous on objective[0]'s stream: d_out (m doubles) is required,
 * d_best (16 bytes {double value; long long index}) may be NULL.  lower / upper are host arrays. */
int gpk_es_cost_multi_dev(gpk_handle* const* objective, gpk_handle* const* cost, int n, const void* d_Xs, long m,
                          const double* lower, const double* upper, int n_bounds, int basis_objective, int basis_cost,
                          double overhead,
                          void* d_out, void* d_best);
/* RandomSampling.maximize of that acquisition (robo/maximizers/random_sampling.py:38-50) on one GPU: count candidates
 * from gpk_generate_candidates's Philox stream in [box_lower, box_upper] (d each; the first n_uniform uniform, the rest
 * clip(incumbent + scale N(0, 1)^d)), scored by gpk_es_cost_multi; only the winner (best_x, d), its value and its index
 * cross PCIe.  The arguments otherwise as for gpk_es_cost_multi; GPK_BAD_ARG when any objective or cost handle has a
 * multi-rank communicator. */
int gpk_maximize_random_es_cost(gpk_handle* const* objective, gpk_handle* const* cost, int n, unsigned long long seed,
                                long count, long n_uniform, const double* box_lower, const double* box_upper,
                                const double* incumbent, double scale, const double* lower, const double* upper,
                                int n_bounds, int basis_objective, int basis_cost, double overhead, double* best_x, double* best_val,
                                long* best_idx);

/* gpk_maximize_de over the entropy change: the same evolution, kernels and Philox stream, with the same two deviations
 * from the reference (updating='deferred'; the counter-based Philox stream keyed by `seed`), minimising
 *   gpk_maximize_de_es:      -(gpk_es_multi's value of the member over objective[0 .. n-1]); n = 1: -(gpk_es_compute's
 *                            value), no reduction;
 *   gpk_maximize_de_es_cost: -(gpk_es_cost_multi's value of the member over the (objective[i], cost[i]) pairs); the
 *                            members live in the extended box lower / upper (d each, the environment column last) and
 *                            are scored raw; cfg_lower / cfg_upper (n_bounds = d - 1), the basis codes and the overhead
 *                            as for gpk_es_cost_multi.
 * pop, maxiter, mut_lo / mut_hi, recombination, tol, atol, lower / upper and the outputs as for gpk_maximize_de (there is
 * no n_negative).  GPK_BAD_ARG as for gpk_maximize_de and gpk_es_multi / gpk_es_cost_multi, and when a handle has a
 * multi-rank communicator: both run on one GPU. */
int gpk_maximize_de_es(gpk_handle* const* objective, int n, unsigned long long seed, long pop, int maxiter,
                       double mut_lo, double mut_hi, double recombination, double tol, double atol,
                       const double* lower, const double* upper, double* best_x, double* best_energy, int* nit,
                       long* nfev, double* population, double* energies);
int gpk_maximize_de_es_cost(gpk_handle* const* objective, gpk_handle* const* cost, int n, unsigned long long seed,
                            long pop, int maxiter, double mut_lo, double mut_hi, double recombination, double tol,
                            double atol, const double* lower, const double* upper, const double* cfg_lower,
                            const double* cfg_upper, int n_bounds, int basis_objective, int basis_cost, double overhead,
                            double* best_x, double* best_energy, int* nit, long* nfev, double* population,
                            double* energies);

/* SciPyOptimizer.maximize (robo/maximizers/scipy_optimizer.py) and posterior_mean(_plus_std)_optimization
 * (robo/util/posterior_optimization.py) on the device: multi-start bounded L-BFGS, the n_starts starts run
 * independently and in lockstep.  Each round scores, for every start still running, its trial point and the d
 * forward-difference neighbours of it in one batched pass (n_active (d + 1) rows); the iteration (free set, two-loop
 * recursion over the last maxcor pairs, projected Armijo backtracking, the stopping tests) runs in one warp per start,
 * and only a 16-byte status record crosses PCIe per round.  The energy minimised is
 *   acquisitions and information gain: -value of the row, x clipped into the box (scipy_optimizer.py:39-49);
 *   GPK_OBJ_MEAN: mu(x); GPK_OBJ_MEAN_STD: mu(x) + sqrt(v(x)) (the mixture moments of gpk_acq_multi mode 1);
 * a value that is not finite becomes DBL_MAX.  The gradient is scipy's 2-point forward difference with the relative
 * step sqrt(DBL_EPSILON) max(1, |x_j|), turned inwards at a bound; there is no analytic gradient in the loop (the
 * reference's with_gradients=True calls predictive_gradients, which no reference model has).
 * Deviation from the reference: this is projected L-BFGS (steepest descent on the free set through the two-loop
 * recursion, projected backtracking from alpha0 = min(1, 1 / ||d||) on the first iteration and 1 afterwards, at most 20
 * halvings), not L-BFGS-B's Cauchy point, subspace minimisation and More-Thuente line search.  Every rounding step is
 * fixed (gpk_lbfgs.cuh states the algorithm and the order), so a host model can restate a run bit for bit.
 * Stopping per start, scipy's tests and defaults: (f_k - f_k+1) / max(|f_k|, |f_k+1|, 1) <= ftol (2.220446049250313e-09),
 * ||P(x - g) - x||_inf <= pgtol (1e-5), nit >= maxiter (15000), nfev >= maxfun (15000 rows scored for the start).
 * x0 (n_starts x d) finite starts, clipped into [lower, upper] before the first round; 1 <= n_starts <= 2^20;
 * 1 <= maxcor <= 32 (scipy: 10).  Out per start: x_out (n_starts x d) the last accepted iterate, energy its energy, nit
 * accepted steps, nfev rows scored, status (gpk_lb_status); energy, nit, nfev and status may be NULL.  n_negative:
 * EI values < 0 over all rows.  GPK_BAD_ARG: d > GPK_LB_MAX_D, maxcor out of range, lower >= upper, a start that is
 * not finite, a handle with a multi-rank communicator, and as for gpk_acq_multi / gpk_es_multi / gpk_es_cost_multi. */
#define GPK_LB_MAX_D 64
typedef enum {
    GPK_LB_FTOL = 0,           /* relative reduction of f <= ftol (scipy: CONVERGENCE, success)        */
    GPK_LB_PGTOL = 1,          /* projected gradient <= pgtol (scipy: CONVERGENCE, success)            */
    GPK_LB_MAXITER = 2,        /* nit reached maxiter (scipy status 1)                                 */
    GPK_LB_MAXFUN = 3,         /* nfev reached maxfun (scipy status 1)                                 */
    GPK_LB_ABNORMAL = 4,       /* no sufficient decrease in 21 trials (ABNORMAL_TERMINATION_IN_LNSRCH) */
    GPK_LB_INVALID = 5         /* the start's energy is DBL_MAX: stopped at once                       */
} gpk_lb_status;
/* acq_kind: GPK_ACQ_EI ... GPK_ACQ_LCB over the mean of the n_models handles (one handle: gpk_acq's value; eta[n_models]
 * and par as for gpk_acq_multi), or GPK_OBJ_MEAN / GPK_OBJ_MEAN_STD (eta and par ignored). */
int gpk_maximize_lbfgs(gpk_handle* const* models, int n_models, int acq_kind, const double* eta, double par,
                       long n_starts, const double* x0, const double* lower, const double* upper, int maxcor,
                       int maxiter, long maxfun, double ftol, double pgtol, double* x_out, double* energy, int* nit,
                       long* nfev, int* status, long* n_negative);
/* -(gpk_es_multi's value over objective[0 .. n-1]); n = 1: -(gpk_es_compute's value) */
int gpk_maximize_lbfgs_es(gpk_handle* const* objective, int n, long n_starts, const double* x0, const double* lower,
                          const double* upper, int maxcor, int maxiter, long maxfun, double ftol, double pgtol,
                          double* x_out, double* energy, int* nit, long* nfev, int* status);
/* -(gpk_es_cost_multi's value over the (objective[i], cost[i]) pairs) in the extended box lower / upper (d each);
 * cfg_lower / cfg_upper (n_bounds = d - 1), the basis codes and the overhead as for gpk_es_cost_multi */
int gpk_maximize_lbfgs_es_cost(gpk_handle* const* objective, gpk_handle* const* cost, int n, long n_starts,
                               const double* x0, const double* lower, const double* upper, const double* cfg_lower,
                               const double* cfg_upper, int n_bounds, int basis_objective, int basis_cost,
                               double overhead, int maxcor, int maxiter, long maxfun, double ftol, double pgtol,
                               double* x_out, double* energy, int* nit, long* nfev, int* status);

/* CMAES.maximize (robo/maximizers/cmaes.py:50-81) on the device: cma.fmin(obj_func, x0, sigma0, restarts, bounds,
 * maxfevals) minimising the energy e = -acq(x) of the reference's obj_func (cmaes.py:66-68), without the `cma` package.
 * The standard (mu/mu_w, lambda)-CMA-ES of Hansen's tutorial ("The CMA Evolution Strategy: A Tutorial", 2016, Table 1
 * defaults, positive weights only): every generation samples lambda members from N(m, sigma^2 C), scores them in one
 * batched pass, ranks them, updates m, sigma, the paths p_sigma / p_c and C, and eigendecomposes C (parallel cyclic
 * Jacobi) when purecma's lazy rule asks for it; all of it stays on the device and only a 24-byte status record crosses
 * PCIe per generation.  robo_b200/csrc/gpk_cmaes.cuh states every step, the Philox counter layout and every rounding.
 * Bounds go through cma's BoundTransform, BoxConstraintsLinQuadTransformation, restated per coordinate with
 *   a_l = min((u - l) / 2, (1 + |l|) / 20),  a_u = min((u - l) / 2, (1 + |u|) / 20):
 * shift periodically into [l - a_l, u + a_u] (period 2 (u - l + a_l + a_u)) when farther out than a_l + (u - l) / 2
 * beyond l - a_l (a_u likewise at the top), mirror at u + a_u and l - a_l, then T(x) = l + (x - (l - a_l))^2 / (4 a_l)
 * on [l - a_l, l + a_l), the identity up to u - a_u and u - (x - (u + a_u))^2 / (4 a_u) above.  The distribution lives
 * in genotype space, scoring sees the phenotype T(x), and the result is the best phenotype seen (an earlier generation,
 * then the lower index, win ties).  The start mean is the genotype of x0: l - a_l + 2 sqrt(a_l (x0 - l)) near l, the
 * identity inside, u + a_u - 2 sqrt(a_u (u - x0)) near u.
 * Stop tests after every generation, the first that holds: maxfevals (evaluations over all runs >= n_func_evals, so the
 * overshoot is below lambda), tolfun 1e-11 (the range of this generation's energies and of the best energies of the
 * last 10 + ceil(30 d / lambda) generations, once that many exist; NaN ignored), tolx 1e-11 (sigma max_j max(|p_c,j|,
 * sqrt(C_jj))), conditioncov 1e14 (the ratio of the largest to the smallest eigenvalue of C), numerical (sigma, m, C or
 * an eigenvalue not finite, or sigma or an eigenvalue <= 0).  IPOP restarts (cma.fmin's incpopsize = 2): run r has
 * lambda_0 2^r members and its own constants, and starts again from the genotype of x0 and sigma0; the budget is
 * shared, and a run that stops on maxfevals ends the restarts.
 * `cma` itself is not restated bit for bit, only in law: the Philox stream replaces numpy's, and these parts of recent
 * `cma` versions are not restated: active CMA (negative recombination weights, on by default there), the resampling of
 * members whose energy is NaN (here a NaN energy ranks last), and the noeffectaxis / noeffectcoord / tolstagnation /
 * tolupsigma stops.
 * consts: (restarts + 1) rows of GPK_CMA_NCONST doubles, one per run, laid out as GPK_CMA_C_* (the constants of
 * robo_b200._lib.cmaes_constants, computed on the host so that no log runs on the device); weights w_0 .. w_mu-1 at
 * GPK_CMA_C_W.  d (the handles' input dimension) 2 .. GPK_CMA_MAX_D; lower < upper and x0 inside [lower, upper] (d each,
 * x0 finite); sigma0 > 0; n_func_evals >= 1; 0 <= restarts; every run's lambda 2 .. GPK_CMA_MAX_LAMBDA, mu = lambda / 2
 * (rounded down), history length <= GPK_CMA_HIST and flat index < lambda; otherwise GPK_BAD_ARG.
 * Out (gpk_cmaes_result; best_x required, every other pointer may be NULL): best_x (d) and best_energy (NaN when no
 * finite energy was seen), nfev_total; per run (restarts + 1 each; runs not started give 0, 0, GPK_CMA_RUNNING) nit
 * generations, nfev evaluations and stop (gpk_cmaes_stop); the last run's final m (genotype, d), sigma, p_sigma (d),
 * p_c (d) and C (d x d). */
#define GPK_CMA_MAX_D 64
#define GPK_CMA_MAX_LAMBDA 2048          /* covers restarts doublings: lambda_0 2^restarts <= this */
#define GPK_CMA_HIST 160                 /* longest tolfun history: 10 + ceil(30 d / lambda) <= 130 for 2 <= d <= 64 */
#define GPK_CMA_C_LAMBDA 0
#define GPK_CMA_C_MU 1
#define GPK_CMA_C_MUEFF 2
#define GPK_CMA_C_CS 3                   /* c_sigma */
#define GPK_CMA_C_DS 4                   /* d_sigma */
#define GPK_CMA_C_CC 5
#define GPK_CMA_C_C1 6
#define GPK_CMA_C_CMU 7
#define GPK_CMA_C_CHI 8                  /* E||N(0, I)|| = sqrt(d) (1 - 1 / (4 d) + 1 / (21 d^2)) */
#define GPK_CMA_C_HIST 9                 /* tolfun history length 10 + ceil(30 d / lambda) */
#define GPK_CMA_C_EIG 10                 /* lambda / ((c1 + cmu) d 10): evaluations between eigendecompositions */
#define GPK_CMA_C_FLAT 11                /* ceil(0.7 lambda) - 1: the rank of the flat-fitness test */
#define GPK_CMA_C_OMCS 12                /* 1 - c_sigma */
#define GPK_CMA_C_CPS 13                 /* sqrt(c_sigma (2 - c_sigma) mueff) */
#define GPK_CMA_C_OMCC 14                /* 1 - c_c */
#define GPK_CMA_C_CCC 15                 /* sqrt(c_c (2 - c_c) mueff) */
#define GPK_CMA_C_CCD 16                 /* c_c (2 - c_c) */
#define GPK_CMA_C_A0 17                  /* 1 - c1 - cmu */
#define GPK_CMA_C_HTH 18                 /* (1.4 + 2 / (d + 1)) chi: the h_sigma threshold */
#define GPK_CMA_C_CSDS 19                /* c_sigma / d_sigma */
#define GPK_CMA_C_W 20
#define GPK_CMA_NCONST (GPK_CMA_C_W + GPK_CMA_MAX_LAMBDA / 2)
typedef enum {
    GPK_CMA_RUNNING = 0,       /* not stopped (a run that was never started reports this too) */
    GPK_CMA_MAXFEVALS = 1,
    GPK_CMA_TOLFUN = 2,
    GPK_CMA_TOLX = 3,
    GPK_CMA_CONDITIONCOV = 4,
    GPK_CMA_NUMERICAL = 5
} gpk_cmaes_stop;
typedef struct {
    double* best_x;
    double* best_energy;
    long* nfev_total;
    int* nit;
    long* nfev;
    int* stop;
    double* m;
    double* sigma;
    double* ps;
    double* pc;
    double* C;
} gpk_cmaes_result;
/* EI / LogEI / PI / LCB over the mean of the n_models handles (one handle: gpk_acq's value; eta[n_models] and par as
 * for gpk_acq_multi); n_negative: EI values < 0 over all evaluations (ei.py:86-88 raises on them). */
int gpk_maximize_cmaes(gpk_handle* const* models, int n_models, int acq_kind, const double* eta, double par,
                       unsigned long long seed, const double* x0, double sigma0, const double* lower,
                       const double* upper, long n_func_evals, int restarts, const double* consts,
                       gpk_cmaes_result* out, long* n_negative);
/* -(gpk_es_multi's value over objective[0 .. n-1]); n = 1: -(gpk_es_compute's value).  One GPU. */
int gpk_maximize_cmaes_es(gpk_handle* const* objective, int n, unsigned long long seed, const double* x0, double sigma0,
                          const double* lower, const double* upper, long n_func_evals, int restarts,
                          const double* consts, gpk_cmaes_result* out);
/* -(gpk_esmc_multi's value); GPK_NOT_PD as for gpk_esmc_compute (checked after every generation).  One GPU. */
int gpk_maximize_cmaes_esmc(gpk_handle* const* objective, int n, unsigned long long seed, const double* x0,
                            double sigma0, const double* lower, const double* upper, long n_func_evals, int restarts,
                            const double* consts, gpk_cmaes_result* out);
/* -(gpk_es_cost_multi's value over the (objective[i], cost[i]) pairs) in the extended box lower / upper (d each);
 * cfg_lower / cfg_upper (n_bounds = d - 1), the basis codes and the overhead as for gpk_es_cost_multi.  One GPU. */
int gpk_maximize_cmaes_es_cost(gpk_handle* const* objective, gpk_handle* const* cost, int n, unsigned long long seed,
                               const double* x0, double sigma0, const double* lower, const double* upper,
                               long n_func_evals, int restarts, const double* consts, const double* cfg_lower,
                               const double* cfg_upper, int n_bounds, int basis_objective, int basis_cost,
                               double overhead, gpk_cmaes_result* out);
/* The standard normals gpk_maximize_cmaes* draw in generations g0 .. g1 - 1 of run `run` with `lambda` members in
 * dimension d: out ((g1 - g0) x lambda x d, row-major); z depends on (seed, run, g, member, coordinate) only.
 * 0 <= run < 256, 0 <= g0 < g1, 1 <= lambda <= GPK_CMA_MAX_LAMBDA, 1 <= d <= GPK_CMA_MAX_D. */
int gpk_cmaes_draws(gpk_handle* h, unsigned long long seed, int run, int g0, int g1, int lambda, int d, double* out);

/* Direct.maximize (robo/maximizers/direct.py:56-85) on the device: DIRECT.solve(obj_func, l, u, maxT = n_iters,
 * maxf = n_func_evals) minimising the energy e = -acq(x) of the reference's _direct_acquisition_fkt_wrapper
 * (direct.py:50-54), without the `DIRECT` package.  Jones' original DIRECT (algmethod = 0, eps = 1e-4) as Gablonsky's
 * DIRECT 2.0.4 runs it: every iteration chooses its potentially optimal rectangles and writes the points it samples
 * (c +- delta e_i over each chosen rectangle's longest sides, mapped to the box as (c + l / (u - l)) (u - l)) into one
 * row buffer in one CTA, scores them in one batched pass, and divides, inserts and updates the incumbent in one CTA;
 * only a 24-byte status record crosses PCIe per iteration.  robo_b200/csrc/gpk_direct.cuh states every step.
 * The level of a rectangle is Gablonsky's n k + j (k: its fewest trisections, j: its sides trisected k + 1 times), of
 * size 0.5 sqrt(n - j + j / 9) / 3^k; one energy-sorted list per level.  Selection: the head of each level on the
 * lower-right hull passing Jones' test f - K d <= minf - 1e-4 |minf|, then every rectangle within 1e-13 of a chosen
 * head at its level.  The rules follow scipy.optimize.direct (scipy's C translation of the same code), the one
 * executable form of it available: a head whose lower slope bound exceeds its upper one is kept without Jones' test.
 * Stop tests after every iteration, the first that holds: a rectangle at level >= GPK_DIRECT_MAXDEEP - 1 was chosen
 * (MAXDEEP_HIT; the chosen ones before it are divided), more than GPK_DIRECT_MAXDIV rectangles were chosen
 * (MAXDIV_HIT; nothing sampled), (minf + 1e100) 100 / 1e100 <= 0.01 (the package's fglobal = -1e100, fglper = 0.01),
 * nfev >= n_func_evals (so the last iteration overshoots); and the run ends without sampling when iteration n_iters
 * would begin (iterations 2 .. n_iters - 1 sample, the first one being the root's division; nit = max(n_iters, 2)
 * then, as scipy counts).  The result x is the package's
 * c (u - l) + (l / (u - l)) (u - l) of the best centre, which can differ from the scored row in the last bit.
 * Non-finite energies: NaN is stored as +inf; +inf and -inf are kept (-inf ends the run on the fglobal test).
 * Not restated: the package's stdout report and log file, its hidden-constraint flag (the reference's wrapper
 * always returns 0), DIRECT-L (algmethod = 1) and its other options.
 * d (the handles' input dimension) 1 .. GPK_DIRECT_MAX_D; lower < upper (d each, finite); n_func_evals >= 1;
 * n_iters >= 1; (2 d + 1) max(n_func_evals, 2 d + 1) <= GPK_DIRECT_MAX_RECTS (the store: every iteration starts
 * below the budget or at the 2 d + 1 initial points and adds at most 2 d rows per stored rectangle); otherwise
 * GPK_BAD_ARG.  Device memory: that many rectangles of d centre doubles and d ints, and as many rows of d doubles.
 * Out (gpk_direct_result; best_x required, every other pointer may be NULL): best_x (d), best_energy, nit, nfev, stop
 * (gpk_direct_stop), rows: the rows sampled by iterations 2 .. nit (nit - 1 of them; nit - 2 when the run stops on
 * n_iters; n_iters - 1 entries reserved by the caller). */
#define GPK_DIRECT_MAX_D 64
#define GPK_DIRECT_MAXDEEP 600
#define GPK_DIRECT_MAXDIV 5000
#define GPK_DIRECT_MAX_RECTS (1L << 22)
typedef enum {
    GPK_DIRECT_RUNNING = 0,
    GPK_DIRECT_MAXF = 1,
    GPK_DIRECT_MAXT = 2,
    GPK_DIRECT_FGLOBAL_HIT = 3,
    GPK_DIRECT_MAXDEEP_HIT = 4,
    GPK_DIRECT_MAXDIV_HIT = 5
} gpk_direct_stop;
typedef struct {
    double* best_x;
    double* best_energy;
    int* nit;
    long* nfev;
    int* stop;
    long* rows;
} gpk_direct_result;
/* EI / LogEI / PI / LCB over the mean of the n_models handles (eta[n_models] and par as for gpk_acq_multi);
 * n_negative: EI values < 0 over all evaluations (ei.py:86-88 raises on them). */
int gpk_maximize_direct(gpk_handle* const* models, int n_models, int acq_kind, const double* eta, double par,
                        const double* lower, const double* upper, long n_func_evals, int n_iters,
                        gpk_direct_result* out, long* n_negative);
/* -(gpk_es_multi's value over objective[0 .. n-1]); n = 1: -(gpk_es_compute's value).  One GPU. */
int gpk_maximize_direct_es(gpk_handle* const* objective, int n, const double* lower, const double* upper,
                           long n_func_evals, int n_iters, gpk_direct_result* out);
/* -(gpk_esmc_multi's value); GPK_NOT_PD as for gpk_esmc_compute (checked after every pass).  One GPU. */
int gpk_maximize_direct_esmc(gpk_handle* const* objective, int n, const double* lower, const double* upper,
                             long n_func_evals, int n_iters, gpk_direct_result* out);
/* -(gpk_es_cost_multi's value over the (objective[i], cost[i]) pairs) in the extended box lower / upper (d each);
 * cfg_lower / cfg_upper (n_bounds = d - 1), the basis codes and the overhead as for gpk_es_cost_multi.  One GPU. */
int gpk_maximize_direct_es_cost(gpk_handle* const* objective, gpk_handle* const* cost, int n, const double* lower,
                                const double* upper, long n_func_evals, int n_iters, const double* cfg_lower,
                                const double* cfg_upper, int n_bounds, int basis_objective, int basis_cost,
                                double overhead, gpk_direct_result* out);

/* The representer points of n entropy-search estimators in one call: the emcee 2.x stretch move (a = 2) of
 * robo_b200/util/ensemble_sampler.py, replacing the host loops of information_gain.py:68-81 and
 * information_gain_per_unit_cost.py:152-172.  Estimator i walks nb walkers of dimension dw on models[i], seeded by
 * seeds[i] alone (Philox4x32-10; the counter layout and every rounding step are in robo_b200/csrc/gpk_rs.cuh): walkers
 * start uniformly in [lower, upper] (dw each), each half of the ensemble proposes in turn, and each model scores its own
 * half-batch of nb / 2 rows on its own stream with the closed form acq_kind (EI / LogEI / PI / LCB, eta[i], par), as
 * gpk_acq would.  The log-density is -inf outside [lower, upper] and where the acquisition is NaN.
 *   fabolas = 0: dw = d, the walker is the scored row.
 *   fabolas = 1: dw = d - 1, the scored row is [walker, env_value] mapped as FabolasGP.normalize maps it
 *                (cfg_lower / cfg_upper: d - 1 entries, basis: gpk_basis), bit-identical to numpy.
 * A run is `steps` steps; an estimator whose final log-probabilities are not all finite runs again (run index + 1) up to
 * max_runs runs, the others keep their result.  Each run ends in one 4-byte-per-estimator device-to-host copy.
 * Out: zb (n x nb x dw) and lmb (n x nb) of the last run of each estimator, runs (n), n_accepted (n x nb, accepted moves
 * of that run per walker; may be NULL), n_negative (may be NULL): the number of in-box EI values < 0 met (ei.py:86-88
 * raises on them).  GPK_BAD_ARG: n < 1, nb odd, nb < 2 dw or nb > 64, steps < 1, max_runs < 1, acq_kind out of range,
 * lower >= upper, dw != d (fabolas = 0) or d - 1 (fabolas = 1), an unknown basis code or cfg_lower >= cfg_upper,
 * handles on different devices, with different d, listed twice, not fitted, or with a multi-rank communicator. */
int gpk_sample_representers(gpk_handle* const* models, int n, const unsigned long long* seeds, int nb, int steps,
                            int max_runs, int acq_kind, const double* eta, double par,
                            const double* lower, const double* upper, int dw,
                            int fabolas, const double* cfg_lower, const double* cfg_upper, int basis, double env_value,
                            double* zb, double* lmb, int* runs, long* n_accepted, long* n_negative);

/* ---- GP-MCMC hyper-parameters on the device (robo_b200/csrc/gpk_hyper.cuh) ---------------------------------------
 * GaussianProcessMCMC.train's stretch-move chain over theta = (kernel parameters, log noise) with every walker's
 * log-posterior computed on chip: the kernel built from theta on the inputs of gpk_set_data, a Cholesky factor in shared
 * memory (n <= GPK_HYPER_MAX_N), the prior restated on the device.
 *
 * gpk_set_hyper_model: how theta maps to the handle's kernel structure (family, axes, groups of the last gpk_set_kernel;
 *   its parameter values are not used).  n_params = len(kernel) (theta has n_params + 1 entries, the log noise last);
 *   amp_slot[p] = 1 when parameter p is an amplitude slot (log_amp = 0.0 + those entries in order), 0 for a metric slot,
 *   2 for log_a and 3 for log_b of the environment factor (one each, exactly when gpk_set_env_factor set a factor; its
 *   axis is the handle's), 4 for an entry of the task factor's Cholesky factor (exactly n_tasks (n_tasks + 1) / 2 of
 *   them, in packed order, when gpk_set_task_factor set a factor; its axis and n_tasks are the handle's);
 *   term_param[t] (n_terms entries) = the metric slot that sets term t (kernels.py flatten()["slots"]).  The diagonal is
 *   fl(sqrt(fl(yerr^2 + tiny)))^2 with yerr = sqrt(exp(theta[-1])), the constant mean `mean`.  prior_kind: gpk_prior_kind;
 *   prior_par (7 entries, NULL for GPK_PRIOR_NONE) = lognormal sigma, lognormal mean (scipy's loc), tophat lower, tophat
 *   upper, horseshoe scale, normal sigma, normal mean (the last two for GPK_PRIOR_ENV); n_ls, n_lr: EnvPrior's slices.
 *   GPK_PRIOR_MTBO (MTBOPrior, env_priors.py:188-206): lognorm(theta_0) + Tophat(theta[1:n_ls+1]) + a second tophat
 *   over theta[n_ls+1:n_ls+1+n_lr] (n_lr = n_kt, the task Cholesky entries) with prior_par[5], prior_par[6] its lower
 *   and upper bound + Horseshoe(theta[-1]).
 * gpk_hyper_lnpost: the log-likelihood ll (-inf for any |theta_j| > 20, a pivot that is not > 0 or a non-finite result)
 *   and the log-prior lp (0 without a prior) of count thetas (count x dim); the sampler's log-posterior is lp + ll where
 *   ll is finite (ll alone without a prior), -inf otherwise, NaN -> -inf.  The same device routine and block shape as
 *   gpk_sample_hypers: the values are the ones the sampler sees, bit for bit.
 * gpk_sample_hypers: one EnsembleSampler.run_mcmc(p0, steps): nwalkers x dim walkers from p0, the initial
 *   log-posteriors, then `steps` steps of two half-steps (one launch each, no host synchronisation), keyed by `seed`
 *   (Philox4x32-10; the counter layout and the rounding are in gpk_hyper.cuh).  Out: pos (nwalkers x dim), lnpost
 *   (nwalkers), n_accepted (nwalkers, may be NULL), copied back in one transfer at the end.
 * GPK_BAD_ARG: no data or kernel, no hyper model, n > GPK_HYPER_MAX_N, dim != n_params + 1, an odd number of walkers or
 * fewer than 2 dim, steps < 0, a slot table that does not cover the kernel's terms, an unknown prior kind. */
int gpk_set_hyper_model(gpk_handle* h, int n_params, const int* amp_slot, const int* term_param, int n_terms,
                        double mean, double tiny, int prior_kind, const double* prior_par, int n_ls, int n_lr);
int gpk_hyper_lnpost(gpk_handle* h, const double* theta, int count, int dim, double* ll, double* lp);
int gpk_sample_hypers(gpk_handle* h, const double* p0, int nwalkers, int dim, int steps, unsigned long long seed,
                      double* pos, double* lnpost, long* n_accepted);

/* ---- GaussianProcess hyper-parameter optimisation on the device (robo_b200/csrc/gpk_hyperopt.cuh) ------------------
 * GaussianProcess.optimize (gaussian_process.py:193-219): scipy.optimize.minimize(nll, p0, method='L-BFGS-B') without a
 * gradient, as one call.  nll is the objective of gpk_hyper_lnpost's two parts (-ll without a prior, -(ll + lp) with
 * one, 1e25 where that is not finite or |theta_j| > 20), the gradient scipy's forward differences with the absolute step
 * eps.  Every round scores the trial point and its dim neighbours in one launch (one CTA each) and runs L-BFGS-B's update
 * (every variable unbounded: the two-loop direction, the More-Thuente search, L-BFGS-B's restarts and skip rule) on the
 * device; the host reads the status once per GPK_HO_CHUNK rounds.  The arguments are scipy's options: maxcor, maxiter,
 * maxfun, ftol, pgtol (gtol), eps, maxls.  Needs gpk_set_data, gpk_set_kernel and gpk_set_hyper_model, as
 * gpk_sample_hypers.  Out: theta (dim) = the last accepted iterate (results.x); f, nit, nfev (evaluations, dim + 1 per
 * scored point) and status (GPK_LB_FTOL, _PGTOL, _MAXITER, _MAXFUN or _ABNORMAL) may be NULL.
 * GPK_BAD_ARG: no data, kernel or hyper model, a handle of another model kind, n > GPK_HYPER_MAX_N, dim != n_params + 1
 * or > GPK_HYPER_MAX_DIM, a non-finite p0, maxcor outside [1, 32], maxls < 1, eps <= 0, maxiter or maxfun < 1. */
#define GPK_HO_CHUNK 16
int gpk_optimize_hypers(gpk_handle* h, const double* p0, int dim, int maxcor, int maxiter, long maxfun, double ftol,
                        double pgtol, double eps, int maxls, double* theta, double* f, int* nit, long* nfev,
                        int* status);

/* ---- the same at large N (robo_b200/csrc/gpk_hyper_blocked.cuh) ---------------------------------------------------
 * gpk_hyper_lnpost_blocked, gpk_sample_hypers_blocked, gpk_optimize_hypers_blocked: the arguments, outputs and
 * gpk_set_hyper_model state of gpk_hyper_lnpost, gpk_sample_hypers and gpk_optimize_hypers, for 2 <= n <=
 * GPK_HYPER_BLOCKED_MAX_N.  The kernel matrix of every theta is built from theta in device memory and factored by the
 * fit's blocked Cholesky (128-row blocks: its diagonal-block kernel once per matrix, its fp64 tile engine with job
 * tables that span the chunk for the panel solves and trailing updates); the chunk holds as many thetas as
 * "hyper_batch_bytes" (gpk_set_option) allows.  ll and lp follow gpk_hyper_lnpost's rules (-inf for any |theta_j| > 20,
 * a pivot that is not > 0 or a non-finite result; lp the same prior routine, bit for bit); ll is another fixed-order
 * evaluation of the same quantity, so it agrees with gpk_hyper_lnpost to rounding, not bit for bit.  The bits of a
 * theta's ll and lp depend on theta, the data and n only, never on the chunk, the batch or the other thetas.  The
 * sampler and the optimiser are gpk_sample_hypers's and gpk_optimize_hypers's runs over these values (the same Philox
 * counters, rounding, L-BFGS-B update and status reads).  The chunk's device memory is released before each returns,
 * whatever the outcome.
 * GPK_BAD_ARG: as the counterpart, with n < 2 or n > GPK_HYPER_BLOCKED_MAX_N in place of n > GPK_HYPER_MAX_N, and one
 * theta's matrix larger than "hyper_batch_bytes".  GPK_CUDA_ERROR: the chunk's memory could not be allocated. */
int gpk_hyper_lnpost_blocked(gpk_handle* h, const double* theta, int count, int dim, double* ll, double* lp);
int gpk_sample_hypers_blocked(gpk_handle* h, const double* p0, int nwalkers, int dim, int steps,
                              unsigned long long seed, double* pos, double* lnpost, long* n_accepted);
int gpk_optimize_hypers_blocked(gpk_handle* h, const double* p0, int dim, int maxcor, int maxiter, long maxfun,
                                double ftol, double pgtol, double eps, int maxls, double* theta, double* f, int* nit,
                                long* nfev, int* status);

/* ---- Bayesian linear regression on the device (robo_b200/csrc/gpk_blr.cuh) ----------------------------------------
 * robo/models/bayesian_linear_regression.py with its default prior (robo/priors/bayesian_linear_regression_prior.py).
 * A handle becomes a BLR handle with gpk_blr_set_data and stays one: the Gaussian-process entry points (gpk_set_data,
 * gpk_set_kernel, gpk_set_input_bounds, gpk_set_output_transform, gpk_fit*, the hyper sampler, gpk_predict_grad,
 * gpk_predict_cov / gpk_posterior_cov / gpk_predict_mean*, gpk_kernel_matrix, gpk_nll_grad, the introspection calls,
 * ES / ESMC / ES_COST and gpk_sample_representers) return GPK_BAD_ARG with a message naming the model kind.  The
 * scoring entry points (gpk_acq, gpk_acq_dev, gpk_predict, gpk_maximize_random and every entry point over several
 * models with an EI / LogEI / PI / LCB or posterior objective: gpk_acq_multi, gpk_maximize_de, gpk_maximize_lbfgs,
 * gpk_maximize_cmaes, gpk_maximize_direct) score a fitted BLR handle through its predictive pass. */
#define GPK_BLR_MAX_F 64       /* most features: linear D <= 63, quadratic D <= 31, none D <= 64 */
typedef enum {
    GPK_BLR_LINEAR = 0,        /* phi(x) = [x, 1]       linear_basis_func    (bayesian_linear_regression.py:11-12) */
    GPK_BLR_QUADRATIC = 1,     /* phi(x) = [x^2, x, 1]  quadratic_basis_func (:15-17)                           */
    GPK_BLR_NONE = 2           /* phi(x) = x            basis_func=None (:154-157)                              */
} gpk_blr_basis;
/* gpk_blr_set_data: X (n x d) and y (n) as train() receives them (:152-160); Phi (n x F) is built on the device, and
 *   Phi^T Phi and Phi^T y are formed once, each entry a fixed-order reduction.  Drops the weight posteriors.  prior_par
 *   = lognormal sigma, lognormal mean (scipy's loc), horseshoe scale (BayesianLinearRegressionPrior: 0.1, -10, 0.1).
 *   GPK_BAD_ARG: an unknown basis, F > GPK_BLR_MAX_F, a handle that holds a Gaussian-process model.
 * gpk_blr_lnpost: marginal_log_likelihood (:76-113) of count thetas = (log alpha, log beta) (count x 2), one CTA each,
 *   NaN -> -inf: the values gpk_blr_sample sees, bit for bit.  The quirks are kept: the 2-norm of the residual, not its
 *   square (:108); log det A taken as +inf / -inf where numpy's det overflows / underflows (:110); the prior
 *   lognorm.logpdf(theta_0, sigma, loc) + Horseshoe(scale).lnprob(1 / theta_1) (prior :45-49).  A pivot that is not > 0
 *   gives -inf where the reference's inv raises LinAlgError.
 * gpk_blr_sample: one EnsembleSampler.run_mcmc(p0, steps) (:162-188 through emcee 2.x, a = 2) of nwalkers x 2 walkers:
 *   one launch for the initial log-posteriors, one per half-step, keyed by `seed` (Philox4x32-10, gpk_blr.cuh).  Out:
 *   pos (nwalkers x 2), lnpost (nwalkers), n_accepted (nwalkers, may be NULL), back in one transfer at the end.
 *   GPK_BAD_ARG: no data, an odd number of walkers or fewer than 4, steps < 0.
 * gpk_blr_fit: the k weight posteriors (:197-210) of hypers (k x 2, (alpha, beta) rows, not logs), resident for the
 *   predictive pass: m_i and L_i^-1 of A_i = beta_i Phi^T Phi + alpha_i I.  GPK_NOT_PD when a pivot of some A_i is not
 *   > 0 (the reference's inv raises LinAlgError or returns a useless inverse).
 * gpk_blr_get_models: the fit's m (k x F) and S = A^-1 (k x F x F) for `models`; dims: n, F, k.
 * The predictive pass (predict, :213-254): mu_i = phi^T m_i, var_i = 1 / beta_i + ||L_i^-1 phi||^2, their sums over i
 * in order divided by k, var clipped to DBL_EPSILON, then the acquisition closed form of gpk_acq_moments (hyper-samples
 * averaged before the closed form, the reference's BLR semantics). */
int gpk_blr_set_data(gpk_handle* h, const double* X, const double* y, int n, int d, int basis, const double* prior_par);
int gpk_blr_lnpost(gpk_handle* h, const double* thetas, int count, double* out);
int gpk_blr_sample(gpk_handle* h, unsigned long long seed, int nwalkers, const double* p0, int steps, double* pos,
                   double* lnpost, long* n_accepted);
int gpk_blr_fit(gpk_handle* h, const double* hypers, int k);
int gpk_blr_get_models(gpk_handle* h, double* m, double* S);
int gpk_blr_dims(gpk_handle* h, int* n, int* F, int* k);

/* ---- Random forest on the device (robo_b200/csrc/gpk_rf.cuh) --------------------------------------------------------
 * robo/models/random_forest.py, with the pyrfr forest it wraps restated (pyrfr's source is not available): bagged CART
 * regression trees on the residual sum of squares, every feature tried at every node, min_samples_to_split 2,
 * min_samples_in_leaf 1, no depth or node limit, a node with max y - min y <= 1e-8 is a leaf.  gpk_rf.cuh states every
 * step and its order; tests/rf_model.py restates them and the device equals it bit for bit.  A handle becomes an RF
 * handle with gpk_rf_set_data and stays one: the Gaussian-process entry points and the BLR ones return GPK_BAD_ARG with a
 * message naming the model kind, and the RF entry points refuse Gaussian-process and BLR handles.  The scoring entry
 * points (gpk_acq, gpk_acq_dev, gpk_predict, gpk_maximize_random and every entry point over several models with an EI /
 * LogEI / PI / LCB or posterior objective: gpk_acq_multi, gpk_maximize_de, gpk_maximize_lbfgs, gpk_maximize_cmaes,
 * gpk_maximize_direct) score a fitted RF handle through its predictive pass. */
#define GPK_RF_MAX_N 16384     /* most training points of a forest */
#define GPK_RF_MAX_D 64        /* most input dimensions of a forest */
#define GPK_RF_MAX_T 512       /* most trees of a forest */
/* gpk_rf_set_data: X (n x d) and y (n) as train() receives them (random_forest.py:59-83, which adds them row by row to
 *   a pyrfr data container); each feature's rows are ordered by (x_f, row index) once here.  Drops the trees.
 *   GPK_BAD_ARG: n > GPK_RF_MAX_N, d > GPK_RF_MAX_D, a non-finite entry, a handle holding another model kind.
 * gpk_rf_fit: rf.fit(data, engine) (:83) with the options of :52-57: T trees (num_trees), n_per_tree draws each
 *   (num_data_points_per_tree; 0: n, :75-76), with replacement when bootstrap (do_bootstrapping) and without otherwise
 *   (n_per_tree <= n), total_variance (compute_law_of_total_variance).  The draws are Philox4x32-10 keyed by seed,
 *   with counter (draw, tree, `counter`, tag): a caller advances `counter` once per fit as pyrfr's engine advances.
 *   Every tree grows on the device; there is no host round trip per node.  GPK_BAD_ARG: T outside 1..GPK_RF_MAX_T,
 *   n_per_tree > n without bootstrap.
 * gpk_rf_dims: n, d, T (0 before a fit) and the node slots per tree (2 n).
 * gpk_rf_get_trees: the trees in breadth-first order, T x slots each (any pointer may be NULL): n_nodes (T), feat (-1:
 *   leaf), thr, left (right = left + 1; -1 at a leaf), and the leaves' W (samples with multiplicity), mean and var (0 at
 *   a split node).  Slots past n_nodes are undefined.
 * gpk_rf_set_trees: the same arrays back onto an RF handle that holds the training set (a pickled or copied model);
 *   GPK_BAD_ARG for a node that is neither a leaf nor a split whose children follow it.
 * The predictive pass (predict_mean_var, :103-109 loops it over the rows): the (m_t, v_t) of the leaf x falls into in
 * every tree; mean = sum m_t / T, var = sum (m_t - mean)^2 / T (+ sum v_t / T with total_variance), sums in ascending t;
 * no clip.  The acquisition closed form of gpk_acq_moments follows, except that EI is 0 where var is 0 (ei.py:72-74). */
int gpk_rf_set_data(gpk_handle* h, const double* X, const double* y, int n, int d);
int gpk_rf_fit(gpk_handle* h, unsigned long long seed, unsigned counter, int T, int n_per_tree, int bootstrap,
               int total_variance);
int gpk_rf_dims(gpk_handle* h, int* n, int* d, int* T, int* slots);
int gpk_rf_get_trees(gpk_handle* h, int* n_nodes, int* feat, double* thr, int* left, double* W, double* mean,
                     double* var);
int gpk_rf_set_trees(gpk_handle* h, int T, int total_variance, const int* n_nodes, const int* feat, const double* thr,
                     const int* left, const double* W, const double* mean, const double* var);

/* ---- Bayesian neural network on the device (robo_b200/csrc/gpk_bnn.cuh) -------------------------------------------
 * robo/models/wrapper_bohamiann.py, with the pybnn network and sampler it wraps restated (pybnn's source is not
 * available): a D -> 50 -> 50 -> 1 tanh network with a homoscedastic log-variance, sampled by adaptive SGHMC.
 * gpk_bnn.cuh states every step and its order; tests/bnn_model.py restates them and the device chain equals it bit for
 * bit on the device's normals.  A handle becomes a BNN handle with gpk_bnn_set_data and stays one: the Gaussian-process,
 * BLR and RF entry points return GPK_BAD_ARG with a message naming the model kind, and the BNN entry points refuse the
 * other kinds.  The scoring entry points (as for an RF handle) score a trained BNN handle through its predictive pass. */
#define GPK_BNN_MAX_D 64         /* most input dimensions */
#define GPK_BNN_MAX_N 4096       /* most training points: the chain keeps an epoch's order (12 bytes a row) in shared
                                    memory beside theta, its gradient and the batch's activations */
#define GPK_BNN_MAX_BATCH 32     /* largest batch */
/* gpk_bnn_set_data: X (n x d) and y (n) as train() receives them.  Each column of X and y is scaled to zero mean and unit
 *   population std on the host (pybnn's normalize_input / normalize_output); the scaled copy and the statistics stay on
 *   the handle.  Drops the samples.  GPK_BAD_ARG: n < 2, a constant column or a constant y (pybnn would divide by zero),
 *   n > GPK_BNN_MAX_N, d > GPK_BNN_MAX_D, a non-finite entry, a handle holding another model kind.
 * gpk_bnn_train: one fresh chain of num_steps adaptive-SGHMC steps in one launch (step size lr, friction mdecay, eps;
 *   adaptation while the step count t <= burn_in; batches of `batch` rows), keeping theta after step s when s > burn_in
 *   and (s - burn_in) % keep_every == 0.  The draws are Philox4x32-10 keyed by seed with `counter` in their counter: a
 *   caller advances it once per train.  GPK_BAD_ARG: lr, mdecay or eps not finite and > 0 (eps >= 0), batch outside
 *   1..GPK_BNN_MAX_BATCH, keep_every < 1, burn_in < 0, num_steps outside 1..2^31 - 1, no network kept.
 * gpk_bnn_dims: n, d, the parameters per network P = 50 d + 2652 and the kept networks S (0 before a train).
 * gpk_bnn_get_samples: the S x P kept networks, in gpk_bnn.cuh's parameter order.
 * gpk_bnn_set_samples: S networks back onto a BNN handle that holds the training set (a pickled or copied model).
 * gpk_bnn_get_state: the chain's final theta, momentum p and adaptation state tau, g, vhat (P each; any may be NULL).
 * gpk_bnn_draws: Z (ns x P): the normals of steps step0 .. step0 + ns - 1 of a chain (seed, counter); step -1 holds the
 *   initial weights' normals.  For tests that restate the chain on the device's normals.
 * The predictive pass: m = mean_k f_k and v = mean_k (f_k - m)^2 + mean_k exp(lv_k) over the kept networks in order, then
 * m y_std + y_mean and v y_std^2; no clip.  The acquisition closed form of gpk_acq_moments follows. */
int gpk_bnn_set_data(gpk_handle* h, const double* X, const double* y, int n, int d);
int gpk_bnn_train(gpk_handle* h, unsigned long long seed, unsigned counter, double lr, double mdecay, double eps,
                  long burn_in, long num_steps, long keep_every, int batch);
int gpk_bnn_dims(gpk_handle* h, int* n, int* d, int* P, int* S);
int gpk_bnn_get_samples(gpk_handle* h, double* samples);
int gpk_bnn_set_samples(gpk_handle* h, int S, const double* samples);
int gpk_bnn_get_state(gpk_handle* h, double* theta, double* p, double* tau, double* g, double* vhat);
int gpk_bnn_draws(gpk_handle* h, unsigned long long seed, unsigned counter, int step0, int ns, double* Z);

/* ---- DNGO on the device (robo_b200/csrc/gpk_dngo.cuh) ------------------------------------------------------------
 * pybnn's DNGO (robo/fmin/bayesian_optimization.py:105-109), restated (pybnn's source is not available): a D -> 50 -> 50
 * -> 50 -> 1 tanh network trained by Adam on minibatches, then Bayesian linear regression over its last hidden layer
 * (the 50 features Theta) with the BLR entry points' log-posterior, sampler and weight posteriors.  gpk_dngo.cuh states
 * every step and its order; tests/dngo_model.py restates them and the device training equals it bit for bit.  A handle
 * becomes a DNGO handle with gpk_dngo_set_data and stays one: the Gaussian-process, RF and BNN entry points,
 * gpk_blr_set_data and gpk_blr_fit return GPK_BAD_ARG with a message naming the model kind, and the DNGO entry points
 * refuse the other kinds.  gpk_blr_lnpost, gpk_blr_sample, gpk_blr_get_models and gpk_blr_dims serve a trained DNGO
 * handle's regression (F = 50, basis none, on the scaled y).  The scoring entry points (as for an RF handle) score a
 * fitted DNGO handle through its predictive pass. */
#define GPK_DNGO_MAX_D 64        /* most input dimensions */
#define GPK_DNGO_MAX_N 4096      /* most training points: the training kernel keeps an epoch's order (12 bytes a row) in
                                    shared memory beside theta, its gradient and the batch's activations */
#define GPK_DNGO_MAX_BATCH 16    /* largest batch, min(batch, n) */
/* gpk_dngo_set_data: X (n x d) and y (n) as train() receives them.  With normalize_input / normalize_output, each column
 *   of X / y is scaled to zero mean and unit population std on the host (gpk_bnn_set_data's code); otherwise that side
 *   is used as given.  prior_par as gpk_blr_set_data's.  Drops the net and the fit.  GPK_BAD_ARG: n < 2 with a flag on,
 *   a constant column or a constant y under its flag, n > GPK_DNGO_MAX_N, d > GPK_DNGO_MAX_D, a non-finite entry, a
 *   handle holding another model kind.
 * gpk_dngo_train: a fresh net trained for `epochs` epochs of floor(n / B) Adam steps (B = min(batch, n); the remaining
 *   rows of each epoch are dropped) at learning rate lr, in one launch; then Theta and the regression's Theta^T Theta and
 *   Theta^T y.  The initial weights and the epoch orders are Philox4x32-10 keyed by seed with `counter` in their counter:
 *   a caller advances it once per train.  Drops the fit.  GPK_BAD_ARG: lr not finite and > 0, batch < 1, epochs < 1,
 *   B > GPK_DNGO_MAX_BATCH.
 * gpk_dngo_fit: the BLR weight posteriors of hypers (k x 2, as gpk_blr_fit), then the collapsed predictive: m_bar = mean
 *   m_i, Q = mean S_i + (1 / k) sum (m_i - m_bar)(m_i - m_bar)^T, its Cholesky factor R and c_bar = mean 1 / beta_i.
 *   GPK_NOT_PD as gpk_blr_fit, or when Q's factorisation fails.
 * gpk_dngo_dims: n, d, the parameters of the net P = 50 d + 5201 and the fit's k (0 before a fit).
 * gpk_dngo_get_net: the trained net (P, gpk_dngo.cuh's parameter order).
 * gpk_dngo_set_net: a net back onto a DNGO handle that holds the training set (a pickled or copied model); Theta and the
 *   regression's products are rebuilt from it, bit for bit as gpk_dngo_train built them.  Drops the fit and the Adam
 *   state.
 * gpk_dngo_features: Theta (m x 50) of the m rows X (m x d, scaled as candidates are), the training pass's arithmetic.
 * gpk_dngo_get_state: Adam's final m and v (P each; either may be NULL) and its step count t of the last train.
 * The predictive pass: at features phi, m = phi^T m_bar and v = c_bar + ||R^T phi||^2 (the mixture of the k posteriors'
 * mean and full variance), v clipped to DBL_EPSILON, then m y_std + y_mean and v y_std^2.  The acquisition closed form of
 * gpk_acq_moments follows. */
int gpk_dngo_set_data(gpk_handle* h, const double* X, const double* y, int n, int d, int normalize_input,
                      int normalize_output, const double* prior_par);
int gpk_dngo_train(gpk_handle* h, unsigned long long seed, unsigned counter, double lr, int batch, int epochs);
int gpk_dngo_fit(gpk_handle* h, const double* hypers, int k);
int gpk_dngo_dims(gpk_handle* h, int* n, int* d, int* P, int* k);
int gpk_dngo_get_net(gpk_handle* h, double* net);
int gpk_dngo_set_net(gpk_handle* h, const double* net);
int gpk_dngo_features(gpk_handle* h, const double* X, long m, double* out);
int gpk_dngo_get_state(gpk_handle* h, double* m, double* v, long long* t);

/* kernel.get_value(X1, X2) (test/test_models/test_gaussian_process.py:44-46) with the
 * handle's current kernel; no input scaling.  out is (n1, n2) row-major. */
int gpk_kernel_matrix(gpk_handle* h, const double* X1, long n1, const double* X2, long n2,
                      int d, double* out);

/* ---- multi-GPU: candidate shards, one 16-byte exchange per arg-max (SURVEY.md section 8e) -------------------- */
/* One process per GPU, one handle per process.  The fit state is replicated (every rank calls gpk_set_data /
 * gpk_set_kernel / gpk_fit with the same inputs: zero communication), rank r scores the contiguous slice
 * gpk_shard_bounds(m, r, world) of the candidate list, and the ranks agree on numpy.argmax of the whole list
 * (robo/maximizers/random_sampling.py:50: first maximum, NaN first) through ONE ncclAllGather of the 16-byte
 * {value, global index} pair on the handle's stream followed by a deterministic merge on the device.  NCCL is bound at
 * run time (dlopen of libnccl.so.2; GPK_NCCL_LIB overrides), so the library itself links cudart only. */
int gpk_comm_unique_id(void* id128);           /* rank 0: ncclGetUniqueId; ship the 128 bytes to the other ranks */
int gpk_comm_init(gpk_handle* h, int rank, int world, const void* id128);    /* collective over all ranks */
int gpk_comm_destroy(gpk_handle* h);
int gpk_comm_info(gpk_handle* h, int* rank, int* world, int* nccl_version);
int gpk_shard_bounds(long m, int rank, int world, long* lo, long* hi);       /* sizes differ by at most one */
/* The exchange alone: this rank's best {value, GLOBAL index} (index < 0: nothing to offer) in, the merged winner out on
 * every rank.  For callers that scored their shard themselves (e.g. EI.compute on a slice, values wanted on the host). */
int gpk_comm_argmax_pair(gpk_handle* h, double val, long idx, double* best_val, long* best_idx);
/* Xs: the FULL candidate batch (m_total, d), identical host array on every rank; each rank copies and scores only its
 * slice.  Returns the global arg-max on every rank. */
int gpk_acq_argmax_sharded(gpk_handle* h, const double* Xs, long m_total, int acq_kind, double eta, double par,
                           double* best_val, long* best_idx);
/* Device-resident shard, asynchronous on the handle's stream, no host synchronisation: d_Xs_shard is this rank's
 * (m_shard, d) slice whose first row has global index first_global (m_shard may be 0); d_best (16 bytes, device)
 * receives the merged {double value; long long global index}. */
int gpk_acq_argmax_sharded_dev(gpk_handle* h, const void* d_Xs_shard, long m_shard, long first_global, int acq_kind,
                               double eta, double par, void* d_best);
/* gpk_maximize_random over n_total device-generated candidates split across the ranks (Philox keyed by the global
 * index: the result does not depend on the number of GPUs); best_x is re-created on every rank from the winning index. */
int gpk_maximize_random_sharded(gpk_handle* h, unsigned long long seed, long n_total, long n_uniform,
                                const double* lower, const double* upper, const double* incumbent, double scale,
                                int acq_kind, double eta, double par,
                                double* best_x, double* best_val, long* best_idx);

/* ---- marginal-likelihood gradient (gaussian_process.py:168-191, corrected noise term) -- */
/* grad[n_terms + 2] = d(-loglik)/d[log_amp, log_metric_t..., log sigma^2]; requires a
 * preceding successful gpk_fit with the same parameters.  noise_var = sigma^2.  With the environment factor
 * (gpk_set_env_factor) grad has n_terms + 4 entries: [log_amp, log_metric_t..., log_a, log_b, log sigma^2]; with the
 * task factor (gpk_set_task_factor) n_terms + 2 + n_kt: [log_amp, log_metric_t..., theta_task (packed)..., log sigma^2],
 * dK_t[a, b] / dtheta_pq = L_pq (delta_ap L_bq + delta_bp L_aq). */
int gpk_nll_grad(gpk_handle* h, double noise_var, double* grad);

/* fp64 issue-rate peaks of this GPU in TFLOP/s, measured with register-resident operands: the DMMA
 * m8n8k4 tensor instruction (every fp64 GEMM of the library) and the DFMA vector pipe (covariance builder).  bench.py
 * uses the DMMA figure as the roofline denominator of the fp64 contraction.  On an H100 the m8n8k4 shape reaches
 * about half of the fp64 tensor-core rate that cuBLAS DGEMM gets (DESIGN.md section 5). */
int gpk_measure_fp64_peaks(gpk_handle* h, double* dmma_tflops, double* dfma_tflops);

/* int8 tensor-pipe issue-rate peak in TOP/s (wgmma m64n128k32 s8 on two warpgroups per SM, operands in shared memory,
 * accumulators in registers): the roofline denominator of the option-"ozaki" contraction. */
int gpk_measure_int8_peak(gpk_handle* h, double* tops);
/* the same kernel launched back to back for `seconds` (<= 10); reports the rate of the second half, i.e. at the SM clock
 * the board's power limit allows for this pipe: the denominator for a kernel timed inside a long step.
 * random_operands = 0: constant operand pattern (no switching activity: does not reach the power limit); 1: pseudo-random
 * bytes, the statistics of real digit slices. */
int gpk_measure_int8_peak_sustained(gpk_handle* h, double seconds, int random_operands, double* tops);

/* ---- introspection (tests / debugging) ----------------------------------------------- */
int gpk_get_factor(gpk_handle* h, double* L /* n x n row-major, lower */);
int gpk_get_linv(gpk_handle* h, double* Linv /* n x n row-major, lower */);
int gpk_get_z(gpk_handle* h, double* z /* n */);
/* The two inputs of the entropy change that gpk_es_compute derives per candidate, read back from the buffers its dH
 * kernel reads (the same passes of ES_CH = 16384 candidates, the same launches): var (m) the predictive variance of the
 * scoring pass, sigma (m x nb row-major) the covariance to the representer points, (k(zb_j, x) - K(x, X) U[:, j]) *
 * y_std^2 (output transform) clipped at DBL_EPSILON.  Xs: m x d raw inputs.  GPK_BAD_ARG before gpk_es_update or after
 * the model changed since. */
int gpk_es_moments(gpk_handle* h, const double* Xs, long m, double* var, double* sigma);
/* U = K^-1 K(X, zb) of the last gpk_es_update (n x nb row-major, fp64, built from L^-1); GPK_BAD_ARG as above. */
int gpk_es_get_u(gpk_handle* h, double* U);
/* n and nb of the last gpk_es_update: the shapes of gpk_es_get_u's U and of gpk_es_moments' sigma rows; GPK_BAD_ARG
 * as above. */
int gpk_es_dims(gpk_handle* h, int* n, int* nb);
/* The int8 variance contraction alone, on caller-supplied operands (tests: tests/ozaki_model.py restates it exactly).
 * P: n x n row-major, lower triangular (the stand-in for L^-1; only its block-lower triangle is read by the contraction,
 * its row maxima by the row exponents).  Ks: m x n row-major, every |entry| <= amp.  Both are zero-padded to NP =
 * round_up(n, 128) columns and to NP / round_up(m, 128) rows, split into 7 balanced base-256 digits (row exponents eP of
 * P, one exponent eK = oz_exponent(amp) for Ks) and contracted with the handle's "ozcluster", "ozpersist" and "ozgrid",
 * whatever "ozaki" says.  Out: part_ssq (nb x m row-major, nb = NP / 128) = sum over the rows of row block ib of V^2,
 * V = P Ks^T; eP (n) and eK.  Uses its own scratch: a fitted model is left untouched.  GPK_BAD_ARG when an entry of Ks
 * exceeds amp or NP > 16384.  Updates out[14] of gpk_get_timings. */
int gpk_oz_contract(gpk_handle* h, const double* P, int n, const double* Ks, long m, double amp,
                    double* part_ssq /* nb x m */, int* eP /* n */, int* eK);
/* last fit/score timings measured with CUDA events on the handle's stream, milliseconds:
 * out[0] fit total, [1] K build, [2] Cholesky, [3] L^-1, [4] last score call total,
 * [5] K* build and [7] epilogue of the last candidate chunk, [6] variance GEMM averaged over the
 * full-size chunk launches of that call;
 * out[8] = variance-GEMM launches so far,
 * out[9] = total kernel launches so far,
 * out[10] = of those, launches of the int8 (Ozaki) contraction; out[11] = largest row exponent of L^-1 seen by it
 * (option "ozaki"); out[12] reserved (zero); out[13] = int8 slice-pair products the int8 contraction spends per
 * fp64 product (28: 7 balanced base-256 digits per operand); out[14] = which int8 kernel ran last (1 gpk_oz_vargemm_kernel;
 * + 8: persistent tile walk; + 16 / + 32: clusters of 2 / 4 CTAs); out[15] reserved (zero). */
int gpk_get_timings(gpk_handle* h, double* out16);
/* diagnostics of the blocked diagonal-block kernel (option "diagprof" = 1): clock64() stamps of the last
 * launched block: out[0] start, out[1] tiles loaded, out[2+2p] panel p factorised + solved, out[3+2p] panel p's
 * rank-16 update applied and panel p+1 published, out[33] end, out[34..41] finer stamps inside panel 3. */
int gpk_get_diag_profile(gpk_handle* h, long long* out64);

#ifdef __cplusplus
}
#endif
#endif /* GPK_H_ */
