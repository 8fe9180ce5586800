/* smcb.h -- C-ABI of libsmcb.so: the H100 (sm_90a) SMC inner loop.
 *
 * Drop-in boundary for the per-step hot path of nchopin/particles
 * (particles.core.SMC: propagate -> log-weight -> normalise/ESS -> resample).
 * The reference is pure Python with no FFI of its own; each entry point below
 * names the reference function it replaces (paths relative to the reference
 * root), and INTEGRATION.md shows the ctypes binding a maintainer would add.
 *
 * Conventions
 *  - every array argument is a DEVICE pointer (fp64 / int64, contiguous) owned by
 *    the caller (torch tensors in the Python host layer); scalars results are
 *    written to device memory too, so no call synchronises the host;
 *  - work is enqueued on the context's stream (smcb_set_stream);
 *  - every function returns 0 on success, a negative SMCB_E* code otherwise,
 *    with a message available from smcb_last_error();
 *  - a context is bound to one device and is not thread-safe;
 *  - results are deterministic: same inputs + same seed -> same bits, whatever
 *    the grid size (all reductions and the scan use a fixed association order).
 */
#ifndef SMCB_H
#define SMCB_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SMCB_OK 0
#define SMCB_EINVAL (-1) /* bad argument (ValueError on the Python side)        */
#define SMCB_ECUDA (-2)  /* CUDA runtime error                                   */
#define SMCB_ENOSYS (-3) /* combination not implemented (NotImplementedError)    */

typedef struct smcb_ctx smcb_ctx;

const char *smcb_last_error(void);
int smcb_version(void);

/* one context per (device, stream); owns a small workspace + the Philox key */
int smcb_create(smcb_ctx **out, int device, uint64_t seed);
int smcb_destroy(smcb_ctx *ctx);
int smcb_set_stream(smcb_ctx *ctx, void *cuda_stream);
/* re-key the counter-based generator (replaces numpy.random.seed for this path) */
int smcb_seed(smcb_ctx *ctx, uint64_t seed);
/* number of kernels this context has launched so far (bench.py "gpu_launches") */
int64_t smcb_launch_count(const smcb_ctx *ctx);

/* ---------------------------------------------------------------------------
 * weights algebra  (particles/resampling.py)
 * ------------------------------------------------------------------------- */

/* Weights.__init__, resampling.py:217-226.  lw is modified in place (NaN -> -inf,
 * line 220).  W_out may be NULL.  stats_out[4] = {max lw, log_mean, ESS, sum w}. */
int smcb_normalise(smcb_ctx *ctx, double *lw, int64_t n, double *W_out, double *stats_out);
/* The second half alone, W = exp(lw - m) / s (resampling.py:223-225) with statistics the caller already holds
 * (stats[0] = m, stats[3] = s: the layout above; the fused filter's device state; for a sharded filter the GLOBAL
 * (m, s), so that W sums to one over all ranks). */
int smcb_weights_from_stats(smcb_ctx *ctx, const double *lw, int64_t n, const double *stats, double *W_out);

#define SMCB_LSE_SUM 0  /* log_sum_exp   resampling.py:247-270            */
#define SMCB_LSE_MEAN 1 /* log_mean_exp  resampling.py:291-317 (W optional) */
#define SMCB_LSE_ESSL 2 /* essl          resampling.py:166-188            */
/* every mode gives NaN when v holds a NaN or a +inf, or is -inf throughout, as the reference does */
int smcb_lse(smcb_ctx *ctx, int mode, const double *v, const double *W, int64_t n,
             double *out);

/* exp_and_normalise, resampling.py:138-163 */
int smcb_exp_and_normalise(smcb_ctx *ctx, const double *lw, int64_t n, double *W_out);

/* wmean_and_var, resampling.py:320-338; x is SoA (d, n) with 1 <= d <= 32; out = {mean[d], var[d]} */
int smcb_wmean_and_var(smcb_ctx *ctx, const double *W, const double *x, int64_t n, int d,
                       double *out);

/* ---------------------------------------------------------------------------
 * resampling  (particles/resampling.py)
 * ------------------------------------------------------------------------- */
#define SMCB_RS_MULTINOMIAL 0 /* resampling.py:540-558 */
#define SMCB_RS_STRATIFIED 1  /* resampling.py:599-603 */
#define SMCB_RS_SYSTEMATIC 2  /* resampling.py:606-610 */
#define SMCB_RS_RESIDUAL 3    /* resampling.py:613-627 */
#define SMCB_RS_SSP 4         /* resampling.py:630-677; sequential recursion, one device thread;
                                 u_in = N - 1 uniforms; synchronises once (ValueError check) */

/* Inclusive prefix sum of non-negative fp64 values (the CDF that inverse_cdf,
 * resampling.py:484-509, walks).  Reduce-then-scan with a fixed association
 * order: deterministic and non-decreasing by construction. */
int smcb_cumsum(smcb_ctx *ctx, const double *w, int64_t n, double *cdf_out);

/* A[k] = min{ j : cdf[j] >= su[k] } clipped to n-1, for sorted su;
 * == np.searchsorted(cdf, su, 'left') bit-exactly (inverse_cdf, resampling.py:484-509) */
int smcb_searchsorted(smcb_ctx *ctx, const double *cdf, int64_t n, const double *su,
                      int64_t m, int64_t *A_out);

/* rs.resampling(scheme, W, M), resampling.py:464-481, 540-627.
 * u_in (device) = the uniforms to use, in the order the reference draws them
 * (systematic 1, stratified m, multinomial m+1, residual m+1, ssp n-1); NULL -> Philox.
 * scratch: at least smcb_resample_scratch_doubles(n, m) doubles (16-byte aligned).
 * Asynchronous on the context's stream except SMCB_RS_SSP, which synchronises once to report the
 * reference's "wrong size for output" ValueError (resampling.py:674-676) as SMCB_EINVAL. */
int64_t smcb_resample_scratch_doubles(int64_t n, int64_t m);
int smcb_resample(smcb_ctx *ctx, int scheme, const double *W, int64_t n, int64_t m,
                  int64_t *A_out, const double *u_in, double *scratch);

/* Xp = X[A]  (core.py:332); X is SoA (d, n), Xp is SoA (d, m) */
int smcb_gather(smcb_ctx *ctx, const double *X, int64_t n, const int64_t *A, int64_t m,
                int d, double *Xp);
/* same for row-major (n, d) particles, the layout user closures index as xp[:, i] */
int smcb_gather_rows(smcb_ctx *ctx, const double *X, int64_t n, const int64_t *A, int64_t m,
                     int d, double *Xp);

/* ---------------------------------------------------------------------------
 * distributions  (particles/distributions.py)
 * an array argument may be NULL, in which case the scalar next to it is used
 * ------------------------------------------------------------------------- */
/* Normal.rvs, distributions.py:270-271; z_in = injected N(0,1) draws or NULL */
int smcb_normal_rvs(smcb_ctx *ctx, const double *loc, double loc0, const double *scale,
                    double scale0, const double *z_in, double *out, int64_t n);
/* Normal.logpdf, distributions.py:273-274 */
int smcb_normal_logpdf(smcb_ctx *ctx, const double *x, double x0, const double *loc,
                       double loc0, const double *scale, double scale0, double *out,
                       int64_t n);
/* other univariate log-densities (distributions.py): kind 0 Student(df = p0, loc, scale) :417-433, 1 Gamma(a = p0,
 * rate) :336-356, 2 Laplace(loc, scale) :399-414, 3 Logistic(loc, scale) :381-396; p1 / p2 arrays or scalars as for
 * Normal; c0 = the host-computed lgamma constant of the density (0 for kinds 2, 3) */
int smcb_logpdf1(smcb_ctx *ctx, int kind, const double *x, double x0, double p0, double c0, const double *p1,
                 double p10, const double *p2, double p20, double *out, int64_t n);
/* MvNormal.rvs / logpdf, distributions.py:946-969; SoA (d, n), d <= 32; L = host (d,d) lower
 * Cholesky factor of cov, row-major; loc/scale: array (d, n), or NULL + host vector[d].
 * d <= 8: factor in the kernel parameters, two particles per thread; 8 < d <= 32: factor in shared
 * memory, one particle per thread (CUDA cores: HBM-bound at every d <= 32, see smcb_api.cu) */
int smcb_mvnormal_rvs(smcb_ctx *ctx, const double *loc, const double *loc0,
                      const double *scale, const double *scale0, const double *L, int d,
                      const double *z_in, double *out, int64_t n);
int smcb_mvnormal_logpdf(smcb_ctx *ctx, const double *x, const double *loc,
                         const double *loc0, const double *scale, const double *scale0,
                         const double *L, int d, double *out, int64_t n);
/* standard normals / uniforms from the context's Philox stream */
int smcb_standard_normal(smcb_ctx *ctx, double *out, int64_t n);
int smcb_uniform(smcb_ctx *ctx, double *out, int64_t n);

/* The laws of distributions.py with a kernel of their own (csrc/smcb_dists.cuh), by law code:
 *   0 InvGamma(a, b)                  :358-377  scipy.stats.invgamma.logpdf(x, a, scale=b); draws b / Gamma(a, 1)
 *   1 LogNormal(mu, sigma)            :379-396  scipy.stats.lognorm.logpdf(x, sigma, scale=exp(mu))
 *   2 TruncNormal(mu, sigma, a, b)    :475-505  scipy.stats.truncnorm.logpdf, mass in log space; exact draws
 *   3 Binomial(n, p)                  :535-549  scipy.stats.binom.logpmf
 *   4 Geometric(p)                    :552-565  scipy.stats.geom.logpmf (support 1, 2, ...)
 *   5 NegativeBinomial(n, p)          :568-595  scipy.stats.nbinom.logpmf(x, n, p), the law its draws follow
 *   6 DiscreteUniform(lo, hi)         :631-649  -log(hi - lo) on lo .. hi - 1
 *   7 Gamma(a, rate b)                draws only: the sampler InvGamma, NegativeBinomial and Dirichlet draw through
 * Parameter k is the array pk of n values, or NULL and the scalar s[k] (s: host array of 4 doubles; unused ones
 * are ignored).  NaN outside a law's parameter domain, -inf outside its support and, for codes 3-6, at non-integer
 * x.  Draws: fp64 into out for codes 0-2 and 7, int64 for the discrete codes 3-6 (INT64_MIN where a parameter is
 * outside its domain); element i's draw depends on (seed, API call, i) only. */
int smcb_dist_logpdf(smcb_ctx *ctx, int law, const double *x, double x0, const double *p0, const double *p1,
                     const double *p2, const double *p3, const double *s, double *out, int64_t n);
int smcb_dist_rvs(smcb_ctx *ctx, int law, const double *p0, const double *p1, const double *p2, const double *p3,
                  const double *s, void *out, int64_t n);
/* Dirichlet(alpha), distributions.py:854-885: alpha (d,) on the device, rows x (n, d) with row stride x_ld (0: one
 * row for all n); c0 = -log B(alpha).  *bad (device int, zeroed by the caller) collects the bits of the tests of
 * scipy.stats.dirichlet's input check that some row fails (the host raises its ValueError): 1 an entry < 0 or > 1,
 * 2 a zero entry where alpha_j < 1, 4 |sum - 1| > 1e-9, 8 a NaN entry (which, as in scipy, voids test 1 and makes
 * the row's density NaN).  rvs: Gamma(alpha_j, 1) draws normalised in log space (finite for small alphas). */
int smcb_dirichlet_logpdf(smcb_ctx *ctx, const double *x, int64_t x_ld, const double *alpha, int d, double c0,
                          double *out, int *bad, int64_t n);
int smcb_dirichlet_rvs(smcb_ctx *ctx, const double *alpha, int d, double *out, int64_t n);
/* VaryingCovNormal, distributions.py:1012-1059, 1 <= d <= 8 (SMCB_ENOSYS above): cov, L (n, d, d) row-major; chol
 * writes the lower factors and sets *bad (device int, zeroed by the caller) when a cov[i] is not positive
 * definite; loc / x rows of d values with row stride loc_ld / x_ld (0: one row for all n). */
int smcb_vcn_chol(smcb_ctx *ctx, const double *cov, int d, double *L, int *bad, int64_t n);
int smcb_vcn_rvs(smcb_ctx *ctx, const double *loc, int64_t loc_ld, const double *L, int d, double *out, int64_t n);
int smcb_vcn_logpdf(smcb_ctx *ctx, const double *x, int64_t x_ld, const double *loc, int64_t loc_ld,
                    const double *L, int d, double *out, int64_t n);
/* Mixture.logpdf, distributions.py:805-810: out[i] = logsumexp_j (logpk[i pk_ld + j] + lp[j n + i]), lp the (k, n)
 * component log-densities, logpk (k,) (pk_ld = 0) or (n, k) (pk_ld = k) */
int smcb_mixture_logpdf(smcb_ctx *ctx, const double *lp, const double *logpk, int64_t pk_ld, int k, double *out,
                        int64_t n);

/* ---------------------------------------------------------------------------
 * SMC samplers: tempering / waste-free move step  (particles/smc_samplers.py)
 * theta is (n, d) row-major, d <= 32
 * ------------------------------------------------------------------------- */
/* Tempering.current_target, smc_samplers.py:836-845, for the logistic-regression static model
 * (book/smc_samplers/logistic_reg.py:60-67): prior MvNormal(0, prior_scale^2 I_d);
 * llik = sum_t -log(1 + exp(-theta . data[t])) (StaticModel.loglik, 263-284); lpost = lprior + epn*llik */
int smcb_logistic_target(smcb_ctx *ctx, const double *theta, int64_t n, int d, const double *data,
                         int64_t n_data, double prior_scale, double epn, double *lprior,
                         double *llik, double *lpost);
/* ArrayRandomWalk.proposal, smc_samplers.py:624-629: prop = theta + z @ L.T; L_dev = device (d, d)
 * row-major lower factor; z_in = injected N(0,1) (n, d) or NULL */
int smcb_rw_propose(smcb_ctx *ctx, const double *theta, int64_t n, int d, const double *L_dev,
                    const double *z_in, double *prop);
/* ArrayMetropolis.step, smc_samplers.py:601-611: accept where u < exp(min(lpost' - lpost, 0)) and
 * copy the proposal's fields in place; mean_acc (device scalar) = mean acceptance probability */
int smcb_mh_accept(smcb_ctx *ctx, int64_t n, int d, double *theta, double *lprior, double *llik,
                   double *lpost, const double *theta_p, const double *lprior_p, const double *llik_p,
                   const double *lpost_p, const double *u_in, double *mean_acc);

/* MCMCSequenceWF.__call__, smc_samplers.py:672-683, fused for the logistic model + random-walk
 * Metropolis: ONE launch runs the P-1 Metropolis steps of all M chains.  Inputs: the M resampled
 * particles; outputs: the P*M particles of the next generation in concatenate(xs) order and the
 * (P-1, M) acceptance probabilities.  z_in (P-1, M, d) / u_in (P-1, M): injected noise or NULL. */
int smcb_logistic_wf_move(smcb_ctx *ctx, int64_t M, int d, int P, const double *theta0,
                          const double *lprior0, const double *llik0, const double *lpost0,
                          const double *data, int64_t n_data, double prior_scale, double epn,
                          const double *L_dev, const double *z_in, const double *u_in,
                          double *theta_out, double *lprior_out, double *llik_out, double *lpost_out,
                          double *pb_out);

/* IBIS.logG, smc_samplers.py:773-776, for the logistic-regression model: logpyt of the data rows [r0, r0 + K) of
 * data (n_data, d) for n particles, added one row at a time in row order (a NaN log-weight becomes -inf after each
 * row).  commit != 0: lw, lpost and llik += every row, in place (lpost / llik may be NULL); commit == 0:
 * scratch (K, n) row k = lw + the rows r0 .. r0 + k, and nothing else is written.  Same per-row bits as a one-row
 * smcb_logistic_target. */
int smcb_logistic_logpyt(smcb_ctx *ctx, const double *theta, int64_t n, int d, const double *data, int64_t n_data,
                         int64_t r0, int64_t K, int commit, double *lw, double *lpost, double *llik, double *scratch);

/* Nested sampling SMC (NestedSamplingSMC, particles/nested.py:281-373, Salomone et al. 2018) for the same model.
 * The target is the prior truncated to llik >= lmin (current_target, 353-363): lpost = lprior where llik >= lmin,
 * -inf elsewhere; lmin = -inf gives the bits of the untempered target (epn = 0).  lmin must not be NaN.
 * smcb_logistic_ns_target: the arguments of smcb_logistic_target with lmin in place of epn.
 * smcb_logistic_ns_move: those of smcb_logistic_wf_move with lmin in place of epn; a proposal below the floor has
 * pb = 0 and is rejected whatever u is.  Same proposals, Philox counters, output order and pb table. */
int smcb_logistic_ns_target(smcb_ctx *ctx, const double *theta, int64_t n, int d, const double *data,
                            int64_t n_data, double prior_scale, double lmin, double *lprior, double *llik,
                            double *lpost);
int smcb_logistic_ns_move(smcb_ctx *ctx, int64_t M, int d, int P, const double *theta0, const double *lprior0,
                          const double *llik0, const double *lpost0, const double *data, int64_t n_data,
                          double prior_scale, double lmin, const double *L_dev, const double *z_in,
                          const double *u_in, double *theta_out, double *lprior_out, double *llik_out,
                          double *lpost_out, double *pb_out);
/* NestedSamplingSMC.logG (nested.py:330-351) in one call, nothing read back inside it.  llik (n): NaN-free.
 * lt = numpy's _lerp of the order statistics k0 and k1 (k1 = k0 or k0 + 1) of llik with weight gamma: the caller gives
 * NumPy's "linear" rule, so lt has the bits of np.percentile(llik, 100 (1 - ESSrmin)) (when llik holds both -0.0
 * and +0.0, a zero lt may carry either sign, as NumPy's partition may).  Then
 * lZt = t log_alpha - log(n) + logsumexp(llik[llik <= lt]), new_evid = log_sum_exp_ab(log_evid, lZt), the same with
 * all of llik (new_evid_final, one reduction tree for both), and stop = |new_evid - new_evid_final| < eps.
 * lw (n): 0 where llik > lt, -inf elsewhere, or all 0 on a stop.  out_dev (3) = (lt, new_evid, stop): (inf,
 * new_evid_final, 1) on a stop.  10 launches; uses the context's workspace. */
int smcb_ns_threshold(smcb_ctx *ctx, const double *llik, int64_t n, int64_t k0, int64_t k1, double gamma, int t,
                      double log_alpha, double log_evid, double eps, double *lw, double *out_dev);

/* SMC samplers on {0,1}^p (particles/binary_smc.py): Bayesian variable selection, p <= 128.  Particles are (n, p)
 * bytes 0 / 1 (torch.bool).  The model: loglik(gamma) = -(coef_len |gamma| + [use_ldet] ldet + coef_log
 * log(coef_in_log - gw wtw)) (BIC 227-230, BayesianVS 258-265 with use_ldet = 1, BayesianVS_gprior 287-293 with
 * gw = g / (g + 1)), prior IID(Bernoulli(q), p) with lq = log(clip(q)), l1q = log(clip(1 - q)). */
typedef struct {
    int32_t p;                 /* predictors, 1..128                                                     */
    int32_t use_ldet;          /* 1: the log-determinant enters loglik (BayesianVS)                      */
    const double *xtx;         /* (p, p) device, X^T X                                                   */
    const double *xty;         /* (p) device, X^T y                                                      */
    double vm2;                /* added to the diagonal of X^T X[gamma, gamma] by the move (iv2)         */
    double coef_len, coef_log, coef_in_log, gw;
    double lq, l1q;
} smcb_vs_desc;

/* chol_and_friends (binary_smc.py:165-180) with diagonal shift vm2 for the n rows of gamma: len_gam, ldet =
 * sum log diag L, wtw = |L^-1 X^T y[gamma]|^2 ((0, 0, 0) for an empty gamma); each output may be NULL.  llik (or
 * NULL): the model's loglik; lprior and lpost (or NULL; lpost needs both): the prior and lprior + epn llik
 * (lprior where epn <= 0).  kmax >= every |gamma| (it sizes shared memory).  *err (device int, zeroed by the
 * caller): bit 0 = a non-positive pivot (that row gets llik = -inf, ldet = wtw = NaN), bit 1 = a row above kmax. */
int smcb_vs_loglik(smcb_ctx *ctx, const smcb_vs_desc *model, const uint8_t *gamma, int64_t n, int kmax, double vm2,
                   double epn, double *len_gam, double *ldet, double *wtw, double *lprior, double *llik,
                   double *lpost, int *err);
/* NestedLogistic (binary_smc.py:83-118) with device coeffs (p, p) and edgy (p): draw != 0: x (n, p) := rvs, from
 * u_in (p, n) (the reference's order of draws) or the context's Philox stream; logpdf (or NULL) = its log-density.
 * draw == 0: logpdf of the given x. */
int smcb_nested_logistic(smcb_ctx *ctx, int p, const double *coeffs, const uint8_t *edgy, int64_t n, int draw,
                         uint8_t *x, const double *u_in, double *logpdf);
/* MCMCSequenceWF.__call__ (smc_samplers.py:672-683) with BinaryMetropolis (binary_smc.py:154-162) under the tempered
 * target at exponent epn: ONE launch runs the P-1 steps of all M chains.  Inputs: the M resampled particles with
 * their lprior / llik / lpost; outputs: the P*M particles in concatenate(xs) order and pb_out (P-1, M), the
 * acceptance probabilities.  u_prop (P-1, p, M) and u_acc (P-1, M): injected uniforms, or both NULL.  *err as for
 * smcb_vs_loglik (bit 0). */
int smcb_binary_wf_move(smcb_ctx *ctx, const smcb_vs_desc *model, const double *coeffs, const uint8_t *edgy,
                        int64_t M, int P, double epn, const uint8_t *x0, const double *lprior0, const double *llik0,
                        const double *lpost0, const double *u_prop, const double *u_acc, uint8_t *x_out,
                        double *lprior_out, double *llik_out, double *lpost_out, double *pb_out, int *err);

/* AdaptiveTempering's control plane on the device (no host round trip inside a tempering step):
 * next_annealing_epn, smc_samplers.py:876-895: the exponent at which ESS(delta * llik) = alpha * n, by an 11-pass
 * 16-way bracketing search whose state stays in device memory; out_dev[0] = new exponent (1.0 if the whole step fits) */
int smcb_next_annealing_epn(smcb_ctx *ctx, const double *llik, int64_t n, double epn, double alpha, double *out_dev);
/* ArrayRandomWalk.calibrate, smc_samplers.py:617-622 (rs.wmean_and_cov, resampling.py:341-358): L_out (d, d)
 * row-major = scale * chol(weighted covariance of the rows of theta), d <= 20 */
int smcb_rw_calibrate(smcb_ctx *ctx, const double *W, const double *theta, int64_t n, int d, double scale,
                      double *L_out);

/* the same control plane in pieces, for a tempering run sharded over ranks (the host layer all-reduces between them):
 * raw ESS sums of one root-find pass; raw weighted-moment sums; the factor from all-reduced sums */
int smcb_essl_grid(smcb_ctx *ctx, const double *llik, int64_t n, double lo, double hi, const double *max_dev,
                   double *out32_dev);
int smcb_wcov_sums(smcb_ctx *ctx, const double *W, const double *theta, int64_t n, int d, const double *mean_dev,
                   double *out_dev);
int smcb_chol_from_sums(smcb_ctx *ctx, const double *tri_dev, const double *sw_dev, int d, double scale, double *L_out);

/* test hook: the kernels' own fp64 exp / log / sincos (csrc/smcb_math.cuh) on an array;
 * fn: 0 exp, 1 log (x > 0, normal), 2 sin(2 pi x), 3 cos(2 pi x), x in [0, 1)   -- polynomial family;
 *     4 exp, 5 log, 6 sin(2 pi x), 7 cos(2 pi x), 8 sqrt (x > 0, normal)        -- table family (step kernels) */
int smcb_device_math(smcb_ctx *ctx, int fn, const double *x, double *out, int64_t n);

/* ---------------------------------------------------------------------------
 * fused filter: the whole step of core.py:369-383 for a recognised model
 * ------------------------------------------------------------------------- */
#define SMCB_FK_BOOTSTRAP 0 /* state_space_models.py:299-349 */
#define SMCB_FK_GUIDED 1    /* state_space_models.py:352-398 */
#define SMCB_FK_APF 2       /* state_space_models.py:406-428 */
#define SMCB_FK_AUXBOOT 3   /* state_space_models.py:431-438 */

#define SMCB_MODEL_STOCHVOL 0      /* state_space_models.py:446-498             */
#define SMCB_MODEL_LINGAUSS 1      /* kalman.py:397-452 (also README ToySSM)    */
#define SMCB_MODEL_GORDON 2        /* state_space_models.py:546-577             */
#define SMCB_MODEL_THETALOGISTIC 3 /* state_space_models.py:657-689             */
#define SMCB_MODEL_BEARINGS 4      /* state_space_models.py:580-608 (d = 4)     */
#define SMCB_MODEL_MVLINGAUSS 5    /* kalman.py:296-394 (d <= 8)                */
#define SMCB_MODEL_DISCRETECOX 6   /* state_space_models.py:611-630             */
#define SMCB_MODEL_STOCHVOLLEV 7   /* state_space_models.py:501-543             */

#define SMCB_MAX_PARAMS 256
#define SMCB_SUMMARY_STRIDE 4 /* per step: ESS, logLt, rs_flag, log_mean_w */

typedef struct smcb_filter smcb_filter;

typedef struct {
    int32_t model, fk, scheme, dim;  /* dim = state dimension d                     */
    int32_t dy, n_params;
    int32_t world, rank;             /* particle shards over `world` GPUs (0/1 = one device) */
    int64_t n;                       /* particles on this device                    */
    int64_t n_global;                /* particles over all ranks (== n if 1 GPU)    */
    int64_t index_offset;            /* global index of local particle 0 (Philox)   */
    int64_t T;                       /* number of data points                       */
    double essrmin;
    uint64_t seed;
    double params[SMCB_MAX_PARAMS];  /* model constants, layout per model (DESIGN.md) */
    /* device buffers, all caller-owned */
    double *X[2];      /* ping-pong state, SoA (d, n)                               */
    double *lw[2];     /* ping-pong log-weights (n)                                 */
    int64_t *A;        /* ancestors of the last resampling step (n)                 */
    double *cdf;       /* (n) scratch: CDF of the last resampling step              */
    double *data;      /* (T, dy) observations                                      */
    double *summaries; /* (T, SMCB_SUMMARY_STRIDE)                                  */
    const double *z_in; /* NULL, or injected N(0,1): (T, n_noise, n)                */
    const double *u_in; /* NULL, or injected uniforms: (T, n + 1)                   */
    double *scratch;    /* NULL, or n + 2 doubles (multinomial: exponential spacings) */
    const double *step_consts; /* NULL, or (T) host-computed per-step model constants */
    double *local_stats;       /* world > 1: 16 doubles, this rank's weight statistics    */
    const double *gathered;    /* world > 1: world x 16 doubles, filled by the all-gather */
    double *mail_local;        /* world > 1, optional: this rank's peer mailbox (smcb_p2p_alloc,
                                  2 * world * 32 doubles) -> statistics are exchanged by the
                                  kernels themselves over NVLink and smcb_filter_step works */
    double *mail_peer[8];      /* every rank's mailbox as mapped in THIS process (own = mail_local) */
    /* world > 1, optional: EXACT global resampling (SURVEY.md section 8e, mode 2).  X[0], X[1] and cdf
       of every rank live in peer-mapped memory (smcb_p2p_alloc); on a resampling step each rank
       searches the global CDF (shard offsets from the exchanged statistics + the owning shard's
       local CDF) and pulls the selected ancestors over NVLink.  Needs mail_local; systematic or
       stratified. */
    int32_t rs_global, reserved0;
    double *moments;           /* NULL, or (T, 8): per step the weighted mean [0..3] and variance [4..7] of the
                                  state components (collectors.Moments with the default wmean_and_var,
                                  collectors.py:301-317, resampling.py:320-338), accumulated by the step kernel */
    double *reserved1;
    const double *peer_X0[8];  /* rank r's X[0] / X[1] / cdf as mapped in THIS process    */
    const double *peer_X1[8];
    const double *peer_cdf[8];
} smcb_filter_desc;

int smcb_filter_create(smcb_ctx *ctx, const smcb_filter_desc *desc, smcb_filter **out);
int smcb_filter_destroy(smcb_filter *f);
/* enqueue nsteps steps of SMC.__next__ (core.py:369-383); no host sync.  ONE kernel launch per step (its
 * prologue finalises the previous step) plus one single-CTA launch that finalises the last step of the batch. */
int smcb_filter_step(smcb_filter *f, int64_t nsteps);
/* sharded filter (SURVEY.md section 8e): particles are partitioned over `world` GPUs, one
 * process each.  With the host-driven exchange a step is step_local (this rank's kernels, ending
 * with its (max, sum exp, sum exp^2 [, moments]) in desc.local_stats), ONE all-gather of 16 doubles
 * per rank into desc.gathered done by the host layer on the same stream (NCCL), and step_finish
 * (global log-normaliser, ESS, logLt recursion and the resampling decision, identical on every
 * rank).  Resampling is per shard with the shard's mass carried in the restart log-weight. */
int smcb_filter_step_local(smcb_filter *f);
int smcb_filter_step_finish(smcb_filter *f);
/* peer memory for the fused exchange: alloc (zeroed) + 64-byte IPC handle to hand to the other
 * ranks (any transport), open a peer's handle, close / free */
int smcb_p2p_alloc(smcb_ctx *ctx, int64_t bytes, void **dev_ptr, unsigned char *handle64);
int smcb_p2p_open(smcb_ctx *ctx, const unsigned char *handle64, void **dev_ptr);
int smcb_p2p_close(void *peer_ptr);
int smcb_p2p_free(void *dev_ptr);
/* same, with a CUDA-event pair around every kernel launch; synchronises at the end.
 * out[0..3] = summed device ms of {init, step kernels of resampling steps, tail, step kernels of
 * non-resampling steps}, out[4..7] = launches of each (bench.py "roofline") */
int smcb_filter_step_timed(smcb_filter *f, int64_t nsteps, double *out8);
/* host-visible snapshot (synchronises the stream):
 * out[0]=t, [1]=cur buffer index, [2]=rs_flag of last step, [3]=logLt, [4]=ESS,
 * [5]=log_mean_w, [6]=max lw, [7]=sum w */
int smcb_filter_state(smcb_filter *f, double *out8);
/* fused pairs of streaming steps (env SMCB_FUSE, read at smcb_filter_create: 0 off, 1 on, 2 fuse whenever
 * allowed): out[0] = launches that ran their step and the next one, out[1] = launches whose step was already
 * done (no-op), out[2] = launches whose pre-computed step resampled after all (misprediction).  Synchronises. */
int smcb_filter_fusion_stats(smcb_filter *f, int64_t *out3);

/* ---------------------------------------------------------------------------
 * sequential quasi-Monte Carlo  (particles/core.py:315-349, rqmc.py, hilbert.py)
 * ------------------------------------------------------------------------- */
/* rqmc.sobol(n, d) for 1 <= d <= 4096: scipy.stats.qmc.Sobol's 30-bit points 0 .. n-1, squeezed into
 * u = 0.5 + (1 - 1e-10) (p - 0.5); u and raw (the 30-bit integers) are component-major (d, n), either may be NULL.
 * scramble != 0: a random lower-triangular bit matrix and digital shift per dimension, drawn from Philox under
 * (seed, call, dimension), so that dimension j's points do not depend on d; scramble = 0: scipy's scramble=False
 * points, bit for bit. */
int smcb_sobol(smcb_ctx *ctx, int d, int64_t n, int scramble, uint64_t seed, uint64_t call, double *u,
               int32_t *raw);
/* hilbert.hilbert_sort(x) for SoA (d, n) points, 1 <= d <= 32: order = np.argsort(x) for d = 1, otherwise the
 * argsort of the int64 Hilbert keys of floor(invlogit(standardised x) * floor(2^(62/d))), which wrap as the
 * reference's do (signed comparison).  keys (d > 1, may be NULL) = the unsorted keys.  Equal keys come out in any
 * order.  scratch: smcb_hilbert_scratch_bytes(n, d) bytes, 256-byte aligned (-1: bad sizes). */
int64_t smcb_hilbert_scratch_bytes(int64_t n, int d);
int smcb_hilbert_sort(smcb_ctx *ctx, const double *x, int64_t n, int d, int64_t *order, int64_t *keys,
                      void *scratch);
/* nsteps SQMC steps (resample_move_qmc, always resampling) of a filter made by smcb_filter_create, which fixes the
 * model, kind, buffers and seed (desc.scheme and desc.essrmin are ignored; desc.moments must be NULL).  Step t draws
 * the points of smcb_sobol(du (+ 1), n, 1, desc.seed, t) with du = the state dimension -- or, when desc.u_in is not
 * NULL, the caller's points: T blocks of (du + 1, n) doubles, component-major, step 0 reading the first du rows of
 * block 0 (parity tests against recorded point sets) -- writes X[t & 1], lw[t & 1],
 * A and summary row t (rs_flag 1 from t = 1).  No host sync.  scratch: smcb_sqmc_scratch_bytes(n, dim) bytes,
 * 256-byte aligned (-1: bad sizes). */
int64_t smcb_sqmc_scratch_bytes(int64_t n, int dim);
/* out = Phi^-1(u) (scipy.special.ndtri, within 8 ulp on the squeezed Sobol' range): the ppf of Normal and MvNormal */
int smcb_ndtri(smcb_ctx *ctx, const double *u, double *out, int64_t n);
int smcb_sqmc_step(smcb_filter *f, int64_t nsteps, void *scratch);

/* ---------------------------------------------------------------------------
 * off-line smoothing: FFBS backward sampling over a stored history (particles/smoothing.py:278-423)
 * ------------------------------------------------------------------------- */
#define SMCB_SMOOTH_ON2 0    /* backward_sampling_ON2,    smoothing.py:291-311 */
#define SMCB_SMOOTH_MCMC 1   /* backward_sampling_mcmc,   smoothing.py:313-350 */
#define SMCB_SMOOTH_REJECT 2 /* backward_sampling_reject, smoothing.py:352-423 (hybrid, Dau & Chopin 2022) */
#define SMCB_SMOOTH_GATHER 3 /* paths[t] = X[t][idx[t]] only (idx given; model ignored) */

typedef struct {
    int32_t method, model, dim, n_params;
    int64_t T, N, M;
    int64_t nsteps;            /* MCMC: Metropolis steps per time                                  */
    int64_t max_trials;        /* reject: proposals per trajectory before the exact O(N) draw      */
    double params[SMCB_MAX_PARAMS];  /* model constants, same layout as smcb_filter_desc.params    */
    const double *step_consts; /* NULL, or (T) per-step model constants (Gordon_etal)              */
    /* the history: device arrays of T device pointers; X[t] holds particle n, component c at
       X[t][n * x_stride_n + c * x_stride_c] (element strides, the same for every t) */
    const double *const *X;
    const double *const *lw;   /* (N) log-weights per t                                             */
    const int64_t *const *A;   /* (N) ancestors per t (entry 0 unused)                              */
    int64_t x_stride_n, x_stride_c;
    const double *log_bound;   /* reject: (T-1), entry t = log C_{t+1} >= log p(x_{t+1} | x_t)       */
    const double *cdf;         /* MCMC / reject: (T-1, cdf_ld) rows, the inclusive prefix sums of W_t */
    int64_t cdf_ld;            /* row stride of cdf (>= N; even, so that every row is 16-byte aligned) */
    const int64_t *idx_T;      /* (M) the final-time indices (drawn by the caller)                  */
    /* injected randomness (parity tests) or NULL -> Philox keyed by (seed, call, m, t, trial):
       ON2 u (M, T-1) [m, t]; MCMC prop / lu (T-1, nsteps, M); reject prop / lu (T-1, M, max_trials)
       and u_exact (T-1, M) for the exact fallback draw */
    const double *u;
    const int64_t *prop;
    const double *lu;
    const double *u_exact;
    int64_t *idx;              /* out (T, M): idx[T-1] = idx_T; GATHER: input                       */
    double *paths;             /* out (T, M, dim) = X[t][idx[t]]                                    */
    int64_t *counts;           /* reject: out (T-1, 2) {accepted, proposals} (zeroed here)          */
    /* ON2 only: NULL (index order), or a device array of T-1 device pointers, order[t] a permutation of 0 .. N-1:
       the draw at t walks the CDF of particles order[t][0], order[t][1], ... (QMC backward sampling over the
       Hilbert orders of an SQMC history, smoothing.py:425-455); idx stays in particle indices */
    const int64_t *const *order;
} smcb_smooth_desc;

/* ONE kernel launch for the whole backward pass (plus a memset of counts for reject); no host sync */
int smcb_backward_sample(smcb_ctx *ctx, const smcb_smooth_desc *desc);

/* ---------------------------------------------------------------------------
 * on-line smoothing of additive functionals (particles/collectors.py:345-449): one step t >= 1 of the PaRIS and
 * O(N^2) collectors.  The caller evaluates the user's add_func psi between the launches.
 * ------------------------------------------------------------------------- */
#define SMCB_ONLINE_PARIS 0     /* B[n, i] ~ p(a | x_t^n) prop. to W_{t-1}[a] p_t(x_t^n | x_{t-1}^a), j = n*Np + i:
                                   at most max_trials proposals a ~ W_{t-1} accepted w.p. p_t / C_t, then the
                                   exact O(N) draw (hybrid PaRIS, Dau & Chopin 2022) */
#define SMCB_ONLINE_ON2_W 1     /* omega (rows, N): omega[r, m] = W_{t-1}[m] p_t(x_t^{row0+r} | x_{t-1}^m), normalised
                                   per row */
#define SMCB_ONLINE_PHI_PARIS 2 /* phi[n] = (sum_i phi_prev[B[n, i]] + psi[n, i]) / Np  (model ignored) */
#define SMCB_ONLINE_PHI_ON2 3   /* phi[r] = sum_m omega[r, m] (phi_prev[m] + psi[r, m]) / sum_m omega[r, m] */

typedef struct {
    int32_t method, model, dim, n_params;
    int64_t t;                 /* the time of X; the density is logpt(t, X_prev, X) */
    int64_t N;                 /* particles at t - 1 and t                                          */
    int64_t Np;                /* PaRIS: draws per particle (Nparis)                                 */
    int64_t max_trials;        /* PaRIS: proposals per draw before the exact draw                     */
    int64_t row0, rows;        /* ON2: the block of rows [row0, row0 + rows) of X                     */
    int64_t k;                 /* PHI: components of phi / psi                                        */
    uint64_t seed;             /* PaRIS: Philox key; the draws are keyed by (seed, t, j, trial)         */
    double log_bound;          /* PaRIS: log C_t >= log p_t(x | xp)                                   */
    double step_const;         /* the model's per-step constant of step t (Gordon_etal), else 0        */
    double params[SMCB_MAX_PARAMS];  /* model constants, same layout as smcb_filter_desc.params         */
    /* X_{t-1} and X_t: particle n, component c at X[n * x_stride_n + c * x_stride_c] (element strides) */
    const double *X_prev;
    const double *X;
    int64_t x_stride_n, x_stride_c;
    const double *lw_prev;     /* (N) log-weights of t - 1                                            */
    const double *cdf;         /* PaRIS: (N) inclusive prefix sum of W_{t-1} (any positive scale)      */
    /* injected randomness (parity tests) or NULL: prop / lu (N, Np, max_trials), u_exact (N, Np)     */
    const int64_t *prop;
    const double *lu;
    const double *u_exact;
    int64_t *B;                /* PaRIS: out (N, Np); PHI_PARIS: in                                    */
    int64_t *counts;           /* PaRIS: {accepted, proposals} += this step's (integer atomics)        */
    double *omega;             /* ON2_W: out (rows, N); PHI_ON2: in                                    */
    const double *phi_prev;    /* PHI: (N, k)                                                          */
    const double *psi;         /* PHI_PARIS: (N, Np, k); PHI_ON2: (rows, N, k)                         */
    double *phi;               /* PHI: out (rows, k) (PARIS: rows = N)                                 */
} smcb_online_desc;

/* one kernel launch, no host sync */
int smcb_online_smooth(smcb_ctx *ctx, const smcb_online_desc *desc);

/* ---------------------------------------------------------------------------
 * two-filter smoothing (particles/smoothing.py:487-566) of a forward generation X_t (N particles, log-weights lw)
 * against an information generation Xinfo (Ninfo particles), one-dimensional states only; the pair density is
 * logpt(t + 1, X_t[n], Xinfo[m]).  The caller evaluates the user's phi between the launches and combines the rows
 * (exp_and_normalise of lwinfo + L, dotted with S).
 * ------------------------------------------------------------------------- */
#define SMCB_TF_ON2_ROWS 0  /* rows [row0, row0 + rows) of Xinfo, one pass over n, omega never stored:
                               L[m] = log sum_n exp(v_nm), S[m] = sum_n exp(v_nm - L[m]) psi[m - row0, n],
                               v_nm = lw[n] + logpt(t + 1, X_t[n], Xinfo[m]); a row with no positive pair weight
                               gives L = -inf, S = 0.  Partial sums merge in a fixed order (bits = f(inputs)) */
#define SMCB_TF_ON_LOGW 1   /* one thread per draw j: log_omega[j] = logpt(t + 1, X_t[J[j]], Xinfo[I[j]])
                               - mf[J[j]] - mi[I[j]] (mf, mi may be NULL); xf[j] = X_t[J[j]], xi[j] = Xinfo[I[j]] */

typedef struct {
    int32_t method, model, dim, n_params;
    int64_t t;                 /* forward time; the density is logpt(t + 1, X_t, Xinfo)                  */
    int64_t N, Ninfo;          /* particles of X_t and of Xinfo                                          */
    int64_t row0, rows;        /* ON2_ROWS: the block of rows of Xinfo                                   */
    int64_t M;                 /* ON_LOGW: draws                                                         */
    double step_const;         /* the model's per-step constant of step t + 1 (Gordon_etal), else 0      */
    double params[SMCB_MAX_PARAMS];  /* model constants, same layout as smcb_filter_desc.params          */
    /* particle n at X[n * x_stride], m at Xinfo[m * xi_stride] (element strides)                        */
    const double *X;
    const double *Xinfo;
    int64_t x_stride, xi_stride;
    const double *lw;          /* ON2_ROWS: (N) forward log-weights at t                                 */
    const double *psi;         /* ON2_ROWS: (rows, N) phi(X_t[n], Xinfo[row0 + r]) at [r, n]             */
    double *L, *S;             /* ON2_ROWS: out (Ninfo), rows [row0, row0 + rows) written               */
    const int64_t *I, *J;      /* ON_LOGW: (M) indices into Xinfo and X_t (in range: not checked)        */
    const double *mf, *mi;     /* ON_LOGW: NULL or (N) / (Ninfo) log-modifiers                           */
    double *log_omega;         /* ON_LOGW: out (M)                                                       */
    double *xf, *xi;           /* ON_LOGW: out (M) the gathered pairs                                    */
} smcb_twofilter_desc;

/* one kernel launch, no host sync; a model whose state is not one-dimensional -> SMCB_ENOSYS */
int smcb_two_filter(smcb_ctx *ctx, const smcb_twofilter_desc *desc);

/* ---------------------------------------------------------------------------
 * genealogy-based variance estimators (particles/variance_estimators.py:93-201): the Eve indices of a running filter
 * and the branch sums  sum_b (sum_{m: B_m = b} v_m)^2  over SORTED rows B, so that each branch is a contiguous run.
 * ------------------------------------------------------------------------- */
#define SMCB_VAR_EVE 0          /* if the step resampled: B[p ^ 1][n] = B[p][A[n]], p = *parity (one launch) */
#define SMCB_VAR_SUMS 1         /* the branch sums of L rows, k components each (four launches, then *parity ^= rs) */
#define SMCB_VAR_CENTRED 0      /* v = W (phi - m), m = sum W phi / sum W; zeros where B[0] == B[N-1] (Var)    */
#define SMCB_VAR_WEIGHTS 1      /* v = W, no centring and no zero rule (Var_logLt)                              */

typedef struct {
    int32_t method, mode;
    int32_t lin_w;             /* lw holds the weights W themselves (var_estimate), else log-weights: W = exp(lw) / sum */
    int32_t rs_host;           /* the step's resampling flag when rs_flag is NULL                                */
    int64_t N, k, L;           /* particles, components of phi (1 in WEIGHTS mode), rows of B                     */
    const double *rs_flag;     /* device: the step resampled when nonzero (the filter's summaries[t, 2]), or NULL */
    int32_t *parity;           /* device word: the Eve row is B[*parity] (B[*parity ^ rs] after EVE); NULL: B[0]   */
    int64_t *B[2];             /* EVE: the ping-pong pair of (N) rows; SUMS: (L, N) rows at B[cur]              */
    const int64_t *A;          /* EVE: the step's ancestors (read only when the step resampled)                  */
    const double *lw;          /* SUMS: (N) log-weights (or W), the mean and the normaliser                       */
    const double *phi;         /* SUMS, CENTRED: (N, k) row-major                                                */
    const double *lw_rows;     /* SUMS: row r reads lw_rows + r * row_ld and phi_rows + r * row_ld * k           */
    const double *phi_rows;
    int64_t row_ld;            /* 0 when every row reads lw and phi (sorted rows)                                 */
    const uint8_t *zero;       /* CENTRED: (L) the B[0] == B[N-1] rule decided by the caller, or NULL: on the row */
    int32_t *unsorted;         /* (L) set to 1 when a row is not sorted (never cleared here)                      */
    double *scratch;           /* smcb_variance_scratch_doubles(N, L, k) doubles                                   */
    double *out;               /* (L, k) the estimates                                                            */
} smcb_variance_desc;

/* no host sync; the chunk size is a function of N only, so the bits do not depend on the device */
int smcb_variance(smcb_ctx *ctx, const smcb_variance_desc *desc);
int64_t smcb_variance_scratch_doubles(int64_t N, int64_t L, int64_t k);

/* ---------------------------------------------------------------------------
 * batched filters (multiSMC): R independent filters of the same model, Feynman-Kac kind, scheme, N and T in ONE
 * launch, one CTA per filter (csrc/smcb_batch.cu).  1-D fused models only.  Run r draws what the single filter
 * with seed seed[r] draws (same Philox counters); the two differ only in reduction order.
 * Per-run rows are padded to ld = N rounded up to even (16-byte aligned rows).
 * ------------------------------------------------------------------------- */
#define SMCB_BATCH_AUTO 0      /* resident if the filter fits in shared memory, else streaming */
#define SMCB_BATCH_RESIDENT 1  /* x, lw and the CDF stay in shared memory for the whole run     */
#define SMCB_BATCH_STREAMING 2 /* per-run buffers in device memory; any N                       */

typedef struct {
    int32_t model, fk, scheme, dim;  /* dim must be 1                                              */
    int32_t dy, n_params;
    int32_t tier, reserved0;         /* SMCB_BATCH_*                                               */
    int64_t N, T, R;
    const uint64_t *seed;      /* (R) Philox key of each run                                        */
    const double *essrmin;     /* (R)                                                               */
    const double *params;      /* (R, n_params) model constants, layout of smcb_filter_desc.params  */
    const double *data;        /* (R, T, dy) observations                                           */
    const double *step_consts; /* (R, T) or NULL                                                    */
    double *X;                 /* (R, 2, ld): generation s of the last two in X[r][s & 1]           */
    double *lw;                /* (R, ld) log-weights of step T - 1                                 */
    int64_t *A;                /* (R, ld) ancestors of step T - 1 (written only if it resampled)    */
    double *cdf;               /* streaming: (R, ld) scratch; resident: unused                      */
    double *scratch;           /* streaming multinomial: (R, ld + 2) exponential spacings           */
    double *summaries;         /* (R, T, SMCB_SUMMARY_STRIDE)                                       */
    double *moments;           /* NULL, or (R, T, 8) as smcb_filter_desc.moments                    */
    const double *z_in;        /* NULL, or injected N(0,1): (R, T, n_noise, N)                      */
    const double *u_in;        /* NULL, or injected uniforms: (R, T, N + 1)                         */
} smcb_batch_desc;

/* out[0] = the tier a run with this descriptor takes, out[1] = its grid (CTAs).  Reads only the shape fields.
 * SMCB_ENOSYS for a combination that is not built (the caller runs those filters one by one). */
int smcb_batch_plan(smcb_ctx *ctx, const smcb_batch_desc *desc, int64_t out[2]);
/* one launch on the context's stream, no host sync */
int smcb_batch_run(smcb_ctx *ctx, const smcb_batch_desc *desc);

/* ---------------------------------------------------------------------------
 * filter bank (SMC^2, particles/smc_samplers.py:1038-1167): R resumable filters of one 1-D fused model, Feynman-Kac
 * kind, scheme, N and data, each with its own model constants and Philox key, kept in device rows between launches
 * (csrc/smcb_bank.cu).  The geometry and the step body are those of the batched filters: advancing a filter over
 * [0, t) and then [t, t1) gives the bits of advancing it over [0, t1) in one call, and filter r draws what the
 * batched run (and the single filter) with seed key[r] draws.  Rows are padded to ld = N rounded up to even.
 * ------------------------------------------------------------------------- */
#define SMCB_BANK_STATE 8 /* per filter: steps done t, logLt, log_mean_w of step t - 1, APF restart constant,
                             max and sum exp of the auxiliary log-weights, resampling decided for step t (0 / 1),
                             loglt of step t - 1 */

typedef struct {
    int32_t model, fk, scheme, tier; /* tier: SMCB_BATCH_*                                          */
    int32_t n_params, restart;       /* restart != 0: every selected filter starts from M0 (step 0) */
    int64_t N, T, R;                 /* particles per filter, data points, filters in the bank       */
    int64_t t1;                      /* advance: every selected filter runs up to (excluding) step t1 */
    const int64_t *idx;        /* (n_idx) the filters to advance, or NULL: all R; the others are not read or written */
    int64_t n_idx;
    double essrmin;
    uint64_t *key;             /* (R) Philox key of each filter                                       */
    double *params;            /* (R, n_params) model constants, layout of smcb_filter_desc.params    */
    const double *data;        /* (T) observations, shared by every filter                            */
    double *step_consts;       /* NULL, or (R, sc_ld) per-filter rows, or one (T) row when sc_ld == 0 */
    int64_t sc_ld;
    double *X;                 /* (R, 2, ld): generation s of the last two in X[r][s & 1]              */
    double *lw;                /* (R, ld) log-weights of the last step                                 */
    double *state;             /* (R, SMCB_BANK_STATE)                                                 */
    int64_t *A;                /* NULL, or (R, ld): ancestors of step t1 - 1 (written only if it resampled) */
    double *summaries;         /* NULL, or (R, T, SMCB_SUMMARY_STRIDE): rows of the steps this call runs */
    double *cdf;               /* streaming: (scratch_rows, ld) scratch, one row per CTA of the grid   */
    double *scratch;           /* streaming multinomial: (scratch_rows, ld + 2) exponential spacings   */
    int64_t scratch_rows;      /* >= the grid smcb_bank_plan returns                                   */
} smcb_bank_desc;

/* out[0] = the tier, out[1] = the grid (CTAs) an advance with this descriptor takes.  Reads only the shape fields,
 * idx and n_idx.  SMCB_ENOSYS for a combination that is not built. */
int smcb_bank_plan(smcb_ctx *ctx, const smcb_bank_desc *desc, int64_t out[2]);
/* SMC.__next__ (core.py:369-383) for every selected filter r from step state[r][0] (0 when restart) up to step t1;
 * writes X, lw, state (logLt in state[r][1], loglt of step t1 - 1 in state[r][7]) and the optional A / summaries.
 * A filter already at t1 or beyond is left as it is.  One launch, no host sync. */
int smcb_bank_advance(smcb_ctx *ctx, const smcb_bank_desc *desc);
/* dst[i] = src[A[i]] for i < m (X, lw, state, params, per-filter step constants, key): the outer sampler's X[A]
 * (FancyList / all_distinct, particles/smc_samplers.py:319-361).  The first copy of an ancestor (lowest i) keeps its
 * key; every further copy gets the key number counter + i under seed (smcb_bank_keys), so copies draw independent
 * streams.  dst must not alias src; first: (src->R) scratch words.  Three launches, no host sync. */
int smcb_bank_gather(smcb_ctx *ctx, const smcb_bank_desc *src, const int64_t *A, int64_t m,
                     const smcb_bank_desc *dst, uint64_t seed, uint64_t counter, uint64_t *first);
/* dst[i] = src[i] (all rows, key included) where accepted[i] != 0: the bank half of the Metropolis copy-where
 * (ThetaParticles.copyto, particles/smc_samplers.py:601-611).  One launch. */
int smcb_bank_merge(smcb_ctx *ctx, const smcb_bank_desc *dst, const smcb_bank_desc *src, const uint8_t *accepted);
/* key[i] = the key number counter + i under seed: fmix64(fmix64(seed) + counter + i), fmix64 the splitmix64
 * finaliser, a bijection -- distinct numbers give distinct keys.  One launch. */
int smcb_bank_keys(smcb_ctx *ctx, uint64_t *key, int64_t n, uint64_t seed, uint64_t counter);
/* smcb_mh_accept that also writes accepted[i] = 1 where the proposal was taken, else 0 (the mask smcb_bank_merge
 * reads) */
int smcb_mh_accept_flags(smcb_ctx *ctx, int64_t n, int d, double *theta, double *lprior, double *llik,
                         double *lpost, const double *theta_p, const double *lprior_p, const double *llik_p,
                         const double *lpost_p, const double *u_in, double *mean_acc, uint8_t *accepted);

/* ---------------------------------------------------------------------------
 * conditional SMC (Particle Gibbs, particles/mcmc.py:453-475 and 594-609): R chains, one filter of N particles each,
 * of one 1-D model and the Bootstrap or Guided kind, multinomial resampling when ESS < ESSrmin N, each with its own
 * model constants, Philox key and reference path x* (csrc/smcb_pmcmc.cu).  Slot 0 is pinned to x*: x*[0] at step 0,
 * then ancestor 0 and state x*[t], weighted by logG(t, x*[t-1], x*[t]).  With pin = 0 the same pass runs
 * unconditionally and chain r gives the bits of the filter bank's multinomial filter with key[r].  The whole history
 * is kept, and the same launch draws one new trajectory per chain from it.  Rows are padded to ld = N rounded up to
 * even.
 * ------------------------------------------------------------------------- */
#define SMCB_CSMC_GENEALOGY 0 /* trace the ancestors of one draw from W_{T-1} (smoothing.py:256-269)     */
#define SMCB_CSMC_BACKWARD 1  /* one backward draw per step, backward_sampling_ON2(1) (smoothing.py:291-311) */

typedef struct {
    int32_t model, fk, n_params, draw; /* fk: SMCB_FK_BOOTSTRAP or SMCB_FK_GUIDED; draw: SMCB_CSMC_*     */
    int32_t pin, reserved0;            /* pin != 0: slot 0 follows xstar                                 */
    int64_t N, T, R;                   /* particles per chain, data points, chains                      */
    double essrmin;
    const uint64_t *key;       /* (R) Philox key of each chain                                         */
    const double *params;      /* (R, n_params) model constants, layout of smcb_filter_desc.params     */
    const double *data;        /* (R, data_ld) observations; data_ld = 0: one (T) row shared by all    */
    int64_t data_ld;
    const double *step_consts; /* NULL, or (R, sc_ld) per-chain rows, or one (T) row when sc_ld == 0   */
    int64_t sc_ld;
    const double *xstar;       /* (R, T) reference paths (read only when pin != 0)                     */
    double *X;                 /* (R, T, ld) particles of every step                                   */
    double *lw;                /* (R, T, ld) log-weights of every step                                 */
    int64_t *A;                /* (R, T, ld) ancestors of every step (arange where a step does not resample) */
    double *traj;              /* (R, T) the drawn trajectory                                          */
    double *logLt;             /* (R) log-likelihood estimate                                          */
    double *summaries;         /* NULL, or (R, T, SMCB_SUMMARY_STRIDE)                                 */
    const double *z_in;        /* NULL, or (R, T, N) injected normals                                  */
    const double *u_in;        /* NULL, or (R, T, N + 1) injected uniforms of the multinomial spacings */
    const double *ud_in;       /* NULL, or (R, T) injected uniforms of the trajectory draw at step t   */
} smcb_csmc_desc;

/* out[0] = the largest N the shared memory of this device holds for this model and kind, out[1] = the grid (CTAs).
 * SMCB_ENOSYS for a combination that is not built or an N above the bound. */
int smcb_csmc_plan(smcb_ctx *ctx, const smcb_csmc_desc *desc, int64_t out[2]);
/* the forward pass and the trajectory draw of every chain: one launch on the context's stream, no host sync */
int smcb_csmc_run(smcb_ctx *ctx, const smcb_csmc_desc *desc);

/* ---------------------------------------------------------------------------
 * hidden Markov models (particles/hmm.py, BaumWelch): B finite-state HMMs with K <= SMCB_HMM_MAX_K states.
 * Per-HMM arrays are time-major rows of a buffer of `ld` rows: element (b, t, k) of pred / filt / logft / smth is
 * at [(b * ld + t) * K + k], logpyt (b, t) at [b * ld + t].  trans (b) is at trans + b * trans_stride (K x K, row
 * j = from-state), init (b) at init + b * init_stride; a stride of 0 shares one matrix / vector across the batch.
 * K <= 32 runs one warp per HMM, 33 <= K <= 128 one CTA per HMM; every sum over states is a fixed tree (warps: xor
 * butterfly; across warps: in warp order), so the bits depend on the inputs only.
 * ------------------------------------------------------------------------- */
#define SMCB_HMM_MAX_K 128
#define SMCB_HMM_FORWARD 0  /* rows [t0, t1): pred_t = filt_{t-1} P (sum in j order; init at t = 0),
                               lp = log pred_t + logft_t, logpyt_t = LSE(lp), filt_t = exp(lp - logpyt_t)       */
#define SMCB_HMM_BACKWARD 1 /* rows [0, t1): ctg_k <- LSE_j(log P_kj + logft_{t+1,j} + ctg_j),
                               smth_t = exp_and_normalise(log filt_t + ctg), smth_{t1-1} = filt_{t1-1}         */
#define SMCB_HMM_SAMPLE 2   /* rows t1-2 .. 0 of N trajectories per HMM, given paths row t1-1: per t the K column
                               CDFs C[j][k] = cumsum_k exp_and_normalise_k(log P_kj + log filt_t,k), the draw
                               #{k : C[path_{t+1}][k] < u}, clipped to K - 1; u = U[(b, t, n)] if U, else
                               Philox(seed; n, t, b) under its own purpose                                   */

typedef struct {
    int32_t method, K;
    int64_t B;                 /* HMMs                                                                     */
    int64_t ld;                /* rows per HMM in the time-major buffers                                   */
    int64_t t0, t1;            /* FORWARD: rows [t0, t1); BACKWARD / SAMPLE: t1 = T rows filled            */
    int64_t N;                 /* SAMPLE: trajectories per HMM                                             */
    uint64_t seed;             /* SAMPLE: Philox key when U is NULL                                        */
    const double *trans;       /* (K, K) per HMM                                                           */
    int64_t trans_stride;
    const double *init;        /* (K) per HMM                                                              */
    int64_t init_stride;
    const double *logft;       /* (B, ld, K) log-density of y_t given x_t = k                              */
    double *pred, *filt;       /* (B, ld, K) FORWARD out; filt read by BACKWARD / SAMPLE                   */
    double *logpyt;            /* (B, ld) FORWARD out                                                      */
    double *smth;              /* (B, ld, K) BACKWARD out                                                  */
    const double *U;           /* SAMPLE: NULL, or (B, t1 - 1, N) injected uniforms                        */
    int64_t *paths;            /* SAMPLE: (B, t1, N); row t1 - 1 is read, rows t1 - 2 .. 0 written         */
} smcb_hmm_desc;

/* one kernel launch on the context's stream, no host sync; K > SMCB_HMM_MAX_K -> SMCB_ENOSYS */
int smcb_hmm(smcb_ctx *ctx, const smcb_hmm_desc *desc);

/* ---------------------------------------------------------------------------
 * Kalman filter and RTS smoother (particles/kalman.py, Kalman): B linear-Gaussian models X_t = F X_{t-1} + U,
 * Y_t = G X_t + V with dx, dy <= SMCB_KALMAN_MAX_D.  Per-model arrays are time-major rows of a buffer of `ld` rows:
 * mean (b, t, i) at [(b * ld + t) * dx + i], cov (b, t, i, j) at [((b * ld + t) * dx + i) * dx + j], logpyt (b, t)
 * at [b * ld + t]; observation (b, t, i) at y[b * y_stride + t * dy + i].  Parameter (b) is at p + b * p_stride
 * (F, covX, cov0: dx x dx; G: dy x dx; covY: dy x dy; mu0: dx, all row-major); a stride of 0 shares it.
 * dx = dy = 1 runs one thread per model, otherwise one warp per model; every sum runs in index order, so the bits
 * depend on the inputs only.  A non-positive Cholesky pivot (S or P_{t+1} not positive definite) gives NaN, which
 * fills that model's rows from that step on.
 * ------------------------------------------------------------------------- */
#define SMCB_KALMAN_MAX_D 32
#define SMCB_KALMAN_FILTER 0 /* rows [t0, t1): pred = (mu0, cov0) at t = 0, else (F m, (F Sig) F' + covX);
                                S = (G P) G' + covY, K = P G' S^-1 through chol(S), filt = (m + K r, P - (K G) P),
                                logpyt: N(G pm, S) log-density of y_t                                           */
#define SMCB_KALMAN_SMOOTH 1 /* rows [0, t1): J = Sig_f F' P_{t+1}^-1 through chol(P_{t+1}),
                                smth = (m_f + J (m_s' - m_{t+1}), Sig_f + (J (Sig_s' - P_{t+1})) J'),
                                smth_{t1-1} = filt_{t1-1}                                                       */

typedef struct {
    int32_t method, dx, dy, pad_;
    int64_t B;                 /* models                                                                   */
    int64_t ld;                /* rows per model in the time-major buffers                                 */
    int64_t t0, t1;            /* FILTER: rows [t0, t1); SMOOTH: t1 = T rows filtered                      */
    const double *F, *G, *covX, *covY, *mu0, *cov0;
    int64_t F_stride, G_stride, covX_stride, covY_stride, mu0_stride, cov0_stride;
    const double *y;           /* FILTER: observations                                                     */
    int64_t y_stride;
    double *pred_mean, *pred_cov, *filt_mean, *filt_cov;   /* FILTER out; read by SMOOTH                   */
    double *logpyt;            /* FILTER out                                                               */
    double *smth_mean, *smth_cov;                          /* SMOOTH out                                   */
} smcb_kalman_desc;

/* one kernel launch on the context's stream, no host sync; dx or dy > SMCB_KALMAN_MAX_D -> SMCB_ENOSYS */
int smcb_kalman(smcb_ctx *ctx, const smcb_kalman_desc *desc);

#ifdef __cplusplus
}
#endif
#endif /* SMCB_H */
