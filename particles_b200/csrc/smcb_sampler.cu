// smcb_sampler.cu -- kernels of the tempering / waste-free SMC sampler move step
// (particles/smc_samplers.py:596-629, 669-683, 797-936; BASELINE config 5):
//   * tempered target of the Bayesian logistic regression: log prior, log-likelihood
//     sum_t -log(1 + exp(-theta . x_t)) and log posterior for N parameter vectors at once
//     (StaticModel.loglik loops over the data rows in Python, smc_samplers.py:263-284);
//   * Gaussian random-walk proposal theta + z @ L.T (ArrayRandomWalk.proposal, 624-629);
//   * Metropolis accept / copy-where (ArrayMetropolis.step, 601-611).
// The log-likelihood is the only dense contraction on the path ((N x d) . (d x n_data) followed by a
// softplus row-reduce).  It stays fp64 on the CUDA cores: the contraction is 2d = 40 flops per
// (particle, datum) against ~50 fp64 instructions of softplus, so tensor cores would not move the
// bound, and lower precision would change results (SURVEY.md section 8 row a23).
#include "smcb_common.cuh"
#include "smcb_math.cuh"
#include "smcb_reduce.cuh"

using namespace smcb;

namespace smcb {

constexpr int kSampBlock = 128;
constexpr int kRowsPerTile = 32;       // data rows staged in shared memory per pass

// -log(1 + exp(-lin)) = -(max(v, 0) + log1p(exp(-|v|))), v = -lin   (np.logaddexp(0, v)).  A NaN lin (a NaN
// parameter, or infinite ones whose products cancel) must give NaN, which the row sum turns into -inf as the
// reference does: fmax drops a NaN and flog_pos reads one as a finite number, so it is passed through explicitly.
__device__ __forceinline__ double neg_softplus_neg(double lin) {
    const double v = -lin;
    const double e = fexp_neg(-fabs(v));
    const double g = -(fmax(v, 0.0) + flog_pos(1.0 + e));
    return (lin != lin) ? lin : g;
}

// theta: (n, d) row-major.  D = d rounded up to a supported size (extra coordinates are zero).
// Each thread owns TWO parameter vectors, so every data value read from shared memory feeds two
// FMAs.  The sum over data rows runs in row order, as the reference's Python loop does.
// FLOOR (NestedSamplingSMC.current_target, nested.py:353-363): the argument epn is the likelihood floor lmin
// and lpost = lprior where llik >= lmin, -inf elsewhere.  Reusing the argument keeps the tempered
// instantiations' parameter layout, so they compile to the same code as before.
template <int D, bool FLOOR = false>
__global__ void __launch_bounds__(kSampBlock) k_logistic_target(
    const double *__restrict__ theta, int64_t n, int d, const double *__restrict__ data, int64_t n_data,
    double prior_scale, double prior_lognorm, double epn, double *__restrict__ lprior,
    double *__restrict__ llik, double *__restrict__ lpost) {
    __shared__ __align__(16) double s_x[kRowsPerTile * D];
    const int64_t i0 = 2 * ((int64_t)blockIdx.x * kSampBlock + threadIdx.x);
    const bool v0 = i0 < n, v1 = i0 + 1 < n;
    double th0[D], th1[D];
#pragma unroll
    for (int j = 0; j < D; j++) {
        th0[j] = (v0 && j < d) ? theta[i0 * d + j] : 0.0;
        th1[j] = (v1 && j < d) ? theta[(i0 + 1) * d + j] : 0.0;
    }
    double l0 = 0.0, l1 = 0.0;
    for (int64_t r0 = 0; r0 < n_data; r0 += kRowsPerTile) {
        const int rows = (int)((n_data - r0) < kRowsPerTile ? (n_data - r0) : kRowsPerTile);
        __syncthreads();
        for (int e = threadIdx.x; e < rows * D; e += kSampBlock) {
            const int r = e / D, j = e - r * D;
            s_x[e] = (j < d) ? data[(r0 + r) * d + j] : 0.0;
        }
        __syncthreads();
        for (int r = 0; r < rows; r++) {
            const double *x = s_x + r * D;
            double a0 = 0.0, a1 = 0.0;
#pragma unroll
            for (int j = 0; j < D; j += 2) {
                const double2 xx = *reinterpret_cast<const double2 *>(x + j);
                a0 = fma(th0[j], xx.x, a0); a1 = fma(th1[j], xx.x, a1);
                a0 = fma(th0[j + 1], xx.y, a0); a1 = fma(th1[j + 1], xx.y, a1);
            }
            l0 += neg_softplus_neg(a0);
            l1 += neg_softplus_neg(a1);
        }
    }
    // prior: MvNormal(loc=0, scale=s, cov=I).logpdf (distributions.py:949-959)
    double q0 = 0.0, q1 = 0.0;
#pragma unroll
    for (int j = 0; j < D; j++) {
        const double z0 = th0[j] / prior_scale, z1 = th1[j] / prior_scale;
        q0 += z0 * z0; q1 += z1 * z1;
    }
    if (l0 != l0) l0 = -CUDART_INF;        // np.nan_to_num(l, nan=-inf), smc_samplers.py:283
    if (l1 != l1) l1 = -CUDART_INF;
    if (v0) {
        const double lp = -0.5 * q0 - prior_lognorm;
        lprior[i0] = lp; llik[i0] = l0;
        if (FLOOR) lpost[i0] = (l0 >= epn) ? lp : -CUDART_INF;
        else lpost[i0] = (epn > 0.0) ? lp + epn * l0 : lp;   // smc_samplers.py:840-843
    }
    if (v1) {
        const double lp = -0.5 * q1 - prior_lognorm;
        lprior[i0 + 1] = lp; llik[i0 + 1] = l1;
        if (FLOOR) lpost[i0 + 1] = (l1 >= epn) ? lp : -CUDART_INF;
        else lpost[i0 + 1] = (epn > 0.0) ? lp + epn * l1 : lp;
    }
}

// prop = theta + z @ L.T   (L lower-triangular, row-major in constant-like kernel argument space)
struct RwParams { double L[32 * 32]; int d; };

__global__ void __launch_bounds__(kSampBlock) k_rw_propose(const double *__restrict__ theta, int64_t n,
                                                          const double *__restrict__ Ldev, int d,
                                                          Philox key, uint64_t call,
                                                          const double *__restrict__ z_in,
                                                          double *__restrict__ prop) {
    extern __shared__ double s_L[];
    for (int e = threadIdx.x; e < d * d; e += kSampBlock) s_L[e] = Ldev[e];
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * kSampBlock + threadIdx.x;
    if (i >= n) return;
    double z[32];
    for (int j = 0; j < d; j += 2) {
        if (z_in) {
            z[j] = z_in[i * d + j];
            if (j + 1 < d) z[j + 1] = z_in[i * d + j + 1];
        } else {
            uint32_t r[4];
            philox4x32_10k((uint32_t)i, (uint32_t)((uint64_t)i >> 32), (uint32_t)call,
                           ((uint32_t)(call >> 32) << 16) | ((uint32_t)(j >> 1) << 8) | kPurposeApi, key, r);
            double za, zb;
            box_muller_fast(r, za, zb);
            z[j] = za;
            if (j + 1 < d) z[j + 1] = zb;
        }
    }
    for (int a = 0; a < d; a++) {
        double acc = 0.0;
        for (int b = 0; b <= a; b++) acc += z[b] * s_L[a * d + b];
        prop[i * d + a] = theta[i * d + a] + acc;
    }
}

// ArrayMetropolis.step (smc_samplers.py:601-611): pb = exp(min(lpost' - lpost, 0)); accept where
// u < pb; copy theta / lprior / llik / lpost of accepted proposals over the current state.
// Block sums of pb go to partials; the last block averages them in a fixed order.
__global__ void __launch_bounds__(kSampBlock) k_mh_accept(int64_t n, int d, double *theta, double *lprior,
                                                         double *llik, double *lpost,
                                                         const double *__restrict__ theta_p,
                                                         const double *__restrict__ lprior_p,
                                                         const double *__restrict__ llik_p,
                                                         const double *__restrict__ lpost_p,
                                                         Philox key, uint64_t call,
                                                         const double *__restrict__ u_in, double *partials,
                                                         unsigned int *ticket, double *mean_acc,
                                                         uint8_t *accepted) {
    __shared__ double s_red[kSampBlock / 32];
    const int64_t i = (int64_t)blockIdx.x * kSampBlock + threadIdx.x;
    double pb = 0.0;
    if (i < n) {
        const double lp_acc = lpost_p[i] - lpost[i] + 0.0;
        pb = exp(fmin(lp_acc, 0.0));                       // np.exp(np.clip(lp_acc, None, 0.))
        if (lp_acc != lp_acc) pb = CUDART_NAN;
        double u;
        if (u_in) u = u_in[i];
        else {
            double u1;
            uniform_pair(key, (uint64_t)i, (uint32_t)call, ((uint32_t)(call >> 32) << 8) | kPurposeApi, u, u1);
        }
        if (u < pb) {
            for (int j = 0; j < d; j++) theta[i * d + j] = theta_p[i * d + j];
            lprior[i] = lprior_p[i]; llik[i] = llik_p[i]; lpost[i] = lpost_p[i];
        }
        if (accepted) accepted[i] = (u < pb) ? 1 : 0;
    }
    const double acc = warp_sum(pb);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < kSampBlock / 32; w++) t += s_red[w];
        partials[blockIdx.x] = t;
    }
    if (!last_block(ticket) || threadIdx.x != 0) return;
    double t = 0.0;
    for (unsigned int b = 0; b < gridDim.x; b++) t += ((volatile double *)partials)[b];
    mean_acc[0] = t / (double)n;
}

// ---------------------------------------------------------------------------
// Fused waste-free move (MCMCSequenceWF.__call__, smc_samplers.py:672-683, with the
// ArrayRandomWalk / ArrayMetropolis step of 601-629 and the tempered logistic target): every
// chain is independent, so ONE launch runs all P-1 Metropolis steps of all M chains and writes
// the (P*M) particles of the next generation in the reference's order (xs[0] | xs[1] | ...).
// kWfLanes lanes of a warp share a chain: each takes every kWfLanes-th data row, a butterfly
// reduction gives all of them the same log-likelihood bits, so they take the same decision.
// The data matrix is staged in shared memory once per CTA when it fits (it is re-used P-1 times).
// FLOOR: the target of nested sampling SMC, the prior truncated to llik >= lmin, with lmin passed as epn (as in
// k_logistic_target): a proposal below the floor has lpost = -inf, so pb = 0 and it is rejected whatever u is.
// ---------------------------------------------------------------------------
constexpr int kWfBlock = 512;
constexpr int kWfLanes = 16;

template <int D, bool FLOOR = false>
__global__ void __launch_bounds__(kWfBlock) k_logistic_wf_move(
    int64_t M, int d, int P, const double *__restrict__ theta0, const double *__restrict__ lprior0,
    const double *__restrict__ llik0, const double *__restrict__ lpost0, const double *__restrict__ data,
    int64_t n_data, int tile_rows, double prior_scale, double prior_lognorm, double epn,
    const double *__restrict__ Ldev, Philox key, uint64_t call, const double *__restrict__ z_in,
    const double *__restrict__ u_in, double *__restrict__ theta_out, double *__restrict__ lprior_out,
    double *__restrict__ llik_out, double *__restrict__ lpost_out, double *__restrict__ pb_out) {
    extern __shared__ __align__(16) double s_mem[];
    double *s_L = s_mem;                 // D x D
    double *s_x = s_mem + D * D;         // tile_rows x D
    const int g = threadIdx.x % kWfLanes;
    const int64_t c = (int64_t)blockIdx.x * (kWfBlock / kWfLanes) + threadIdx.x / kWfLanes;
    const bool valid = c < M;
    for (int e = threadIdx.x; e < D * D; e += kWfBlock) {
        const int a = e / D, b = e - a * D;
        s_L[e] = (a < d && b < d) ? Ldev[a * d + b] : 0.0;
    }
    const bool resident = tile_rows >= n_data;     // whole data set in shared memory
    if (resident) {
        for (int e = threadIdx.x; e < (int)n_data * D; e += kWfBlock) {
            const int r = e / D, j = e - r * D;
            s_x[e] = (j < d) ? data[(int64_t)r * d + j] : 0.0;
        }
    }
    __syncthreads();
    double th[D], lpr = 0.0, ll = 0.0, lp = 0.0;
#pragma unroll
    for (int j = 0; j < D; j++) th[j] = (valid && j < d) ? theta0[c * d + j] : 0.0;
    if (valid) { lpr = lprior0[c]; ll = llik0[c]; lp = lpost0[c]; }
    // generation row 0: the resampled particles themselves
    if (valid) {
        for (int j = g; j < d; j += kWfLanes) theta_out[c * d + j] = th[j];
        if (g == 0) { lprior_out[c] = lpr; llik_out[c] = ll; lpost_out[c] = lp; }
    }
    for (int s = 1; s < P; s++) {
        double z[D], pr[D];
#pragma unroll
        for (int j = 0; j < D; j += 2) {
            if (z_in) {
                z[j] = (valid && j < d) ? z_in[((int64_t)(s - 1) * M + c) * d + j] : 0.0;
                z[j + 1] = (valid && j + 1 < d) ? z_in[((int64_t)(s - 1) * M + c) * d + j + 1] : 0.0;
            } else {
                uint32_t r[4];
                philox4x32_10k((uint32_t)c, (uint32_t)((uint64_t)c >> 32), (uint32_t)call,
                               ((uint32_t)s << 16) | ((uint32_t)(j >> 1) << 8) | kPurposeNormal, key, r);
                box_muller_fast(r, z[j], z[j + 1]);
            }
        }
#pragma unroll
        for (int a = 0; a < D; a++) {
            double acc = 0.0;
#pragma unroll
            for (int b = 0; b <= a; b++) acc += z[b] * s_L[a * D + b];
            pr[a] = th[a] + acc;
        }
        double part = 0.0;
        for (int64_t r0 = 0; r0 < n_data; r0 += tile_rows) {
            const int rows = (int)((n_data - r0) < tile_rows ? (n_data - r0) : tile_rows);
            if (!resident) {
                __syncthreads();
                for (int e = threadIdx.x; e < rows * D; e += kWfBlock) {
                    const int r = e / D, j = e - r * D;
                    s_x[e] = (j < d) ? data[(r0 + r) * d + j] : 0.0;
                }
                __syncthreads();
            }
            for (int r = g; r < rows; r += kWfLanes) {
                const double *x = s_x + r * D;
                double a0 = 0.0, a1 = 0.0;
#pragma unroll
                for (int j = 0; j < D; j += 2) {
                    const double2 xx = *reinterpret_cast<const double2 *>(x + j);
                    a0 = fma(pr[j], xx.x, a0);
                    a1 = fma(pr[j + 1], xx.y, a1);
                }
                part += neg_softplus_neg(a0 + a1);
            }
        }
#pragma unroll
        for (int m = kWfLanes / 2; m > 0; m >>= 1) part += __shfl_xor_sync(0xffffffffu, part, m);
        double llp = (part != part) ? -CUDART_INF : part;
        double q = 0.0;
#pragma unroll
        for (int j = 0; j < D; j++) { const double zz = pr[j] / prior_scale; q += zz * zz; }
        const double lprp = -0.5 * q - prior_lognorm;
        const double lpp = FLOOR ? ((llp >= epn) ? lprp : -CUDART_INF) : (epn > 0.0) ? lprp + epn * llp : lprp;
        const double lp_acc = lpp - lp + 0.0;
        double pb = exp(fmin(lp_acc, 0.0));
        if (lp_acc != lp_acc) pb = CUDART_NAN;
        double u;
        if (u_in) u = valid ? u_in[(int64_t)(s - 1) * M + c] : 1.0;
        else {
            double u1;
            uniform_pair(key, (uint64_t)c, (uint32_t)call, ((uint32_t)s << 16) | kPurposeUniform, u, u1);
        }
        if (u < pb) {
#pragma unroll
            for (int j = 0; j < D; j++) th[j] = pr[j];
            lpr = lprp; ll = llp; lp = lpp;
        }
        if (valid) {
            const int64_t row = (int64_t)s * M + c;
            for (int j = g; j < d; j += kWfLanes) theta_out[row * d + j] = th[j];
            if (g == 0) {
                lprior_out[row] = lpr; llik_out[row] = ll; lpost_out[row] = lp;
                pb_out[(int64_t)(s - 1) * M + c] = pb;
            }
        }
    }
}

}  // namespace smcb

template <int D, bool FLOOR>
static int launch_wf(smcb_ctx *c, int64_t M, int d, int P, const double *theta0, const double *lprior0,
                     const double *llik0, const double *lpost0, const double *data, int64_t n_data, double s,
                     double lognorm, double epn, const double *L, const double *z_in, const double *u_in,
                     double *theta_out, double *lprior_out, double *llik_out, double *lpost_out, double *pb_out) {
    const size_t budget = 200 * 1024;                 // of the 227 KB a CTA may use
    const size_t fixed = (size_t)D * D * sizeof(double);
    int64_t tile_rows = (int64_t)((budget - fixed) / (D * sizeof(double)));
    if (tile_rows > n_data) tile_rows = n_data;
    const size_t smem = fixed + (size_t)tile_rows * D * sizeof(double);
    SMCB_TRY(set_smem(k_logistic_wf_move<D, FLOOR>, smem));
    const int chains_per_block = kWfBlock / kWfLanes;
    const int grid = (int)((M + chains_per_block - 1) / chains_per_block);
    const uint64_t call = (z_in && u_in) ? 0 : c->api_counter++;
    return launch(c, k_logistic_wf_move<D, FLOOR>, grid, kWfBlock, smem, M, d, P, theta0, lprior0, llik0, lpost0, data,
                  n_data, (int)tile_rows, s, lognorm, epn, L, key_of(c->seed), call, z_in, u_in, theta_out, lprior_out,
                  llik_out, lpost_out, pb_out);
}

template <bool FLOOR>
static int logistic_wf_move(smcb_ctx *c, int64_t M, int d, int P, const double *theta0, const double *lprior0,
                            const double *llik0, const double *lpost0, const double *data, int64_t n_data,
                            double prior_scale, double epn, const double *L_dev, const double *z_in,
                            const double *u_in, double *theta_out, double *lprior_out, double *llik_out,
                            double *lpost_out, double *pb_out) {
    SMCB_REQUIRE(c && theta0 && lprior0 && llik0 && lpost0 && data && L_dev && theta_out && lprior_out &&
                     llik_out && lpost_out && pb_out, "smcb_logistic_wf_move: NULL argument");
    SMCB_REQUIRE(M >= 1 && P >= 2 && n_data >= 1 && d >= 1 && d <= 32, "smcb_logistic_wf_move: bad sizes");
    SMCB_REQUIRE(P < 65536, "smcb_logistic_wf_move: len_chain must be < 65536");
    const double lognorm = (double)d * log(prior_scale) + 0.0 + (double)d * kHalfLog2Pi;
#define WF(DD) return launch_wf<DD, FLOOR>(c, M, d, P, theta0, lprior0, llik0, lpost0, data, n_data, prior_scale, \
                                           lognorm, epn, L_dev, z_in, u_in, theta_out, lprior_out, llik_out, lpost_out, \
                                           pb_out)
    if (d <= 4) WF(4);
    if (d <= 8) WF(8);
    if (d <= 12) WF(12);
    if (d <= 16) WF(16);
    if (d <= 20) WF(20);
    if (d <= 24) WF(24);
    WF(32);
#undef WF
}

// MCMCSequenceWF.__call__ (smc_samplers.py:672-683) for the logistic model + random-walk Metropolis:
// inputs = the M resampled particles (theta0 (M,d), lprior0, llik0, lpost0), outputs = the P*M
// particles of the next generation in concatenate(xs) order, pb_out (P-1, M) acceptance probabilities.
extern "C" int smcb_logistic_wf_move(smcb_ctx *c, int64_t M, int d, int P, const double *theta0,
                                     const double *lprior0, const double *llik0, const double *lpost0,
                                     const double *data, int64_t n_data, double prior_scale, double epn,
                                     const double *L_dev, const double *z_in, const double *u_in,
                                     double *theta_out, double *lprior_out, double *llik_out,
                                     double *lpost_out, double *pb_out) {
    return logistic_wf_move<false>(c, M, d, P, theta0, lprior0, llik0, lpost0, data, n_data, prior_scale, epn, L_dev,
                                   z_in, u_in, theta_out, lprior_out, llik_out, lpost_out, pb_out);
}

// The same move under the target of NestedSamplingSMC (nested.py:353-373): the prior truncated to llik >= lmin.
extern "C" int smcb_logistic_ns_move(smcb_ctx *c, int64_t M, int d, int P, const double *theta0,
                                     const double *lprior0, const double *llik0, const double *lpost0,
                                     const double *data, int64_t n_data, double prior_scale, double lmin,
                                     const double *L_dev, const double *z_in, const double *u_in,
                                     double *theta_out, double *lprior_out, double *llik_out,
                                     double *lpost_out, double *pb_out) {
    SMCB_REQUIRE(lmin == lmin, "smcb_logistic_ns_move: lmin is NaN");
    return logistic_wf_move<true>(c, M, d, P, theta0, lprior0, llik0, lpost0, data, n_data, prior_scale, lmin, L_dev,
                                  z_in, u_in, theta_out, lprior_out, llik_out, lpost_out, pb_out);
}

template <int D, bool FLOOR>
static int launch_target(smcb_ctx *c, const double *theta, int64_t n, int d, const double *data,
                         int64_t n_data, double s, double lognorm, double epn, double *lprior, double *llik,
                         double *lpost) {
    const int64_t pairs = (n + 1) / 2;
    const int grid = (int)((pairs + kSampBlock - 1) / kSampBlock);
    return launch(c, k_logistic_target<D, FLOOR>, grid, kSampBlock, 0, theta, n, d, data, n_data, s, lognorm, epn,
                  lprior, llik, lpost);
}

template <bool FLOOR>
static int logistic_target(smcb_ctx *c, const double *theta, int64_t n, int d, const double *data, int64_t n_data,
                           double prior_scale, double epn, double *lprior, double *llik, double *lpost) {
    SMCB_REQUIRE(c && theta && data && lprior && llik && lpost, "smcb_logistic_target: NULL argument");
    SMCB_REQUIRE(n >= 1 && n_data >= 1 && d >= 1 && d <= 32, "smcb_logistic_target: need 1 <= d <= 32");
    SMCB_REQUIRE(prior_scale > 0.0, "smcb_logistic_target: prior scale must be positive");
    const double lognorm = (double)d * log(prior_scale) + 0.0 + (double)d * kHalfLog2Pi;
#define TG(DD) return launch_target<DD, FLOOR>(c, theta, n, d, data, n_data, prior_scale, lognorm, epn, lprior, llik, lpost)
    if (d <= 4) TG(4);
    if (d <= 8) TG(8);
    if (d <= 12) TG(12);
    if (d <= 16) TG(16);
    if (d <= 20) TG(20);
    if (d <= 24) TG(24);
    TG(32);
#undef TG
}

// Tempering.current_target (smc_samplers.py:836-845) for the logistic-regression model with an
// MvNormal(loc=0, scale=prior_scale, cov=I_d) prior: lprior, llik, lpost = lprior + epn * llik.
extern "C" int smcb_logistic_target(smcb_ctx *c, const double *theta, int64_t n, int d, const double *data,
                                    int64_t n_data, double prior_scale, double epn, double *lprior,
                                    double *llik, double *lpost) {
    return logistic_target<false>(c, theta, n, d, data, n_data, prior_scale, epn, lprior, llik, lpost);
}

// NestedSamplingSMC.current_target (nested.py:353-363) for the same model: lpost = lprior where llik >= lmin, else -inf.
extern "C" int smcb_logistic_ns_target(smcb_ctx *c, const double *theta, int64_t n, int d, const double *data,
                                       int64_t n_data, double prior_scale, double lmin, double *lprior,
                                       double *llik, double *lpost) {
    SMCB_REQUIRE(lmin == lmin, "smcb_logistic_ns_target: lmin is NaN");
    return logistic_target<true>(c, theta, n, d, data, n_data, prior_scale, lmin, lprior, llik, lpost);
}

// ArrayRandomWalk.proposal (smc_samplers.py:624-629); L: DEVICE (d, d) row-major lower factor
extern "C" int smcb_rw_propose(smcb_ctx *c, const double *theta, int64_t n, int d, const double *L_dev,
                               const double *z_in, double *prop) {
    SMCB_REQUIRE(c && theta && L_dev && prop, "smcb_rw_propose: NULL argument");
    SMCB_REQUIRE(n >= 1 && d >= 1 && d <= 32, "smcb_rw_propose: need 1 <= d <= 32");
    const uint64_t call = z_in ? 0 : c->api_counter++;
    const int grid = (int)((n + kSampBlock - 1) / kSampBlock);
    return launch(c, k_rw_propose, grid, kSampBlock, (size_t)d * d * sizeof(double), theta, n, L_dev, d,
                  key_of(c->seed), call, z_in, prop);
}

// ArrayMetropolis.step accept / copyto (smc_samplers.py:605-611); mean_acc: device scalar; accepted: NULL or (n)
extern "C" int smcb_mh_accept_flags(smcb_ctx *c, int64_t n, int d, double *theta, double *lprior, double *llik,
                                    double *lpost, const double *theta_p, const double *lprior_p,
                                    const double *llik_p, const double *lpost_p, const double *u_in,
                                    double *mean_acc, uint8_t *accepted) {
    SMCB_REQUIRE(c && theta && lprior && llik && lpost && theta_p && lprior_p && llik_p && lpost_p && mean_acc,
                 "smcb_mh_accept: NULL argument");
    SMCB_REQUIRE(n >= 1 && d >= 1, "smcb_mh_accept: bad sizes");
    const int grid = (int)((n + kSampBlock - 1) / kSampBlock);
    SMCB_REQUIRE((size_t)grid <= kWsPartials, "smcb_mh_accept: too many particles for the workspace");
    const uint64_t call = u_in ? 0 : c->api_counter++;
    return launch(c, k_mh_accept, grid, kSampBlock, 0, n, d, theta, lprior, llik, lpost, theta_p, lprior_p, llik_p,
                  lpost_p, key_of(c->seed), call, u_in, c->ws, c->counters + kTicketMhAccept, mean_acc, accepted);
}

extern "C" int smcb_mh_accept(smcb_ctx *c, int64_t n, int d, double *theta, double *lprior, double *llik,
                              double *lpost, const double *theta_p, const double *lprior_p,
                              const double *llik_p, const double *lpost_p, const double *u_in,
                              double *mean_acc) {
    return smcb_mh_accept_flags(c, n, d, theta, lprior, llik, lpost, theta_p, lprior_p, llik_p, lpost_p, u_in,
                                mean_acc, nullptr);
}

// ---------------------------------------------------------------------------
// the control plane of adaptive tempering on the device (no host round trip inside a tempering step)
// ---------------------------------------------------------------------------
namespace smcb {

constexpr int kRootWays = 16;          // candidate exponents evaluated per pass
constexpr int kRootPasses = 11;        // 16^11 > 1e13: the bracket shrinks below brentq's 2e-12 tolerance
constexpr int kCtlBlock = 256;
constexpr int kCtlGrid = kSMs * 2;

// max of v (NaN-free log-likelihoods): one pass, last block merges
__global__ void __launch_bounds__(kCtlBlock) k_ctl_max(const double *__restrict__ v, int64_t n, double *partials,
                                                      unsigned int *ticket, double *out) {
    __shared__ double s[kCtlBlock / 32];
    double m = -CUDART_INF;
    for (int64_t i = (int64_t)blockIdx.x * kCtlBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kCtlBlock)
        m = fmax(m, v[i]);
    m = warp_max(m);
    if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < kCtlBlock / 32; w++) m = fmax(m, s[w]);
        partials[blockIdx.x] = m;
    }
    if (!last_block(ticket) || threadIdx.x != 0) return;
    double r = -CUDART_INF;
    for (unsigned int b = 0; b < gridDim.x; b++) r = fmax(r, reinterpret_cast<volatile double *>(partials)[b]);
    out[0] = r;
}

// one pass of the root-find of next_annealing_epn (smc_samplers.py:876-895): ESS(delta * lw) at the kRootWays
// points delta_j = lo + (hi - lo) (j + 1) / kRootWays, then the bracket [lo, hi] := the sub-interval in which
// ESS crosses alpha N (ESS is non-increasing in delta).  state = {lo, hi, max lw, done flag, result}.
__global__ void __launch_bounds__(kCtlBlock) k_ctl_root_pass(const double *__restrict__ lw, int64_t n, double target,
                                                            double *state, double *partials, unsigned int *ticket,
                                                            int final_pass, double *raw_out) {
    __shared__ double s_red[kCtlBlock / 32][2 * kRootWays];
    const double lo = state[0], hi = state[1], M = state[2];
    if (state[3] != 0.0) return;                                   // already decided (delta = full step)
    double dj[kRootWays], s[kRootWays], q[kRootWays];
#pragma unroll
    for (int j = 0; j < kRootWays; j++) { dj[j] = lo + (hi - lo) * ((double)(j + 1) / kRootWays); s[j] = 0.0; q[j] = 0.0; }
    for (int64_t i = (int64_t)blockIdx.x * kCtlBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kCtlBlock) {
        const double a = lw[i] - M;                                // <= 0
#pragma unroll
        for (int j = 0; j < kRootWays; j++) {
            const double e = fexp_neg(dj[j] * a);
            s[j] += e;
            q[j] = fma(e, e, q[j]);
        }
    }
#pragma unroll
    for (int j = 0; j < kRootWays; j++) {
        s[j] = warp_sum(s[j]);
        q[j] = warp_sum(q[j]);
        if ((threadIdx.x & 31) == 0) { s_red[threadIdx.x >> 5][2 * j] = s[j]; s_red[threadIdx.x >> 5][2 * j + 1] = q[j]; }
    }
    __syncthreads();
    if (threadIdx.x < 2 * kRootWays) {
        double v = 0.0;
        for (int w = 0; w < kCtlBlock / 32; w++) v += s_red[w][threadIdx.x];
        partials[(size_t)blockIdx.x * 2 * kRootWays + threadIdx.x] = v;
    }
    if (!last_block(ticket)) return;
    __shared__ double tot[2 * kRootWays];
    if (threadIdx.x < 2 * kRootWays) {                             // fixed block order: deterministic
        double v = 0.0;
        for (unsigned int b = 0; b < gridDim.x; b++)
            v += reinterpret_cast<volatile double *>(partials)[(size_t)b * 2 * kRootWays + threadIdx.x];
        tot[threadIdx.x] = v;
    }
    __syncthreads();
    if (raw_out != nullptr) {                                      // sharded run: the caller sums these over the ranks
        if (threadIdx.x < 2 * kRootWays) raw_out[threadIdx.x] = tot[threadIdx.x];
        return;
    }
    if (threadIdx.x == 0) {
        // f(delta) = ESS - target; f(lo) >= 0 by construction.  First j with f(delta_j) < 0 brackets the root.
        int jx = kRootWays;
        for (int j = 0; j < kRootWays; j++) {
            const double ess = tot[2 * j] * tot[2 * j] / tot[2 * j + 1];
            if (ess - target < 0.0) { jx = j; break; }
        }
        if (jx == kRootWays && (final_pass & 2)) {                 // first pass, ESS(hi) >= target: the whole step is allowed
            state[3] = 1.0;
            state[4] = hi;
        } else {
            if (jx == kRootWays) jx = kRootWays - 1;               // (rounding at the bracket's end in a later pass)
            const double nlo = lo + (hi - lo) * ((double)jx / kRootWays), nhi = lo + (hi - lo) * ((double)(jx + 1) / kRootWays);
            state[0] = nlo;
            state[1] = nhi;
            if (final_pass & 1) state[4] = 0.5 * (nlo + nhi);
        }
    }
}

__global__ void k_ctl_root_finish(const double *st, double epn, double *out) {
    out[0] = (st[3] != 0.0) ? 1.0 : epn + st[4];
}

// weighted mean and covariance of the rows of theta (rs.wmean_and_cov, resampling.py:341-358, as
// ArrayRandomWalk.calibrate uses it), then L = scale * chol(cov): two passes, fixed-order block merges
__device__ __forceinline__ void chol_scaled(const double *cov, int d, double scale, double *L_out) {
    // numpy.linalg.cholesky (smc_samplers.py:617-622), then the 2.38 / sqrt(d) scale; NaN if not positive definite
    for (int j = 0; j < d; j++) {
        double s = cov[j * d + j];
        for (int k = 0; k < j; k++) s -= L_out[j * d + k] * L_out[j * d + k];
        const double ljj = sqrt(s);
        L_out[j * d + j] = ljj;
        for (int i = j + 1; i < d; i++) {
            double t = cov[i * d + j];
            for (int k = 0; k < j; k++) t -= L_out[i * d + k] * L_out[j * d + k];
            L_out[i * d + j] = t / ljj;
        }
        for (int i = 0; i < j; i++) L_out[i * d + j] = 0.0;
    }
    for (int i = 0; i < d * d; i++) L_out[i] *= scale;
}

// sharded runs: covariance from the (all-reduced) lower-triangular sums and the sum of weights, then the factor
__global__ void k_ctl_chol(const double *tri, const double *sw, int d, double scale, double *work, double *L_out) {
    if (threadIdx.x != 0) return;
    for (int a_ = 0; a_ < d; a_++)
        for (int b_ = 0; b_ <= a_; b_++) { const double c = tri[a_ * (a_ + 1) / 2 + b_] / sw[0]; work[a_ * d + b_] = c; work[b_ * d + a_] = c; }
    chol_scaled(work, d, scale, L_out);
}

// FINAL: the last block turns the sums into the mean (pass 0) / the scaled Cholesky factor (pass 1); otherwise it
// leaves the raw sums in `work` (pass 0: sum w x_j, sum w; pass 1: the lower triangle) for the caller to reduce
// over ranks.  `mean` (pass 1) = the mean the deviations are taken from.
template <int PASS, bool FINAL>
__global__ void __launch_bounds__(kCtlBlock) k_ctl_wcov(const double *__restrict__ W, const double *__restrict__ theta,
                                                       int64_t n, int d, double *work /* [0..d) mean | d x d cov */,
                                                       double *partials, unsigned int *ticket, double scale,
                                                       double *L_out, const double *mean) {
    extern __shared__ double s_acc[];                              // (kCtlBlock/32) x nvals
    const int nvals = (PASS == 0) ? d + 1 : d * (d + 1) / 2;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // each WARP walks rows; lane l accumulates the values v = l, l + 32, ... of the row's contribution
    constexpr int kMaxPerLane = 8;                                 // d <= 20: d (d + 1) / 2 = 210 <= 256
    double acc[kMaxPerLane];
#pragma unroll
    for (int k = 0; k < kMaxPerLane; k++) acc[k] = 0.0;
    const int64_t wstride = (int64_t)gridDim.x * (kCtlBlock / 32);
    for (int64_t r = (int64_t)blockIdx.x * (kCtlBlock / 32) + warp; r < n; r += wstride) {
        const double w = W[r];
        const double *row = theta + r * d;
#pragma unroll
        for (int k = 0; k < kMaxPerLane; k++) {
            const int v = lane + 32 * k;
            if (v < nvals) {
                if (PASS == 0) acc[k] += (v < d) ? w * row[v] : w;               // sum w x_j | sum w
                else {
                    // v -> (a, b), a >= b (row-major lower triangle)
                    int a_ = (int)((sqrt(8.0 * v + 1.0) - 1.0) * 0.5);
                    while ((a_ + 1) * (a_ + 2) / 2 <= v) a_++;
                    while (a_ * (a_ + 1) / 2 > v) a_--;
                    const int b_ = v - a_ * (a_ + 1) / 2;
                    acc[k] += w * (row[a_] - mean[a_]) * (row[b_] - mean[b_]);
                }
            }
        }
    }
#pragma unroll
    for (int k = 0; k < kMaxPerLane; k++) {
        const int v = lane + 32 * k;
        if (v < nvals) s_acc[warp * nvals + v] = acc[k];
    }
    __syncthreads();
    for (int v = threadIdx.x; v < nvals; v += kCtlBlock) {
        double t = 0.0;
        for (int w2 = 0; w2 < kCtlBlock / 32; w2++) t += s_acc[w2 * nvals + v];
        partials[(size_t)blockIdx.x * nvals + v] = t;
    }
    if (!last_block(ticket)) return;
    double *tot = s_acc;
    for (int v = threadIdx.x; v < nvals; v += kCtlBlock) {
        double t = 0.0;
        for (unsigned int b = 0; b < gridDim.x; b++) t += reinterpret_cast<volatile double *>(partials)[(size_t)b * nvals + v];
        tot[v] = t;
    }
    __syncthreads();
    if (!FINAL) {
        for (int v = threadIdx.x; v < nvals; v += kCtlBlock) work[v] = tot[v];
    } else if (PASS == 0) {
        for (int j = threadIdx.x; j <= d; j += kCtlBlock) work[j] = (j < d) ? tot[j] / tot[d] : tot[d];     // mean | sum w
    } else if (threadIdx.x == 0) {
        const double sw = work[d];
        double *cov = work + d + 1;                                // d x d, symmetric
        for (int a_ = 0; a_ < d; a_++)
            for (int b_ = 0; b_ <= a_; b_++) { const double c = tot[a_ * (a_ + 1) / 2 + b_] / sw; cov[a_ * d + b_] = c; cov[b_ * d + a_] = c; }
        chol_scaled(cov, d, scale, L_out);
    }
}

}  // namespace smcb

// next_annealing_epn (smc_samplers.py:876-895) without the host: out_dev[0] = the new exponent.
// 1 + kRootPasses launches, the bracket lives in the context's workspace.
extern "C" int smcb_next_annealing_epn(smcb_ctx *c, const double *lw, int64_t n, double epn, double alpha, double *out_dev) {
    SMCB_REQUIRE(c && lw && out_dev && n >= 1, "smcb_next_annealing_epn: bad argument");
    SMCB_REQUIRE(epn >= 0.0 && epn <= 1.0 && alpha > 0.0 && alpha < 1.0, "smcb_next_annealing_epn: epn in [0, 1], alpha in (0, 1)");
    double *state = c->ws;                                         // 8 doubles
    double *partials = c->ws + 64;
    const double init[5] = {0.0, 1.0 - epn, 0.0, 0.0, 0.0};
    SMCB_CUDA(cudaMemcpyAsync(state, init, sizeof(init), cudaMemcpyHostToDevice, c->stream));
    const int grid = (int)((n + kCtlBlock - 1) / kCtlBlock < kCtlGrid ? (n + kCtlBlock - 1) / kCtlBlock : kCtlGrid);
    SMCB_TRY(launch(c, k_ctl_max, grid, kCtlBlock, 0, lw, n, partials, c->counters + kTicketCtlMax, state + 2));
    for (int p = 0; p < kRootPasses; p++)
        SMCB_TRY(launch(c, k_ctl_root_pass, grid, kCtlBlock, 0, lw, n, alpha * (double)n, state, partials,
                        c->counters + kTicketCtlRoot, (p == kRootPasses - 1 ? 1 : 0) | (p == 0 ? 2 : 0),
                        (double *)nullptr));
    return launch(c, k_ctl_root_finish, 1, 1, 0, state, epn, out_dev);     // result = epn + delta
}

// ArrayRandomWalk.calibrate (smc_samplers.py:617-622): L = scale * chol(wcov(W, theta)) on the device
extern "C" int smcb_rw_calibrate(smcb_ctx *c, const double *W, const double *theta, int64_t n, int d, double scale,
                                 double *L_out) {
    SMCB_REQUIRE(c && W && theta && L_out && n >= 1, "smcb_rw_calibrate: bad argument");
    SMCB_REQUIRE(d >= 1 && d <= 20, "smcb_rw_calibrate: 1 <= d <= 20 (got %d)", d);
    double *work = c->ws;                                          // mean[d] | sum w | cov[d x d]
    double *partials = c->ws + 1024;
    const int grid = (int)((n + 7) / 8 < kCtlGrid ? (n + 7) / 8 : kCtlGrid);
    const int nv0 = d + 1, nv1 = d * (d + 1) / 2;
    SMCB_TRY(launch(c, k_ctl_wcov<0, true>, grid, kCtlBlock, (kCtlBlock / 32) * (nv0 > 32 ? nv0 : 32) * sizeof(double), W,
                    theta, n, d, work, partials, c->counters + kTicketCtlWcov0, scale, L_out, (const double *)nullptr));
    return launch(c, k_ctl_wcov<1, true>, grid, kCtlBlock, (kCtlBlock / 32) * nv1 * sizeof(double), W, theta, n, d, work,
                  partials, c->counters + kTicketCtlWcov1, scale, L_out, (const double *)work);
}

// the same in pieces for a run sharded over ranks (the caller all-reduces between them):
//   pass 0 (mean_dev == NULL): out_dev[0..d) = sum w x_j, out_dev[d] = sum w
//   pass 1:                    out_dev[0..d(d+1)/2) = lower triangle of sum w (x - mean)(x - mean)^T
extern "C" int smcb_wcov_sums(smcb_ctx *c, const double *W, const double *theta, int64_t n, int d, const double *mean_dev,
                              double *out_dev) {
    SMCB_REQUIRE(c && W && theta && out_dev && n >= 1 && d >= 1 && d <= 20, "smcb_wcov_sums: bad argument");
    double *partials = c->ws + 1024;
    const int grid = (int)((n + 7) / 8 < kCtlGrid ? (n + 7) / 8 : kCtlGrid);
    const int nv0 = d + 1, nv1 = d * (d + 1) / 2;
    if (mean_dev == nullptr)
        return launch(c, k_ctl_wcov<0, false>, grid, kCtlBlock, (kCtlBlock / 32) * (nv0 > 32 ? nv0 : 32) * sizeof(double),
                      W, theta, n, d, out_dev, partials, c->counters + kTicketCtlWcov0, 1.0, (double *)nullptr,
                      (const double *)nullptr);
    return launch(c, k_ctl_wcov<1, false>, grid, kCtlBlock, (kCtlBlock / 32) * nv1 * sizeof(double), W, theta, n, d,
                  out_dev, partials, c->counters + kTicketCtlWcov1, 1.0, (double *)nullptr, mean_dev);
}

extern "C" int smcb_chol_from_sums(smcb_ctx *c, const double *tri_dev, const double *sw_dev, int d, double scale,
                                   double *L_out) {
    SMCB_REQUIRE(c && tri_dev && sw_dev && L_out && d >= 1 && d <= 20, "smcb_chol_from_sums: bad argument");
    return launch(c, k_ctl_chol, 1, 32, 0, tri_dev, sw_dev, d, scale, c->ws, L_out);
}

// one pass of the root-find's ESS grid without the bracket update (sharded runs): out32_dev = {s_j, q_j} for the 16
// exponents lo + (hi - lo)(j + 1)/16, relative to the shift max_dev[0] (the GLOBAL maximum of lw)
extern "C" int smcb_essl_grid(smcb_ctx *c, const double *lw, int64_t n, double lo, double hi, const double *max_dev,
                              double *out32_dev) {
    SMCB_REQUIRE(c && lw && max_dev && out32_dev && n >= 1, "smcb_essl_grid: bad argument");
    double *state = c->ws;
    double *partials = c->ws + 64;
    const double init[5] = {lo, hi, 0.0, 0.0, 0.0};
    SMCB_CUDA(cudaMemcpyAsync(state, init, sizeof(init), cudaMemcpyHostToDevice, c->stream));
    SMCB_CUDA(cudaMemcpyAsync(state + 2, max_dev, sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
    const int grid = (int)((n + kCtlBlock - 1) / kCtlBlock < kCtlGrid ? (n + kCtlBlock - 1) / kCtlBlock : kCtlGrid);
    return launch(c, k_ctl_root_pass, grid, kCtlBlock, 0, lw, n, 0.0, state, partials, c->counters + kTicketCtlRoot, 0,
                  out32_dev);
}

// ---------------------------------------------------------------------------
// IBIS reweighting (IBIS.logG, smc_samplers.py:773-776, for the logistic model): the log-likelihood of the data rows
// [r0, r0 + K) for n particles, added to the log-weights ONE ROW AT A TIME, in row order.
//   scan   (COMMIT = false): scratch[k * n + i] = lw[i] + sum_{r <= k} logpyt_r(theta_i); lw is not written.
//   commit (COMMIT = true):  lw[i], lpost[i] and llik[i] += logpyt_r(theta_i) for r = r0 .. r0 + K - 1, in place
//                            (lpost / llik may be NULL).
// A NaN log-weight becomes -inf after each row, as smcb_normalise rewrites it after each step of the per-step path,
// so scratch row k and a commit through row k hold the bits of k + 1 single-row steps.  The dot product and
// neg_softplus_neg are those of k_logistic_target (theta in registers, two particles per thread, rows staged in
// shared memory, fma over the padded coordinates in order): a one-row logpyt has the bits of a one-row target.
// ---------------------------------------------------------------------------
namespace smcb {

template <int D, bool COMMIT>
__global__ void __launch_bounds__(kSampBlock) k_logistic_logpyt(
    const double *__restrict__ theta, int64_t n, int d, const double *__restrict__ data, int64_t r0, int64_t K,
    double *__restrict__ lw, double *__restrict__ lpost, double *__restrict__ llik, double *__restrict__ scratch) {
    __shared__ __align__(16) double s_x[kRowsPerTile * D];
    const int64_t i0 = 2 * ((int64_t)blockIdx.x * kSampBlock + threadIdx.x);
    const bool v0 = i0 < n, v1 = i0 + 1 < n;
    double th0[D], th1[D];
#pragma unroll
    for (int j = 0; j < D; j++) {
        th0[j] = (v0 && j < d) ? theta[i0 * d + j] : 0.0;
        th1[j] = (v1 && j < d) ? theta[(i0 + 1) * d + j] : 0.0;
    }
    double w0 = v0 ? lw[i0] : 0.0, w1 = v1 ? lw[i0 + 1] : 0.0;
    double p0 = 0.0, p1 = 0.0, q0 = 0.0, q1 = 0.0;
    if (COMMIT && lpost) { p0 = v0 ? lpost[i0] : 0.0; p1 = v1 ? lpost[i0 + 1] : 0.0; }
    if (COMMIT && llik) { q0 = v0 ? llik[i0] : 0.0; q1 = v1 ? llik[i0 + 1] : 0.0; }
    for (int64_t k0 = 0; k0 < K; k0 += kRowsPerTile) {
        const int rows = (int)((K - k0) < kRowsPerTile ? (K - k0) : kRowsPerTile);
        __syncthreads();
        for (int e = threadIdx.x; e < rows * D; e += kSampBlock) {
            const int r = e / D, j = e - r * D;
            s_x[e] = (j < d) ? data[(r0 + k0 + r) * d + j] : 0.0;
        }
        __syncthreads();
        for (int r = 0; r < rows; r++) {
            const double *x = s_x + r * D;
            double a0 = 0.0, a1 = 0.0;
#pragma unroll
            for (int j = 0; j < D; j += 2) {
                const double2 xx = *reinterpret_cast<const double2 *>(x + j);
                a0 = fma(th0[j], xx.x, a0); a1 = fma(th1[j], xx.x, a1);
                a0 = fma(th0[j + 1], xx.y, a0); a1 = fma(th1[j + 1], xx.y, a1);
            }
            const double g0 = neg_softplus_neg(a0), g1 = neg_softplus_neg(a1);
            w0 += g0; w1 += g1;
            if (w0 != w0) w0 = -CUDART_INF;
            if (w1 != w1) w1 = -CUDART_INF;
            if (COMMIT) {
                p0 += g0; p1 += g1;
                q0 += g0; q1 += g1;
            } else {
                double *row = scratch + (k0 + r) * n;
                if (v0) row[i0] = w0;
                if (v1) row[i0 + 1] = w1;
            }
        }
    }
    if (COMMIT) {
        if (v0) lw[i0] = w0;
        if (v1) lw[i0 + 1] = w1;
        if (lpost && v0) lpost[i0] = p0;
        if (lpost && v1) lpost[i0 + 1] = p1;
        if (llik && v0) llik[i0] = q0;
        if (llik && v1) llik[i0 + 1] = q1;
    }
}

}  // namespace smcb

template <int D>
static int launch_logpyt(smcb_ctx *c, const double *theta, int64_t n, int d, const double *data, int64_t r0,
                         int64_t K, int commit, double *lw, double *lpost, double *llik, double *scratch) {
    const int64_t pairs = (n + 1) / 2;
    const int grid = (int)((pairs + kSampBlock - 1) / kSampBlock);
    return launch(c, commit ? k_logistic_logpyt<D, true> : k_logistic_logpyt<D, false>, grid, kSampBlock, 0, theta, n,
                  d, data, r0, K, lw, lpost, llik, scratch);
}

// IBIS.logG (smc_samplers.py:773-776) for the logistic-regression model over the rows [r0, r0 + K) of data
// (n_data, d): commit != 0 adds them to lw / lpost / llik in place, row by row; commit == 0 writes the cumulative
// log-weights of every row into scratch (K, n) and leaves lw, lpost and llik alone.
extern "C" int smcb_logistic_logpyt(smcb_ctx *c, const double *theta, int64_t n, int d, const double *data,
                                    int64_t n_data, int64_t r0, int64_t K, int commit, double *lw, double *lpost,
                                    double *llik, double *scratch) {
    SMCB_REQUIRE(c && theta && data && lw && (commit || scratch), "smcb_logistic_logpyt: NULL argument");
    SMCB_REQUIRE(n >= 1 && d >= 1 && d <= 32, "smcb_logistic_logpyt: need n >= 1 and 1 <= d <= 32");
    SMCB_REQUIRE(K >= 1 && r0 >= 0 && r0 + K <= n_data, "smcb_logistic_logpyt: rows [%lld, %lld) outside the %lld data rows",
                 (long long)r0, (long long)(r0 + K), (long long)n_data);
#define LP(DD) return launch_logpyt<DD>(c, theta, n, d, data, r0, K, commit, lw, lpost, llik, scratch)
    if (d <= 4) LP(4);
    if (d <= 8) LP(8);
    if (d <= 12) LP(12);
    if (d <= 16) LP(16);
    if (d <= 20) LP(20);
    if (d <= 24) LP(24);
    LP(32);
#undef LP
}
