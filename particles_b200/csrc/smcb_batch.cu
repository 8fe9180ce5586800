// smcb_batch.cu -- many independent filters in one launch, one CTA per filter (multiSMC).
//
//   k_batch<Model, FK, SCHEME, RESIDENT>: a persistent grid; CTA b runs filters r = b, b + grid, ... and each of
//   them runs its whole T-step loop (core.py:369-383) inside the CTA.  Filters are independent, so there is no grid
//   barrier, no cross-CTA partial row, no programmatic dependent launch and no launch per step.
//
//   Per step, every thread takes the pairs of particles p = tid, tid + BS, ... (the pair is the unit of the Philox
//   normals, as in k_step):
//     resampling step: W = exp(lw - m) / s (auxiliary weights for an APF) -> CTA scan into a non-decreasing CDF
//                      (scan_range of smcb_step.cuh) -> su_k -> A_k = searchsorted(cdf, su_k, 'left') clipped to
//                      N - 1 -> xp = X[A_k], restart weight
//     every step:      x' ~ M_t(xp), lw' = base + logG, thread accumulators (max, sum exp, sum exp^2 [, moments])
//     then:            CTA-wide merge (fixed order, every thread gets the totals), log-mean, ESS = s^2 / q, the
//                      logLt recursion, the strict ESS < N ESSrmin test and the APF restart constant; thread 0
//                      writes the summaries row and the moments row.
//
//   Tiers.  RESIDENT: x (ping-pong), lw, the CDF (and the multinomial spacings) live in shared memory next to the
//   64 KB of math tables for the whole run; device memory sees the data, the per-step rows and the final generation.
//   STREAMING: the same buffers are per-run rows in device memory (any N).  Both tiers run the same code on the same
//   thread-to-pair map, so they give the same bits.
//
//   Randomness: the Philox counters of k_step (normals: pair index, t, component; uniforms: purpose kPurposeUniform,
//   pair index, t) under the run's own key, and the table-family Box-Muller, so run r draws exactly what
//   SMC(seed = seed[r]) draws.  The bits of a run depend on N and the block size only -- not on R, on the run's
//   position in the batch or on the grid.
#include "smcb_step.cuh"

namespace smcb {

constexpr int kBatchBS = 256;

// plain loads (shared or device memory written earlier by this CTA): the multinomial spacings
struct LoadPlain {
    const double *v;
    __device__ __forceinline__ void operator()(int64_t i0, int64_t n, double (&o)[8]) const {
#pragma unroll
        for (int j = 0; j < 8; j++) o[j] = (i0 + j < n) ? v[i0 + j] : 0.0;
    }
};

// np.searchsorted(cdf, key, 'left') on [0, n) with plain loads
__device__ __forceinline__ int64_t lower_bound_plain(const double *cdf, int64_t n, double key) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = lo + ((hi - lo) >> 1);
        if (cdf[mid] < key) lo = mid + 1; else hi = mid;
    }
    return lo;
}

__host__ __device__ inline int64_t batch_ld(int64_t n) { return (n + 1) & ~(int64_t)1; }

// doubles of shared memory the resident tier needs besides the math tables
__host__ __device__ inline int64_t resident_doubles(int64_t n, int scheme) {
    const int64_t ld = batch_ld(n);
    return 4 * ld + (scheme == SMCB_RS_MULTINOMIAL ? ld + 2 : 0);
}

template <class M, int FK, int SCHEME, bool RESIDENT>
__global__ void __launch_bounds__(kBatchBS) k_batch(const smcb_batch_desc d, const double *math_tab) {
    static_assert(M::D == 1, "the batched filter runs the 1-D models");
    constexpr bool APF = FkTraits<FK>::apf;
    constexpr bool MULTI = (SCHEME == SMCB_RS_MULTINOMIAL);
    constexpr int NZ = M::NZ, BS = kBatchBS;
    extern __shared__ __align__(128) double s_dyn[];     // math tables | resident buffers
    __shared__ M s_model;
    __shared__ Philox s_key;
    __shared__ double s_red[(BS / 32 + 1) * 6];
    __shared__ double s_warp[BS / 32];
    __shared__ __align__(8) uint64_t s_tabbar;
    if (threadIdx.x == 0) mtab_issue(math_tab, &s_tabbar);
    __syncthreads();
    mbar_wait(&s_tabbar, 0);
    const int64_t n = d.N, ld = batch_ld(n), T = d.T, npairs = (n + 1) >> 1;
    const double Nd = (double)n;
    const bool mom = d.moments != nullptr;
    for (int64_t r = blockIdx.x; r < d.R; r += gridDim.x) {
        __syncthreads();                                 // the previous run is done with s_model, s_key, the buffers
        if (threadIdx.x == 0) {
            s_model.load(d.params + r * d.n_params);
            s_key = key_of(d.seed[r]);
        }
        __syncthreads();
        const M &model = s_model;
        const Philox &key = s_key;
        double *X[2], *lw, *cdf, *su;
        if (RESIDENT) {
            double *b = s_dyn + kMathTabDoubles;
            X[0] = b; X[1] = b + ld; lw = b + 2 * ld; cdf = b + 3 * ld; su = b + 4 * ld;
        } else {
            X[0] = d.X + r * 2 * ld; X[1] = X[0] + ld; lw = d.lw + r * ld; cdf = d.cdf + r * ld;
            su = MULTI ? d.scratch + r * (ld + 2) : nullptr;
        }
        FilterArgs fa = {};                              // what step_consts reads: this run's data
        fa.data = d.data + r * T * d.dy;
        fa.sc = d.step_consts ? d.step_consts + r * T : nullptr;
        fa.dy = d.dy;
        fa.T = T;
        const double essrmin = d.essrmin[r];
        const double *zr = d.z_in ? d.z_in + r * T * NZ * n : nullptr;
        const double *ur = d.u_in ? d.u_in + r * T * (n + 1) : nullptr;
        double *summ = d.summaries + r * T * SMCB_SUMMARY_STRIDE;
        double *momr = mom ? d.moments + r * T * 2 * kMaxD : nullptr;
        // the recursion's state: identical bits in every thread
        double logLt = 0.0, lm_prev = 0.0, reset_c = 0.0, xm = 0.0, xs = 1.0;
        bool rs = false;                                 // does step t resample (decided at the end of step t - 1)
        for (int64_t t = 0; t < T; t++) {
            const StepK k = step_consts(fa, t);
            const StepK kprev = step_consts(fa, t - 1);
            const int cur = (int)((t - 1) & 1), nxt = (int)(t & 1);
            const double *zt = zr ? zr + t * NZ * n : nullptr;
            const double *ut = ur ? ur + t * (n + 1) : nullptr;
            double u_sys = 0.0, zlast = 1.0;
            if (rs) {
                // A = resampling(scheme, aux.W, M=N) (core.py:329-331)
                LoadWeights<M, FK> load;
                load.lw = lw; load.X = X[cur]; load.ntot = ld; load.m = xm; load.s = xs;
                load.model = model; load.kprev = kprev;
                scan_range<BS>(load, 0, n, 0.0, CUDART_INF, cdf, s_warp);
                if (MULTI) {                             // exponential spacings, n + 1 of them (resampling.py:536-537)
                    for (int64_t i = 2 * (int64_t)threadIdx.x; i <= n; i += 2 * BS) {
                        double v0, v1;
                        spacings_pair(key, (uint32_t)t, ut, i, n + 1, v0, v1);
                        su[i] = v0;
                        if (i + 1 <= n) su[i + 1] = v1;
                    }
                    __syncthreads();
                    scan_range<BS>(LoadPlain{su}, 0, n + 1, 0.0, CUDART_INF, su, s_warp);
                    zlast = su[n];
                }
                if (SCHEME == SMCB_RS_SYSTEMATIC) u_sys = systematic_u(key, t, ut);
            }
            const bool last_apf = APF && t + 1 < T;
            const bool write_A = rs && t == T - 1;
            Acc<1> acc;
            acc_init(acc);
            Lse3 aux = lse3_empty();
            for (int64_t p = threadIdx.x; p < npairs; p += BS) {
                const bool two = 2 * p + 1 < n;
                double z[2][NZ];
                pair_normals<NZ>(key, (uint64_t)p, (uint32_t)t, zt, n, p, z);
                double x[2][1], l[2], av[2];
                if (t == 0) {                            // generate_particles + reweight (core.py:315-324)
#pragma unroll
                    for (int j = 0; j < 2; j++) {
                        double dd;
                        model_init<M, FK>(model, k, z[j], x[j], dd);
                        l[j] = fix_nan(dd);
                        av[j] = last_apf ? fix_nan(l[j] + model_logeta<M>(model, k, x[j])) : -CUDART_INF;
                    }
                } else {
                    double xp[2][1], base[2];
                    if (rs) {
                        double us[2] = {0.0, 0.0};
                        if (SCHEME == SMCB_RS_STRATIFIED) {
                            if (ut) { us[0] = ut[2 * p]; us[1] = two ? ut[2 * p + 1] : 0.0; }
                            else uniform_pair(key, (uint64_t)p, (uint32_t)t, kPurposeUniform, us[0], us[1]);
                        }
#pragma unroll
                        for (int j = 0; j < 2; j++) {
                            const int64_t kk = two ? 2 * p + j : 2 * p;
                            double s_k;
                            if (SCHEME == SMCB_RS_SYSTEMATIC) s_k = (u_sys + (double)kk) / Nd;          // resampling.py:609
                            else if (SCHEME == SMCB_RS_STRATIFIED) s_k = (us[j] + (double)kk) / Nd;     // resampling.py:602
                            else s_k = su[kk] / zlast;                                                   // resampling.py:537
                            int64_t a = lower_bound_plain(cdf, n, s_k);
                            a = a < n - 1 ? a : n - 1;
                            if (write_A && (j == 0 || two)) d.A[r * ld + kk] = a;
                            xp[j][0] = X[cur][a];
                            // core.py:302-305: lw = log_mean_exp(logetat, W) - logetat[A] for an APF, else 0
                            base[j] = APF ? reset_c - model_logeta<M>(model, kprev, xp[j]) : reset_c;
                        }
                    } else {                             // A = arange(N), Xp = X (core.py:335-336)
                        xp[0][0] = X[cur][2 * p]; base[0] = lw[2 * p];
                        xp[1][0] = two ? X[cur][2 * p + 1] : 0.0; base[1] = two ? lw[2 * p + 1] : 0.0;
                    }
#pragma unroll
                    for (int j = 0; j < 2; j++) {
                        double dd;
                        model_move<M, FK>(model, k, xp[j], z[j], x[j], dd);
                        l[j] = fix_nan(base[j] + dd);    // Weights.add, resampling.py:241-244
                        av[j] = last_apf ? fix_nan(l[j] + model_logeta<M>(model, k, x[j])) : -CUDART_INF;
                    }
                }
                X[nxt][2 * p] = x[0][0];
                lw[2 * p] = l[0];
                if (two) {
                    X[nxt][2 * p + 1] = x[1][0];
                    lw[2 * p + 1] = l[1];
                } else {                                 // masked slot contributes exactly 0
                    x[1][0] = 0.0; l[1] = -CUDART_INF; av[1] = -CUDART_INF;
                }
                acc_add_batch<2, 1>(acc, l, x, mom);
                if (APF) lse3_add_batch<2>(aux, av);
            }
            // CTA-wide (max, sum exp, sum exp^2) [+ auxiliary] [+ moments]: maximum first, then one exponential per
            // accumulator, fixed butterfly order
            double mx[2] = {acc.w.m, APF ? aux.m : -CUDART_INF};
            block_max_all<2, BS>(mx, s_red);
            const double ew = shift_factor_t(acc.w.m, mx[0]);
            const double ea = APF ? shift_factor_t(aux.m, mx[1]) : 0.0;
            double v[6] = {acc.w.s * ew, acc.w.q * (ew * ew), APF ? aux.s * ea : 0.0, APF ? aux.q * (ea * ea) : 0.0,
                           mom ? acc.sx[0] * ew : 0.0, mom ? acc.sxx[0] * ew : 0.0};
            block_sum_all<6, BS>(v, s_red);
            // compute_summaries (core.py:351-367) and time_to_resample of step t + 1 (core.py:181-183)
            const Lse3 w{mx[0], v[0], v[1]}, xa{APF ? mx[1] : mx[0], APF ? v[2] : v[0], APF ? v[3] : v[1]};
            double log_mean, ess, lm_aux, ess_aux;
            weights_scalars(w, Nd, log_mean, ess);
            if (APF) weights_scalars(xa, Nd, lm_aux, ess_aux);
            else { lm_aux = log_mean; ess_aux = ess; }
            const bool fresh = (t == 0) || rs;
            logLt = logLt + (fresh ? log_mean : (log_mean - lm_prev));
            if (threadIdx.x == 0) {
                double *row = summ + t * SMCB_SUMMARY_STRIDE;
                row[0] = ess; row[1] = logLt; row[2] = rs ? 1.0 : 0.0; row[3] = log_mean;
                if (mom) {                               // wmean_and_var, resampling.py:320-338
                    double *mrow = momr + t * 2 * kMaxD;
                    const double mean = v[4] / w.s;
#pragma unroll
                    for (int c = 0; c < kMaxD; c++) { mrow[c] = 0.0; mrow[kMaxD + c] = 0.0; }
                    mrow[0] = mean;
                    mrow[kMaxD] = v[5] / w.s - mean * mean;
                }
            }
            lm_prev = log_mean;
            reset_c = APF ? (log(xa.s) + xa.m) - (log(w.s) + w.m) : 0.0;
            xm = xa.m;
            xs = xa.s;
            rs = (t + 1 < T) && (ess_aux < Nd * essrmin);           // strict <, NaN -> False
        }
        if (RESIDENT) {                                  // the last two generations and the last weights
            double *Xo = d.X + r * 2 * ld, *lwo = d.lw + r * ld;
            for (int64_t i = threadIdx.x; i < n; i += BS) {
                Xo[i] = X[0][i];
                Xo[ld + i] = X[1][i];
                lwo[i] = lw[i];
            }
        }
    }
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
template <class M, int FK, int SCHEME, bool RES>
static int batch_kernel_setup(smcb_ctx *c, const smcb_batch_desc &d, size_t smem, int &grid) {
    auto kern = k_batch<M, FK, SCHEME, RES>;
    SMCB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int nb = 0, sms = 0;
    SMCB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kern, kBatchBS, smem));
    SMCB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device));
    if (nb < 1) {
        set_error("batched filter: the kernel does not fit on an SM of this device");
        return SMCB_ECUDA;
    }
    const int64_t g = (int64_t)nb * sms;
    grid = (int)(d.R < g ? d.R : g);
    return SMCB_OK;
}

// plan (out != NULL) or launch one group
template <class M, int FK, int SCHEME>
static int batch_one(smcb_ctx *c, const smcb_batch_desc &d, int64_t *out) {
    int optin = 0;
    SMCB_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, c->device));
    cudaFuncAttributes fa;
    SMCB_CUDA(cudaFuncGetAttributes(&fa, k_batch<M, FK, SCHEME, true>));
    const size_t smem_res = kMathTabBytes + (size_t)resident_doubles(d.N, SCHEME) * sizeof(double);
    const bool fits = smem_res + fa.sharedSizeBytes <= (size_t)optin;
    int tier = d.tier == SMCB_BATCH_AUTO ? (fits ? SMCB_BATCH_RESIDENT : SMCB_BATCH_STREAMING) : d.tier;
    if (tier == SMCB_BATCH_RESIDENT && !fits) {
        set_error("batched filter: N=%lld does not fit the resident tier", (long long)d.N);
        return SMCB_EINVAL;
    }
    int grid = 0, rc;
    if (tier == SMCB_BATCH_RESIDENT) rc = batch_kernel_setup<M, FK, SCHEME, true>(c, d, smem_res, grid);
    else rc = batch_kernel_setup<M, FK, SCHEME, false>(c, d, kMathTabBytes, grid);
    if (rc != SMCB_OK) return rc;
    if (out) {
        out[0] = tier;
        out[1] = grid;
        return SMCB_OK;
    }
    SMCB_REQUIRE(tier == SMCB_BATCH_RESIDENT || (d.cdf && (SCHEME != SMCB_RS_MULTINOMIAL || d.scratch)),
                 "smcb_batch_run: the streaming tier needs cdf (and scratch for multinomial)");
    if (tier == SMCB_BATCH_RESIDENT)
        k_batch<M, FK, SCHEME, true><<<grid, kBatchBS, smem_res, c->stream>>>(d, c->math_tab);
    else
        k_batch<M, FK, SCHEME, false><<<grid, kBatchBS, kMathTabBytes, c->stream>>>(d, c->math_tab);
    c->launches++;
    SMCB_CUDA(cudaGetLastError());
    return SMCB_OK;
}

template <class M, int FK>
static int batch_scheme(smcb_ctx *c, const smcb_batch_desc &d, int64_t *out) {
    bool built = false;
    const int rc = with_scheme(d.scheme, [&](auto scheme) {
        built = true;
        return batch_one<M, FK, decltype(scheme)::value>(c, d, out);
    });
    if (!built) set_error("batched filter: resampling scheme %d is not built", d.scheme);
    return rc;
}

template <class M>
static int batch_fk(smcb_ctx *c, const smcb_batch_desc &d, int64_t *out) {
    bool built = false;
    const int rc = with_fk<M>(d.fk, [&](auto fk) {
        built = true;
        return batch_scheme<M, decltype(fk)::value>(c, d, out);
    });
    if (!built) set_error("batched filter: Feynman-Kac kind %d is not built for model %d", d.fk, d.model);
    return rc;
}

static int batch_dispatch(smcb_ctx *c, const smcb_batch_desc *dp, int64_t *out) {
    SMCB_REQUIRE(c && dp, "smcb_batch: NULL argument");
    const smcb_batch_desc &d = *dp;
    SMCB_REQUIRE(d.N >= 1 && d.T >= 1 && d.R >= 1, "smcb_batch: bad shape N=%lld T=%lld R=%lld", (long long)d.N,
                 (long long)d.T, (long long)d.R);
    SMCB_REQUIRE(d.n_params >= 0 && d.n_params <= SMCB_MAX_PARAMS, "smcb_batch: bad n_params %d", d.n_params);
    if (d.dim != 1 || d.dy != 1) {
        set_error("batched filter: d-dimensional models are not built (dim=%d, dy=%d)", d.dim, d.dy);
        return SMCB_ENOSYS;
    }
    SMCB_REQUIRE(d.tier >= SMCB_BATCH_AUTO && d.tier <= SMCB_BATCH_STREAMING, "smcb_batch: bad tier %d", d.tier);
    if (!out) {
        SMCB_REQUIRE(d.seed && d.essrmin && d.params && d.data && d.X && d.lw && d.A && d.summaries,
                     "smcb_batch: NULL buffer");
    }
    bool built = false;
    const int rc = with_model(d.model, d.dim, [&](auto m) {
        using M = decltype(m);
        if constexpr (M::D == 1) {
            built = true;
            return batch_fk<M>(c, d, out);
        } else {
            return SMCB_ENOSYS;
        }
    });
    if (!built) set_error("batched filter: model id %d is not built", d.model);
    return rc;
}

}  // namespace smcb

extern "C" int smcb_batch_plan(smcb_ctx *c, const smcb_batch_desc *d, int64_t out[2]) {
    SMCB_REQUIRE(out, "smcb_batch_plan: NULL out");
    return smcb::batch_dispatch(c, d, out);
}

extern "C" int smcb_batch_run(smcb_ctx *c, const smcb_batch_desc *d) {
    return smcb::batch_dispatch(c, d, nullptr);
}
