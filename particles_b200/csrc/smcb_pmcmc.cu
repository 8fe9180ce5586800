// smcb_pmcmc.cu -- conditional SMC with its whole history and a trajectory draw, one CTA per chain: the
// state update of Particle Gibbs (particles/mcmc.py:453-475 and 594-609).
//
//   k_csmc<Model, FK>: the geometry of k_bank (smcb_bank.cu): 256 threads, one CTA per chain, a persistent grid and
//   the math tables staged by TMA.  The step body is the one of k_bank with multinomial resampling -- same thread-to-
//   pair map, same Philox counters under the chain's key, same LoadWeights / scan_range / spacings_pair /
//   lower_bound_plain / model_move / acc_add_batch and the same fixed-order CTA merge -- so with the pin off a chain
//   gives the bits of the bank filter with the same key.  Differences:
//     * every generation stays in device memory: X, lw, A (R, T, ld); step t reads generation t - 1 back from its own
//       history row, so there is one tier.  The CDF and the spacings live in shared memory next to the tables, which
//       bounds N (smcb_csmc_plan);
//     * pin on: slot 0 is x*[t] with ancestor 0, and its log-weight increment is logG(t, x*[t-1], x*[t]) computed at
//       that state (fk_logG0 / fk_logG).  The reference leaves Xp[0] at the discarded resampled ancestor; here the
//       previous state of the pinned path is used, so its weight is that of the conditional path.  Slot 0 still
//       draws its normals, so every other slot keeps the counters of k_bank;
//     * after step T - 1 the same launch draws one trajectory: one multinomial draw on W_{T-1}, then either the
//       ancestors are traced back (extract_one_trajectory, smoothing.py:256-269) or one backward draw per step is made
//       from lw_t + logpt(t + 1, X_t, x_{t+1}) (backward_sampling_ON2 with M = 1, smoothing.py:291-311).  Its
//       uniforms come from purpose kPurposeTraj, a stream the forward pass never uses.
#include "smcb_batch.cuh"

namespace smcb {

// the uniform of the trajectory draw at step t: injected (ud[t]) or Philox
__device__ __forceinline__ double traj_uniform(const Philox &key, int64_t t, const double *ud) {
    if (ud) return ud[t];
    double u0, u1;
    uniform_pair(key, 0ull, (uint32_t)t, kPurposeTraj, u0, u1);
    return u0;
}

// exp(v[i] - m) of a shared-memory row: the unnormalised weights of one backward draw
struct LoadShiftedExp {
    const double *v;
    double m;
    __device__ __forceinline__ void operator()(int64_t i0, int64_t n, double (&o)[8]) const {
#pragma unroll
        for (int j = 0; j < 8; j++) o[j] = (i0 + j < n) ? texp(v[i0 + j] - m) : 0.0;
    }
};

__device__ __forceinline__ int64_t search_clamped(const double *cdf, int64_t n, double key) {
    const int64_t a = lower_bound_plain(cdf, n, key);
    return a < n - 1 ? a : n - 1;
}

template <class M, int FK>
__global__ void __launch_bounds__(kBatchBS) k_csmc(const smcb_csmc_desc d, const double *math_tab) {
    static_assert(M::D == 1 && M::NZ == 1, "the conditional filter runs the 1-D models");
    static_assert(!FkTraits<FK>::apf, "the conditional filter has no auxiliary kinds");
    constexpr int BS = kBatchBS;
    extern __shared__ __align__(128) double s_dyn[];     // math tables | cdf (ld) | spacings / backward weights (ld + 2)
    __shared__ M s_model;
    __shared__ Philox s_key;
    __shared__ double s_red[(BS / 32 + 1) * 6];
    __shared__ double s_warp[BS / 32];
    __shared__ __align__(8) uint64_t s_tabbar;
    if (threadIdx.x == 0) mtab_issue(math_tab, &s_tabbar);
    __syncthreads();
    mbar_wait(&s_tabbar, 0);
    const int64_t n = d.N, ld = batch_ld(n), T = d.T, npairs = (n + 1) >> 1;
    const double Nd = (double)n, essrmin = d.essrmin;
    const bool pin = d.pin != 0;
    double *const cdf = s_dyn + kMathTabDoubles, *const su = cdf + ld;
    for (int64_t r = blockIdx.x; r < d.R; r += gridDim.x) {
        __syncthreads();                                 // the previous chain is done with s_model, s_key, cdf, su
        if (threadIdx.x == 0) {
            s_model.load(d.params + r * d.n_params);
            s_key = key_of(d.key[r]);
        }
        __syncthreads();
        const M &model = s_model;
        const Philox &key = s_key;
        double *Xh = d.X + r * T * ld, *lwh = d.lw + r * T * ld;
        int64_t *Ah = d.A + r * T * ld;
        const double *xs = d.xstar ? d.xstar + r * T : nullptr;
        FilterArgs fa = {};                              // what step_consts reads: this chain's data row
        fa.data = d.data + r * d.data_ld;
        fa.sc = d.step_consts ? d.step_consts + r * d.sc_ld : nullptr;
        fa.dy = 1;
        fa.T = T;
        const double *zr = d.z_in ? d.z_in + r * T * n : nullptr;
        const double *ur = d.u_in ? d.u_in + r * T * (n + 1) : nullptr;
        const double *udr = d.ud_in ? d.ud_in + r * T : nullptr;
        double *summ = d.summaries ? d.summaries + r * T * SMCB_SUMMARY_STRIDE : nullptr;
        // the recursion's state: identical bits in every thread
        double logLt = 0.0, lm_prev = 0.0, xm = 0.0, xsum = 1.0;
        bool rs = false;                                 // does step t resample (decided at the end of step t - 1)
        for (int64_t t = 0; t < T; t++) {
            const StepK k = step_consts(fa, t);
            const StepK kprev = step_consts(fa, t - 1);
            double *Xt = Xh + t * ld, *lwt = lwh + t * ld;
            int64_t *At = Ah + t * ld;
            const double *Xq = Xh + (t - 1) * ld, *lwq = lwh + (t - 1) * ld;    // generation t - 1 (t > 0)
            const double *zt = zr ? zr + t * n : nullptr;
            double zlast = 1.0;
            if (rs) {
                // A = multinomial(W, M=N) (core.py:329-331, resampling.py:536-537)
                LoadWeights<M, FK> load;
                load.lw = lwq; load.X = Xq; load.ntot = ld; load.m = xm; load.s = xsum;
                load.model = model; load.kprev = kprev;
                scan_range<BS>(load, 0, n, 0.0, CUDART_INF, cdf, s_warp);
                const double *ut = ur ? ur + t * (n + 1) : nullptr;
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
            Acc<1> acc;
            acc_init(acc);
            for (int64_t p = threadIdx.x; p < npairs; p += BS) {
                const bool two = 2 * p + 1 < n;
                const bool pinned = pin && p == 0;       // slot 0 of this pair follows x*
                double z[2][1];
                pair_normals<1>(key, (uint64_t)p, (uint32_t)t, zt, n, p, z);
                double x[2][1], l[2];
                int64_t a[2] = {2 * p, 2 * p + 1};
                if (t == 0) {                            // generate_particles + reweight (core.py:315-324)
#pragma unroll
                    for (int jj = 0; jj < 2; jj++) {
                        double dd;
                        model_init<M, FK>(model, k, z[jj], x[jj], dd);
                        l[jj] = fix_nan(dd);
                    }
                    if (pinned) {                        // CSMC.generate_particles (mcmc.py:468-470)
                        x[0][0] = xs[0];
                        l[0] = fix_nan(fk_logG0<M, FK>(model, k, x[0][0]));
                    }
                } else {
                    double xp[2][1], base[2];
                    if (rs) {
#pragma unroll
                        for (int jj = 0; jj < 2; jj++) {
                            const int64_t kk = two ? 2 * p + jj : 2 * p;
                            a[jj] = search_clamped(cdf, n, su[kk] / zlast);                  // resampling.py:537
                            xp[jj][0] = Xq[a[jj]];
                            base[jj] = 0.0;
                        }
                    } else {                             // A = arange(N), Xp = X (core.py:335-336)
                        xp[0][0] = Xq[2 * p]; base[0] = lwq[2 * p];
                        xp[1][0] = two ? Xq[2 * p + 1] : 0.0; base[1] = two ? lwq[2 * p + 1] : 0.0;
                    }
#pragma unroll
                    for (int jj = 0; jj < 2; jj++) {
                        double dd;
                        model_move<M, FK>(model, k, xp[jj], z[jj], x[jj], dd);
                        l[jj] = fix_nan(base[jj] + dd);  // Weights.add, resampling.py:241-244
                    }
                    if (pinned) {                        // CSMC.resample_move (mcmc.py:472-475), Xp[0] = x*[t-1]
                        a[0] = 0;
                        x[0][0] = xs[t];
                        l[0] = fix_nan((rs ? 0.0 : lwq[0]) + fk_logG<M, FK>(model, k, xs[t - 1], x[0][0]));
                    }
                }
                Xt[2 * p] = x[0][0];
                lwt[2 * p] = l[0];
                At[2 * p] = a[0];
                if (two) {
                    Xt[2 * p + 1] = x[1][0];
                    lwt[2 * p + 1] = l[1];
                    At[2 * p + 1] = a[1];
                } else {                                 // masked slot contributes exactly 0
                    x[1][0] = 0.0; l[1] = -CUDART_INF;
                }
                acc_add_batch<2, 1>(acc, l, x, false);
            }
            // CTA-wide (max, sum exp, sum exp^2): the merge of k_bank, in the same fixed order
            double mx[2] = {acc.w.m, -CUDART_INF};
            block_max_all<2, BS>(mx, s_red);
            const double ew = shift_factor_t(acc.w.m, mx[0]);
            double v[6] = {acc.w.s * ew, acc.w.q * (ew * ew), 0.0, 0.0, 0.0, 0.0};
            block_sum_all<6, BS>(v, s_red);
            // compute_summaries (core.py:351-367) and time_to_resample of step t + 1 (core.py:181-183)
            const Lse3 w{mx[0], v[0], v[1]};
            double log_mean, ess;
            weights_scalars(w, Nd, log_mean, ess);
            const bool fresh = (t == 0) || rs;
            logLt = logLt + (fresh ? log_mean : (log_mean - lm_prev));
            if (summ && threadIdx.x == 0) {
                double *row = summ + t * SMCB_SUMMARY_STRIDE;
                row[0] = ess; row[1] = logLt; row[2] = rs ? 1.0 : 0.0; row[3] = log_mean;
            }
            lm_prev = log_mean;
            xm = w.m;
            xsum = w.s;
            rs = (t + 1 < T) && (ess < Nd * essrmin);   // strict <, NaN -> False
        }
        if (threadIdx.x == 0) d.logLt[r] = logLt;
        // the trajectory draw: its final index from W_{T-1} (block barriers in the reductions above order the
        // history writes before these reads)
        double *traj = d.traj + r * T;
        {
            LoadWeights<M, FK> load;
            load.lw = lwh + (T - 1) * ld; load.X = Xh + (T - 1) * ld; load.ntot = ld; load.m = xm; load.s = xsum;
            load.model = model; load.kprev = step_consts(fa, T - 1);
            scan_range<BS>(load, 0, n, 0.0, CUDART_INF, cdf, s_warp);
        }
        int64_t idx = search_clamped(cdf, n, traj_uniform(key, T - 1, udr));
        if (d.draw == SMCB_CSMC_GENEALOGY) {
            if (threadIdx.x == 0) {
                for (int64_t t = T - 1; t >= 0; t--) {
                    traj[t] = Xh[t * ld + idx];
                    if (t > 0) idx = Ah[t * ld + idx];
                }
            }
        } else {
            TransDensity<M> td;
            td.init(model);
            double xnext = Xh[(T - 1) * ld + idx];
            if (threadIdx.x == 0) traj[T - 1] = xnext;
            double *lwm = su;
            for (int64_t t = T - 2; t >= 0; t--) {
                // lw_t + logpt(t + 1, X_t, x_{t+1}), exp_and_normalise, multinomial_once (smoothing.py:303-308)
                const StepK k1 = step_consts(fa, t + 1);
                const double *Xt = Xh + t * ld, *lwt = lwh + t * ld;
                double mloc = -CUDART_INF;
                for (int64_t i = threadIdx.x; i < n; i += BS) {
                    double lc[1];
                    td.loc(model, k1, Xt + i, lc);
                    const double e = fix_nan(lwt[i] + td.lpdf(model, lc, &xnext));
                    lwm[i] = e;
                    mloc = fmax(mloc, e);
                }
                double mxb[1] = {mloc};
                block_max_all<1, BS>(mxb, s_red);        // its barriers also publish lwm
                scan_range<BS>(LoadShiftedExp{lwm, mxb[0]}, 0, n, 0.0, CUDART_INF, cdf, s_warp);
                // a row with no positive weight (every term -inf) gives 0, the rule of smcb_smooth.cuh: m = -inf makes
                // every exp(v - m) texp(NaN) = NaN, so the key is NaN and the search stops at 0
                idx = search_clamped(cdf, n, traj_uniform(key, t, udr) * cdf[n - 1]);
                xnext = Xt[idx];
                if (threadIdx.x == 0) traj[t] = xnext;
                __syncthreads();                         // every thread has searched cdf before it is rewritten
            }
        }
    }
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
// shared memory a launch needs besides the math tables: the cdf (ld) and the spacings (ld + 2)
static size_t csmc_smem(int64_t n) { return kMathTabBytes + (size_t)(2 * batch_ld(n) + 2) * sizeof(double); }

// plan (out != NULL) or launch
template <class M, int FK>
static int csmc_one(smcb_ctx *c, const smcb_csmc_desc &d, int64_t *out) {
    auto kern = k_csmc<M, FK>;
    int optin = 0, sms = 0, nb = 0;
    SMCB_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, c->device));
    SMCB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device));
    cudaFuncAttributes fa;
    SMCB_CUDA(cudaFuncGetAttributes(&fa, kern));
    // the largest N whose buffers fit: 2 ld + 2 doubles after the tables and the static shared memory
    const int64_t room = ((int64_t)optin - (int64_t)fa.sharedSizeBytes - (int64_t)kMathTabBytes) / 8 - 2;
    const int64_t nmax = (room / 2) & ~(int64_t)1;
    if (d.N > nmax) {
        set_error("conditional SMC: N=%lld is above the shared-memory bound %lld", (long long)d.N, (long long)nmax);
        return SMCB_ENOSYS;
    }
    const size_t smem = csmc_smem(d.N);
    SMCB_TRY(set_smem(kern, smem));
    SMCB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kern, kBatchBS, smem));
    if (nb < 1) {
        set_error("conditional SMC: the kernel does not fit on an SM of this device");
        return SMCB_ECUDA;
    }
    const int64_t g = (int64_t)nb * sms;
    const int grid = (int)(d.R < g ? (d.R > 0 ? d.R : 1) : g);
    if (out) {
        out[0] = nmax;
        out[1] = grid;
        return SMCB_OK;
    }
    if (d.R == 0) return SMCB_OK;
    return launch(c, kern, grid, kBatchBS, smem, d, c->math_tab);
}

static int csmc_dispatch(smcb_ctx *c, const smcb_csmc_desc *dp, int64_t *out) {
    SMCB_REQUIRE(c && dp, "smcb_csmc: NULL argument");
    const smcb_csmc_desc &d = *dp;
    SMCB_REQUIRE(d.N >= 1 && d.T >= 1 && d.R >= 0, "smcb_csmc: bad shape N=%lld T=%lld R=%lld", (long long)d.N,
                 (long long)d.T, (long long)d.R);
    SMCB_REQUIRE(d.n_params >= 0 && d.n_params <= SMCB_MAX_PARAMS, "smcb_csmc: bad n_params %d", d.n_params);
    SMCB_REQUIRE(d.draw == SMCB_CSMC_GENEALOGY || d.draw == SMCB_CSMC_BACKWARD, "smcb_csmc: bad draw mode %d",
                 d.draw);
    if (!out) {
        SMCB_REQUIRE(d.key && d.params && d.data && d.X && d.lw && d.A && d.traj && d.logLt,
                     "smcb_csmc_run: NULL buffer");
        SMCB_REQUIRE(!d.pin || d.xstar, "smcb_csmc_run: the pinned path needs xstar");
        SMCB_REQUIRE(d.data_ld == 0 || d.data_ld >= d.T, "smcb_csmc_run: bad data_ld");
        SMCB_REQUIRE(!d.step_consts || d.sc_ld == 0 || d.sc_ld >= d.T, "smcb_csmc_run: bad sc_ld");
    }
    bool built = false;
    const int rc = with_model(d.model, 1, [&](auto m) {
        using M = decltype(m);
        if constexpr (M::D == 1) {
            return with_fk<M>(d.fk, [&](auto fk) {
                constexpr int FK = decltype(fk)::value;
                if constexpr (FK == SMCB_FK_BOOTSTRAP || FK == SMCB_FK_GUIDED) {
                    built = true;
                    return csmc_one<M, FK>(c, d, out);
                } else {
                    return SMCB_ENOSYS;
                }
            });
        } else {
            return SMCB_ENOSYS;
        }
    });
    if (!built) {
        set_error("conditional SMC: model %d, Feynman-Kac kind %d is not built", d.model, d.fk);
        return SMCB_ENOSYS;
    }
    return rc;
}

}  // namespace smcb

using namespace smcb;

extern "C" int smcb_csmc_plan(smcb_ctx *c, const smcb_csmc_desc *d, int64_t out[2]) {
    SMCB_REQUIRE(out, "smcb_csmc_plan: NULL out");
    return csmc_dispatch(c, d, out);
}

extern "C" int smcb_csmc_run(smcb_ctx *c, const smcb_csmc_desc *d) { return csmc_dispatch(c, d, nullptr); }
