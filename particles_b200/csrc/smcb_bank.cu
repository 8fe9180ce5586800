// smcb_bank.cu -- a bank of resumable filters (the inner filters of SMC^2, particles/smc_samplers.py:1038-1167) and
// the row operations the outer sampler applies to it.
//
//   k_bank<Model, FK, SCHEME, RESIDENT>: the geometry of k_batch (smcb_batch.cu): 256 threads, one CTA per filter,
//   a persistent grid, the resident tier when the filter fits in shared memory and the streaming tier otherwise.
//   Filter r runs from the step t0 its state row records (0: from M0) to the common step t1 and writes its state
//   back: the last two generations X, lw, and the scalars of the recursion (SMCB_BANK_STATE).  The step body is the
//   one of k_batch -- same thread-to-pair map, same Philox counters under the filter's key, same LoadWeights /
//   scan_range / lower_bound_plain / model_move / acc_add_batch and the same fixed-order CTA merge -- so
//     * advancing [0, t) and then [t, T) gives the bits of advancing [0, T) in one call, in both tiers;
//     * filter r gives the bits of the k_batch run with seed key[r] (multiSMC), i.e. what SMC(seed = key[r]) draws.
//
//   Row operations (one CTA per destination row, plain copies):
//     gather:  dst[i] = src[A[i]] (the outer sampler's X[A]); the first copy of an ancestor (lowest i) keeps its
//              key, every further copy gets bank_key(seed, counter + i), so no two filters share a random stream;
//     merge:   dst[i] = src[i] where accepted[i] (the Metropolis copy-where of the outer move);
//     keys:    key[i] = bank_key(seed, counter + i).
#include "smcb_batch.cuh"

namespace smcb {

// the splitmix64 finaliser: a bijection of the 64-bit integers
__host__ __device__ inline uint64_t fmix64(uint64_t z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// key number c under the sampler's seed: a bijection of c for a fixed seed, so distinct counters give distinct keys
__host__ __device__ inline uint64_t bank_key(uint64_t seed, uint64_t c) { return fmix64(fmix64(seed) + c); }

template <class M, int FK, int SCHEME, bool RESIDENT>
__global__ void __launch_bounds__(kBatchBS) k_bank(const smcb_bank_desc d, const double *math_tab) {
    static_assert(M::D == 1, "the filter bank runs the 1-D models");
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
    const int64_t n = d.N, ld = batch_ld(n), T = d.T, npairs = (n + 1) >> 1, t1 = d.t1;
    const int64_t nrun = d.idx ? d.n_idx : d.R;
    const double Nd = (double)n, essrmin = d.essrmin;
    for (int64_t j = blockIdx.x; j < nrun; j += gridDim.x) {
        const int64_t r = d.idx ? d.idx[j] : j;
        double *st = d.state + r * SMCB_BANK_STATE;
        const int64_t t0 = d.restart ? 0 : (int64_t)st[0];
        if (t0 >= t1) continue;                          // nothing to do: the rows stay as they are
        __syncthreads();                                 // the previous filter is done with s_model, s_key, buffers
        if (threadIdx.x == 0) {
            s_model.load(d.params + r * d.n_params);
            s_key = key_of(d.key[r]);
        }
        const M &model = s_model;
        const Philox &key = s_key;
        double *Xd = d.X + r * 2 * ld, *lwd = d.lw + r * ld;
        double *X[2], *lw, *cdf, *su;
        if (RESIDENT) {
            double *b = s_dyn + kMathTabDoubles;
            X[0] = b; X[1] = b + ld; lw = b + 2 * ld; cdf = b + 3 * ld; su = b + 4 * ld;
            if (t0 > 0) {                                // resume: the last two generations and the weights
                for (int64_t i = threadIdx.x; i < n; i += BS) {
                    X[0][i] = Xd[i];
                    X[1][i] = Xd[ld + i];
                    lw[i] = lwd[i];
                }
            }
        } else {
            X[0] = Xd; X[1] = Xd + ld; lw = lwd; cdf = d.cdf + blockIdx.x * ld;
            su = MULTI ? d.scratch + blockIdx.x * (ld + 2) : nullptr;
        }
        __syncthreads();
        FilterArgs fa = {};                              // what step_consts reads: the data and this filter's row
        fa.data = d.data;
        fa.sc = d.step_consts ? d.step_consts + r * d.sc_ld : nullptr;
        fa.dy = 1;
        fa.T = T;
        double *summ = d.summaries ? d.summaries + r * T * SMCB_SUMMARY_STRIDE : nullptr;
        // the recursion's state: identical bits in every thread
        double logLt = 0.0, lm_prev = 0.0, reset_c = 0.0, xm = 0.0, xs = 1.0, loglt = 0.0;
        bool rs = false;                                 // does step t resample (decided at the end of step t - 1)
        if (t0 > 0) {
            logLt = st[1]; lm_prev = st[2]; reset_c = st[3]; xm = st[4]; xs = st[5]; rs = st[6] != 0.0;
        }
        for (int64_t t = t0; t < t1; t++) {
            const StepK k = step_consts(fa, t);
            const StepK kprev = step_consts(fa, t - 1);
            const int cur = (int)((t - 1) & 1), nxt = (int)(t & 1);
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
                        spacings_pair(key, (uint32_t)t, nullptr, i, n + 1, v0, v1);
                        su[i] = v0;
                        if (i + 1 <= n) su[i + 1] = v1;
                    }
                    __syncthreads();
                    scan_range<BS>(LoadPlain{su}, 0, n + 1, 0.0, CUDART_INF, su, s_warp);
                    zlast = su[n];
                }
                if (SCHEME == SMCB_RS_SYSTEMATIC) u_sys = systematic_u(key, t, nullptr);
            }
            const bool last_apf = APF && t + 1 < T;
            const bool write_A = rs && t == t1 - 1 && d.A != nullptr;
            Acc<1> acc;
            acc_init(acc);
            Lse3 aux = lse3_empty();
            for (int64_t p = threadIdx.x; p < npairs; p += BS) {
                const bool two = 2 * p + 1 < n;
                double z[2][NZ];
                pair_normals<NZ>(key, (uint64_t)p, (uint32_t)t, nullptr, n, p, z);
                double x[2][1], l[2], av[2];
                if (t == 0) {                            // generate_particles + reweight (core.py:315-324)
#pragma unroll
                    for (int jj = 0; jj < 2; jj++) {
                        double dd;
                        model_init<M, FK>(model, k, z[jj], x[jj], dd);
                        l[jj] = fix_nan(dd);
                        av[jj] = last_apf ? fix_nan(l[jj] + model_logeta<M>(model, k, x[jj])) : -CUDART_INF;
                    }
                } else {
                    double xp[2][1], base[2];
                    if (rs) {
                        double us[2] = {0.0, 0.0};
                        if (SCHEME == SMCB_RS_STRATIFIED)
                            uniform_pair(key, (uint64_t)p, (uint32_t)t, kPurposeUniform, us[0], us[1]);
#pragma unroll
                        for (int jj = 0; jj < 2; jj++) {
                            const int64_t kk = two ? 2 * p + jj : 2 * p;
                            double s_k;
                            if (SCHEME == SMCB_RS_SYSTEMATIC) s_k = (u_sys + (double)kk) / Nd;          // resampling.py:609
                            else if (SCHEME == SMCB_RS_STRATIFIED) s_k = (us[jj] + (double)kk) / Nd;    // resampling.py:602
                            else s_k = su[kk] / zlast;                                                   // resampling.py:537
                            int64_t a = lower_bound_plain(cdf, n, s_k);
                            a = a < n - 1 ? a : n - 1;
                            if (write_A && (jj == 0 || two)) d.A[r * ld + kk] = a;
                            xp[jj][0] = X[cur][a];
                            // core.py:302-305: lw = log_mean_exp(logetat, W) - logetat[A] for an APF, else 0
                            base[jj] = APF ? reset_c - model_logeta<M>(model, kprev, xp[jj]) : reset_c;
                        }
                    } else {                             // A = arange(N), Xp = X (core.py:335-336)
                        xp[0][0] = X[cur][2 * p]; base[0] = lw[2 * p];
                        xp[1][0] = two ? X[cur][2 * p + 1] : 0.0; base[1] = two ? lw[2 * p + 1] : 0.0;
                    }
#pragma unroll
                    for (int jj = 0; jj < 2; jj++) {
                        double dd;
                        model_move<M, FK>(model, k, xp[jj], z[jj], x[jj], dd);
                        l[jj] = fix_nan(base[jj] + dd);  // Weights.add, resampling.py:241-244
                        av[jj] = last_apf ? fix_nan(l[jj] + model_logeta<M>(model, k, x[jj])) : -CUDART_INF;
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
                acc_add_batch<2, 1>(acc, l, x, false);
                if (APF) lse3_add_batch<2>(aux, av);
            }
            // CTA-wide (max, sum exp, sum exp^2) [+ auxiliary]: the merge of k_batch, in the same fixed order
            double mx[2] = {acc.w.m, APF ? aux.m : -CUDART_INF};
            block_max_all<2, BS>(mx, s_red);
            const double ew = shift_factor_t(acc.w.m, mx[0]);
            const double ea = APF ? shift_factor_t(aux.m, mx[1]) : 0.0;
            double v[6] = {acc.w.s * ew, acc.w.q * (ew * ew), APF ? aux.s * ea : 0.0, APF ? aux.q * (ea * ea) : 0.0,
                           0.0, 0.0};
            block_sum_all<6, BS>(v, s_red);
            // compute_summaries (core.py:351-367) and time_to_resample of step t + 1 (core.py:181-183)
            const Lse3 w{mx[0], v[0], v[1]}, xa{APF ? mx[1] : mx[0], APF ? v[2] : v[0], APF ? v[3] : v[1]};
            double log_mean, ess, lm_aux, ess_aux;
            weights_scalars(w, Nd, log_mean, ess);
            if (APF) weights_scalars(xa, Nd, lm_aux, ess_aux);
            else { lm_aux = log_mean; ess_aux = ess; }
            const bool fresh = (t == 0) || rs;
            loglt = fresh ? log_mean : (log_mean - lm_prev);
            logLt = logLt + loglt;
            if (summ && threadIdx.x == 0) {
                double *row = summ + t * SMCB_SUMMARY_STRIDE;
                row[0] = ess; row[1] = logLt; row[2] = rs ? 1.0 : 0.0; row[3] = log_mean;
            }
            lm_prev = log_mean;
            reset_c = APF ? (log(xa.s) + xa.m) - (log(w.s) + w.m) : 0.0;
            xm = xa.m;
            xs = xa.s;
            rs = (t + 1 < T) && (ess_aux < Nd * essrmin);           // strict <, NaN -> False
        }
        if (RESIDENT) {                                  // the generations this call holds, and the last weights
            const bool both = t0 > 0 || t1 - t0 >= 2;
            const int last = (int)((t1 - 1) & 1);
            for (int64_t i = threadIdx.x; i < n; i += BS) {
                Xd[last * ld + i] = X[last][i];
                if (both) Xd[(last ^ 1) * ld + i] = X[last ^ 1][i];
                lwd[i] = lw[i];
            }
        }
        if (threadIdx.x == 0) {                          // every thread read st before the first step's barriers
            st[0] = (double)t1; st[1] = logLt; st[2] = lm_prev; st[3] = reset_c;
            st[4] = xm; st[5] = xs; st[6] = rs ? 1.0 : 0.0; st[7] = loglt;
        }
    }
}

// ---------------------------------------------------------------------------
// row operations
// ---------------------------------------------------------------------------
constexpr int kRowBS = 128;

__global__ void k_first_fill(unsigned long long *first, int64_t R) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < R; i += (int64_t)gridDim.x * blockDim.x)
        first[i] = ~0ull;
}

// first[a] = the lowest destination index whose ancestor is a
__global__ void k_first_min(const int64_t *A, int64_t m, unsigned long long *first) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x)
        atomicMin(first + A[i], (unsigned long long)i);
}

__device__ __forceinline__ void copy_row(double *dst, const double *src, int64_t n) {
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
}

// one CTA per destination row i: source row A[i] (gather) or i (merge, where accepted[i])
__global__ void __launch_bounds__(kRowBS) k_bank_rows(const smcb_bank_desc s, const smcb_bank_desc dd,
                                                     const int64_t *A, const uint8_t *accepted,
                                                     const unsigned long long *first, uint64_t seed,
                                                     uint64_t counter, int64_t m) {
    const int64_t ld = batch_ld(s.N);
    for (int64_t i = blockIdx.x; i < m; i += gridDim.x) {
        if (accepted && !accepted[i]) continue;
        const int64_t a = A ? A[i] : i;
        copy_row(dd.X + i * 2 * ld, s.X + a * 2 * ld, 2 * ld);
        copy_row(dd.lw + i * ld, s.lw + a * ld, ld);
        copy_row(dd.state + i * SMCB_BANK_STATE, s.state + a * SMCB_BANK_STATE, SMCB_BANK_STATE);
        copy_row(dd.params + i * dd.n_params, s.params + a * s.n_params, s.n_params);
        if (dd.sc_ld > 0) copy_row(dd.step_consts + i * dd.sc_ld, s.step_consts + a * s.sc_ld, s.T);
        if (threadIdx.x == 0) {
            const bool keep = !first || first[a] == (unsigned long long)i;
            dd.key[i] = keep ? s.key[a] : bank_key(seed, counter + (uint64_t)i);
        }
    }
}

__global__ void k_bank_keys(uint64_t *key, int64_t n, uint64_t seed, uint64_t counter) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        key[i] = bank_key(seed, counter + (uint64_t)i);
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
template <class M, int FK, int SCHEME, bool RES>
static int bank_kernel_setup(smcb_ctx *c, int64_t nrun, size_t smem, int &grid) {
    auto kern = k_bank<M, FK, SCHEME, RES>;
    SMCB_TRY(set_smem(kern, smem));
    int nb = 0, sms = 0;
    SMCB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kern, kBatchBS, smem));
    SMCB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->device));
    if (nb < 1) {
        set_error("filter bank: the kernel does not fit on an SM of this device");
        return SMCB_ECUDA;
    }
    const int64_t g = (int64_t)nb * sms;
    grid = (int)(nrun < g ? (nrun > 0 ? nrun : 1) : g);
    return SMCB_OK;
}

// plan (out != NULL) or launch
template <class M, int FK, int SCHEME>
static int bank_one(smcb_ctx *c, const smcb_bank_desc &d, int64_t *out) {
    int optin = 0;
    SMCB_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, c->device));
    cudaFuncAttributes fa;
    SMCB_CUDA(cudaFuncGetAttributes(&fa, k_bank<M, FK, SCHEME, true>));
    const size_t smem_res = kMathTabBytes + (size_t)resident_doubles(d.N, SCHEME) * sizeof(double);
    const bool fits = smem_res + fa.sharedSizeBytes <= (size_t)optin;
    const int tier = d.tier == SMCB_BATCH_AUTO ? (fits ? SMCB_BATCH_RESIDENT : SMCB_BATCH_STREAMING) : d.tier;
    if (tier == SMCB_BATCH_RESIDENT && !fits) {
        set_error("filter bank: N=%lld does not fit the resident tier", (long long)d.N);
        return SMCB_EINVAL;
    }
    const int64_t nrun = d.idx ? d.n_idx : d.R;
    int grid = 0, rc;
    if (tier == SMCB_BATCH_RESIDENT) rc = bank_kernel_setup<M, FK, SCHEME, true>(c, nrun, smem_res, grid);
    else rc = bank_kernel_setup<M, FK, SCHEME, false>(c, nrun, kMathTabBytes, grid);
    if (rc != SMCB_OK) return rc;
    if (out) {
        out[0] = tier;
        out[1] = grid;
        return SMCB_OK;
    }
    if (nrun == 0) return SMCB_OK;
    SMCB_REQUIRE(tier == SMCB_BATCH_RESIDENT || (d.cdf && (SCHEME != SMCB_RS_MULTINOMIAL || d.scratch)),
                 "smcb_bank_advance: the streaming tier needs cdf (and scratch for multinomial)");
    SMCB_REQUIRE(tier == SMCB_BATCH_RESIDENT || d.scratch_rows >= grid,
                 "smcb_bank_advance: the streaming tier needs %d scratch rows (got %lld)", grid,
                 (long long)d.scratch_rows);
    if (tier == SMCB_BATCH_RESIDENT)
        return launch(c, k_bank<M, FK, SCHEME, true>, grid, kBatchBS, smem_res, d, c->math_tab);
    return launch(c, k_bank<M, FK, SCHEME, false>, grid, kBatchBS, kMathTabBytes, d, c->math_tab);
}

static int bank_dispatch(smcb_ctx *c, const smcb_bank_desc *dp, int64_t *out) {
    SMCB_REQUIRE(c && dp, "smcb_bank: NULL argument");
    const smcb_bank_desc &d = *dp;
    SMCB_REQUIRE(d.N >= 1 && d.T >= 1 && d.R >= 0, "smcb_bank: bad shape N=%lld T=%lld R=%lld", (long long)d.N,
                 (long long)d.T, (long long)d.R);
    SMCB_REQUIRE(d.n_params >= 0 && d.n_params <= SMCB_MAX_PARAMS, "smcb_bank: bad n_params %d", d.n_params);
    SMCB_REQUIRE(d.tier >= SMCB_BATCH_AUTO && d.tier <= SMCB_BATCH_STREAMING, "smcb_bank: bad tier %d", d.tier);
    SMCB_REQUIRE(!d.idx || (d.n_idx >= 0 && d.n_idx <= d.R), "smcb_bank: bad n_idx %lld", (long long)d.n_idx);
    if (!out) {
        SMCB_REQUIRE(d.t1 >= 1 && d.t1 <= d.T, "smcb_bank_advance: t1=%lld outside [1, T=%lld]", (long long)d.t1,
                     (long long)d.T);
        SMCB_REQUIRE(d.key && d.params && d.data && d.X && d.lw && d.state, "smcb_bank_advance: NULL buffer");
        SMCB_REQUIRE(!d.step_consts || d.sc_ld == 0 || d.sc_ld >= d.T, "smcb_bank_advance: bad sc_ld");
    }
    bool built = false;
    const int rc = with_model(d.model, 1, [&](auto m) {
        using M = decltype(m);
        if constexpr (M::D == 1) {
            return with_fk<M>(d.fk, [&](auto fk) {
                return with_scheme(d.scheme, [&](auto scheme) {
                    built = true;
                    return bank_one<M, decltype(fk)::value, decltype(scheme)::value>(c, d, out);
                });
            });
        } else {
            return SMCB_ENOSYS;
        }
    });
    if (!built) {
        set_error("filter bank: model %d, Feynman-Kac kind %d, scheme %d is not built", d.model, d.fk, d.scheme);
        return SMCB_ENOSYS;
    }
    return rc;
}

static int rows_check(const smcb_bank_desc *s, const smcb_bank_desc *d, const char *who) {
    SMCB_REQUIRE(s && d, "%s: NULL argument", who);
    SMCB_REQUIRE(s->N == d->N && s->T == d->T && s->n_params == d->n_params && s->sc_ld == d->sc_ld,
                 "%s: the two banks differ in N, T, n_params or step-constant rows", who);
    SMCB_REQUIRE(s->X && s->lw && s->state && s->params && s->key && d->X && d->lw && d->state && d->params &&
                     d->key && (d->sc_ld == 0 || (s->step_consts && d->step_consts)),
                 "%s: NULL buffer", who);
    return SMCB_OK;
}

static int rows_grid(int64_t m) { return (int)(m < 65535 ? m : 65535); }

}  // namespace smcb

using namespace smcb;

extern "C" int smcb_bank_plan(smcb_ctx *c, const smcb_bank_desc *d, int64_t out[2]) {
    SMCB_REQUIRE(out, "smcb_bank_plan: NULL out");
    return bank_dispatch(c, d, out);
}

extern "C" int smcb_bank_advance(smcb_ctx *c, const smcb_bank_desc *d) { return bank_dispatch(c, d, nullptr); }

extern "C" int smcb_bank_gather(smcb_ctx *c, const smcb_bank_desc *src, const int64_t *A, int64_t m,
                                const smcb_bank_desc *dst, uint64_t seed, uint64_t counter, uint64_t *first) {
    SMCB_REQUIRE(c && A && first, "smcb_bank_gather: NULL argument");
    const int rc = rows_check(src, dst, "smcb_bank_gather");
    if (rc != SMCB_OK) return rc;
    SMCB_REQUIRE(m >= 0 && dst->R >= m, "smcb_bank_gather: the destination holds %lld < %lld rows",
                 (long long)dst->R, (long long)m);
    if (m == 0 || src->R == 0) return SMCB_OK;
    auto *f = reinterpret_cast<unsigned long long *>(first);
    SMCB_TRY(launch(c, k_first_fill, grid_for(src->R, 256), 256, 0, f, src->R));
    SMCB_TRY(launch(c, k_first_min, grid_for(m, 256), 256, 0, A, m, f));
    return launch(c, k_bank_rows, rows_grid(m), kRowBS, 0, *src, *dst, A, nullptr, f, seed, counter, m);
}

extern "C" int smcb_bank_merge(smcb_ctx *c, const smcb_bank_desc *dst, const smcb_bank_desc *src,
                               const uint8_t *accepted) {
    SMCB_REQUIRE(c && accepted, "smcb_bank_merge: NULL argument");
    const int rc = rows_check(src, dst, "smcb_bank_merge");
    if (rc != SMCB_OK) return rc;
    SMCB_REQUIRE(src->R == dst->R, "smcb_bank_merge: %lld proposals for %lld slots", (long long)src->R,
                 (long long)dst->R);
    if (dst->R == 0) return SMCB_OK;
    return launch(c, k_bank_rows, rows_grid(dst->R), kRowBS, 0, *src, *dst, nullptr, accepted, nullptr, 0, 0, dst->R);
}

extern "C" int smcb_bank_keys(smcb_ctx *c, uint64_t *key, int64_t n, uint64_t seed, uint64_t counter) {
    SMCB_REQUIRE(c && key && n >= 0, "smcb_bank_keys: bad argument");
    if (n == 0) return SMCB_OK;
    return launch(c, k_bank_keys, grid_for(n, 256), 256, 0, key, n, seed, counter);
}
