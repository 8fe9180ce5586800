// smcb_smooth.cu -- off-line smoothing on the device: FFBS backward sampling over a stored particle history
// (particles/smoothing.py:278-423).  Trajectories are independent of each other, so each method is ONE kernel
// launch that loops over t = T-2 ... 0 inside, with no grid-wide synchronisation:
//   ON2     one CTA owns 256 trajectories; per t it walks tiles of (loc(X_t[n]), lw_t[n]) staged in shared memory
//           (the transition location computed ONCE per particle and shared by the CTA's trajectories), pass 1 an
//           online (max, sum exp) per trajectory, pass 2 the re-walk to the crossing of u * S with early exit;
//   MCMC    one thread per trajectory: chain started at the genealogy, nsteps independent Metropolis steps with
//           multinomial proposals from W_t (inverse CDF on the caller's per-t CDF);
//   REJECT  one thread per trajectory, lanes in lockstep over t: at most max_trials proposals, then a
//           warp-cooperative exact O(N) draw for every lane still rejected.
// Randomness: Philox keyed by (context seed, API call, trajectory m, time t, trial, purpose): results depend on the
// seed only, never on the launch geometry.
#include "smcb_dispatch.cuh"
#include "smcb_smooth.cuh"

using namespace smcb;

namespace {

template <int D>
__device__ __forceinline__ void put_path(const smcb_smooth_desc &d, int64_t t, int64_t j, int64_t n, const double *x) {
    d.idx[t * d.M + j] = n;
    double *o = d.paths + (t * d.M + j) * D;
#pragma unroll
    for (int c = 0; c < D; c++) o[c] = x[c];
}

__device__ __forceinline__ StepK step_at(const smcb_smooth_desc &d, int64_t t) {
    StepK k{};
    k.t = t;
    k.sc0 = d.step_consts ? d.step_consts[t] : 0.0;
    return k;
}

// ---------------------------------------------------------------------------
// ON2 -- smoothing.py:291-311
// ---------------------------------------------------------------------------
template <class M>
__global__ void __launch_bounds__(kSmBlock) k_bs_on2(M m, smcb_smooth_desc d, Philox key, uint64_t call,
                                                    const double *tab) {
    constexpr int D = M::D;
    __shared__ __align__(8) uint64_t s_bar;
    stage_tables<M>(tab, &s_bar, true);
    double *s_loc = const_cast<double *>(mtab()) + kMathTabDoubles;   // (D, kSmBlock) locations of the tile
    double *s_lw = s_loc + D * kSmBlock;                               // (kSmBlock) log-weights of the tile
    const int64_t j = (int64_t)blockIdx.x * kSmBlock + threadIdx.x;
    const bool live = j < d.M;
    const int64_t N = d.N, T = d.T;
    TransDensity<M> td;
    td.init(m);
    double xn[D];
    int64_t nxt = live ? d.idx_T[j] : 0;
    if (live) {
        load_x<D>(d, T - 1, nxt, xn);
        put_path<D>(d, T - 1, j, nxt, xn);
    }
    for (int64_t t = T - 2; t >= 0; t--) {
        const StepK k = step_at(d, t + 1);
        const double *lw = d.lw[t];
        auto fill = [&](int64_t base) {
            __syncthreads();                               // the previous tile is consumed
            const int64_t n = base + threadIdx.x;
            if (n < N) {
                double xp[D], lc[D];
                load_x<D>(d, t, n, xp);
                td.loc(m, k, xp, lc);
#pragma unroll
                for (int c = 0; c < D; c++) s_loc[c * kSmBlock + threadIdx.x] = lc[c];
                s_lw[threadIdx.x] = lw[n];
            }
            __syncthreads();
        };
        auto value = [&](int i) {
            double lc[D];
#pragma unroll
            for (int c = 0; c < D; c++) lc[c] = s_loc[c * kSmBlock + i];
            return s_lw[i] + td.lpdf(m, lc, xn);
        };
        // pass 1: log-sum-exp of lw_t + logpt(t + 1, X_t, xn), in index order
        double mx = -CUDART_INF, s = 0.0;
        for (int64_t base = 0; base < N; base += kSmBlock) {
            fill(base);
            const int cnt = (int)min((int64_t)kSmBlock, N - base);
            if (live)
                for (int i = 0; i < cnt; i++) lse_add<true>(mx, s, value(i));
        }
        // pass 2: first n with sum_{i <= n} exp(v_i - mx) >= u * S
        double u = 0.5, tmp;
        if (live) {
            if (d.u) u = d.u[j * (T - 1) + t];
            else smooth_uniforms(key, call, j, t, 0, kPurposeSmoothExact, u, tmp);
        }
        const double target = u * s;
        double cacc = 0.0;
        int64_t found = -1, last = -1;
        for (int64_t base = 0; base < N; base += kSmBlock) {
            fill(base);
            const int cnt = (int)min((int64_t)kSmBlock, N - base);
            if (live && found < 0) {
                for (int i = 0; i < cnt; i++) {
                    const double v = value(i);
                    const double e = (v > -CUDART_INF) ? texp_neg(v - mx) : 0.0;
                    cacc += e;
                    if (e > 0.0) last = base + i;
                    if (cacc >= target && e > 0.0) { found = base + i; break; }
                }
            }
            if (__syncthreads_and(!live || found >= 0)) break;
        }
        if (live) {
            if (found < 0) found = last >= 0 ? last : N - 1;   // round-off: clip to the last positive weight
            nxt = found;
            load_x<D>(d, t, nxt, xn);
            put_path<D>(d, t, j, nxt, xn);
        }
    }
}

// ---------------------------------------------------------------------------
// MCMC -- smoothing.py:313-350
// ---------------------------------------------------------------------------
template <class M>
__global__ void __launch_bounds__(kSmBlock) k_bs_mcmc(M m, smcb_smooth_desc d, Philox key, uint64_t call,
                                                     const double *tab) {
    constexpr int D = M::D;
    __shared__ __align__(8) uint64_t s_bar;
    stage_tables<M>(tab, &s_bar, TransUsesTable<M>::value);
    const int64_t j = (int64_t)blockIdx.x * kSmBlock + threadIdx.x;
    if (j >= d.M) return;
    const int64_t N = d.N, T = d.T, Mt = d.M;
    TransDensity<M> td;
    td.init(m);
    double xn[D], xp[D], lc[D];
    int64_t nxt = d.idx_T[j];
    load_x<D>(d, T - 1, nxt, xn);
    put_path<D>(d, T - 1, j, nxt, xn);
    for (int64_t t = T - 2; t >= 0; t--) {
        const StepK k = step_at(d, t + 1);
        int64_t cur = d.A[t + 1][nxt];                       // the genealogy, smoothing.py:342
        load_x<D>(d, t, cur, xp);
        td.loc(m, k, xp, lc);
        double lcur = td.lpdf(m, lc, xn);
        for (int64_t i = 0; i < d.nsteps; i++) {
            int64_t prop;
            double lu;
            if (d.prop) {
                const int64_t off = (t * d.nsteps + i) * Mt + j;
                prop = d.prop[off];
                lu = d.lu[off];
            } else {
                double u0, u1;
                smooth_uniforms(key, call, j, t, (uint32_t)i, kPurposeSmooth, u0, u1);
                prop = draw_cdf(d.cdf + t * d.cdf_ld, N, u0);
                lu = log(u1);
            }
            load_x<D>(d, t, prop, xp);
            td.loc(m, k, xp, lc);
            const double lprop = td.lpdf(m, lc, xn);
            if (lu < lprop - lcur) {                         // smoothing.py:346-349
                cur = prop;
                lcur = lprop;
            }
        }
        nxt = cur;
        load_x<D>(d, t, nxt, xn);
        put_path<D>(d, t, j, nxt, xn);
    }
}

// ---------------------------------------------------------------------------
// REJECT (hybrid) -- smoothing.py:352-423
// ---------------------------------------------------------------------------
template <class M>
__global__ void __launch_bounds__(kSmBlock) k_bs_reject(M m, smcb_smooth_desc d, Philox key, uint64_t call,
                                                       const double *tab) {
    constexpr int D = M::D;
    __shared__ __align__(8) uint64_t s_bar;
    stage_tables<M>(tab, &s_bar, TransUsesTable<M>::value);
    const int lane = threadIdx.x & 31;
    const int64_t j = (int64_t)blockIdx.x * kSmBlock + threadIdx.x;
    const bool live = j < d.M;
    if (__all_sync(kFull, !live)) return;                   // whole warp past M; partial warps stay for the fallback
    const int64_t T = d.T, Mt = d.M, mt = d.max_trials;
    TransDensity<M> td;
    td.init(m);
    double xn[D];
    int64_t nxt = live ? d.idx_T[j] : 0;
    if (live) {
        load_x<D>(d, T - 1, nxt, xn);
        put_path<D>(d, T - 1, j, nxt, xn);
    } else {
#pragma unroll
        for (int c = 0; c < D; c++) xn[c] = 0.0;
    }
    for (int64_t t = T - 2; t >= 0; t--) {
        const StepK k = step_at(d, t + 1);
        const double bound = d.log_bound[t];
        bool acc = !live;
        int64_t choice = 0, nprop = 0;
        // the first trials: every lane its own trajectory
        const int64_t solo = mt < kSoloTrials ? mt : kSoloTrials;
        for (int64_t trial = 0; trial < solo; trial++) {
            if (__all_sync(kFull, acc)) break;
            if (!acc) {
                int64_t prop;
                nprop++;
                if (reject_trial<M>(m, td, d, k, key, call, j, t, trial, xn, bound, prop)) {
                    acc = true;
                    choice = prop;
                }
            }
        }
        // the stragglers, one at a time by the whole warp: lane l runs trial base + l, the first accepted trial in
        // trial order wins -- the same trajectory, proposal and count as running the trials one after another
        unsigned slow = __ballot_sync(kFull, live && !acc && mt > solo);
        while (slow) {
            const int src = __ffs(slow) - 1;
            slow &= slow - 1;
            double xs[D];
#pragma unroll
            for (int c = 0; c < D; c++) xs[c] = __shfl_sync(kFull, xn[c], src);
            const int64_t js = j - lane + src;
            int64_t hit_trial = -1, hit_prop = 0;
            for (int64_t base = solo; base < mt && hit_trial < 0; base += 32) {
                const int64_t trial = base + lane;
                int64_t prop = 0;
                const bool ok = trial < mt && reject_trial<M>(m, td, d, k, key, call, js, t, trial, xs, bound, prop);
                const unsigned b = __ballot_sync(kFull, ok);
                if (b) {
                    const int f = __ffs(b) - 1;
                    hit_trial = base + f;
                    hit_prop = __shfl_sync(kFull, prop, f);
                }
            }
            if (lane == src) {
                nprop = hit_trial >= 0 ? hit_trial + 1 : mt;
                if (hit_trial >= 0) {
                    acc = true;
                    choice = hit_prop;
                }
            }
        }
        // acceptance statistics: integer sums, one atomic pair per warp (order-independent -> deterministic)
        const long long na = warp_sum((live && acc) ? 1 : 0), np = warp_sum(nprop);
        if (lane == 0) {
            atomicAdd(reinterpret_cast<unsigned long long *>(d.counts + 2 * t), (unsigned long long)na);
            atomicAdd(reinterpret_cast<unsigned long long *>(d.counts + 2 * t + 1), (unsigned long long)np);
        }
        // the exact fallback (smoothing.py:416-421), served by the whole warp, one rejected lane at a time
        unsigned need = __ballot_sync(kFull, live && !acc);
        while (need) {
            const int src = __ffs(need) - 1;
            need &= need - 1;
            double xs[D];
#pragma unroll
            for (int c = 0; c < D; c++) xs[c] = __shfl_sync(kFull, xn[c], src);
            const int64_t js = j - lane + src;
            double u, tmp;
            if (d.u_exact) u = d.u_exact[t * Mt + js];
            else smooth_uniforms(key, call, js, t, 0, kPurposeSmoothExact, u, tmp);
            const int64_t r = warp_exact_draw<M>(m, td, d, k, t, xs, u, lane);
            if (lane == src) choice = r;
        }
        if (live) {
            nxt = choice;
            load_x<D>(d, t, nxt, xn);
            put_path<D>(d, t, j, nxt, xn);
        }
    }
}

// ---------------------------------------------------------------------------
// paths[t][m] = X[t][idx[t][m]] for indices computed elsewhere (the plugin path)
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlock) k_bs_gather(smcb_smooth_desc d) {
    const int64_t total = d.T * d.M * d.dim;
    const int64_t stride = (int64_t)gridDim.x * kBlock;
    for (int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x; i < total; i += stride) {
        const int64_t c = i % d.dim, tm = i / d.dim, t = tm / d.M;
        d.paths[i] = d.X[t][d.idx[tm] * d.x_stride_n + c * d.x_stride_c];
    }
}

template <class M>
int run_model(smcb_ctx *c, const smcb_smooth_desc &d) {
    SMCB_REQUIRE(d.dim == M::D, "smcb_backward_sample: dim %d does not match the model's %d", (int)d.dim, M::D);
    M m;
    m.load(d.params);
    const Philox key = key_of(c->seed);
    const uint64_t call = c->api_counter++;
    const int grid = (int)((d.M + kSmBlock - 1) / kSmBlock);
    const size_t tab = TransUsesTable<M>::value ? kMathTabBytes : 0;
    int rc;
    if (d.method == SMCB_SMOOTH_ON2) {
        const size_t smem = kMathTabBytes + (size_t)(M::D + 1) * kSmBlock * sizeof(double);
        if ((rc = set_smem(k_bs_on2<M>, smem)) != SMCB_OK) return rc;
        k_bs_on2<M><<<grid, kSmBlock, smem, c->stream>>>(m, d, key, call, c->math_tab);
    } else if (d.method == SMCB_SMOOTH_MCMC) {
        if ((rc = set_smem(k_bs_mcmc<M>, tab)) != SMCB_OK) return rc;
        k_bs_mcmc<M><<<grid, kSmBlock, tab, c->stream>>>(m, d, key, call, c->math_tab);
    } else {
        if ((rc = set_smem(k_bs_reject<M>, tab)) != SMCB_OK) return rc;
        SMCB_CUDA(cudaMemsetAsync(d.counts, 0, (size_t)(d.T - 1) * 2 * sizeof(int64_t), c->stream));
        k_bs_reject<M><<<grid, kSmBlock, tab, c->stream>>>(m, d, key, call, c->math_tab);
    }
    c->launches++;
    SMCB_CUDA(cudaGetLastError());
    return SMCB_OK;
}

}  // namespace

extern "C" int smcb_backward_sample(smcb_ctx *c, const smcb_smooth_desc *dp) {
    SMCB_REQUIRE(c && dp, "smcb_backward_sample: NULL argument");
    const smcb_smooth_desc &d = *dp;
    SMCB_REQUIRE(d.T >= 1 && d.N >= 1 && d.M >= 1 && d.M <= 0xffffffffLL && d.T <= 0xffffffffLL,
                 "smcb_backward_sample: bad sizes T=%lld N=%lld M=%lld", (long long)d.T, (long long)d.N,
                 (long long)d.M);
    SMCB_REQUIRE(d.X && d.idx && d.paths && d.dim >= 1, "smcb_backward_sample: NULL history or output");
    if (d.method == SMCB_SMOOTH_GATHER) {
        k_bs_gather<<<grid_for(d.T * d.M * d.dim, kBlock * 4), kBlock, 0, c->stream>>>(d);
        c->launches++;
        SMCB_CUDA(cudaGetLastError());
        return SMCB_OK;
    }
    SMCB_REQUIRE(d.method >= SMCB_SMOOTH_ON2 && d.method <= SMCB_SMOOTH_REJECT, "smcb_backward_sample: bad method %d",
                 (int)d.method);
    SMCB_REQUIRE(d.lw && d.idx_T, "smcb_backward_sample: NULL log-weights or final indices");
    if (d.method == SMCB_SMOOTH_MCMC) {
        SMCB_REQUIRE(d.nsteps >= 0 && d.nsteps < (1 << 24), "smcb_backward_sample: nsteps out of range");
        SMCB_REQUIRE(d.T == 1 || d.A, "smcb_backward_sample: MCMC needs the ancestors");
        SMCB_REQUIRE(d.T == 1 || d.nsteps == 0 || d.prop || (d.cdf && d.cdf_ld >= d.N),
                     "smcb_backward_sample: MCMC needs the CDFs");
        SMCB_REQUIRE((d.prop == nullptr) == (d.lu == nullptr), "smcb_backward_sample: prop and lu go together");
    }
    if (d.method == SMCB_SMOOTH_REJECT) {
        SMCB_REQUIRE(d.max_trials >= 0 && d.max_trials < (1 << 24), "smcb_backward_sample: max_trials out of range");
        SMCB_REQUIRE(d.T == 1 || (d.log_bound && d.counts), "smcb_backward_sample: reject needs the bounds and counts");
        SMCB_REQUIRE(d.T == 1 || d.max_trials == 0 || d.prop || (d.cdf && d.cdf_ld >= d.N),
                     "smcb_backward_sample: reject needs the CDFs");
        SMCB_REQUIRE((d.prop == nullptr) == (d.lu == nullptr), "smcb_backward_sample: prop and lu go together");
    }
    bool known = false;
    const int rc = with_model(d.model, d.dim, [&](auto m) {
        known = true;
        return run_model<decltype(m)>(c, d);
    });
    if (!known) set_error("smcb_backward_sample: no transition density for model %d, dim %d", (int)d.model, (int)d.dim);
    return rc;
}
