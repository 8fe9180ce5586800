// smcb_sqmc.cu -- sequential quasi-Monte Carlo (particles/core.py:315-349): device Sobol' points (rqmc.sobol), the
// Hilbert sort (hilbert.hilbert_sort) and the SQMC step of the fused stock models, which always resamples:
//   t = 0:  u = sobol(N, du),      X = Gamma0(u)                          (fk_init / model_init, z = Phi^-1(u))
//   t >= 1: u = sobol(N, du + 1),  tau = argsort(u[:, 0]),  h = hilbert_sort(X),
//           A = h[inverse_cdf(u[tau, 0], aux.W[h])],  X = Gamma(t, X[A], u[tau, 1:])   (fk_move / model_move)
// The argsort of u[:, 0] sorts the 30-bit integers (the squeeze is monotone); both sorts are CUB radix sorts.  The
// CDF and its search are the library's scan and search (smcb_cumsum, smcb_searchsorted); the weights and the
// summary row come from smcb_normalise.  Nothing here synchronises with the host.
#include <cub/device/device_radix_sort.cuh>

#include "smcb_dispatch.cuh"
#include "smcb_sqmc.cuh"
#include "smcb_step.cuh"

using namespace smcb;
using namespace smcb::sqmc;

namespace {

constexpr int kThreads = 256;
constexpr int kColBlocks = 128;   // most CTAs per column of the Hilbert standardisation (col_stats)

// ------------------------------------------------------------------------------------------------------------- Sobol
constexpr int kSobolSlab = 32;    // dimensions per CTA row of the grid (blockIdx.y)

// every CTA builds the scrambled direction numbers of its slab of up to kSobolSlab dimensions in shared memory, then
// writes their points; dimension j's numbers are keyed by j alone, so its points do not depend on d or on the slab
__global__ void k_sobol(int d, int64_t n, int scramble, Philox key, uint64_t call, double *u, int32_t *raw) {
    __shared__ uint32_t words[kSobolSlab][32];
    __shared__ uint32_t sv[kSobolSlab][kSobolBits];
    __shared__ uint32_t shift[kSobolSlab];
    auto gen = [&](uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t r[4]) {
        philox4x32_10(c0, c1, c2, c3, key.k0, key.k1, r);
    };
    const int j0 = blockIdx.y * kSobolSlab, dj = min(kSobolSlab, d - j0);
    for (int j = threadIdx.x; j < dj; j += blockDim.x) {
        sobol_scramble_words(gen, j0 + j, call, words[j]);
        uint32_t v[kSobolBits], s;
        sobol_dims(j0 + j, scramble, words[j], v, s);
        for (int k = 0; k < kSobolBits; k++) sv[j][k] = v[k];
        shift[j] = s;
    }
    __syncthreads();
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        for (int j = 0; j < dj; j++) {
            const uint32_t q = sobol_int(sv[j], shift[j], (uint64_t)i);
            if (raw) raw[(j0 + j) * n + i] = (int32_t)q;
            if (u) u[(j0 + j) * n + i] = squeeze(q);
        }
    }
}

int sobol(smcb_ctx *c, int d, int64_t n, int scramble, uint64_t seed, uint64_t call, double *u, int32_t *raw) {
    const dim3 grid(grid_for(n, kThreads), (d + kSobolSlab - 1) / kSobolSlab);
    return launch(c, k_sobol, grid, kThreads, 0, d, n, scramble, key_of(seed), call, u, raw);
}

// ----------------------------------------------------------------------------------------------------------- Hilbert
// scratch of one Hilbert sort of n points of dimension d (256-byte aligned sections)
struct HilbertWs {
    int64_t *iota, *keys, *keys_out;
    double *stats;        // mean[d], std[d]
    double *partials;     // per column, one partial sum per CTA of col_stats
    void *cub;
    size_t cub_bytes;
};

inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

size_t hilbert_cub_bytes(int64_t n) {
    size_t a = 0, b = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, a, (const int64_t *)nullptr, (int64_t *)nullptr,
                                    (const int64_t *)nullptr, (int64_t *)nullptr, (int)n);
    cub::DeviceRadixSort::SortPairs(nullptr, b, (const double *)nullptr, (double *)nullptr,
                                    (const int64_t *)nullptr, (int64_t *)nullptr, (int)n);
    return a > b ? a : b;
}

size_t hilbert_ws_bytes(int64_t n, int d) {
    return 3 * align256(8 * (size_t)n) + align256(16 * (size_t)d) + align256(8 * (size_t)d * kColBlocks) +
           align256(hilbert_cub_bytes(n));
}

HilbertWs hilbert_ws(char *p, int64_t n, int d) {
    HilbertWs w;
    const size_t s = align256(8 * (size_t)n);
    w.iota = (int64_t *)p; w.keys = (int64_t *)(p + s); w.keys_out = (int64_t *)(p + 2 * s);
    w.stats = (double *)(p + 3 * s);
    w.partials = (double *)(p + 3 * s + align256(16 * (size_t)d));
    w.cub = p + 3 * s + align256(16 * (size_t)d) + align256(8 * (size_t)d * kColBlocks);
    w.cub_bytes = align256(hilbert_cub_bytes(n));
    return w;
}

__global__ void k_iota(int64_t *v, int64_t n) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        v[i] = i;
}

// np.mean and np.std (ddof = 0) of every column of the SoA (d, n) points, in two passes (sum, then the sum of squared
// deviations), each a grid of (kColBlocks or fewer) x d CTAs writing one partial per CTA and one CTA per column adding
// them in a fixed order: the whole device works on every column and the result does not depend on timing.
inline int col_blocks(int64_t n) {
    const int64_t b = (n + 8 * kThreads - 1) / (8 * kThreads);
    return (int)(b < 1 ? 1 : (b > kColBlocks ? kColBlocks : b));
}

template <int PASS>
__global__ void k_col_partial(const double *x, int64_t n, const double *stats, double *partials) {
    const int j = blockIdx.y, nb = gridDim.x;
    const double *col = x + j * n;
    const double m = PASS == 1 ? stats[j] : 0.0;
    __shared__ double red[kThreads / 32];
    double s = 0.0;
    for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)nb * kThreads) {
        const double v = col[i];
        if (PASS == 0) s += v;
        else s += (v - m) * (v - m);
    }
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < kThreads / 32; w++) t += red[w];
        partials[j * nb + blockIdx.x] = t;
    }
}

// PASS 0: stats[j] = mean; PASS 1: stats[d + j] = std
template <int PASS>
__global__ void k_col_finish(const double *partials, int nb, int64_t n, int d, double *stats) {
    const int j = blockIdx.x;
    if (threadIdx.x != 0) return;
    double t = 0.0;
    for (int b = 0; b < nb; b++) t += partials[j * nb + b];
    if (PASS == 0) stats[j] = t / (double)n;
    else stats[d + j] = sqrt(t / (double)n);
}

int col_stats(smcb_ctx *c, const double *x, int64_t n, int d, double *stats, double *partials) {
    const int nb = col_blocks(n);
    SMCB_TRY(launch(c, k_col_partial<0>, dim3(nb, d), kThreads, 0, x, n, (const double *)stats, partials));
    SMCB_TRY(launch(c, k_col_finish<0>, d, 32, 0, (const double *)partials, nb, n, d, stats));
    SMCB_TRY(launch(c, k_col_partial<1>, dim3(nb, d), kThreads, 0, x, n, (const double *)stats, partials));
    return launch(c, k_col_finish<1>, d, 32, 0, (const double *)partials, nb, n, d, stats);
}

// key of point i: Hilbert_to_int(floor(invlogit((x - mean) / std) * maxint))
__global__ void k_hilbert_keys(const double *x, int64_t n, int d, const double *stats, double maxint, int64_t *keys) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t c[kHilbertMaxDim];
        for (int j = 0; j < d; j++) {
            const double xs = 1.0 / (1.0 + exp(-((x[j * n + i] - stats[j]) / stats[d + j])));
            c[j] = (int64_t)floor(xs * maxint);
        }
        keys[i] = hilbert_key(c, d);
    }
}

// order = hilbert_sort(x) for SoA (d, n) points; keys_out (NULL: not written) = the unsorted int64 keys (d > 1)
int hilbert_order(smcb_ctx *c, const double *x, int64_t n, int d, int64_t *order, int64_t *keys_out, char *scratch) {
    HilbertWs w = hilbert_ws(scratch, n, d);
    SMCB_TRY(launch(c, k_iota, grid_for(n, kThreads), kThreads, 0, w.iota, n));
    size_t cb = w.cub_bytes;
    if (d == 1) {      // np.argsort(x)
        SMCB_CUDA(cub::DeviceRadixSort::SortPairs(w.cub, cb, x, (double *)w.keys_out, w.iota, order, (int)n, 0, 64,
                                                  c->stream));
        return SMCB_OK;
    }
    int64_t *keys = keys_out ? keys_out : w.keys;
    SMCB_TRY(col_stats(c, x, n, d, w.stats, w.partials));
    const double maxint = floor(pow(2.0, 62.0 / d));
    SMCB_TRY(launch(c, k_hilbert_keys, grid_for(n, kThreads), kThreads, 0, x, n, d, w.stats, maxint, keys));
    SMCB_CUDA(cub::DeviceRadixSort::SortPairs(w.cub, cb, keys, w.keys_out, w.iota, order, (int)n, 0, 64, c->stream));
    return SMCB_OK;
}

// -------------------------------------------------------------------------------------------------------- SQMC step
// scratch of smcb_sqmc_step: the points (du + 1 rows), their integers, tau, the Hilbert order and its scratch, the
// aux weights in Hilbert order, the sorted first coordinate, the searched indices, logeta, W_{t-1} and statistics
struct SqmcWs {
    double *u;
    int32_t *raw;
    uint32_t *raw0s;
    int64_t *iota, *tau, *h, *idx;
    double *la, *wh, *su, *le, *wprev, *stats;    // stats: [0, 4) aux, [4, 8) W_{t-1}, [8, 12) step, 12 log-mean
    char *hws;
    void *cub;
    size_t cub_bytes;
};

size_t sqmc_cub_bytes(int64_t n) {
    size_t a = 0, b = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, a, (const uint32_t *)nullptr, (uint32_t *)nullptr,
                                    (const int64_t *)nullptr, (int64_t *)nullptr, (int)n);
    cub::DeviceRadixSort::SortPairs(nullptr, b, (const double *)nullptr, (double *)nullptr,
                                    (const int64_t *)nullptr, (int64_t *)nullptr, (int)n);
    return a > b ? a : b;
}

size_t sqmc_ws_layout(int64_t n, int du, char *p, SqmcWs *w) {
    const size_t s8 = align256(8 * (size_t)n), s4 = align256(4 * (size_t)n);
    size_t o = 0;
    auto take = [&](size_t b) { char *q = p ? p + o : nullptr; o += b; return q; };
    char *u = take(align256(8 * (size_t)n * (du + 1)));
    char *raw = take(align256(4 * (size_t)n * (du + 1)));
    char *raw0s = take(s4);
    char *iota = take(s8), *tau = take(s8), *h = take(s8), *idx = take(s8);
    char *la = take(s8), *wh = take(s8), *su = take(s8), *le = take(s8), *wprev = take(s8);
    char *stats = take(256);
    char *hws = take(align256(hilbert_ws_bytes(n, du)));
    const size_t cb = align256(sqmc_cub_bytes(n));
    char *cub = take(cb);
    if (w) {
        w->u = (double *)u; w->raw = (int32_t *)raw; w->raw0s = (uint32_t *)raw0s;
        w->iota = (int64_t *)iota; w->tau = (int64_t *)tau; w->h = (int64_t *)h; w->idx = (int64_t *)idx;
        w->la = (double *)la; w->wh = (double *)wh; w->su = (double *)su; w->le = (double *)le;
        w->wprev = (double *)wprev; w->stats = (double *)stats; w->hws = hws; w->cub = cub; w->cub_bytes = cb;
    }
    return o;
}

// X = Gamma0(u), lw = logG(0, X): z_j = Phi^-1(u_j) for the first NZ coordinates (BearingsOnly's Dirac coordinates
// take no normal).  The per-step data come from the filter's own FilterArgs (step_consts of smcb_step.cuh).
template <class M, int FK>
__global__ void k_sqmc_init(const double *tab, const M m, const FilterArgs a, const double *u, int64_t n, double *X,
                            double *lw) {
    __shared__ __align__(8) uint64_t s_bar;
    stage_math_tables(tab, &s_bar);          // the models' table-assisted exp (mexp) reads them
    const StepK k = step_consts(a, 0);
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        double z[M::D], x[M::D], d;
        for (int j = 0; j < M::NZ; j++) z[j] = ndtri(u[j * n + i]);
        model_init<M, FK>(m, k, z, x, d);
        for (int j = 0; j < M::D; j++) X[j * n + i] = x[j];
        lw[i] = d;
    }
}

// la[i] = aux log-weight of particle h[i] (lw + logeta for the APF kinds); le[h[i]] = its logeta
template <class M, int FK>
__global__ void k_sqmc_aux(const double *tab, const M m, const FilterArgs a, int64_t t, const double *X,
                           const double *lw, const int64_t *h, int64_t n, double *la, double *le) {
    __shared__ __align__(8) uint64_t s_bar;
    stage_math_tables(tab, &s_bar);
    const StepK k = step_consts(a, t - 1);
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t p = h[i];
        double v = lw[p];
        if (FkTraits<FK>::apf) {
            double x[M::D];
            for (int j = 0; j < M::D; j++) x[j] = X[j * n + p];
            const double e = model_logeta(m, k, x);
            le[p] = e;
            v = v + e;
        }
        la[i] = v;
    }
}

// su = the sorted first coordinate of the points (from its sorted integers)
__global__ void k_sqmc_su(const uint32_t *raw0s, int64_t n, double *su) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        su[i] = squeeze(raw0s[i]);
}

// A = h[idx]; X = Gamma(t, X_{t-1}[A], u[tau, 1:]); lw = reset + logG(t, Xp, X), reset = log_mean_exp(logeta, W) -
// logeta[A] for the APF kinds (core.py:299-305), 0 otherwise
template <class M, int FK>
__global__ void k_sqmc_move(const double *tab, const M m, const FilterArgs a, int64_t t, const double *Xp,
                            const int64_t *h, const int64_t *idx, const int64_t *tau, const double *u, const double *le,
                            const double *stats, int64_t n, long long *A, double *X, double *lw) {
    __shared__ __align__(8) uint64_t s_bar;
    stage_math_tables(tab, &s_bar);
    const StepK k = step_consts(a, t);
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t p = h[idx[i]], r = tau[i];
        A[i] = p;
        double xp[M::D], z[M::D], x[M::D], d;
        for (int j = 0; j < M::D; j++) xp[j] = Xp[j * n + p];
        for (int j = 0; j < M::NZ; j++) z[j] = ndtri(u[(1 + j) * n + r]);
        model_move<M, FK>(m, k, xp, z, x, d);
        for (int j = 0; j < M::D; j++) X[j * n + i] = x[j];
        lw[i] = FkTraits<FK>::apf ? (stats[12] - le[p]) + d : d;
    }
}

// summary row t (ESS, logLt, rs_flag, log_mean_w) from the statistics {max, log_mean, ESS, sum} of the new weights
__global__ void k_sqmc_row(double *summ, int64_t t, const double *st) {
    const double lm = st[1];
    summ[t * SMCB_SUMMARY_STRIDE + 0] = st[2];
    summ[t * SMCB_SUMMARY_STRIDE + 1] = (t == 0 ? 0.0 : summ[(t - 1) * SMCB_SUMMARY_STRIDE + 1]) + lm;
    summ[t * SMCB_SUMMARY_STRIDE + 2] = t == 0 ? 0.0 : 1.0;
    summ[t * SMCB_SUMMARY_STRIDE + 3] = lm;
}

// the points of step t: the Sobol' points of key (seed, t), or the caller's (desc.u_in: per step du + 1 rows of n,
// component-major; step 0 reads the first du rows).  For t >= 1 also tau = argsort(u[0]) and su = u[0][tau].
int sqmc_points(smcb_filter *f, const SqmcWs &w, int du, int64_t t) {
    smcb_ctx *c = f->ctx;
    const smcb_filter_desc &d = f->desc;
    const int64_t n = d.n;
    const int rows = t == 0 ? du : du + 1;
    size_t cb = w.cub_bytes;
    if (d.u_in) {
        SMCB_CUDA(cudaMemcpyAsync(w.u, d.u_in + (size_t)t * (du + 1) * n, sizeof(double) * rows * n,
                                  cudaMemcpyDeviceToDevice, c->stream));
        if (t == 0) return SMCB_OK;
        SMCB_TRY(launch(c, k_iota, grid_for(n, kThreads), kThreads, 0, w.iota, n));
        SMCB_CUDA(cub::DeviceRadixSort::SortPairs(w.cub, cb, (const double *)w.u, w.su, w.iota, w.tau, (int)n, 0, 64,
                                                  c->stream));
        return SMCB_OK;
    }
    SMCB_TRY(sobol(c, rows, n, 1, d.seed, (uint64_t)t, w.u, t == 0 ? nullptr : w.raw));
    if (t == 0) return SMCB_OK;
    SMCB_TRY(launch(c, k_iota, grid_for(n, kThreads), kThreads, 0, w.iota, n));
    SMCB_CUDA(cub::DeviceRadixSort::SortPairs(w.cub, cb, (const uint32_t *)w.raw, w.raw0s, w.iota, w.tau, (int)n, 0, 30,
                                              c->stream));
    return launch(c, k_sqmc_su, grid_for(n, kThreads), kThreads, 0, (const uint32_t *)w.raw0s, n, w.su);
}

template <class M, int FK>
int sqmc_one(smcb_filter *f, char *scratch) {
    smcb_ctx *c = f->ctx;
    const smcb_filter_desc &d = f->desc;
    const FilterArgs &fa = f->args;
    const int64_t n = d.n, t = f->t_host;
    constexpr int du = M::D;
    SqmcWs w;
    sqmc_ws_layout(n, du, scratch, &w);
    M m;                                   // the model constants travel by value: desc.params is host memory
    m.load(d.params);
    // the math tables take kMathTabBytes of shared memory; the opt-in is per device, so it is made on every call
    SMCB_TRY(set_smem(k_sqmc_init<M, FK>, kMathTabBytes));
    SMCB_TRY(set_smem(k_sqmc_aux<M, FK>, kMathTabBytes));
    SMCB_TRY(set_smem(k_sqmc_move<M, FK>, kMathTabBytes));
    const double *tab = c->math_tab;
    const int g = grid_for(n, kThreads);
    double *X = d.X[t & 1], *lw = d.lw[t & 1];
    SMCB_TRY(sqmc_points(f, w, du, t));
    if (t == 0) {
        SMCB_TRY(launch(c, k_sqmc_init<M, FK>, g, kThreads, kMathTabBytes, tab, m, fa, (const double *)w.u, n, X, lw));
    } else {
        const double *Xprev = d.X[(t - 1) & 1];
        double *lwprev = d.lw[(t - 1) & 1];
        SMCB_TRY(hilbert_order(c, Xprev, n, du, w.h, nullptr, w.hws));
        SMCB_TRY(launch(c, k_sqmc_aux<M, FK>, g, kThreads, kMathTabBytes, tab, m, fa, t, Xprev,
                        (const double *)lwprev, (const int64_t *)w.h, n, w.la, w.le));
        SMCB_TRY(smcb_normalise(c, w.la, n, w.wh, w.stats));
        SMCB_TRY(smcb_cumsum(c, w.wh, n, d.cdf));
        SMCB_TRY(smcb_searchsorted(c, d.cdf, n, w.su, n, w.idx));
        if (FkTraits<FK>::apf) {     // log_mean_exp(logeta, W = W_{t-1}) into stats[12]
            SMCB_TRY(smcb_normalise(c, lwprev, n, w.wprev, w.stats + 4));
            SMCB_TRY(smcb_lse(c, SMCB_LSE_MEAN, w.le, w.wprev, n, w.stats + 12));
        }
        SMCB_TRY(launch(c, k_sqmc_move<M, FK>, g, kThreads, kMathTabBytes, tab, m, fa, t, Xprev, (const int64_t *)w.h,
                        (const int64_t *)w.idx, (const int64_t *)w.tau, (const double *)w.u, (const double *)w.le,
                        (const double *)w.stats, n, reinterpret_cast<long long *>(d.A), X, lw));
    }
    SMCB_TRY(smcb_normalise(c, lw, n, nullptr, w.stats + 8));
    return launch(c, k_sqmc_row, 1, 1, 0, d.summaries, t, (const double *)(w.stats + 8));
}

__global__ void k_ndtri(const double *u, double *out, int64_t n) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        out[i] = ndtri(u[i]);
}

}  // namespace

extern "C" int smcb_ndtri(smcb_ctx *c, const double *u, double *out, int64_t n) {
    SMCB_REQUIRE(c && u && out, "smcb_ndtri: NULL argument");
    SMCB_REQUIRE(n >= 0, "smcb_ndtri: n must be >= 0");
    if (n == 0) return SMCB_OK;
    return launch(c, k_ndtri, grid_for(n, kThreads), kThreads, 0, u, out, n);
}

extern "C" int smcb_sobol(smcb_ctx *c, int d, int64_t n, int scramble, uint64_t seed, uint64_t call, double *u,
                          int32_t *raw) {
    SMCB_REQUIRE(c && (u || raw), "smcb_sobol: NULL argument");
    SMCB_REQUIRE(d >= 1 && d <= kSobolMaxDim, "smcb_sobol: d must be 1..%d (got %d)", kSobolMaxDim, d);
    SMCB_REQUIRE(n >= 1 && n <= (int64_t)1 << 30, "smcb_sobol: n must be 1..2^30");
    return sobol(c, d, n, scramble ? 1 : 0, seed, call, u, raw);
}

extern "C" int64_t smcb_hilbert_scratch_bytes(int64_t n, int d) {
    if (n < 1 || n > INT32_MAX || d < 1 || d > kHilbertMaxDim) return -1;
    return (int64_t)hilbert_ws_bytes(n, d);
}

extern "C" int smcb_hilbert_sort(smcb_ctx *c, const double *x, int64_t n, int d, int64_t *order, int64_t *keys,
                                 void *scratch) {
    SMCB_REQUIRE(c && x && order && scratch, "smcb_hilbert_sort: NULL argument");
    SMCB_REQUIRE(n >= 1 && n <= INT32_MAX, "smcb_hilbert_sort: n must be 1..2^31-1");
    SMCB_REQUIRE(d >= 1 && d <= kHilbertMaxDim, "smcb_hilbert_sort: d must be 1..%d (got %d)", kHilbertMaxDim, d);
    SMCB_REQUIRE(((uintptr_t)scratch & 255) == 0, "smcb_hilbert_sort: scratch must be 256-byte aligned");
    return hilbert_order(c, x, n, d, order, keys, (char *)scratch);
}

extern "C" int64_t smcb_sqmc_scratch_bytes(int64_t n, int dim) {
    if (n < 1 || n > INT32_MAX || dim < 1 || dim > 4) return -1;
    return (int64_t)sqmc_ws_layout(n, dim, nullptr, nullptr);
}

extern "C" int smcb_sqmc_step(smcb_filter *f, int64_t nsteps, void *scratch) {
    SMCB_REQUIRE(f && scratch, "smcb_sqmc_step: NULL argument");
    SMCB_REQUIRE(((uintptr_t)scratch & 255) == 0, "smcb_sqmc_step: scratch must be 256-byte aligned");
    SMCB_REQUIRE(f->args.world == 1, "smcb_sqmc_step: SQMC runs on one device");
    SMCB_REQUIRE(f->t_host + nsteps <= f->desc.T, "smcb_sqmc_step: past the last step (StopIteration)");
    const smcb_filter_desc &d = f->desc;
    for (int64_t s = 0; s < nsteps; s++) {
        const int rc = with_model(d.model, d.dim, [&](auto m) {
            using M = decltype(m);
            if (M::D != d.dim) return (int)SMCB_ENOSYS;
            return with_fk<M>(d.fk, [&](auto fk) { return sqmc_one<M, decltype(fk)::value>(f, (char *)scratch); });
        });
        if (rc == SMCB_ENOSYS) set_error("smcb_sqmc_step: no SQMC kernel for model %d, kind %d, dim %d", d.model, d.fk,
                                         d.dim);
        if (rc) return rc;
        f->t_host++;
    }
    return SMCB_OK;
}
