// smcb_api.cu -- context + the L0 numerics of the path as stand-alone entry points:
// weights algebra and resampling (particles/resampling.py), distributions
// (particles/distributions.py).  The fused filter lives in smcb_filter.cu.
#include <stdarg.h>
#include <string.h>

#include <new>

#include "smcb_common.cuh"
#include "smcb_math.cuh"
#include "smcb_reduce.cuh"
#include "smcb_scan.cuh"
#include "smcb_search.cuh"

// ---------------------------------------------------------------------------
// errors / context
// ---------------------------------------------------------------------------
static thread_local char g_err[512] = "";
namespace smcb {
void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
}  // namespace smcb
using namespace smcb;

extern "C" const char *smcb_last_error(void) { return g_err; }
extern "C" int smcb_version(void) { return 100; }

extern "C" int smcb_create(smcb_ctx **out, int device, uint64_t seed) {
    SMCB_REQUIRE(out != nullptr, "smcb_create: out is NULL");
    SMCB_CUDA(cudaSetDevice(device));
    smcb_ctx *c = new smcb_ctx();
    c->device = device;
    c->stream = 0;
    c->seed = seed;
    c->api_counter = 0;
    c->launches = 0;
    c->ws_bytes = kWsBytes;
    SMCB_CUDA(cudaMalloc(&c->ws, c->ws_bytes));
    SMCB_CUDA(cudaMalloc(&c->counters, kTicketSlots * sizeof(unsigned int)));
    SMCB_CUDA(cudaMemset(c->counters, 0, kTicketSlots * sizeof(unsigned int)));
    {   // lookup tables of the step kernels' elementary functions (long double on the host, once)
        double *h = new (std::nothrow) double[kMathTabDoubles];
        SMCB_REQUIRE(h != nullptr, "smcb_create: out of host memory");
        fill_math_tables(h);
        cudaError_t e = cudaMalloc(&c->math_tab, kMathTabBytes);
        if (e == cudaSuccess) e = cudaMemcpy(c->math_tab, h, kMathTabBytes, cudaMemcpyHostToDevice);
        delete[] h;
        SMCB_CUDA(e);
    }
    *out = c;
    return SMCB_OK;
}

extern "C" int smcb_destroy(smcb_ctx *c) {
    if (!c) return SMCB_OK;
    cudaSetDevice(c->device);
    cudaFree(c->ws);
    cudaFree(c->counters);
    cudaFree(c->math_tab);
    delete c;
    return SMCB_OK;
}

extern "C" int smcb_set_stream(smcb_ctx *c, void *s) {
    SMCB_REQUIRE(c != nullptr, "smcb_set_stream: ctx is NULL");
    c->stream = (cudaStream_t)s;
    return SMCB_OK;
}

extern "C" int smcb_seed(smcb_ctx *c, uint64_t seed) {
    SMCB_REQUIRE(c != nullptr, "smcb_seed: ctx is NULL");
    c->seed = seed;
    c->api_counter = 0;
    return SMCB_OK;
}

extern "C" int64_t smcb_launch_count(const smcb_ctx *c) { return c ? c->launches : 0; }

static int check_ws(smcb_ctx *c, size_t need) {
    if (need <= c->ws_bytes) return SMCB_OK;
    SMCB_CUDA(cudaStreamSynchronize(c->stream));
    SMCB_CUDA(cudaFree(c->ws));
    c->ws_bytes = need + (need >> 2);
    SMCB_CUDA(cudaMalloc(&c->ws, c->ws_bytes));
    return SMCB_OK;
}

// ---------------------------------------------------------------------------
// weights algebra
// ---------------------------------------------------------------------------
enum { kModeNormalise = 10, kModeWeightedMean = 11 };

// one pass: (max, sum exp, sum exp^2) of v, deterministic grid merge, scalars out.
// mode kModeNormalise also rewrites NaN -> -inf in place (resampling.py:220).
// The other modes follow the reference's m + log(sum(exp(v - m))) at the edges: a NaN anywhere, a +inf anywhere or
// every entry -inf gives NaN (NaN - m, inf - inf, -inf - -inf).  A NaN marks its accumulator's max as well as its sum,
// so that no merge drops it as an empty (max -inf) partial.
template <int MODE>
__global__ void __launch_bounds__(kBlock) k_lse(double *v, const double *__restrict__ W, int64_t n,
                                               double *partials, unsigned int *ticket,
                                               double *out) {
    __shared__ Lse3 smem[kBlock / 32];
    Lse3 acc[1] = {lse3_empty()};
    double sw = 0.0;  // sum of W (weighted mean only)
    const int64_t stride = (int64_t)gridDim.x * kBlock;
    int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x;
    if (MODE != kModeWeightedMean) {
        // eight independent loads in flight per thread and ONE running-max update per batch of eight (one exp per
        // value, branch-free polynomial exp).  A table-assisted exp with a third of the instructions did not move the
        // time: the kernel is bound by the latency of its four rounds of loads per thread, not by issue
        bool saw_nan = false;
        for (; i + 7 * stride < n; i += 8 * stride) {
            double x[8];
#pragma unroll
            for (int j = 0; j < 8; j++) x[j] = v[i + j * stride];
#pragma unroll
            for (int j = 0; j < 8; j++) {
                if (x[j] != x[j]) {
                    x[j] = -CUDART_INF;
                    if (MODE == kModeNormalise) v[i + j * stride] = x[j];      // resampling.py:220
                    else saw_nan = true;                                       // NumPy: max() of a NaN array is NaN
                }
            }
            lse3_add_batch_f<8>(acc[0], x);
        }
        for (; i < n; i += stride) {
            double x[1] = {v[i]};
            if (x[0] != x[0]) {
                x[0] = -CUDART_INF;
                if (MODE == kModeNormalise) v[i] = x[0];
                else saw_nan = true;
            }
            lse3_add_batch_f<1>(acc[0], x);
        }
        if (saw_nan) { acc[0].m = CUDART_NAN; acc[0].s = CUDART_NAN; }
    } else {
        for (; i < n; i += stride) {
            double x = v[i];
            // log_mean_exp(v, W): m + log( sum W e^{v-m} / sum W )  (resampling.py:312-317)
            double w = W[i];
            sw += w;
            if (x != x) { acc[0].m = CUDART_NAN; acc[0].s = CUDART_NAN; continue; }
            if (x == -CUDART_INF) continue;
            double d = x - acc[0].m;
            double e = exp(-fabs(d));
            if (d > 0.0) { acc[0].s = acc[0].s * e + w; acc[0].m = x; }
            else acc[0].s += w * e;
        }
    }
    if (MODE == kModeWeightedMean) {
        // carry sum W in the q slot; it must NOT be rescaled by the merges, so reduce it apart
        __shared__ double s_sw[kBlock / 32];
        sw = warp_sum(sw);
        if ((threadIdx.x & 31) == 0) s_sw[threadIdx.x >> 5] = sw;
        __syncthreads();
        if (threadIdx.x == 0) {
            double t = 0.0;
            for (int w = 0; w < kBlock / 32; w++) t += s_sw[w];
            partials[(size_t)blockIdx.x * 4 + 3] = t;
        }
        acc[0].q = 0.0;
    }
    Lse3 tot[1];
    if (!grid_merge_lse3<kBlock, 1>(acc, partials, ticket, smem, tot)) return;
    if (MODE == kModeWeightedMean) {
        __shared__ double s_tot;
        if (threadIdx.x == 0) {
            double t = 0.0;
            for (int k = 0; k < (int)gridDim.x; k++) t += ((volatile double *)partials)[(size_t)k * 4 + 3];
            s_tot = t;
        }
        __syncthreads();
        if (threadIdx.x == 0) out[0] = (fabs(tot[0].m) == CUDART_INF) ? CUDART_NAN : tot[0].m + log(tot[0].s / s_tot);
        return;
    }
    if (threadIdx.x != 0) return;
    const Lse3 t = tot[0];
    const bool edge = (fabs(t.m) == CUDART_INF);             // all -inf, or a +inf: NaN, as NumPy gives
    if (MODE == kModeNormalise) {
        double lm, ess;
        weights_scalars(t, (double)n, lm, ess);
        out[0] = t.m; out[1] = lm; out[2] = ess;
        out[3] = (lm != lm) ? CUDART_NAN : t.s;
    } else if (MODE == SMCB_LSE_SUM) {
        out[0] = edge ? CUDART_NAN : t.m + log(t.s);
    } else if (MODE == SMCB_LSE_MEAN) {
        out[0] = edge ? CUDART_NAN : t.m + log(t.s / (double)n);
    } else if (MODE == SMCB_LSE_ESSL) {
        out[0] = edge ? CUDART_NAN : (t.s * t.s) / t.q;
    }
}

// W = exp(lw - m) / s   (resampling.py:223-225, 162-163); stats = {m, ., ., s}
__global__ void __launch_bounds__(kBlock) k_exp_normalise(const double *__restrict__ lw, int64_t n,
                                                         const double *__restrict__ stats,
                                                         double *__restrict__ W) {
    const double m = stats[0], s = stats[3];
    const double r = 1.0 / s;
    const int64_t stride = (int64_t)gridDim.x * kBlock;
    int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x;
    // w / s as q + fma(-q, s, w) * r with q = w * r: the correctly rounded quotient without the division sequence
    for (; i + 3 * stride < n; i += 4 * stride) {
        double x[4];
#pragma unroll
        for (int j = 0; j < 4; j++) x[j] = lw[i + j * stride];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const double w = fexp(x[j] - m);
            const double q = w * r;
            W[i + j * stride] = (s == s && s > 0.0 && s < CUDART_INF) ? fma(fma(-q, s, w), r, q) : w / s;
        }
    }
    for (; i < n; i += stride) {
        const double w = fexp(lw[i] - m);
        const double q = w * r;
        W[i] = (s == s && s > 0.0 && s < CUDART_INF) ? fma(fma(-q, s, w), r, q) : w / s;
    }
}

extern "C" int smcb_normalise(smcb_ctx *c, double *lw, int64_t n, double *W_out,
                              double *stats_out) {
    SMCB_REQUIRE(c && lw && stats_out, "smcb_normalise: NULL argument");
    SMCB_REQUIRE(n >= 1, "smcb_normalise: n must be >= 1 (got %lld)", (long long)n);
    const int grid = grid_for(n, kBlock * 4);
    SMCB_TRY(launch(c, k_lse<kModeNormalise>, grid, kBlock, 0, lw, nullptr, n, c->ws, c->counters + kTicketLse,
                    stats_out));
    if (!W_out) return SMCB_OK;
    return launch(c, k_exp_normalise, grid_for(n, kBlock * 4), kBlock, 0, lw, n, stats_out, W_out);
}

// W = exp(lw - m) / s from statistics the caller already holds (stats = {m, ., ., s}: the layout smcb_normalise
// writes; the fused filter's device state; for a sharded filter the GLOBAL (m, s), so that W sums to one over all ranks)
extern "C" int smcb_weights_from_stats(smcb_ctx *c, const double *lw, int64_t n, const double *stats, double *W_out) {
    SMCB_REQUIRE(c && lw && stats && W_out, "smcb_weights_from_stats: NULL argument");
    SMCB_REQUIRE(n >= 1, "smcb_weights_from_stats: n must be >= 1");
    return launch(c, k_exp_normalise, grid_for(n, kBlock * 4), kBlock, 0, lw, n, stats, W_out);
}

extern "C" int smcb_lse(smcb_ctx *c, int mode, const double *v, const double *W, int64_t n,
                        double *out) {
    SMCB_REQUIRE(c && v && out, "smcb_lse: NULL argument");
    SMCB_REQUIRE(n >= 1, "smcb_lse: n must be >= 1");
    const int grid = grid_for(n, kBlock * 4);
    double *vv = const_cast<double *>(v);
    unsigned int *ticket = c->counters + kTicketLse;
    if (mode == SMCB_LSE_SUM) return launch(c, k_lse<SMCB_LSE_SUM>, grid, kBlock, 0, vv, nullptr, n, c->ws, ticket, out);
    if (mode == SMCB_LSE_MEAN && W == nullptr)
        return launch(c, k_lse<SMCB_LSE_MEAN>, grid, kBlock, 0, vv, nullptr, n, c->ws, ticket, out);
    if (mode == SMCB_LSE_MEAN) return launch(c, k_lse<kModeWeightedMean>, grid, kBlock, 0, vv, W, n, c->ws, ticket, out);
    if (mode == SMCB_LSE_ESSL)
        return launch(c, k_lse<SMCB_LSE_ESSL>, grid, kBlock, 0, vv, nullptr, n, c->ws, ticket, out);
    set_error("smcb_lse: unknown mode %d", mode);
    return SMCB_EINVAL;
}

// exp_and_normalise: m = max, w = exp(lw - m), W = w / sum(w)  (no NaN rewrite)
__global__ void __launch_bounds__(kBlock) k_max_sum(const double *__restrict__ v, int64_t n,
                                                   double *partials, unsigned int *ticket,
                                                   double *stats) {
    __shared__ Lse3 smem[kBlock / 32];
    Lse3 acc[1] = {lse3_empty()};
    const int64_t stride = (int64_t)gridDim.x * kBlock;
    for (int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x; i < n; i += stride) {
        double x = v[i];
        if (x != x) { acc[0].m = CUDART_NAN; acc[0].s = CUDART_NAN; continue; }     // kept through every merge
        lse3_add(acc[0], x);
    }
    Lse3 tot[1];
    if (!grid_merge_lse3<kBlock, 1>(acc, partials, ticket, smem, tot)) return;
    if (threadIdx.x == 0) {
        bool bad = (tot[0].m == -CUDART_INF || tot[0].m == CUDART_INF);
        stats[0] = tot[0].m; stats[1] = 0.0; stats[2] = 0.0;
        stats[3] = bad ? CUDART_NAN : tot[0].s;
    }
}

extern "C" int smcb_exp_and_normalise(smcb_ctx *c, const double *lw, int64_t n, double *W_out) {
    SMCB_REQUIRE(c && lw && W_out, "smcb_exp_and_normalise: NULL argument");
    SMCB_REQUIRE(n >= 1, "smcb_exp_and_normalise: n must be >= 1");
    double *stats = c->ws + kWsPartials;  // 4 doubles right after the partials
    SMCB_TRY(launch(c, k_max_sum, grid_for(n, kBlock * 4), kBlock, 0, lw, n, c->ws, c->counters + kTicketLse, stats));
    return launch(c, k_exp_normalise, grid_for(n, kBlock * 4), kBlock, 0, lw, n, stats, W_out);
}

// wmean_and_var (resampling.py:320-338): np.average(x, weights=W), np.average(x^2, weights=W)
// one block row per component; partial sums merged in a fixed order by the last block
__global__ void __launch_bounds__(kBlock) k_wmoments(const double *__restrict__ W,
                                                    const double *__restrict__ x, int64_t n, int d,
                                                    double *partials, unsigned int *ticket,
                                                    double *out) {
    // partials layout: [block][3*d + 1]: sum W, then per component sum W x, sum W x^2
    __shared__ double s_red[9][kBlock / 32];
    const int nv = 1 + 2 * d;
    const int64_t stride = (int64_t)gridDim.x * kBlock;
    // ONE pass over W and x per chunk of 4 components (d <= 4: one pass in all; the first version re-read W for every
    // one of the 1 + 2 d sums), two elements in flight per thread
    for (int c0 = 0; c0 < d; c0 += 4) {
        const int dc = d - c0 < 4 ? d - c0 : 4;
        double a[9];
#pragma unroll
        for (int q = 0; q < 9; q++) a[q] = 0.0;
        int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x;
        for (; i + stride < n; i += 2 * stride) {
            const double w0 = W[i], w1 = W[i + stride];
            double x0[4], x1[4];
#pragma unroll
            for (int c = 0; c < 4; c++) {
                x0[c] = (c < dc) ? x[(size_t)(c0 + c) * n + i] : 0.0;
                x1[c] = (c < dc) ? x[(size_t)(c0 + c) * n + i + stride] : 0.0;
            }
            a[0] += w0;
            a[0] += w1;
#pragma unroll
            for (int c = 0; c < 4; c++) {
                a[1 + 2 * c] += w0 * x0[c]; a[2 + 2 * c] += w0 * (x0[c] * x0[c]);
                a[1 + 2 * c] += w1 * x1[c]; a[2 + 2 * c] += w1 * (x1[c] * x1[c]);
            }
        }
        for (; i < n; i += stride) {
            const double w0 = W[i];
            a[0] += w0;
#pragma unroll
            for (int c = 0; c < 4; c++) {
                const double xv = (c < dc) ? x[(size_t)(c0 + c) * n + i] : 0.0;
                a[1 + 2 * c] += w0 * xv; a[2 + 2 * c] += w0 * (xv * xv);
            }
        }
#pragma unroll
        for (int q = 0; q < 9; q++) {
            const double acc = warp_sum(a[q]);
            if ((threadIdx.x & 31) == 0) s_red[q][threadIdx.x >> 5] = acc;
        }
        __syncthreads();
        if (threadIdx.x < 9) {
            const int q = threadIdx.x;
            double t = 0.0;
            for (int w = 0; w < kBlock / 32; w++) t += s_red[q][w];
            const int slot = (q == 0) ? 0 : 2 * c0 + q;                 // sum W | per component sum W x, sum W x^2
            if ((q == 0 && c0 == 0) || (q > 0 && (q - 1) / 2 < dc)) partials[(size_t)blockIdx.x * nv + slot] = t;
        }
        __syncthreads();
    }
    if (!last_block(ticket)) return;
    if (threadIdx.x < nv) {
        double t = 0.0;
        for (int k = 0; k < (int)gridDim.x; k++)
            t += ((volatile double *)partials)[(size_t)k * nv + threadIdx.x];
        partials[(size_t)gridDim.x * nv + threadIdx.x] = t;
    }
    __syncthreads();
    if (threadIdx.x < d) {
        const double *tot = partials + (size_t)gridDim.x * nv;
        double sw = tot[0];
        double m = tot[1 + 2 * threadIdx.x] / sw;
        double m2 = tot[2 + 2 * threadIdx.x] / sw;
        out[threadIdx.x] = m;
        out[d + threadIdx.x] = m2 - m * m;
    }
}

extern "C" int smcb_wmean_and_var(smcb_ctx *c, const double *W, const double *x, int64_t n, int d,
                                  double *out) {
    SMCB_REQUIRE(c && W && x && out, "smcb_wmean_and_var: NULL argument");
    // d <= 32, the samplers' largest dimension: (592 + 1) (2 d + 1) partials fit kWsPartials, 2 d + 1 <= kBlock
    SMCB_REQUIRE(n >= 1 && d >= 1 && d <= 32, "smcb_wmean_and_var: need n >= 1, 1 <= d <= 32 (got n=%lld d=%d)",
                 (long long)n, d);
    int grid = grid_for(n, kBlock * 4);
    if (grid > 592) grid = 592;
    return launch(c, k_wmoments, grid, kBlock, 0, W, x, n, d, c->ws, c->counters + kTicketWmoments, out);
}

// ---------------------------------------------------------------------------
// prefix sums
// ---------------------------------------------------------------------------
struct LoadPlain {
    const double *w;
    __device__ __forceinline__ void operator()(int64_t i0, int64_t n, double (&v)[8]) const {
        if (i0 + 8 <= n) {
#pragma unroll
            for (int j = 0; j < 8; j += 2) { double2 t = ld2(w + i0 + j); v[j] = t.x; v[j + 1] = t.y; }
        } else {
#pragma unroll
            for (int j = 0; j < 8; j++) v[j] = (i0 + j < n) ? w[i0 + j] : 0.0;
        }
    }
};
// -log(u): the exponential spacings of uniform_spacings (resampling.py:536)
struct LoadNegLog {
    const double *u;
    __device__ __forceinline__ void operator()(int64_t i0, int64_t n, double (&v)[8]) const {
#pragma unroll
        for (int j = 0; j < 8; j++) v[j] = (i0 + j < n) ? -log(u[i0 + j]) : 0.0;
    }
};
// residual resampling (resampling.py:617-621): intpart = floor(M W), res = M W - intpart
struct LoadIntPart {
    const double *W; double M;
    __device__ __forceinline__ void operator()(int64_t i0, int64_t n, long long (&v)[8]) const {
#pragma unroll
        for (int j = 0; j < 8; j++) v[j] = (i0 + j < n) ? (long long)floor(M * W[i0 + j]) : 0ll;
    }
};
struct LoadResidual {
    const double *W; double M; const long long *cum_ip;  // sres = M - cum_ip[n-1]
    int64_t nn;
    __device__ __forceinline__ void operator()(int64_t i0, int64_t n, double (&v)[8]) const {
        const double sres = (double)((long long)M - cum_ip[nn - 1]);
#pragma unroll
        for (int j = 0; j < 8; j++) {
            double mw = (i0 + j < n) ? M * W[i0 + j] : 0.0;
            v[j] = (i0 + j < n) ? (mw - floor(mw)) / sres : 0.0;
        }
    }
};

// carve the scan slot out of the context workspace (after the partials area)
static int scan_state(smcb_ctx *c, int64_t n, ScanState *st, int slot) {
    const size_t bytes = scan_state_bytes(n);
    const size_t base = (kWsPartials + 16) * sizeof(double);
    int rc = check_ws(c, base + 2 * bytes + 64);
    if (rc) return rc;
    const size_t half = ((c->ws_bytes - base) / 2) & ~(size_t)15;  // two slots: scans may chain
    st->chunk_sum = (char *)c->ws + base + (size_t)slot * half;
    return SMCB_OK;
}

template <typename T, typename LOAD>
__global__ void __launch_bounds__(kBlock) k_scan_sums(LOAD load, int64_t n, int tiles_per_chunk, T *chunk_sum) {
    scan_chunk_sums<T, LOAD>(load, n, tiles_per_chunk, chunk_sum);
}
template <typename T, typename LOAD>
__global__ void __launch_bounds__(kBlock) k_scan_chunks(LOAD load, int64_t n, int tiles_per_chunk, const T *chunk_sum,
                                                       int nchunks, T *out) {
    scan_chunks<T, LOAD>(load, n, tiles_per_chunk, chunk_sum, nchunks, out);
}

// reduce-then-scan (smcb_scan.cuh); `slot` 0 / 1: two scans may be in flight on the stream (multinomial, residual)
template <typename T, typename LOAD>
static int run_scan(smcb_ctx *c, const LOAD &load, int64_t n, T *out, int slot = 0) {
    ScanState st;
    int rc = scan_state(c, n, &st, slot);
    if (rc) return rc;
    const int64_t tiles = scan_tiles(n);
    // one chunk per CTA that can be resident (occupancy of the scan kernel x SMs): a grid of 1.1 - 1.4 waves, as the
    // fixed "6 per SM" gave, ends with a half-empty second round
    static int occ = 0;
    if (occ == 0) {
        int o = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, k_scan_chunks<T, LOAD>, kBlock, 0) != cudaSuccess || o < 1) o = 4;
        occ = o;
    }
    int64_t want = (int64_t)kSMs * occ;
    if (want > kScanMaxChunks) want = kScanMaxChunks;
    const int tpc = (int)((tiles + want - 1) / want);
    const int nchunks = (int)((tiles + tpc - 1) / tpc);
    T *sums = reinterpret_cast<T *>(st.chunk_sum);
    SMCB_TRY(launch(c, k_scan_sums<T, LOAD>, nchunks, kBlock, 0, load, n, tpc, sums));
    return launch(c, k_scan_chunks<T, LOAD>, nchunks, kBlock, 0, load, n, tpc, sums, nchunks, out);
}

extern "C" int smcb_cumsum(smcb_ctx *c, const double *w, int64_t n, double *cdf_out) {
    SMCB_REQUIRE(c && w && cdf_out, "smcb_cumsum: NULL argument");
    SMCB_REQUIRE(n >= 1, "smcb_cumsum: n must be >= 1");
    SMCB_REQUIRE(((uintptr_t)w & 15) == 0 && ((uintptr_t)cdf_out & 15) == 0,
                 "smcb_cumsum: arrays must be 16-byte aligned");
    return run_scan<double>(c, LoadPlain{w}, n, cdf_out);
}

// ---------------------------------------------------------------------------
// inverse-CDF search
// ---------------------------------------------------------------------------
constexpr int kSearchPer = 4;                       // outputs per thread
constexpr int kSearchTile = kBlock * kSearchPer;    // outputs per tile

// SU: functor double operator()(int64_t k) giving the k-th sorted uniform
struct SuArray { const double *su; __device__ __forceinline__ double operator()(int64_t k) const { return su[k]; } };
struct SuSystematic {  // resampling.py:609  (rand(1) + arange(M)) / M
    const double *u; double M;
    __device__ __forceinline__ double operator()(int64_t k) const { return (u[0] + (double)k) / M; }
};
struct SuStratified {  // resampling.py:602  (rand(M) + arange(M)) / M
    const double *u; double M;
    __device__ __forceinline__ double operator()(int64_t k) const { return (u[k] + (double)k) / M; }
};
struct SuSpacings {    // resampling.py:537  z[:-1] / z[-1]
    const double *z; int64_t M;
    __device__ __forceinline__ double operator()(int64_t k) const { return z[k] / z[M]; }
};

// Tile boundaries first, all at once: thread t finds where the first uniform of tile t lands (one global bisection
// each, ~10^4 of them in parallel), so the tile kernel below knows its slice of the CDF without any block-wide
// search; the slice is then staged in shared memory with coalesced loads and every output bisects THERE.  The first
// version bracketed every tile with two block-cooperative searches of the whole CDF and bisected in global memory:
// 174 us for 1e7 outputs.
constexpr int kSearchStage = 4096;                  // CDF entries staged per tile (32 KB)

template <typename SU>
__global__ void __launch_bounds__(kBlock) k_search_bounds(const double *__restrict__ cdf, int64_t n, SU su, int64_t m,
                                                         int64_t ntiles, int64_t *__restrict__ bnd) {
    const int64_t t = (int64_t)blockIdx.x * kBlock + threadIdx.x;
    if (t > ntiles) return;
    const int64_t k = t < ntiles ? t * kSearchTile : m - 1;
    bnd[t] = lower_bound(cdf, 0, n, su(k));
}

template <typename SU>
__global__ void __launch_bounds__(kBlock) k_search(const double *__restrict__ cdf, int64_t n, SU su,
                                                  int64_t m, int64_t *__restrict__ A,
                                                  int64_t a_offset, const int64_t *__restrict__ bnd) {
    __shared__ double s_cdf[kSearchStage];
    const int64_t ntiles = (m + kSearchTile - 1) / kSearchTile;
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t k0 = tile * kSearchTile;
        // the uniforms are sorted, so the tile's answers lie in [lo, hi]
        const int64_t lo = bnd[tile];
        const int64_t hi = bnd[tile + 1];
        const int64_t hi1 = hi < n ? hi + 1 : n;
        const int len = (hi1 - lo <= (int64_t)kSearchStage) ? (int)(hi1 - lo) : -1;
        if (len >= 0) {
            for (int i = threadIdx.x; i < len; i += kBlock) s_cdf[i] = cdf[lo + i];
            __syncthreads();
        }
#pragma unroll
        for (int j = 0; j < kSearchPer; j++) {
            const int64_t k = k0 + (int64_t)j * kBlock + threadIdx.x;
            if (k < m) {
                const double v = su(k);
                int64_t a;
                if (len >= 0) {
                    int l = 0, h = len;
                    while (l < h) { const int mid = (l + h) >> 1; if (s_cdf[mid] < v) l = mid + 1; else h = mid; }
                    a = lo + l;
                } else {
                    a = lower_bound(cdf, lo, hi1, v);
                }
                A[a_offset + k] = a < n - 1 ? a : n - 1;
            }
        }
        if (len >= 0) __syncthreads();
    }
}

template <typename SU>
static int run_search(smcb_ctx *c, const double *cdf, int64_t n, const SU &su, int64_t m,
                      int64_t *A, int64_t a_offset) {
    if (m <= 0) return SMCB_OK;
    int64_t tiles = (m + kSearchTile - 1) / kSearchTile;
    // tile boundaries live in scan slot 0 of the workspace (the CDF's scan, stream-ordered before us, is done with it)
    const size_t base = (kWsPartials + 16) * sizeof(double);
    const size_t need = (size_t)(tiles + 2) * sizeof(int64_t);
    const size_t sc = scan_state_bytes(n);
    int rc = check_ws(c, base + 2 * (need > sc ? need : sc) + 64);
    if (rc) return rc;
    int64_t *bnd = reinterpret_cast<int64_t *>((char *)c->ws + base);
    SMCB_TRY(launch(c, k_search_bounds<SU>, (int)((tiles + 1 + kBlock - 1) / kBlock), kBlock, 0, cdf, n, su, m, tiles,
                    bnd));
    static int occ = 0;                        // resident CTAs per SM of this instantiation: the grid is ONE full wave
    if (occ == 0) {
        int o = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, k_search<SU>, kBlock, 0) != cudaSuccess || o < 1) o = 4;
        occ = o;
    }
    const int64_t wave = (int64_t)kSMs * occ;
    int grid = (int)(tiles < wave ? tiles : wave);
    return launch(c, k_search<SU>, grid, kBlock, 0, cdf, n, su, m, A, a_offset, bnd);
}

extern "C" int smcb_searchsorted(smcb_ctx *c, const double *cdf, int64_t n, const double *su,
                                 int64_t m, int64_t *A_out) {
    SMCB_REQUIRE(c && cdf && su && A_out, "smcb_searchsorted: NULL argument");
    SMCB_REQUIRE(n >= 1 && m >= 0, "smcb_searchsorted: bad sizes");
    return run_search(c, cdf, n, SuArray{su}, m, A_out, 0);
}

// uniforms from the context stream: block `call` of the API counter space
__global__ void __launch_bounds__(kBlock) k_uniform(Philox key, uint64_t call, double *out,
                                                   int64_t n) {
    const int64_t npairs = (n + 1) >> 1;
    const int64_t stride = (int64_t)gridDim.x * kBlock;
    for (int64_t p = (int64_t)blockIdx.x * kBlock + threadIdx.x; p < npairs; p += stride) {
        double u0, u1;
        uniform_pair(key, (uint64_t)p, (uint32_t)call, ((uint32_t)(call >> 32) << 8) | kPurposeApi, u0, u1);
        out[2 * p] = u0;
        if (2 * p + 1 < n) out[2 * p + 1] = u1;
    }
}
__global__ void __launch_bounds__(kBlock) k_std_normal(Philox key, uint64_t call, double *out,
                                                      int64_t n) {
    const int64_t npairs = (n + 1) >> 1;
    const int64_t stride = (int64_t)gridDim.x * kBlock;
    for (int64_t p = (int64_t)blockIdx.x * kBlock + threadIdx.x; p < npairs; p += stride) {
        uint32_t r[4];
        philox4x32_10((uint32_t)p, (uint32_t)((uint64_t)p >> 32), (uint32_t)call,
                      ((uint32_t)(call >> 32) << 8) | kPurposeApi, key.k0, key.k1, r);
        double z0, z1;
        box_muller(r, z0, z1);
        out[2 * p] = z0;
        if (2 * p + 1 < n) out[2 * p + 1] = z1;
    }
}

extern "C" int smcb_uniform(smcb_ctx *c, double *out, int64_t n) {
    SMCB_REQUIRE(c && out && n >= 0, "smcb_uniform: bad argument");
    if (n == 0) return SMCB_OK;
    return launch(c, k_uniform, grid_for((n + 1) / 2, kBlock * 4), kBlock, 0, key_of(c->seed), c->api_counter++, out,
                  n);
}
extern "C" int smcb_standard_normal(smcb_ctx *c, double *out, int64_t n) {
    SMCB_REQUIRE(c && out && n >= 0, "smcb_standard_normal: bad argument");
    if (n == 0) return SMCB_OK;
    return launch(c, k_std_normal, grid_for((n + 1) / 2, kBlock * 4), kBlock, 0, key_of(c->seed), c->api_counter++,
                  out, n);
}

// residual resampling, deterministic part (resampling.py:622):
//   A[k] = j  for  cum_ip[j-1] <= k < cum_ip[j],  k < sip = cum_ip[n-1]
// == np.arange(N).repeat(intpart); one binary search per output on the int64 CDF.
__global__ void __launch_bounds__(kBlock) k_repeat(const long long *__restrict__ cum_ip, int64_t n,
                                                  int64_t m, int64_t *__restrict__ A) {
    const int64_t sip = cum_ip[n - 1] < m ? cum_ip[n - 1] : m;
    const int64_t stride = (int64_t)gridDim.x * kBlock;
    for (int64_t k = (int64_t)blockIdx.x * kBlock + threadIdx.x; k < sip; k += stride) {
        int64_t lo = 0, hi = n;  // first j with cum_ip[j] > k
        while (lo < hi) {
            int64_t mid = lo + ((hi - lo) >> 1);
            if (cum_ip[mid] <= k) lo = mid + 1; else hi = mid;
        }
        A[k] = lo;
    }
}

// stochastic part of residual resampling: multinomial on res/sres with M - sip draws whose
// number is only known on the device -> the search kernel reads it from cum_ip.
struct SuSpacingsDyn {
    const double *z; const long long *cum_ip; int64_t n; int64_t M;
    __device__ __forceinline__ int64_t count() const { return M - cum_ip[n - 1]; }
};
__global__ void __launch_bounds__(kBlock) k_search_residual(const double *__restrict__ cdf, int64_t n,
                                                           SuSpacingsDyn sd, int64_t *__restrict__ A) {
    const int64_t sres = sd.count();
    if (sres <= 0) return;
    const int64_t sip = sd.M - sres;
    const double zl = sd.z[sres];
    const int64_t stride = (int64_t)gridDim.x * kBlock;
    for (int64_t k = (int64_t)blockIdx.x * kBlock + threadIdx.x; k < sres; k += stride) {
        int64_t a = lower_bound(cdf, 0, n, sd.z[k] / zl);
        A[sip + k] = a < n - 1 ? a : n - 1;
    }
}

// SSP resampling (Srinivasan sampling process, resampling.py:630-677): the pairwise process is a
// sequential recursion over the particles (each step depends on which of the two active indices
// survived the previous one), so ONE thread walks it with the two active (index, fractional part,
// offspring count) triples in registers -- same operations in the same order as the reference,
// hence identical offspring counts for the same uniforms.  O(N) serial: a completeness feature,
// not a hot path.  status[0] = sum of the offspring counts after the reference's round-off fix.
struct LoadCounts {
    const long long *c;
    __device__ __forceinline__ void operator()(int64_t i0, int64_t n, long long (&v)[8]) const {
#pragma unroll
        for (int j = 0; j < 8; j++) v[j] = (i0 + j < n) ? c[i0 + j] : 0ll;
    }
};

__global__ void k_ssp_counts(const double *__restrict__ W, int64_t n, int64_t m, const double *__restrict__ u,
                             long long *__restrict__ nr, long long *__restrict__ status) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const double M = (double)m;
    auto split = [&](int64_t idx, double &xi, long long &cnt) {
        const double mw = M * W[idx];
        const double fl = floor(mw);
        cnt = (long long)fl;
        xi = mw - fl;
    };
    long long total = 0;
    if (n == 1) {
        double x; long long c0;
        split(0, x, c0);
        nr[0] = c0;
        status[0] = c0;
        return;
    }
    int64_t i = 0, j = 1;
    double xi_i, xi_j;
    long long c_i, c_j;
    split(0, xi_i, c_i);
    split(1, xi_j, c_j);
    for (int64_t k = 0; k < n - 1; k++) {
        double delta_i = fmin(xi_j, 1.0 - xi_i);          // increase i, decrease j
        const double delta_j = fmin(xi_i, 1.0 - xi_j);    // the opposite
        const double sum_delta = delta_i + delta_j;
        const double pj = sum_delta > 0.0 ? delta_i / sum_delta : 0.0;
        if (u[k] < pj) {                                  // swap, so that we always increase i
            const int64_t ti = i; i = j; j = ti;
            const double tx = xi_i; xi_i = xi_j; xi_j = tx;
            const long long tc = c_i; c_i = c_j; c_j = tc;
            delta_i = delta_j;
        }
        const int64_t nxt = k + 2;
        if (xi_j < 1.0 - xi_i) {
            xi_i += delta_i;
            nr[j] = c_j; total += c_j;                    // j retires with its integer part
            j = nxt;
            if (nxt < n) split(nxt, xi_j, c_j); else { xi_j = 0.0; c_j = 0; }
        } else {
            xi_j -= delta_i;
            c_i += 1;
            nr[i] = c_i; total += c_i;                    // i retires with one more offspring
            i = nxt;
            if (nxt < n) split(nxt, xi_i, c_i); else { xi_i = 0.0; c_i = 0; }
        }
    }
    // the index that is still in range keeps its count; round-off may have lost one particle
    const int64_t last = (j == n) ? i : j;
    double xl = (j == n) ? xi_i : xi_j;
    long long cl = (j == n) ? c_i : c_j;
    if (total + cl == m - 1 && xl > 0.99) cl += 1;
    nr[last] = cl;
    status[0] = total + cl;
}

extern "C" int64_t smcb_resample_scratch_doubles(int64_t n, int64_t m) {
    return 3 * n + 2 * (m + 2) + 24;
}

extern "C" int smcb_resample(smcb_ctx *c, int scheme, const double *W, int64_t n, int64_t m,
                             int64_t *A_out, const double *u_in, double *scratch) {
    SMCB_REQUIRE(c && W && A_out && scratch, "smcb_resample: NULL argument");
    SMCB_REQUIRE(n >= 1 && m >= 1, "smcb_resample: bad sizes n=%lld m=%lld", (long long)n, (long long)m);
    SMCB_REQUIRE(((uintptr_t)W & 15) == 0 && ((uintptr_t)scratch & 15) == 0,
                 "smcb_resample: arrays must be 16-byte aligned");
    // scratch layout (doubles): cdf[n] | su/z[m+2] | u[m+2] | aux[n]
    double *cdf = scratch;
    double *z = cdf + ((n + 1) & ~(int64_t)1);
    double *u = z + ((m + 3) & ~(int64_t)1);
    double *aux = u + ((m + 3) & ~(int64_t)1);
    int rc;
    if (scheme == SMCB_RS_SSP) {
        // scratch reuse: uniforms (n - 1) in the cdf slot | counts in aux | their scan + status behind it
        double *us = cdf;
        long long *nr = reinterpret_cast<long long *>(aux);
        long long *cum = nr + ((n + 1) & ~(int64_t)1);
        long long *status = cum + ((n + 1) & ~(int64_t)1);
        if (u_in == nullptr) {
            if (n > 1 && (rc = smcb_uniform(c, us, n - 1))) return rc;
            u_in = us;
        }
        SMCB_TRY(launch(c, k_ssp_counts, 1, 32, 0, W, n, m, u_in, nr, status));
        long long total = 0;
        SMCB_CUDA(cudaMemcpyAsync(&total, status, sizeof(total), cudaMemcpyDeviceToHost, c->stream));
        SMCB_CUDA(cudaStreamSynchronize(c->stream));
        if (total != m) {                                 // resampling.py:674-676
            set_error("ssp resampling: wrong size for output");
            return SMCB_EINVAL;
        }
        if ((rc = run_scan<long long>(c, LoadCounts{nr}, n, cum))) return rc;
        return launch(c, k_repeat, grid_for(m, kBlock * 4), kBlock, 0, cum, n, m, A_out);
    }
    const int64_t nu = (scheme == SMCB_RS_SYSTEMATIC) ? 1 : (scheme == SMCB_RS_STRATIFIED ? m : m + 1);
    if (u_in == nullptr) {
        if ((rc = smcb_uniform(c, u, nu))) return rc;
        u_in = u;
    }
    if (scheme == SMCB_RS_SYSTEMATIC || scheme == SMCB_RS_STRATIFIED || scheme == SMCB_RS_MULTINOMIAL) {
        if ((rc = run_scan<double>(c, LoadPlain{W}, n, cdf))) return rc;
        if (scheme == SMCB_RS_SYSTEMATIC) return run_search(c, cdf, n, SuSystematic{u_in, (double)m}, m, A_out, 0);
        if (scheme == SMCB_RS_STRATIFIED) return run_search(c, cdf, n, SuStratified{u_in, (double)m}, m, A_out, 0);
        // multinomial: z = cumsum(-log u) over m+1 uniforms (second scan), su = z[:-1]/z[-1]
        if ((rc = run_scan<double>(c, LoadNegLog{u_in}, m + 1, z, 1))) return rc;
        return run_search(c, cdf, n, SuSpacings{z, m}, m, A_out, 0);
    }
    if (scheme == SMCB_RS_RESIDUAL) {
        long long *cum_ip = reinterpret_cast<long long *>(aux);
        if ((rc = run_scan<long long>(c, LoadIntPart{W, (double)m}, n, cum_ip))) return rc;
        SMCB_TRY(launch(c, k_repeat, grid_for(m, kBlock * 4), kBlock, 0, cum_ip, n, m, A_out));
        // residual weights res/sres -> cdf; spacings over (sres + 1) uniforms: only the first
        // sres + 1 entries of z are meaningful, and z[k]/z[sres] needs exactly those.
        if ((rc = run_scan<double>(c, LoadResidual{W, (double)m, cum_ip, n}, n, cdf))) return rc;
        if ((rc = run_scan<double>(c, LoadNegLog{u_in}, m + 1, z, 1))) return rc;
        return launch(c, k_search_residual, grid_for(m, kBlock * 4), kBlock, 0, cdf, n, SuSpacingsDyn{z, cum_ip, n, m},
                      A_out);
    }
    set_error("smcb_resample: %d is not a valid resampling scheme", scheme);
    return SMCB_EINVAL;
}

// Xp = X[A]  (core.py:332), SoA
__global__ void __launch_bounds__(kBlock) k_gather(const double *__restrict__ X, int64_t n,
                                                  const int64_t *__restrict__ A, int64_t m, int d,
                                                  double *__restrict__ Xp) {
    const int64_t stride = (int64_t)gridDim.x * kBlock;
    for (int64_t k = (int64_t)blockIdx.x * kBlock + threadIdx.x; k < m; k += stride) {
        const int64_t a = A[k];
        for (int j = 0; j < d; j++) Xp[(size_t)j * m + k] = __ldg(X + (size_t)j * n + a);
    }
}

extern "C" int smcb_gather(smcb_ctx *c, const double *X, int64_t n, const int64_t *A, int64_t m,
                           int d, double *Xp) {
    SMCB_REQUIRE(c && X && A && Xp, "smcb_gather: NULL argument");
    SMCB_REQUIRE(n >= 1 && m >= 1 && d >= 1, "smcb_gather: bad sizes");
    return launch(c, k_gather, grid_for(m, kBlock * 4), kBlock, 0, X, n, A, m, d, Xp);
}

__global__ void __launch_bounds__(kBlock) k_gather_rows(const double *__restrict__ X, int64_t n,
                                                       const int64_t *__restrict__ A, int64_t m,
                                                       int d, double *__restrict__ Xp) {
    const int64_t total = m * d;
    const int64_t stride = (int64_t)gridDim.x * kBlock;
    for (int64_t e = (int64_t)blockIdx.x * kBlock + threadIdx.x; e < total; e += stride) {
        const int64_t k = e / d;
        const int j = (int)(e - k * d);
        Xp[e] = __ldg(X + A[k] * d + j);
    }
}

extern "C" int smcb_gather_rows(smcb_ctx *c, const double *X, int64_t n, const int64_t *A,
                                int64_t m, int d, double *Xp) {
    SMCB_REQUIRE(c && X && A && Xp, "smcb_gather_rows: NULL argument");
    SMCB_REQUIRE(n >= 1 && m >= 1 && d >= 1, "smcb_gather_rows: bad sizes");
    return launch(c, k_gather_rows, grid_for(m * d, kBlock * 4), kBlock, 0, X, n, A, m, d, Xp);
}

// ---------------------------------------------------------------------------
// distributions
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlock) k_normal_rvs(Philox key, uint64_t call,
                                                      const double *__restrict__ loc, double loc0,
                                                      const double *__restrict__ scale, double scale0,
                                                      const double *__restrict__ z_in,
                                                      double *__restrict__ out, int64_t n) {
    const int64_t npairs = (n + 1) >> 1;
    const int64_t stride = (int64_t)gridDim.x * kBlock;
    for (int64_t p = (int64_t)blockIdx.x * kBlock + threadIdx.x; p < npairs; p += stride) {
        double z[2];
        if (z_in) {
            z[0] = z_in[2 * p];
            z[1] = (2 * p + 1 < n) ? z_in[2 * p + 1] : 0.0;
        } else {
            uint32_t r[4];
            philox4x32_10((uint32_t)p, (uint32_t)((uint64_t)p >> 32), (uint32_t)call,
                          ((uint32_t)(call >> 32) << 8) | kPurposeApi, key.k0, key.k1, r);
            box_muller(r, z[0], z[1]);
        }
#pragma unroll
        for (int j = 0; j < 2; j++) {
            const int64_t i = 2 * p + j;
            if (i < n) {
                const double l = loc ? loc[i] : loc0, s = scale ? scale[i] : scale0;
                out[i] = l + s * z[j];  // numpy legacy normal: loc + scale * gauss (no FMA: -fmad=false)
            }
        }
    }
}

__global__ void __launch_bounds__(kBlock) k_normal_logpdf(const double *__restrict__ x, double x0,
                                                         const double *__restrict__ loc, double loc0,
                                                         const double *__restrict__ scale, double scale0,
                                                         double *__restrict__ out, int64_t n) {
    const int64_t stride = (int64_t)gridDim.x * kBlock;
    for (int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x; i < n; i += stride)
        out[i] = normal_logpdf(x ? x[i] : x0, loc ? loc[i] : loc0, scale ? scale[i] : scale0);
}

extern "C" int smcb_normal_rvs(smcb_ctx *c, const double *loc, double loc0, const double *scale,
                               double scale0, const double *z_in, double *out, int64_t n) {
    SMCB_REQUIRE(c && out && n >= 1, "smcb_normal_rvs: bad argument");
    uint64_t call = z_in ? 0 : c->api_counter++;
    return launch(c, k_normal_rvs, grid_for((n + 1) / 2, kBlock * 4), kBlock, 0, key_of(c->seed), call, loc, loc0,
                  scale, scale0, z_in, out, n);
}

extern "C" int smcb_normal_logpdf(smcb_ctx *c, const double *x, double x0, const double *loc,
                                  double loc0, const double *scale, double scale0, double *out,
                                  int64_t n) {
    SMCB_REQUIRE(c && out && n >= 1, "smcb_normal_logpdf: bad argument");
    return launch(c, k_normal_logpdf, grid_for(n, kBlock * 4), kBlock, 0, x, x0, loc, loc0, scale, scale0, out, n);
}

// ---------------------------------------------------------------------------
// more univariate log-densities of distributions.py (the ones a state-space model's PY / PX may use): one
// elementwise kernel, parameters scalar or per-particle arrays as for Normal.
//   kind 0 Student(df, loc, scale)  distributions.py:417-433  (scipy.stats.t.logpdf)
//   kind 1 Gamma(a, b)              distributions.py:336-356  (scipy.stats.gamma.logpdf(x, a, scale = 1 / b))
//   kind 2 Laplace(loc, scale)      distributions.py:399-414
//   kind 3 Logistic(loc, scale)     distributions.py:381-396
// p0 is a scalar (df resp. a); its lgamma terms come in as host-computed constants c0.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlock) k_logpdf1(int kind, const double *__restrict__ x, double x0, double p0, double c0,
                                                   const double *__restrict__ p1, double p10,
                                                   const double *__restrict__ p2, double p20,
                                                   double *__restrict__ out, int64_t n) {
    const int64_t stride = (int64_t)gridDim.x * kBlock;
    for (int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x; i < n; i += stride) {
        const double xv = x ? x[i] : x0, a = p1 ? p1[i] : p10, b = p2 ? p2[i] : p20;
        double r;
        if (kind == 0) {                  // c0 = gammaln((df+1)/2) - gammaln(df/2) - log(df pi)/2
            const double z = (xv - a) / b;
            r = c0 - 0.5 * (p0 + 1.0) * log1p(z * z / p0) - log(b);
        } else if (kind == 1) {           // a = rate b (array or scalar); c0 = -gammaln(a_shape)
            // scipy's xlogy(a - 1, x): the term is 0 when a == 1, also at x = 0 and x = +inf; at x = 0 it is +inf for
            // a < 1 and -inf for a > 1, and x = +inf gives -inf for a <= 1 and NaN (inf - inf) for a > 1
            const double xl = (p0 == 1.0) ? 0.0 : (p0 - 1.0) * log(xv);
            r = (xv != xv) ? xv : (xv >= 0.0) ? p0 * log(a) + c0 + xl - a * xv : -CUDART_INF;
        } else if (kind == 2) {
            r = -log(2.0 * b) - fabs(xv - a) / b;
        } else {                          // scipy's symmetric form: exp(-|z|) cannot overflow
            const double y = -fabs((xv - a) / b);
            r = y - 2.0 * log1p(exp(y)) - log(b);
        }
        out[i] = r;
    }
}

extern "C" int smcb_logpdf1(smcb_ctx *c, int kind, const double *x, double x0, double p0, double c0, const double *p1,
                            double p10, const double *p2, double p20, double *out, int64_t n) {
    SMCB_REQUIRE(c && out && n >= 1 && kind >= 0 && kind <= 3, "smcb_logpdf1: bad argument");
    return launch(c, k_logpdf1, grid_for(n, kBlock * 4), kBlock, 0, kind, x, x0, p0, c0, p1, p10, p2, p20, out, n);
}

constexpr int kMaxDim = 8;
struct MvnParams {
    double L[kMaxDim * kMaxDim];   // lower Cholesky factor, row-major
    double loc0[kMaxDim], scale0[kMaxDim];
    double halflogdet;             // sum log diag L
    int d;
};

// MvNormal.rvs: loc + scale * (z @ L.T)   (distributions.py:946-947, 961-969)
__global__ void __launch_bounds__(kBlock) k_mvn_rvs(Philox key, uint64_t call, MvnParams P,
                                                   const double *__restrict__ loc,
                                                   const double *__restrict__ scale,
                                                   const double *__restrict__ z_in,
                                                   double *__restrict__ out, int64_t n) {
    const int d = P.d;
    const int64_t npairs = (n + 1) >> 1;
    const int64_t stride = (int64_t)gridDim.x * kBlock;
    for (int64_t p = (int64_t)blockIdx.x * kBlock + threadIdx.x; p < npairs; p += stride) {
        double z[2][kMaxDim];
        for (int k = 0; k < d; k++) {
            if (z_in) {
                z[0][k] = z_in[(size_t)k * n + 2 * p];
                z[1][k] = (2 * p + 1 < n) ? z_in[(size_t)k * n + 2 * p + 1] : 0.0;
            } else {
                uint32_t r[4];
                philox4x32_10((uint32_t)p, (uint32_t)((uint64_t)p >> 32), (uint32_t)call,
                              ((uint32_t)(call >> 32) << 16) | ((uint32_t)k << 8) | kPurposeApi,
                              key.k0, key.k1, r);
                box_muller(r, z[0][k], z[1][k]);
            }
        }
#pragma unroll
        for (int j = 0; j < 2; j++) {
            const int64_t i = 2 * p + j;
            if (i >= n) continue;
            for (int a = 0; a < d; a++) {
                double acc = 0.0;
                for (int b = 0; b <= a; b++) acc += z[j][b] * P.L[a * kMaxDim + b];
                const double l = loc ? loc[(size_t)a * n + i] : P.loc0[a];
                const double s = scale ? scale[(size_t)a * n + i] : P.scale0[a];
                out[(size_t)a * n + i] = l + s * acc;
            }
        }
    }
}

// MvNormal.logpdf (distributions.py:949-959): forward substitution with L
__global__ void __launch_bounds__(kBlock) k_mvn_logpdf(MvnParams P, const double *__restrict__ x,
                                                      const double *__restrict__ loc,
                                                      const double *__restrict__ scale,
                                                      double *__restrict__ out, int64_t n) {
    const int d = P.d;
    const int64_t stride = (int64_t)gridDim.x * kBlock;
    for (int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x; i < n; i += stride) {
        double z[kMaxDim];
        double ss = 0.0, logdet = 0.0;
        for (int a = 0; a < d; a++) {
            const double l = loc ? loc[(size_t)a * n + i] : P.loc0[a];
            const double s = scale ? scale[(size_t)a * n + i] : P.scale0[a];
            double acc = (x[(size_t)a * n + i] - l) / s;
            for (int b = 0; b < a; b++) acc -= P.L[a * kMaxDim + b] * z[b];
            z[a] = acc / P.L[a * kMaxDim + a];
            ss += z[a] * z[a];
            logdet += log(s);
        }
        out[i] = -0.5 * ss - (logdet + P.halflogdet) - (double)d * kHalfLog2Pi;
    }
}

static int fill_mvn(MvnParams *P, const double *loc0, const double *scale0, const double *L, int d) {
    SMCB_REQUIRE(d >= 1 && d <= kMaxDim, "MvNormal: dimension %d not in [1, %d]", d, kMaxDim);
    SMCB_REQUIRE(L != nullptr, "MvNormal: L is NULL");
    memset(P, 0, sizeof(*P));
    P->d = d;
    double hl = 0.0;
    for (int a = 0; a < d; a++) {
        for (int b = 0; b < d; b++) P->L[a * kMaxDim + b] = L[a * d + b];
        SMCB_REQUIRE(L[a * d + a] > 0.0, "MvNormal: argument cov must be a (d, d) pos. definite matrix");
        hl += log(L[a * d + a]);
        P->loc0[a] = loc0 ? loc0[a] : 0.0;
        P->scale0[a] = scale0 ? scale0[a] : 1.0;
    }
    P->halflogdet = hl;
    return SMCB_OK;
}

// ---------------------------------------------------------------------------
// 8 < d <= 32: the factor L (8 KB at d = 32) no longer fits the kernel parameters: it is staged in shared memory
// (with 1 / L_aa next to it), one particle per thread, z kept in registers through fully unrolled, predicated loops.
// No tensor cores, and that is a measured decision, not an omission: the Cholesky matvec costs d (d + 1) / 2 fp64 FMAs
// per particle against 16 d bytes of compulsory traffic (loc in, x out) -- (d + 1) / 32 FMA per byte, 1.03 at
// d = 32 -- while an H100 SXM is rated (data sheet) at 17e12 fp64 FMA/s per 3.35e12 B/s of HBM3 = 5 FMA/B.
// The kernel is HBM-bound at every d <= 32; fp64 DMMA doubles the FMA rate but cannot move the HBM bound, so a
// tensor-core formulation would not make it faster.
// ---------------------------------------------------------------------------
constexpr int kBigDim = 32;

struct MvnBig {
    const double *L;        // device: d x d row-major lower factor, then d reciprocals of the diagonal
    const double *loc0;     // device: d (or NULL)
    const double *scale0;   // device: d (or NULL)
    double halflogdet;
    int d;
};

template <bool LOGPDF>
__global__ void __launch_bounds__(kBlock) k_mvn_big(Philox key, uint64_t call, MvnBig P, const double *__restrict__ xin,
                                                   const double *__restrict__ loc, const double *__restrict__ scale,
                                                   const double *__restrict__ z_in, double *__restrict__ out, int64_t n) {
    __shared__ double sL[kBigDim * kBigDim + 3 * kBigDim];
    const int d = P.d;
    for (int e = threadIdx.x; e < d * d + d; e += kBlock) sL[e] = P.L[e];
    double *sInv = sL + d * d, *sLoc = sInv + kBigDim, *sSc = sLoc + kBigDim;
    for (int e = threadIdx.x; e < d; e += kBlock) { sLoc[e] = P.loc0 ? P.loc0[e] : 0.0; sSc[e] = P.scale0 ? P.scale0[e] : 1.0; }
    __syncthreads();
    const int64_t stride = (int64_t)gridDim.x * kBlock;
    for (int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x; i < n; i += stride) {
        double z[kBigDim];
        if (!LOGPDF) {
#pragma unroll
            for (int k = 0; k < kBigDim; k += 2) {
                if (k < d) {
                    if (z_in) {
                        z[k] = z_in[(size_t)k * n + i];
                        z[k + 1] = (k + 1 < d) ? z_in[(size_t)(k + 1) * n + i] : 0.0;
                    } else {                       // one Philox block -> components k, k + 1 of particle i
                        uint32_t r[4];
                        philox4x32_10((uint32_t)i, (uint32_t)((uint64_t)i >> 32), (uint32_t)call,
                                      ((uint32_t)(call >> 32) << 16) | ((uint32_t)(k >> 1) << 8) | kPurposeApi, key.k0, key.k1, r);
                        box_muller(r, z[k], z[k + 1]);
                    }
                } else { z[k] = 0.0; z[k + 1] = 0.0; }
            }
#pragma unroll
            for (int a = 0; a < kBigDim; a++) {
                if (a < d) {
                    double acc = 0.0;
#pragma unroll
                    for (int b = 0; b < kBigDim; b++)
                        if (b <= a) acc += z[b] * sL[a * d + b];
                    const double l = loc ? loc[(size_t)a * n + i] : sLoc[a];
                    const double s = scale ? scale[(size_t)a * n + i] : sSc[a];
                    out[(size_t)a * n + i] = l + s * acc;
                }
            }
        } else {
            double ss = 0.0, logdet = 0.0;
#pragma unroll
            for (int a = 0; a < kBigDim; a++) {
                if (a < d) {
                    const double l = loc ? loc[(size_t)a * n + i] : sLoc[a];
                    const double s = scale ? scale[(size_t)a * n + i] : sSc[a];
                    double acc = (xin[(size_t)a * n + i] - l) / s;
#pragma unroll
                    for (int b = 0; b < kBigDim; b++)
                        if (b < a) acc -= sL[a * d + b] * z[b];
                    z[a] = acc / sL[a * d + a];
                    ss += z[a] * z[a];
                    if (scale) logdet += log(s);
                } else z[a] = 0.0;
            }
            if (!scale) for (int a = 0; a < d; a++) logdet += log(sSc[a]);
            out[i] = -0.5 * ss - (logdet + P.halflogdet) - (double)d * kHalfLog2Pi;
        }
    }
}

// stage L (+ reciprocal diagonal), loc0, scale0 in the context's workspace (stream-ordered copies)
static int fill_mvn_big(smcb_ctx *c, MvnBig *P, const double *loc0, const double *scale0, const double *L, int d) {
    SMCB_REQUIRE(d > kMaxDim && d <= kBigDim, "MvNormal: dimension %d not in [1, %d]", d, kBigDim);
    SMCB_REQUIRE(L != nullptr, "MvNormal: L is NULL");
    double h[kBigDim * kBigDim + 3 * kBigDim];
    double hl = 0.0;
    for (int a = 0; a < d; a++) {
        for (int b = 0; b < d; b++) h[a * d + b] = (b <= a) ? L[a * d + b] : 0.0;
        SMCB_REQUIRE(L[a * d + a] > 0.0, "MvNormal: argument cov must be a (d, d) pos. definite matrix");
        hl += log(L[a * d + a]);
        h[d * d + a] = 1.0 / L[a * d + a];
        h[d * d + d + a] = loc0 ? loc0[a] : 0.0;
        h[d * d + 2 * d + a] = scale0 ? scale0[a] : 1.0;
    }
    double *w = c->ws + 4096;            // clear of the control-plane scratch at the start of the workspace
    // the workspace copy must not race with a previous call still reading it on the stream
    SMCB_CUDA(cudaStreamSynchronize(c->stream));
    SMCB_CUDA(cudaMemcpyAsync(w, h, sizeof(double) * (d * d + 3 * d), cudaMemcpyHostToDevice, c->stream));
    P->L = w; P->loc0 = w + d * d + d; P->scale0 = w + d * d + 2 * d; P->halflogdet = hl; P->d = d;
    return SMCB_OK;
}

extern "C" int smcb_mvnormal_rvs(smcb_ctx *c, const double *loc, const double *loc0,
                                 const double *scale, const double *scale0, const double *L, int d,
                                 const double *z_in, double *out, int64_t n) {
    SMCB_REQUIRE(c && out && n >= 1, "smcb_mvnormal_rvs: bad argument");
    uint64_t call = z_in ? 0 : c->api_counter++;
    if (d > kMaxDim) {
        MvnBig B;
        int rc = fill_mvn_big(c, &B, loc0, scale0, L, d);
        if (rc) return rc;
        return launch(c, k_mvn_big<false>, grid_for(n, kBlock), kBlock, 0, key_of(c->seed), call, B,
                      (const double *)nullptr, loc, scale, z_in, out, n);
    }
    MvnParams P;
    int rc = fill_mvn(&P, loc0, scale0, L, d);
    if (rc) return rc;
    return launch(c, k_mvn_rvs, grid_for((n + 1) / 2, kBlock * 2), kBlock, 0, key_of(c->seed), call, P, loc, scale,
                  z_in, out, n);
}

extern "C" int smcb_mvnormal_logpdf(smcb_ctx *c, const double *x, const double *loc,
                                    const double *loc0, const double *scale, const double *scale0,
                                    const double *L, int d, double *out, int64_t n) {
    SMCB_REQUIRE(c && x && out && n >= 1, "smcb_mvnormal_logpdf: bad argument");
    if (d > kMaxDim) {
        MvnBig B;
        int rc = fill_mvn_big(c, &B, loc0, scale0, L, d);
        if (rc) return rc;
        return launch(c, k_mvn_big<true>, grid_for(n, kBlock), kBlock, 0, key_of(c->seed), 0ull, B, x, loc, scale,
                      (const double *)nullptr, out, n);
    }
    MvnParams P;
    int rc = fill_mvn(&P, loc0, scale0, L, d);
    if (rc) return rc;
    return launch(c, k_mvn_logpdf, grid_for(n, kBlock * 2), kBlock, 0, P, x, loc, scale, out, n);
}

// ---------------------------------------------------------------------------
// test hook: evaluate the kernels' fp64 elementary functions (smcb_math.cuh) on an array
// fn: 0 fexp, 1 flog_pos, 2 sin(2 pi u), 3 cos(2 pi u)            (polynomial family)
//     4 texp, 5 tlog_pos, 6 sin(2 pi u), 7 cos(2 pi u), 8 tsqrt_pos (table family of the step kernels)
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlock) k_device_math(int fn, const double *__restrict__ x,
                                                       double *__restrict__ out, int64_t n, const double *tab) {
    __shared__ __align__(8) uint64_t s_bar;
    if (fn >= 4) {
        if (threadIdx.x == 0) mtab_issue(tab, &s_bar);
        __syncthreads();
        mbar_wait(&s_bar, 0);
    }
    const int64_t stride = (int64_t)gridDim.x * kBlock;
    for (int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x; i < n; i += stride) {
        const double v = x[i];
        double r, s, c;
        if (fn == 0) r = fexp(v);
        else if (fn == 1) r = flog_pos(v);
        else if (fn == 2 || fn == 3) { fsincos2pi(v, s, c); r = (fn == 2) ? s : c; }
        else if (fn == 4) r = texp(v);
        else if (fn == 5) r = tlog_pos(v);
        else if (fn == 8) r = tsqrt_pos(v);
        else { tsincos2pi(v, s, c); r = (fn == 6) ? s : c; }
        out[i] = r;
    }
}

extern "C" int smcb_device_math(smcb_ctx *c, int fn, const double *x, double *out, int64_t n) {
    SMCB_REQUIRE(c && x && out && n >= 1 && fn >= 0 && fn <= 8, "smcb_device_math: bad argument");
    static bool attr_set = false;
    if (!attr_set) {
        SMCB_TRY(set_smem(k_device_math, kMathTabBytes));
        attr_set = true;
    }
    return launch(c, k_device_math, grid_for(n, kBlock * 4), kBlock, fn >= 4 ? kMathTabBytes : 0, fn, x, out, n,
                  c->math_tab);
}
