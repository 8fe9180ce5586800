// smcb_variance.cu -- the genealogy-based variance estimators (particles/variance_estimators.py:93-201) on the device:
//   EVE     B_t = B_{t-1}[A_t] into the other half of a ping-pong pair, only when the step resampled (the flag is read
//           on the device, so a non-resampling step costs one tiny launch and no traffic);
//   SUMS    sum_b (sum_{m: B_m = b} v_m)^2 over sorted rows, four launches:
//           k_var_p1   per chunk of kVarChunk particles: the max-shifted (max, sum e, sum e phi_c), e = exp(lw - max);
//           k_var_f1   one CTA: merges the chunk triples into (max, S, m_c = sum e phi_c / S);
//           k_var_p2   per chunk, row and component: v = W (phi_c - m_c) or W, folded into a VarSeg (smcb_variance.cuh);
//           k_var_f2   one CTA: merges the chunk segments, applies the B[0] == B[N-1] rule and the "not sorted" flag,
//                      writes out[r, c], and flips the Eve parity.
// Every reduction runs in an order fixed by N: kVarChunk is a constant, each thread's share of a chunk is fixed (in
// pass 2 kVarPer contiguous elements, folded in index order), and the merges are pairwise trees over fixed positions.
#include "smcb_common.cuh"
#include "smcb_variance.cuh"

using namespace smcb;

namespace {

constexpr int kVarThreads = 256;
constexpr int kVarPer = 8;                                   // contiguous elements per thread
constexpr int64_t kVarChunk = (int64_t)kVarThreads * kVarPer;
constexpr int kVarFin = 512;                                 // threads of the one-CTA merges
constexpr int kVarRec1 = 3;                                  // doubles per pass-1 record: max, sum e, sum e phi
constexpr int kVarRec2 = (int)(sizeof(VarSeg) / sizeof(double));
static_assert(sizeof(VarSeg) % sizeof(double) == 0, "VarSeg is a whole number of doubles");

int64_t n_chunks(int64_t N) { return (N + kVarChunk - 1) / kVarChunk; }

struct Lse1 {
    double m, s, p;            // max, sum exp(v - m), sum exp(v - m) phi
};

__device__ __forceinline__ Lse1 lse1_merge(const Lse1 &a, const Lse1 &b) {
    if (b.m == -CUDART_INF) return a;
    if (a.m == -CUDART_INF) return b;
    const double M = fmax(a.m, b.m);
    const double ea = exp(a.m - M), eb = exp(b.m - M);
    return Lse1{M, a.s * ea + b.s * eb, a.p * ea + b.p * eb};
}

// the Eve row of this step; B[0] when there is no parity word
__device__ __forceinline__ const int64_t *cur_rows(const smcb_variance_desc &d) {
    if (!d.parity) return d.B[0];
    const int rs = d.rs_flag ? (*d.rs_flag != 0.0) : (d.rs_host != 0);
    return d.B[(*d.parity ^ rs) & 1];
}

__global__ void __launch_bounds__(kBlock) k_var_eve(smcb_variance_desc d) {
    if (d.rs_flag ? *d.rs_flag == 0.0 : d.rs_host == 0) return;
    const int p = d.parity ? (*d.parity & 1) : 0;
    const int64_t *src = d.B[p];
    int64_t *dst = d.B[p ^ 1];
    for (int64_t n = (int64_t)blockIdx.x * kBlock + threadIdx.x; n < d.N; n += (int64_t)gridDim.x * kBlock)
        dst[n] = src[d.A[n]];
}

// pairwise tree over smem[0, n), the order of varseg_tree: level w merges positions i and i + w, i a multiple of 2w
template <class R, class F>
__device__ __forceinline__ void block_tree(R *rec, int n, F merge) {
    for (int w = 1; w < n; w <<= 1) {
        __syncthreads();
        const int i = 2 * w * (int)threadIdx.x;
        if (i + w < n) rec[i] = merge(rec[i], rec[i + w]);
    }
    __syncthreads();
}

// pass 1: blockIdx.x = chunk, blockIdx.y = component
__global__ void __launch_bounds__(kVarThreads) k_var_p1(smcb_variance_desc d, double *rec1) {
    __shared__ Lse1 s_rec[kVarThreads];
    const int64_t c = blockIdx.y, k = d.k;
    const int64_t i0 = (int64_t)blockIdx.x * kVarChunk + threadIdx.x;
    // all loads first, then the thread's max and ONE exp per element: no dependent chain between the elements
    double v[kVarPer];
    double mx = -CUDART_INF;
#pragma unroll
    for (int j = 0; j < kVarPer; j++) {
        const int64_t i = i0 + (int64_t)j * kVarThreads;      // coalesced: the order is still fixed by N
        v[j] = i < d.N ? d.lw[i] : (d.lin_w ? 0.0 : -CUDART_INF);
        mx = fmax(mx, v[j]);
    }
    auto f = [&](int j) {
        const int64_t i = i0 + (int64_t)j * kVarThreads;
        return (i < d.N && d.phi) ? d.phi[i * k + c] : 0.0;
    };
    Lse1 a{-CUDART_INF, 0.0, 0.0};
    if (d.lin_w) {                                          // W given: sum W, sum W phi (no shift)
        a.m = 0.0;
#pragma unroll
        for (int j = 0; j < kVarPer; j++) {
            a.s += v[j];
            a.p += v[j] * f(j);
        }
    } else if (mx > -CUDART_INF) {
        a.m = mx;
#pragma unroll
        for (int j = 0; j < kVarPer; j++) {
            const double e = exp(v[j] - mx);                // exp(-inf) = 0
            a.s += e;
            a.p += e * f(j);
        }
    }
    s_rec[threadIdx.x] = a;
    block_tree(s_rec, kVarThreads, lse1_merge);
    if (threadIdx.x == 0) {
        double *r = rec1 + ((int64_t)c * gridDim.x + blockIdx.x) * kVarRec1;
        r[0] = s_rec[0].m;
        r[1] = s_rec[0].s;
        r[2] = s_rec[0].p;
    }
}

// pass-1 merge: one CTA, component by component; stats[c] = {max, S, m_c}
__global__ void __launch_bounds__(kVarFin) k_var_f1(smcb_variance_desc d, const double *rec1, int64_t nch,
                                                    double *stats) {
    __shared__ Lse1 s_rec[kVarFin];
    const int64_t per = (nch + kVarFin - 1) / kVarFin;
    for (int64_t c = 0; c < d.k; c++) {
        Lse1 a{-CUDART_INF, 0.0, 0.0};
        for (int64_t j = (int64_t)threadIdx.x * per; j < min(nch, (int64_t)(threadIdx.x + 1) * per); j++) {
            const double *r = rec1 + (c * nch + j) * kVarRec1;
            a = lse1_merge(a, Lse1{r[0], r[1], r[2]});
        }
        s_rec[threadIdx.x] = a;
        block_tree(s_rec, kVarFin, lse1_merge);
        if (threadIdx.x == 0) {
            stats[3 * c] = d.lin_w ? 0.0 : s_rec[0].m;
            stats[3 * c + 1] = s_rec[0].s;
            stats[3 * c + 2] = s_rec[0].p / s_rec[0].s;     // np.average(phi, weights=W)
        }
        __syncthreads();
    }
}

__device__ __forceinline__ VarSeg seg_merge(const VarSeg &a, const VarSeg &b) { return varseg_merge(a, b); }

// pass 2: blockIdx.x = chunk, blockIdx.y = row * k + component.  The chunk is staged in shared memory by coalesced
// loads (one pad slot per kVarPer elements keeps the folds' strided reads off a single bank), then thread j folds
// elements [j * kVarPer, (j + 1) * kVarPer) in index order and the CTA merges the thread segments by a fixed tree.
constexpr int kVarPad = kVarChunk + kVarChunk / kVarPer;
constexpr int kVarStage = kVarPad * (int)(sizeof(double) + sizeof(int64_t));
constexpr int kVarP2Smem = kVarStage > kVarThreads * (int)sizeof(VarSeg) ? kVarStage : kVarThreads * (int)sizeof(VarSeg);

__global__ void __launch_bounds__(kVarThreads) k_var_p2(smcb_variance_desc d, const double *stats, double *rec2) {
    __shared__ __align__(16) unsigned char s_raw[kVarP2Smem];
    double *s_v = reinterpret_cast<double *>(s_raw);
    int64_t *s_b = reinterpret_cast<int64_t *>(s_raw + kVarPad * sizeof(double));
    VarSeg *s_rec = reinterpret_cast<VarSeg *>(s_raw);
    const int64_t k = d.k, N = d.N;
    const int64_t r = blockIdx.y / k, c = blockIdx.y % k;
    const int64_t *B = cur_rows(d) + r * N;
    const double *lw = d.lw_rows + r * d.row_ld;
    const double *phi = d.phi_rows ? d.phi_rows + r * d.row_ld * k : nullptr;
    const double mx = stats[3 * c], S = stats[3 * c + 1], m = stats[3 * c + 2];
    const bool centred = d.mode == SMCB_VAR_CENTRED;
    const int64_t base = (int64_t)blockIdx.x * kVarChunk;
    const int n = (int)min((int64_t)kVarChunk, N - base);
#pragma unroll
    for (int j = 0; j < kVarPer; j++) {
        const int e = j * kVarThreads + threadIdx.x;
        if (e < n) {
            const int64_t i = base + e;
            // W = exp(lw - max) / S as exp_and_normalise; var_estimate's W are used as given
            const double W = d.lin_w ? lw[i] : exp(lw[i] - mx) / S;
            s_v[e + e / kVarPer] = centred ? W * (phi[i * k + c] - m) : W;
            s_b[e + e / kVarPer] = B[i];
        }
    }
    __syncthreads();
    VarSeg s = varseg_empty();
    const int e0 = threadIdx.x * kVarPer;
#pragma unroll
    for (int j = 0; j < kVarPer; j++) {
        const int e = e0 + j;
        if (e < n) s = varseg_merge(s, varseg_leaf(s_b[e + e / kVarPer], s_v[e + e / kVarPer]));
    }
    __syncthreads();                                         // s_rec reuses the staging buffer
    s_rec[threadIdx.x] = s;
    block_tree(s_rec, kVarThreads, seg_merge);
    if (threadIdx.x == 0) {
        VarSeg *o = reinterpret_cast<VarSeg *>(rec2) + (int64_t)blockIdx.y * gridDim.x + blockIdx.x;
        *o = s_rec[0];
    }
}

// pass-2 merge: one CTA, (row, component) by (row, component)
__global__ void __launch_bounds__(kVarFin) k_var_f2(smcb_variance_desc d, const double *rec2, int64_t nch) {
    __shared__ VarSeg s_rec[kVarFin];
    const int64_t per = (nch + kVarFin - 1) / kVarFin;
    const VarSeg *recs = reinterpret_cast<const VarSeg *>(rec2);
    for (int64_t rc = 0; rc < d.L * d.k; rc++) {
        VarSeg a = varseg_empty();
        for (int64_t j = (int64_t)threadIdx.x * per; j < min(nch, (int64_t)(threadIdx.x + 1) * per); j++)
            a = varseg_merge(a, recs[rc * nch + j]);
        s_rec[threadIdx.x] = a;
        block_tree(s_rec, kVarFin, seg_merge);
        if (threadIdx.x == 0) {
            const VarSeg &t = s_rec[0];
            const int64_t r = rc / d.k;
            bool zero = false;
            if (d.mode == SMCB_VAR_CENTRED) zero = d.zero ? d.zero[r] != 0 : t.b0 == t.b1;   // B[0] == B[-1]
            d.out[rc] = zero ? 0.0 : varseg_total(t);
            if (t.bad) d.unsorted[r] = 1;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0 && d.parity) {
        const int rs = d.rs_flag ? (*d.rs_flag != 0.0) : (d.rs_host != 0);
        *d.parity ^= rs;
    }
}

}  // namespace

extern "C" int64_t smcb_variance_scratch_doubles(int64_t N, int64_t L, int64_t k) {
    const int64_t nch = n_chunks(N);
    return 3 * k + kVarRec1 * k * nch + (int64_t)kVarRec2 * L * k * nch;
}

extern "C" int smcb_variance(smcb_ctx *c, const smcb_variance_desc *dp) {
    SMCB_REQUIRE(c && dp, "smcb_variance: NULL argument");
    const smcb_variance_desc &d = *dp;
    SMCB_REQUIRE(d.N >= 1, "smcb_variance: bad N=%lld", (long long)d.N);
    SMCB_REQUIRE(d.B[0] && (!d.parity || d.B[1]), "smcb_variance: NULL Eve rows");
    if (d.method == SMCB_VAR_EVE) {
        SMCB_REQUIRE(d.parity && d.A, "smcb_variance: EVE needs the parity word and the ancestors");
        return launch(c, k_var_eve, grid_for(d.N, kBlock), kBlock, 0, d);
    }
    SMCB_REQUIRE(d.method == SMCB_VAR_SUMS, "smcb_variance: bad method %d", (int)d.method);
    SMCB_REQUIRE(d.mode == SMCB_VAR_CENTRED || d.mode == SMCB_VAR_WEIGHTS, "smcb_variance: bad mode %d", (int)d.mode);
    SMCB_REQUIRE(d.k >= 1 && d.L >= 1 && d.L * d.k <= 65535, "smcb_variance: bad shape L=%lld k=%lld",
                 (long long)d.L, (long long)d.k);
    SMCB_REQUIRE(d.mode == SMCB_VAR_WEIGHTS ? d.k == 1 : (d.phi && d.phi_rows), "smcb_variance: phi and mode disagree");
    SMCB_REQUIRE(d.lw && d.lw_rows && d.row_ld >= 0 && d.unsorted && d.scratch && d.out,
                 "smcb_variance: NULL argument");
    SMCB_REQUIRE(!d.lin_w || d.mode == SMCB_VAR_CENTRED, "smcb_variance: linear weights in CENTRED mode only");
    const int64_t nch = n_chunks(d.N);
    SMCB_REQUIRE(nch <= 0x7fffffffLL, "smcb_variance: N too large");
    double *stats = d.scratch, *rec1 = stats + 3 * d.k, *rec2 = rec1 + kVarRec1 * d.k * nch;
    SMCB_TRY(launch(c, k_var_p1, dim3((unsigned)nch, (unsigned)d.k), kVarThreads, 0, d, rec1));
    SMCB_TRY(launch(c, k_var_f1, 1, kVarFin, 0, d, rec1, nch, stats));
    SMCB_TRY(launch(c, k_var_p2, dim3((unsigned)nch, (unsigned)(d.L * d.k)), kVarThreads, 0, d, stats, rec2));
    return launch(c, k_var_f2, 1, kVarFin, 0, d, rec2, nch);
}
