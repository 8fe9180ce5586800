// smcb_binary.cu -- SMC samplers on {0,1}^p (particles/binary_smc.py; Schäfer & Chopin 2013, waste-free moves of
// Dau & Chopin 2022): Bayesian variable selection with a nested-logistic independent Metropolis move.
//
//   smcb_vs_loglik        chol_and_friends (binary_smc.py:165-180) and the loglik of BIC / BayesianVS /
//                         BayesianVS_gprior (216-293), plus the IID(Bernoulli(q), p) prior and the tempered target,
//                         for n particles.  One WARP per particle: the selected columns of X^T X (ascending, as the
//                         reference's boolean indexing takes them) are gathered into a packed lower triangle in
//                         shared memory, with X^T y[gamma] appended as one more row, and factored in place by a
//                         right-looking warp-cooperative Cholesky.  The appended row ends up holding w = L^-1 X^T y,
//                         so the triangular solve costs nothing extra.
//   smcb_nested_logistic  NestedLogistic.rvs / logpdf (binary_smc.py:98-118): one thread per particle, the bits of a
//                         particle packed in four registers, coordinates in order.
//   smcb_binary_wf_move   MCMCSequenceWF.__call__ (smc_samplers.py:672-683) with the BinaryMetropolis step
//                         (binary_smc.py:154-162 + smc_samplers.py:601-611): all P-1 steps of all M chains in one
//                         launch, one warp per chain.  Lane l owns the coordinates l, l + 32, l + 64, l + 96, so the
//                         nested-logistic dot product of coordinate i is a warp sum and the owner of i draws its bit.
//
// Shared memory per warp is (k + 1)(k + 2) / 2 doubles for |gamma| <= k (k = the batch's largest |gamma| for
// smcb_vs_loglik, k = p for the move, whose proposals may select anything): p <= 128 keeps at least three warps in a
// CTA.  A pivot that is not positive (where scipy.linalg.cholesky raises LinAlgError) gives llik = -inf and sets
// bit 0 of *err; it never yields a NaN silently.  All arithmetic is fp64.
#include "smcb_common.cuh"
#include "smcb_reduce.cuh"

using namespace smcb;

namespace smcb {

constexpr int kBinMaxP = 128;
constexpr int kBinWords = kBinMaxP / 32;
constexpr int kBinThreads = 128;                   // smcb_nested_logistic
constexpr size_t kBinSmemBudget = 200 * 1024;      // of the 227 KB a CTA may use

__host__ __device__ __forceinline__ int tri(int a) { return a * (a + 1) / 2; }

__device__ __forceinline__ double log_no_warn(double x) { return log(x > 1e-300 ? x : 1e-300); }   // :62-64
__device__ __forceinline__ double expit(double x) { return 1.0 / (1.0 + exp(-x)); }

// the uniform of coordinate i of particle / chain n at step s (s = 0: smcb_nested_logistic)
__device__ __forceinline__ double bin_uniform(const Philox &key, uint64_t n, uint64_t call, int s, int i,
                                              uint32_t purpose) {
    uint32_t r[4];
    philox4x32_10k((uint32_t)n, (uint32_t)(n >> 32), (uint32_t)call,
                   ((uint32_t)s << 16) | ((uint32_t)i << 8) | purpose, key, r);
    return u53(r[0], r[1]);
}

// IID(Bernoulli(q), p).logpdf: IndepProd sums the p coordinates' terms in order (distributions.py:1101-1102)
__device__ __forceinline__ double iid_prior(const smcb_vs_desc &m, const uint32_t mask[kBinWords]) {
    double lp = 0.0;
    for (int i = 0; i < m.p; i++) lp += ((mask[i >> 5] >> (i & 31)) & 1u) ? m.lq : m.l1q;
    return lp;
}

// chol_and_friends for the gamma whose coordinate masks (bit l of mask[w] = gamma[32 w + l]) every lane holds.
// A: this warp's (k + 1)(k + 2) / 2 doubles, idx: its kBinMaxP ints.  Returns |gamma| and, in every lane, ldet and
// wtw; ok = false on a non-positive pivot.
__device__ int vs_chol(const smcb_vs_desc &m, const uint32_t mask[kBinWords], double vm2, double *A, int *idx,
                       double &ldet, double &wtw, bool &ok) {
    const int lane = threadIdx.x & 31;
    int k = 0;
#pragma unroll
    for (int w = 0; w < kBinWords; w++) {
        if ((mask[w] >> lane) & 1u) idx[k + __popc(mask[w] & ((1u << lane) - 1u))] = 32 * w + lane;
        k += __popc(mask[w]);
    }
    ldet = 0.0; wtw = 0.0; ok = true;
    if (k == 0) return 0;
    __syncwarp();
    // the augmented lower triangle, row-major packed: rows 0..k-1 = X^T X[gamma, gamma] + vm2 I, row k = X^T y[gamma]
    // (its diagonal is never read)
    const int tot = tri(k + 1) - 1;
    int a = 0, b = lane;
    while (b > a) { b -= a + 1; a++; }
    for (int e = lane; e < tot; e += 32) {
        double v;
        if (a < k) {
            v = m.xtx[(int64_t)idx[a] * m.p + idx[b]];
            if (a == b) v += vm2;
        } else {
            v = m.xty[idx[b]];
        }
        A[e] = v;
        b += 32;
        while (b > a) { b -= a + 1; a++; }
    }
    __syncwarp();
    for (int j = 0; j < k; j++) {
        const double piv = A[tri(j) + j];
        if (!(piv > 0.0)) { ok = false; break; }            // warp-uniform
        const double ljj = sqrt(piv);
        ldet += log(ljj);
        for (int i = j + 1 + lane; i <= k; i += 32) A[tri(i) + j] /= ljj;
        __syncwarp();
        // trailing update of rows j+1..k, columns j+1..row (row k: columns j+1..k-1)
        const int mm = k - j;
        int r = 0, c = lane;
        while (c > r) { c -= r + 1; r++; }
        for (int t = lane; t < tri(mm); t += 32) {
            const int i = j + 1 + r, l = j + 1 + c;
            if (l < k) A[tri(i) + l] -= A[tri(i) + j] * A[tri(l) + j];
            c += 32;
            while (c > r) { c -= r + 1; r++; }
        }
        __syncwarp();
    }
    if (!ok) return k;
    double s = 0.0;
    for (int b2 = lane; b2 < k; b2 += 32) { const double w = A[tri(k) + b2]; s += w * w; }
    wtw = warp_sum(s);
    return k;
}

// loglik of the three models (binary_smc.py:227-230, 258-265, 287-293), -inf where the factorisation failed
__device__ __forceinline__ double vs_loglik_of(const smcb_vs_desc &m, int k, double ldet, double wtw, bool ok) {
    if (!ok) return -CUDART_INF;
    const double in_log = m.coef_in_log - m.gw * wtw;     // gw = 1 except for the g-prior (gogp1)
    const double lead = m.coef_len * (double)k;
    const double s = m.use_ldet ? lead + ldet + m.coef_log * log(in_log) : lead + m.coef_log * log(in_log);
    return -s;
}

// the masks of a bool row
__device__ __forceinline__ void load_mask(const uint8_t *row, int p, uint32_t mask[kBinWords]) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int w = 0; w < kBinWords; w++) {
        const int j = 32 * w + lane;
        mask[w] = __ballot_sync(0xffffffffu, j < p && row[j] != 0);
    }
}

__global__ void k_vs_loglik(smcb_vs_desc m, const uint8_t *__restrict__ gamma, int64_t n, int kmax, double vm2,
                            double epn, double *len_gam, double *ldet_out, double *wtw_out, double *lprior,
                            double *llik, double *lpost, int *err) {
    extern __shared__ __align__(16) double s_bin[];
    const int wpc = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double *A = s_bin + (size_t)warp * tri(kmax + 1);
    int *idx = reinterpret_cast<int *>(s_bin + (size_t)wpc * tri(kmax + 1)) + warp * kBinMaxP;
    const int64_t i = (int64_t)blockIdx.x * wpc + warp;
    if (i >= n) return;                                      // warp-uniform
    uint32_t mask[kBinWords];
    load_mask(gamma + i * m.p, m.p, mask);
    int k = 0;
#pragma unroll
    for (int w = 0; w < kBinWords; w++) k += __popc(mask[w]);
    double ldet = 0.0, wtw = 0.0;
    bool ok = true;
    if (k > kmax) {                                          // the caller's bound is wrong: refuse, loudly
        if (lane == 0) atomicOr(err, 2);
        ldet = wtw = CUDART_NAN;
    } else {
        vs_chol(m, mask, vm2, A, idx, ldet, wtw, ok);
        if (!ok && lane == 0) atomicOr(err, 1);
    }
    if (lane != 0) return;
    if (len_gam) len_gam[i] = (double)k;
    if (ldet_out) ldet_out[i] = ok ? ldet : CUDART_NAN;
    if (wtw_out) wtw_out[i] = ok ? wtw : CUDART_NAN;
    if (llik) {
        const double ll = (k > kmax) ? CUDART_NAN : vs_loglik_of(m, k, ldet, wtw, ok);
        llik[i] = ll;
        if (lprior) {
            const double lp = iid_prior(m, mask);
            lprior[i] = lp;
            if (lpost) lpost[i] = (epn > 0.0) ? lp + epn * ll : lp;      // smc_samplers.py:840-843
        }
    }
}

// NestedLogistic.predict_prob (binary_smc.py:98-106) for coordinate i, given the bits of coordinates < i
__device__ __forceinline__ double nl_prob_thread(const double *__restrict__ coeffs, const uint8_t *__restrict__ edgy,
                                                 int p, int i, const uint32_t x[kBinWords]) {
    const double *ci = coeffs + (int64_t)i * p;
    if (edgy[i]) return ci[i];
    double lin = 0.0;
    for (int j = 0; j < i; j++) lin += ((x[j >> 5] >> (j & 31)) & 1u) ? ci[j] : 0.0;
    return expit(ci[i] + lin);
}

// DRAW: x := NestedLogistic.rvs (u_in (p, n) or Philox), logpdf of the draw; else logpdf of x (binary_smc.py:108-118)
template <bool DRAW>
__global__ void __launch_bounds__(kBinThreads) k_nested_logistic(int p, const double *__restrict__ coeffs,
                                                                 const uint8_t *__restrict__ edgy, int64_t n,
                                                                 uint8_t *x, const double *__restrict__ u_in,
                                                                 Philox key, uint64_t call, double *logpdf) {
    const int64_t t = (int64_t)blockIdx.x * kBinThreads + threadIdx.x;
    if (t >= n) return;
    uint32_t bits[kBinWords] = {0u, 0u, 0u, 0u};
    if (!DRAW)
        for (int j = 0; j < p; j++) bits[j >> 5] |= (x[t * p + j] ? 1u : 0u) << (j & 31);
    double lp = 0.0;
    for (int i = 0; i < p; i++) {
        const double pr = nl_prob_thread(coeffs, edgy, p, i, bits);
        bool b;
        if (DRAW) {
            const double u = u_in ? u_in[(int64_t)i * n + t] : bin_uniform(key, (uint64_t)t, call, 0, i, kPurposeBinRvs);
            b = u < pr;                                      // Bernoulli.rvs, :73-77
            bits[i >> 5] |= (b ? 1u : 0u) << (i & 31);
            x[t * p + i] = b ? 1 : 0;
        } else {
            b = (bits[i >> 5] >> (i & 31)) & 1u;
        }
        lp += b ? log_no_warn(pr) : log_no_warn(1.0 - pr);  // Bernoulli.logpdf, :79-80
    }
    if (logpdf) logpdf[t] = lp;
}

// The warp version for the fused move: lane l holds bit w of `own` = coordinate 32 w + l.  DRAW: draw the bits
// (the owner of coordinate i compares its uniform) and return the draw's logpdf; else the logpdf of `own`.
template <bool DRAW>
__device__ __forceinline__ double nl_warp(const double *__restrict__ coeffs, const uint8_t *__restrict__ edgy, int p,
                                          uint32_t &own, const double *u_own) {
    const int lane = threadIdx.x & 31;
    double lp = 0.0;
    if (DRAW) own = 0u;
    for (int i = 0; i < p; i++) {
        const double *ci = coeffs + (int64_t)i * p;
        double pr;
        if (edgy[i]) {
            pr = ci[i];
        } else {
            double part = 0.0;
#pragma unroll
            for (int w = 0; w < kBinWords; w++) {
                const int j = 32 * w + lane;
                if (j < i && ((own >> w) & 1u)) part += ci[j];
            }
            pr = expit(ci[i] + warp_sum(part));
        }
        const int owner = i & 31, w = i >> 5;
        uint32_t b;
        if (DRAW) {
            b = (lane == owner) ? (u_own[w] < pr ? 1u : 0u) : 0u;
            b = __shfl_sync(0xffffffffu, b, owner);
            if (lane == owner) own |= b << w;
        } else {
            b = __shfl_sync(0xffffffffu, (own >> w) & 1u, owner);
        }
        lp += b ? log_no_warn(pr) : log_no_warn(1.0 - pr);
    }
    return lp;
}

// One warp per chain.  Row s of the output (s = 0..P-1) holds the chains' states after s Metropolis steps.
// u_prop (P-1, p, M) / u_acc (P-1, M): the reference's order of draws (rvs coordinate by coordinate, then the
// acceptance uniforms), or NULL for Philox keyed by (chain, step, coordinate, purpose).
__global__ void k_binary_wf_move(smcb_vs_desc m, const double *__restrict__ coeffs, const uint8_t *__restrict__ edgy,
                                 int64_t M, int P, double epn, const uint8_t *__restrict__ x0,
                                 const double *__restrict__ lprior0, const double *__restrict__ llik0,
                                 const double *__restrict__ lpost0, Philox key, uint64_t call,
                                 const double *__restrict__ u_prop, const double *__restrict__ u_acc, uint8_t *x_out,
                                 double *lprior_out, double *llik_out, double *lpost_out, double *pb_out, int *err) {
    extern __shared__ __align__(16) double s_bin[];
    const int wpc = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int p = m.p;
    double *A = s_bin + (size_t)warp * tri(p + 1);
    int *idx = reinterpret_cast<int *>(s_bin + (size_t)wpc * tri(p + 1)) + warp * kBinMaxP;
    const int64_t c = (int64_t)blockIdx.x * wpc + warp;
    if (c >= M) return;                                      // warp-uniform
    uint32_t cur = 0u;                                       // this lane's bits of the chain's state
#pragma unroll
    for (int w = 0; w < kBinWords; w++) {
        const int j = 32 * w + lane;
        if (j < p && x0[c * p + j]) cur |= 1u << w;
    }
    double lpr = lprior0[c], ll = llik0[c], lp = lpost0[c];
    for (int j = lane; j < p; j += 32) x_out[c * p + j] = x0[c * p + j];
    if (lane == 0) { lprior_out[c] = lpr; llik_out[c] = ll; lpost_out[c] = lp; }
    double lq_cur = nl_warp<false>(coeffs, edgy, p, cur, nullptr);
    for (int s = 1; s < P; s++) {
        double u_own[kBinWords];
#pragma unroll
        for (int w = 0; w < kBinWords; w++) {
            const int j = 32 * w + lane;
            u_own[w] = 1.0;
            if (j < p) u_own[w] = u_prop ? u_prop[((int64_t)(s - 1) * p + j) * M + c]
                                         : bin_uniform(key, (uint64_t)c, call, s, j, kPurposeBinProp);
        }
        uint32_t prop = 0u;
        const double lq_prop = nl_warp<true>(coeffs, edgy, p, prop, u_own);
        const double delta_lp = lq_cur - lq_prop;            // BinaryMetropolis.proposal, :158-162
        uint32_t mask[kBinWords];
#pragma unroll
        for (int w = 0; w < kBinWords; w++) mask[w] = __ballot_sync(0xffffffffu, (prop >> w) & 1u);
        double ldet, wtw;
        bool ok;
        const int k = vs_chol(m, mask, m.vm2, A, idx, ldet, wtw, ok);
        if (!ok && lane == 0) atomicOr(err, 1);
        const double llp = vs_loglik_of(m, k, ldet, wtw, ok);
        const double lprp = iid_prior(m, mask);
        const double lpp = (epn > 0.0) ? lprp + epn * llp : lprp;
        const double lp_acc = lpp - lp + delta_lp;           // smc_samplers.py:606-609
        double pb = exp(fmin(lp_acc, 0.0));
        if (lp_acc != lp_acc) pb = CUDART_NAN;
        const double u = u_acc ? u_acc[(int64_t)(s - 1) * M + c] : bin_uniform(key, (uint64_t)c, call, s, 0, kPurposeBinAcc);
        if (u < pb) {                                        // warp-uniform
            cur = prop; lq_cur = lq_prop;
            lpr = lprp; ll = llp; lp = lpp;
        }
        const int64_t row = (int64_t)s * M + c;
#pragma unroll
        for (int w = 0; w < kBinWords; w++) {
            const int j = 32 * w + lane;
            if (j < p) x_out[row * p + j] = (cur >> w) & 1u;
        }
        if (lane == 0) {
            lprior_out[row] = lpr; llik_out[row] = ll; lpost_out[row] = lp;
            pb_out[(int64_t)(s - 1) * M + c] = pb;
        }
    }
}

// warps per CTA for a per-warp triangle of tri(k + 1) doubles
inline int bin_warps(int k) {
    const size_t per = (size_t)tri(k + 1) * sizeof(double) + kBinMaxP * sizeof(int);
    size_t w = kBinSmemBudget / per;
    if (w > 8) w = 8;
    return (int)w;
}

inline size_t bin_smem(int k, int wpc) {
    return (size_t)wpc * ((size_t)tri(k + 1) * sizeof(double) + kBinMaxP * sizeof(int));
}

}  // namespace smcb

static int check_desc(const smcb_vs_desc *m, const char *who) {
    SMCB_REQUIRE(m && m->xtx && m->xty, "%s: NULL model", who);
    SMCB_REQUIRE(m->p >= 1 && m->p <= kBinMaxP, "%s: p = %d outside 1..%d", who, m->p, kBinMaxP);
    return SMCB_OK;
}

extern "C" int smcb_vs_loglik(smcb_ctx *c, const smcb_vs_desc *m, const uint8_t *gamma, int64_t n, int kmax,
                              double vm2, double epn, double *len_gam, double *ldet, double *wtw, double *lprior,
                              double *llik, double *lpost, int *err) {
    SMCB_REQUIRE(c && gamma && err, "smcb_vs_loglik: NULL argument");
    if (int rc = check_desc(m, "smcb_vs_loglik")) return rc;
    SMCB_REQUIRE(n >= 1 && kmax >= 0 && kmax <= m->p, "smcb_vs_loglik: need n >= 1 and 0 <= kmax <= p");
    SMCB_REQUIRE(!lpost || (lprior && llik), "smcb_vs_loglik: lpost needs lprior and llik");
    const int wpc = bin_warps(kmax);
    const size_t smem = bin_smem(kmax, wpc);
    SMCB_TRY(set_smem(k_vs_loglik, smem));
    const int64_t grid = (n + wpc - 1) / wpc;
    SMCB_REQUIRE(grid < (1ll << 31), "smcb_vs_loglik: too many particles");
    return launch(c, k_vs_loglik, (unsigned)grid, 32 * wpc, smem, *m, gamma, n, kmax, vm2, epn, len_gam, ldet, wtw,
                  lprior, llik, lpost, err);
}

extern "C" int smcb_nested_logistic(smcb_ctx *c, int p, const double *coeffs, const uint8_t *edgy, int64_t n,
                                    int draw, uint8_t *x, const double *u_in, double *logpdf) {
    SMCB_REQUIRE(c && coeffs && edgy && x, "smcb_nested_logistic: NULL argument");
    SMCB_REQUIRE(p >= 1 && p <= kBinMaxP && n >= 1, "smcb_nested_logistic: need 1 <= p <= %d and n >= 1", kBinMaxP);
    SMCB_REQUIRE(draw || logpdf, "smcb_nested_logistic: nothing to compute");
    const int64_t grid = (n + kBinThreads - 1) / kBinThreads;
    const uint64_t call = (draw && !u_in) ? c->api_counter++ : 0;
    return launch(c, draw ? k_nested_logistic<true> : k_nested_logistic<false>, (unsigned)grid, kBinThreads, 0, p,
                  coeffs, edgy, n, x, u_in, key_of(c->seed), call, logpdf);
}

extern "C" int smcb_binary_wf_move(smcb_ctx *c, const smcb_vs_desc *m, const double *coeffs, const uint8_t *edgy,
                                   int64_t M, int P, double epn, const uint8_t *x0, const double *lprior0,
                                   const double *llik0, const double *lpost0, const double *u_prop,
                                   const double *u_acc, uint8_t *x_out, double *lprior_out, double *llik_out,
                                   double *lpost_out, double *pb_out, int *err) {
    SMCB_REQUIRE(c && coeffs && edgy && x0 && lprior0 && llik0 && lpost0 && x_out && lprior_out && llik_out &&
                     lpost_out && pb_out && err, "smcb_binary_wf_move: NULL argument");
    if (int rc = check_desc(m, "smcb_binary_wf_move")) return rc;
    SMCB_REQUIRE(M >= 1 && P >= 2 && P < 65536, "smcb_binary_wf_move: need M >= 1 and 2 <= len_chain < 65536");
    SMCB_REQUIRE((u_prop == nullptr) == (u_acc == nullptr), "smcb_binary_wf_move: inject both uniforms or neither");
    const int wpc = bin_warps(m->p);
    const size_t smem = bin_smem(m->p, wpc);
    SMCB_TRY(set_smem(k_binary_wf_move, smem));
    const int64_t grid = (M + wpc - 1) / wpc;
    const uint64_t call = u_prop ? 0 : c->api_counter++;
    return launch(c, k_binary_wf_move, (unsigned)grid, 32 * wpc, smem, *m, coeffs, edgy, M, P, epn, x0, lprior0,
                  llik0, lpost0, key_of(c->seed), call, u_prop, u_acc, x_out, lprior_out, llik_out, lpost_out, pb_out,
                  err);
}
