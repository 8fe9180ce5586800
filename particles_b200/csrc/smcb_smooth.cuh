// smcb_smooth.cuh -- device pieces shared by the backward samplers (smcb_smooth.cu) and the on-line smoothers
// (smcb_online.cu): Philox uniforms of a draw, inverse-CDF multinomial draw, online log-sum-exp, the warp-cooperative
// exact draw and one rejection trial.
//
// The history-reading helpers are templated on the descriptor.  A descriptor `d` provides the pointer tables
// d.X[t] and d.lw[t], the element strides d.x_stride_n / d.x_stride_c, the sizes d.N (particles at t), d.M (draws)
// and d.max_trials, the CDF rows d.cdf + t * d.cdf_ld, and the injected proposals / log-uniforms d.prop / d.lu laid
// out (t, M, max_trials).
//
// The rule every exact draw of a backward kernel follows (k_bs_on2, warp_exact_draw, and the plugin path of
// smoothing.py / collectors.py): with v_n = lw_t[n] + logpt(t + 1, X_t[n], x) and e_n = exp(v_n - max v), the draw is
// the first n with e_n > 0 and e_0 + ... + e_n >= u * sum e; a target above the re-summed total (round-off) gives the
// last n with e_n > 0.  A row with no positive weight (every v_n is -inf) gives 0, as the reference's
// searchsorted(cumsum(exp_and_normalise(v)), u) does on its all-NaN CDF.  A NaN v_n has weight zero here; in the
// reference it makes the whole row NaN.
#pragma once
#include "smcb_common.cuh"
#include "smcb_math.cuh"
#include "smcb_models.cuh"
#include "smcb_reduce.cuh"

namespace smcb {

constexpr int kSmBlock = 256;                  // threads per CTA; ON2: trajectories per CTA = particles per tile

__device__ __forceinline__ void smooth_uniforms(const Philox &key, uint64_t call, int64_t m, int64_t t, uint32_t trial,
                                                uint32_t purpose, double &u0, double &u1) {
    uint32_t r[4];
    philox4x32_10k((uint32_t)m, (uint32_t)t, (uint32_t)call, (trial << 8) | purpose, key, r);
    u0 = u53_open(r[0], r[1]);
    u1 = u53_open(r[2], r[3]);
}

template <int D, class Desc>
__device__ __forceinline__ void load_x(const Desc &d, int64_t t, int64_t n, double *x) {
    const double *p = d.X[t] + n * d.x_stride_n;
#pragma unroll
    for (int c = 0; c < D; c++) x[c] = p[c * d.x_stride_c];
}

// multinomial draw from an inclusive prefix sum: first j with cdf[j] >= u * cdf[N-1], u in (0, 1), so that a
// particle of weight zero is never selected
__device__ __forceinline__ int64_t draw_cdf(const double *cdf, int64_t N, double u) {
    const double v = u * cdf[N - 1];
    int64_t lo = 0, hi = N - 1;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (cdf[mid] >= v) hi = mid;
        else lo = mid + 1;
    }
    return lo;
}

// online (max, sum exp(v - max)) with ONE exp per value; -inf and NaN contribute nothing
template <bool TAB>
__device__ __forceinline__ void lse_add(double &mx, double &s, double v) {
    if (!(v > -CUDART_INF)) return;
    if (v > mx) {
        s = s * (TAB ? texp_neg(mx - v) : fexp_neg(mx - v)) + 1.0;
        mx = v;
    } else {
        s += TAB ? texp_neg(v - mx) : fexp_neg(v - mx);
    }
}

// merge the partial (mo, so) of a disjoint set of values into (mx, s): both rescaled to the larger max, so that s is
// again sum exp(v - mx); two empty partials (max -inf) stay empty.  A sum of exp(v - mx) * psi kept beside s merges
// the same way, from a copy of mx taken before.
__device__ __forceinline__ void lse_merge(double &mx, double &s, double mo, double so) {
    const double Mx = fmax(mx, mo);
    if (Mx > -CUDART_INF) {
        s = s * fexp_neg(mx - Mx) + so * fexp_neg(mo - Mx);
        mx = Mx;
    }
}

// lse_merge of the lanes' (mx, s) by the xor butterfly, strides 16 -> 1: every lane gets the same bits
__device__ __forceinline__ void warp_lse_merge(double &mx, double &s) {
#pragma unroll
    for (int mask = 16; mask > 0; mask >>= 1) {
        const double mo = __shfl_xor_sync(kFull, mx, mask), so = __shfl_xor_sync(kFull, s, mask);
        lse_merge(mx, s, mo, so);
    }
}

template <class M>
__device__ __forceinline__ void stage_tables(const double *tab, uint64_t *bar, bool needed) {
    if (needed) stage_math_tables(tab, bar);
}

// the exact draw of smoothing.py:418-421 for ONE target xs, by the whole warp:
// searchsorted(cumsum(exp_and_normalise(lw_t + logpt(t+1, X_t, xs))), u).  Pass 1: lane-strided online (max, sum)
// merged by a fixed butterfly; pass 2: chunks of 32 in index order, warp inclusive scan, first crossing.
template <class M, class Desc>
__device__ int64_t warp_exact_draw(const M &m, const TransDensity<M> &td, const Desc &d, const StepK &k,
                                   int64_t t, const double *xs, double u, int lane) {
    constexpr int D = M::D;
    const double *lw = d.lw[t];
    const int64_t N = d.N;
    auto value = [&](int64_t n) {
        double xp[D], lc[D];
        load_x<D>(d, t, n, xp);
        td.loc(m, k, xp, lc);
        return lw[n] + td.lpdf(m, lc, xs);
    };
    double mx = -CUDART_INF, s = 0.0;
    for (int64_t n = lane; n < N; n += 32) lse_add<false>(mx, s, value(n));
    warp_lse_merge(mx, s);
    const double target = u * s;
    double c = 0.0;
    int64_t last = -1;
    for (int64_t base = 0; base < N; base += 32) {
        const int64_t n = base + lane;
        double e = 0.0;
        if (n < N) {
            const double v = value(n);
            e = (v > -CUDART_INF) ? fexp_neg(v - mx) : 0.0;
        }
        double sc = e;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const double up = __shfl_up_sync(kFull, sc, o);
            if (lane >= o) sc += up;
        }
        const double cc = c + sc;
        const unsigned hit = __ballot_sync(kFull, n < N && cc >= target);
        if (hit) return base + __ffs(hit) - 1;
        const unsigned pos = __ballot_sync(kFull, e > 0.0);
        if (pos) last = base + 31 - __clz(pos);
        c = __shfl_sync(kFull, cc, 31);
    }
    // round-off: the target lies above the re-summed total -> the last particle of positive weight (an all-zero row
    // never gets here: its target is 0, which lane 0 meets at once)
    return last >= 0 ? last : 0;
}

// trial `trial` of draw jj at time t: proposal (returned in prop) and acceptance test (smoothing.py:405-410)
template <class M, class Desc>
__device__ __forceinline__ bool reject_trial(const M &m, const TransDensity<M> &td, const Desc &d,
                                             const StepK &k, const Philox &key, uint64_t call, int64_t jj, int64_t t,
                                             int64_t trial, const double *xn, double bound, int64_t &prop) {
    constexpr int D = M::D;
    double lu;
    if (d.prop) {
        const int64_t off = (t * d.M + jj) * d.max_trials + trial;
        prop = d.prop[off];
        lu = d.lu[off];
    } else {
        double u0, u1;
        smooth_uniforms(key, call, jj, t, (uint32_t)trial, kPurposeSmooth, u0, u1);
        prop = draw_cdf(d.cdf + t * d.cdf_ld, d.N, u0);
        lu = log(u1);
    }
    double xp[D], lc[D];
    load_x<D>(d, t, prop, xp);
    td.loc(m, k, xp, lc);
    return lu < td.lpdf(m, lc, xn) - bound;
}

// trials each lane runs on its own before the warp serves the lanes still rejected together
constexpr int64_t kSoloTrials = 4;

}  // namespace smcb
