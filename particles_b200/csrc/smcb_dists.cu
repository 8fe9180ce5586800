// smcb_dists.cu -- kernels and C entry points of the laws in smcb_dists.cuh, of Dirichlet, of VaryingCovNormal and of
// the row log-sum-exp behind Mixture.logpdf (particles_b200/distributions.py).  Every kernel is elementwise over the
// n particles (grid-stride); the draws follow the counters of smcb_dists.cuh.
#include "smcb_dists.cuh"

using namespace smcb;
using namespace smcb::dists;

namespace {

// a parameter: per-element array, or the scalar next to it
struct Par4 {
    const double *p[4];
    double s[4];
    __device__ __forceinline__ double operator()(int k, int64_t i) const { return p[k] ? p[k][i] : s[k]; }
};

// one instantiation per law: the law's branch is resolved at compile time, so each kernel holds only its own code.
// Two elements per pass for the continuous laws: the compiler then keeps the parameters' array-or-scalar tests on
// uniform registers instead of redoing them per element (Student, the most arithmetic per byte, is 3 % faster at
// 10^7).  The discrete laws' series loops would spill at two.
template <int LAW>
__global__ void __launch_bounds__(kBlock) k_dist_logpdf(const double *__restrict__ x, double x0, Par4 P,
                                                       double *__restrict__ out, int64_t n) {
    const int64_t stride = (int64_t)gridDim.x * kBlock;
#pragma unroll (discrete_law(LAW) ? 1 : 2)
    for (int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x; i < n; i += stride)
        out[i] = law_logpdf(LAW, x ? x[i] : x0, P(0, i), P(1, i), P(2, i), P(3, i));
}

// continuous laws write fp64, the discrete ones int64 (INT64_MIN for a NaN draw: a parameter outside the domain)
template <int LAW>
__global__ void __launch_bounds__(kBlock) k_dist_rvs(Philox key, uint64_t call, Par4 P, void *__restrict__ out,
                                                    int64_t n) {
    const int64_t stride = (int64_t)gridDim.x * kBlock;
    for (int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x; i < n; i += stride) {
        const Rng g{key.k0, key.k1, (uint32_t)call, (uint64_t)i};
        const double v = law_rvs(LAW, g, P(0, i), P(1, i), P(2, i), P(3, i));
        if (discrete_law(LAW))
            static_cast<int64_t *>(out)[i] = (v == v) ? (int64_t)v : INT64_MIN;
        else
            static_cast<double *>(out)[i] = v;
    }
}

// Dirichlet(alpha) log-density of the rows of x (n, d), scipy.stats.dirichlet.logpdf: c0 + sum_j xlogy(a_j - 1, x_j)
// with c0 = -log B(alpha) from the host.  scipy's _dirichlet_check_input, row by row, sets bits of *bad (the host
// raises its ValueError): kDirRange an entry < 0 or > 1, kDirZero a zero entry where a_j < 1, kDirSum
// |sum - 1| > 1e-9, kDirNaN a NaN entry.  scipy takes the min and max over the whole array, so a NaN anywhere
// disables its range test (the host ignores kDirRange when kDirNaN is set) and the row's density is NaN.
enum : int { kDirRange = 1, kDirZero = 2, kDirSum = 4, kDirNaN = 8 };
__global__ void __launch_bounds__(kBlock) k_dirichlet_logpdf(const double *__restrict__ x, int64_t x_ld,
                                                            const double *__restrict__ alpha, int d, double c0,
                                                            double *__restrict__ out, int *__restrict__ bad,
                                                            int64_t n) {
    const int64_t stride = (int64_t)gridDim.x * kBlock;
    for (int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x; i < n; i += stride) {
        const double *xi = x + i * x_ld;
        double s = 0.0, lp = c0;
        int flags = 0;
        for (int j = 0; j < d; j++) {
            const double v = xi[j], a = __ldg(alpha + j);
            if (v != v) flags |= kDirNaN;
            if (v < 0.0 || v > 1.0) flags |= kDirRange;
            if (v == 0.0 && a < 1.0) flags |= kDirZero;
            s += v;
            lp += (a == 1.0 && v == v) ? 0.0 : (a - 1.0) * log(v);
        }
        if (fabs(s - 1.0) > 1e-9) flags |= kDirSum;
        if (flags) atomicOr(bad, flags);
        out[i] = lp;
    }
}

// Dirichlet draws: row i is (G_j / sum G), G_j ~ Gamma(a_j, 1) the draw of element i d + j, normalised in log space
// (exp(log G_j - max) / sum) so that rows of small alphas, whose G_j all underflow, stay finite
__global__ void __launch_bounds__(kBlock) k_dirichlet_rvs(Philox key, uint64_t call, const double *__restrict__ alpha,
                                                         int d, double *__restrict__ out, int64_t n) {
    const int64_t stride = (int64_t)gridDim.x * kBlock;
    for (int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x; i < n; i += stride) {
        double m = -CUDART_INF;
        for (int j = 0; j < d; j++) {
            const Rng g{key.k0, key.k1, (uint32_t)call, (uint64_t)(i * d + j)};
            const double l = gamma_log_rvs(g, 0, __ldg(alpha + j));
            out[i * d + j] = l;
            m = fmax(m, l);
        }
        double s = 0.0;
        for (int j = 0; j < d; j++) {
            const double e = exp(out[i * d + j] - m);
            out[i * d + j] = e;
            s += e;
        }
        for (int j = 0; j < d; j++) out[i * d + j] /= s;
    }
}

// ---------------------------------------------------------------------------
// VaryingCovNormal: one thread per particle, its lower factor (D (D + 1) / 2 values) in registers.  cov, L are
// (n, D, D) row-major; loc / x rows of D values with row stride ld (0: one row for every particle).
// ---------------------------------------------------------------------------
template <int D>
__global__ void __launch_bounds__(kBlock) k_vcn_chol(const double *__restrict__ cov, double *__restrict__ L,
                                                    int *__restrict__ bad, int64_t n) {
    const int64_t stride = (int64_t)gridDim.x * kBlock;
    for (int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x; i < n; i += stride) {
        const double *C = cov + i * D * D;
        double l[D * (D + 1) / 2], inv[D];     // inv: 1 / L_cc, through rsqrt (no division or square-root calls)
#pragma unroll
        for (int r = 0; r < D; r++) {
#pragma unroll
            for (int c = 0; c <= r; c++) {
                double s = C[r * D + c];
#pragma unroll
                for (int k = 0; k < c; k++) s -= l[r * (r + 1) / 2 + k] * l[c * (c + 1) / 2 + k];
                if (r == c) {
                    if (!(s > 0.0)) atomicOr(bad, 1);   // NaN or a non-positive pivot: numpy's LinAlgError
                    inv[r] = rsqrt(s);
                    l[r * (r + 1) / 2 + c] = s * inv[r];
                } else {
                    l[r * (r + 1) / 2 + c] = s * inv[c];
                }
            }
        }
        double *Li = L + i * D * D;
#pragma unroll
        for (int r = 0; r < D; r++)
#pragma unroll
            for (int c = 0; c < D; c++) Li[r * D + c] = (c <= r) ? l[r * (r + 1) / 2 + c] : 0.0;
    }
}

template <int D>
__device__ __forceinline__ void load_lower(const double *__restrict__ Li, double (&l)[D * (D + 1) / 2]) {
#pragma unroll
    for (int r = 0; r < D; r++)
#pragma unroll
        for (int c = 0; c <= r; c++) l[r * (r + 1) / 2 + c] = Li[r * D + c];
}

// loc + L z, z the Box-Muller normals of element i, block k giving components 2k, 2k + 1
template <int D>
__global__ void __launch_bounds__(kBlock) k_vcn_rvs(Philox key, uint64_t call, const double *__restrict__ loc,
                                                   int64_t loc_ld, const double *__restrict__ L,
                                                   double *__restrict__ out, int64_t n) {
    const int64_t stride = (int64_t)gridDim.x * kBlock;
    for (int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x; i < n; i += stride) {
        const Rng g{key.k0, key.k1, (uint32_t)call, (uint64_t)i};
        double z[D + 1];
#pragma unroll 1
        for (int k = 0; k < (D + 1) / 2; k++) {
            uint32_t r[4];
            g.block(k, r);
            double z0, z1;
            box_muller(r, z0, z1);
#pragma unroll
            for (int j = 0; j < (D + 1) / 2; j++)
                if (j == k) { z[2 * j] = z0; z[2 * j + 1] = z1; }
        }
        double l[D * (D + 1) / 2];
        load_lower<D>(L + i * D * D, l);
#pragma unroll
        for (int r = 0; r < D; r++) {
            double s = 0.0;
#pragma unroll
            for (int c = 0; c <= r; c++) s += l[r * (r + 1) / 2 + c] * z[c];
            out[i * D + r] = loc[i * loc_ld + r] + s;
        }
    }
}

// -|L^-1 (x - loc)|^2 / 2 - sum log L_jj - D log(2 pi) / 2, by forward substitution
template <int D>
__global__ void __launch_bounds__(kBlock) k_vcn_logpdf(const double *__restrict__ x, int64_t x_ld,
                                                      const double *__restrict__ loc, int64_t loc_ld,
                                                      const double *__restrict__ L, double *__restrict__ out,
                                                      int64_t n) {
    const int64_t stride = (int64_t)gridDim.x * kBlock;
    for (int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x; i < n; i += stride) {
        double l[D * (D + 1) / 2];
        load_lower<D>(L + i * D * D, l);
        double z[D], q = 0.0, hld = 0.0;
#pragma unroll
        for (int r = 0; r < D; r++) {
            double s = x[i * x_ld + r] - loc[i * loc_ld + r];
#pragma unroll
            for (int c = 0; c < r; c++) s -= l[r * (r + 1) / 2 + c] * z[c];
            z[r] = s / l[r * (r + 1) / 2 + r];
            q += z[r] * z[r];
            hld += log(l[r * (r + 1) / 2 + r]);
        }
        out[i] = -0.5 * q - (D * kLogSqrt2Pi + hld);
    }
}

// Mixture.logpdf: out[i] = logsumexp_j (logpk[i pk_ld + j] + lp[j n + i]), scipy.special.logsumexp's conventions
// (-inf when every term is, +inf when one is, NaN when one is NaN)
__global__ void __launch_bounds__(kBlock) k_mixture_logpdf(const double *__restrict__ lp,
                                                          const double *__restrict__ logpk, int64_t pk_ld, int k,
                                                          double *__restrict__ out, int64_t n) {
    const int64_t stride = (int64_t)gridDim.x * kBlock;
    for (int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x; i < n; i += stride) {
        double m = -CUDART_INF;
        for (int j = 0; j < k; j++) m = fmax(m, __ldg(logpk + i * pk_ld + j) + lp[(int64_t)j * n + i]);
        const double sh = (fabs(m) < CUDART_INF) ? m : 0.0;
        double s = 0.0;
        for (int j = 0; j < k; j++) s += exp(__ldg(logpk + i * pk_ld + j) + lp[(int64_t)j * n + i] - sh);
        out[i] = log(s) + sh;
    }
}

template <template <int> class K, class... A>
int launch_vcn(smcb_ctx *c, int d, int64_t n, A... args) {
    const int g = grid_for(n, kBlock);
    switch (d) {
        case 1: return launch(c, K<1>::fn, g, kBlock, 0, args...);
        case 2: return launch(c, K<2>::fn, g, kBlock, 0, args...);
        case 3: return launch(c, K<3>::fn, g, kBlock, 0, args...);
        case 4: return launch(c, K<4>::fn, g, kBlock, 0, args...);
        case 5: return launch(c, K<5>::fn, g, kBlock, 0, args...);
        case 6: return launch(c, K<6>::fn, g, kBlock, 0, args...);
        case 7: return launch(c, K<7>::fn, g, kBlock, 0, args...);
        default: return launch(c, K<8>::fn, g, kBlock, 0, args...);
    }
}
// launches K<law> for a law in [LAW, END): one instance per code of that range, and none outside it
template <template <int> class K, int LAW, int END, class... A>
int launch_law(smcb_ctx *c, int law, int64_t n, A... args) {
    if constexpr (LAW + 1 < END)
        if (law != LAW) return launch_law<K, LAW + 1, END>(c, law, n, args...);
    return launch(c, K<LAW>::fn, grid_for(n, kBlock * 4), kBlock, 0, args...);
}
template <int L> struct LLogpdf { static constexpr auto fn = k_dist_logpdf<L>; };
template <int L> struct LRvs { static constexpr auto fn = k_dist_rvs<L>; };
template <int D> struct Chol { static constexpr auto fn = k_vcn_chol<D>; };
template <int D> struct VRvs { static constexpr auto fn = k_vcn_rvs<D>; };
template <int D> struct VLogpdf { static constexpr auto fn = k_vcn_logpdf<D>; };

Par4 par4(const double *p0, const double *p1, const double *p2, const double *p3, const double *s) {
    return Par4{{p0, p1, p2, p3}, {s[0], s[1], s[2], s[3]}};
}

}  // namespace

extern "C" int smcb_dist_logpdf(smcb_ctx *c, int law, const double *x, double x0, const double *p0, const double *p1,
                                const double *p2, const double *p3, const double *s, double *out, int64_t n) {
    SMCB_REQUIRE(c && out && s && n >= 1, "smcb_dist_logpdf: bad argument");
    SMCB_REQUIRE(law >= 0 && law < kNumLaws, "smcb_dist_logpdf: %d is not a law code", law);
    return launch_law<LLogpdf, 0, kNumLaws>(c, law, n, x, x0, par4(p0, p1, p2, p3, s), out, n);
}

extern "C" int smcb_dist_rvs(smcb_ctx *c, int law, const double *p0, const double *p1, const double *p2,
                             const double *p3, const double *s, void *out, int64_t n) {
    SMCB_REQUIRE(c && out && s && n >= 1, "smcb_dist_rvs: bad argument");
    SMCB_REQUIRE(law >= 0 && law < kNumSampled, "smcb_dist_rvs: %d is not a law with a sampler here", law);
    return launch_law<LRvs, 0, kNumSampled>(c, law, n, key_of(c->seed), c->api_counter++, par4(p0, p1, p2, p3, s),
                                            out, n);
}

extern "C" int smcb_dirichlet_logpdf(smcb_ctx *c, const double *x, int64_t x_ld, const double *alpha, int d, double c0,
                                     double *out, int *bad, int64_t n) {
    SMCB_REQUIRE(c && x && alpha && out && bad && d >= 1 && n >= 1 && x_ld >= 0, "smcb_dirichlet_logpdf: bad argument");
    return launch(c, k_dirichlet_logpdf, grid_for(n, kBlock * 4), kBlock, 0, x, x_ld, alpha, d, c0, out, bad, n);
}

extern "C" int smcb_dirichlet_rvs(smcb_ctx *c, const double *alpha, int d, double *out, int64_t n) {
    SMCB_REQUIRE(c && alpha && out && d >= 1 && n >= 1, "smcb_dirichlet_rvs: bad argument");
    return launch(c, k_dirichlet_rvs, grid_for(n, kBlock * 4), kBlock, 0, key_of(c->seed), c->api_counter++, alpha, d,
                  out, n);
}

extern "C" int smcb_vcn_chol(smcb_ctx *c, const double *cov, int d, double *L, int *bad, int64_t n) {
    SMCB_REQUIRE(c && cov && L && bad && n >= 1, "smcb_vcn_chol: bad argument");
    if (d < 1 || d > 8) {
        set_error("VaryingCovNormal: d = %d, the device kernels take 1 <= d <= 8", d);
        return SMCB_ENOSYS;
    }
    return launch_vcn<Chol>(c, d, n, cov, L, bad, n);
}

extern "C" int smcb_vcn_rvs(smcb_ctx *c, const double *loc, int64_t loc_ld, const double *L, int d, double *out,
                            int64_t n) {
    SMCB_REQUIRE(c && loc && L && out && n >= 1 && d >= 1 && d <= 8 && loc_ld >= 0, "smcb_vcn_rvs: bad argument");
    return launch_vcn<VRvs>(c, d, n, key_of(c->seed), c->api_counter++, loc, loc_ld, L, out, n);
}

extern "C" int smcb_vcn_logpdf(smcb_ctx *c, const double *x, int64_t x_ld, const double *loc, int64_t loc_ld,
                               const double *L, int d, double *out, int64_t n) {
    SMCB_REQUIRE(c && x && loc && L && out && n >= 1 && d >= 1 && d <= 8 && x_ld >= 0 && loc_ld >= 0,
                 "smcb_vcn_logpdf: bad argument");
    return launch_vcn<VLogpdf>(c, d, n, x, x_ld, loc, loc_ld, L, out, n);
}

extern "C" int smcb_mixture_logpdf(smcb_ctx *c, const double *lp, const double *logpk, int64_t pk_ld, int k,
                                   double *out, int64_t n) {
    SMCB_REQUIRE(c && lp && logpk && out && k >= 1 && n >= 1 && pk_ld >= 0, "smcb_mixture_logpdf: bad argument");
    return launch(c, k_mixture_logpdf, grid_for(n, kBlock * 4), kBlock, 0, lp, logpk, pk_ld, k, out, n);
}
