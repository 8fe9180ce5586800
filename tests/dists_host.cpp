// Host build of particles_b200/csrc/smcb_dists.cuh: the log-densities and the samplers of the laws with a kernel of
// their own, compiled for the CPU so that tests/test_dists_host.py can check them against scipy / mpmath and run the
// goodness-of-fit tests of the samplers on 10^6 draws, and so that tests/test_gpu_dists.py can replay the device's
// draws from the same Philox counters.  The CUDA intrinsics the header uses are restated below; compile with
// -ffp-contract=off so that nothing fuses, as nvcc -fmad=false does.
//   g++ -O2 -ffp-contract=off -shared -fPIC -I particles_b200/csrc tests/dists_host.cpp
#include <cmath>
#include <cstdint>

#define SMCB_DISTS_HOST_TEST 1
#define __device__
#define __host__
#define __forceinline__ inline
using std::ceil; using std::erf; using std::erfc; using std::exp; using std::expm1; using std::fabs; using std::floor;
using std::fmax; using std::fmin; using std::lgamma; using std::log; using std::log1p; using std::pow; using std::sqrt;

namespace smcb {
constexpr uint32_t kPurposeDists = 8;   // as in smcb_common.cuh
// Philox4x32-10 and the 53-bit uniforms of smcb_common.cuh
static inline void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1,
                                 uint32_t out[4]) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
    for (int r = 0; r < 10; r++) {
        const uint64_t p0 = (uint64_t)M0 * c0, p1 = (uint64_t)M1 * c2;
        const uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0, hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
        const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
        c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
        k0 += W0; k1 += W1;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}
static inline double u53(uint32_t a, uint32_t b) {
    return (double)(((uint64_t)(a >> 5) << 26) | (uint64_t)(b >> 6)) * (1.0 / 9007199254740992.0);
}
static inline double u53_open(uint32_t a, uint32_t b) {
    return ((double)(((uint64_t)(a >> 5) << 26) | (uint64_t)(b >> 6)) + 0.5) * (1.0 / 9007199254740992.0);
}
}  // namespace smcb
// (sin, cos)(pi x) as CUDA's sincospi: reduced to |r| <= 1/4 first, so that pi r carries no absolute error
static inline void sincospi(double x, double *s, double *c) {
    const double q = std::nearbyint(2.0 * x);
    const double r = x - 0.5 * q;
    const double sr = std::sin(M_PI * r), cr = std::cos(M_PI * r);
    switch (((long long)q) & 3) {
        case 0: *s = sr; *c = cr; break;
        case 1: *s = cr; *c = -sr; break;
        case 2: *s = -sr; *c = -cr; break;
        default: *s = -cr; *c = sr; break;
    }
}

#include "smcb_dists.cuh"

using namespace smcb::dists;

extern "C" {
// per-element parameter arrays (p2, p3 may be NULL)
void dh_logpdf(int law, const double *x, const double *p0, const double *p1, const double *p2, const double *p3,
               double *out, long n) {
    for (long i = 0; i < n; i++)
        out[i] = law_logpdf(law, x[i], p0[i], p1 ? p1[i] : 0.0, p2 ? p2[i] : 0.0, p3 ? p3[i] : 0.0);
}
// the draws k_dist_rvs makes for elements offset .. offset + n - 1 of API call `call` under key `seed` (discrete
// draws as fp64)
void dh_rvs(int law, uint64_t seed, uint64_t call, long offset, const double *p0, const double *p1, const double *p2,
            const double *p3, double *out, long n) {
    for (long i = 0; i < n; i++) {
        const Rng g{(uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)call, (uint64_t)(offset + i)};
        out[i] = law_rvs(law, g, p0[i], p1 ? p1[i] : 0.0, p2 ? p2[i] : 0.0, p3 ? p3[i] : 0.0);
    }
}
// k_dirichlet_rvs, rows (n, d)
void dh_dirichlet_rvs(uint64_t seed, uint64_t call, const double *alpha, int d, double *out, long n) {
    for (long i = 0; i < n; i++) {
        double m = -INFINITY, s = 0.0;
        for (int j = 0; j < d; j++) {
            const Rng g{(uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)call, (uint64_t)(i * d + j)};
            out[i * d + j] = gamma_log_rvs(g, 0, alpha[j]);
            m = fmax(m, out[i * d + j]);
        }
        for (int j = 0; j < d; j++) {
            out[i * d + j] = exp(out[i * d + j] - m);
            s += out[i * d + j];
        }
        for (int j = 0; j < d; j++) out[i * d + j] /= s;
    }
}
// Philox block `block` of element `elem` in API call `call` (Rng::block), for the check against tests/philox_ref.py
void dh_block(uint64_t seed, uint64_t call, uint64_t elem, uint32_t block, uint32_t *out) {
    const Rng g{(uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)call, elem};
    g.block(block, out);
}
// the uniform and the normal a block gives (Rng::uniform, Rng::normal)
void dh_block_draws(uint64_t seed, uint64_t call, uint64_t elem, uint32_t block, double *out) {
    const Rng g{(uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)call, elem};
    out[0] = g.uniform(block);
    out[1] = g.normal(block);
}
}
