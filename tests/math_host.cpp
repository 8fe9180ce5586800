// Host build of particles_b200/csrc/smcb_math.cuh (the step kernel's fp64 exp / log / sincos / batch
// log-sum-exp), smcb_models.cuh (the model / Feynman-Kac maps of the fused step kernel), the library's table of
// (model, Feynman-Kac kind) combinations in smcb_dispatch.cuh and the step kernel's in-tile CDF search of
// smcb_search.cuh so that their
// ALGORITHMS can be checked on the CPU against NumPy / mpmath and against the oracle
// (tests/test_math_host.py, tests/test_models_host.py).  CUDA intrinsics are restated bit-for-bit below; compile with
// -ffp-contract=off so that only the explicit fma() calls fuse, as nvcc -fmad=false does.
//   g++ -O2 -ffp-contract=off -shared -fPIC -I particles_b200/csrc tests/math_host.cpp
// Both families of smcb_math.cuh are exported: `tab` = 0 polynomial (stand-alone kernels), 1 table-assisted (step
// kernels; the tables of smcb_tables.h are built here by the same host function the library uses).
#include <cmath>
#include <cstdint>
#include <cstring>

#define SMCB_MATH_HOST_TEST 1
#define __device__
#define __host__
#define __forceinline__ inline
#define __constant__ const
#define CUDART_INF INFINITY
#define CUDART_NAN NAN
struct double2 { double x, y; };
static inline int __double2hiint(double v) { uint64_t b; std::memcpy(&b, &v, 8); return (int)(uint32_t)(b >> 32); }
static inline int __double2loint(double v) { uint64_t b; std::memcpy(&b, &v, 8); return (int)(uint32_t)b; }
static inline double __hiloint2double(int hi, int lo) {
    uint64_t b = ((uint64_t)(uint32_t)hi << 32) | (uint32_t)lo; double v; std::memcpy(&v, &b, 8); return v;
}
template <class T> static inline T __ldg(const T *p) { return *p; }
static inline unsigned int __funnelshift_r(unsigned int lo, unsigned int hi, unsigned int sh) {
    return (unsigned int)((((uint64_t)hi << 32) | lo) >> (sh & 31));
}
using std::fma; using std::fmax; using std::sqrt; using std::floor; using std::atan; using std::lgamma;
using std::log; using std::exp; using std::fabs; using std::cos;
#include "smcb.h"                 // model / Feynman-Kac ids
namespace smcb {
constexpr double kHalfLog2Pi = 0.91893853320467274178;      // log(2 pi) / 2, as in smcb_common.cuh
static inline double normal_logpdf(double x, double loc, double scale) {
    double z = (x - loc) / scale;
    return -z * z / 2.0 - kHalfLog2Pi - log(scale);
}
struct Lse3 { double m, s, q; };
struct Philox { uint32_t k0, k1, rk[20]; };
constexpr uint32_t kPurposeNormal = 1;
// the two uniform constructions of smcb_common.cuh (53-bit mantissa from two 32-bit words)
static inline double u53(uint32_t a, uint32_t b) {
    return (double)(((uint64_t)(a >> 5) << 26) | (b >> 6)) * 1.1102230246251565404e-16;
}
static inline double u53_open(uint32_t a, uint32_t b) {
    return ((double)(((uint64_t)(a >> 5) << 26) | (b >> 6)) + 0.5) * 1.1102230246251565404e-16;
}
static inline void philox4x32_10k(uint32_t, uint32_t, uint32_t, uint32_t, const Philox &, uint32_t *) {}
}  // namespace smcb
#include "smcb_math.cuh"
#include "smcb_models.cuh"
#include "smcb_dispatch.cuh"
#include "smcb_search.cuh"

namespace {
using namespace smcb;
// same construction as step_consts() of smcb_step.cuh
StepK make_step(const double *data, long T, int dy, const double *sc, long t) {
    StepK k;
    k.t = t;
    for (int i = 0; i < kMaxDy; i++) {
        k.yv[i] = (i < dy) ? data[t * dy + i] : 0.0;
        k.yn[i] = (i < dy && t + 1 < T) ? data[(t + 1) * dy + i] : 0.0;
    }
    k.y = k.yv[0];
    k.y_next = k.yn[0];
    k.sc0 = sc ? sc[t] : 0.0;
    return k;
}
// one step of the fused kernel's per-particle work, no resampling: x' and the log-weight increment from
// (xp, z), plus logeta(t, x') for the auxiliary kinds.  SoA arrays: xp / x (D, n), z (NZ, n).
template <class M, int FK>
void step_all(const double *params, const StepK &k, const double *xp, const double *z, long n, double *x,
              double *delta, double *leta) {
    M m;
    m.load(params);
    constexpr int D = M::D, NZ = M::NZ;
    for (long i = 0; i < n; i++) {
        double zi[NZ], xpi[D], xi[D], d;
        for (int c = 0; c < NZ; c++) zi[c] = z[(size_t)c * n + i];
        if (xp) {
            for (int c = 0; c < D; c++) xpi[c] = xp[(size_t)c * n + i];
            model_move<M, FK>(m, k, xpi, zi, xi, d);
        } else {
            model_init<M, FK>(m, k, zi, xi, d);
        }
        for (int c = 0; c < D; c++) x[(size_t)c * n + i] = xi[c];
        delta[i] = d;
        if (leta) leta[i] = model_logeta<M>(m, k, xi);
    }
}
}  // namespace

extern "C" {
// returns 0, or -3 (SMCB_ENOSYS) when the (model, Feynman-Kac kind, dimension) combination has no fused kernel:
// the library's own table, smcb_dispatch.cuh, decides
int mh_model_step(int model, int fk, int dim, const double *params, const double *data, long T, int dy,
                  const double *sc, long t, const double *xp, const double *z, long n, double *x, double *delta,
                  double *leta) {
    const StepK k = make_step(data, T, dy, sc, t);
    return with_model(model, dim, [&](auto m) {
        using M = decltype(m);
        return with_fk<M>(fk, [&](auto kind) {
            constexpr int FK = decltype(kind)::value;
            step_all<M, FK>(params, k, xp, z, n, x, delta, FkTraits<FK>::apf ? leta : nullptr);
            return 0;
        });
    });
}

static double g_tables[smcb::kMathTabDoubles];
void mh_init() { smcb::fill_math_tables(g_tables); smcb::g_mtab_host = g_tables; }
const double *mh_tables() { return g_tables; }
int mh_table_doubles() { return smcb::kMathTabDoubles; }
void mh_exp(const double *x, double *y, long n, int kind, int tab) {
    for (long i = 0; i < n; i++) {
        if (tab) y[i] = kind == 0 ? smcb::texp(x[i]) : (kind == 1 ? smcb::texp_neg(x[i]) : smcb::texp_sat(x[i]));
        else y[i] = kind == 0 ? smcb::fexp(x[i]) : (kind == 1 ? smcb::fexp_neg(x[i]) : smcb::fexp_mid(x[i]));
    }
}
void mh_log(const double *x, double *y, long n, int tab) {
    for (long i = 0; i < n; i++) y[i] = tab ? smcb::tlog_pos(x[i]) : smcb::flog_pos(x[i]);
}
void mh_sqrt(const double *x, double *y, long n) { for (long i = 0; i < n; i++) y[i] = smcb::tsqrt_pos(x[i]); }
void mh_sincos2pi(const double *u, double *s, double *c, long n, int tab) {
    for (long i = 0; i < n; i++) { if (tab) smcb::tsincos2pi(u[i], s[i], c[i]); else smcb::fsincos2pi(u[i], s[i], c[i]); }
}
void mh_box_muller(const uint32_t *r, double *z, long npairs, int tab) {
    for (long i = 0; i < npairs; i++) {
        if (tab) smcb::box_muller_tab(r + 4 * i, z[2 * i], z[2 * i + 1]);
        else smcb::box_muller_fast(r + 4 * i, z[2 * i], z[2 * i + 1]);
    }
}
// (m, s, q) of v accumulated in batches of 4, as the step kernel does
void mh_lse3(const double *v, long n, double *out3) {
    smcb::Lse3 a{-INFINITY, 0.0, 0.0};
    long i = 0;
    for (; i + 4 <= n; i += 4) { const double b[4] = {v[i], v[i + 1], v[i + 2], v[i + 3]}; smcb::lse3_add_batch<4>(a, b); }
    for (; i < n; i++) { const double b[1] = {v[i]}; smcb::lse3_add_batch<1>(a, b); }
    out3[0] = a.m; out3[1] = a.s; out3[2] = a.q;
}
// the step kernel's in-tile search: for each query i, the answers for keys v[2i] <= v[2i+1] on the slice s[0, cnt)
// searched from l0[i]
void mh_tile_search(const double *s, int cnt, const int *l0, const double *v, long m, int *out) {
    for (long i = 0; i < m; i++) smcb::tile_search(s, l0[i], cnt, v[2 * i], v[2 * i + 1], out[2 * i], out[2 * i + 1]);
}
}
