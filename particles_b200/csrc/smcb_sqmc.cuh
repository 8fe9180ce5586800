// smcb_sqmc.cuh -- the pieces of sequential quasi-Monte Carlo (particles/core.py:315-349, rqmc.py, hilbert.py) that
// are pure functions: the inverse normal CDF, scrambled Sobol' points and Hilbert keys.  Every function is
// __host__ __device__ and uses only +, -, *, /, sqrt, fma and integer operations, so the CPU test harness
// (tests/sqmc_host.cpp, g++ -ffp-contract=off) reproduces the kernels of smcb_sqmc.cu bit for bit.
#pragma once
#include <stdint.h>
#ifndef SMCB_SQMC_HOST_TEST
#include "smcb_common.cuh"
#define SMCB_SOBOL_CONST __constant__ const
#define SMCB_SOBOL_GLOBAL __device__ const
#else
#define SMCB_SOBOL_CONST static const
#define SMCB_SOBOL_GLOBAL static const
#endif

namespace smcb {
namespace sqmc {

#define SMCB_HD __host__ __device__ __forceinline__

#include "smcb_sobol_dirs.inc"
#include "smcb_sobol_init.inc"

#ifdef SMCB_SQMC_HOST_TEST
constexpr uint32_t kPurposeSobol = 9;     // as in smcb_common.cuh
#endif
// rqmc.py: v = 0.5 + (1 - TOL) (u - 0.5), TOL = 1e-10, keeps the points off 0 and 1
constexpr double kSqueeze = 1.0 - 1e-10;
constexpr double kTwoM30 = 1.0 / 1073741824.0;     // 2^-30: scipy's scale of the 30-bit integers
constexpr int kHilbertMaxDim = 32;

SMCB_HD uint64_t dbits(double x) {
#ifdef __CUDA_ARCH__
    return (uint64_t)__double_as_longlong(x);
#else
    uint64_t b;
    __builtin_memcpy(&b, &x, 8);
    return b;
#endif
}
SMCB_HD double bitsd(uint64_t b) {
#ifdef __CUDA_ARCH__
    return __longlong_as_double((long long)b);
#else
    double x;
    __builtin_memcpy(&x, &b, 8);
    return x;
#endif
}

// log(x) for a positive normal x: x = 2^e m with m in [sqrt(1/2), sqrt(2)), log m = 2 atanh(f), f = (m - 1)/(m + 1),
// |f| <= 0.1716; the odd series to f^23 leaves < 1e-19 relative; e ln 2 in two parts (the high part has 32 bits).
SMCB_HD double plog(double x) {
    uint64_t b = dbits(x);
    int e = (int)((b >> 52) & 0x7ff) - 1023;
    b = (b & 0x000fffffffffffffull) | 0x3ff0000000000000ull;     // m in [1, 2)
    double m = bitsd(b);
    if (m > 1.4142135623730951) { m *= 0.5; e += 1; }
    const double f = (m - 1.0) / (m + 1.0), f2 = f * f;
    double p = 1.0 / 23.0;
    p = fma(p, f2, 1.0 / 21.0); p = fma(p, f2, 1.0 / 19.0); p = fma(p, f2, 1.0 / 17.0);
    p = fma(p, f2, 1.0 / 15.0); p = fma(p, f2, 1.0 / 13.0); p = fma(p, f2, 1.0 / 11.0);
    p = fma(p, f2, 1.0 / 9.0); p = fma(p, f2, 1.0 / 7.0); p = fma(p, f2, 1.0 / 5.0); p = fma(p, f2, 1.0 / 3.0);
    const double s = fma(f * f2, p, f);                          // atanh(f)
    const double ln2_hi = 6.93147180369123816490e-01, ln2_lo = 1.90821492927058770002e-10;
    return fma((double)e, ln2_hi, fma((double)e, ln2_lo, 2.0 * s));
}

// Phi^-1(p) for p in (0, 1): Wichura's algorithm AS 241 (PPND16, Appl. Statist. 37 (1988) 477-484), rational
// approximations of relative accuracy ~1e-16 on |p - 1/2| <= 0.425 and, in r = sqrt(-log min(p, 1 - p)), on r <= 5
// and beyond.  The maximum error against scipy.special.ndtri over the squeezed range of the Sobol' points is measured
// by tests/test_sqmc_host.py (DESIGN.md section 5.17).
SMCB_HD double ndtri(double p) {
    const double q = p - 0.5;
    if (fabs(q) <= 0.425) {
        const double r = 0.180625 - q * q;
        double a = 2.5090809287301226727e+3;
        a = fma(a, r, 3.3430575583588128105e+4); a = fma(a, r, 6.7265770927008700853e+4);
        a = fma(a, r, 4.5921953931549871457e+4); a = fma(a, r, 1.3731693765509461125e+4);
        a = fma(a, r, 1.9715909503065514427e+3); a = fma(a, r, 1.3314166789178437745e+2);
        a = fma(a, r, 3.3871328727963666080e0);
        double b = 5.2264952788528545610e+3;
        b = fma(b, r, 2.8729085735721942674e+4); b = fma(b, r, 3.9307895800092710610e+4);
        b = fma(b, r, 2.1213794301586595867e+4); b = fma(b, r, 5.3941960214247511077e+3);
        b = fma(b, r, 6.8718700749205790830e+2); b = fma(b, r, 4.2313330701600911252e+1);
        b = fma(b, r, 1.0);
        return q * a / b;
    }
    double r = q < 0.0 ? p : 1.0 - p;
    r = sqrt(-plog(r));
    double v;
    if (r <= 5.0) {
        r -= 1.6;
        double a = 7.74545014278341407640e-4;
        a = fma(a, r, 2.27238449892691845833e-2); a = fma(a, r, 2.41780725177450611770e-1);
        a = fma(a, r, 1.27045825245236838258e0); a = fma(a, r, 3.64784832476320460504e0);
        a = fma(a, r, 5.76949722146069140550e0); a = fma(a, r, 4.63033784615654529590e0);
        a = fma(a, r, 1.42343711074968357734e0);
        double b = 1.05075007164441684324e-9;
        b = fma(b, r, 5.47593808499534494600e-4); b = fma(b, r, 1.51986665636164571966e-2);
        b = fma(b, r, 1.48103976427480074590e-1); b = fma(b, r, 6.89767334985100004550e-1);
        b = fma(b, r, 1.67638483018380384940e0); b = fma(b, r, 2.05319162663775882187e0);
        b = fma(b, r, 1.0);
        v = a / b;
    } else {
        r -= 5.0;
        double a = 2.01033439929228813265e-7;
        a = fma(a, r, 2.71155556874348757815e-5); a = fma(a, r, 1.24266094738807843860e-3);
        a = fma(a, r, 2.65321895265761230930e-2); a = fma(a, r, 2.96560571828504891230e-1);
        a = fma(a, r, 1.78482653991729133580e0); a = fma(a, r, 5.46378491116411436990e0);
        a = fma(a, r, 6.65790464350110377720e0);
        double b = 2.04426310338993978564e-15;
        b = fma(b, r, 1.42151175831644588870e-7); b = fma(b, r, 1.84631831751005468180e-5);
        b = fma(b, r, 7.86869131145613259100e-4); b = fma(b, r, 1.48753612908506148525e-2);
        b = fma(b, r, 1.36929880922735805310e-1); b = fma(b, r, 5.99832206555887937690e-1);
        b = fma(b, r, 1.0);
        v = a / b;
    }
    return q < 0.0 ? -v : v;
}

// ---------------------------------------------------------------------------------------------------------------------
// Sobol' points (scipy.stats.qmc.Sobol, 30 bits).  Point i is shift ^ XOR of the direction numbers selected by the
// bits of the Gray code i ^ (i >> 1): scipy's sequence, computed for every i independently.  Scrambling, as scipy's:
// a random lower-triangular bit matrix with unit diagonal applied to every direction number (bit 29 - p of the result
// is the parity of row p and the number; row p mixes in bits 29 - k, k < p) and a random digital shift.  Both are
// drawn from Philox under key(seed), counter (word block, dimension, call lo, (call hi << 8) | kPurposeSobol): the
// points of call `call` depend on (seed, call) only.
// ---------------------------------------------------------------------------------------------------------------------
template <class KEY>
SMCB_HD void sobol_scramble_words(const KEY &key_fn, int j, uint64_t call, uint32_t w[32]) {
    for (int blk = 0; blk < 8; blk++) {
        uint32_t r[4];
        key_fn((uint32_t)blk, (uint32_t)j, (uint32_t)call, ((uint32_t)(call >> 32) << 8) | kPurposeSobol, r);
        for (int q = 0; q < 4; q++) w[4 * blk + q] = r[q];
    }
}

// the direction numbers of dimension j, 1 <= j < kSobolMaxDim, from its primitive polynomial p of degree s and its s
// initial numbers (smcb_sobol_init.inc), by scipy's recurrence (_initialize_v):
//   m_k = m_{k-s} ^ (2^s m_{k-s}) ^ XOR_{i < s-1, bit s-1-i of p} 2^(i+1) m_{k-i-1},
// then number k = m_k 2^(29-k).  For j < kSobolTabDim this reproduces kSobolDirs (tests/test_ffbs_qmc_host.py).
SMCB_HD void sobol_expand(int j, uint32_t v[kSobolBits]) {
    const uint32_t *row = kSobolInit + kSobolInitOff[j];
    const uint32_t p = row[0];
    int s = 0;
    while ((p >> (s + 1)) != 0u) s++;
    for (int k = 0; k < s; k++) v[k] = row[1 + k];
    for (int k = s; k < kSobolBits; k++) {
        uint32_t m = v[k - s];
        for (int i = 0; i < s; i++)
            if ((p >> (s - 1 - i)) & 1u) m ^= v[k - i - 1] << (i + 1);
        v[k] = m;
    }
    for (int k = 0; k < kSobolBits; k++) v[k] <<= kSobolBits - 1 - k;
}

// the (scrambled) direction numbers and shift of dimension j from its 32 random words (words 0..29: the rows of the
// matrix, word 30: the shift); scramble = 0 gives scipy's scramble=False numbers and a zero shift
SMCB_HD void sobol_dims(int j, int scramble, const uint32_t w[32], uint32_t sv[kSobolBits], uint32_t &shift) {
    const uint32_t full = (1u << kSobolBits) - 1u;
    if (j < kSobolTabDim) {
        for (int k = 0; k < kSobolBits; k++) sv[k] = kSobolDirs[j][k];
    } else {
        sobol_expand(j, sv);
    }
    shift = 0;
    if (!scramble) return;
    uint32_t rows[kSobolBits];
    for (int p = 0; p < kSobolBits; p++) {        // row p: the diagonal bit 29 - p and random bits above it
        const uint32_t above = p == 0 ? 0u : ((w[p] & ((1u << p) - 1u)) << (kSobolBits - p));
        rows[p] = ((1u << (kSobolBits - 1 - p)) | above) & full;
    }
    for (int k = 0; k < kSobolBits; k++) {
        uint32_t out = 0;
        for (int p = 0; p < kSobolBits; p++) {
            uint32_t x = rows[p] & sv[k];
            x ^= x >> 16; x ^= x >> 8; x ^= x >> 4; x ^= x >> 2; x ^= x >> 1;
            out |= (x & 1u) << (kSobolBits - 1 - p);
        }
        sv[k] = out;
    }
    shift = w[30] & full;
}

SMCB_HD uint32_t sobol_int(const uint32_t sv[kSobolBits], uint32_t shift, uint64_t i) {
    uint64_t g = i ^ (i >> 1);
    uint32_t q = shift;
    for (int k = 0; k < kSobolBits && g; k++, g >>= 1)
        if (g & 1) q ^= sv[k];
    return q;
}

// rqmc.py's squeeze of scipy's float point q 2^-30
SMCB_HD double squeeze(uint32_t q) { return 0.5 + kSqueeze * ((double)q * kTwoM30 - 0.5); }

// ---------------------------------------------------------------------------------------------------------------------
// Hilbert keys: hilbert.py's Hilbert_to_int (Witham's codec) on int64 coordinates, with numba's int64 semantics kept
// exactly: products wrap mod 2^64, // is a floor division, pack_index wraps, and the keys compare as signed values.
// The number of chunks is the bit length of the point's largest coordinate (ceil(log2(max + 1)), at least 1).
// ---------------------------------------------------------------------------------------------------------------------
SMCB_HD int64_t fdiv(int64_t a, int64_t b) {
    int64_t q = a / b;
    if ((a % b != 0) && ((a < 0) != (b < 0))) q -= 1;
    return q;
}
SMCB_HD int64_t wmul(int64_t a, int64_t b) { return (int64_t)((uint64_t)a * (uint64_t)b); }
SMCB_HD int64_t gray_encode(int64_t bn) { return bn ^ fdiv(bn, 2); }
SMCB_HD int64_t gray_decode(int64_t n) {
    for (int sh = 1;; sh <<= 1) {
        const int64_t div = sh < 64 ? (n >> sh) : (n < 0 ? -1 : 0);
        n ^= div;
        if (div <= 1) return n;
    }
}
SMCB_HD int64_t gray_encode_travel(int64_t start, int64_t end, int64_t mask, int64_t i) {
    const int64_t travel_bit = start ^ end, modulus = mask + 1;
    const int64_t g = wmul(gray_encode(i), travel_bit * 2);
    return ((g | fdiv(g, modulus)) & mask) ^ start;
}
SMCB_HD int64_t gray_decode_travel(int64_t start, int64_t end, int64_t mask, int64_t g) {
    const int64_t travel_bit = start ^ end, modulus = mask + 1;
    const int64_t rg = wmul(g ^ start, fdiv(modulus, travel_bit * 2));
    return gray_decode((rg | fdiv(rg, modulus)) & mask);
}

// Hilbert_to_int(coords[0..d)), coords >= 0, 2 <= d <= 32
SMCB_HD int64_t hilbert_key(const int64_t *c, int d) {
    int64_t biggest = c[0];
    for (int k = 1; k < d; k++) biggest = c[k] > biggest ? c[k] : biggest;
    int nchunks = 0;
    for (uint64_t v = (uint64_t)biggest; v; v >>= 1) nchunks++;
    if (nchunks < 1) nchunks = 1;
    const int64_t mask = (int64_t)((1ull << d) - 1ull);
    int64_t start = 0, end = (int64_t)1 << (((-nchunks - 1) % d + d) % d);
    uint64_t z = 0;
    const uint64_t p = 1ull << d;
    for (int j = 0; j < nchunks; j++) {
        const int bit = nchunks - 1 - j;                       // chunk j: bit `bit` of every coordinate
        int64_t chunk = 0;
        for (int k = 0; k < d; k++) chunk = chunk * 2 + ((c[k] >> bit) & 1);
        const int64_t i = gray_decode_travel(start, end, mask, chunk);
        z = j == 0 ? (uint64_t)i : p * z + (uint64_t)i;        // pack_index, mod 2^64
        const int64_t si = (i - 1) & ~(int64_t)1, ei = (i + 1) | 1;
        const int64_t s2 = gray_encode_travel(start, end, mask, si > 0 ? si : 0);
        const int64_t e2 = gray_encode_travel(start, end, mask, ei < mask ? ei : mask);
        start = s2; end = e2;
    }
    return (int64_t)z;
}

}  // namespace sqmc
}  // namespace smcb
