// Host build of particles_b200/csrc/smcb_sqmc.cuh: the inverse normal CDF, the (scrambled) Sobol' points and the
// Hilbert keys, compiled for the CPU so that tests/test_sqmc_host.py can check them against scipy and the reference's
// codec, and so that tests/test_gpu_sqmc.py can replay the device's points and keys.  Compile with -ffp-contract=off
// so that nothing fuses, as nvcc -fmad=false does.
//   g++ -O2 -ffp-contract=off -shared -fPIC -I particles_b200/csrc tests/sqmc_host.cpp
#include <cmath>
#include <cstdint>

#define SMCB_SQMC_HOST_TEST 1
#define __device__
#define __host__
#define __forceinline__ inline
using std::fabs; using std::floor; using std::fma; using std::sqrt;

namespace smcb {
// Philox4x32-10 of smcb_common.cuh
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
}  // namespace smcb

#include "smcb_sqmc.cuh"

using namespace smcb;
using namespace smcb::sqmc;

extern "C" {

void sh_ndtri(const double *p, double *out, long n) {
    for (long i = 0; i < n; i++) out[i] = ndtri(p[i]);
}

// points i0 .. i0 + n - 1 of dimensions 0 .. d - 1, component-major (d, n): squeezed u and the 30-bit integers
void sh_sobol(int d, long i0, long n, int scramble, uint64_t seed, uint64_t call, double *u, int32_t *raw) {
    const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
    auto key = [&](uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t r[4]) {
        philox4x32_10(c0, c1, c2, c3, k0, k1, r);
    };
    for (int j = 0; j < d; j++) {
        uint32_t w[32], sv[kSobolBits], shift;
        sobol_scramble_words(key, j, call, w);
        sobol_dims(j, scramble, w, sv, shift);
        for (long i = 0; i < n; i++) {
            const uint32_t q = sobol_int(sv, shift, (uint64_t)(i0 + i));
            if (raw) raw[(long)j * n + i] = (int32_t)q;
            if (u) u[(long)j * n + i] = squeeze(q);
        }
    }
}

// Hilbert_to_int of n points of d int64 coordinates, row-major (n, d)
void sh_hilbert_keys(const int64_t *c, long n, int d, int64_t *out) {
    for (long i = 0; i < n; i++) out[i] = hilbert_key(c + i * d, d);
}

}  // extern "C"
