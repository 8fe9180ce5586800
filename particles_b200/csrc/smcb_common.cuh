// smcb_common.cuh -- shared device/host helpers of libsmcb (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <math_constants.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/smcb.h"

namespace smcb {

constexpr int kSMs = 132;          // H100 SXM
constexpr int kBlock = 256;        // threads per CTA for the streaming kernels
constexpr int kCtasPerSM = 8;      // 8 x 256 = 2048 resident threads / SM
constexpr int kMaxGrid = kSMs * kCtasPerSM;
constexpr double kHalfLog2Pi = 0.91893853320467274178;  // distributions.py:212

// ---------------------------------------------------------------------------
// error plumbing
// ---------------------------------------------------------------------------
void set_error(const char *fmt, ...);
#define SMCB_CUDA(call)                                                          \
    do {                                                                         \
        cudaError_t e__ = (call);                                                \
        if (e__ != cudaSuccess) {                                                \
            smcb::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call,        \
                            cudaGetErrorString(e__));                            \
            return SMCB_ECUDA;                                                   \
        }                                                                        \
    } while (0)
#define SMCB_REQUIRE(cond, ...)                                                  \
    do {                                                                         \
        if (!(cond)) {                                                           \
            smcb::set_error(__VA_ARGS__);                                        \
            return SMCB_EINVAL;                                                  \
        }                                                                        \
    } while (0)
// returns from the caller with expr's code unless it is SMCB_OK
#define SMCB_TRY(expr)                                                           \
    do {                                                                         \
        const int smcb_rc_ = (expr);                                             \
        if (smcb_rc_ != SMCB_OK) return smcb_rc_;                                \
    } while (0)

constexpr unsigned kFull = 0xffffffffu;   // every lane of a warp

inline int grid_for(int64_t work_items, int items_per_block) {
    int64_t b = (work_items + items_per_block - 1) / items_per_block;
    if (b < 1) b = 1;
    if (b > kMaxGrid) b = kMaxGrid;  // persistent: grid-stride beyond kSMs x 8 CTAs
    return (int)b;
}

// ---------------------------------------------------------------------------
// Philox4x32-10 (Salmon et al. 2011), counter-based: the draw for particle n at
// step t does not depend on the launch geometry or the number of GPUs.
// ---------------------------------------------------------------------------
struct Philox {
    uint32_t k0, k1;
    uint32_t rk[20];   // the 10 round keys (k0 + r*W0, k1 + r*W1), bumped once on the host
};

__host__ __device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2,
                                                       uint32_t c3, uint32_t k0, uint32_t k1,
                                                       uint32_t out[4]) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < 10; r++) {
        uint64_t p0 = (uint64_t)M0 * c0;
        uint64_t p1 = (uint64_t)M1 * c2;
        uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0;
        uint32_t hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
        uint32_t n0 = hi1 ^ c1 ^ k0;
        uint32_t n2 = hi0 ^ c3 ^ k1;
        c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
        k0 += W0; k1 += W1;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// same permutation with the round keys taken from the (constant-bank) Philox struct: saves the
// 18 uniform key bumps per call that the generic version spends
__device__ __forceinline__ void philox4x32_10k(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                               const Philox &key, uint32_t out[4]) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
#pragma unroll
    for (int r = 0; r < 10; r++) {
        const uint32_t hi0 = __umulhi(M0, c0), lo0 = M0 * c0;
        const uint32_t hi1 = __umulhi(M1, c2), lo1 = M1 * c2;
        const uint32_t n0 = hi1 ^ c1 ^ key.rk[2 * r];
        const uint32_t n2 = hi0 ^ c3 ^ key.rk[2 * r + 1];
        c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// Philox purposes: the low byte of counter word 3, so that streams never collide.  Pick a new feature's value here.
// The values used twice are kept apart by another counter word or by the key:
//   4, 5  the backward samplers (Smooth*) and the binary-space kernels (Bin*) both key on the context seed and put the
//         API call number, which every random entry point takes afresh from smcb_ctx::api_counter, in word 2;
//         the on-line smoothers' 5 is under their own key, seed ^ kOnlineSeedMix.
//   6     the binary-space draws (BinRvs) key on the context seed, the conditional SMC trajectory (Traj) on the
//         filter bank's per-filter keys.
enum : uint32_t {
    kPurposeNormal = 1, kPurposeUniform = 2, kPurposeApi = 3,
    kPurposeSmooth = 4,       // a backward draw's proposal + acceptance uniforms of trial `trial`
    kPurposeSmoothExact = 5,  // the uniform of an exact O(N) backward draw
    kPurposeBinProp = 4, kPurposeBinAcc = 5, kPurposeBinRvs = 6,
    kPurposeTraj = 6,         // the uniform of the conditional SMC trajectory draw at step t
    kPurposeHmm = 7,          // the uniform of trajectory n's draw at step t of HMM b
    kPurposeDists = 8,        // block b of element n's draw in the samplers of smcb_dists.cuh (API call in word 2)
    kPurposeSobol = 9,        // word block b of the Sobol' scrambling of dimension j (smcb_sqmc.cuh; call in word 2)
};
constexpr uint64_t kOnlineSeedMix = 0x9E3779B97F4A7C15ull;   // the on-line smoothers' key: seed ^ kOnlineSeedMix

// 53-bit uniform in [0, 1), the construction numpy's legacy rand uses
__host__ __device__ __forceinline__ double u53(uint32_t a, uint32_t b) {
    return (double)(((uint64_t)(a >> 5) << 26) | (uint64_t)(b >> 6)) * (1.0 / 9007199254740992.0);
}
// 53-bit uniform in (0, 1): safe under log()
__host__ __device__ __forceinline__ double u53_open(uint32_t a, uint32_t b) {
    return ((double)(((uint64_t)(a >> 5) << 26) | (uint64_t)(b >> 6)) + 0.5) *
           (1.0 / 9007199254740992.0);
}

// two N(0,1) from one Philox block: Box-Muller, branch-free, fp64
__device__ __forceinline__ void box_muller(const uint32_t r[4], double &z0, double &z1) {
    double u1 = u53_open(r[0], r[1]);
    double u2 = u53(r[2], r[3]);
    double rad = sqrt(-2.0 * log(u1));
    double s, c;
    sincospi(2.0 * u2, &s, &c);
    z0 = rad * c;
    z1 = rad * s;
}

// standard normals for the pair of particles (2p, 2p+1), component k, step t
__device__ __forceinline__ void normal_pair(const Philox &key, uint64_t pair, uint32_t t,
                                            uint32_t comp, double &z0, double &z1) {
    uint32_t r[4];
    philox4x32_10k((uint32_t)pair, (uint32_t)(pair >> 32), t, (comp << 8) | kPurposeNormal, key, r);
    box_muller(r, z0, z1);
}

// uniforms [0,1) for the pair of indices (2p, 2p+1), step t
__device__ __forceinline__ void uniform_pair(const Philox &key, uint64_t pair, uint32_t t,
                                             uint32_t purpose, double &u0, double &u1) {
    uint32_t r[4];
    philox4x32_10k((uint32_t)pair, (uint32_t)(pair >> 32), t, purpose, key, r);
    u0 = u53(r[0], r[1]);
    u1 = u53(r[2], r[3]);
}

// ---------------------------------------------------------------------------
// max-shifted (max, sum exp, sum exp^2) accumulators -- the algebra behind
// Weights.__init__ (resampling.py:217-226), log_sum_exp (247-270), essl (166-188)
// ---------------------------------------------------------------------------
struct Lse3 {
    double m, s, q;  // max, sum exp(v - m), sum exp(2 (v - m))
};

__device__ __forceinline__ Lse3 lse3_empty() { return Lse3{-CUDART_INF, 0.0, 0.0}; }

// add one value with ONE exp: e = exp(-|v - m|) serves both the "new max" rescale
// and the ordinary accumulate
__device__ __forceinline__ void lse3_add(Lse3 &a, double v) {
    if (v == -CUDART_INF) return;  // exp(-inf) = 0 contributes nothing (also avoids inf-inf)
    double d = v - a.m;
    double e = exp(-fabs(d));      // a.m = -inf first time: d = +inf, e = 0
    if (d > 0.0) {
        a.s = a.s * e + 1.0;
        a.q = a.q * (e * e) + 1.0;
        a.m = v;
    } else {
        a.s += e;
        a.q += e * e;
    }
}

__device__ __forceinline__ Lse3 lse3_merge(const Lse3 &a, const Lse3 &b) {
    if (b.m == -CUDART_INF) return a;
    if (a.m == -CUDART_INF) return b;
    double M = fmax(a.m, b.m);
    double ea = exp(a.m - M), eb = exp(b.m - M);
    Lse3 r;
    r.m = M;
    r.s = a.s * ea + b.s * eb;
    r.q = a.q * (ea * ea) + b.q * (eb * eb);
    return r;
}

__device__ __forceinline__ Lse3 lse3_shfl_xor(const Lse3 &a, int mask) {
    Lse3 b;
    b.m = __shfl_xor_sync(0xffffffffu, a.m, mask);
    b.s = __shfl_xor_sync(0xffffffffu, a.s, mask);
    b.q = __shfl_xor_sync(0xffffffffu, a.q, mask);
    return b;
}

// block-wide merge, result valid in thread 0; fixed butterfly order -> deterministic
template <int BLOCK>
__device__ __forceinline__ Lse3 lse3_block_reduce(Lse3 a, Lse3 *smem /* BLOCK/32 */) {
#pragma unroll
    for (int mask = 16; mask > 0; mask >>= 1) a = lse3_merge(a, lse3_shfl_xor(a, mask));
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) smem[warp] = a;
    __syncthreads();
    if (warp == 0) {
        a = (lane < BLOCK / 32) ? smem[lane] : lse3_empty();
#pragma unroll
        for (int mask = 16; mask > 0; mask >>= 1) a = lse3_merge(a, lse3_shfl_xor(a, mask));
    }
    __syncthreads();
    return a;
}

// Normal.logpdf, distributions.py:273-274 (scipy.stats.norm.logpdf): the operation
// order of SURVEY.md section 9 item 2
__device__ __forceinline__ double normal_logpdf(double x, double loc, double scale) {
    double z = (x - loc) / scale;
    return -z * z / 2.0 - kHalfLog2Pi - log(scale);
}

// streaming 16-byte accesses (two fp64 particles per thread)
__device__ __forceinline__ double2 ld2(const double *p) {
    return *reinterpret_cast<const double2 *>(p);
}
__device__ __forceinline__ void st2(double *p, double a, double b) {
    *reinterpret_cast<double2 *>(p) = make_double2(a, b);
}

// ---------------------------------------------------------------------------
// TMA bulk copy global -> shared with mbarrier completion (sm_90+ PTX; SASS UBLKCP + SYNCS).
// One thread arms the barrier with the byte count and issues the copy; every consumer thread
// waits on the barrier's phase parity.  Addresses and sizes are multiples of 16 bytes.
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t arrivals) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(arrivals) : "memory");
}
__device__ __forceinline__ void mbar_init_fence() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(__cvta_generic_to_global(src_gmem)), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// bounded: a barrier that never completes (wrong byte count, faulted copy) traps instead of hanging
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    uint32_t ok = 0;
    for (unsigned int spin = 0; !ok; spin++) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                     "selp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
        if (spin > (1u << 22)) __trap();
    }
}

}  // namespace smcb

struct smcb_ctx {
    int device;
    cudaStream_t stream;
    uint64_t seed;
    uint64_t api_counter;   // advances with every API-level random call
    int64_t launches;
    double *ws;             // workspace: partials / scan slots
    size_t ws_bytes;
    unsigned int *counters; // "last block done" tickets (zeroed, self-resetting)
    double *math_tab;       // smcb_tables.h (64 KB): exp / log / sincos tables of the step kernels
};

namespace smcb {
// workspace layout (doubles): [0, kWsPartials) block partials | 16 scalars | two scan slots
constexpr size_t kWsPartials = 65536;
constexpr size_t kWsBytes = 8u << 20;  // 8 MiB: partials + up to ~1M scan tiles
__host__ __device__ inline Philox key_of(uint64_t seed) {
    Philox k;
    k.k0 = (uint32_t)seed;
    k.k1 = (uint32_t)(seed >> 32);
    for (int r = 0; r < 10; r++) {
        k.rk[2 * r] = k.k0 + (uint32_t)r * 0x9E3779B9u;
        k.rk[2 * r + 1] = k.k1 + (uint32_t)r * 0xBB67AE85u;
    }
    return k;
}

// Launches kern on the context's stream and counts it in ctx->launches (smcb_launch_count).  A launch the runtime
// rejects returns SMCB_ECUDA at once, so no later launch of the same entry point runs on its missing results.
template <class... P, class... A>
int launch(smcb_ctx *ctx, void (*kern)(P...), dim3 grid, dim3 block, size_t smem, A &&...args) {
    kern<<<grid, block, smem, ctx->stream>>>(static_cast<A &&>(args)...);
    ctx->launches++;
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_error("kernel launch: %s", cudaGetErrorString(e));
        return SMCB_ECUDA;
    }
    return SMCB_OK;
}

// lets launches of `kern` use `bytes` of dynamic shared memory
template <class K>
int set_smem(K kern, size_t bytes) {
    SMCB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    return SMCB_OK;
}
}  // namespace smcb
