// smcb_scan.cuh -- inclusive prefix sum of non-negative fp64 (or int64) values
// (the CDF walked by inverse_cdf, particles/resampling.py:484-509).
//
// Reduce-then-scan.  The tiles of kScanTile values are grouped into <= kScanMaxChunks contiguous chunks, one CTA
// each: pass 1 (scan_chunk_sums) sums every chunk, with no dependence between chunks; pass 2 (scan_chunks) lets
// every CTA derive its chunk's base from the chunk sums and scan its chunk tile by tile with a local carry.  One
// more read of the input than a single-pass scan (3 N instead of 2 N words of traffic), but no serial chain of
// dependent global round trips over all tiles.  Two properties make the result a pure function of the input:
//   * every association order is fixed: the chunk bases come from one CTA-wide scan of the chunk sums in a fixed
//     order (identical bits in every CTA), and inside a chunk the tile bases are P_{t+1} = fl(P_t + a_t) in tile
//     order.  Timing and scheduling never change the output.
//   * every level (thread, warp, tile, chunk) clamps its values into the interval spanned by its own base and the
//     base of its successor, which makes the output non-decreasing BY CONSTRUCTION.  np.searchsorted on it is then
//     well defined and the search kernel can be held to it bit-exactly.
#pragma once
#include "smcb_common.cuh"

namespace smcb {

constexpr int kScanItems = 8;                       // fp64 values per thread
constexpr int kScanTile = kBlock * kScanItems;      // 2048 values per tile


struct ScanState {          // a scan slot of the context workspace
    void *chunk_sum;        // [<= kScanMaxChunks] chunk sums of pass 1
};

inline int64_t scan_tiles(int64_t n) { return (n + kScanTile - 1) / kScanTile; }
// bytes the context workspace reserves per scan slot (it grows with the tile count; run_search keeps its tile
// bounds in slot 0)
inline size_t scan_state_bytes(int64_t n) {
    int64_t t = scan_tiles(n);
    return 16 + 8 * (size_t)t + 8 * (size_t)(t + 2);
}

template <typename T> __device__ __forceinline__ T tmin(T a, T b) { return b < a ? b : a; }
template <typename T> __device__ __forceinline__ T tmax(T a, T b) { return a < b ? b : a; }
__device__ __forceinline__ void store_items(double *out, int64_t i0, const double (&o)[8]) {
#pragma unroll
    for (int j = 0; j < 8; j += 2) st2(out + i0 + j, o[j], o[j + 1]);
}
__device__ __forceinline__ void store_items(long long *out, int64_t i0, const long long (&o)[8]) {
#pragma unroll
    for (int j = 0; j < 8; j += 2)
        *reinterpret_cast<longlong2 *>(out + i0 + j) = make_longlong2(o[j], o[j + 1]);
}

// inclusive warp scan (Kogge-Stone) followed by a running max: non-decreasing in lane
template <typename T>
__device__ __forceinline__ T warp_scan_monotone(T v, int lane) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        T o = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= d) v = v + o;
    }
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        T o = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= d) v = tmax(v, o);
    }
    return v;
}

constexpr int kScanMaxChunks = 4 * kBlock;          // the chunk-sum prefix is taken by one CTA-wide scan, 4 per thread

// LOAD: struct with  __device__ void operator()(int64_t i0, int64_t n, T (&v)[8]) const
// filling v[j] with the value at index i0 + j (0 beyond n).  T = double or long long.
template <typename T, typename LOAD>
__device__ __forceinline__ void scan_chunk_sums(const LOAD &load, int64_t n, int tiles_per_chunk, T *chunk_sum) {
    __shared__ T s_w[kBlock / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t t0 = (int64_t)blockIdx.x * tiles_per_chunk;
    T acc = 0;
    for (int k = 0; k < tiles_per_chunk; k++) {
        const int64_t i0 = (t0 + k) * kScanTile + (int64_t)tid * kScanItems;
        if ((t0 + k) * kScanTile >= n) break;
        T r[kScanItems];
        load(i0, n, r);
        T a = r[0];
#pragma unroll
        for (int j = 1; j < kScanItems; j++) a = a + r[j];
        acc = acc + a;
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) acc = acc + __shfl_xor_sync(0xffffffffu, acc, d);
    if (lane == 0) s_w[warp] = acc;
    __syncthreads();
    if (tid == 0) {
        T t = 0;
#pragma unroll
        for (int w = 0; w < kBlock / 32; w++) t = t + s_w[w];
        chunk_sum[blockIdx.x] = t;
    }
}

template <typename T, typename LOAD>
__device__ __forceinline__ void scan_chunks(const LOAD &load, int64_t n, int tiles_per_chunk, const T *chunk_sum,
                                            int nchunks, T *out) {
    __shared__ T s_warp[kBlock / 32];
    __shared__ T s_pref[2];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // base of this chunk: inclusive scan of the chunk sums, 4 consecutive sums per thread, fixed order
    {
        T c[4];
#pragma unroll
        for (int j = 0; j < 4; j++) c[j] = (4 * tid + j < nchunks) ? chunk_sum[4 * tid + j] : (T)0;
#pragma unroll
        for (int j = 1; j < 4; j++) c[j] = c[j - 1] + c[j];
        const T iw = warp_scan_monotone(c[3], lane);
        if (lane == 31) s_warp[warp] = iw;
        __syncthreads();
        T woff = 0;
#pragma unroll
        for (int w = 0; w < kBlock / 32; w++)
            if (w < warp) woff = woff + s_warp[w];
        const T up = __shfl_up_sync(0xffffffffu, iw, 1);
        const T excl = (lane == 0) ? woff : (woff + up);
        const int b = (int)blockIdx.x;
        // the base of chunk b is the LARGEST inclusive prefix of chunks 0..b-1, not the prefix of chunk b - 1 alone:
        // excl + c[j] rounds differently on either side of a thread boundary, so after a chunk that sums to 0 the
        // prefix of chunk b - 1 can fall below that of chunk b - 2 -- and below what CTA b - 1 clamped its last
        // value to.  The max is exact, so CTA b's base is bit for bit CTA b - 1's upper clamp p_next.
        __shared__ T s_max[kBlock / 32];
        T pm = (T)0;
#pragma unroll
        for (int j = 0; j < 4; j++)
            if (4 * tid + j < b) pm = tmax(pm, excl + c[j]);
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) pm = tmax(pm, __shfl_xor_sync(0xffffffffu, pm, d));
        if (lane == 0) s_max[warp] = pm;
#pragma unroll
        for (int j = 0; j < 4; j++)
            if (4 * tid + j == b) s_pref[1] = excl + c[j];               // inclusive prefix of chunk b
        __syncthreads();
        if (tid == 0) {
            T m = s_max[0];
#pragma unroll
            for (int w = 1; w < kBlock / 32; w++) m = tmax(m, s_max[w]);
            s_pref[0] = m;
        }
        __syncthreads();
    }
    const T p_b = s_pref[0];
    const T p_next = tmax(s_pref[1], p_b);
    __syncthreads();
    const int64_t t0 = (int64_t)blockIdx.x * tiles_per_chunk;
    T carry = 0;
    T nxt[kScanItems];                                   // the next tile's values are requested before this one is scanned
    if (t0 * kScanTile < n) load(t0 * kScanTile + (int64_t)tid * kScanItems, n, nxt);
    for (int k = 0; k < tiles_per_chunk; k++) {
        if ((t0 + k) * kScanTile >= n) break;
        const int64_t i0 = (t0 + k) * kScanTile + (int64_t)tid * kScanItems;
        T r[kScanItems];
#pragma unroll
        for (int j = 0; j < kScanItems; j++) r[j] = nxt[j];
        if (k + 1 < tiles_per_chunk && (t0 + k + 1) * kScanTile < n) load(i0 + kScanTile, n, nxt);
#pragma unroll
        for (int j = 1; j < kScanItems; j++) r[j] = r[j - 1] + r[j];
        const T iw = warp_scan_monotone(r[kScanItems - 1], lane);
        if (lane == 31) s_warp[warp] = iw;
        __syncthreads();
        T woff = 0, total = 0;
#pragma unroll
        for (int w = 0; w < kBlock / 32; w++) {
            if (w < warp) woff = woff + s_warp[w];
            total = total + s_warp[w];
        }
        const T incl = woff + iw;
        const T up = __shfl_up_sync(0xffffffffu, iw, 1);
        const T excl = (lane == 0) ? woff : (woff + up);
        const T b_i = tmin(p_b + carry, p_next);
        const T carry_next = carry + total;
        const T b_next = tmin(p_b + carry_next, p_next);
        const T tb = b_i + excl;
        const T cap = tmin(b_i + incl, b_next);
        T o[kScanItems];
#pragma unroll
        for (int j = 0; j < kScanItems; j++) o[j] = tmin(tb + r[j], cap);
        if (i0 + kScanItems <= n) {
            store_items(out, i0, o);
        } else {
#pragma unroll
            for (int j = 0; j < kScanItems; j++)
                if (i0 + j < n) out[i0 + j] = o[j];
        }
        carry = carry_next;
        __syncthreads();
    }
}

}  // namespace smcb
