// smcb_variance.cuh -- the branch-sum algebra of the genealogy-based variance estimators
// (particles/variance_estimators.py): sum over Eve values b of (sum_{m: B_m = b} v_m)^2 for a SORTED row B, so that
// every branch is a contiguous run.  A row is cut into fixed chunks; each chunk folds into a VarSeg, and segments
// merge left to right.  The merge is associative in exact arithmetic; the device fixes the order of every merge as a
// function of N alone, so the bits never depend on the launch geometry.
//
// These functions are plain __host__ __device__ code: tests/variance_host.cpp compiles them for the CPU.
#pragma once
#include <stdint.h>

namespace smcb {

// A segment of a row: empty (n == 0); one run (one != 0: Eve b0 == b1, partial sum s0); or a first run (b0, s0), a
// last run (b1, s1) and q = the sum of the squared sums of the complete runs in between.  b0 / b1 are also the first
// and last Eve values of the segment, so a merge sees a decreasing step (bad: the row is not sorted).
struct VarSeg {
    int64_t b0, b1;
    double s0, s1, q;
    int32_t one, bad;
    int64_t n;
};

__host__ __device__ __forceinline__ VarSeg varseg_empty() {
    VarSeg r;
    r.b0 = r.b1 = 0;
    r.s0 = r.s1 = r.q = 0.0;
    r.one = 1;
    r.bad = 0;
    r.n = 0;
    return r;
}

__host__ __device__ __forceinline__ VarSeg varseg_leaf(int64_t b, double v) {
    VarSeg r;
    r.b0 = r.b1 = b;
    r.s0 = v;
    r.s1 = r.q = 0.0;
    r.one = 1;
    r.bad = 0;
    r.n = 1;
    return r;
}

// a followed by c
__host__ __device__ __forceinline__ VarSeg varseg_merge(const VarSeg &a, const VarSeg &c) {
    if (a.n == 0) return c;
    if (c.n == 0) return a;
    VarSeg r;
    r.n = a.n + c.n;
    r.bad = a.bad | c.bad | (a.b1 > c.b0 ? 1 : 0);
    const bool join = a.b1 == c.b0;                 // the last run of a continues into c
    r.b0 = a.b0;
    r.b1 = c.b1;
    if (a.one && c.one) {
        if (join) {
            r.one = 1;
            r.s0 = a.s0 + c.s0;
            r.s1 = r.q = 0.0;
        } else {
            r.one = 0;
            r.s0 = a.s0;
            r.s1 = c.s0;
            r.q = 0.0;
        }
    } else if (a.one) {
        r.one = 0;
        r.s1 = c.s1;
        if (join) {
            r.s0 = a.s0 + c.s0;
            r.q = c.q;
        } else {
            r.s0 = a.s0;
            r.q = c.s0 * c.s0 + c.q;
        }
    } else if (c.one) {
        r.one = 0;
        r.s0 = a.s0;
        if (join) {
            r.s1 = a.s1 + c.s0;
            r.q = a.q;
        } else {
            r.s1 = c.s0;
            r.q = a.q + a.s1 * a.s1;
        }
    } else {
        r.one = 0;
        r.s0 = a.s0;
        r.s1 = c.s1;
        const double mid = join ? (a.s1 + c.s0) * (a.s1 + c.s0) : a.s1 * a.s1 + c.s0 * c.s0;
        r.q = a.q + mid + c.q;
    }
    return r;
}

// the sum over the segment's branches of the squared branch sums
__host__ __device__ __forceinline__ double varseg_total(const VarSeg &a) {
    if (a.n == 0) return 0.0;
    if (a.one) return a.s0 * a.s0;
    return a.s0 * a.s0 + a.q + a.s1 * a.s1;
}

// One chunk [i0, i1) of a row, folded element by element in index order: v(i) is the summand of element i.
template <class V>
__host__ __device__ __forceinline__ VarSeg varseg_fold(const int64_t *B, int64_t i0, int64_t i1, V v) {
    VarSeg s = varseg_empty();
    for (int64_t i = i0; i < i1; i++) s = varseg_merge(s, varseg_leaf(B[i], v(i)));
    return s;
}

// Merge of n records in a fixed pairwise tree over their positions (level by level, neighbours 2^l apart): the
// order of every addition depends on n only.  Works in place on rec[0, n).
__host__ __device__ __forceinline__ VarSeg varseg_tree(VarSeg *rec, int64_t n) {
    for (int64_t w = 1; w < n; w <<= 1)
        for (int64_t i = 0; i + w < n; i += 2 * w) rec[i] = varseg_merge(rec[i], rec[i + w]);
    return n > 0 ? rec[0] : varseg_empty();
}

}  // namespace smcb
