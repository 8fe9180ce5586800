// The branch-sum algebra of csrc/smcb_variance.cuh compiled for the CPU (tests/test_variance_host.py): rows cut into
// chunks of C elements, each folded in index order, the chunk segments merged left to right or by the fixed tree.
#include <cmath>
#include <cstdint>
#include <vector>

#define __device__
#define __host__
#define __forceinline__ inline

#include "smcb_variance.cuh"

using smcb::VarSeg;

extern "C" {

// out[0] = the branch sum of squares, out[1] = B[0] == B[N-1], out[2] = "not sorted"
void vh_branch_sums(const int64_t *B, const double *v, int64_t N, int64_t C, int tree, double *out) {
    std::vector<VarSeg> rec;
    for (int64_t i0 = 0; i0 < N; i0 += C) {
        const int64_t i1 = i0 + C < N ? i0 + C : N;
        rec.push_back(smcb::varseg_fold(B, i0, i1, [&](int64_t i) { return v[i]; }));
    }
    VarSeg all = smcb::varseg_empty();
    if (tree) {
        all = smcb::varseg_tree(rec.data(), (int64_t)rec.size());
    } else {
        for (const VarSeg &s : rec) all = smcb::varseg_merge(all, s);
    }
    out[0] = smcb::varseg_total(all);
    out[1] = all.b0 == all.b1 ? 1.0 : 0.0;
    out[2] = all.bad ? 1.0 : 0.0;
}
}
