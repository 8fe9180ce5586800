// Host build of the backward samplers' transition density (TransDensity / trans_logpdf, particles_b200/csrc/
// smcb_models.cuh) so that it can be checked on the CPU against the oracle's PX(t, xp).logpdf(x)
// (tests/test_smoothing_host.py).  It reuses the CUDA shim and the model headers of tests/math_host.cpp by including
// that file whole, and adds one export; compile it the same way, with -ffp-contract=off:
//   g++ -O2 -std=c++17 -ffp-contract=off -shared -fPIC -I particles_b200/csrc -I include tests/trans_host.cpp
#include "math_host.cpp"

namespace {
using namespace smcb;
template <class M>
void trans_all(const double *params, const StepK &k, const double *xp, const double *x, long n, double *out) {
    M m;
    m.load(params);
    constexpr int D = M::D;
    for (long i = 0; i < n; i++) {
        double xpi[D], xi[D];
        for (int c = 0; c < D; c++) { xpi[c] = xp[(size_t)c * n + i]; xi[c] = x[(size_t)c * n + i]; }
        out[i] = trans_logpdf<M>(m, k, xpi, xi);
    }
}
}  // namespace

extern "C" {
// PX(t, xp).logpdf(x); xp / x SoA (dim, n); `t` is the time of x (Gordon's step constant sc[t]).
// Returns 0, or -3 when the model has no device transition density.
int mh_trans_logpdf(int model, int dim, const double *params, const double *sc, long t, const double *xp,
                    const double *x, long n, double *out) {
    StepK k{};
    k.t = t;
    k.sc0 = sc ? sc[t] : 0.0;
    switch (model) {
        case SMCB_MODEL_STOCHVOL: trans_all<StochVolM>(params, k, xp, x, n, out); return 0;
        case SMCB_MODEL_LINGAUSS: trans_all<LinGaussM>(params, k, xp, x, n, out); return 0;
        case SMCB_MODEL_GORDON: trans_all<GordonM>(params, k, xp, x, n, out); return 0;
        case SMCB_MODEL_THETALOGISTIC: trans_all<ThetaLogisticM>(params, k, xp, x, n, out); return 0;
        case SMCB_MODEL_DISCRETECOX: trans_all<DiscreteCoxM>(params, k, xp, x, n, out); return 0;
        case SMCB_MODEL_STOCHVOLLEV: trans_all<StochVolLevM>(params, k, xp, x, n, out); return 0;
        case SMCB_MODEL_BEARINGS: trans_all<BearingsM>(params, k, xp, x, n, out); return 0;
        case SMCB_MODEL_MVLINGAUSS:
            if (dim == 2) { trans_all<MvLinGaussM<2>>(params, k, xp, x, n, out); return 0; }
            if (dim == 3) { trans_all<MvLinGaussM<3>>(params, k, xp, x, n, out); return 0; }
            if (dim == 4) { trans_all<MvLinGaussM<4>>(params, k, xp, x, n, out); return 0; }
            return -3;
        default: return -3;
    }
}
}
