// Host build of the pinned particle's weight of the conditional filter (fk_logG0 / fk_logG, particles_b200/csrc/
// smcb_models.cuh) so that it can be checked on the CPU against the oracle's logG at given states
// (tests/test_pmcmc_host.py).  It reuses the CUDA shim, the model headers and the dispatch table of
// tests/math_host.cpp by including that file whole; compile it the same way, with -ffp-contract=off:
//   g++ -O2 -std=c++17 -ffp-contract=off -shared -fPIC -I particles_b200/csrc -I include tests/pmcmc_host.cpp
#include "math_host.cpp"

extern "C" {
// out[i] = logG(t, xp[i], x[i]) of the 1-D model / kind (t = 0: logG(0, None, x[i]), xp unread).  Returns 0, or -3
// when the combination has no fused kernel.
int mh_fk_logG(int model, int fk, const double *params, const double *data, long T, const double *sc, long t,
               const double *xp, const double *x, long n, double *out) {
    using namespace smcb;
    const StepK k = make_step(data, T, 1, sc, t);
    return with_model(model, 1, [&](auto m) {
        using M = decltype(m);
        if constexpr (M::D != 1) {
            return -3;
        } else {
            return with_fk<M>(fk, [&](auto kind) {
                constexpr int FK = decltype(kind)::value;
                M mm;
                mm.load(params);
                for (long i = 0; i < n; i++)
                    out[i] = t == 0 ? fk_logG0<M, FK>(mm, k, x[i]) : fk_logG<M, FK>(mm, k, xp[i], x[i]);
                return 0;
            });
        }
    });
}
}
