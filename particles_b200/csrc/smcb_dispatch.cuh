// smcb_dispatch.cuh -- the one table from the run-time ids of the C ABI (model and dim, Feynman-Kac kind,
// resampling scheme) to the template arguments of the kernels.  Host code only; tests/math_host.cpp compiles it
// with g++.
//
// Each function calls f with a tag of the selected type or value and returns what f returns.  An id that names
// nothing, or a kind the model cannot run, returns SMCB_ENOSYS without calling f and without setting an error:
// the caller words its own message.
#pragma once
#include <type_traits>

#include "smcb_models.cuh"

namespace smcb {

// f(M{}) for the model of `model`; `dim` picks MvLinGaussM<2|3|4> and is not checked for the other models
template <class F>
int with_model(int model, int dim, F &&f) {
    switch (model) {
        case SMCB_MODEL_STOCHVOL: return f(StochVolM{});
        case SMCB_MODEL_LINGAUSS: return f(LinGaussM{});
        case SMCB_MODEL_GORDON: return f(GordonM{});
        case SMCB_MODEL_THETALOGISTIC: return f(ThetaLogisticM{});
        case SMCB_MODEL_BEARINGS: return f(BearingsM{});
        case SMCB_MODEL_MVLINGAUSS:
            if (dim == 2) return f(MvLinGaussM<2>{});
            if (dim == 3) return f(MvLinGaussM<3>{});
            if (dim == 4) return f(MvLinGaussM<4>{});
            return SMCB_ENOSYS;
        case SMCB_MODEL_DISCRETECOX: return f(DiscreteCoxM{});
        case SMCB_MODEL_STOCHVOLLEV: return f(StochVolLevM{});
        default: return SMCB_ENOSYS;
    }
}

// f(std::integral_constant<int, FK>) for the Feynman-Kac kind `fk`; the kinds that need the model's proposal and
// logeta exist only for models that have them
template <class M, class F>
int with_fk(int fk, F &&f) {
    if (fk == SMCB_FK_BOOTSTRAP) return f(std::integral_constant<int, SMCB_FK_BOOTSTRAP>{});
    if constexpr (M::has_proposal) {
        if (fk == SMCB_FK_GUIDED) return f(std::integral_constant<int, SMCB_FK_GUIDED>{});
        if (fk == SMCB_FK_APF) return f(std::integral_constant<int, SMCB_FK_APF>{});
        if (fk == SMCB_FK_AUXBOOT) return f(std::integral_constant<int, SMCB_FK_AUXBOOT>{});
    }
    return SMCB_ENOSYS;
}

// f(std::integral_constant<int, SCHEME>) for the three resampling schemes of the fused kernels
template <class F>
int with_scheme(int scheme, F &&f) {
    switch (scheme) {
        case SMCB_RS_SYSTEMATIC: return f(std::integral_constant<int, SMCB_RS_SYSTEMATIC>{});
        case SMCB_RS_STRATIFIED: return f(std::integral_constant<int, SMCB_RS_STRATIFIED>{});
        case SMCB_RS_MULTINOMIAL: return f(std::integral_constant<int, SMCB_RS_MULTINOMIAL>{});
        default: return SMCB_ENOSYS;
    }
}

}  // namespace smcb
