// smcb_filter_1d.cu -- instantiations of the fused step kernels for the remaining 1-D stock models
// (Gordon et al, ThetaLogistic, DiscreteCox, StochVolLeverage); a separate translation unit only so
// that the library builds in parallel.  See smcb_step.cuh.
#include "smcb_step.cuh"

int smcb_bind_1d_more(smcb_filter *f) {
    switch (f->desc.model) {
        case SMCB_MODEL_GORDON: return bind_fk<GordonM>(f);
        case SMCB_MODEL_THETALOGISTIC: return bind_fk<ThetaLogisticM>(f);
        case SMCB_MODEL_DISCRETECOX: return bind_fk<DiscreteCoxM>(f);
        case SMCB_MODEL_STOCHVOLLEV: return bind_fk<StochVolLevM>(f);
        default:
            set_error("fused filter: model id %d is not available in the fused 1-D family", f->desc.model);
            return SMCB_ENOSYS;
    }
}
