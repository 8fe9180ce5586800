// smcb_filter_nd.cu -- instantiations of the fused step kernels for the d-dimensional models
// (SoA state): BearingsOnly (d = 4) and MVLinearGauss (dx = 2..4).  See smcb_step.cuh.
#include "smcb_step.cuh"

int smcb_bind_nd(smcb_filter *f) {
    const smcb_filter_desc *d = &f->desc;
    switch (d->model) {
        case SMCB_MODEL_BEARINGS:
            if (d->dim != 4) { set_error("fused BearingsOnly: state dimension must be 4"); return SMCB_EINVAL; }
            return bind_fk<BearingsM>(f);
        case SMCB_MODEL_MVLINGAUSS:
            if (d->dim == 2) return bind_fk<MvLinGaussM<2>>(f);
            if (d->dim == 3) return bind_fk<MvLinGaussM<3>>(f);
            if (d->dim == 4) return bind_fk<MvLinGaussM<4>>(f);
            set_error("fused MVLinearGauss: dx must be 2, 3 or 4 (got %d)", d->dim);
            return SMCB_ENOSYS;
        default:
            set_error("fused filter: model id %d has no d-dimensional kernel", d->model);
            return SMCB_ENOSYS;
    }
}
