// smcb_filter_nd.cu -- instantiations of the fused step kernels for the d-dimensional models
// (SoA state): BearingsOnly (d = 4) and MVLinearGauss (dx = 2..4).  smcb_filter.cu dispatches to them.
// See smcb_step.cuh.
#include "smcb_step.cuh"

template int bind_fk<BearingsM>(smcb_filter *);
template int bind_fk<MvLinGaussM<2>>(smcb_filter *);
template int bind_fk<MvLinGaussM<3>>(smcb_filter *);
template int bind_fk<MvLinGaussM<4>>(smcb_filter *);
