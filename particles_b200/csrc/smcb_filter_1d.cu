// smcb_filter_1d.cu -- instantiations of the fused step kernels for the remaining 1-D stock models
// (Gordon et al, ThetaLogistic, DiscreteCox, StochVolLeverage); a separate translation unit only so
// that the library builds in parallel.  smcb_filter.cu dispatches to them.  See smcb_step.cuh.
#include "smcb_step.cuh"

template int bind_fk<GordonM>(smcb_filter *);
template int bind_fk<ThetaLogisticM>(smcb_filter *);
template int bind_fk<DiscreteCoxM>(smcb_filter *);
template int bind_fk<StochVolLevM>(smcb_filter *);
