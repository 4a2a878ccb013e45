// SwiFTly -- size dispatch of finish_facet (one translation unit per primitive keeps
// the heavy FP64 template instantiations compiling in parallel).
#include "dispatch_finish_facet.cuh"

namespace swiftly {

template int run_finish_facet<FinishFacetOp>(const swiftly_b200*, const FinishFacetOp&, bool,
                                             cudaStream_t);

}  // namespace swiftly
