// SwiFTly -- size dispatch of finish_facet with a real output from half-row accumulators (real
// images), in a translation unit of its own so that it compiles in parallel with the other forms.
#include "dispatch_finish_facet.cuh"

namespace swiftly {

template int run_finish_facet<FinishFacetRealHalfOp>(const swiftly_b200*,
                                                     const FinishFacetRealHalfOp&, bool,
                                                     cudaStream_t);

}  // namespace swiftly
