// SwiFTly -- size dispatch of finish_facet with a real output (real images), in a translation
// unit of its own so that it compiles in parallel with the complex form.
#include "dispatch_finish_facet.cuh"

namespace swiftly {

template int run_finish_facet<FinishFacetRealOp>(const swiftly_b200*, const FinishFacetRealOp&,
                                                 bool, cudaStream_t);

}  // namespace swiftly
