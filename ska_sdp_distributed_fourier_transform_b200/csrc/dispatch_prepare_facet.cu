// SwiFTly -- size dispatch of prepare_facet (one translation unit per primitive keeps
// the heavy FP64 template instantiations compiling in parallel).
#include "dispatch.cuh"

namespace swiftly {

int run_prepare_facet(const swiftly_b200* h, const PrepareFacetOp& op, bool lf, cudaStream_t s) {
    return run_line_op<+1>(h, op, lf, s);
}

}  // namespace swiftly
