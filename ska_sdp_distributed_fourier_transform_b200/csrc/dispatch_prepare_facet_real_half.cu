// SwiFTly -- size dispatch of prepare_facet from a real facet into half rows (real images).
#include "dispatch.cuh"

namespace swiftly {

int run_prepare_facet_real_half(const swiftly_b200* h, const PrepareFacetRealHalfOp& op, bool lf,
                                cudaStream_t s) {
    return run_line_op<+1>(h, op, lf, s);
}

}  // namespace swiftly
