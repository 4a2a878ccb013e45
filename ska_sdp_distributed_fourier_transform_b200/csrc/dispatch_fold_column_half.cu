// SwiFTly -- size dispatch of fold_column into half-row facet accumulators (real images).
#include "dispatch.cuh"

namespace swiftly {

int run_fold_column_half(const swiftly_b200* h, const FoldColumnHalfOp& op, bool lf,
                         cudaStream_t s) {
    return run_line_op<-1>(h, op, lf, s);
}

}  // namespace swiftly
