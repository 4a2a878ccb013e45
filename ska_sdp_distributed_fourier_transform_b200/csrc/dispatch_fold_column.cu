// SwiFTly -- size dispatch of fold_column (one translation unit per primitive keeps
// the heavy FP64 template instantiations compiling in parallel).
#include "dispatch.cuh"

namespace swiftly {

int run_fold_column(const swiftly_b200* h, const FoldColumnOp& op, bool lf, cudaStream_t s) {
    return run_line_op<-1>(h, op, lf, s);
}

}  // namespace swiftly
