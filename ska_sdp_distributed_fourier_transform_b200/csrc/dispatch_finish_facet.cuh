// SwiFTly -- size dispatch of finish_facet, shared by the complex (FinishFacetOp) and the real
// (FinishFacetRealOp) output; each op is instantiated in its own translation unit.
#pragma once

#include "dispatch.cuh"

namespace swiftly {

template <class Op>
int run_finish_facet(const swiftly_b200* h, const Op& op, bool lf, cudaStream_t s) {
    return run_line_op<-1>(h, op, lf, s);
}

}  // namespace swiftly
