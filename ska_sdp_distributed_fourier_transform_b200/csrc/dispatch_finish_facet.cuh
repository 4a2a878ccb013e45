// SwiFTly -- size dispatch of finish_facet, shared by the complex (FinishFacetOp) and the real
// (FinishFacetRealOp) output; each op is instantiated in its own translation unit.
#pragma once

#include "dispatch.cuh"

namespace swiftly {

template <class Op>
int run_finish_facet(const swiftly_b200* h, const Op& op, bool lf, cudaStream_t s) {
    const int n = op.n;
    if (h->force_split && n >= 2 * MIN_FFT && n <= MAX_DIRECT_FFT) {
        switch (n) {
#if defined(SWIFTLY_EMU)
            case 128: return launch_split<64, -1, Op>(h, op, s);
            case 512: return launch_split<256, -1, Op>(h, op, s);
#endif
            default: break;
        }
    }
    switch (n) {
        SW_DIRECT_CASES(-1, Op)
        case 16384: return launch_split<8192, -1, Op>(h, op, s);
        default: break;
    }
    {
        int M = 0, F = 0;
        if (split_f_plan(n, &M, &F)) {
            SW_SPLIT_F_CASES(-1, Op, M, F)
        }
    }
    return unsupported(n);
}

}  // namespace swiftly
