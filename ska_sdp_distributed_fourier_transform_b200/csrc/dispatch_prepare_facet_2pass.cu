// SwiFTly -- dispatch of the two-pass (four-step) strided prepare_facet.
#include "dispatch.cuh"

namespace swiftly {

// sub-transform lengths used by the two-pass kernels
#define SW_2PASS_CASES(Op, NN)                                           \
    switch (NN) {                                                        \
        case 16: return launch_lines<16, +1, Op>(h, op, true, s);        \
        case 32: return launch_lines<32, +1, Op>(h, op, true, s);        \
        case 64: return launch_lines<64, +1, Op>(h, op, true, s);        \
        case 128: return launch_lines<128, +1, Op>(h, op, true, s);      \
        case 256: return launch_lines<256, +1, Op>(h, op, true, s);      \
        default: return unsupported(NN);                                 \
    }

int run_prepare_facet_pass_a(const swiftly_b200* h, const PrepareFacetPassAOp& op, cudaStream_t s) {
    SW_2PASS_CASES(PrepareFacetPassAOp, op.n1)
}

int run_prepare_facet_pass_b(const swiftly_b200* h, const PrepareFacetPassBOp& op, cudaStream_t s) {
    SW_2PASS_CASES(PrepareFacetPassBOp, op.n2)
}

// real facet into half rows (real images)
int run_prepare_facet_pass_a_real(const swiftly_b200* h, const PrepareFacetPassARealOp& op,
                                  cudaStream_t s) {
    SW_2PASS_CASES(PrepareFacetPassARealOp, op.n1)
}

int run_prepare_facet_pass_b_half(const swiftly_b200* h, const PrepareFacetPassBHalfOp& op,
                                  cudaStream_t s) {
    SW_2PASS_CASES(PrepareFacetPassBHalfOp, op.n2)
}

}  // namespace swiftly
