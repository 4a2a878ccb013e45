// SwiFTly -- dispatch of the fused subgrid split kernel (backward direction) over (m, xM) pairs.
#include "dispatch.cuh"

namespace swiftly {

template <int M, int XM, int LINES>
static int launch_split_pair_l(const swiftly_b200* h, const SubgridSplitArgs& a, cudaStream_t s) {
    SubgridSplitAxisKernel<M, XM, LINES> k;
    for (int i = 0; i < SW_MAX_SOURCES; ++i) k.tgt[i] = a.tgt[i];
    for (int g = 0; g < SW_MAX_GROUPS; ++g) k.grp[g] = a.grp[g];
    k.n_groups = a.n_groups;
    k.n_lines = a.n_lines;
    k.add = a.add;
    k.yN = (int)h->yN;
    k.fn = h->d_Fn;
    k.tw_m = twiddles(h, M);
    k.tw_x = twiddles(h, XM);
    if (!k.tw_m || !k.tw_x) return SWIFTLY_B200_ECUDA;
    k.scale = 1.0 / (double)M;
    int grid = grid_for((a.n_lines + LINES - 1) / LINES, 1);
    if (h->max_blocks > 0 && grid > h->max_blocks) grid = h->max_blocks;  // (test hook)
    cudaError_t e = launch_body(k, grid, k.SMEM, s);
    return e == cudaSuccess ? SWIFTLY_B200_OK : cuda_fail(e, "subgrid split kernel launch");
}

// two adjacent lines per CTA when the inputs and every target have unit line stride (axis-0
// work on C-ordered arrays) and two lines' shared memory fits, as for SubgridAxisKernel
template <int M, int XM>
static int launch_split_pair(const swiftly_b200* h, const SubgridSplitArgs& a, cudaStream_t s) {
    bool adjacent = a.n_lines > 1;
    for (int g = 0; g < a.n_groups && adjacent; ++g)
        if (a.grp[g].in_ls != 1) adjacent = false;
    for (int i = 0; i < SW_MAX_SOURCES && adjacent; ++i)
        if (a.tgt[i].base && a.tgt[i].ls != 1) adjacent = false;
    if constexpr (SubgridSplitAxisKernel<M, XM, 2>::SMEM <= 227 * 1024) {
        if (adjacent) return launch_split_pair_l<M, XM, 2>(h, a, s);
    }
    return launch_split_pair_l<M, XM, 1>(h, a, s);
}

// the pairs of SW_SG_PAIRS (dispatch_subgrid_axis.cu): every (m, xM) of the parameter catalogue
#define SW_SPLIT_PAIRS(X) \
    X(32, 64) X(32, 128) X(64, 128) X(64, 256) X(128, 256) X(128, 512) X(256, 512) X(256, 1024) \
    X(512, 1024) X(512, 2048) X(1024, 2048) X(1024, 4096) X(2048, 4096) X(2048, 8192)         \
    X(128, 1024) X(256, 256) X(128, 384) X(160, 320) X(192, 384) X(224, 448)

int subgrid_split_conc(int m, int xM) {
#define X(M, XM) if (m == M && xM == XM) return SubgridSplitAxisKernel<M, XM, 1>::CONC;
    SW_SPLIT_PAIRS(X)
#undef X
    return 0;
}

int run_subgrid_split(const swiftly_b200* h, const SubgridSplitArgs& a, cudaStream_t s) {
    const int m = (int)h->m, xM = (int)h->xM;
#define X(M, XM) if (m == M && xM == XM) return launch_split_pair<M, XM>(h, a, s);
    SW_SPLIT_PAIRS(X)
#undef X
    set_error("no fused subgrid split kernel for m=" + std::to_string(m) +
              ", xM=" + std::to_string(xM));
    return SWIFTLY_B200_EUNSUPPORTED;
}

}  // namespace swiftly
