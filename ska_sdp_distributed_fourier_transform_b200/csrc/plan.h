// SwiFTly -- plan (handle) definition shared by the C-ABI translation units.
#pragma once

#include <map>
#include <mutex>
#include <string>

#include "../../include/swiftly_b200.h"
#include "common.cuh"
#include "kernels.cuh"

struct swiftly_b200 {
    double W;
    int64_t N, xM, yN, m;
    int device;
    double* d_Fb;  // yN - 1
    double* d_Fn;  // m
    // twiddle tables keyed by n (compact per-pass table) or -n (full table, t < n/2)
    mutable std::mutex mu;
    mutable std::map<int, swiftly::cplx*> tw;
    // scratch lines of the split (2 x n/2) kernels, one buffer per stream: (pointer, samples)
    mutable std::map<cudaStream_t, std::pair<swiftly::cplx*, size_t>> scratch;
    int force_split;  // debug / test: transform yN lines with the 2 x yN/2 split path
    int sg_variant;   // debug / test: fused subgrid kernel variant (dispatch_subgrid_axis.cu)
    int max_blocks;   // debug / test: cap of the persistent kernels' grid (0: none), so that a
                      // small test problem walks several lines per CTA
    // debug / test: what the last fused subgrid, line, split, window-copy or extract_columns
    // launch ran (kernel, lines per CTA or F or chunks per tensor load, output path or
    // line-fastest flag or staging capacity, grid), see swiftly_b200_debug_last_launch
    mutable int last_launch[4];
};

namespace swiftly {

void set_error(const std::string& msg);
int cuda_fail(cudaError_t e, const char* what);

// returns the table for size n (creating it on first use), nullptr on failure
const cplx* twiddles(const swiftly_b200* h, int n);
// full table exp(-2 pi i t / n), t < n / 2
const cplx* twiddles_full(const swiftly_b200* h, int n);
// per-stream scratch of at least `samples` complex samples (grown on demand)
cplx* split_scratch(const swiftly_b200* h, cudaStream_t s, size_t samples);

// kernel codes of swiftly_b200_debug_last_launch; 1 .. 3 are the fused subgrid kernels
// (dispatch_subgrid_axis.cu, dispatch_subgrid_split.cu)
enum {
    LAUNCH_LINE = 4,        // LineKernel: lines per CTA, line-fastest flag
    LAUNCH_SPLIT_LINE = 5,  // SplitLineKernel: F = 2, flag 0
    LAUNCH_SPLIT_F = 6,     // SplitFKernel: F, flag 0
    LAUNCH_WINDOW_COPY = 7, // WindowCopyKernel: 0, line-fastest flag
    // the TMA-staged extract_columns kernels (dispatch_extract_columns.cu): chunks per tensor
    // load when the rows are staged swizzled, 0 when by linear bulk copies; capacity of the
    // staging buffer in samples
    LAUNCH_K2_TMA = 8,         // ExtractColumnsTmaKernel<yN, false>
    LAUNCH_K2_TMA_SPLIT = 9,   // ExtractColumnsTmaKernel<yN / 2, true>
    LAUNCH_K2_TMA4 = 10,       // ExtractColumnsTma4Kernel<yN / 4>
    LAUNCH_K2_DIF = 11,        // ExtractColumnsTmaDifKernel<yN / 4, BOTH>
    LAUNCH_K2_PARK_DIF = 12,   // ExtractColumnsParkKernel<yN / 4, 0>: facets of at most yN / 2
    LAUNCH_K2_PARK_DIF2 = 13,  // ExtractColumnsParkKernel<yN / 4, 1>: longer facets
    LAUNCH_K2_PARK_DIT = 14,   // ExtractColumnsParkKernel<yN / 4, 2>
    LAUNCH_K2_PARK_SKEW = 15   // ExtractColumnsParkSkewKernel<yN / 4>
};

// records the form of a launch for swiftly_b200_debug_last_launch (one host-side store)
inline void note_launch(const swiftly_b200* h, int kernel, int lines, int out_path, int grid) {
    h->last_launch[0] = kernel;
    h->last_launch[1] = lines;
    h->last_launch[2] = out_path;
    h->last_launch[3] = grid;
}

// SMs of the H100 SXM: grid size of the persistent kernels and cap of the grid-stride ones
static const int NUM_SMS = 132;

// largest directly supported power-of-two line length (fits shared memory)
static const int MAX_DIRECT_FFT = 8192;
static const int MIN_FFT = 16;
inline bool is_pow2(int64_t n) { return n > 0 && (n & (n - 1)) == 0; }

// dispatchers, one translation unit each (compile time!): launch `op` over all
// its lines with an n-point transform.  dir = -1 forward, +1 inverse.
int run_prepare_facet(const swiftly_b200* h, const PrepareFacetOp& op, bool line_fastest, cudaStream_t s);
int run_finish_facet(const swiftly_b200* h, const FinishFacetOp& op, bool line_fastest, cudaStream_t s);
int run_add_to_subgrid(const swiftly_b200* h, const AddToSubgridOp& op, bool line_fastest, cudaStream_t s);
int run_extract_from_subgrid(const swiftly_b200* h, const ExtractFromSubgridOp& op, bool line_fastest, cudaStream_t s);
int run_finish_subgrid(const swiftly_b200* h, const FinishSubgridOp& op, bool line_fastest, cudaStream_t s);
int run_prepare_subgrid(const swiftly_b200* h, const PrepareSubgridOp& op, bool line_fastest, cudaStream_t s);
int run_prepare_facet_pass_a(const swiftly_b200* h, const PrepareFacetPassAOp& op, cudaStream_t s);
int run_prepare_facet_pass_b(const swiftly_b200* h, const PrepareFacetPassBOp& op, cudaStream_t s);
int run_subgrid_to_facets(const swiftly_b200* h, const SubgridToFacetsOp& op, bool line_fastest, cudaStream_t s);
int run_fold_column(const swiftly_b200* h, const FoldColumnOp& op, bool line_fastest, cudaStream_t s);
int run_extract_columns(const swiftly_b200* h, const ExtractColumnsOp& op, bool line_fastest, cudaStream_t s);

// fused subgrid axis kernel (dispatch_subgrid_axis.cu); `k` carries everything but the tables
struct SubgridAxisArgs {
    SgSource src[SW_MAX_SOURCES];
    int n_slots;   // per group
    int n_groups;
    int64_t n_lines;  // per group
    cplx* out;
    int64_t out_ls, out_es, out_gs;
    int sz;
    int start[SW_MAX_GROUPS];
    const double* mask[SW_MAX_GROUPS];
    int first_round_tiles;
    int accumulate_out;  // add to `out` instead of overwriting it (later pieces of a split job)
    // optional per-group output base pointers (groups that live in DIFFERENT allocations,
    // e.g. the peers' receive buffers of the multi-GPU driver); null: out + g * out_gs
    cplx* out_g[SW_MAX_GROUPS];
};
// rank-4 tensor map over an output array with arbitrary line / sample / group strides
// (tensor_map.cu); slot[0..2] receive the coordinate slots of line / sample / group
bool make_out_map(TensorMap4* tm, cplx* out, int64_t out_ls, int64_t out_es, int64_t out_gs,
                  int64_t n_lines, int64_t sz, int64_t n_groups, int box_rows, int* slot);

// rank-4 map for staging rows of a complex128 array in shared memory, 128-byte swizzled
bool make_row_map(TensorMap4* tm, const cplx* base, int64_t ls, int64_t n_rows, int64_t fs,
                  int box_chunks);

// returns SWIFTLY_B200_EUNSUPPORTED (without setting up anything) when the (m, xM) pair has no
// fused instantiation; conc_out receives the number of sources processed concurrently
int subgrid_axis_conc(int m, int xM);
int run_subgrid_axis(const swiftly_b200* h, const SubgridAxisArgs& a, cudaStream_t s);

// fused subgrid split kernel (dispatch_subgrid_split.cu), the backward direction's adjoint of
// the above: groups share the line count; targets are [grp[g].first, + grp[g].count)
struct SubgridSplitArgs {
    SplitTarget tgt[SW_MAX_SOURCES];
    SplitGroup grp[SW_MAX_GROUPS];
    int n_groups;
    int64_t n_lines;
    int add;
};
// concurrent m-point transforms per line (xM / m, at least 1), 0 if the pair has no kernel
int subgrid_split_conc(int m, int xM);
int run_subgrid_split(const swiftly_b200* h, const SubgridSplitArgs& a, cudaStream_t s);

}  // namespace swiftly
