// SwiFTly -- size dispatch of extract_columns (one translation unit per primitive keeps
// the heavy FP64 template instantiations compiling in parallel).
#include "dispatch.cuh"
#include "extract_tma.cuh"
#include "extract_park.cuh"

namespace swiftly {

// TMA-staged K2 (extract_tma.cuh): persistent CTAs, the facet row of the next line is copied
// into shared memory by the bulk-copy engine while the current line is transformed
template <int H, bool SPLIT, bool HALF>
static int launch_extract_tma(const swiftly_b200* h, const ExtractColumnsOp& op, int max_fs,
                              cudaStream_t s) {
    typedef ExtractColumnsTmaKernel<H, SPLIT, HALF> K;
    K k;
    static thread_local typename K::Maps maps;
    k.op = op;
    k.tw = twiddles(h, H);
    k.tw2 = SPLIT ? twiddles_full(h, 2 * H) : nullptr;
    if (!k.tw || (SPLIT && !k.tw2)) return SWIFTLY_B200_ECUDA;
    k.in_cap = (max_fs + 1) & ~1;
    // swizzled tensor loads when every facet row is whole 128-byte chunks (sg_variant 6: linear)
    const int n_facets = (int)(op.g.n_lines / op.lines_per);
    k.swizzled = h->sg_variant != 6 ? 1 : 0;
    k.box_chunks = 8;
    for (int f = 0; f < n_facets && k.swizzled; ++f)
        if (op.fac[f].fs % 8 != 0 || op.fac[f].in_ls < op.fac[f].fs) k.swizzled = 0;
    if (k.swizzled) {
        int chunks = max_fs / 8;
        k.box_chunks = chunks >= 256 ? 256 : (chunks & ~7);
        if (k.box_chunks < 8) k.swizzled = 0;
    }
    if (k.swizzled) {
        // staging capacity: whole boxes
        const int boxes = (max_fs / 8 + k.box_chunks - 1) / k.box_chunks;
        k.in_cap = boxes * k.box_chunks * 8;
        for (int f = 0; f < n_facets && k.swizzled; ++f)
            if (!make_row_map(&maps.in_map[f], op.fac[f].in, op.fac[f].in_ls, op.rows, op.fac[f].fs,
                              k.box_chunks))
                k.swizzled = 0;
        if (!k.swizzled) k.in_cap = (max_fs + 1) & ~1;
    }
    if (K::smem_bytes(k.in_cap) > (size_t)227 * 1024) {
        k.swizzled = 0;
        k.in_cap = (max_fs + 1) & ~1;
    }
    const size_t smem = K::smem_bytes(k.in_cap);
    int per_sm = (int)((size_t)227 * 1024 / smem);
    if (per_sm > 512 / K::THREADS) per_sm = 512 / K::THREADS;
    if (per_sm < 1) per_sm = 1;
    int64_t blocks = (int64_t)NUM_SMS * per_sm;
    if (blocks > op.g.n_lines) blocks = op.g.n_lines;
    if (h->max_blocks > 0 && blocks > h->max_blocks) blocks = h->max_blocks;
    k.scratch = nullptr;
    if (SPLIT) {
        k.scratch = split_scratch(h, s, (size_t)blocks * H);
        if (!k.scratch) return SWIFTLY_B200_ECUDA;
    }
    note_launch(h, SPLIT ? LAUNCH_K2_TMA_SPLIT : LAUNCH_K2_TMA, k.swizzled ? k.box_chunks : 0,
                k.in_cap, (int)blocks);
    cudaError_t e = launch_body_maps(k, maps, (int)blocks, smem, s);
    return e == cudaSuccess ? SWIFTLY_B200_OK : cuda_fail(e, "extract_columns (TMA) kernel launch");
}

// kernel code of swiftly_b200_debug_last_launch (plan.h)
template <class K>
struct K2Code;
template <int Q, bool HALF>
struct K2Code<ExtractColumnsTma4Kernel<Q, HALF>> {
    static const int value = LAUNCH_K2_TMA4;
};
template <int Q, bool BOTH>
struct K2Code<ExtractColumnsTmaDifKernel<Q, BOTH>> {
    static const int value = LAUNCH_K2_DIF;
};
template <int Q, int MODE>
struct K2Code<ExtractColumnsParkKernel<Q, MODE>> {
    static const int value = MODE == 0 ? LAUNCH_K2_PARK_DIF
                           : MODE == 1 ? LAUNCH_K2_PARK_DIF2 : LAUNCH_K2_PARK_DIT;
};
template <int Q>
struct K2Code<ExtractColumnsParkSkewKernel<Q>> {
    static const int value = LAUNCH_K2_PARK_SKEW;
};

// staging of the 4 x Q kernels: swizzled tensor loads when every facet row is whole 128-byte
// chunks and the buffer in whole boxes fits (sg_variant 6: linear), else linear bulk copies.
// Fills k.in_cap / swizzled / box_chunks and the row maps; returns the shared memory of a CTA,
// 0 when even the linear staging does not fit
template <class K>
static size_t stage_extract_tma4(const swiftly_b200* h, const ExtractColumnsOp& op, int max_fs,
                                 K& k, typename K::Maps& maps) {
    const int n_facets = (int)(op.g.n_lines / op.lines_per);
    k.in_cap = (max_fs + 1) & ~1;
    k.swizzled = h->sg_variant != 6 ? 1 : 0;
    k.box_chunks = 8;
    for (int f = 0; f < n_facets && k.swizzled; ++f)
        if (op.fac[f].fs % 8 != 0 || op.fac[f].in_ls < op.fac[f].fs) k.swizzled = 0;
    if (k.swizzled) {
        int chunks = max_fs / 8;
        k.box_chunks = chunks >= 256 ? 256 : (chunks & ~7);
        if (k.box_chunks < 8) k.swizzled = 0;
    }
    if (k.swizzled) {
        const int boxes = (max_fs / 8 + k.box_chunks - 1) / k.box_chunks;
        k.in_cap = boxes * k.box_chunks * 8;
        for (int f = 0; f < n_facets && k.swizzled; ++f)
            if (!make_row_map(&maps.in_map[f], op.fac[f].in, op.fac[f].in_ls, op.rows, op.fac[f].fs,
                              k.box_chunks))
                k.swizzled = 0;
        if (!k.swizzled) k.in_cap = (max_fs + 1) & ~1;
    }
    if (K::smem_bytes(k.in_cap) > (size_t)227 * 1024) {
        k.swizzled = 0;
        k.in_cap = (max_fs + 1) & ~1;
    }
    const size_t smem = K::smem_bytes(k.in_cap);
    return smem > (size_t)227 * 1024 ? 0 : smem;
}

// 4 x Q split with two thread groups (extract_tma.cuh)
template <int Q, class K>
static int launch_extract_tma4(const swiftly_b200* h, const ExtractColumnsOp& op, int max_fs,
                               cudaStream_t s, int scratch_lines) {
    K k;
    static thread_local typename K::Maps maps;
    k.op = op;
    k.tw = twiddles(h, Q);
    k.twf = twiddles_full(h, 4 * Q);
    if (!k.tw || !k.twf) return SWIFTLY_B200_ECUDA;
    const size_t smem = stage_extract_tma4(h, op, max_fs, k, maps);
    if (!smem) return -1;
    int per_sm = (int)((size_t)227 * 1024 / smem);
    if (per_sm > 512 / K::THREADS) per_sm = 512 / K::THREADS;  // 128 registers per thread
    if (per_sm < 1) per_sm = 1;
    int64_t blocks = (int64_t)NUM_SMS * per_sm;
    if (blocks > op.g.n_lines) blocks = op.g.n_lines;
    if (h->max_blocks > 0 && blocks > h->max_blocks) blocks = h->max_blocks;
    k.scratch = nullptr;
    if (scratch_lines > 0) {
        k.scratch = split_scratch(h, s, (size_t)blocks * scratch_lines * Q);
        if (!k.scratch) return SWIFTLY_B200_ECUDA;
    }
    note_launch(h, K2Code<K>::value, k.swizzled ? k.box_chunks : 0, k.in_cap, (int)blocks);
    cudaError_t e = launch_body_maps(k, maps, (int)blocks, smem, s);
    return e == cudaSuccess ? SWIFTLY_B200_OK
                            : cuda_fail(e, "extract_columns (TMA, 4-way split) kernel launch");
}

// 4 x Q split on two-CTA clusters (extract_tma.cuh): the grid of the single-CTA form (one CTA per
// SM, at most one per line, at most max_blocks), its CTAs paired.  Returns -1 when that grid is
// odd or the device cannot hold all its clusters at once (then the single-CTA form runs on it).
template <int Q, bool HALF>
static int launch_extract_cluster(const swiftly_b200* h, const ExtractColumnsOp& op, int max_fs,
                                  cudaStream_t s) {
    typedef ExtractColumnsClusterKernel<Q, HALF> K;
    K k;
    static thread_local typename K::Maps maps;
    k.op = op;
    k.tw = twiddles(h, Q);
    k.twf = twiddles_full(h, 4 * Q);
    if (!k.tw || !k.twf) return SWIFTLY_B200_ECUDA;
    const size_t smem = stage_extract_tma4(h, op, max_fs, k, maps);
    if (!smem) return -1;
    int64_t blocks = NUM_SMS;  // one CTA of 512 threads per SM, as launch_extract_tma4
    if (blocks > op.g.n_lines) blocks = op.g.n_lines;
    if (h->max_blocks > 0 && blocks > h->max_blocks) blocks = h->max_blocks;
    if (blocks % K::CLUSTER != 0) return -1;
    int clusters = 0;
    cudaError_t e = launch_body_maps_cluster(k, maps, 0, smem, s, &clusters);
    if (e != cudaSuccess) return cuda_fail(e, "extract_columns (TMA, cluster) occupancy query");
    if (clusters < blocks / K::CLUSTER) return -1;
    note_launch(h, LAUNCH_K2_TMA4, k.swizzled ? k.box_chunks : 0, k.in_cap, (int)blocks, K::CLUSTER);
    e = launch_body_maps_cluster(k, maps, (int)blocks, smem, s, nullptr);
    return e == cudaSuccess ? SWIFTLY_B200_OK
                            : cuda_fail(e, "extract_columns (TMA, cluster) kernel launch");
}

// K2 with intermediate results parked in L2-resident scratch (extract_park.cuh): PARK samples
// per CTA, i.e. PARK / Q scratch lines
template <int Q, class K>
static int launch_extract_park(const swiftly_b200* h, const ExtractColumnsOp& op, int max_fs,
                               cudaStream_t s) {
    return launch_extract_tma4<Q, K>(h, op, max_fs, s, K::PARK / Q);
}

// the MODE 0 / 1 parking kernels store pairs of samples as one 32-byte sector: every output line
// must start on a 32-byte boundary
static bool pair_store_ok(const ExtractColumnsOp& op, int n_facets) {
    for (int f = 0; f < n_facets; ++f) {
        if ((op.fac[f].out_ls & 1) != 0) return false;
#if !defined(SWIFTLY_EMU)  // (the emulated pair store is two plain stores: host buffers are only 16-byte aligned)
        if (((uintptr_t)op.fac[f].out & 31) != 0) return false;
#endif
    }
    return true;
}

// returns -1 when the TMA-staged kernel does not apply (then the generic kernels run).  HALF:
// half rows (op.rows = yN/2 + 1) through the default forms only; the debug-selectable ones
// (sg_variant 15, 17, 18, 19 and the emulator's force_split 3 .. 6) have no half instantiation
template <bool HALF>
static int try_extract_tma(const swiftly_b200* h, const ExtractColumnsOp& op, cudaStream_t s) {
    const int n = op.n;
    const int n_facets = (int)(op.g.n_lines / op.lines_per);
    int max_fs = 0;
    for (int f = 0; f < n_facets; ++f) {
        if (op.fac[f].fs > max_fs) max_fs = op.fac[f].fs;
        if (op.fac[f].fs < 1) return -1;
    }
    const bool split = n > MAX_DIRECT_FFT || h->force_split;
    const int hh = split ? n / 2 : n;
    // staging buffer + exchange buffer must fit the 227 KiB of one SM
    if ((size_t)((max_fs + 1) & ~1) * 16 + (size_t)(hh + hh / 16) * 8 + 16 > (size_t)227 * 1024)
        return -1;
    if (split) {
        // 4 x (n/4) with two thread groups (default for 16384; sg_variant 7 / force_split 1:
        // the 2 x (n/2) kernel)
        if (h->sg_variant != 7 && h->force_split != 1) {
            switch (n) {
                case 16384: {
                    // DEFAULT: the 4 x Q form on two-CTA clusters that combine through
                    // distributed shared memory (extract_tma.cuh); 26: the same on one CTA with
                    // the combine through an L2 scratch, which also runs when the grid cannot be
                    // paired.  The forms that park intermediate results per thread in
                    // L2-resident scratch (extract_park.cuh) stay selectable: 19 = DIT within and
                    // across the groups, store phases half a line apart; 18 = the same without the
                    // skew; 17 = DIF across the groups, 32-byte pair stores; 15 = two independent
                    // groups, 16-byte stores at 32-byte stride.  Measured on an H100 80GB HBM3
                    // (700 W), 8 facets of pre-windowed rows (tools/quick_k2.py): default 1.56 ms,
                    // 26: 2.19 (2.23 in an earlier session, with 17: 3.14, 18: 3.78, 19: 4.01,
                    // 15: 3.98).
                    if (!HALF && h->sg_variant == 17 && pair_store_ok(op, n_facets)) {
                        int rc = max_fs <= n / 2
                            ? launch_extract_park<4096, ExtractColumnsParkKernel<4096, 0>>(h, op, max_fs, s)
                            : launch_extract_park<4096, ExtractColumnsParkKernel<4096, 1>>(h, op, max_fs, s);
                        if (rc != -1) return rc;
                    }
                    if (!HALF && h->sg_variant == 18) {
                        int rc = launch_extract_park<4096, ExtractColumnsParkKernel<4096, 2>>(h, op, max_fs, s);
                        if (rc != -1) return rc;
                    }
                    if (!HALF && h->sg_variant == 19) {
                        int rc = launch_extract_park<4096, ExtractColumnsParkSkewKernel<4096>>(h, op, max_fs, s);
                        if (rc != -1) return rc;
                    }
                    if (HALF || (h->sg_variant != 15 && h->sg_variant != 26)) {
                        int rc = launch_extract_cluster<4096, HALF>(h, op, max_fs, s);
                        if (rc != -1) return rc;
                    }
                    int rc = HALF || h->sg_variant != 15
                        ? launch_extract_tma4<4096, ExtractColumnsTma4Kernel<4096, HALF>>(h, op, max_fs, s, 4)
                        : (max_fs <= n / 2
                           ? launch_extract_tma4<4096, ExtractColumnsTmaDifKernel<4096, false>>(h, op, max_fs, s, 2)
                           : launch_extract_tma4<4096, ExtractColumnsTmaDifKernel<4096, true>>(h, op, max_fs, s, 2));
                    if (rc != -1) return rc;
                    break;
                }
#if defined(SWIFTLY_EMU)
                case 512: {
                    if (!HALF && h->force_split == 4 && pair_store_ok(op, n_facets)) {
                        int rc = max_fs <= n / 2
                            ? launch_extract_park<128, ExtractColumnsParkKernel<128, 0>>(h, op, max_fs, s)
                            : launch_extract_park<128, ExtractColumnsParkKernel<128, 1>>(h, op, max_fs, s);
                        if (rc != -1) return rc;
                    }
                    if (!HALF && h->force_split == 5) {
                        int rc = launch_extract_park<128, ExtractColumnsParkKernel<128, 2>>(h, op, max_fs, s);
                        if (rc != -1) return rc;
                    }
                    if (!HALF && h->force_split == 6) {
                        int rc = launch_extract_park<128, ExtractColumnsParkSkewKernel<128>>(h, op, max_fs, s);
                        if (rc != -1) return rc;
                    }
                    // force_split 2: as the default at yN = 16384, 7: as sg_variant 26
                    if (h->force_split == 2) {
                        int rc = launch_extract_cluster<128, HALF>(h, op, max_fs, s);
                        if (rc != -1) return rc;
                    }
                    int rc = HALF || h->force_split != 3
                        ? launch_extract_tma4<128, ExtractColumnsTma4Kernel<128, HALF>>(h, op, max_fs, s, 4)
                        : (max_fs <= n / 2
                           ? launch_extract_tma4<128, ExtractColumnsTmaDifKernel<128, false>>(h, op, max_fs, s, 2)
                           : launch_extract_tma4<128, ExtractColumnsTmaDifKernel<128, true>>(h, op, max_fs, s, 2));
                    if (rc != -1) return rc;
                    break;
                }
#endif
                default: break;
            }
        }
        switch (n) {
            case 16384: return launch_extract_tma<8192, true, HALF>(h, op, max_fs, s);
#if defined(SWIFTLY_EMU)
            case 512: return launch_extract_tma<256, true, HALF>(h, op, max_fs, s);
#endif
            default: return -1;
        }
    }
    switch (n) {
#if defined(SWIFTLY_EMU)
        case 128: return launch_extract_tma<128, false, HALF>(h, op, max_fs, s);
        case 512: return launch_extract_tma<512, false, HALF>(h, op, max_fs, s);
#endif
        case 1024: return launch_extract_tma<1024, false, HALF>(h, op, max_fs, s);
        case 2048: return launch_extract_tma<2048, false, HALF>(h, op, max_fs, s);
        case 4096: return launch_extract_tma<4096, false, HALF>(h, op, max_fs, s);
        case 8192: return launch_extract_tma<8192, false, HALF>(h, op, max_fs, s);
        default: return -1;
    }
}

// Op: ExtractColumnsOp, or ExtractColumnsHalfOp for half rows (no debug forms: sg_variant 3 and 4
// do not apply to it either)
template <class Op>
static int run_extract_columns_op(const swiftly_b200* h, const Op& op, bool lf, cudaStream_t s) {
    constexpr bool HALF = std::is_same<Op, ExtractColumnsHalfOp>::value;
    const int n = op.n;
    if (HALF || (h->sg_variant != 4 && h->sg_variant != 3)) {  // 4: round-1 kernels (debug hook)
        int rc = try_extract_tma<HALF>(h, op, s);
        if (rc != -1) return rc;
    }
    if (h->force_split && n >= 2 * MIN_FFT && n <= MAX_DIRECT_FFT) {
        switch (n) {
#if defined(SWIFTLY_EMU)
            case 128: return launch_split<64, +1, Op>(h, op, s);
            case 512: return launch_split<256, +1, Op>(h, op, s);
#endif
            default: break;
        }
    }
    if (!HALF && h->sg_variant == 3 && n == 16384)  // experiment: 4 x 4096 split, 256-thread CTAs
        return launch_split_f<4096, +1, Op>(h, op, 4, s);
    switch (n) {
        SW_DIRECT_CASES(+1, Op)
        case 16384: return launch_split<8192, +1, Op>(h, op, s);
        default: break;
    }
    {
        int M = 0, F = 0;
        if (split_f_plan(n, &M, &F)) {
            SW_SPLIT_F_CASES(+1, Op, M, F)
        }
    }
    return unsupported(n);
}

int run_extract_columns(const swiftly_b200* h, const ExtractColumnsOp& op, bool lf, cudaStream_t s) {
    return run_extract_columns_op(h, op, lf, s);
}

int run_extract_columns_half(const swiftly_b200* h, const ExtractColumnsHalfOp& op, bool lf,
                             cudaStream_t s) {
    return run_extract_columns_op(h, op, lf, s);
}

}  // namespace swiftly
