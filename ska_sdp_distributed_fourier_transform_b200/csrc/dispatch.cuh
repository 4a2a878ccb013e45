// SwiFTly -- size dispatch for the line-FFT kernels (included by the
// per-primitive translation units dispatch_*.cu).
#pragma once

#include <math.h>

#include "plan.h"

namespace swiftly {

template <int N>
struct LinesPerCta {
    static constexpr int T = FftCfg<N>::T;
    static constexpr int V = T >= 256 ? 1 : ((256 / T) > 16 ? 16 : (256 / T));
};

inline int grid_for(int64_t n_lines, int lpc) {
    int64_t blocks = (n_lines + lpc - 1) / lpc;
    const int64_t cap = NUM_SMS * 32;  // grid-stride loop covers the rest
    return (int)(blocks < cap ? blocks : cap);
}

// grid_for, further capped by the plan's max_blocks (test hook)
inline int grid_for(const swiftly_b200* h, int64_t n_lines, int lpc) {
    int grid = grid_for(n_lines, lpc);
    return h->max_blocks > 0 && grid > h->max_blocks ? h->max_blocks : grid;
}

template <int N, int DIR, class Op>
int launch_lines(const swiftly_b200* h, const Op& op, bool line_fastest, cudaStream_t s) {
    const cplx* tw = twiddles(h, N);
    if (!tw) return SWIFTLY_B200_ECUDA;
    constexpr int LPC = LinesPerCta<N>::V;
    const int grid = grid_for(h, op.g.n_lines, LPC);
    cudaError_t e;
    if (line_fastest && LPC > 1) {
        note_launch(h, LAUNCH_LINE, LPC, 1, grid);
        LineKernel<N, DIR, LPC, true, Op> k{op, tw};
        e = launch_body(k, grid, k.SMEM, s);
    } else {
        note_launch(h, LAUNCH_LINE, LPC, 0, grid);
        LineKernel<N, DIR, LPC, false, Op> k{op, tw};
        e = launch_body(k, grid, k.SMEM, s);
    }
    return e == cudaSuccess ? SWIFTLY_B200_OK : cuda_fail(e, "line FFT kernel launch");
}

template <int H, int DIR, class Op>
int launch_split(const swiftly_b200* h, const Op& op, cudaStream_t s) {
    const cplx* tw = twiddles(h, H);
    const cplx* tw2 = twiddles_full(h, 2 * H);
    if (!tw || !tw2) return SWIFTLY_B200_ECUDA;
    // persistent CTAs: two per SM's worth of lines in flight keeps the scratch L2 resident
    int64_t blocks = op.g.n_lines < 296 ? op.g.n_lines : 296;
    if (h->max_blocks > 0 && blocks > h->max_blocks) blocks = h->max_blocks;  // (test hook)
    cplx* scratch = split_scratch(h, s, (size_t)blocks * H);
    if (!scratch) return SWIFTLY_B200_ECUDA;
    note_launch(h, LAUNCH_SPLIT_LINE, 2, 0, (int)blocks);
    SplitLineKernel<H, DIR, Op> k{op, tw, tw2, scratch};
    cudaError_t e = launch_body(k, (int)blocks, k.SMEM, s);
    return e == cudaSuccess ? SWIFTLY_B200_OK : cuda_fail(e, "split line FFT kernel launch");
}

template <int M, int DIR, class Op>
int launch_split_f(const swiftly_b200* h, const Op& op, int F, cudaStream_t s) {
    const int64_t n = (int64_t)F * M;
    const cplx* tw = twiddles(h, M);
    const cplx* twf = twiddles_full(h, (int)n);
    if (!tw || !twf) return SWIFTLY_B200_ECUDA;
    int64_t blocks = op.g.n_lines < 296 ? op.g.n_lines : 296;
    if (h->max_blocks > 0 && blocks > h->max_blocks) blocks = h->max_blocks;  // (test hook)
    cplx* scratch = split_scratch(h, s, (size_t)blocks * (size_t)(F - 1) * M);
    if (!scratch) return SWIFTLY_B200_ECUDA;
    note_launch(h, LAUNCH_SPLIT_F, F, 0, (int)blocks);
    SplitFKernel<M, DIR, Op> k;
    k.op = op;
    k.tw = tw;
    k.twf = twf;
    k.scratch = scratch;
    k.F = F;
    const long double two_pi = 6.283185307179586476925286766559005768L;
    for (int t = 0; t < SW_MAX_SPLIT_F; ++t) {
        long double a = two_pi * (long double)(t % F) / (long double)F;
        k.wf[t].x = (double)cosl(a);
        k.wf[t].y = (double)(-sinl(a));
    }
    cudaError_t e = launch_body(k, (int)blocks, k.SMEM, s);
    return e == cudaSuccess ? SWIFTLY_B200_OK : cuda_fail(e, "split-F line FFT kernel launch");
}

// n = F * M with M the largest power of two <= 8192 dividing n and 2 <= F <= 16
inline bool split_f_plan(int64_t n, int* M, int* F) {
    if (n < 2 * MIN_FFT || (n & 1)) return false;
    int64_t m = 1;
    while ((n % (2 * m)) == 0 && 2 * m <= MAX_DIRECT_FFT) m *= 2;
    int64_t f = n / m;
    while (f < 2 && m > MIN_FFT) {  // pure power of two above MAX_DIRECT_FFT handled by caller
        m /= 2;
        f = n / m;
    }
    if (m < MIN_FFT || f < 2 || f > SW_MAX_SPLIT_F) return false;
    *M = (int)m;
    *F = (int)f;
    return true;
}

#define SW_SPLIT_F_CASES(DIR, Op, MM, FF)                                       \
    switch (MM) {                                                               \
        case 16: return launch_split_f<16, DIR, Op>(h, op, FF, s);              \
        case 32: return launch_split_f<32, DIR, Op>(h, op, FF, s);              \
        case 64: return launch_split_f<64, DIR, Op>(h, op, FF, s);              \
        case 128: return launch_split_f<128, DIR, Op>(h, op, FF, s);            \
        case 256: return launch_split_f<256, DIR, Op>(h, op, FF, s);            \
        case 512: return launch_split_f<512, DIR, Op>(h, op, FF, s);            \
        case 1024: return launch_split_f<1024, DIR, Op>(h, op, FF, s);          \
        case 2048: return launch_split_f<2048, DIR, Op>(h, op, FF, s);          \
        case 4096: return launch_split_f<4096, DIR, Op>(h, op, FF, s);          \
        case 8192: return launch_split_f<8192, DIR, Op>(h, op, FF, s);          \
        default: break;                                                         \
    }

inline int unsupported(int n) {
    set_error("FFT length " + std::to_string(n) +
              " is not supported by this build (need n = F * 2^k, F <= 16, 16 <= 2^k <= 8192)");
    return SWIFTLY_B200_EUNSUPPORTED;
}

#define SW_DIRECT_CASES(DIR, Op)                                         \
    case 16: return launch_lines<16, DIR, Op>(h, op, lf, s);             \
    case 32: return launch_lines<32, DIR, Op>(h, op, lf, s);             \
    case 64: return launch_lines<64, DIR, Op>(h, op, lf, s);             \
    case 128: return launch_lines<128, DIR, Op>(h, op, lf, s);           \
    case 256: return launch_lines<256, DIR, Op>(h, op, lf, s);           \
    case 512: return launch_lines<512, DIR, Op>(h, op, lf, s);           \
    case 1024: return launch_lines<1024, DIR, Op>(h, op, lf, s);         \
    case 2048: return launch_lines<2048, DIR, Op>(h, op, lf, s);         \
    case 4096: return launch_lines<4096, DIR, Op>(h, op, lf, s);         \
    case 8192: return launch_lines<8192, DIR, Op>(h, op, lf, s);

// The length dispatch of the facet-side line ops (op.n points, DIR = +1 inverse, -1 forward): one
// CTA per line up to 8192, the 2 x 8192 split at 16384, split-F for F * 2^k; force_split (test
// hook) runs the emulator's 128 and 512 as 2 x n/2.
template <int DIR, class Op>
int run_line_op(const swiftly_b200* h, const Op& op, bool lf, cudaStream_t s) {
    const int n = op.n;
    if (h->force_split && n >= 2 * MIN_FFT && n <= MAX_DIRECT_FFT) {
        switch (n) {
#if defined(SWIFTLY_EMU)
            case 128: return launch_split<64, DIR, Op>(h, op, s);
            case 512: return launch_split<256, DIR, Op>(h, op, s);
#endif
            default: break;
        }
    }
    switch (n) {
        SW_DIRECT_CASES(DIR, Op)
        case 16384: return launch_split<8192, DIR, Op>(h, op, s);
        default: break;
    }
    {
        int M = 0, F = 0;
        if (split_f_plan(n, &M, &F)) {
            SW_SPLIT_F_CASES(DIR, Op, M, F)
        }
    }
    return unsupported(n);
}

}  // namespace swiftly
