// SwiFTly -- C ABI (include/swiftly_b200.h): plan management, argument
// validation, host staging and the per-primitive entry points.
#include <math.h>
#include <stdio.h>

#include <string>
#include <vector>

#include "capi_util.h"

using namespace swiftly;

// ------------------------------------------------------------------ errors
namespace swiftly {

static thread_local std::string g_last_error;

void set_error(const std::string& msg) { g_last_error = msg; }

int cuda_fail(cudaError_t e, const char* what) {
    set_error(std::string(what) + ": " + cudaGetErrorString(e));
    return SWIFTLY_B200_ECUDA;
}

static const cplx* upload_table(const swiftly_b200* h, int key, const std::vector<cplx>& host) {
    cplx* dev = nullptr;
    cudaError_t e = cudaMalloc((void**)&dev, sizeof(cplx) * host.size());
    if (e != cudaSuccess) {
        cuda_fail(e, "cudaMalloc(twiddles)");
        return nullptr;
    }
    e = cudaMemcpy(dev, host.data(), sizeof(cplx) * host.size(), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        cudaFree(dev);
        cuda_fail(e, "cudaMemcpy(twiddles)");
        return nullptr;
    }
    h->tw[key] = dev;
    return dev;
}

static cplx unit_root(long double num, long double den) {  // exp(-2 pi i num / den)
    const long double two_pi = 6.283185307179586476925286766559005768L;
    long double a = two_pi * num / den;
    cplx w;
    w.x = (double)cosl(a);
    w.y = (double)(-sinl(a));
    return w;
}

// Compact per-pass table of the n-point Stockham plan (fft_engine.cuh): for every pass
// after the first, with sub-transform size Ns (16, 256, 4096) and radix R, the Ns entries
// exp(-2 pi i k / (Ns R)), k < Ns, stored pass after pass.  A mixed-radix length n = F * p
// (p the power-of-two part, line_fft_mixed in fft_engine.cuh) gets the table of the p-point
// plan followed by exp(-2 pi i t / n), t < n.
const cplx* twiddles(const swiftly_b200* h, int n) {
    std::lock_guard<std::mutex> lock(h->mu);
    auto it = h->tw.find(n);
    if (it != h->tw.end()) return it->second;
    std::vector<cplx> host;
    const int p = n & -n;
    for (int ns = 16; ns < p; ns *= 16) {
        const int r = (p / ns >= 16) ? 16 : p / ns;
        for (int k = 0; k < ns; ++k) host.push_back(unit_root(k, (long double)ns * r));
    }
    if (host.empty()) host.push_back(unit_root(0, 1));
    if (p != n)
        for (int t = 0; t < n; ++t) host.push_back(unit_root(t, n));
    return upload_table(h, n, host);
}

// Full table exp(-2 pi i t / n), t < n / 2 (split kernels: the radix-2 DIF pre-twiddle).
const cplx* twiddles_full(const swiftly_b200* h, int n) {
    std::lock_guard<std::mutex> lock(h->mu);
    auto it = h->tw.find(-n);
    if (it != h->tw.end()) return it->second;
    std::vector<cplx> host((size_t)(n / 2));
    for (int t = 0; t < n / 2; ++t) host[t] = unit_root(t, n);
    return upload_table(h, -n, host);
}

cplx* split_scratch(const swiftly_b200* h, cudaStream_t s, size_t samples) {
    std::lock_guard<std::mutex> lock(h->mu);
    auto& slot = h->scratch[s];
    if (slot.first && slot.second >= samples) return slot.first;
    if (slot.first) {
        cudaStreamSynchronize(s);  // kernels on this stream may still use the old buffer
        cudaFree(slot.first);
        slot.first = nullptr;
        slot.second = 0;
    }
    cplx* dev = nullptr;
    cudaError_t e = cudaMalloc((void**)&dev, sizeof(cplx) * samples);
    if (e != cudaSuccess) {
        cuda_fail(e, "cudaMalloc(split scratch)");
        return nullptr;
    }
    slot.first = dev;
    slot.second = samples;
    return dev;
}

}  // namespace swiftly

// ------------------------------------------------------------------ plan
extern "C" const char* swiftly_b200_last_error(void) { return g_last_error.c_str(); }

extern "C" const char* swiftly_b200_build_info(void) {
#if defined(SWIFTLY_EMU)
    return "swiftly_b200 0.1 EMULATED (host fibres; test tooling only)";
#else
    return "swiftly_b200 0.1 cuda sm_90a";
#endif
}

extern "C" int swiftly_b200_create(double W, int64_t N, int64_t xM, int64_t yN, const double* Fb,
                                   const double* Fn, int device, swiftly_b200** plan) {
    if (!plan) return einval("plan output pointer is NULL");
    *plan = nullptr;
    if (N <= 0 || xM <= 0 || yN <= 0) return einval("sizes must be positive");
    // SwiftlyCore.check_params, core.py:55-74
    if (N % yN != 0)
        return einval("Image size " + std::to_string(N) + " not divisible by facet size " +
                      std::to_string(yN) + "!");
    if (N % xM != 0)
        return einval("Image size " + std::to_string(N) + " not divisible by subgrid size " +
                      std::to_string(xM) + "!");
    if ((xM * yN) % N != 0)
        return einval("Contribution size not integer with image size " + std::to_string(N) +
                      ", subgrid size " + std::to_string(xM) + " and facet size " +
                      std::to_string(yN) + "!");
    if (!Fb || !Fn) return einval("Fb / Fn tables must be given");
    DeviceGuard guard(device);
    if (!guard.ok()) return cuda_fail(guard.err, "cudaSetDevice");
    swiftly_b200* h = new swiftly_b200();
    h->W = W;
    h->N = N;
    h->xM = xM;
    h->yN = yN;
    h->m = xM * yN / N;
    h->device = device;
    h->d_Fb = nullptr;
    h->d_Fn = nullptr;
    h->force_split = 0;
    h->sg_variant = 0;
    h->max_blocks = 0;
    for (int i = 0; i < 4; ++i) h->last_launch[i] = 0;
    h->last_cluster = 1;
    h->n_fold_runs = 0;
    cudaError_t e = cudaMalloc((void**)&h->d_Fb, sizeof(double) * (size_t)(yN > 1 ? yN - 1 : 1));
    if (e == cudaSuccess) e = cudaMalloc((void**)&h->d_Fn, sizeof(double) * (size_t)h->m);
    if (e == cudaSuccess)
        e = cudaMemcpy(h->d_Fb, Fb, sizeof(double) * (size_t)(yN - 1), cudaMemcpyHostToDevice);
    if (e == cudaSuccess)
        e = cudaMemcpy(h->d_Fn, Fn, sizeof(double) * (size_t)h->m, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        swiftly_b200_destroy(h);
        return cuda_fail(e, "plan allocation");
    }
    *plan = h;
    return SWIFTLY_B200_OK;
}

extern "C" void swiftly_b200_destroy(swiftly_b200* h) {
    if (!h) return;
    DeviceGuard guard(h->device);
    if (h->d_Fb) cudaFree(h->d_Fb);
    if (h->d_Fn) cudaFree(h->d_Fn);
    for (auto& kv : h->tw) cudaFree(kv.second);
    for (auto& kv : h->scratch)
        if (kv.second.first) cudaFree(kv.second.first);
    delete h;
}

// Free the per-stream scratch buffers of the plan (the two-pass prepare_facet keeps up to 2 GiB
// at N = 65536).  The streaming drivers call this once stage 1 is over, so that the memory is
// available again to the caller's allocator; the small scratch lines of the split kernels are
// re-created on demand.  Synchronises the streams that own a buffer.
extern "C" void swiftly_b200_release_scratch(swiftly_b200* h) {
    if (!h) return;
    DeviceGuard guard(h->device);
    std::lock_guard<std::mutex> lock(h->mu);
    for (auto& kv : h->scratch) {
        if (kv.second.first) {
            cudaStreamSynchronize(kv.first);
            cudaFree(kv.second.first);
            kv.second.first = nullptr;
            kv.second.second = 0;
        }
    }
}

extern "C" int64_t swiftly_b200_contribution_size(const swiftly_b200* h) { return h ? h->m : -1; }

// test hook (not in the public header): force the 2 x n/2 split path
extern "C" void swiftly_b200_debug_force_split(swiftly_b200* h, int on) {
    if (h) h->force_split = on;
}

// test hook (not in the public header): select the fused subgrid kernel variant
extern "C" void swiftly_b200_debug_max_blocks(swiftly_b200* h, int blocks) {
    if (h) h->max_blocks = blocks;
}

extern "C" void swiftly_b200_debug_sg_variant(swiftly_b200* h, int variant) {
    if (h) h->sg_variant = variant;
}

// test hook (not in the public header): the form of the last kernel launch of the plan, so that
// a test can assert the kernel it was written for.  out[0]: kernel (0 none yet, 1 round-1
// SubgridAxisKernel, 2 two-group SubgridAxisKernelPP, 3 split SubgridSplitAxisKernel,
// 4 LineKernel, 5 SplitLineKernel, 6 SplitFKernel, 7 WindowCopyKernel; the TMA-staged
// extract_columns kernels: 8 ExtractColumnsTmaKernel<yN, false>, 9 its 2 x yN/2 split,
// 10 ExtractColumnsTma4Kernel, 11 ExtractColumnsTmaDifKernel, 12 / 13 / 14
// ExtractColumnsParkKernel MODE 0 / 1 / 2, 15 ExtractColumnsParkSkewKernel; 16
// MirrorSubgridKernel and 17 MergeMirrorSubgridKernel, with 0 in out[1] and out[2]); out[1]:
// lines per CTA (1 .. 4), F (5, 6: 2 for SplitLineKernel), 0 (7), or for 8 .. 15 the 128-byte chunks per
// tensor load when the rows are staged swizzled and 0 when they are staged by linear bulk
// copies; out[2]: output path of the fused kernels (0 direct stores, 1 TMA with one tensor map,
// 2 TMA with one tensor map per group), the line-fastest flag of 4 and 7, 0 for 5 and 6, the
// capacity of the staging buffer in samples for 8 .. 15; out[3]: grid size.  An extract_columns
// launch that leaves the TMA-staged kernels records the generic kernel it ran (4, 5 or 6).
extern "C" void swiftly_b200_debug_last_launch(const swiftly_b200* h, int* out) {
    if (h && out)
        for (int i = 0; i < 4; ++i) out[i] = h->last_launch[i];
}

// test hook: CTAs per cluster of the last launch recorded by swiftly_b200_debug_last_launch (2
// when the 4 x Q form of extract_columns ran on two-CTA clusters, else 1)
extern "C" int swiftly_b200_debug_last_cluster(const swiftly_b200* h) {
    return h ? h->last_cluster : 0;
}

// test hook: the runs of the last fold_column call into half-row accumulators, in launch order:
// out[3 i .. 3 i + 2] = (first window row u, rows, pass 1 or 2); returns the number of runs (<= 8)
extern "C" int swiftly_b200_debug_fold_runs(const swiftly_b200* h, int* out) {
    if (!h) return 0;
    if (out)
        for (int i = 0; i < 3 * h->n_fold_runs; ++i) out[i] = h->fold_runs[i];
    return h->n_fold_runs;
}

// ------------------------------------------------------------------ host staging
namespace {

// A device-side view of a caller-provided batch of lines.  Device arrays are used
// in place; host arrays are copied into a temporary device buffer (and back).
struct Staged {
    const swiftly_b200_lines* src;
    cplx* dev = nullptr;        // device base pointer
    int64_t ls = 0, es = 0;     // device strides
    bool owned = false;         // dev is a temporary
    // host copy geometry (2-D copy: rows x width elements)
    int64_t rows = 0, width = 0, host_pitch = 0, dev_pitch = 0;
    ~Staged() {
        if (owned && dev) cudaFree(dev);
    }
};

int stage_in(Staged& st, const swiftly_b200_lines* a, bool copy_contents, cudaStream_t s,
             const char* name) {
    st.src = a;
    if (a->location == SWIFTLY_B200_DEVICE) {
        st.dev = (cplx*)a->data;
        st.ls = a->line_stride;
        st.es = a->elem_stride;
        return SWIFTLY_B200_OK;
    }
    if (a->location != SWIFTLY_B200_HOST) return einval(std::string(name) + ": bad location");
    // a single line has no meaningful line stride: treat a strided one as a column
    const int64_t ls_eff = (a->n_lines == 1 && a->elem_stride != 1) ? 1 : a->line_stride;
    if (a->elem_stride == 1) {
        // lines are rows: device layout [n_lines][size]
        st.rows = a->n_lines;
        st.width = a->size;
        st.host_pitch = a->n_lines == 1 ? a->size : a->line_stride;
        st.dev_pitch = a->size;
        st.ls = a->size;
        st.es = 1;
    } else if (ls_eff == 1) {
        // lines are columns (axis-0 view of a C-ordered array): device layout [size][n_lines]
        st.rows = a->size;
        st.width = a->n_lines;
        st.host_pitch = a->elem_stride;
        st.dev_pitch = a->n_lines;
        st.ls = 1;
        st.es = a->n_lines;
    } else {
        return einval(std::string(name) +
                      ": host arrays must have unit element stride or unit line stride");
    }
    size_t bytes = sizeof(cplx) * (size_t)(st.rows * st.width);
    SW_CUDA(cudaMalloc((void**)&st.dev, bytes ? bytes : 16), "cudaMalloc(staging)");
    st.owned = true;
    if (copy_contents && bytes) {
        SW_CUDA(cudaMemcpy2DAsync(st.dev, sizeof(cplx) * (size_t)st.dev_pitch, a->data,
                                  sizeof(cplx) * (size_t)st.host_pitch,
                                  sizeof(cplx) * (size_t)st.width, (size_t)st.rows,
                                  cudaMemcpyHostToDevice, s),
                "cudaMemcpy2DAsync(H2D)");
    }
    return SWIFTLY_B200_OK;
}

int stage_out(Staged& st, cudaStream_t s) {
    if (!st.owned) return SWIFTLY_B200_OK;
    size_t bytes = sizeof(cplx) * (size_t)(st.rows * st.width);
    if (bytes) {
        SW_CUDA(cudaMemcpy2DAsync(st.src->data, sizeof(cplx) * (size_t)st.host_pitch, st.dev,
                                  sizeof(cplx) * (size_t)st.dev_pitch,
                                  sizeof(cplx) * (size_t)st.width, (size_t)st.rows,
                                  cudaMemcpyDeviceToHost, s),
                "cudaMemcpy2DAsync(D2H)");
    }
    SW_CUDA(cudaStreamSynchronize(s), "cudaStreamSynchronize(staging)");
    return SWIFTLY_B200_OK;
}

// optional per-sample mask living where `out` lives
struct StagedMask {
    const double* dev = nullptr;
    double* tmp = nullptr;
    ~StagedMask() {
        if (tmp) cudaFree(tmp);
    }
};

int stage_mask(StagedMask& sm, const double* mask, int64_t n, int location, cudaStream_t s) {
    if (!mask) return SWIFTLY_B200_OK;
    if (location == SWIFTLY_B200_DEVICE) {
        sm.dev = mask;
        return SWIFTLY_B200_OK;
    }
    SW_CUDA(cudaMalloc((void**)&sm.tmp, sizeof(double) * (size_t)n), "cudaMalloc(mask)");
    SW_CUDA(cudaMemcpyAsync(sm.tmp, mask, sizeof(double) * (size_t)n, cudaMemcpyHostToDevice, s),
            "cudaMemcpyAsync(mask)");
    sm.dev = sm.tmp;
    return SWIFTLY_B200_OK;
}

int check_lines(const swiftly_b200_lines* in, const swiftly_b200_lines* out, int64_t in_size,
                int64_t out_size, const char* what) {
    if (!in || !out) return einval(std::string(what) + ": NULL array descriptor");
    if (!in->data || !out->data) return einval(std::string(what) + ": NULL data pointer");
    if (in->n_lines != out->n_lines)
        return einval(std::string(what) + ": input has " + std::to_string(in->n_lines) +
                      " lines, output " + std::to_string(out->n_lines));
    if (in_size >= 0 && in->size != in_size)
        return einval(std::string(what) + ": input line length is " + std::to_string(in->size) +
                      ", expected " + std::to_string(in_size) + "!");
    if (out_size >= 0 && out->size != out_size)
        return einval(std::string(what) + ": output line length is " + std::to_string(out->size) +
                      ", expected " + std::to_string(out_size) + "!");
    if (in->n_lines < 0 || in->size < 0) return einval(std::string(what) + ": negative shape");
    return SWIFTLY_B200_OK;
}

Lines make_lines(const Staged& in, const Staged& out, int64_t n_lines) {
    Lines g;
    g.in = in.dev;
    g.out = out.dev;
    g.in_ls = in.ls;
    g.in_es = in.es;
    g.out_ls = out.ls;
    g.out_es = out.es;
    g.n_lines = n_lines;
    return g;
}

// lines adjacent in memory (stride 1 between lines): let warps run across lines
bool lines_adjacent(const Lines& g) {
    return g.n_lines > 1 && (g.in_ls == 1 || g.out_ls == 1) && g.in_es != 1;
}

// grid of WindowCopyKernel for `total` samples: one per thread up to 64 CTAs per SM, a
// grid-stride loop beyond; capped by the plan's max_blocks (test hook)
int window_copy_grid(const swiftly_b200* h, int64_t total) {
    const int64_t per_cta = WindowCopyKernel<false>::THREADS;
    int64_t grid = (total + per_cta - 1) / per_cta;
    if (grid > NUM_SMS * 64) grid = NUM_SMS * 64;
    if (h->max_blocks > 0 && grid > h->max_blocks) grid = h->max_blocks;
    return (int)grid;
}

}  // namespace

#define SW_PROLOGUE(what, in_size, out_size, copy_out)                          \
    if (!h) return einval(what ": NULL plan");                                  \
    SW_TRY(check_lines(in, out, in_size, out_size, what));                      \
    if (in->n_lines == 0) return SWIFTLY_B200_OK;                               \
    cudaStream_t s = (cudaStream_t)stream;                                      \
    SW_DEVICE_GUARD(h);                         \
    Staged sin, sout;                                                           \
    SW_TRY(stage_in(sin, in, true, s, what " input"));                          \
    SW_TRY(stage_in(sout, out, copy_out, s, what " output"));                   \
    Lines g = make_lines(sin, sout, in->n_lines);

// ------------------------------------------------------------------ facet -> subgrid
// real_half (always windowed): `in` holds doubles (strides counted in doubles), device arrays
// only, and `out` receives the yN/2 + 1 half rows (PrepareFacetRealHalfOp)
static int prepare_facet_impl(const swiftly_b200* h, const swiftly_b200_lines* in,
                              const swiftly_b200_lines* out, int64_t facet_off, bool windowed,
                              bool real_half, void* stream) {
    if (real_half) {
        if (!h) return einval("prepare_facet_real_half: NULL plan");
        if (h->yN % 2) return einval("prepare_facet_real_half: yN_size must be even");
        if (in && out && (in->location != SWIFTLY_B200_DEVICE || out->location != SWIFTLY_B200_DEVICE))
            return einval("prepare_facet_real_half: device arrays only");
    }
    SW_PROLOGUE("prepare_facet", -1, h ? (real_half ? h->yN / 2 + 1 : h->yN) : -1, false)
    const int64_t yN = h->yN, fs = in->size;
    const double* rin = real_half ? (const double*)in->data : nullptr;
    // windowed: line l of the output is additionally multiplied by Fb_c[l], the window the
    // NEXT prepare_facet (along the other axis) would apply to sample l of its lines
    const double* lw = nullptr;
    if (windowed) {
        if (g.n_lines > yN - 1)
            return einval("prepare_facet_windowed: more lines than the window is long");
        lw = h->d_Fb + ((yN - 1) / 2 - g.n_lines / 2);
    }
    // extract_mid(Fb, fs) needs fs <= len(Fb) = yN - 1 (core.py:213-215)
    if (fs > yN - 1) return einval("prepare_facet: facet size must be at most yN_size - 1");
    // Strided axis with many adjacent lines: two-pass transform with coalesced column runs.
    if (g.in_ls == 1 && g.out_ls == 1 && g.n_lines >= 16 && is_pow2(yN) && yN >= 256 &&
        yN <= 65536 && !h->force_split) {
        int lg = 0;
        while (((int64_t)1 << lg) < yN) ++lg;
        const int n1 = 1 << ((lg + 1) / 2), n2 = (int)(yN / n1);
        const cplx* twf = twiddles_full(h, (int)yN);
        // Column tiles bound the scratch T (yN x tile samples) to 2 GiB.  Tiles small enough to
        // keep T in L2 between the passes make launches so short that their tails cost more
        // than the L2 hits save.
        int64_t tile = ((int64_t)128 << 20) / yN;  // 2 GiB of complex128
        tile = tile / 16 * 16;
        if (tile < 16) tile = 16;
        if (h->sg_variant == 9) tile = ((int64_t)4 << 20) / yN;  // debug hook: 64 MiB tiles
        if (h->sg_variant == 10) tile = 32;  // tests: several tiles, ragged last one
        if (tile > g.n_lines) tile = g.n_lines;
        cplx* scratch = split_scratch(h, s, (size_t)yN * (size_t)tile);
        if (!twf || !scratch) return SWIFTLY_B200_ECUDA;
        for (int64_t c0 = 0; c0 < g.n_lines; c0 += tile) {
            const int64_t nc = g.n_lines - c0 < tile ? g.n_lines - c0 : tile;
            PrepareFacetPassAOp a;
            a.g = g;
            a.g.in = g.in + c0;
            a.g.out = scratch;
            a.g.n_lines = (int64_t)n2 * nc;
            a.fb = h->d_Fb + ((yN - 1) / 2 - fs / 2);
            a.twf = twf;
            a.n = (int)yN;
            a.n1 = n1;
            a.n2 = n2;
            a.fs = (int)fs;
            a.shift_in = (int)pmod(fs / 2 - facet_off, yN);
            a.ncols = (int)nc;
            a.lw = lw ? lw + c0 : nullptr;
            if (real_half) {
                PrepareFacetPassARealOp ar;
                static_cast<PrepareFacetPassAOp&>(ar) = a;
                ar.rin = rin + c0;
                SW_TRY(run_prepare_facet_pass_a_real(h, ar, s));
            } else {
                SW_TRY(run_prepare_facet_pass_a(h, a, s));
            }
            PrepareFacetPassBOp b;
            b.g = g;
            b.g.in = scratch;
            b.g.out = g.out + c0;
            b.g.n_lines = (int64_t)n1 * nc;
            b.n = (int)yN;
            b.n1 = n1;
            b.n2 = n2;
            b.ncols = (int)nc;
            b.scale = 1.0 / (double)yN;
            if (real_half) {
                PrepareFacetPassBHalfOp bh;
                static_cast<PrepareFacetPassBOp&>(bh) = b;
                SW_TRY(run_prepare_facet_pass_b_half(h, bh, s));
            } else {
                SW_TRY(run_prepare_facet_pass_b(h, b, s));
            }
        }
        return stage_out(sout, s);
    }
    PrepareFacetOp op;
    op.g = g;
    op.n = (int)yN;
    op.fs = (int)fs;
    // Fb_c[k] = Fb[(yN-1)//2 - fs//2 + k]   (extract_mid on the yN-1 long table)
    op.fb = h->d_Fb + ((yN - 1) / 2 - fs / 2);
    op.shift_in = (int)pmod(fs / 2 - facet_off, yN);
    op.scale = 1.0 / (double)yN;
    op.rm_m = 0;
    op.rm_s_m = op.rm_base = 0;
    op.rm_mod = 1;
    op.lw = lw;
    if (real_half) {
        PrepareFacetRealHalfOp rop;
        static_cast<PrepareFacetOp&>(rop) = op;
        rop.rin = rin;
        SW_TRY(run_prepare_facet_real_half(h, rop, lines_adjacent(g), s));
    } else {
        SW_TRY(run_prepare_facet(h, op, lines_adjacent(g), s));
    }
    return stage_out(sout, s);
}

extern "C" int swiftly_b200_prepare_facet(const swiftly_b200* h, const swiftly_b200_lines* in,
                                          const swiftly_b200_lines* out, int64_t facet_off,
                                          void* stream) {
    return prepare_facet_impl(h, in, out, facet_off, false, false, stream);
}

// prepare_facet whose output lines are pre-multiplied by the Fb window of the other axis
// (fused forward path: stage 1 hands K2 rows that need no window fetch per sample)
extern "C" int swiftly_b200_prepare_facet_windowed(const swiftly_b200* h,
                                                   const swiftly_b200_lines* in,
                                                   const swiftly_b200_lines* out,
                                                   int64_t facet_off, void* stream) {
    return prepare_facet_impl(h, in, out, facet_off, true, false, stream);
}

// prepare_facet_windowed of a real facet (doubles), only the half rows d <= yN/2 stored
extern "C" int swiftly_b200_prepare_facet_real_half(const swiftly_b200* h,
                                                    const swiftly_b200_lines* in,
                                                    const swiftly_b200_lines* out,
                                                    int64_t facet_off, void* stream) {
    return prepare_facet_impl(h, in, out, facet_off, true, true, stream);
}

extern "C" int swiftly_b200_extract_from_facet(const swiftly_b200* h,
                                               const swiftly_b200_lines* in,
                                               const swiftly_b200_lines* out,
                                               int64_t subgrid_off, void* stream) {
    SW_PROLOGUE("extract_from_facet", h ? h->yN : -1, h ? h->m : -1, false)
    const int64_t yN = h->yN, m = h->m;
    const int64_t sc = floordiv(subgrid_off * yN, h->N);
    WindowCopyKernel<false> k;
    k.g = g;
    k.m = (int)m;
    k.yN = (int)yN;
    k.s_m = (int)pmod(sc, m);
    k.base = (int)pmod(yN / 2 - m / 2 + sc, yN);
    k.line_fastest = lines_adjacent(g) ? 1 : 0;
    const int grid = window_copy_grid(h, g.n_lines * m);
    note_launch(h, LAUNCH_WINDOW_COPY, 0, k.line_fastest, grid);
    SW_CUDA(launch_body(k, grid, 0, s), "extract_from_facet launch");
    return stage_out(sout, s);
}

extern "C" int swiftly_b200_add_to_subgrid(const swiftly_b200* h, const swiftly_b200_lines* in,
                                           const swiftly_b200_lines* out, int64_t facet_off,
                                           void* stream) {
    SW_PROLOGUE("add_to_subgrid", h ? h->m : -1, h ? h->xM : -1, true)
    const int64_t xM = h->xM, m = h->m;
    const int64_t sf = floordiv(facet_off * xM, h->N);
    AddToSubgridOp op;
    op.g = g;
    op.fn = h->d_Fn;
    op.m = (int)m;
    op.xM = (int)xM;
    op.sf_m = (int)pmod(sf, m);
    op.base = (int)pmod(xM / 2 - m / 2 + sf, xM);
    SW_TRY(run_add_to_subgrid(h, op, lines_adjacent(g), s));
    return stage_out(sout, s);
}

extern "C" int swiftly_b200_finish_subgrid(const swiftly_b200* h, const swiftly_b200_lines* in,
                                           const swiftly_b200_lines* out, int64_t subgrid_off,
                                           const double* mask, void* stream) {
    SW_PROLOGUE("finish_subgrid", h ? h->xM : -1, -1, false)
    const int64_t xM = h->xM, sz = out->size;
    if (sz > xM) return einval("finish_subgrid: subgrid size exceeds padded subgrid size");
    StagedMask sm;
    SW_TRY(stage_mask(sm, mask, sz, out->location, s));
    FinishSubgridOp op;
    op.g = g;
    op.xM = (int)xM;
    op.sz = (int)sz;
    op.start = (int)pmod(xM / 2 - sz / 2 + subgrid_off, xM);
    op.scale = 1.0 / (double)xM;
    op.mask = sm.dev;
    SW_TRY(run_finish_subgrid(h, op, lines_adjacent(g), s));
    return stage_out(sout, s);
}

// ------------------------------------------------------------------ subgrid -> facet
extern "C" int swiftly_b200_prepare_subgrid(const swiftly_b200* h, const swiftly_b200_lines* in,
                                            const swiftly_b200_lines* out, int64_t subgrid_off,
                                            void* stream) {
    SW_PROLOGUE("prepare_subgrid", -1, h ? h->xM : -1, false)
    const int64_t xM = h->xM, sz = in->size;
    if (sz > xM) return einval("prepare_subgrid: subgrid size exceeds padded subgrid size");
    PrepareSubgridOp op;
    op.g = g;
    op.xM = (int)xM;
    op.sz = (int)sz;
    op.start = (int)pmod(xM / 2 - sz / 2 + subgrid_off, xM);
    SW_TRY(run_prepare_subgrid(h, op, lines_adjacent(g), s));
    return stage_out(sout, s);
}

extern "C" int swiftly_b200_extract_from_subgrid(const swiftly_b200* h,
                                                 const swiftly_b200_lines* in,
                                                 const swiftly_b200_lines* out,
                                                 int64_t facet_off, void* stream) {
    SW_PROLOGUE("extract_from_subgrid", h ? h->xM : -1, h ? h->m : -1, false)
    const int64_t xM = h->xM, m = h->m;
    const int64_t sf = floordiv(facet_off * xM, h->N);
    ExtractFromSubgridOp op;
    op.g = g;
    op.fn = h->d_Fn;
    op.m = (int)m;
    op.xM = (int)xM;
    op.sf_m = (int)pmod(sf, m);
    op.base = (int)pmod(xM / 2 - m / 2 + sf, xM);
    op.scale = 1.0 / (double)m;
    SW_TRY(run_extract_from_subgrid(h, op, lines_adjacent(g), s));
    return stage_out(sout, s);
}

extern "C" int swiftly_b200_add_to_facet(const swiftly_b200* h, const swiftly_b200_lines* in,
                                         const swiftly_b200_lines* out, int64_t subgrid_off,
                                         void* stream) {
    SW_PROLOGUE("add_to_facet", h ? h->m : -1, h ? h->yN : -1, true)
    const int64_t yN = h->yN, m = h->m;
    const int64_t sc = floordiv(subgrid_off * yN, h->N);
    WindowCopyKernel<true> k;
    k.g = g;
    k.m = (int)m;
    k.yN = (int)yN;
    k.s_m = (int)pmod(sc, m);
    k.base = (int)pmod(yN / 2 - m / 2 + sc, yN);
    k.line_fastest = lines_adjacent(g) ? 1 : 0;
    const int grid = window_copy_grid(h, g.n_lines * m);
    note_launch(h, LAUNCH_WINDOW_COPY, 0, k.line_fastest, grid);
    SW_CUDA(launch_body(k, grid, 0, s), "add_to_facet launch");
    return stage_out(sout, s);
}

extern "C" int swiftly_b200_finish_facet(const swiftly_b200* h, const swiftly_b200_lines* in,
                                         const swiftly_b200_lines* out, int64_t facet_off,
                                         const double* mask, void* stream) {
    SW_PROLOGUE("finish_facet", h ? h->yN : -1, -1, false)
    const int64_t yN = h->yN, fs = out->size;
    if (fs > yN - 1) return einval("finish_facet: facet size must be at most yN_size - 1");
    StagedMask sm;
    SW_TRY(stage_mask(sm, mask, fs, out->location, s));
    FinishFacetOp op;
    op.g = g;
    op.fb = h->d_Fb + ((yN - 1) / 2 - fs / 2);
    op.n = (int)yN;
    op.fs = (int)fs;
    op.start = (int)pmod(yN / 2 - fs / 2 + facet_off, yN);
    op.mask = sm.dev;
    SW_TRY(run_finish_facet(h, op, lines_adjacent(g), s));
    return stage_out(sout, s);
}

// half: `in` holds yN/2 + 1 half-row samples per line (FinishFacetRealHalfOp)
static int finish_facet_real_impl(const swiftly_b200* h, const swiftly_b200_lines* in,
                                  const swiftly_b200_lines* out, int64_t facet_off,
                                  const double* mask, bool half, void* stream) {
    if (!h) return einval("finish_facet_real: NULL plan");
    if (half && h->yN % 2) return einval("finish_facet_real_half: yN_size must be even");
    SW_TRY(check_lines(in, out, half ? h->yN / 2 + 1 : h->yN, -1, "finish_facet_real"));
    if (in->location != SWIFTLY_B200_DEVICE || out->location != SWIFTLY_B200_DEVICE)
        return einval("finish_facet_real: device arrays only");
    const int64_t yN = h->yN, fs = out->size;
    if (fs > yN - 1) return einval("finish_facet_real: facet size must be at most yN_size - 1");
    if (in->n_lines == 0) return SWIFTLY_B200_OK;
    cudaStream_t s = (cudaStream_t)stream;
    SW_DEVICE_GUARD(h);
    FinishFacetRealOp op;
    op.g.in = (const cplx*)in->data;
    op.g.out = nullptr;
    op.g.in_ls = in->line_stride;
    op.g.in_es = in->elem_stride;
    // (strides in doubles: only their adjacency enters the choice of the kernel form)
    op.g.out_ls = out->line_stride;
    op.g.out_es = out->elem_stride;
    op.g.n_lines = in->n_lines;
    op.fb = h->d_Fb + ((yN - 1) / 2 - fs / 2);
    op.n = (int)yN;
    op.fs = (int)fs;
    op.start = (int)pmod(yN / 2 - fs / 2 + facet_off, yN);
    op.mask = nullptr;
    op.rout = (double*)out->data;
    op.rout_ls = out->line_stride;
    op.rout_es = out->elem_stride;
    op.rmask = mask;
    if (half) {
        FinishFacetRealHalfOp hop;
        static_cast<FinishFacetRealOp&>(hop) = op;
        SW_TRY(run_finish_facet(h, hop, lines_adjacent(op.g), s));
    } else {
        SW_TRY(run_finish_facet(h, op, lines_adjacent(op.g), s));
    }
    return SWIFTLY_B200_OK;
}

extern "C" int swiftly_b200_finish_facet_real(const swiftly_b200* h,
                                              const swiftly_b200_lines* in,
                                              const swiftly_b200_lines* out, int64_t facet_off,
                                              const double* mask, void* stream) {
    return finish_facet_real_impl(h, in, out, facet_off, mask, false, stream);
}

extern "C" int swiftly_b200_finish_facet_real_half(const swiftly_b200* h,
                                                   const swiftly_b200_lines* in,
                                                   const swiftly_b200_lines* out,
                                                   int64_t facet_off, const double* mask,
                                                   void* stream) {
    return finish_facet_real_impl(h, in, out, facet_off, mask, true, stream);
}
