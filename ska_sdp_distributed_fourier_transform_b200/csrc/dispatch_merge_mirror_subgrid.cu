// SwiFTly -- a Hermitian pair of subgrids merged into one, for the backward transform of a real
// image (the adjoint of mirror_subgrid).
//
// The backward transform L is linear with real, even windows, so for the subgrid B of size sz
// at -off, L(B) = conj(L(B')) with B' the subgrid of size S = 2h + 1 (h = sz // 2) at +off,
// B'[2h - r, 2h - c] = conj(B[r, c]).  For a pair A at off and B at -off the real parts add up:
//
//   Re L(A) + Re L(B) = Re L(C),   C = A + B'   (one subgrid of size S at off)
//
//   out[r, c] = [r, c < sz] sg[r, c] + [2h - r, 2h - c < sz] conj(mirror[2h - r, 2h - c])
#include "capi_util.h"

using namespace swiftly;

namespace swiftly {

// One CTA per output row r (grid-stride over rows): row r of `sg` is read forward and row 2h - r
// of `mirror` reversed, where those rows exist.  A warp's reversed loads cover the same 128-byte
// lines as forward ones, in descending order.
struct MergeMirrorSubgridKernel {
    static constexpr int THREADS = 256;
    const cplx* sg;
    int64_t sg_ls, sg_es;
    const cplx* mir;
    int64_t mir_ls, mir_es;
    cplx* out;
    int64_t out_ls, out_es;
    int sz, h;
    template <class Ctx>
    SW_HD void operator()(Ctx& ctx) const {
        const int S = 2 * h + 1;
        for (int r = ctx.bid; r < S; r += ctx.nblocks) {
            const int rm = 2 * h - r;
            const bool row_sg = r < sz, row_mir = rm < sz;
            const cplx* a = sg + (int64_t)r * sg_ls;
            const cplx* b = mir + (int64_t)rm * mir_ls;
            cplx* o = out + (int64_t)r * out_ls;
            for (int c = ctx.tid; c < S; c += THREADS) {
                const int cm = 2 * h - c;
                const bool has_a = row_sg && c < sz, has_b = row_mir && cm < sz;
                cplx v = mk(0.0, 0.0);
                if (has_a) v = ld_stream(a + (int64_t)c * sg_es);
                if (has_b) {
                    const cplx w = cconj(ld_stream(b + (int64_t)cm * mir_es));
                    v = has_a ? mk(v.x + w.x, v.y + w.y) : w;
                }
                st_stream(o + (int64_t)c * out_es, v);
            }
        }
    }
};

}  // namespace swiftly

extern "C" int swiftly_b200_merge_mirror_subgrid(const swiftly_b200* h,
                                                 const swiftly_b200_lines* sg,
                                                 const swiftly_b200_lines* mirror,
                                                 const swiftly_b200_lines* out, void* stream) {
    if (!h || !sg || !mirror || !out) return einval("merge_mirror_subgrid: NULL argument");
    if (sg->location != SWIFTLY_B200_DEVICE || mirror->location != SWIFTLY_B200_DEVICE ||
        out->location != SWIFTLY_B200_DEVICE)
        return einval("merge_mirror_subgrid: device arrays only");
    const int64_t sz = sg->size;
    if (sz < 0) return einval("merge_mirror_subgrid: negative shape");
    if (sg->n_lines != sz || mirror->n_lines != sz || mirror->size != sz)
        return einval("merge_mirror_subgrid: sg and mirror must both be square of one size, got " +
                      std::to_string(sg->n_lines) + " x " + std::to_string(sz) + " and " +
                      std::to_string(mirror->n_lines) + " x " + std::to_string(mirror->size));
    const int64_t S = 2 * (sz / 2) + 1;
    if (out->n_lines != S || out->size != S)
        return einval("merge_mirror_subgrid: out is " + std::to_string(out->n_lines) + " x " +
                      std::to_string(out->size) + ", expected " + std::to_string(S) + " x " +
                      std::to_string(S));
    if (!sg->data || !mirror->data || !out->data)
        return einval("merge_mirror_subgrid: NULL data pointer");
    SW_DEVICE_GUARD(h);
    MergeMirrorSubgridKernel k;
    k.sg = (const cplx*)sg->data;
    k.sg_ls = sg->line_stride;
    k.sg_es = sg->elem_stride;
    k.mir = (const cplx*)mirror->data;
    k.mir_ls = mirror->line_stride;
    k.mir_es = mirror->elem_stride;
    k.out = (cplx*)out->data;
    k.out_ls = out->line_stride;
    k.out_es = out->elem_stride;
    k.sz = (int)sz;
    k.h = (int)(sz / 2);
    int grid = (int)S;
    if (h->max_blocks > 0 && grid > h->max_blocks) grid = h->max_blocks;  // (test hook)
    note_launch(h, LAUNCH_MERGE_MIRROR, 0, 0, grid);
    SW_CUDA(launch_body(k, grid, 0, (cudaStream_t)stream), "merge_mirror_subgrid launch");
    return SWIFTLY_B200_OK;
}
