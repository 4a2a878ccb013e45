// SwiFTly -- the two finished subgrids of a Hermitian pair from one unmasked source.
//
// The Fourier plane of a real image is Hermitian, G(-u, -v) = conj(G(u, v)).  A subgrid of size
// sz at offset `off` holds the samples at off - h + r, r < sz, h = sz // 2 (finish_subgrid,
// core.py:287-325); the subgrid of the same size at -off holds -off - h + r', the conjugates of
// the samples at off + h - r' = off - h + (2h - r').  So both come from ONE source subgrid of
// size S = 2h + 1 at `off` (its first sz x sz samples are the subgrid at `off` itself):
//
//   out[r, c]    = m0[r] * m1[c] * src[r, c]
//   mirror[r, c] = n0[r] * n1[c] * conj(src[2h - r, 2h - c])        r, c < sz
#include "capi_util.h"

using namespace swiftly;

namespace swiftly {

// One CTA per source row r (grid-stride over rows): the row is read once and written to row r
// of `out` and reversed to row 2h - r of `mirror`, where those rows exist.  A warp's reversed
// stores cover the same 128-byte lines as forward ones, in descending order.
struct MirrorSubgridKernel {
    static constexpr int THREADS = 256;
    const cplx* src;
    int64_t src_ls, src_es;
    cplx* out;
    int64_t out_ls, out_es;
    cplx* mir;
    int64_t mir_ls, mir_es;
    const double *m0, *m1, *n0, *n1;  // null: all ones
    int sz, h;
    template <class Ctx>
    SW_HD void operator()(Ctx& ctx) const {
        const int S = 2 * h + 1;
        for (int r = ctx.bid; r < S; r += ctx.nblocks) {
            const int rm = 2 * h - r;
            const bool row_out = r < sz, row_mir = rm < sz;
            const double w0 = row_out && m0 ? ldg_d(m0 + r) : 1.0;
            const double v0 = row_mir && n0 ? ldg_d(n0 + rm) : 1.0;
            const cplx* in = src + (int64_t)r * src_ls;
            for (int c = ctx.tid; c < S; c += THREADS) {
                const cplx v = ld_stream(in + (int64_t)c * src_es);
                if (row_out && c < sz) {
                    const double w = w0 * (m1 ? ldg_d(m1 + c) : 1.0);
                    st_stream(out + (int64_t)r * out_ls + (int64_t)c * out_es, cscale(v, w));
                }
                const int cm = 2 * h - c;
                if (row_mir && cm < sz) {
                    const double w = v0 * (n1 ? ldg_d(n1 + cm) : 1.0);
                    st_stream(mir + (int64_t)rm * mir_ls + (int64_t)cm * mir_es,
                              cscale(cconj(v), w));
                }
            }
        }
    }
};

}  // namespace swiftly

extern "C" int swiftly_b200_mirror_subgrid(const swiftly_b200* h, const swiftly_b200_lines* src,
                                           const swiftly_b200_lines* out,
                                           const swiftly_b200_lines* mirror, const double* mask0,
                                           const double* mask1, const double* mirror_mask0,
                                           const double* mirror_mask1, void* stream) {
    if (!h || !src || !out || !mirror) return einval("mirror_subgrid: NULL argument");
    if (src->location != SWIFTLY_B200_DEVICE || out->location != SWIFTLY_B200_DEVICE ||
        mirror->location != SWIFTLY_B200_DEVICE)
        return einval("mirror_subgrid: device arrays only");
    const int64_t sz = out->size;
    if (out->n_lines != sz || mirror->n_lines != sz || mirror->size != sz)
        return einval("mirror_subgrid: out and mirror must both be " + std::to_string(sz) + " x " +
                      std::to_string(sz) + ", got " + std::to_string(out->n_lines) + " x " +
                      std::to_string(sz) + " and " + std::to_string(mirror->n_lines) + " x " +
                      std::to_string(mirror->size));
    if (sz < 0) return einval("mirror_subgrid: negative shape");
    const int64_t S = 2 * (sz / 2) + 1;
    if (src->n_lines < S || src->size < S)
        return einval("mirror_subgrid: source is " + std::to_string(src->n_lines) + " x " +
                      std::to_string(src->size) + ", need at least " + std::to_string(S) +
                      " x " + std::to_string(S));
    if (sz == 0) return SWIFTLY_B200_OK;
    if (!src->data || !out->data || !mirror->data)
        return einval("mirror_subgrid: NULL data pointer");
    SW_DEVICE_GUARD(h);
    MirrorSubgridKernel k;
    k.src = (const cplx*)src->data;
    k.src_ls = src->line_stride;
    k.src_es = src->elem_stride;
    k.out = (cplx*)out->data;
    k.out_ls = out->line_stride;
    k.out_es = out->elem_stride;
    k.mir = (cplx*)mirror->data;
    k.mir_ls = mirror->line_stride;
    k.mir_es = mirror->elem_stride;
    k.m0 = mask0;
    k.m1 = mask1;
    k.n0 = mirror_mask0;
    k.n1 = mirror_mask1;
    k.sz = (int)sz;
    k.h = (int)(sz / 2);
    int grid = (int)S;
    if (h->max_blocks > 0 && grid > h->max_blocks) grid = h->max_blocks;  // (test hook)
    note_launch(h, LAUNCH_MIRROR, 0, 0, grid);
    SW_CUDA(launch_body(k, grid, 0, (cudaStream_t)stream), "mirror_subgrid launch");
    return SWIFTLY_B200_OK;
}
