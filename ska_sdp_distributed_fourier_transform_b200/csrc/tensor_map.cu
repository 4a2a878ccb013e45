// SwiFTly -- descriptors for the TMA engine (bulk tensor stores of finished lines).
//
// The fused subgrid kernels stage a finished line in shared memory and hand it to the TMA
// engine, which scatters it into the output array -- with ANY line / sample / group strides,
// in particular transposed ("sample stride = number of lines") -- without spending LSU
// wavefronts or SM issue slots on 16-byte scattered stores.  The descriptor is a rank-4 tiled
// tensor map over the output array seen as doubles: dimension 0 = (re, im), dimensions 1..3 =
// line / sample / group in ascending stride order.
#include <algorithm>

#include "capi_util.h"

namespace swiftly {

#if !defined(SWIFTLY_EMU)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_tiled() {
    static EncodeTiledFn fn = []() -> EncodeTiledFn {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) !=
                cudaSuccess || q != cudaDriverEntryPointSuccess)
            return nullptr;
        return (EncodeTiledFn)p;
    }();
    return fn;
}
#endif

// slot[0..2]: which tensor coordinate (1..3) carries the line / sample / group index
bool make_out_map(TensorMap4* tm, cplx* out, int64_t out_ls, int64_t out_es, int64_t out_gs,
                  int64_t n_lines, int64_t sz, int64_t n_groups, int box_rows, int* slot) {
    struct Dim {
        int which;
        int64_t size, stride;
    } d[3] = {{0, n_lines, out_ls}, {1, sz, out_es}, {2, n_groups, out_gs}};
    for (auto& x : d)
        if (x.size < 1 || (x.size > 1 && x.stride < 1)) return false;
    // ascending stride; dimensions of size one go last (their stride is immaterial)
    std::stable_sort(d, d + 3, [](const Dim& a, const Dim& b) {
        if ((a.size == 1) != (b.size == 1)) return b.size == 1;
        return a.stride < b.stride;
    });
    int64_t prev = 1;
    for (auto& x : d) {
        if (x.size == 1) x.stride = prev > x.stride ? prev : x.stride;
        if (x.stride < 1) x.stride = 1;
        prev = x.stride * x.size;
    }
    for (int i = 0; i < 3; ++i) slot[d[i].which] = i + 1;
    int box[4] = {2, 1, 1, 1};
    box[slot[1]] = box_rows;
    if (box_rows < 1 || box_rows > 256) return false;
#if defined(SWIFTLY_EMU)
    tm->base = (double*)out;
    tm->stride[0] = 1;
    tm->dim[0] = 2;
    for (int i = 0; i < 3; ++i) {
        tm->stride[i + 1] = 2 * d[i].stride;
        tm->dim[i + 1] = d[i].size;
    }
    for (int i = 0; i < 4; ++i) tm->box[i] = box[i];
    tm->swizzle128 = 0;
    return true;
#else
    EncodeTiledFn fn = encode_tiled();
    if (!fn) return false;
    if (((uintptr_t)out & 15) != 0) return false;
    cuuint64_t gdim[4] = {2, (cuuint64_t)d[0].size, (cuuint64_t)d[1].size, (cuuint64_t)d[2].size};
    cuuint64_t gstr[3] = {(cuuint64_t)d[0].stride * 16, (cuuint64_t)d[1].stride * 16,
                          (cuuint64_t)d[2].stride * 16};
    for (int i = 0; i < 3; ++i)
        if (gstr[i] >= ((cuuint64_t)1 << 40)) return false;
    cuuint32_t bdim[4] = {(cuuint32_t)box[0], (cuuint32_t)box[1], (cuuint32_t)box[2],
                          (cuuint32_t)box[3]};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = fn(&tm->map, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 4, (void*)out, gdim, gstr, bdim,
                    estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                    CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
#endif
}

// Map for staging the ROWS of a 2-D complex128 array (row stride `ls` samples, `fs` samples per
// row, fs a multiple of 8) in shared memory with the 128-byte swizzle: the row is seen as
// fs / 8 chunks of 128 bytes; dimension 0 = the 16 doubles of a chunk, 1 = chunk, 2 = row.
// One box = `box_chunks` chunks of one row.
bool make_row_map(TensorMap4* tm, const cplx* base, int64_t ls, int64_t n_rows, int64_t fs,
                  int box_chunks) {
    if (fs < 8 || (fs & 7) || box_chunks < 8 || box_chunks > 256 || (box_chunks & 7)) return false;
    if (n_rows < 1 || ls < fs) return false;
#if defined(SWIFTLY_EMU)
    tm->base = (double*)base;
    tm->stride[0] = 1;
    tm->stride[1] = 16;
    tm->stride[2] = 2 * ls;
    tm->stride[3] = 2 * ls * n_rows;
    tm->dim[0] = 16;
    tm->dim[1] = fs / 8;
    tm->dim[2] = n_rows;
    tm->dim[3] = 1;
    tm->box[0] = 16;
    tm->box[1] = box_chunks;
    tm->box[2] = 1;
    tm->box[3] = 1;
    tm->swizzle128 = 1;
    return true;
#else
    EncodeTiledFn fn = encode_tiled();
    if (!fn) return false;
    if (((uintptr_t)base & 15) != 0) return false;
    cuuint64_t gdim[4] = {16, (cuuint64_t)(fs / 8), (cuuint64_t)n_rows, 1};
    cuuint64_t gstr[3] = {128, (cuuint64_t)ls * 16, (cuuint64_t)ls * 16 * (cuuint64_t)n_rows};
    for (int i = 0; i < 3; ++i)
        if (gstr[i] >= ((cuuint64_t)1 << 40)) return false;
    cuuint32_t bdim[4] = {16, (cuuint32_t)box_chunks, 1, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = fn(&tm->map, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 4, (void*)base, gdim, gstr, bdim,
                    estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                    CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
#endif
}

#if defined(SWIFTLY_EMU)
// the bytes a tensor load reports to its mbarrier: the whole box, the zero fill outside the tensor
// included
uint32_t emu_tensor_box_bytes(const TensorMap4* tm) {
    return (uint32_t)(tm->box[0] * tm->box[1] * tm->box[2] * tm->box[3]) * (uint32_t)sizeof(double);
}

// what the TMA engine does with a (128-byte swizzled) tensor load of box (0, c1, c2, 0)
void emu_tensor_load(const TensorMap4* tm, double* dst, int c1, int c2) {
    for (int i1 = 0; i1 < tm->box[1]; ++i1)
        for (int u = 0; u < 8; ++u) {  // 16-byte units of the 128-byte row
            const int64_t x1 = c1 + i1;
            const int pu = tm->swizzle128 ? (u ^ (i1 & 7)) : u;
            for (int w = 0; w < 2; ++w) {
                double v = 0.0;
                if (x1 < tm->dim[1] && c2 < tm->dim[2])
                    v = tm->base[(2 * u + w) * tm->stride[0] + x1 * tm->stride[1] +
                                 (int64_t)c2 * tm->stride[2]];
                dst[(size_t)i1 * 16 + 2 * pu + w] = v;
            }
        }
}

// what the TMA engine does with a tensor store: copy the dense box, clipped to the tensor
void emu_tensor_store(const TensorMap4* tm, const double* src, int c1, int c2, int c3) {
    const int c[4] = {0, c1, c2, c3};
    for (int i3 = 0; i3 < tm->box[3]; ++i3)
        for (int i2 = 0; i2 < tm->box[2]; ++i2)
            for (int i1 = 0; i1 < tm->box[1]; ++i1)
                for (int i0 = 0; i0 < tm->box[0]; ++i0) {
                    const int64_t x[4] = {c[0] + i0, c[1] + i1, c[2] + i2, c[3] + i3};
                    bool inside = true;
                    for (int k = 0; k < 4; ++k)
                        if (x[k] < 0 || x[k] >= tm->dim[k]) inside = false;
                    const double v = *src++;
                    if (!inside) continue;
                    tm->base[x[0] * tm->stride[0] + x[1] * tm->stride[1] + x[2] * tm->stride[2] +
                             x[3] * tm->stride[3]] = v;
                }
}
#endif

}  // namespace swiftly
