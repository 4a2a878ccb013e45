/*
 * swiftly_b200.h -- C ABI of the B200-native SwiFTly facet<->subgrid hot path.
 *
 * This is the drop-in boundary: the entry points below are what the reference's
 * native-backend adapter binds.  In the reference
 * (ska-sdp-distributed-fourier-transform, src/ska_sdp_exec_swiftly/
 * fourier_transform/core.py) the adapter class `SwiftlyCoreFunc` (core.py:487-929)
 * forwards each of the eight SwiFTly primitives to a method of the native object
 * `ska_sdp_func.fourier_transforms.swiftly.Swiftly(N, yN_size, xM_size, W)`
 * (core.py:508-510).  Those native methods always transform along the LAST axis
 * of a 2-D array and receive axis-0 work as strided transposed views
 * (core.py:577-630).  The functions here take the same information in plain C:
 * a batch of 1-D "lines" described by a base pointer, a line count, a line
 * length, and line/element strides -- so a C-ordered 2-D array along axis 1, the
 * same array along axis 0 (transposed view) and 1-D arrays are all one call.
 *
 * All samples are complex128 (interleaved re, im doubles).  Offsets are in image
 * / grid pixels exactly as in the reference (any integer, taken modulo).
 * Functions return 0 on success, a negative SWIFTLY_B200_E* code otherwise;
 * swiftly_b200_last_error() gives the message of the calling thread's last
 * failure.  A handle is immutable after creation: concurrent calls on
 * different streams are safe.  There is NO CPU implementation behind this ABI:
 * if no CUDA device is usable every call fails.
 */
#ifndef SWIFTLY_B200_H
#define SWIFTLY_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SWIFTLY_B200_OK 0
#define SWIFTLY_B200_EINVAL (-1)      /* bad argument / shape (Python: ValueError)     */
#define SWIFTLY_B200_ECUDA (-2)       /* CUDA runtime failure (Python: RuntimeError)   */
#define SWIFTLY_B200_EUNSUPPORTED (-3) /* FFT size not supported by this build          */

#define SWIFTLY_B200_DEVICE 0 /* `data` is a device pointer (cudaMalloc / torch)  */
#define SWIFTLY_B200_HOST 1   /* `data` is a host pointer; the library stages it  */

typedef struct swiftly_b200 swiftly_b200; /* opaque plan: tables live on one device */

/* A batch of 1-D lines of complex128 samples.
 * sample (line l, index i) lives at data[(l * line_stride + i * elem_stride)] (complex elements). */
typedef struct swiftly_b200_lines {
    void* data;
    int64_t n_lines;
    int64_t size;
    int64_t line_stride;
    int64_t elem_stride;
    int32_t location; /* SWIFTLY_B200_DEVICE or SWIFTLY_B200_HOST */
} swiftly_b200_lines;

/* Plan creation.  Replaces `Swiftly(N, yN_size, xM_size, W)` (core.py:508-510) and
 * `SwiftlyCore.__init__` / `check_params` (core.py:39-74).  Fb (yN_size-1 doubles,
 * core.py:104-108) and Fn (xM_size*yN_size/N doubles, core.py:110-117) are the
 * PSWF-derived window tables computed by the caller with the reference's scipy
 * formula (core.py:119-150); they are copied to the device.
 * Parameter violations (N % yN, N % xM, xM*yN % N) return SWIFTLY_B200_EINVAL. */
int swiftly_b200_create(double W, int64_t N, int64_t xM_size, int64_t yN_size,
                        const double* Fb, const double* Fn, int device, swiftly_b200** plan);
void swiftly_b200_destroy(swiftly_b200* plan);
const char* swiftly_b200_last_error(void);
/* Free the plan's per-stream scratch buffers (up to 2 GiB after prepare_facet along the strided
 * axis at N = 65536); they are re-created on demand.  Synchronises the owning streams. */
void swiftly_b200_release_scratch(swiftly_b200* plan);
/* Library identification: "swiftly_b200 <version> cuda sm_90a" (or "... EMULATED" for
 * the test-only host build, which the product never loads). */
const char* swiftly_b200_build_info(void);

int64_t swiftly_b200_contribution_size(const swiftly_b200* plan); /* xM_yN_size, core.py:48 */

/* ---- facet -> subgrid ------------------------------------------------------------ */
/* SwiftlyCore.prepare_facet (core.py:189-222) / Swiftly.prepare_facet (core.py:684-692).
 * in: n_lines x facet_size, out: n_lines x yN_size (overwritten). */
int swiftly_b200_prepare_facet(const swiftly_b200* plan, const swiftly_b200_lines* in,
                               const swiftly_b200_lines* out, int64_t facet_off, void* stream);
/* SwiftlyCore.extract_from_facet (core.py:224-253) / Swiftly.extract_from_facet (:713-721).
 * in: n_lines x yN_size, out: n_lines x xM_yN_size (overwritten). */
int swiftly_b200_extract_from_facet(const swiftly_b200* plan, const swiftly_b200_lines* in,
                                    const swiftly_b200_lines* out, int64_t subgrid_off,
                                    void* stream);
/* SwiftlyCore.add_to_subgrid (core.py:255-285) / Swiftly.add_to_subgrid (:742-750).
 * in: n_lines x xM_yN_size, out: n_lines x xM_size, ACCUMULATED into (out +=). */
int swiftly_b200_add_to_subgrid(const swiftly_b200* plan, const swiftly_b200_lines* in,
                                const swiftly_b200_lines* out, int64_t facet_off, void* stream);
/* One axis of SwiftlyCore.finish_subgrid (core.py:287-325) / Swiftly.finish_subgrid
 * (core.py:795-812, called once per axis).  in: n_lines x xM_size, out: n_lines x
 * subgrid_size (overwritten).  mask: optional subgrid_size doubles on the same
 * location as `out` data (0/1 mask of api_helper.py:107-111 folded into the store) or NULL. */
int swiftly_b200_finish_subgrid(const swiftly_b200* plan, const swiftly_b200_lines* in,
                                const swiftly_b200_lines* out, int64_t subgrid_off,
                                const double* mask, void* stream);

/* ---- subgrid -> facet ------------------------------------------------------------ */
/* One axis of SwiftlyCore.prepare_subgrid (core.py:328-368) / Swiftly.prepare_subgrid_inplace
 * (core.py:837-853).  in: n_lines x subgrid_size, out: n_lines x xM_size (overwritten). */
int swiftly_b200_prepare_subgrid(const swiftly_b200* plan, const swiftly_b200_lines* in,
                                 const swiftly_b200_lines* out, int64_t subgrid_off, void* stream);
/* SwiftlyCore.extract_from_subgrid (core.py:370-406) / Swiftly.extract_from_subgrid (:866-876).
 * in: n_lines x xM_size, out: n_lines x xM_yN_size (overwritten). */
int swiftly_b200_extract_from_subgrid(const swiftly_b200* plan, const swiftly_b200_lines* in,
                                      const swiftly_b200_lines* out, int64_t facet_off,
                                      void* stream);
/* SwiftlyCore.add_to_facet (core.py:408-449) / Swiftly.add_to_facet (:890-900).
 * in: n_lines x xM_yN_size, out: n_lines x yN_size, ACCUMULATED into (out +=). */
int swiftly_b200_add_to_facet(const swiftly_b200* plan, const swiftly_b200_lines* in,
                              const swiftly_b200_lines* out, int64_t subgrid_off, void* stream);
/* SwiftlyCore.finish_facet (core.py:452-484) / Swiftly.finish_facet (:916-926).
 * in: n_lines x yN_size, out: n_lines x facet_size (overwritten).  mask as in finish_subgrid
 * (api_helper.py:175-176, 195-196) or NULL. */
int swiftly_b200_finish_facet(const swiftly_b200* plan, const swiftly_b200_lines* in,
                              const swiftly_b200_lines* out, int64_t facet_off,
                              const double* mask, void* stream);
/* finish_facet of a real image: the real part only, as float64 samples,
 *   out[k] = (Re(fft_c(in))[(yN/2 - fs//2 + k + facet_off) mod yN] * Fb[k]) * mask[k],
 * in that product order, i.e. bitwise Re(swiftly_b200_finish_facet(mask = NULL)) * mask.
 * in: n_lines x yN_size complex128; out: n_lines x facet_size DOUBLES (overwritten) whose
 * line_stride and elem_stride count doubles, not complex elements.  mask: facet_size device
 * doubles or NULL.  Device arrays only (SWIFTLY_B200_EINVAL otherwise). */
int swiftly_b200_finish_facet_real(const swiftly_b200* plan, const swiftly_b200_lines* in,
                                   const swiftly_b200_lines* out, int64_t facet_off,
                                   const double* mask, void* stream);
/* swiftly_b200_finish_facet_real of a line kept as half rows (see "Half rows" below): in has
 * yN_size/2 + 1 samples per line, stored sample q being natural FFT index q.  The transform input
 * is the Hermitian part of the full line, 0.5 in[q] (0 < q < yN/2), 0.5 conj(in[yN - q])
 * (q > yN/2), (Re in[q], 0) (q = 0, yN/2): bitwise swiftly_b200_finish_facet_real of the full
 * line built that way.  Same contract otherwise; SWIFTLY_B200_EINVAL for an odd yN_size. */
int swiftly_b200_finish_facet_real_half(const swiftly_b200* plan, const swiftly_b200_lines* in,
                                        const swiftly_b200_lines* out, int64_t facet_off,
                                        const double* mask, void* stream);

/* ---- fused forward path (device memory only) ---------------------------------------- */
/* The reference's `extract_column` task (api_helper.py:200-210) in one kernel:
 * extract_from_facet(BF_F, subgrid_off0, axis=0) followed by prepare_facet(., facet_off1,
 * axis=1).  bf_f: yN_size lines (rows of the axis-0 prepared facet) of facet_size samples;
 * out: xM_yN_size lines of yN_size samples (overwritten). */
int swiftly_b200_extract_column(const swiftly_b200* plan, const swiftly_b200_lines* bf_f,
                                const swiftly_b200_lines* out, int64_t subgrid_off0,
                                int64_t facet_off1, void* stream);

/* One input of swiftly_b200_sum_finish_axis: `n_lines` lines (n_lines of the output) of
 * `size` samples.  size == yN_size: lines of a prepared facet, the contribution window for
 * `subgrid_off` is extracted on the fly (extract_from_facet, core.py:224-253);
 * size == xM_yN_size: lines that already are contributions. */
typedef struct swiftly_b200_source {
    const void* data; /* device pointer */
    int64_t line_stride;
    int64_t elem_stride;
    int64_t size;
    int64_t facet_off; /* facet offset along the transformed axis */
} swiftly_b200_source;

/* One axis of the reference's `sum_and_finish_subgrid` task (api_helper.py:73-112) in one
 * kernel: for every line, sum_g add_to_subgrid(extract(source_g), facet_off_g) is built in
 * shared memory and finished (finish_subgrid along this axis, mask folded in).  out:
 * n_lines x subgrid_size (overwritten).  Returns SWIFTLY_B200_EUNSUPPORTED when the
 * (xM_yN_size, xM_size) pair has no fused instantiation (callers then use the primitives). */
int swiftly_b200_sum_finish_axis(const swiftly_b200* plan, const swiftly_b200_source* sources,
                                 int n_sources, const swiftly_b200_lines* out,
                                 int64_t subgrid_off, const double* mask, void* stream);
/* The same for several independent source groups in ONE launch (e.g. all facet rows of a
 * subgrid): group g takes sources [sum(group_sizes[:g]), ... + group_sizes[g]) and writes
 * out->data + g * out_group_stride (complex elements); `out` describes one group's lines. */
int swiftly_b200_sum_finish_axis_grouped(const swiftly_b200* plan,
                                         const swiftly_b200_source* sources,
                                         const int32_t* group_sizes, int n_groups,
                                         const swiftly_b200_lines* out, int64_t out_group_stride,
                                         int64_t subgrid_off, const double* mask, void* stream);
/* As above, but the groups may belong to different subgrids (a batch of the multi-GPU
 * driver): subgrid_offs[g] and masks[g] (masks or masks[g] may be NULL) per group
 * (any number of groups: larger jobs are cut into several launches). */
int swiftly_b200_sum_finish_axis_batched(const swiftly_b200* plan,
                                         const swiftly_b200_source* sources,
                                         const int32_t* group_sizes, int n_groups,
                                         const swiftly_b200_lines* out, int64_t out_group_stride,
                                         const int64_t* subgrid_offs, const double* const* masks,
                                         void* stream);
/* As swiftly_b200_sum_finish_axis_batched, but every group writes to its OWN buffer:
 * out_ptrs[g] is the base address of group g's output, `out` gives the (common) shape and
 * strides.  The sharded driver passes the owners' peer-mapped receive buffers, so the strips
 * of a subgrid travel over NVLink as the kernel's epilogue (TMA bulk tensor stores) instead
 * of through a separate collective (replaces the Dask transfer of contributions,
 * reference api.py:263-277). */
int swiftly_b200_sum_finish_axis_scattered(const swiftly_b200* plan,
                                           const swiftly_b200_source* sources,
                                           const int32_t* group_sizes, int n_groups,
                                           const swiftly_b200_lines* out, void* const* out_ptrs,
                                           const int64_t* subgrid_offs,
                                           const double* const* masks, void* stream);
/* Ordering between the ranks of the sharded transform (peer_sync.cu): `flags_dev_table` is a
 * DEVICE array of n_peers device pointers -- this rank's mappings of every rank's flag array
 * (n_peers int64 each, peer-mapped / symmetric memory).  signal stores `value` into entry
 * my_rank of every rank's array (system-scope release, after everything queued before on the
 * stream); wait spins (system-scope acquire) until all n_peers entries of `my_flags` are
 * >= value, or sets *status (device int) to 1 + peer after timeout_s. */
int swiftly_b200_peer_signal(const swiftly_b200* plan, void* const* flags_dev_table, int n_peers,
                             int my_rank, int64_t value, void* stream);
int swiftly_b200_peer_wait(const swiftly_b200* plan, const void* my_flags, int n_peers,
                           int64_t value, double timeout_s, void* status, void* stream);
/* Row rings.  A subgrid column reads (extract_columns) or adds into (fold_column) only an
 * xM_yN_size-row window of each yN_size-row facet array: rows (yN/2 - m/2 + s) mod yN + u,
 * u < m, with m = xM_yN_size and s = subgrid_off0 * yN_size // N.  Instead of the whole array
 * a caller may pass a RING of m rows: facet row r lives at ring line r mod m (m divides yN, so
 * the mapping holds across the wrap at yN).  The ring must hold the window's rows of the
 * column at hand; rows that stay when the window slides keep their line.  In one call every
 * bf_f[f] (every facet_accs[f]) has yN_size lines, or every one has xM_yN_size lines; any other
 * line count is rejected.  A ring runs the same kernel form as the whole array with the same
 * facet size and row stride. */
/* Half rows.  For a real image every column of BF_F (and the part of a facet accumulator that
 * finish_facet_real reads) is conjugate-symmetric in the centred row index: rows yN/2 + d and
 * yN/2 - d are conjugates.  A caller may then pass yN_size/2 + 1 rows (yN_size even): stored row
 * d, 0 <= d <= yN/2, holds centred row (yN/2 + d) mod yN.  Centred row r is stored row
 * i = (r - yN/2) mod yN when that is <= yN/2, else yN - i, conjugated.  extract_columns[_windowed]
 * reads a conjugated row with every imaginary part negated (bitwise the call on the full
 * Hermitian rows); fold_column adds conj(w v) into a conjugated row, w v elsewhere, in at most two
 * passes in stream order: a window across centred offset 0 or yN/2 holds rows r and -r, and the
 * unconjugated one is added first.  One call takes half rows for every facet or for none. */
/* swiftly_b200_extract_column for n_facets (<= 64) facets in ONE launch: bf_f[f] / out[f]
 * as in swiftly_b200_extract_column (contiguous rows, or row rings), facet_off1[f] per facet. */
int swiftly_b200_extract_columns(const swiftly_b200* plan, int n_facets,
                                 const swiftly_b200_lines* bf_f, const swiftly_b200_lines* out,
                                 int64_t subgrid_off0, const int64_t* facet_off1, void* stream);
/* The pair the fused forward driver uses between stage 1 and K2: prepare_facet whose output
 * LINES are pre-multiplied by the Fb window of the other axis (line l by Fb_c[l], the factor
 * prepare_facet(axis 1) would apply to sample l), and extract_columns that takes such rows and
 * skips its own window multiply.  Together they equal prepare_facet + extract_columns
 * (core.py:189-222 applied along axis 0, then api_helper.py:200-210). */
int swiftly_b200_prepare_facet_windowed(const swiftly_b200* plan, const swiftly_b200_lines* in,
                                        const swiftly_b200_lines* out, int64_t facet_off,
                                        void* stream);
int swiftly_b200_extract_columns_windowed(const swiftly_b200* plan, int n_facets,
                                          const swiftly_b200_lines* bf_f,
                                          const swiftly_b200_lines* out, int64_t subgrid_off0,
                                          const int64_t* facet_off1, void* stream);
/* swiftly_b200_prepare_facet_windowed of a REAL facet, keeping only its half rows (see "Half
 * rows" below): in: n_lines x facet_size DOUBLES (line_stride and elem_stride count doubles);
 * out: n_lines x (yN_size/2 + 1) complex128, line l sample d = the windowed prepared facet's
 * line l at centred index (yN/2 + d) mod yN.  Bitwise equal to those samples of
 * swiftly_b200_prepare_facet_windowed applied to the facet promoted to complex.  Device arrays
 * only; SWIFTLY_B200_EINVAL for an odd yN_size. */
int swiftly_b200_prepare_facet_real_half(const swiftly_b200* plan, const swiftly_b200_lines* in,
                                         const swiftly_b200_lines* out, int64_t facet_off,
                                         void* stream);
/* The two finished subgrids of a Hermitian pair (real image: G(-u, -v) = conj(G(u, v))) from
 * ONE unmasked source, finish_subgrid (core.py:287-325) with api_helper.py:107-111's masks:
 *   out[r, c]    = mask0[r] * mask1[c] * src[r, c]
 *   mirror[r, c] = mirror_mask0[r] * mirror_mask1[c] * conj(src[2h - r, 2h - c])
 * for r, c < sz, h = sz // 2.  src: the subgrid at (off0, off1) of size 2h + 1 (or larger:
 * only the first 2h + 1 lines and samples are read), lines = rows; out: the subgrid of size sz
 * at (off0, off1); mirror: the subgrid of size sz at (-off0, -off1).  out and mirror are sz x sz
 * (overwritten), any line and element strides; every mask may be NULL (all ones), else sz
 * device doubles.  Device arrays only.  SWIFTLY_B200_EINVAL when src is smaller than 2h + 1 in
 * either dimension, out and mirror are not both sz x sz, or an array is on the host. */
int swiftly_b200_mirror_subgrid(const swiftly_b200* plan, const swiftly_b200_lines* src,
                                const swiftly_b200_lines* out, const swiftly_b200_lines* mirror,
                                const double* mask0, const double* mask1,
                                const double* mirror_mask0, const double* mirror_mask1,
                                void* stream);
/* The adjoint of swiftly_b200_mirror_subgrid (unmasked), for the backward transform of a real
 * image: the subgrids sg at (off0, off1) and mirror at (-off0, -off1), both sz x sz, merged into
 * ONE subgrid of size S = 2h + 1, h = sz // 2, at (off0, off1) whose backward transform has the
 * same real part as the sum of theirs:
 *   out[r, c] = [r, c < sz] sg[r, c] + [2h - r, 2h - c < sz] conj(mirror[2h - r, 2h - c])
 * for r, c < S.  Where both terms exist: one complex add; where one exists: that term
 * unchanged; where neither does (even sz: the last row and column): 0.  out: S x S
 * (overwritten).  Any line and element strides; device arrays only.  Reads and writes
 * 16 * (2 sz^2 + S^2) bytes.  SWIFTLY_B200_EINVAL when sg and mirror are not both sz x sz, out
 * is not S x S, or an array is on the host. */
int swiftly_b200_merge_mirror_subgrid(const swiftly_b200* plan, const swiftly_b200_lines* sg,
                                      const swiftly_b200_lines* mirror,
                                      const swiftly_b200_lines* out, void* stream);
/* ---- fused backward path (device memory only) --------------------------------------- */
/* One subgrid into the column accumulators of n_facets (<= 64) facets in ONE launch: per
 * facet `extract_from_subgrid(block, facet_off1, axis=1)` followed by `accumulate_column` =
 * `add_to_facet(., subgrid_off1, axis=1, out=acc)` (api_helper.py:115-152).  blocks[f]: the
 * (xM_yN_size x xM_size) result of extract_from_subgrid(axis 0) for the facet's off0;
 * accs[f]: (xM_yN_size x yN_size) accumulator NAF_MNAF, ACCUMULATED into. */
int swiftly_b200_subgrid_to_facets(const swiftly_b200* plan, int n_facets,
                                   const swiftly_b200_lines* blocks,
                                   const swiftly_b200_lines* accs, const int64_t* facet_off1,
                                   int64_t subgrid_off1, void* stream);
/* Fold a finished subgrid column into n_facets facet accumulators in ONE launch: per facet
 * `finish_facet(acc, facet_off1, size, axis=1)`, optional mask1, `add_to_facet(., subgrid_off0,
 * axis=0, out=facet_acc)` (api_helper.py:155-179).  facet_accs[f]: (yN_size x facet_size)
 * accumulator MNAF_BMNAF (or its row ring, see "Row rings" above), ACCUMULATED into; mask1 or
 * mask1[f] may be NULL. */
int swiftly_b200_fold_column(const swiftly_b200* plan, int n_facets,
                             const swiftly_b200_lines* accs,
                             const swiftly_b200_lines* facet_accs, const int64_t* facet_off1,
                             const double* const* mask1, int64_t subgrid_off0, void* stream);

/* xM_size / xM_yN_size (1, 2, 3, 4 or 8: the sources one round of the fused kernel adds) if the
 * fused kernel exists for this plan, else 0.  It exists for every (xM_yN_size, xM_size) pair of
 * the parameter catalogue. */
int swiftly_b200_sum_finish_axis_supported(const swiftly_b200* plan);

/* One output of swiftly_b200_split_subgrid_axis: n_lines lines (the input's line count),
 * sample (l, i) at data[l * line_stride + i * elem_stride] (complex elements). */
typedef struct swiftly_b200_split_target {
    void* data; /* device pointer */
    int64_t n_lines;
    int64_t line_stride;
    int64_t elem_stride;
    int64_t facet_off; /* facet offset along the transformed axis */
} swiftly_b200_split_target;

#define SWIFTLY_B200_SPLIT_STORE 0 /* targets: xM_yN_size samples per line, overwritten    */
#define SWIFTLY_B200_SPLIT_ADD 1   /* targets: yN_size samples per line, ACCUMULATED into  */

/* The subgrid side of the backward transform along one axis in one kernel, the adjoint of
 * swiftly_b200_sum_finish_axis.  For every line of inputs[g] (n_lines lines of size <=
 * xM_size samples, the same n_lines in every group): prepare_subgrid along this axis with
 * subgrid_offs[g] (core.py:328-368), kept in shared memory, then for every target of the group
 * extract_from_subgrid(., facet_off) (core.py:370-406).
 *   SWIFTLY_B200_SPLIT_STORE: the xM_yN_size contribution samples are stored (a strip line).
 *   SWIFTLY_B200_SPLIT_ADD: they are added at the subgrid's position of a yN_size facet column
 *     accumulator line: add_to_facet(., subgrid_offs[g]) (core.py:408-449; together
 *     api_helper.py:115-152, extract_from_subgrid + accumulate_column).
 * Group g takes targets [sum(group_sizes[:g]), ... + group_sizes[g]).  Targets only read the
 * prepared line: their windows may overlap or repeat.  In add mode the targets of ONE group must
 * be distinct accumulators; targets of different groups may share one (groups are applied in
 * order, every line by one CTA: no atomics, deterministic sums).  Any number of groups and
 * targets (larger jobs are cut into several launches).  Offsets are taken modulo N.  Returns
 * SWIFTLY_B200_EUNSUPPORTED when swiftly_b200_split_axis_supported(plan) is 0. */
int swiftly_b200_split_subgrid_axis(const swiftly_b200* plan, const swiftly_b200_lines* inputs,
                                    int n_groups, const int64_t* subgrid_offs,
                                    const swiftly_b200_split_target* targets,
                                    const int32_t* group_sizes, int mode, void* stream);
/* xM_size / xM_yN_size (at least 1: the targets one round transforms) if the fused split kernel
 * exists for this plan, else 0; non-zero exactly for the pairs of
 * swiftly_b200_sum_finish_axis_supported. */
int swiftly_b200_split_axis_supported(const swiftly_b200* plan);

#ifdef __cplusplus
}
#endif
#endif /* SWIFTLY_B200_H */
