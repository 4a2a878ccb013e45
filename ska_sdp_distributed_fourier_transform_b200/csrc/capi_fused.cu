// SwiFTly -- C ABI of the fused forward-path entry points (device memory only).
#include <vector>

#include "capi_util.h"

using namespace swiftly;

// Fused extract_from_facet(axis 0) + prepare_facet(axis 1): the reference's
// `extract_column` task (api_helper.py:200-210).
extern "C" int swiftly_b200_extract_column(const swiftly_b200* h, const swiftly_b200_lines* bf_f,
                                           const swiftly_b200_lines* out, int64_t subgrid_off0,
                                           int64_t facet_off1, void* stream) {
    if (!h || !bf_f || !out) return einval("extract_column: NULL argument");
    if (bf_f->location != SWIFTLY_B200_DEVICE || out->location != SWIFTLY_B200_DEVICE)
        return einval("extract_column: device arrays only");
    const int64_t yN = h->yN, m = h->m, fs = bf_f->size;
    if (bf_f->n_lines != yN)
        return einval("extract_column: prepared facet must have yN_size lines, has " +
                      std::to_string(bf_f->n_lines));
    if (out->n_lines != m || out->size != yN)
        return einval("extract_column: output must be xM_yN_size lines of yN_size samples");
    if (fs > yN - 1) return einval("extract_column: facet size must be at most yN_size - 1");
    SW_DEVICE_GUARD(h);
    const int64_t sc = floordiv(subgrid_off0 * yN, h->N);
    PrepareFacetOp op;
    op.g.in = (const cplx*)bf_f->data;
    op.g.out = (cplx*)out->data;
    op.g.in_ls = bf_f->line_stride;
    op.g.in_es = bf_f->elem_stride;
    op.g.out_ls = out->line_stride;
    op.g.out_es = out->elem_stride;
    op.g.n_lines = m;
    op.n = (int)yN;
    op.fs = (int)fs;
    op.fb = h->d_Fb + ((yN - 1) / 2 - fs / 2);
    op.shift_in = (int)pmod(fs / 2 - facet_off1, yN);
    op.scale = 1.0 / (double)yN;
    op.rm_m = (int)m;
    op.rm_s_m = (int)pmod(sc, m);
    op.rm_base = (int)pmod(yN / 2 - m / 2 + sc, yN);
    op.rm_mod = (int)yN;
    op.lw = nullptr;
    return run_prepare_facet(h, op, false, (cudaStream_t)stream);
}

extern "C" int swiftly_b200_sum_finish_axis_supported(const swiftly_b200* h) {
    return h ? subgrid_axis_conc((int)h->m, (int)h->xM) : 0;
}

// Fused extract_from_facet + add_to_subgrid (summed over sources) + finish_subgrid along
// one axis (SubgridAxisKernel, kernels.cuh), for several independent source groups in one
// launch: group g = sources [first_g, first_g + group_sizes[g]) -> out + g * out_group_stride.
static int sum_finish_groups(const swiftly_b200* h, const swiftly_b200_source* sources,
                             const int32_t* group_sizes, int n_groups,
                             const swiftly_b200_lines* out, int64_t out_group_stride,
                             const int64_t* subgrid_offs, const double* const* masks,
                             void* stream, void* const* out_ptrs = nullptr) {
    if (!h || !sources || !out || !group_sizes) return einval("sum_finish_axis: NULL argument");
    if (out->location != SWIFTLY_B200_DEVICE) return einval("sum_finish_axis: device arrays only");
    const int64_t yN = h->yN, xM = h->xM, m = h->m;
    const int conc = subgrid_axis_conc((int)m, (int)xM);
    if (!conc) {
        set_error("sum_finish_axis: no fused kernel for m=" + std::to_string(m) +
                  ", xM=" + std::to_string(xM));
        return SWIFTLY_B200_EUNSUPPORTED;
    }
    if (n_groups < 1) return einval("sum_finish_axis: need at least one group");
    const int64_t sz = out->size;
    if (sz > xM) return einval("sum_finish_axis: subgrid size exceeds padded subgrid size");
    SW_DEVICE_GUARD(h);

    // per group: schedule sources into rounds of `conc` with pairwise disjoint windows
    std::vector<std::vector<std::vector<int>>> rounds((size_t)n_groups);
    std::vector<int> pos_of;
    int first = 0;
    for (int g = 0; g < n_groups; ++g) {
        if (group_sizes[g] < 0) return einval("sum_finish_axis: negative group size");
        for (int i = first; i < first + group_sizes[g]; ++i) {
            const swiftly_b200_source& sr = sources[i];
            if (!sr.data) return einval("sum_finish_axis: NULL source pointer");
            if (sr.size != yN && sr.size != m)
                return einval("sum_finish_axis: source line length must be yN_size or xM_yN_size");
            const int64_t sf = floordiv(sr.facet_off * xM, h->N);
            pos_of.push_back((int)pmod(xM / 2 - m / 2 + sf, xM));
            bool placed = false;
            for (auto& r : rounds[g]) {
                if ((int)r.size() >= conc) continue;
                bool clash = false;
                for (int j : r) {
                    int64_t d1 = pmod(pos_of[j] - pos_of[i], xM);
                    int64_t d2 = pmod(pos_of[i] - pos_of[j], xM);
                    if (d1 < m || d2 < m) {
                        clash = true;
                        break;
                    }
                }
                if (!clash) {
                    r.push_back(i);
                    placed = true;
                    break;
                }
            }
            if (!placed) rounds[g].push_back(std::vector<int>(1, i));
        }
        first += group_sizes[g];
    }

    // One launch carries at most SW_MAX_GROUPS groups and SW_MAX_SOURCES source slots (the
    // descriptors travel as kernel parameters).  Larger jobs -- any number of facets, like
    // the reference's sum_and_finish_subgrid (api_helper.py:73-112) -- are cut into pieces:
    // whole groups are packed greedily; a single group with more rounds than fit is cut along
    // its rounds, later pieces ADD their finished lines to the output (finishing is linear).
    const int max_rounds_per_launch = SW_MAX_SOURCES / conc;
    auto launch_piece = [&](int g0, int g1, size_t r0, size_t r1, bool accumulate) -> int {
        const int ng = g1 - g0;
        const int slots = (int)(r1 - r0) * conc;
        SubgridAxisArgs a;
        for (int i = 0; i < SW_MAX_SOURCES; ++i) {
            a.src[i].base = nullptr;
            a.src[i].ls = a.src[i].es = 0;
            a.src[i].wbase = a.src[i].s_m = a.src[i].sf_m = a.src[i].pos_base = 0;
            a.src[i].wmod = 1;
        }
        a.first_round_tiles = (r0 == 0 && !accumulate && (int64_t)conc * m == xM) ? 1 : 0;
        for (int g = g0; g < g1; ++g) {
            const int64_t sc = floordiv(subgrid_offs[g] * yN, h->N);
            const size_t rhi = r1 < rounds[g].size() ? r1 : rounds[g].size();
            for (size_t r = r0; r < rhi; ++r) {
                for (size_t c = 0; c < rounds[g][r].size(); ++c) {
                    const int i = rounds[g][r][c];
                    const swiftly_b200_source& sr = sources[i];
                    SgSource& d = a.src[(size_t)(g - g0) * slots + (r - r0) * conc + c];
                    d.base = (const cplx*)sr.data;
                    d.ls = sr.line_stride;
                    d.es = sr.elem_stride;
                    if (sr.size == yN && yN != m) {  // window of a prepared facet line
                        d.wbase = (int)pmod(yN / 2 - m / 2 + sc, yN);
                        d.s_m = (int)pmod(sc, m);
                        d.wmod = (int)yN;
                    } else {  // already a contribution
                        d.wbase = 0;
                        d.s_m = 0;
                        d.wmod = (int)m;
                    }
                    const int64_t sf = floordiv(sr.facet_off * xM, h->N);
                    d.sf_m = (int)pmod(sf, m);
                    d.pos_base = pos_of[i];
                }
            }
            // the first round may store instead of accumulate when its windows tile the
            // accumulator (conc disjoint windows of m samples with conc * m == xM)
            if (rounds[g].size() <= r0 || (int)rounds[g][r0].size() != conc)
                a.first_round_tiles = 0;
        }
        a.n_slots = slots;
        a.n_groups = ng;
        a.n_lines = out->n_lines;
        a.out = (cplx*)out->data + (int64_t)g0 * out_group_stride;
        a.out_ls = out->line_stride;
        a.out_es = out->elem_stride;
        a.out_gs = out_group_stride;
        a.sz = (int)sz;
        a.accumulate_out = accumulate ? 1 : 0;
        for (int g = 0; g < SW_MAX_GROUPS; ++g) {
            const int gg = g < ng ? g0 + g : g0;
            a.start[g] = (int)pmod(xM / 2 - sz / 2 + subgrid_offs[gg], xM);
            a.mask[g] = masks ? masks[gg] : nullptr;
            a.out_g[g] = (out_ptrs && g < ng) ? (cplx*)out_ptrs[gg] : nullptr;
        }
        if (out_ptrs) a.out = (cplx*)out_ptrs[g0];
        return run_subgrid_axis(h, a, (cudaStream_t)stream);
    };

    int g0 = 0;
    while (g0 < n_groups) {
        size_t nr = rounds[g0].empty() ? 1 : rounds[g0].size();
        if ((int)nr > max_rounds_per_launch) {
            // one group, several launches along its rounds
            for (size_t r0 = 0; r0 < nr; r0 += (size_t)max_rounds_per_launch) {
                size_t r1 = r0 + (size_t)max_rounds_per_launch;
                if (r1 > nr) r1 = nr;
                SW_TRY(launch_piece(g0, g0 + 1, r0, r1, r0 > 0));
            }
            ++g0;
            continue;
        }
        int g1 = g0 + 1;
        while (g1 < n_groups && g1 - g0 < SW_MAX_GROUPS) {
            size_t cand = rounds[g1].empty() ? 1 : rounds[g1].size();
            size_t mx = cand > nr ? cand : nr;
            if ((int)cand > max_rounds_per_launch ||
                (int64_t)mx * conc * (g1 - g0 + 1) > SW_MAX_SOURCES)
                break;
            nr = mx;
            ++g1;
        }
        SW_TRY(launch_piece(g0, g1, 0, nr, false));
        g0 = g1;
    }
    return SWIFTLY_B200_OK;
}

extern "C" int swiftly_b200_sum_finish_axis_grouped(const swiftly_b200* h,
                                                    const swiftly_b200_source* sources,
                                                    const int32_t* group_sizes, int n_groups,
                                                    const swiftly_b200_lines* out,
                                                    int64_t out_group_stride,
                                                    int64_t subgrid_off, const double* mask,
                                                    void* stream) {
    if (n_groups < 1) return einval("sum_finish_axis: need at least one group");
    std::vector<int64_t> offs((size_t)n_groups, subgrid_off);
    std::vector<const double*> masks((size_t)n_groups, mask);
    return sum_finish_groups(h, sources, group_sizes, n_groups, out, out_group_stride,
                             offs.data(), masks.data(), stream);
}

// Groups that belong to DIFFERENT subgrids (a batch of the multi-GPU driver): per-group
// subgrid offset and mask.
extern "C" int swiftly_b200_sum_finish_axis_batched(const swiftly_b200* h,
                                                    const swiftly_b200_source* sources,
                                                    const int32_t* group_sizes, int n_groups,
                                                    const swiftly_b200_lines* out,
                                                    int64_t out_group_stride,
                                                    const int64_t* subgrid_offs,
                                                    const double* const* masks, void* stream) {
    if (!subgrid_offs) return einval("sum_finish_axis: NULL subgrid offsets");
    return sum_finish_groups(h, sources, group_sizes, n_groups, out, out_group_stride,
                             subgrid_offs, masks, stream);
}

// Groups whose outputs live in DIFFERENT buffers (same shape and strides): out_ptrs[g] is the
// base of group g's output, `out` describes shape and strides.  The multi-GPU driver passes
// the peers' receive buffers here: the strips leave the kernel straight into the owner's
// memory over NVLink (bulk tensor stores of the TMA engine, or plain stores).
extern "C" int swiftly_b200_sum_finish_axis_scattered(const swiftly_b200* h,
                                                      const swiftly_b200_source* sources,
                                                      const int32_t* group_sizes, int n_groups,
                                                      const swiftly_b200_lines* out,
                                                      void* const* out_ptrs,
                                                      const int64_t* subgrid_offs,
                                                      const double* const* masks, void* stream) {
    if (!subgrid_offs || !out_ptrs) return einval("sum_finish_axis: NULL argument");
    for (int g = 0; g < n_groups; ++g)
        if (!out_ptrs[g]) return einval("sum_finish_axis: NULL output pointer");
    return sum_finish_groups(h, sources, group_sizes, n_groups, out, 0, subgrid_offs, masks,
                             stream, out_ptrs);
}

extern "C" int swiftly_b200_sum_finish_axis(const swiftly_b200* h,
                                            const swiftly_b200_source* sources, int n_sources,
                                            const swiftly_b200_lines* out, int64_t subgrid_off,
                                            const double* mask, void* stream) {
    if (n_sources < 0) return einval("sum_finish_axis: negative source count");
    int32_t one = n_sources;
    return swiftly_b200_sum_finish_axis_grouped(h, sources, &one, 1, out, 0, subgrid_off, mask,
                                                stream);
}

// extract_column for several facets in one launch (same subgrid_off0; per-facet off1).
static int extract_columns_impl(const swiftly_b200* h, int n_facets,
                                const swiftly_b200_lines* bf_f, const swiftly_b200_lines* out,
                                int64_t subgrid_off0, const int64_t* facet_off1, int prewindowed,
                                void* stream) {
    if (!h || !bf_f || !out || !facet_off1) return einval("extract_columns: NULL argument");
    if (n_facets < 1 || n_facets > SW_MAX_COLUMN_FACETS)
        return einval("extract_columns: between 1 and " + std::to_string(SW_MAX_COLUMN_FACETS) +
                      " facets per call");
    const int64_t yN = h->yN, m = h->m;
    // whole prepared facets (yN rows), row rings (m rows) or half rows of a real image (yN/2 + 1),
    // the same for every facet of a call
    const int64_t rows = bf_f[0].n_lines == m                          ? m
                         : yN % 2 == 0 && bf_f[0].n_lines == yN / 2 + 1 ? yN / 2 + 1
                                                                        : yN;
    const bool half = rows != m && rows == yN / 2 + 1;
    ExtractColumnsHalfOp op;
    for (int f = 0; f < n_facets; ++f) {
        const swiftly_b200_lines& i = bf_f[f];
        const swiftly_b200_lines& o = out[f];
        if (i.location != SWIFTLY_B200_DEVICE || o.location != SWIFTLY_B200_DEVICE)
            return einval("extract_columns: device arrays only");
        if (i.n_lines != rows || i.elem_stride != 1 || o.elem_stride != 1)
            return einval("extract_columns: prepared facets must be yN_size (or, all of them, "
                          "an xM_yN_size ring, or yN_size/2 + 1 half rows, yN_size even) "
                          "contiguous rows");
        if (o.n_lines != m || o.size != yN)
            return einval("extract_columns: output must be xM_yN_size lines of yN_size samples");
        if (i.size > yN - 1) return einval("extract_columns: facet size must be at most yN_size - 1");
        ColumnFacet& F = op.fac[f];
        F.in = (const cplx*)i.data;
        F.out = (cplx*)o.data;
        F.in_ls = i.line_stride;
        F.out_ls = o.line_stride;
        F.fs = (int)i.size;
        F.shift_in = (int)pmod(i.size / 2 - facet_off1[f], yN);
        F.fb_off = (int)((yN - 1) / 2 - i.size / 2);
        F.pad_ = 0;
    }
    SW_DEVICE_GUARD(h);
    const int64_t sc = floordiv(subgrid_off0 * yN, h->N);
    op.g.in = nullptr;
    op.g.out = nullptr;
    op.g.in_ls = op.g.in_es = op.g.out_ls = op.g.out_es = 0;
    op.g.n_lines = (int64_t)n_facets * m;
    op.fb = prewindowed ? nullptr : h->d_Fb;
    op.n = (int)yN;
    op.lines_per = (int)m;
    op.scale = 1.0 / (double)yN;
    op.rm_s_m = (int)pmod(sc, m);
    op.rm_base = (int)pmod(yN / 2 - m / 2 + sc, yN);
    op.rows = (int)rows;
    if (rows == m) {
        // row ring: window row r = (rm_base + ((l - s) mod m)) mod yN lives at line r mod m =
        // (l - (s - rm_base)) mod m (m divides yN), which the kernels' row map yields with
        // rm_base 0 and the shift s - rm_base -- the kernel code is the same for both forms
        op.rm_s_m = (int)pmod(op.rm_s_m - op.rm_base, m);
        op.rm_base = 0;
    }
    if (half) return run_extract_columns_half(h, op, false, (cudaStream_t)stream);
    return run_extract_columns(h, op, false, (cudaStream_t)stream);
}

extern "C" int swiftly_b200_extract_columns(const swiftly_b200* h, int n_facets,
                                            const swiftly_b200_lines* bf_f,
                                            const swiftly_b200_lines* out,
                                            int64_t subgrid_off0, const int64_t* facet_off1,
                                            void* stream) {
    return extract_columns_impl(h, n_facets, bf_f, out, subgrid_off0, facet_off1, 0, stream);
}

// the rows of bf_f come from swiftly_b200_prepare_facet_windowed: no Fb multiply here
extern "C" int swiftly_b200_extract_columns_windowed(const swiftly_b200* h, int n_facets,
                                                     const swiftly_b200_lines* bf_f,
                                                     const swiftly_b200_lines* out,
                                                     int64_t subgrid_off0,
                                                     const int64_t* facet_off1, void* stream) {
    return extract_columns_impl(h, n_facets, bf_f, out, subgrid_off0, facet_off1, 1, stream);
}

// ---------------------------------------------------------------------- fused backward path
// One subgrid -> column accumulators of all facets (SubgridToFacetsOp, kernels.cuh).
extern "C" int swiftly_b200_subgrid_to_facets(const swiftly_b200* h, int n_facets,
                                              const swiftly_b200_lines* blocks,
                                              const swiftly_b200_lines* accs,
                                              const int64_t* facet_off1, int64_t subgrid_off1,
                                              void* stream) {
    if (!h || !blocks || !accs || !facet_off1) return einval("subgrid_to_facets: NULL argument");
    if (n_facets < 1 || n_facets > SW_MAX_COLUMN_FACETS)
        return einval("subgrid_to_facets: between 1 and " +
                      std::to_string(SW_MAX_COLUMN_FACETS) + " facets per call");
    const int64_t yN = h->yN, xM = h->xM, m = h->m;
    SubgridToFacetsOp op;
    for (int f = 0; f < n_facets; ++f) {
        const swiftly_b200_lines& i = blocks[f];
        const swiftly_b200_lines& o = accs[f];
        if (i.location != SWIFTLY_B200_DEVICE || o.location != SWIFTLY_B200_DEVICE)
            return einval("subgrid_to_facets: device arrays only");
        if (i.n_lines != m || i.size != xM || i.elem_stride != 1)
            return einval("subgrid_to_facets: blocks must be xM_yN_size contiguous lines of xM_size");
        if (o.n_lines != m || o.size != yN || o.elem_stride != 1)
            return einval("subgrid_to_facets: accumulators must be xM_yN_size lines of yN_size");
        const int64_t sf = floordiv(facet_off1[f] * xM, h->N);
        BackFacet& F = op.fac[f];
        F.in = (const cplx*)i.data;
        F.out = (cplx*)o.data;
        F.in_ls = i.line_stride;
        F.out_ls = o.line_stride;
        F.sf_m = (int)pmod(sf, m);
        F.base_x = (int)pmod(xM / 2 - m / 2 + sf, xM);
    }
    SW_DEVICE_GUARD(h);
    const int64_t sc = floordiv(subgrid_off1 * yN, h->N);
    op.g.in = nullptr;
    op.g.out = nullptr;
    op.g.in_ls = op.g.in_es = op.g.out_ls = op.g.out_es = 0;
    op.g.n_lines = (int64_t)n_facets * m;
    op.fn = h->d_Fn;
    op.m = (int)m;
    op.xM = (int)xM;
    op.yN = (int)yN;
    op.lines_per = (int)m;
    op.s_m = (int)pmod(sc, m);
    op.base_y = (int)pmod(yN / 2 - m / 2 + sc, yN);
    op.scale = 1.0 / (double)m;
    return run_subgrid_to_facets(h, op, false, (cudaStream_t)stream);
}

// fold_column into half-row accumulators.  Window row u (centred row base0 + u) goes to stored
// row half_row(base0 + u); two rows of the window share a target when they are centred rows r and
// -r (mod yN) -- a window across centred offset 0 or yN/2.  Pass 1 adds every row but the
// conjugated member of such a pair, pass 2 those members, so that no launch has two lines with
// one target (plain read-modify-write, no atomics: the sums are deterministic).  Each pass is
// cut into runs of consecutive u, one launch each, in stream order.
static int fold_column_half(const swiftly_b200* h, const FoldColumnOp& base, cudaStream_t s) {
    const int n = base.n, m = base.lines_per;
    auto second = [&](int u) {  // conjugated member of a shared target
        bool cj;
        const int i = half_row(wrap_add(base.base0, u, n), n, cj);
        if (!cj) return false;
        const int partner = wrap_sub(wrap_add(i, n / 2, n), base.base0, n);  // centred n/2 + i
        return partner < m;
    };
    int runs[3 * 8];
    int n_runs = 0;
    for (int pass = 1; pass <= 2; ++pass) {
        for (int u = 0; u < m;) {
            if (second(u) != (pass == 2)) {
                ++u;
                continue;
            }
            int u1 = u + 1;
            while (u1 < m && second(u1) == (pass == 2)) ++u1;
            if (n_runs == 8) return einval("fold_column: window cut into more than 8 runs");
            runs[3 * n_runs] = u;
            runs[3 * n_runs + 1] = u1 - u;
            runs[3 * n_runs + 2] = pass;
            ++n_runs;
            u = u1;
        }
    }
    const int n_facets = (int)(base.g.n_lines / m);
    for (int r = 0; r < n_runs; ++r) {
        FoldColumnHalfOp op;
        static_cast<FoldColumnOp&>(op) = base;
        op.m = m;
        op.u_lo = runs[3 * r];
        op.lines_per = runs[3 * r + 1];
        op.g.n_lines = (int64_t)n_facets * op.lines_per;
        SW_TRY(run_fold_column_half(h, op, false, s));
    }
    for (int i = 0; i < 3 * n_runs; ++i) h->fold_runs[i] = runs[i];
    h->n_fold_runs = n_runs;
    return SWIFTLY_B200_OK;
}

// Fold one finished subgrid column into all facet accumulators (FoldColumnOp, kernels.cuh).
extern "C" int swiftly_b200_fold_column(const swiftly_b200* h, int n_facets,
                                        const swiftly_b200_lines* accs,
                                        const swiftly_b200_lines* facet_accs,
                                        const int64_t* facet_off1, const double* const* mask1,
                                        int64_t subgrid_off0, void* stream) {
    if (!h || !accs || !facet_accs || !facet_off1) return einval("fold_column: NULL argument");
    if (n_facets < 1 || n_facets > SW_MAX_COLUMN_FACETS)
        return einval("fold_column: between 1 and " + std::to_string(SW_MAX_COLUMN_FACETS) +
                      " facets per call");
    const int64_t yN = h->yN, m = h->m;
    // whole facet accumulators (yN rows), row rings (m rows) or half rows of a real image
    // (yN/2 + 1), the same for every facet
    const int64_t rows = facet_accs[0].n_lines == m                          ? m
                         : yN % 2 == 0 && facet_accs[0].n_lines == yN / 2 + 1 ? yN / 2 + 1
                                                                             : yN;
    const bool half = rows != m && rows == yN / 2 + 1;
    FoldColumnOp op;
    for (int f = 0; f < n_facets; ++f) {
        const swiftly_b200_lines& i = accs[f];
        const swiftly_b200_lines& o = facet_accs[f];
        if (i.location != SWIFTLY_B200_DEVICE || o.location != SWIFTLY_B200_DEVICE)
            return einval("fold_column: device arrays only");
        if (i.n_lines != m || i.size != yN || i.elem_stride != 1)
            return einval("fold_column: column accumulators must be xM_yN_size lines of yN_size");
        if (o.n_lines != rows || o.elem_stride != 1 || o.size > yN - 1)
            return einval("fold_column: facet accumulators must be yN_size (or, all of them, an "
                          "xM_yN_size ring, or yN_size/2 + 1 half rows, yN_size even) lines of "
                          "facet size");
        FoldFacet& F = op.fac[f];
        F.in = (const cplx*)i.data;
        F.out = (cplx*)o.data;
        F.mask = mask1 ? mask1[f] : nullptr;
        F.in_ls = i.line_stride;
        F.out_ls = o.line_stride;
        F.fs = (int)o.size;
        F.start1 = (int)pmod(yN / 2 - o.size / 2 + facet_off1[f], yN);
        F.fb_off = (int)((yN - 1) / 2 - o.size / 2);
        F.pad_ = 0;
    }
    SW_DEVICE_GUARD(h);
    const int64_t sc = floordiv(subgrid_off0 * yN, h->N);
    op.g.in = nullptr;
    op.g.out = nullptr;
    op.g.in_ls = op.g.in_es = op.g.out_ls = op.g.out_es = 0;
    op.g.n_lines = (int64_t)n_facets * m;
    op.fb = h->d_Fb;
    op.n = (int)yN;
    op.lines_per = (int)m;
    op.s0_m = (int)pmod(sc, m);
    op.base0 = (int)pmod(yN / 2 - m / 2 + sc, yN);
    if (rows == m) {  // row ring: line r mod m of window row r, as in extract_columns_impl
        op.s0_m = (int)pmod(op.s0_m - op.base0, m);
        op.base0 = 0;
    }
    if (half) return fold_column_half(h, op, (cudaStream_t)stream);
    return run_fold_column(h, op, false, (cudaStream_t)stream);
}
