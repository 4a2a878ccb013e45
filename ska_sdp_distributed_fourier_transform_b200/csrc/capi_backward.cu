// SwiFTly -- C ABI of the fused subgrid side of the backward path (device memory only).
#include <vector>

#include "capi_util.h"

using namespace swiftly;

extern "C" int swiftly_b200_split_axis_supported(const swiftly_b200* h) {
    return h ? subgrid_split_conc((int)h->m, (int)h->xM) : 0;
}

// prepare_subgrid along one axis + extract_from_subgrid for every target (+ add_to_facet in
// add mode), SubgridSplitAxisKernel (kernels.cuh).  Group g: input lines inputs[g], subgrid
// offset subgrid_offs[g], targets [sum(group_sizes[:g]), ... + group_sizes[g]).
extern "C" int swiftly_b200_split_subgrid_axis(const swiftly_b200* h,
                                               const swiftly_b200_lines* inputs, int n_groups,
                                               const int64_t* subgrid_offs,
                                               const swiftly_b200_split_target* targets,
                                               const int32_t* group_sizes, int mode,
                                               void* stream) {
    if (!h || !inputs || !subgrid_offs || !group_sizes)
        return einval("split_subgrid_axis: NULL argument");
    if (mode != SWIFTLY_B200_SPLIT_STORE && mode != SWIFTLY_B200_SPLIT_ADD)
        return einval("split_subgrid_axis: mode must be SWIFTLY_B200_SPLIT_STORE or _ADD");
    if (n_groups < 1) return einval("split_subgrid_axis: need at least one group");
    for (int g = 0; g < n_groups; ++g) {
        if (group_sizes[g] < 0) return einval("split_subgrid_axis: negative group size");
        if (group_sizes[g] > 0 && !targets) return einval("split_subgrid_axis: NULL argument");
    }
    const int64_t N = h->N, yN = h->yN, xM = h->xM, m = h->m;
    if (!subgrid_split_conc((int)m, (int)xM)) {
        set_error("split_subgrid_axis: no fused kernel for m=" + std::to_string(m) +
                  ", xM=" + std::to_string(xM));
        return SWIFTLY_B200_EUNSUPPORTED;
    }
    const int64_t n_lines = inputs[0].n_lines;
    int64_t total = 0;
    for (int g = 0; g < n_groups; ++g) {
        const swiftly_b200_lines& in = inputs[g];
        if (in.location != SWIFTLY_B200_DEVICE)
            return einval("split_subgrid_axis: device arrays only");
        if (in.n_lines != n_lines)
            return einval("split_subgrid_axis: every group must have the same number of lines");
        if (in.size < 0 || in.size > xM)
            return einval("split_subgrid_axis: subgrid size exceeds padded subgrid size");
        if (in.n_lines > 0 && in.size > 0 && !in.data)
            return einval("split_subgrid_axis: NULL input pointer");
        for (int i = (int)total; i < total + group_sizes[g]; ++i) {
            const swiftly_b200_split_target& t = targets[i];
            if (!t.data) return einval("split_subgrid_axis: NULL target pointer");
            if (t.n_lines != n_lines)
                return einval("split_subgrid_axis: target has " + std::to_string(t.n_lines) +
                              " lines, input " + std::to_string(n_lines));
            // one round adds several targets of a group at once: they must not share memory
            if (mode == SWIFTLY_B200_SPLIT_ADD)
                for (int j = (int)total; j < i; ++j)
                    if (targets[j].data == t.data)
                        return einval("split_subgrid_axis: add-mode targets of one group must "
                                      "be distinct accumulators");
        }
        total += group_sizes[g];
    }
    if (n_lines <= 0 || total == 0) return SWIFTLY_B200_OK;
    SW_DEVICE_GUARD(h);

    // pieces of at most SW_MAX_SOURCES targets (a longer group is split: each piece prepares
    // the input again), packed in order into launches of at most SW_MAX_GROUPS pieces and
    // SW_MAX_SOURCES targets; targets are independent, so the pieces need no ordering
    // beyond what shared accumulators get from the stream order
    struct Piece {
        int g, first, count;
    };
    std::vector<Piece> pieces;
    int first = 0;
    for (int g = 0; g < n_groups; ++g) {
        for (int k = 0; k < group_sizes[g]; k += SW_MAX_SOURCES) {
            const int cnt = group_sizes[g] - k < SW_MAX_SOURCES ? group_sizes[g] - k : SW_MAX_SOURCES;
            pieces.push_back({g, first + k, cnt});
        }
        first += group_sizes[g];
    }
    size_t p0 = 0;
    while (p0 < pieces.size()) {
        size_t p1 = p0;
        int used = 0;
        while (p1 < pieces.size() && (int)(p1 - p0) < SW_MAX_GROUPS &&
               used + pieces[p1].count <= SW_MAX_SOURCES)
            used += pieces[p1++].count;
        SubgridSplitArgs a;
        for (int i = 0; i < SW_MAX_SOURCES; ++i) {
            a.tgt[i].base = nullptr;
            a.tgt[i].ls = a.tgt[i].es = 0;
            a.tgt[i].sf_m = a.tgt[i].pos_base = 0;
        }
        for (int g = 0; g < SW_MAX_GROUPS; ++g) a.grp[g] = SplitGroup{nullptr, 0, 0, 0, 0, 0, 0, 0, 0};
        int slot = 0;
        for (size_t p = p0; p < p1; ++p) {
            const Piece& pc = pieces[p];
            const swiftly_b200_lines& in = inputs[pc.g];
            const int64_t off = subgrid_offs[pc.g];
            const int64_t sc = floordiv(off * yN, N);
            SplitGroup& G = a.grp[p - p0];
            G.in = (const cplx*)in.data;
            G.in_ls = in.line_stride;
            G.in_es = in.elem_stride;
            G.sz = (int)in.size;
            G.start = (int)pmod(xM / 2 - in.size / 2 + off, xM);
            G.s_m = (int)pmod(sc, m);
            G.base_y = (int)pmod(yN / 2 - m / 2 + sc, yN);
            G.first = slot;
            G.count = pc.count;
            for (int i = pc.first; i < pc.first + pc.count; ++i) {
                const swiftly_b200_split_target& t = targets[i];
                const int64_t sf = floordiv(t.facet_off * xM, N);
                SplitTarget& T = a.tgt[slot++];
                T.base = (cplx*)t.data;
                T.ls = t.line_stride;
                T.es = t.elem_stride;
                T.sf_m = (int)pmod(sf, m);
                T.pos_base = (int)pmod(xM / 2 - m / 2 + sf, xM);
            }
        }
        a.n_groups = (int)(p1 - p0);
        a.n_lines = n_lines;
        a.add = mode == SWIFTLY_B200_SPLIT_ADD ? 1 : 0;
        SW_TRY(run_subgrid_split(h, a, (cudaStream_t)stream));
        p0 = p1;
    }
    return SWIFTLY_B200_OK;
}
