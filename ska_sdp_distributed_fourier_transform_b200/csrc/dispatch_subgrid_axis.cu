// SwiFTly -- dispatch of the fused subgrid axis kernel over (m, xM) pairs.
#include "dispatch.cuh"
#include "subgrid_pp.cuh"

namespace swiftly {

template <int M, int XM, int LINES>
static int launch_sg_axis_l(const swiftly_b200* h, const SubgridAxisArgs& a, cudaStream_t s) {
    SubgridAxisKernel<M, XM, LINES> k;
    for (int i = 0; i < SW_MAX_SOURCES; ++i) k.src[i] = a.src[i];
    k.n_slots = a.n_slots;
    k.n_groups = a.n_groups;
    k.fn = h->d_Fn;
    k.tw_m = twiddles(h, M);
    k.tw_x = twiddles(h, XM);
    if (!k.tw_m || !k.tw_x) return SWIFTLY_B200_ECUDA;
    k.n_lines = a.n_lines;
    k.out = a.out;
    k.out_ls = a.out_ls;
    k.out_es = a.out_es;
    k.out_gs = a.out_gs;
    k.sz = a.sz;
    for (int g = 0; g < SW_MAX_GROUPS; ++g) {
        k.start[g] = a.start[g];
        k.mask[g] = a.mask[g];
        k.out_g[g] = a.out_g[g];
    }
    k.scale = 1.0 / (double)XM;
    k.first_round_tiles = a.first_round_tiles;
    k.accumulate_out = a.accumulate_out;
    int grid = grid_for(((a.n_lines + LINES - 1) / LINES) * a.n_groups, 1);
    if (h->max_blocks > 0 && grid > h->max_blocks) grid = h->max_blocks;  // (test hook)
    cudaError_t e = launch_body(k, grid, k.SMEM, s);
    return e == cudaSuccess ? SWIFTLY_B200_OK : cuda_fail(e, "subgrid axis kernel launch");
}

// ping-pong variant: two thread groups (two lines) per CTA, LSU token between them
template <int M, int XM, bool TOKENS>
static int launch_sg_axis_pp(const swiftly_b200* h, const SubgridAxisArgs& a, cudaStream_t s) {
    typedef SubgridAxisKernelPP<M, XM, TOKENS> K;
    K k;
    static thread_local typename K::Maps maps;
    for (int i = 0; i < SW_MAX_SOURCES; ++i) k.src[i] = a.src[i];
    k.n_slots = a.n_slots;
    k.n_groups = a.n_groups;
    k.fn = h->d_Fn;
    k.tw_m = twiddles(h, M);
    k.tw_x = twiddles(h, XM);
    if (!k.tw_m || !k.tw_x) return SWIFTLY_B200_ECUDA;
    k.n_lines = a.n_lines;
    k.out = a.out;
    k.out_ls = a.out_ls;
    k.out_es = a.out_es;
    k.out_gs = a.out_gs;
    k.sz = a.sz;
    for (int g = 0; g < SW_MAX_GROUPS; ++g) {
        k.start[g] = a.start[g];
        k.mask[g] = a.mask[g];
        k.out_g[g] = a.out_g[g];
    }
    k.scale = 1.0 / (double)XM;
    k.first_round_tiles = a.first_round_tiles;
    k.accumulate_out = a.accumulate_out;
    // finished lines through the TMA engine when the staging buffer (the work area) holds a
    // line and the output can be described by a tensor map; sg_variant 5: direct stores
    k.tma_out = 0;
    k.tma_box = a.sz < 256 ? a.sz : 256;
    k.tma_slot_line = k.tma_slot_elem = k.tma_slot_group = 1;
    k.tma_per_group = a.out_g[0] != nullptr ? 1 : 0;
    k.pf_mode = h->sg_variant == 11 ? 1 : (h->sg_variant == 12 ? 2 : 0);
    k.stagger_ns = h->sg_variant == 13 ? 5000 : (h->sg_variant == 14 ? 2500 : 0);
    // CTA b starts (b mod 16) * 400 ns late: all CTAs of a launch run identical work and would
    // stay in phase chip-wide (every SM loading at the same moment, then none).  sg_variant 24:
    // no stagger; 22 / 23: 800 / 1300 ns (tools/quick_k3.py times them)
    k.stagger_cta_ns = h->sg_variant == 24 ? 0 : (h->sg_variant == 22 ? 800 : (h->sg_variant == 23 ? 1300 : 400));
    // sg_variant 16: the first round exchanges complex samples through the (still empty)
    // accumulator.  Measured slower: the group barrier it needs before the
    // round's stores re-aligns the transforms that the split-exchange form lets drift apart.
    k.cx_round0 = (h->sg_variant == 16 && XM == (XM / M) * M && M > 16) ? 1 : 0;
    // sg_variant 25: the former round scheme -- transform slots without a source transform
    // zeros, and the accumulator is cleared ahead of the rounds unless the first round tiles it
    // (tools/quick_k3.py compares it with the default)
    k.compute_empty = h->sg_variant == 25 ? 1 : 0;
    // (the last box may be partial: the engine still reads a whole box from shared memory)
    const size_t staged = (size_t)((a.sz + k.tma_box - 1) / (k.tma_box > 0 ? k.tma_box : 1)) *
                          (size_t)k.tma_box * sizeof(cplx);
    if (!a.accumulate_out && h->sg_variant != 5 && a.sz >= 1 &&
        staged <= (size_t)k.WORK * sizeof(double)) {
        int slot[3];
        bool ok = true;
        if (k.tma_per_group) {
            // (the slots depend on the strides only, which all groups share)
            for (int g = 0; g < a.n_groups && ok; ++g)
                ok = make_out_map(&maps.out_map[g], a.out_g[g], a.out_ls, a.out_es, 0, a.n_lines,
                                  a.sz, 1, k.tma_box, slot);
        } else {
            ok = make_out_map(&maps.out_map[0], a.out, a.out_ls, a.out_es, a.out_gs, a.n_lines,
                              a.sz, a.n_groups, k.tma_box, slot);
        }
        if (ok) {
            k.tma_out = 1;
            k.tma_slot_line = slot[0];
            k.tma_slot_elem = slot[1];
            k.tma_slot_group = slot[2];
        }
    }
    // persistent: one CTA per SM, every CTA walks over line pairs
    int64_t pairs = ((a.n_lines + 1) / 2) * a.n_groups;
    int grid = (int)(pairs < NUM_SMS ? pairs : NUM_SMS);
    cudaError_t e = launch_body_maps(k, maps, grid, k.SMEM, s);
    return e == cudaSuccess ? SWIFTLY_B200_OK : cuda_fail(e, "subgrid axis (two-group) kernel launch");
}

// The two-group kernel takes power-of-two lengths with CONC = 2 or 4.  The catalogue's other
// pairs run the round-1 kernel: CONC = 8 (m = 128, xM = 1024: eight-thread transforms), CONC = 1
// (m = xM = 256: one source per round) and the mixed-radix lengths (3, 5, 7 * 2^k).
template <int M, int XM>
struct PingPongFits {
    static constexpr bool POW2 = (M & (M - 1)) == 0 && (XM & (XM - 1)) == 0 && XM / M >= 2;
#if defined(SWIFTLY_EMU)
    static constexpr bool V = POW2 && (XM / M) <= 4;
#else
    static constexpr bool V = POW2 && (XM / M) <= 4 && (XM / 16) % 32 == 0 &&
                              2 * ((size_t)(XM + XM / 16) * 16 + (size_t)(XM + XM / 16 + 24) * 8) <=
                                  227 * 1024;
#endif
};

// two adjacent lines per CTA when every source and the output have unit line stride
template <int M, int XM>
static int launch_sg_axis(const swiftly_b200* h, const SubgridAxisArgs& a, cudaStream_t s) {
    bool adjacent = a.out_ls == 1 && a.n_lines > 1;
    for (int i = 0; i < SW_MAX_SOURCES && adjacent; ++i)
        if (a.src[i].base && a.src[i].ls != 1) adjacent = false;
    if constexpr (PingPongFits<M, XM>::V) {
        // sg_variant (debug hook): 0 = two-group kernel (default), 1 = round-1 kernel,
        // 2 = two-group kernel WITH the LSU token (measured slower: a single group cannot
        // saturate either pipe alone, see subgrid_pp.cuh), 5 = two-group, direct stores
        if (!adjacent && h->sg_variant != 1)
            return h->sg_variant == 2 ? launch_sg_axis_pp<M, XM, true>(h, a, s)
                                      : launch_sg_axis_pp<M, XM, false>(h, a, s);
    }
    // 2 lines need 2 x (acc + work) of shared memory: only the pairs that fit
    if constexpr (2 * ((size_t)(XM + 4) * sizeof(cplx) + (size_t)(XM + XM / 16 + 40) * 8) <=
                      227 * 1024 &&
                  SubgridAxisKernel<M, XM, 2>::SMEM <= 227 * 1024) {
        if (adjacent) return launch_sg_axis_l<M, XM, 2>(h, a, s);
    }
    return launch_sg_axis_l<M, XM, 1>(h, a, s);
}

// the last six: the catalogue pairs outside xM / m in {2, 4} (swift_configs.json)
#define SW_SG_PAIRS(X) \
    X(32, 64) X(32, 128) X(64, 128) X(64, 256) X(128, 256) X(128, 512) X(256, 512) X(256, 1024) \
    X(512, 1024) X(512, 2048) X(1024, 2048) X(1024, 4096) X(2048, 4096) X(2048, 8192)         \
    X(128, 1024) X(256, 256) X(128, 384) X(160, 320) X(192, 384) X(224, 448)

int subgrid_axis_conc(int m, int xM) {
#define X(M, XM) if (m == M && xM == XM) return XM / M;
    SW_SG_PAIRS(X)
#undef X
    return 0;
}

int run_subgrid_axis(const swiftly_b200* h, const SubgridAxisArgs& a, cudaStream_t s) {
    const int m = (int)h->m, xM = (int)h->xM;
#define X(M, XM) if (m == M && xM == XM) return launch_sg_axis<M, XM>(h, a, s);
    SW_SG_PAIRS(X)
#undef X
    set_error("no fused subgrid kernel for m=" + std::to_string(m) + ", xM=" + std::to_string(xM));
    return SWIFTLY_B200_EUNSUPPORTED;
}

}  // namespace swiftly
