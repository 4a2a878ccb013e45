// SwiFTly -- two-group variant of the fused subgrid axis kernel.
//
// Same mathematics and the same parameters as SubgridAxisKernel (kernels.cuh): for every
// output line the m-point transforms of the sources are overlap-added (Fn weighted) into an
// xM accumulator in shared memory, the xM-point inverse transform runs from there and the
// wanted xA samples are stored (api_helper.py:73-112, core.py:224-325).
//
// ONE persistent CTA per SM holds two thread groups, each with its own line, accumulator and
// exchange buffers (209 KiB of shared memory at m = 1024, xM = 4096).  What the layout buys:
//   * finished lines leave through the TMA engine: they are staged in the group's (idle) work
//     area and scattered by bulk tensor stores with ANY output strides -- transposed strips
//     for the axis-0 kernel, the owner's receive buffer on a peer GPU -- at no LSU cost;
//   * the next windows are pulled into L2 by bulk prefetches (one instruction per window);
//   * the xM-point transform exchanges COMPLEX samples (one trip per pass, two barriers)
//     through the accumulator's own storage: the accumulator is dead once the first pass has
//     loaded it;
//   * per-group output pointers / tensor maps (groups in different buffers).
//
// TOKENS (kept as a measured experiment, off by default): a line alternates between
// shared-memory exchange phases (LSU bound) and butterfly phases (FP64 bound); with the token
// the groups are forced into anti-phase through a pair of named barriers (bar.sync /
// bar.arrive), one exchanging while the other multiplies.  It measured slower than the
// default: a single 256-thread group reaches neither pipe's peak alone (tools/pipe_lab.cu) --
// the phases are latency bound at two warps per scheduler, so serialising them loses more than
// the overlap gains.
#pragma once

#include "kernels.cuh"

namespace swiftly {

template <int M, int XM, bool TOKENS>
struct SubgridAxisKernelPP {
    static constexpr int T_M = FftCfg<M>::T;
    static constexpr int T_X = FftCfg<XM>::T;
    static constexpr int GROUPS = 2;
    static constexpr int THREADS = T_X * GROUPS;
    static constexpr int CONC = T_X / T_M;  // concurrent m-point transforms per line
    static_assert(CONC >= 1 && CONC <= 4, "at most four concurrent m-point transforms");
    static constexpr int WSTRIDE = FftCfg<M>::PADDED | 1;
    // doubles per group; a multiple of 128 bytes: the work area doubles as the staging buffer of
    // the bulk tensor stores, whose shared-memory address must be 128-byte aligned
    static constexpr int WORK = (CONC * WSTRIDE + 15) & ~15;
    static constexpr int ACCS = XM + XM / 16;  // cplx per group: accumulator / xM exchange
    static constexpr size_t SMEM =
        (size_t)GROUPS * ((size_t)ACCS * sizeof(cplx) + (size_t)WORK * sizeof(double));
    static_assert(T_X % 32 == 0, "a thread group must be whole warps");
    // named barriers need whole warps; smaller transforms use the group barrier
    static constexpr bool SUB_BARRIERS = (T_M % 32 == 0) && CONC > 1;
    // a slot without a source can sit its round out only when its transform's barriers are its
    // own (with the group barrier or the token every slot has to take part in every exchange)
    static constexpr bool CAN_SKIP = SUB_BARRIERS && !TOKENS;

    // identical to SubgridAxisKernel
    SgSource src[SW_MAX_SOURCES];
    int n_slots;
    int n_groups;
    const double* fn;
    const cplx* tw_m;
    const cplx* tw_x;
    int64_t n_lines;
    cplx* out;
    int64_t out_ls, out_es, out_gs;
    int sz;
    int start[SW_MAX_GROUPS];
    const double* mask[SW_MAX_GROUPS];
    double scale;
    int first_round_tiles;
    int accumulate_out;
    // finished lines leave through the TMA engine: staged in the (idle) work buffer, then
    // bulk tensor stores scatter them with the output's strides
    int tma_out;
    int tma_box;                                       // samples per bulk tensor store
    int tma_slot_line, tma_slot_elem, tma_slot_group;  // coordinate slots (1..3)
    int tma_per_group;                 // one tensor map per group (groups in different buffers)
    int stagger_ns;                    // group 1 starts this much later than group 0 (see below)
    int stagger_cta_ns;                // CTA b starts (b mod 16) * this much later (see below)
    int cx_round0;                     // first round exchanges complex samples in the accumulator
    int pf_mode;                       // L2 prefetch: 0 bulk at the first exchange (default),
                                       // 1 none, 2 per-thread prefetch at the start of the round
    int compute_empty;                 // empty slots transform zeros and the accumulator is
                                       // cleared first unless the first round tiles it (the
                                       // former scheme, kept to compare against)
    cplx* out_g[SW_MAX_GROUPS];        // optional per-group output base (null: out + g * out_gs)
    // tensor maps travel as a separate __grid_constant__ kernel parameter (ctx.tmaps)
    struct Maps {
        TensorMap4 out_map[SW_MAX_GROUPS];  // [0] covers all groups unless tma_per_group
    };

    // barrier ids: 0 = whole CTA, 1 + g = group g, 3 + g * CONC + c = transform c of group g,
    // 11 + g = token of group g
    template <class Ctx>
    struct GroupSync {
        const Ctx& ctx;
        int bar_id, bar_count;  // barrier of the threads that share the exchange buffer
        int grp, t;
        // set at the start of a line whose predecessor left through the TMA engine: the first
        // exchange of the line is the first use of the work area (= the staging buffer), so
        // only THERE -- after the line's global loads and first butterflies -- thread 0 makes
        // sure the bulk stores have read it, and the barrier is widened to the whole group
        bool tma_pending;
        // L2 prefetch of the transform's NEXT window, issued at the first exchange of the round
        // and not together with the round's own loads: both at once would just double the burst
        // every SM sends to DRAM at the same moment
        const void* pf_ptr[2];
        uint32_t pf_bytes[2];
        // the accumulator update of a later round must come after ALL transforms of the
        // earlier rounds have stored (their windows overlap): one group barrier right before
        // the stores, instead of one after every round -- the concurrent transforms of a line
        // run on through the round boundary and drift apart, so that their load, exchange and
        // butterfly phases overlap instead of hitting the same pipe at the same moment
        bool order_stores;
        SW_HD void pre_store() const {
            if (order_stores) ctx.group_sync(1 + grp, T_X);
        }
        SW_HD void operator()() const { ctx.group_sync(bar_id, bar_count); }
        SW_HD void prefetch() {
            if (pf_bytes[0]) {
                ctx.bulk_prefetch_l2(pf_ptr[0], pf_bytes[0]);
                if (pf_bytes[1]) ctx.bulk_prefetch_l2(pf_ptr[1], pf_bytes[1]);
                pf_bytes[0] = pf_bytes[1] = 0;
            }
        }
        // a transform slot without a source in this round (no TOKENS): what the slot's threads
        // owe the rest of the group when they skip the transform -- the L2 prefetch of the
        // slot's next window and, after a line that left through the TMA engine, the wait for
        // the bulk stores together with the group-wide barrier of the first exchange.  The
        // transform's own barriers (3 + g * CONC + c) involve nobody else and are skipped; the
        // caller still owes pre_store().
        SW_HD void idle() {
            prefetch();
            if (tma_pending) {
                tma_pending = false;
                if (t == 0) ctx.bulk_wait_read();
                ctx.group_sync(1 + grp, T_X);
            }
        }
        // start of an exchange phase: with TOKENS wait for the token (the other group's
        // release); either way a barrier over (at least) the transform's threads
        SW_HD void acquire() {
            prefetch();
            if (tma_pending) {
                tma_pending = false;
                if (t == 0) ctx.bulk_wait_read();
                if (!TOKENS) {
                    ctx.group_sync(1 + grp, T_X);
                    return;
                }
            }
            if (TOKENS)
                ctx.group_sync(11 + grp, THREADS);
            else
                ctx.group_sync(bar_id, bar_count);
        }
        SW_HD void release() const {
            if (TOKENS) ctx.group_arrive(11 + (1 - grp), THREADS);
        }
    };

    template <class Ctx>
    SW_HD void operator()(Ctx& ctx) const {
        const int grp = ctx.tid / T_X;  // thread group = which of the CTA's two lines
        const int t = ctx.tid % T_X;    // thread within the group
        cplx* acc = (cplx*)ctx.smem + (size_t)grp * ACCS;
        double* work = (double*)((cplx*)ctx.smem + (size_t)GROUPS * ACCS) + (size_t)grp * WORK;
        const int c = t / T_M;
        const int lt = t % T_M;
        // slots without a source sit their round out (a sparse facet cover leaves up to three
        // of four slots of a round empty; otherwise they transform zeros)
        const bool skip_empty = CAN_SKIP && !compute_empty;
        GroupSync<Ctx> gsync{ctx, 1 + grp, T_X, grp, t, false, {nullptr, nullptr}, {0, 0}, false};
        GroupSync<Ctx> msync{ctx, SUB_BARRIERS ? 3 + grp * CONC + c : 1 + grp,
                             SUB_BARRIERS ? T_M : T_X, grp, t, false, {nullptr, nullptr}, {0, 0},
                             false};
        // group 1 hands the token to group 0 to start with
        if (TOKENS && grp == 1) ctx.group_arrive(11, THREADS);
        // The two groups run identical work and would stay in step: both waiting for their
        // windows at the same time, both in the lockstep xM transform at the same time.  Group 1
        // starts about half a line late, so that one group's load / xM phases fall into the
        // other group's m-point rounds.
        if (grp == 1 && stagger_ns > 0) {
            for (int left = stagger_ns; left > 0; left -= 1000) ctx.nap(1000);
        }
        // All CTAs of a launch start together and run identical work: chip-wide, the load phases
        // of every SM fall onto each other (HBM sees bursts) and so do the phases that leave the
        // memory system idle.  Spreading the start times over about one line de-phases the SMs.
        if (stagger_cta_ns > 0) {
            for (int left = (int)(ctx.bid % 16) * stagger_cta_ns; left > 0; left -= 1000)
                ctx.nap(left < 1000 ? left : 1000);
        }
        const int64_t pairs = (n_lines + GROUPS - 1) / GROUPS;  // line pairs per source group
        const int64_t total = pairs * n_groups;
        for (int64_t gl = ctx.bid; gl < total; gl += ctx.nblocks) {
            const int sgrp = (int)(gl / pairs);
            const int64_t line = (gl - (int64_t)sgrp * pairs) * GROUPS + grp;
            const bool line_ok = line < n_lines;
            // the previous line's bulk stores must have read the staging (= work) buffer before
            // the first exchange THROUGH THE WORK AREA writes it (see GroupSync::acquire)
            bool tma_wait_due = tma_out != 0;
            if (!skip_empty && !first_round_tiles) {
                for (int i = t; i < XM; i += T_X) acc[i] = mk(0.0, 0.0);
                gsync();
            }
            for (int slot0 = 0; slot0 < n_slots; slot0 += CONC) {
                // Which transforms of the round have a source (the same answer in every thread
                // of the group).  The windows of a round are pairwise disjoint, so the first
                // round stores instead of accumulating; the accumulator positions that no
                // window of the first round covers are cleared by the threads of its empty
                // slots, before the pre-store barrier of the next round (or the barrier ahead
                // of the xM-point transform).  CONC * M == XM: a first round without an empty
                // slot tiles the accumulator.
                unsigned act = 0;
#pragma unroll
                for (int k = 0; k < CONC; ++k)
                    if (line_ok && slot0 + k < n_slots && src[sgrp * n_slots + slot0 + k].base != nullptr)
                        act |= 1u << k;
                const bool overwrite = skip_empty ? slot0 == 0 : (first_round_tiles && slot0 == 0);
                const int slot = sgrp * n_slots + slot0 + c;
                const bool active = (act >> c) & 1u;
                const cplx* base = active ? src[slot].base + line * src[slot].ls : nullptr;
                const int64_t es = active ? src[slot].es : 0;
                const int wbase = active ? src[slot].wbase : 0;
                const int s_m = active ? src[slot].s_m : 0;
                const int wmod = active ? src[slot].wmod : 1;
                const int sf_m = active ? src[slot].sf_m : 0;
                const int pos_base = active ? src[slot].pos_base : 0;
                auto ld = [&](int q) {
                    if (!active) return mk(0.0, 0.0);
                    int tc = wrap_add(q, M / 2, M);
                    int idx = wrap_add(wbase, wrap_sub(tc, s_m, M), wmod);
                    return ld_stream(base + (int64_t)idx * es);
                };
                auto st = [&](int w, cplx v) {
                    if (!active) return;
                    int wc = wrap_add(w, M / 2, M);
                    int u = wrap_sub(wc, sf_m, M);
                    int pos = wrap_add(pos_base, u, XM);
                    double f = ldg_d(fn + u);
                    if (overwrite) {
                        acc[pos] = mk(f * v.x, f * v.y);
                    } else {
                        cplx a = acc[pos];
                        acc[pos] = mk(a.x + f * v.x, a.y + f * v.y);
                    }
                };
                // L2 prefetch of what this transform loads next -- the next round of this line, or
                // the first round of the group's next line: ONE bulk prefetch per window
                // (cp.async.bulk.prefetch.L2; the window is M contiguous samples, in two pieces
                // when it wraps), prepared here by the transform's first thread and issued at
                // the round's first exchange (GroupSync::acquire)
                if (pf_mode == 2 || (pf_mode == 0 && lt == 0)) {
                    int pslot0 = slot0 + CONC, psgrp = sgrp;
                    int64_t pline = line;
                    if (pslot0 >= n_slots) {
                        pslot0 = 0;
                        const int64_t ngl = gl + ctx.nblocks;
                        psgrp = (int)(ngl / pairs);
                        pline = (ngl - (int64_t)psgrp * pairs) * GROUPS + grp;
                        if (ngl >= total || pline >= n_lines) psgrp = -1;
                    }
                    if (psgrp >= 0 && pslot0 + c < n_slots) {
                        const SgSource& ps = src[psgrp * n_slots + pslot0 + c];
                        if (ps.base != nullptr && ps.es == 1) {
                            const cplx* pb = ps.base + pline * ps.ls;
                            const int first = ps.wbase;  // samples [first, first + M) mod wmod
                            const int n1 = first + M <= ps.wmod ? M : ps.wmod - first;
                            if (pf_mode == 2) {
#pragma unroll
                                for (int r = 0; r < 16; ++r) {
                                    int tc = wrap_add(lt + r * T_M, M / 2, M);
                                    int idx = wrap_add(ps.wbase, wrap_sub(tc, ps.s_m, M), ps.wmod);
                                    prefetch_l2(pb + idx);
                                }
                            } else {
                            msync.pf_ptr[0] = pb + first;
                            msync.pf_bytes[0] = (uint32_t)n1 * (uint32_t)sizeof(cplx);
                            msync.pf_ptr[1] = pb;
                            msync.pf_bytes[1] = (uint32_t)(M - n1) * (uint32_t)sizeof(cplx);
                            }
                        }
                    }
                }
                if (skip_empty && act == 0) {
                    // no transform in this round (a group with fewer rounds than the launch,
                    // a line past the end): the first round leaves a cleared accumulator
                    msync.prefetch();
                    if (slot0 == 0)
                        for (int i = t; i < XM; i += T_X) acc[i] = mk(0.0, 0.0);
                    continue;
                }
                // The transform's per-thread shared-memory offsets and twiddle addresses depend
                // on lt alone.  Left visible, the compiler computes them once per kernel and
                // keeps them live across every line, which overflows the 128-register budget and
                // spills them (plus transform data) to local memory, reloaded inside each pass
                // through an L1 the 209 KiB carveout has shrunk to ~28 KB.  An opaque copy of lt
                // per round makes them a few integer instructions per pass instead.
                int lt_r = lt;
                asm volatile("" : "+r"(lt_r));
                const bool cx = overwrite && cx_round0 && (!skip_empty || act == (1u << CONC) - 1);
                if (tma_wait_due && !cx) {
                    msync.tma_pending = true;
                    tma_wait_due = false;
                }
                if (skip_empty && !active) {
                    msync.idle();
                    if (overwrite) {
                        // the first round's uncovered positions, shared by its empty slots
                        int rank = 0, n_idle = 0;
#pragma unroll
                        for (int k = 0; k < CONC; ++k)
                            if (!((act >> k) & 1u)) {
                                rank += k < c;
                                ++n_idle;
                            }
                        for (int i = rank * T_M + lt; i < XM; i += n_idle * T_M) {
                            bool covered = false;
#pragma unroll
                            for (int k = 0; k < CONC; ++k)
                                if ((act >> k) & 1u)
                                    covered |= wrap_sub(i, src[sgrp * n_slots + slot0 + k].pos_base, XM) < M;
                            if (!covered) acc[i] = mk(0.0, 0.0);
                        }
                    }
                    msync.order_stores = slot0 > 0;
                    msync.pre_store();
                } else if (cx) {
                    // First round of a tiling layout: the accumulator holds nothing yet, so its
                    // storage serves as COMPLEX exchange buffers of the round's transforms (one
                    // trip, two barriers per pass instead of two trips and four; CONC * (M +
                    // M / 16) samples = exactly the accumulator's padded size).  The stores into
                    // the accumulator then have to wait until every transform of the round has
                    // left its buffer: the pre-store group barrier.
                    msync.order_stores = true;
                    line_fft_cx<M, -1, false>(lt_r, acc + (size_t)c * (M + M / 16), tw_m, ld, st, msync);
                } else {
                    msync.order_stores = slot0 > 0;
                    line_fft<M, -1>(lt_r, work + (size_t)c * WSTRIDE, tw_m, ld, st, msync);
                }
            }
            if (tma_wait_due && t == 0) ctx.bulk_wait_read();  // (no round used the work area)
            gsync();  // accumulator complete
            {
                cplx* o = (out_g[sgrp] ? out_g[sgrp] : out + (int64_t)sgrp * out_gs) + line * out_ls;
                const int gstart = start[sgrp];
                const double* gmask = mask[sgrp];
                auto ld = [&](int q) { return acc[wrap_add(q, XM / 2, XM)]; };
                cplx* stage = (cplx*)work;
                auto st = [&](int p, cplx v) {
                    int pc = wrap_add(p, XM / 2, XM);
                    int r = wrap_sub(pc, gstart, XM);
                    if (line_ok && r < sz) {
                        double f = gmask ? scale * ldg_d(gmask + r) : scale;
                        cplx* dst = o + (int64_t)r * out_es;
                        if (tma_out) {
                            stage[r] = cscale(v, f);
                        } else if (accumulate_out) {
                            cplx a = *dst;
                            *dst = mk(a.x + f * v.x, a.y + f * v.y);
                        } else {
                            st_stream(dst, cscale(v, f));
                        }
                    }
                };
                // the exchange buffer IS the accumulator: the acquire() (a group barrier) of
                // the first pass comes after every thread's loads; t_r: as lt_r above
                int t_r = t;
                asm volatile("" : "+r"(t_r));
                line_fft_cx<XM, +1, true>(t_r, acc, tw_x, ld, st, gsync);
            }
            gsync();  // accumulator is rewritten by the next line; staged line complete
            if (tma_out && t == 0 && line_ok) {
                ctx.fence_async();
                int c[4] = {0, 0, 0, 0};
                c[tma_slot_line] = (int)line;
                c[tma_slot_group] = tma_per_group ? 0 : sgrp;
                const TensorMap4* map = &((const Maps*)ctx.tmaps)->out_map[tma_per_group ? sgrp : 0];
                for (int r0 = 0; r0 < sz; r0 += tma_box) {
                    c[tma_slot_elem] = r0;
                    ctx.tensor_store(map, (const cplx*)work + r0, c[1], c[2], c[3]);
                }
                ctx.bulk_commit();
            }
        }
        // the strips may go to a peer GPU: the kernel ends only when the bulk stores are performed
        if (tma_out && t == 0) ctx.bulk_wait_all();
        // consume group 1's last release so that every barrier ends balanced
        if (TOKENS && grp == 0) ctx.group_sync(11, THREADS);
    }
};

}  // namespace swiftly
