// SwiFTly -- K2 ("Fb . FFT . extract", the reference's extract_column task,
// api_helper.py:200-210 = extract_from_facet(axis 0) + prepare_facet(axis 1),
// core.py:189-253) with the facet rows staged in shared memory by the TMA engine.
//
// One persistent CTA per SM walks over output lines.  A line's input is one contiguous row of
// the axis-0 prepared facet BF_F (fs samples; the row gather of extract_from_facet is just the
// choice of the row).  The row is brought into shared memory by ONE bulk asynchronous copy
// (cp.async.bulk.shared.global, completion on an mbarrier) that is issued while the PREVIOUS
// line is still being transformed: as soon as the last first-pass load of the current line has
// read the staging buffer, the copy of the next row starts and runs under the remaining
// passes, the combine and the stores.  The first-pass loads therefore hit shared memory instead
// of exposing a DRAM round trip with every warp of the SM waiting in the same phase.
//
// SPLIT = true : line length 2 H (yN = 16384 = 2 x 8192), decimation in time; E = FFT_H(even
//                samples) is parked in a per-CTA scratch line (L2), O = FFT_H(odd samples),
//                X[k] = E[k] + w^k O[k], X[k + H] = E[k] - w^k O[k] (as SplitLineKernel).
// SPLIT = false: line length H, one transform straight from the staging buffer.
#pragma once

#include "kernels.cuh"

namespace swiftly {

// Start the asynchronous copy of the input row of output line `line` into the staging buffer
// `in` (called by ONE thread; completion on the mbarrier `bar`): bulk TENSOR loads with the
// 128-byte swizzle when the rows are whole 128-byte chunks (tensor_map.cu make_row_map; a box
// that sticks out of the row is zero filled and still counts in full), else 1-D bulk copies in
// pieces of at most 64 KiB.  Shared by all TMA-staged K2 kernels.
// PAIR: the row goes to the same offsets in both CTAs of a two-CTA cluster (multicast); the
// issuing thread, of either CTA, arms both CTAs' barriers.
// HALF: the rows are half rows (include/swiftly_b200.h): the window row's stored row is fetched.
template <class Maps, bool PAIR = false, bool HALF = false, class Ctx>
SW_HD void k2_issue_row(const Ctx& ctx, const ExtractColumnsOp& op, int swizzled, int box_chunks,
                        cplx* in, uint64_t* bar, int64_t line) {
    const int f = (int)(line / op.lines_per);
    const int l = (int)(line - (int64_t)f * op.lines_per);
    const ColumnFacet& F = op.fac[f];
    int64_t row = wrap_add(op.rm_base, wrap_sub(l, op.rm_s_m, op.lines_per), op.n);
    if constexpr (HALF) {
        bool cj;
        row = half_row((int)row, op.n, cj);
    }
    auto expect = [&](uint32_t bytes) {
        if constexpr (PAIR) {
            ctx.tx_expect_peer(bar, 0, bytes);
            ctx.tx_expect_peer(bar, 1, bytes);
        } else {
            ctx.tx_expect(bar, bytes);
        }
    };
    if (swizzled) {
        const int chunks = F.fs / 8;
        const int boxes = (chunks + box_chunks - 1) / box_chunks;
        expect((uint32_t)boxes * (uint32_t)box_chunks * 128u);
        for (int c0 = 0; c0 < chunks; c0 += box_chunks) {
            const TensorMap4* map = &((const Maps*)ctx.tmaps)->in_map[f];
            if constexpr (PAIR)
                ctx.tensor_load_mc((char*)in + (size_t)c0 * 128, map, c0, (int)row, bar, 3);
            else
                ctx.tensor_load((char*)in + (size_t)c0 * 128, map, c0, (int)row, bar);
        }
        return;
    }
    const uint32_t bytes = (uint32_t)F.fs * (uint32_t)sizeof(cplx);
    expect(bytes);
    const char* src = (const char*)(F.in + row * F.in_ls);
    for (uint32_t o = 0; o < bytes; o += 65536u) {
        const uint32_t piece = bytes - o < 65536u ? bytes - o : 65536u;
        if constexpr (PAIR)
            ctx.tx_copy_mc((char*)in + o, src + o, piece, bar, 3);
        else
            ctx.tx_copy((char*)in + o, src + o, piece, bar);
    }
}

// HALF (every TMA form the default dispatch runs): the rows are half rows; a line whose window
// row is stored conjugated negates the imaginary part of every staged sample it reads.
template <int H, bool SPLIT, bool HALF = false>
struct ExtractColumnsTmaKernel {
    static constexpr int DIR = +1;
    static constexpr int T = FftCfg<H>::T;
    static constexpr int THREADS = T;
    static constexpr int N = SPLIT ? 2 * H : H;  // line length yN
    // staging buffer: up to N - 1 facet samples (fs <= yN - 1); exchange buffer; mbarrier
    static constexpr size_t smem_bytes(int in_cap) {
        return (size_t)in_cap * sizeof(cplx) + (size_t)FftCfg<H>::PADDED * sizeof(double) + 16;
    }

    ExtractColumnsOp op;
    const cplx* tw;   // compact table of the H-point plan
    const cplx* tw2;  // exp(-2 pi i t / 2H), t < H (SPLIT only)
    cplx* scratch;    // gridDim.x * H samples (SPLIT only)
    int in_cap;       // capacity of the staging buffer in samples (>= every facet's fs, even)
    // rows staged by bulk TENSOR loads with the 128-byte swizzle (tensor_map.cu make_row_map):
    // the E / O transforms read every second sample of the row -- 32-byte stride, a 2-way
    // bank conflict on a linear buffer, conflict free on the swizzled one
    int swizzled;
    int box_chunks;  // 128-byte chunks per tensor load
    // tensor maps travel as a separate __grid_constant__ kernel parameter (ctx.tmaps)
    struct Maps {
        TensorMap4 in_map[SW_MAX_COLUMN_FACETS];
    };

    // first-pass loads must be done before the staging buffer is refilled: the refill is issued
    // by thread 0 right after the first barrier that follows them
    template <class Ctx>
    struct RefillSync {
        const Ctx& ctx;
        const ExtractColumnsTmaKernel& k;
        cplx* in;
        uint64_t* bar;
        int64_t next_line;
        bool pending;
        SW_HD void operator()() {
            ctx.sync();
            if (pending) {
                pending = false;
                if (ctx.tid == 0 && next_line < k.op.g.n_lines) k.issue(ctx, in, bar, next_line);
            }
        }
    };

    template <class Ctx>
    SW_HD void issue(const Ctx& ctx, cplx* in, uint64_t* bar, int64_t line) const {
        k2_issue_row<Maps, false, HALF>(ctx, op, swizzled, box_chunks, in, bar, line);
    }

    template <class Ctx>
    SW_HD void operator()(Ctx& ctx) const {
        cplx* in = (cplx*)ctx.smem;
        double* sm = (double*)(in + in_cap);
        uint64_t* bar = (uint64_t*)(sm + ((FftCfg<H>::PADDED + 1) & ~1));
        cplx* stash = SPLIT ? scratch + (size_t)ctx.bid * H : nullptr;
        const int lt = ctx.tid;
        const int n = op.n;
        if (ctx.tid == 0) {
            ctx.tx_init(bar);
            if ((int64_t)ctx.bid < op.g.n_lines) issue(ctx, in, bar, ctx.bid);
        }
        ctx.sync();
        uint32_t parity = 0;
        for (int64_t line = ctx.bid; line < op.g.n_lines; line += ctx.nblocks) {
            const int f = (int)(line / op.lines_per);
            const int l = (int)(line - (int64_t)f * op.lines_per);
            const ColumnFacet& F = op.fac[f];
            const int shift_in = F.shift_in, fs = F.fs;
            const double* fb = op.fb ? op.fb + F.fb_off : nullptr;
            cplx* o = F.out + (int64_t)l * F.out_ls;
            const double scale = op.scale;
            const bool swz = swizzled != 0;
            // natural-order input sample q of the zero-padded, rotated, Fb-weighted row
            bool cj = false;
            if constexpr (HALF) half_row(wrap_add(op.rm_base, wrap_sub(l, op.rm_s_m, op.lines_per), n), n, cj);
            auto sample = [&](int q) {
                int k = wrap_add(q, shift_in, n);
                if (k >= fs) return mk(0.0, 0.0);
                const int ks = swz ? ((k & ~7) | ((k ^ (k >> 3)) & 7)) : k;
                if constexpr (HALF) {
                    const cplx x = fb ? cscale(in[ks], ldg_d(fb + k)) : in[ks];
                    return cj ? cconj(x) : x;
                } else {
                    return fb ? cscale(in[ks], ldg_d(fb + k)) : in[ks];
                }
            };
            auto put = [&](int p, cplx v) {
                int pc = wrap_add(p, n / 2, n);
                st_stream(o + pc, cscale(v, scale));
            };
            ctx.tx_wait(bar, parity);  // this line's row has landed
            parity ^= 1;
            RefillSync<Ctx> refill{ctx, *this, in, bar, line + ctx.nblocks, false};
            if constexpr (SPLIT) {
                {
                    auto sync = [&]() { ctx.sync(); };
                    auto ld = [&](int q) { return sample(2 * q); };
                    auto st = [&](int k, cplx v) { stash[k] = v; };
                    line_fft<H, DIR>(lt, sm, tw, ld, st, sync);
                }
                ctx.sync();
                {
                    auto ld = [&](int q) { return sample(2 * q + 1); };
                    // w^k for the thread's outputs k = j0 + it * T + r * NS by recurrence: one
                    // table load per thread, then multiplications by the two step factors
                    // w^T and w^NS (loading every w^k exposed an L2 round trip per output)
                    typedef LastPass<H> LP;
                    auto unit = [&](int t) {  // exp(DIR 2 pi i t / 2H), 0 <= t < 2H
                        const bool neg = t >= H;
                        cplx w = ldg_c(tw2 + (neg ? t - H : t));
                        if (DIR > 0) w.y = -w.y;
                        return neg ? mk(-w.x, -w.y) : w;
                    };
                    const cplx step_it = unit(T), step_r = unit(LP::NS % (2 * H));
                    cplx w_it = mk(1.0, 0.0), w = mk(1.0, 0.0);
                    auto st = [&](int k, cplx od, int it, int r) {
                        if (r == 0) {
                            w_it = it == 0 ? unit(k) : cmul(w_it, step_it);
                            w = w_it;
                        } else {
                            w = cmul(w, step_r);
                        }
                        cplx e = stash[k];
                        cplx wo = cmul(od, w);
                        put(k, cadd(e, wo));
                        put(k + H, csub(e, wo));
                    };
                    refill.pending = true;
                    line_fft<H, DIR>(lt, sm, tw, ld, st, refill);
                }
            } else {
                auto ld = [&](int q) { return sample(q); };
                refill.pending = true;
                line_fft<H, DIR>(lt, sm, tw, ld, put, refill);
            }
            ctx.sync();  // exchange buffer is reused by the next line
        }
    }
};

// ---------------------------------------------------------------------------------------
// yN = 4 Q: the line as FOUR Q-point transforms (decimation in time by 4), two thread groups.
//
//   e_q[j] = z[4 j + q],  E_q = FFT_Q(e_q),  t_q[k] = w^(q k) E_q[k],  w = exp(+2 pi i / yN)
//   X[k + Q s] = sum_q t_q[k] (+i)^(q s)                      (radix-4 butterfly over q)
//
// Compared with the 2 x (yN/2) split above: a Q = 4096 point transform needs two exchanges
// instead of three (a third less shared-memory traffic for the same samples), and -- more
// important -- the CTA is TWO independent groups of Q/16 threads, each with its own exchange
// buffer and named barrier, working on different sub-transforms of the SAME staged row
// (group g: q = 2g, 2g + 1): their exchange (LSU) and butterfly (FP64) phases drift apart and
// overlap, where 512 threads in lockstep leave one pipe idle while the other works.  The
// stride-4 reads of the staged row are conflict free thanks to the 128-byte swizzle.  All
// four t_q are parked in a per-CTA scratch (L2 resident); after a CTA barrier every thread
// combines its share of the k range and writes four unit-stride output streams.
template <int Q, bool HALF = false>
struct ExtractColumnsTma4Kernel {
    static constexpr int DIR = +1;
    static constexpr int TG = FftCfg<Q>::T;  // threads per group
    static constexpr int THREADS = 2 * TG;
    static constexpr int N = 4 * Q;
    static constexpr int XBUF = (FftCfg<Q>::PADDED + 1) & ~1;  // doubles per exchange buffer
    static constexpr size_t smem_bytes(int in_cap) {
        return (size_t)in_cap * sizeof(cplx) + 2 * (size_t)XBUF * sizeof(double) + 32;
    }

    ExtractColumnsOp op;
    const cplx* tw;   // compact table of the Q-point plan
    const cplx* twf;  // exp(-2 pi i t / yN), t < yN / 2
    cplx* scratch;    // gridDim.x * 4 Q samples
    int in_cap;
    int swizzled;
    int box_chunks;
    struct Maps {
        TensorMap4 in_map[SW_MAX_COLUMN_FACETS];
    };

    SW_HD cplx root(int t) const {  // exp(DIR 2 pi i t / N), 0 <= t < N
        const bool neg = t >= N / 2;
        cplx w = ldg_c(twf + (neg ? t - N / 2 : t));
        if (DIR > 0) w.y = -w.y;
        return neg ? mk(-w.x, -w.y) : w;
    }

    template <class Ctx>
    SW_HD void issue(const Ctx& ctx, cplx* in, uint64_t* bar, int64_t line) const {
        k2_issue_row<Maps, false, HALF>(ctx, op, swizzled, box_chunks, in, bar, line);
    }

    // group barrier; after the first-pass loads of the group's LAST sub-transform the staging
    // buffer is dead for this group: the second group to get there starts the next row's copy
    template <class Ctx>
    struct GroupSync {
        const Ctx& ctx;
        const ExtractColumnsTma4Kernel& k;
        int grp, tg;
        cplx* in;
        uint64_t* bar;
        int* done;  // shared counter
        int64_t next_line;
        bool pending;
        SW_HD void operator()() {
            ctx.group_sync(1 + grp, TG);
            if (pending) {
                pending = false;
                if (tg == 0) {
#if defined(__CUDA_ARCH__)
                    const int prev = atomicAdd(done, 1);
#else
                    const int prev = (*done)++;
#endif
                    if ((prev & 1) == 1 && next_line < k.op.g.n_lines)
                        k.issue(ctx, in, bar, next_line);
                }
            }
        }
    };

    template <class Ctx>
    SW_HD void operator()(Ctx& ctx) const {
        cplx* in = (cplx*)ctx.smem;
        double* xb = (double*)(in + in_cap);
        uint64_t* bar = (uint64_t*)(xb + 2 * XBUF);
        int* done = (int*)(bar + 1);
        const int grp = ctx.tid / TG;
        const int tg = ctx.tid % TG;
        double* sm = xb + (size_t)grp * XBUF;
        cplx* stash = scratch + (size_t)ctx.bid * N;
        const int n = op.n;
        if (ctx.tid == 0) {
            ctx.tx_init(bar);
            *done = 0;
            if ((int64_t)ctx.bid < op.g.n_lines) issue(ctx, in, bar, ctx.bid);
        }
        ctx.sync();
        uint32_t parity = 0;
        for (int64_t line = ctx.bid; line < op.g.n_lines; line += ctx.nblocks) {
            const int f = (int)(line / op.lines_per);
            const int l = (int)(line - (int64_t)f * op.lines_per);
            const ColumnFacet& F = op.fac[f];
            const int shift_in = F.shift_in, fs = F.fs;
            const double* fb = op.fb ? op.fb + F.fb_off : nullptr;
            cplx* o = F.out + (int64_t)l * F.out_ls;
            const double scale = op.scale;
            const bool swz = swizzled != 0;
            bool cj = false;
            if constexpr (HALF) half_row(wrap_add(op.rm_base, wrap_sub(l, op.rm_s_m, op.lines_per), n), n, cj);
            auto sample = [&](int q) {
                int k = wrap_add(q, shift_in, n);
                if (k >= fs) return mk(0.0, 0.0);
                const int ks = swz ? ((k & ~7) | ((k ^ (k >> 3)) & 7)) : k;
                if constexpr (HALF) {
                    const cplx x = fb ? cscale(in[ks], ldg_d(fb + k)) : in[ks];
                    return cj ? cconj(x) : x;
                } else {
                    return fb ? cscale(in[ks], ldg_d(fb + k)) : in[ks];
                }
            };
            ctx.tx_wait(bar, parity);
            parity ^= 1;
            GroupSync<Ctx> gs{ctx, *this, grp, tg, in, bar, done, line + ctx.nblocks, false};
#pragma unroll 1
            for (int qi = 0; qi < 2; ++qi) {
                const int q4 = 2 * grp + qi;
                cplx* sq = stash + (size_t)q4 * Q;
                auto ld = [&](int j) { return sample(4 * j + q4); };
                // t_q[k] = w^(q k) E_q[k]; w^(q k) for the thread's outputs k = j0 + it * T +
                // r * NS by recurrence: one table load, then multiplications by w^(q T), w^(q NS)
                typedef LastPass<Q> LP;
                const cplx step_it = root((q4 * TG) % N), step_r = root((q4 * LP::NS) % N);
                cplx w_it = mk(1.0, 0.0), w = mk(1.0, 0.0);
                auto st = [&](int k, cplx v, int it, int r) {
                    if (r == 0) {
                        w_it = it == 0 ? root((q4 * k) % N) : cmul(w_it, step_it);
                        w = w_it;
                    } else {
                        w = cmul(w, step_r);
                    }
                    sq[k] = q4 ? cmul(v, w) : v;
                };
                gs.pending = (qi == 1);
                line_fft<Q, DIR>(tg, sm, tw, ld, st, gs);
                gs();  // the group's exchange buffer is reused by its next sub-transform
            }
            ctx.sync();  // all four t_q are in the scratch
            // (four k per trip: sixteen independent scratch loads in flight per thread)
            for (int k0 = ctx.tid; k0 < Q; k0 += 4 * THREADS) {
                cplx t[4][4];
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int q4 = 0; q4 < 4; ++q4) {
                        const int k = k0 + i * THREADS;
                        t[i][q4] = k < Q ? stash[(size_t)q4 * Q + k] : mk(0.0, 0.0);
                    }
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int k = k0 + i * THREADS;
                    if (k >= Q) break;
                    Radix<4, DIR>::run(t[i]);
#pragma unroll
                    for (int s4 = 0; s4 < 4; ++s4) {
                        int pc = wrap_add(k + Q * s4, n / 2, n);
                        st_stream(o + pc, cscale(t[i][s4], scale));
                    }
                }
            }
            ctx.sync();  // scratch and exchange buffers are reused by the next line
        }
    }
};

// ---------------------------------------------------------------------------------------
// yN = 4 Q as above, on a CLUSTER of two CTAs that share every line: no L2 scratch.
//
// The row is staged once for both CTAs by multicast loads.  CTA c runs t_c in group 0 and
// t_(c+2) in group 1, one Q-point transform per group and line; a thread owns the same outputs
// k = tg + TG i (i < 16) in every sub-transform and keeps half of its t_q[k] in registers.  The
// radix-4 butterfly over q (bfly4) pairs q with q + 2 first:
//   P+ = t_0 + t_2,  P- = t_0 - t_2          (CTA 0)
//   R+ = t_1 + t_3,  R- = i (t_1 - t_3)      (CTA 1)
//   X_0 = P+ + R+,  X_2 = P+ - R+            (stored by CTA 0)
//   X_1 = P- + R-,  X_3 = P- - R-            (stored by CTA 1)
// 1. inside the CTA the groups swap the other half of their t_q through their exchange buffers
//    (dead after the last pass's reads): group g then holds both operands for i in [8 g, 8 g + 8)
//    and forms P or R there;
// 2. CTA 0 writes P-, CTA 1 writes R+ into the partner's exchange buffers (distributed shared
//    memory, Q samples each way), and after a cluster barrier each CTA finishes two outputs.
// Same operations in the same order as ExtractColumnsTma4Kernel, so the same bits.  The staging
// buffer is dead once all four groups of the pair have done their first-pass loads: the last of
// them to get there issues the next row (counter in CTA 0).
template <int Q, bool HALF = false>
struct ExtractColumnsClusterKernel {
    static constexpr int DIR = +1;
    static constexpr int CLUSTER = 2;
    static constexpr int TG = FftCfg<Q>::T;
    static constexpr int THREADS = 2 * TG;
    static constexpr int N = 4 * Q;
    static constexpr int XBUF = (FftCfg<Q>::PADDED + 1) & ~1;
    // the half of a group's 16 outputs that changes hands fits its exchange buffer
    static_assert(8 * TG * 2 <= XBUF, "exchange buffer too small for the combine");
    static constexpr size_t smem_bytes(int in_cap) {
        return (size_t)in_cap * sizeof(cplx) + 2 * (size_t)XBUF * sizeof(double) + 32;
    }

    ExtractColumnsOp op;
    const cplx* tw;   // compact table of the Q-point plan
    const cplx* twf;  // exp(-2 pi i t / yN), t < yN / 2
    int in_cap;
    int swizzled;
    int box_chunks;
    struct Maps {
        TensorMap4 in_map[SW_MAX_COLUMN_FACETS];
    };

    SW_HD cplx root(int t) const {  // exp(DIR 2 pi i t / N), 0 <= t < N
        const bool neg = t >= N / 2;
        cplx w = ldg_c(twf + (neg ? t - N / 2 : t));
        if (DIR > 0) w.y = -w.y;
        return neg ? mk(-w.x, -w.y) : w;
    }

    template <class Ctx>
    SW_HD void issue(const Ctx& ctx, cplx* in, uint64_t* bar, int64_t line) const {
        k2_issue_row<Maps, true, HALF>(ctx, op, swizzled, box_chunks, in, bar, line);
    }

    template <class Ctx>
    struct GroupSync {
        const Ctx& ctx;
        const ExtractColumnsClusterKernel& k;
        int grp, tg;
        cplx* in;
        uint64_t* bar;
        int* done;  // counter in CTA 0
        int64_t next_line;
        bool pending;
        SW_HD void operator()() {
            ctx.group_sync(1 + grp, TG);
            if (pending) {
                pending = false;
                if (tg == 0 && (ctx.peer_atomic_add(done, 0, 1) & 3) == 3 &&
                    next_line < k.op.g.n_lines)
                    k.issue(ctx, in, bar, next_line);
            }
        }
        SW_HD void pre_store() { ctx.group_sync(1 + grp, TG); }
    };

    template <class Ctx>
    SW_HD void operator()(Ctx& ctx) const {
        cplx* in = (cplx*)ctx.smem;
        double* xb = (double*)(in + in_cap);
        uint64_t* bar = (uint64_t*)(xb + 2 * XBUF);
        int* done = (int*)(bar + 1);
        const int rank = ctx.cluster_rank();
        const int cid = ctx.bid / CLUSTER, ncl = ctx.nblocks / CLUSTER;
        const int grp = ctx.tid / TG;
        const int tg = ctx.tid % TG;
        double* sm = xb + (size_t)grp * XBUF;
        cplx* mine = (cplx*)sm;                        // this group's exchange buffer
        cplx* other = (cplx*)(xb + (size_t)(1 - grp) * XBUF);
        constexpr int n = N;  // op.n
        const int q4 = rank + 2 * grp;
        const int lo = 8 * grp;  // the outputs i in [lo, lo + 8) are combined by this group
        if (ctx.tid == 0) {
            ctx.tx_init(bar);
            *done = 0;
        }
        ctx.cluster_sync();  // both barriers initialised before the first multicast
        if (rank == 0 && ctx.tid == 0 && cid < op.g.n_lines) issue(ctx, in, bar, cid);
        uint32_t parity = 0;
        typedef LastPass<Q> LP;
        for (int64_t line = cid; line < op.g.n_lines; line += ncl) {
            const int f = (int)(line / op.lines_per);
            const int l = (int)(line - (int64_t)f * op.lines_per);
            const ColumnFacet& F = op.fac[f];
            const int shift_in = F.shift_in, fs = F.fs;
            const double* fb = op.fb ? op.fb + F.fb_off : nullptr;
            cplx* o = F.out + (int64_t)l * F.out_ls;
            const double scale = op.scale;
            const bool swz = swizzled != 0;
            bool cj = false;
            if constexpr (HALF) half_row(wrap_add(op.rm_base, wrap_sub(l, op.rm_s_m, op.lines_per), n), n, cj);
            auto sample = [&](int q) {
                int k = wrap_add(q, shift_in, n);
                if (k >= fs) return mk(0.0, 0.0);
                const int ks = swz ? ((k & ~7) | ((k ^ (k >> 3)) & 7)) : k;
                if constexpr (HALF) {
                    const cplx x = fb ? cscale(in[ks], ldg_d(fb + k)) : in[ks];
                    return cj ? cconj(x) : x;
                } else {
                    return fb ? cscale(in[ks], ldg_d(fb + k)) : in[ks];
                }
            };
            ctx.tx_wait(bar, parity);
            parity ^= 1;
            GroupSync<Ctx> gs{ctx, *this, grp, tg, in, bar, done, line + ncl, true};
            // t_q[k] of the thread's outputs k = tg + TG i, i = it + ITERS r of the last pass:
            // group 0 combines i < 8 and keeps those, group 1 the others; the other half goes to
            // the group's exchange buffer as soon as the group has done its last exchange reads
            // (GroupSync::pre_store)
            cplx t[8];
            {
                auto ld = [&](int j) { return sample(4 * j + q4); };
                const cplx step_it = root((q4 * TG) % N), step_r = root((q4 * LP::NS) % N);
                cplx w_it = mk(1.0, 0.0), w = mk(1.0, 0.0);
                auto st = [&](int k, cplx v, int it, int r) {
                    if (r == 0) {
                        w_it = it == 0 ? root((q4 * k) % N) : cmul(w_it, step_it);
                        w = w_it;
                    } else {
                        w = cmul(w, step_r);
                    }
                    const int i = it + LP::ITERS * r;  // (output i - 8 comes before i)
                    const cplx tq = q4 ? cmul(v, w) : v;
                    if (i < 8) {
                        t[i] = tq;
                    } else {  // outputs i - 8 and i: keep one, pass the other on
                        const cplx keep = grp ? tq : t[i - 8];
                        mine[(i - 8) * TG + tg] = grp ? t[i - 8] : tq;
                        t[i - 8] = keep;
                    }
                };
                line_fft<Q, DIR>(tg, sm, tw, ld, st, gs);
            }
            ctx.sync();  // both halves are in the exchange buffers
            // (a, b) = (t_rank, t_(rank+2)) at output lo + i; CTA 0: P+ / P-, CTA 1: R+ / R-
            cplx keep[8], send[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const cplx u = other[i * TG + tg];  // the CTA's other q
                const cplx a = grp ? u : t[i], b = grp ? t[i] : u;
                const cplx s = cadd(a, b), d = csub(a, b);
                keep[i] = rank ? mul_i<DIR>(d) : s;  // R- or P+
                send[i] = rank ? s : d;              // R+ to CTA 0, P- to CTA 1
            }
            // trade with the partner CTA once it has read its exchange buffers
            ctx.cluster_sync();
#pragma unroll
            for (int i = 0; i < 8; ++i) ctx.peer_st(mine + i * TG + tg, 1 - rank, send[i]);
            ctx.cluster_sync();
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int k = tg + TG * (lo + i);
                const cplx r = mine[i * TG + tg];  // R+ (CTA 0) or P- (CTA 1)
                // CTA 0: X_0 = P+ + R+, X_2 = P+ - R+;  CTA 1: X_1 = P- + R-, X_3 = P- - R-
                const cplx x_lo = rank ? cadd(r, keep[i]) : cadd(keep[i], r);
                const cplx x_hi = rank ? csub(r, keep[i]) : csub(keep[i], r);
                // (bit operations, which the compiler recomputes instead of keeping sixteen
                // loop-invariant positions in spilled registers)
                st_stream(o + ((k + Q * rank + n / 2) & (n - 1)), cscale(x_lo, scale));
                st_stream(o + ((k + Q * (rank + 2) + n / 2) & (n - 1)), cscale(x_hi, scale));
            }
            ctx.group_sync(1 + grp, TG);  // the group's exchange buffer is reused by its next line
        }
    }
};

// ---------------------------------------------------------------------------------------
// yN = 4 Q, two FULLY independent thread groups: decimation in frequency by two ACROSS the
// groups, decimation in time by two WITHIN a group.
//
//   group g (0: even outputs, 1: odd outputs):   y_g[j] = (z[j] + (-1)^g z[j + 2Q]) w^(g j),
//       j < 2Q, w = exp(+2 pi i / yN);  X[2 k + g] = FFT_2Q(y_g)[k]
//   inside the group:  E0 = FFT_Q(y_g[2 j]),  E1 = FFT_Q(y_g[2 j + 1]),  v = exp(+2 pi i / 2Q)
//       FFT_2Q(y_g)[k] = E0[k] + v^k E1[k],   FFT_2Q(y_g)[k + Q] = E0[k] - v^k E1[k]
//
// For facets of at most yN/2 samples only one of z[j], z[j + 2Q] is non-zero: both groups
// transform the SAME staged row, group 1 with a twiddle at load time (by recurrence).  Unlike
// the 4 x Q form above there is no CTA-wide combine phase, no CTA barrier inside a line and
// half the scratch traffic (each group parks only its own E0): the groups meet only at the
// staging buffer (mbarrier wait at the top of a line, the second group past its last
// first-pass load refills it).  The price: every group stores 16-byte samples at a 32-byte
// stride (the other group fills the gaps; the sectors merge in L2).  Kept selectable
// (sg_variant 15; tools/quick_k2.py times it against the other forms).
// BOTH: facets longer than yN/2 exist, z[j] and z[j + 2Q] may both be non-zero (two reads per
// sample; the common fs <= yN/2 case reads one).
template <int Q, bool BOTH>
struct ExtractColumnsTmaDifKernel {
    static constexpr int DIR = +1;
    static constexpr int TG = FftCfg<Q>::T;
    static constexpr int THREADS = 2 * TG;
    static constexpr int H = 2 * Q;
    static constexpr int N = 4 * Q;
    static constexpr int XBUF = (FftCfg<Q>::PADDED + 1) & ~1;
    static constexpr size_t smem_bytes(int in_cap) {
        return (size_t)in_cap * sizeof(cplx) + 2 * (size_t)XBUF * sizeof(double) + 32;
    }

    ExtractColumnsOp op;
    const cplx* tw;   // compact table of the Q-point plan
    const cplx* twf;  // exp(-2 pi i t / yN), t < yN / 2
    cplx* scratch;    // gridDim.x * 2 Q samples (E0 of both groups)
    int in_cap;
    int swizzled;
    int box_chunks;
    struct Maps {
        TensorMap4 in_map[SW_MAX_COLUMN_FACETS];
    };

    SW_HD cplx root(int t) const {  // exp(DIR 2 pi i t / N), 0 <= t < N
        const bool neg = t >= N / 2;
        cplx w = ldg_c(twf + (neg ? t - N / 2 : t));
        if (DIR > 0) w.y = -w.y;
        return neg ? mk(-w.x, -w.y) : w;
    }

    template <class Ctx>
    SW_HD void issue(const Ctx& ctx, cplx* in, uint64_t* bar, int64_t line) const {
        k2_issue_row<Maps>(ctx, op, swizzled, box_chunks, in, bar, line);
    }

    template <class Ctx>
    struct GroupSync {
        const Ctx& ctx;
        const ExtractColumnsTmaDifKernel& k;
        int grp, tg;
        cplx* in;
        uint64_t* bar;
        int* done;
        int64_t next_line;
        bool pending;
        SW_HD void operator()() {
            ctx.group_sync(1 + grp, TG);
            if (pending) {
                pending = false;
                if (tg == 0) {
#if defined(__CUDA_ARCH__)
                    const int prev = atomicAdd(done, 1);
#else
                    const int prev = (*done)++;
#endif
                    if ((prev & 1) == 1 && next_line < k.op.g.n_lines)
                        k.issue(ctx, in, bar, next_line);
                }
            }
        }
    };

    template <class Ctx>
    SW_HD void operator()(Ctx& ctx) const {
        cplx* in = (cplx*)ctx.smem;
        double* xb = (double*)(in + in_cap);
        uint64_t* bar = (uint64_t*)(xb + 2 * XBUF);
        int* done = (int*)(bar + 1);
        const int grp = ctx.tid / TG;
        const int tg = ctx.tid % TG;
        double* sm = xb + (size_t)grp * XBUF;
        cplx* stash = scratch + ((size_t)ctx.bid * 2 + grp) * Q;
        const int n = op.n;
        if (ctx.tid == 0) {
            ctx.tx_init(bar);
            *done = 0;
            if ((int64_t)ctx.bid < op.g.n_lines) issue(ctx, in, bar, ctx.bid);
        }
        ctx.sync();
        uint32_t parity = 0;
        typedef LastPass<Q> LP;
        for (int64_t line = ctx.bid; line < op.g.n_lines; line += ctx.nblocks) {
            const int f = (int)(line / op.lines_per);
            const int l = (int)(line - (int64_t)f * op.lines_per);
            const ColumnFacet& F = op.fac[f];
            const int shift_in = F.shift_in, fs = F.fs;
            const double* fb = op.fb ? op.fb + F.fb_off : nullptr;
            cplx* o = F.out + (int64_t)l * F.out_ls;
            const double scale = op.scale;
            const bool swz = swizzled != 0;
            auto sample = [&](int q) {  // natural-order sample q of the padded, rotated row
                int k = wrap_add(q, shift_in, n);
                if (k >= fs) return mk(0.0, 0.0);
                const int ks = swz ? ((k & ~7) | ((k ^ (k >> 3)) & 7)) : k;
                return fb ? cscale(in[ks], ldg_d(fb + k)) : in[ks];
            };
            ctx.tx_wait(bar, parity);
            parity ^= 1;
            GroupSync<Ctx> gs{ctx, *this, grp, tg, in, bar, done, line + ctx.nblocks, false};
            // sub-transform `half` of the group's sequence: y_g[2 j + half], j = tg + r * NB
            {
                constexpr int half = 0;
                // group 1's load twiddle w^(2 j + half): four table loads per thread (r = 0, 4, 8,
                // 12), the samples in between by three multiplications with the step w^(2 NB)
                const cplx w_step = root((2 * (Q / 16)) % N);
                cplx w_ld = mk(1.0, 0.0);
                int calls = 0;
                auto ld = [&](int j) {
                    const int q = 2 * j + half;
                    cplx y;
                    if constexpr (BOTH) {
                        cplx a = sample(q), b = sample(q + H);
                        y = grp ? csub(a, b) : cadd(a, b);
                    } else {
                        // fs <= 2Q: at most one of the two is inside the facet
                        int k = wrap_add(q, shift_in, n);
                        const bool second = k >= fs;
                        if (second) k = wrap_add(k, H, n);
                        if (k >= fs) {
                            y = mk(0.0, 0.0);
                        } else {
                            const int ks = swz ? ((k & ~7) | ((k ^ (k >> 3)) & 7)) : k;
                            y = fb ? cscale(in[ks], ldg_d(fb + k)) : in[ks];
                            if (second && grp) y = mk(-y.x, -y.y);
                        }
                    }
                    if (grp) {
                        w_ld = (calls & 3) == 0 ? root(q % N) : cmul(w_ld, w_step);
                        y = cmul(y, w_ld);
                    }
                    ++calls;
                    return y;
                };
                auto st = [&](int k, cplx v) { stash[k] = v; };
                line_fft<Q, DIR>(tg, sm, tw, ld, st, gs);
                gs();  // the group's exchange buffer is reused by its second sub-transform
            }
            {
                constexpr int half = 1;
                // group 1's load twiddle w^(2 j + half): four table loads per thread (r = 0, 4, 8,
                // 12), the samples in between by three multiplications with the step w^(2 NB)
                const cplx w_step = root((2 * (Q / 16)) % N);
                cplx w_ld = mk(1.0, 0.0);
                int calls = 0;
                auto ld = [&](int j) {
                    const int q = 2 * j + half;
                    cplx y;
                    if constexpr (BOTH) {
                        cplx a = sample(q), b = sample(q + H);
                        y = grp ? csub(a, b) : cadd(a, b);
                    } else {
                        // fs <= 2Q: at most one of the two is inside the facet
                        int k = wrap_add(q, shift_in, n);
                        const bool second = k >= fs;
                        if (second) k = wrap_add(k, H, n);
                        if (k >= fs) {
                            y = mk(0.0, 0.0);
                        } else {
                            const int ks = swz ? ((k & ~7) | ((k ^ (k >> 3)) & 7)) : k;
                            y = fb ? cscale(in[ks], ldg_d(fb + k)) : in[ks];
                            if (second && grp) y = mk(-y.x, -y.y);
                        }
                    }
                    if (grp) {
                        w_ld = (calls & 3) == 0 ? root(q % N) : cmul(w_ld, w_step);
                        y = cmul(y, w_ld);
                    }
                    ++calls;
                    return y;
                };
                // v^k = exp(DIR 2 pi i k / 2Q) = root(2 k) by recurrence over the outputs
                const cplx v_it = root((2 * TG) % N), v_r = root((2 * LP::NS) % N);
                cplx w_it = mk(1.0, 0.0), w = mk(1.0, 0.0);
                auto st = [&](int k, cplx od, int it, int r) {
                    if (r == 0) {
                        w_it = it == 0 ? root((2 * k) % N) : cmul(w_it, v_it);
                        w = w_it;
                    } else {
                        w = cmul(w, v_r);
                    }
                    const cplx e = stash[k];
                    const cplx wo = cmul(od, w);
                    // FFT_2Q(y_g)[k] -> X[2 k + g],  FFT_2Q(y_g)[k + Q] -> X[2 (k + Q) + g]
                    int pc = wrap_add(2 * k + grp, n / 2, n);
                    st_stream(o + pc, cscale(cadd(e, wo), scale));
                    pc = wrap_add(2 * (k + Q) + grp, n / 2, n);
                    st_stream(o + pc, cscale(csub(e, wo), scale));
                };
                gs.pending = true;
                line_fft<Q, DIR>(tg, sm, tw, ld, st, gs);
                gs();  // exchange buffer / scratch line are reused by the group's next line
            }
        }
    }
};

}  // namespace swiftly
