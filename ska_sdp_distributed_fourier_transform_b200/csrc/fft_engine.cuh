// SwiFTly -- in-CTA complex128 FFT engine.
//
// One "line" (a 1-D transform of N complex128 samples, N a power of two,
// 16 <= N <= 8192) is transformed by T = N/16 threads with the Stockham
// autosort algorithm: radix-16 passes (and one final radix-2/4/8 pass when
// log2 N is not a multiple of 4).  Every thread keeps its 16 samples in registers
// for the whole transform; between passes the samples change owner through a
// shared-memory exchange buffer of N (+1/16 padding) DOUBLES: real parts first,
// then imaginary parts through the same buffer.  The FIRST pass reads its input
// through a caller-supplied loader functor (global memory gather: window multiply,
// zero padding and cyclic shifts are index arithmetic there) and the LAST pass
// hands its output to a storer functor (scatter / accumulate / window multiply),
// so a line makes exactly one trip HBM -> registers -> HBM.
//
// Twiddles: a pass with sub-transform size Ns and radix R multiplies input r of
// butterfly j by w^r, w = exp(-2 pi i (j mod Ns) / (Ns R)).  Only w is loaded -- one
// coalesced 16-byte load per butterfly from a compact per-pass table (Ns entries,
// laid out pass after pass, < 4.4 K entries per FFT size) -- and the powers w^2..w^15
// are formed in registers with 14 complex multiplies (product depth <= 3).  Loading
// all 15 factors from a W_N^t table instead costs up to 16 L1 wavefronts per load
// instruction and made the kernels LSU-bound; the FP64 pipe has
// the headroom.  The inverse direction conjugates on the fly; the first pass needs
// no twiddles at all.
//
// Lines of 2N samples that do not fit shared memory (yN = 16384) are done as
// two N-point transforms after one decimation-in-frequency radix-2 step that
// is folded into the loader (split2_*), see kernels.cuh.
#pragma once

#include <type_traits>
#include <utility>

#include "common.cuh"

namespace swiftly {

// A Sync object is a callable CTA (or thread-group) barrier.  It may additionally offer
// acquire() / release(): hooks around the shared-memory exchange of every pass.  The
// ping-pong kernels (subgrid_pp.cuh) use them to hand an "LSU token" back and forth between
// two thread groups of one CTA, so that one group moves data through shared memory (LSU
// bound) exactly while the other one runs its butterflies (FP64 bound).  acquire() must be
// at least as strong as the barrier itself (everybody of the transform has arrived).
// A storer functor is called as st(k, value).  It may instead take st(k, value, it, r) -- the
// butterfly (it) and output (r) numbers of the last pass, compile-time constants after
// unrolling, with k = j0 + it * T + r * NS -- which lets it derive per-output factors (e.g. the
// twiddles of a split transform's combine step) by recurrence instead of loading each one.
template <class St>
SW_HD void call_store(St& st, int k, cplx v, int it, int r) {
    if constexpr (std::is_invocable_v<St&, int, cplx, int, int>)
        st(k, v, it, r);
    else
        st(k, v);
}

// geometry of the LAST pass of the N-point plan: radix, sub-transform size, butterflies per thread
template <int N>
struct LastPass {
    static constexpr int passes_radix16 = (N >= 65536) ? 4 : (N >= 4096) ? 3 : (N >= 256) ? 2 : 1;
    static constexpr int pow16 = passes_radix16 == 4 ? 65536 : passes_radix16 == 3 ? 4096
                                 : passes_radix16 == 2 ? 256 : 16;
    // N = 16^a * R with R in {1 (then the last pass is radix 16), 2, 4, 8}
    static constexpr int R = (N == pow16) ? 16 : N / pow16;
    static constexpr int NS = N / R;
    static constexpr int ITERS = 16 / R;
};

// optional hook: sync.pre_store() right before the stores of the LAST pass (e.g. a barrier that
// orders them after another transform's stores to the same destination)
template <class S, class = void>
struct HasPreStore : std::false_type {};
template <class S>
struct HasPreStore<S, std::void_t<decltype(std::declval<S&>().pre_store())>> : std::true_type {};

template <class S, class = void>
struct HasPhaseHooks : std::false_type {};
template <class S>
struct HasPhaseHooks<S, std::void_t<decltype(std::declval<S&>().acquire())>> : std::true_type {};

// ---------------------------------------------------------------- radix kernels
// v * (c + i * DIR * s)
template <int DIR>
SW_HD cplx mul_w(cplx v, double c, double s) {
    return DIR < 0 ? mk(v.x * c + v.y * s, v.y * c - v.x * s)
                   : mk(v.x * c - v.y * s, v.y * c + v.x * s);
}

template <int DIR>
SW_HD void bfly2(cplx& a, cplx& b) {
    cplx t = a;
    a = cadd(t, b);
    b = csub(t, b);
}

// in-place 4-point DFT, natural order
template <int DIR>
SW_HD void bfly4(cplx& a0, cplx& a1, cplx& a2, cplx& a3) {
    cplx t0 = cadd(a0, a2), t1 = csub(a0, a2);
    cplx t2 = cadd(a1, a3), t3 = mul_i<DIR>(csub(a1, a3));
    a0 = cadd(t0, t2);
    a1 = cadd(t1, t3);
    a2 = csub(t0, t2);
    a3 = csub(t1, t3);
}

#define SW_SQRT1_2 0.70710678118654752440
#define SW_COS_PI_8 0.92387953251128673848
#define SW_SIN_PI_8 0.38268343236508978178

template <int R, int DIR>
struct Radix;

template <int DIR>
struct Radix<2, DIR> {
    static SW_HD void run(cplx* v) { bfly2<DIR>(v[0], v[1]); }
};

template <int DIR>
struct Radix<4, DIR> {
    static SW_HD void run(cplx* v) { bfly4<DIR>(v[0], v[1], v[2], v[3]); }
};

template <int DIR>
struct Radix<8, DIR> {
    // j = c + 2a, k = a' + 4c'
    static SW_HD void run(cplx* v) {
        bfly4<DIR>(v[0], v[2], v[4], v[6]);
        bfly4<DIR>(v[1], v[3], v[5], v[7]);
        v[3] = mul_w<DIR>(v[3], SW_SQRT1_2, SW_SQRT1_2);
        v[5] = mul_i<DIR>(v[5]);
        v[7] = mul_w<DIR>(v[7], -SW_SQRT1_2, SW_SQRT1_2);
        cplx x0 = cadd(v[0], v[1]), x4 = csub(v[0], v[1]);
        cplx x1 = cadd(v[2], v[3]), x5 = csub(v[2], v[3]);
        cplx x2 = cadd(v[4], v[5]), x6 = csub(v[4], v[5]);
        cplx x3 = cadd(v[6], v[7]), x7 = csub(v[6], v[7]);
        v[0] = x0; v[1] = x1; v[2] = x2; v[3] = x3;
        v[4] = x4; v[5] = x5; v[6] = x6; v[7] = x7;
    }
};

template <int DIR>
struct Radix<16, DIR> {
    // j = c + 4a, k = a' + 4c'
    static SW_HD void run(cplx* v) {
        bfly4<DIR>(v[0], v[4], v[8], v[12]);
        bfly4<DIR>(v[1], v[5], v[9], v[13]);
        bfly4<DIR>(v[2], v[6], v[10], v[14]);
        bfly4<DIR>(v[3], v[7], v[11], v[15]);
        // v[c + 4a'] *= W16^(c a')
        v[5] = mul_w<DIR>(v[5], SW_COS_PI_8, SW_SIN_PI_8);     // 1
        v[9] = mul_w<DIR>(v[9], SW_SQRT1_2, SW_SQRT1_2);       // 2
        v[13] = mul_w<DIR>(v[13], SW_SIN_PI_8, SW_COS_PI_8);   // 3
        v[6] = mul_w<DIR>(v[6], SW_SQRT1_2, SW_SQRT1_2);       // 2
        v[10] = mul_i<DIR>(v[10]);                             // 4
        v[14] = mul_w<DIR>(v[14], -SW_SQRT1_2, SW_SQRT1_2);    // 6
        v[7] = mul_w<DIR>(v[7], SW_SIN_PI_8, SW_COS_PI_8);     // 3
        v[11] = mul_w<DIR>(v[11], -SW_SQRT1_2, SW_SQRT1_2);    // 6
        v[15] = mul_w<DIR>(v[15], -SW_COS_PI_8, -SW_SIN_PI_8); // 9
        bfly4<DIR>(v[0], v[1], v[2], v[3]);
        bfly4<DIR>(v[4], v[5], v[6], v[7]);
        bfly4<DIR>(v[8], v[9], v[10], v[11]);
        bfly4<DIR>(v[12], v[13], v[14], v[15]);
        // now v[c' + 4a'] = X[a' + 4c']: transpose the 4x4
        cplx t;
        t = v[1]; v[1] = v[4]; v[4] = t;
        t = v[2]; v[2] = v[8]; v[8] = t;
        t = v[3]; v[3] = v[12]; v[12] = t;
        t = v[6]; v[6] = v[9]; v[9] = t;
        t = v[7]; v[7] = v[13]; v[13] = t;
        t = v[11]; v[11] = v[14]; v[14] = t;
    }
};

// ---------------------------------------------------------------- plan
template <int N>
struct FftCfg {
    static_assert(N >= 16 && (N & (N - 1)) == 0, "FFT size must be a power of two >= 16");
    static constexpr int T = N / 16;           // threads per line
    static constexpr int PADDED = N + N / 16;  // shared memory DOUBLES per line
};

// exchange buffer index: one pad slot per 16 keeps the stride-16 scatter of the first
// pass conflict free (17 j + r hits 16 distinct 8-byte bank pairs per half warp)
SW_HD int sm_phys(int a) { return a + (a >> 4); }

template <int N, int NS>
struct PassRadix {
    static constexpr int R = (N / NS >= 16) ? 16 : (N / NS);
};

// offset of the pass with sub-transform size NS (16, 256 or 4096) in the compact table
template <int NS>
struct TwOffset {
    static constexpr int V = TwOffset<NS / 16>::V + NS / 16;
};
template <>
struct TwOffset<16> {
    static constexpr int V = 0;
};
template <>
struct TwOffset<1> {
    static constexpr int V = 0;
};

SW_HD cplx csqr(cplx a) { return mk(a.x * a.x - a.y * a.y, (a.x + a.x) * a.y); }

// v[r] *= w^r, r = 1..R-1
template <int R>
struct TwiddlePowers;
template <>
struct TwiddlePowers<2> {
    static SW_HD void apply(cplx* v, cplx w1) { v[1] = cmul(v[1], w1); }
};
template <>
struct TwiddlePowers<4> {
    static SW_HD void apply(cplx* v, cplx w1) {
        cplx w2 = csqr(w1);
        v[1] = cmul(v[1], w1);
        v[2] = cmul(v[2], w2);
        v[3] = cmul(v[3], cmul(w2, w1));
    }
};
template <>
struct TwiddlePowers<8> {
    static SW_HD void apply(cplx* v, cplx w1) {
        cplx w2 = csqr(w1), w3 = cmul(w2, w1), w4 = csqr(w2);
        v[1] = cmul(v[1], w1);
        v[2] = cmul(v[2], w2);
        v[3] = cmul(v[3], w3);
        v[4] = cmul(v[4], w4);
        v[5] = cmul(v[5], cmul(w4, w1));
        v[6] = cmul(v[6], cmul(w4, w2));
        v[7] = cmul(v[7], cmul(w4, w3));
    }
};
template <>
struct TwiddlePowers<16> {
    static SW_HD void apply(cplx* v, cplx w1) {
        cplx w2 = csqr(w1), w3 = cmul(w2, w1), w4 = csqr(w2), w8 = csqr(w4), w12 = cmul(w8, w4);
        v[1] = cmul(v[1], w1);
        v[2] = cmul(v[2], w2);
        v[3] = cmul(v[3], w3);
        v[4] = cmul(v[4], w4);
        v[5] = cmul(v[5], cmul(w4, w1));
        v[6] = cmul(v[6], cmul(w4, w2));
        v[7] = cmul(v[7], cmul(w4, w3));
        v[8] = cmul(v[8], w8);
        v[9] = cmul(v[9], cmul(w8, w1));
        v[10] = cmul(v[10], cmul(w8, w2));
        v[11] = cmul(v[11], cmul(w8, w3));
        v[12] = cmul(v[12], w12);
        v[13] = cmul(v[13], cmul(w12, w1));
        v[14] = cmul(v[14], cmul(w12, w2));
        v[15] = cmul(v[15], cmul(w12, w3));
    }
};

// Passes from sub-transform size NS (> 1) to N.  On entry v[it * RP + r] holds the OUTPUT
// of the previous pass (radix RP, sub-transform size NS / RP) in registers: output r of
// butterfly j = lt + it * T, which belongs at exchange index (j / NSP) * NS + j % NSP + r * NSP.
// The exchange through shared memory moves real parts, then imaginary parts, through ONE
// buffer of N (+ padding) doubles -- half the footprint of a complex exchange, which is what
// lets two CTAs of the big kernels share an SM; every thread keeps its 16 samples in
// registers throughout.
template <int N, int NS, int RP, int DIR, class St, class Sync>
SW_HD void stockham_tail(int lt, double* sm, const cplx* tw, cplx* v, St& st, Sync& sync) {
    constexpr int T = FftCfg<N>::T;
    constexpr int NSP = NS / RP;
    constexpr int ITP = 16 / RP;
    constexpr int R = PassRadix<N, NS>::R;
    constexpr int NB = N / R;
    constexpr int ITERS = 16 / R;
    constexpr bool LAST = (NS * R == N);
    constexpr bool HOOKS = HasPhaseHooks<Sync>::value;
    double nx[16];
    if constexpr (HOOKS) sync.acquire();
#pragma unroll
    for (int it = 0; it < ITP; ++it) {
        const int j = lt + it * T;
        const int base = (j / NSP) * NS + (j & (NSP - 1));
#pragma unroll
        for (int r = 0; r < RP; ++r) sm[sm_phys(base + r * NSP)] = v[it * RP + r].x;
    }
    sync();
#pragma unroll
    for (int it = 0; it < ITERS; ++it) {
        const int j = lt + it * T;
#pragma unroll
        for (int r = 0; r < R; ++r) nx[it * R + r] = sm[sm_phys(j + r * NB)];
    }
    sync();
#pragma unroll
    for (int it = 0; it < ITP; ++it) {
        const int j = lt + it * T;
        const int base = (j / NSP) * NS + (j & (NSP - 1));
#pragma unroll
        for (int r = 0; r < RP; ++r) sm[sm_phys(base + r * NSP)] = v[it * RP + r].y;
    }
    sync();
#pragma unroll
    for (int it = 0; it < ITERS; ++it) {
        const int j = lt + it * T;
#pragma unroll
        for (int r = 0; r < R; ++r) v[it * R + r] = mk(nx[it * R + r], sm[sm_phys(j + r * NB)]);
    }
    if constexpr (HOOKS) sync.release();
    // twiddle + butterflies of this pass
#pragma unroll
    for (int it = 0; it < ITERS; ++it) {
        const int j = lt + it * T;
        const int k = j & (NS - 1);
        cplx w1 = ldg_c(tw + TwOffset<NS>::V + k);
        if (DIR > 0) w1.y = -w1.y;
        TwiddlePowers<R>::apply(v + it * R, w1);
        Radix<R, DIR>::run(v + it * R);
    }
    if constexpr (LAST) {
        if constexpr (HasPreStore<Sync>::value) sync.pre_store();
#pragma unroll
        for (int it = 0; it < ITERS; ++it) {
            const int j = lt + it * T;
            const int base = (j / NS) * (NS * R) + (j & (NS - 1));
#pragma unroll
            for (int r = 0; r < R; ++r) call_store(st, base + r * NS, v[it * R + r], it, r);
        }
    } else {
        // everybody has read the imaginary parts before the buffer is rewritten (with hooks
        // the acquire() of the next pass is that barrier)
        if constexpr (!HOOKS) sync();
        stockham_tail<N, NS * R, R, DIR>(lt, sm, tw, v, st, sync);
    }
}

// Same passes with a COMPLEX exchange buffer (N + N/16 cplx): one trip (16-byte accesses)
// and two barriers per pass instead of two trips and four barriers; twice the footprint.
// 16-byte accesses are served per quarter warp; the pad per 16 keeps the stride-16 scatter
// on 8 distinct 16-byte bank groups.
template <int N, int NS, int RP, int DIR, class St, class Sync>
SW_HD void stockham_tail_cx(int lt, cplx* sm, const cplx* tw, cplx* v, St& st, Sync& sync) {
    constexpr int T = FftCfg<N>::T;
    constexpr int NSP = NS / RP;
    constexpr int ITP = 16 / RP;
    constexpr int R = PassRadix<N, NS>::R;
    constexpr int NB = N / R;
    constexpr int ITERS = 16 / R;
    constexpr bool LAST = (NS * R == N);
    constexpr bool HOOKS = HasPhaseHooks<Sync>::value;
    if constexpr (HOOKS) sync.acquire();
#pragma unroll
    for (int it = 0; it < ITP; ++it) {
        const int j = lt + it * T;
        const int base = (j / NSP) * NS + (j & (NSP - 1));
#pragma unroll
        for (int r = 0; r < RP; ++r) sm[sm_phys(base + r * NSP)] = v[it * RP + r];
    }
    sync();
#pragma unroll
    for (int it = 0; it < ITERS; ++it) {
        const int j = lt + it * T;
#pragma unroll
        for (int r = 0; r < R; ++r) v[it * R + r] = sm[sm_phys(j + r * NB)];
    }
    if constexpr (HOOKS) sync.release();
#pragma unroll
    for (int it = 0; it < ITERS; ++it) {
        const int j = lt + it * T;
        const int k = j & (NS - 1);
        cplx w1 = ldg_c(tw + TwOffset<NS>::V + k);
        if (DIR > 0) w1.y = -w1.y;
        TwiddlePowers<R>::apply(v + it * R, w1);
        Radix<R, DIR>::run(v + it * R);
    }
    if constexpr (LAST) {
        if constexpr (HasPreStore<Sync>::value) sync.pre_store();
#pragma unroll
        for (int it = 0; it < ITERS; ++it) {
            const int j = lt + it * T;
            const int base = (j / NS) * (NS * R) + (j & (NS - 1));
#pragma unroll
            for (int r = 0; r < R; ++r) call_store(st, base + r * NS, v[it * R + r], it, r);
        }
    } else {
        if constexpr (!HOOKS) sync();
        stockham_tail_cx<N, NS * R, R, DIR>(lt, sm, tw, v, st, sync);
    }
}

// Full N-point transform of one line.
//   lt  : thread index within the line group, 0 <= lt < T = N/16
//   sm  : this line's exchange buffer, FftCfg<N>::PADDED doubles
//   tw  : compact per-pass twiddle table of size N (see twiddles() in capi.cu)
//   ld(q)    -> cplx   natural-order input sample q
//   st(p, v)          natural-order output sample p
//   sync()            CTA barrier
// The caller guarantees that nobody is still reading `sm` from a previous line (barrier
// before re-use).
template <int N, int DIR, class Ld, class St, class Sync>
SW_HD void line_fft(int lt, double* sm, const cplx* tw, Ld& ld, St& st, Sync& sync) {
    constexpr int T = FftCfg<N>::T;
    constexpr int R = PassRadix<N, 1>::R;  // 16
    constexpr int NB = N / R;
    cplx v[16];
#pragma unroll
    for (int r = 0; r < R; ++r) v[r] = ld(lt + r * NB);
    Radix<R, DIR>::run(v);
    if constexpr (R == N) {
#pragma unroll
        for (int r = 0; r < R; ++r) call_store(st, lt * R + r, v[r], 0, r);  // N == 16: lt == 0
    } else {
        stockham_tail<N, R, R, DIR>(lt, sm, tw, v, st, sync);
    }
    (void)T;
}

}  // namespace swiftly

namespace swiftly {

// line_fft with the complex exchange buffer.  ALIAS: the loader reads from the exchange
// buffer's own memory (an accumulator that turns into the exchange buffer): everybody must
// have loaded before the first exchange writes, which costs one extra barrier.
template <int N, int DIR, bool ALIAS, class Ld, class St, class Sync>
SW_HD void line_fft_cx(int lt, cplx* sm, const cplx* tw, Ld& ld, St& st, Sync& sync) {
    constexpr int R = PassRadix<N, 1>::R;  // 16
    constexpr int NB = N / R;
    static_assert(N > 16, "complex-exchange variant is for multi-pass transforms");
    cplx v[16];
#pragma unroll
    for (int r = 0; r < R; ++r) v[r] = ld(lt + r * NB);
    if constexpr (ALIAS && !HasPhaseHooks<Sync>::value) sync();
    Radix<R, DIR>::run(v);
    stockham_tail_cx<N, R, R, DIR>(lt, sm, tw, v, st, sync);
}

// ---------------------------------------------------------------- mixed-radix lines
// Lengths N = F * P with F in {3, 5, 7} and P a power of two >= 32 (the xM and m of the
// catalogue's non power-of-two geometries: 320, 384, 448 and 160, 192, 224), still with
// T = N / 16 threads per line.  Decimation in time by F, all in shared memory:
//   E_q = FFT_P(z[F j + q]),  q < F      (F concurrent P-point transforms, P / 16 threads each)
//   X[o] = sum_q w^(q o) E_q[o mod P],  w = exp(DIR 2 pi i / N)
// (the split-F decomposition of the line kernels, SplitFKernel in kernels.cuh, with the
// sub-transform outputs kept in the line's work area instead of the L2 scratch).  Every thread
// combines 16 outputs o = lt + i * T: F - 1 complex multiplies each, twiddles from the table
// exp(-2 pi i t / N), t < N, that follows the P-point plan's compact table in `tw`.
// Work area (doubles): F exchange buffers of the P-point transforms, then the F * P outputs E.
template <int N, bool POW2 = (N & (N - 1)) == 0>
struct LineCfg {  // power of two: the Stockham plan of FftCfg
    static constexpr int T = FftCfg<N>::T;
    static constexpr int SCRATCH = FftCfg<N>::PADDED;  // doubles of work area per line
};

constexpr int odd_part(int n) { return n % 2 ? n : odd_part(n / 2); }

// entries of the compact per-pass table of the P-point plan (twiddles() in capi.cu)
constexpr int compact_tw_size(int p) {
    int s = 0;
    for (int ns = 16; ns < p; ns *= 16) s += ns;
    return s ? s : 1;
}

template <int N>
struct LineCfg<N, false> {
    static constexpr int F = odd_part(N);
    static constexpr int P = N / F;
    static_assert(F == 3 || F == 5 || F == 7, "mixed-radix lines: N = F * 2^k, F in {3, 5, 7}");
    static_assert(P >= 32 && P <= 8192, "mixed-radix lines: 32 <= 2^k <= 8192");
    static constexpr int T = N / 16;
    static constexpr int TP = P / 16;                     // threads per P-point transform
    static constexpr int XSTRIDE = FftCfg<P>::PADDED | 1;  // odd: the exchanges hit other banks
    static constexpr int EOFF = (F * XSTRIDE + 1) & ~1;   // E is complex: 16-byte aligned
    static constexpr int SCRATCH = EOFF + 2 * N;
    static constexpr int TW_FULL = compact_tw_size(P);    // offset of exp(-2 pi i t / N) in tw
};

// Mixed-radix line (see LineCfg<N, false>).  Same arguments as line_fft; `sm` holds
// LineCfg<N>::SCRATCH doubles; sync() is a plain barrier over (at least) the line's threads.
// The storer is called as st(o, v) or st(o, v, i, 0) with o = lt + i * T.
template <int N, int DIR, class Ld, class St, class Sync>
SW_HD void line_fft_mixed(int lt, double* sm, const cplx* tw, Ld& ld, St& st, Sync& sync) {
    typedef LineCfg<N> C;
    constexpr int F = C::F, P = C::P;
    static_assert(!HasPhaseHooks<Sync>::value, "mixed-radix lines take a plain barrier");
    const int q = lt / C::TP;
    cplx* e = (cplx*)(sm + C::EOFF);
    {
        auto ldq = [&](int j) { return ld(F * j + q); };
        cplx* eq = e + q * P;
        auto stq = [&](int k, cplx v) { eq[k] = v; };
        line_fft<P, DIR>(lt - q * C::TP, sm + q * C::XSTRIDE, tw, ldq, stq, sync);
    }
    sync();  // every E_q complete
    const cplx* wn = tw + C::TW_FULL;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        const int o = lt + i * C::T;
        const int k = o & (P - 1);
        cplx x = e[k];
        int t = 0;  // q * o mod N
#pragma unroll
        for (int qq = 1; qq < F; ++qq) {
            t += o;
            if (t >= N) t -= N;
            cplx w = ldg_c(wn + t);
            if (DIR > 0) w.y = -w.y;
            x = cadd(x, cmul(e[qq * P + k], w));
        }
        call_store(st, o, x, i, 0);
    }
}

// Number of sync() calls one line_fft_any<N> makes (plain barrier, no phase hooks): 4 per
// Stockham pass after the first radix-16 pass, less one (the last pass stores straight from
// registers), plus one for the combine of a mixed-radix line.  Threads that skip a transform
// whose barrier is CTA-wide call sync() this many times instead (SubgridSplitAxisKernel).
constexpr int ilog2_floor(int n) { return n <= 1 ? 0 : 1 + ilog2_floor(n / 2); }
template <int N, bool POW2 = (N & (N - 1)) == 0>
struct LineBarriers {
    static constexpr int PASSES = (ilog2_floor(N) + 3) / 4 - 1;  // Stockham passes after the first
    static constexpr int V = PASSES > 0 ? 4 * PASSES - 1 : 0;
};
template <int N>
struct LineBarriers<N, false> {
    static constexpr int V = LineBarriers<LineCfg<N>::P>::V + 1;
};

// line_fft for every length the fused subgrid kernels take: the Stockham plan for powers of
// two, the mixed-radix line otherwise (work area: LineCfg<N>::SCRATCH doubles)
template <int N, int DIR, class Ld, class St, class Sync>
SW_HD void line_fft_any(int lt, double* sm, const cplx* tw, Ld& ld, St& st, Sync& sync) {
    if constexpr ((N & (N - 1)) == 0)
        line_fft<N, DIR>(lt, sm, tw, ld, st, sync);
    else
        line_fft_mixed<N, DIR>(lt, sm, tw, ld, st, sync);
}

}  // namespace swiftly
