// SwiFTly -- kernel bodies for the eight SwiFTly primitives.
//
// Every primitive is "a batch of independent 1-D lines": the Python/C caller
// passes a line stride and an element stride (in complex128 elements) for input
// and output, so `axis=0` and `axis=1` of a C-ordered 2-D array, 1-D arrays and
// strided (transposed) views are all the same kernel.  pad / extract / roll /
// fftshift of the reference (core.py, fourier_algorithm.py) are closed-form
// modular index maps inside the loader / storer functors of the FFT engine;
// nothing but the FFT input is read and nothing but the result is written.
//
// Centred transforms: fft_c(x) = fftshift(FFT(ifftshift(x))) -- for even n both
// shifts are a cyclic rotation by n/2, so natural FFT index q' corresponds to
// centred index (q' + n/2) mod n on input and output alike
// (fourier_algorithm.py:96-122).
#pragma once

#include "fft_engine.cuh"

namespace swiftly {

struct Lines {
    const cplx* in;
    cplx* out;
    int64_t in_ls, in_es;    // input line stride / element stride (elements)
    int64_t out_ls, out_es;  // output line stride / element stride
    int64_t n_lines;
};

SW_HD int wrap_add(int a, int b, int n) {  // (a + b) mod n for 0 <= a,b < n
    int r = a + b;
    return r >= n ? r - n : r;
}
SW_HD int wrap_sub(int a, int b, int n) {  // (a - b) mod n for 0 <= a,b < n
    int r = a - b;
    return r < 0 ? r + n : r;
}

// Half rows of a real image (include/swiftly_b200.h, "Half rows"): stored row d, 0 <= d <= n/2,
// holds centred row (n/2 + d) mod n, i.e. natural FFT index d.  Centred row r is stored row
// half_row(r, n, conj), conjugated when `conj` is set (rows n/2 + d and n/2 - d are conjugates).
SW_HD int half_row(int r, int n, bool& conj) {
    const int d = wrap_sub(r, n / 2, n);
    conj = d > n / 2;
    return conj ? n - d : d;
}

// ------------------------------------------------------------------ ops
// prepare_facet (core.py:189-222): out = ifft_c(roll(pad_mid(facet * Fb_c, yN), facet_off))
struct PrepareFacetOp {
    Lines g;
    const double* fb;  // Fb window already offset: fb[k] = Fb_c[k], k < fs
    int n;             // yN
    int fs;            // facet size along the axis
    int shift_in;      // k = (q' + shift_in) mod n  with shift_in = (fs//2 - facet_off) mod n
    double scale;      // 1 / yN
    // optional input row map (fused extract_from_facet along the OTHER axis,
    // api_helper.py:200-210): input line = (rm_base + ((line - rm_s_m) mod rm_m)) mod rm_mod
    int rm_m, rm_s_m, rm_base, rm_mod;
    // optional per-LINE weights applied to the output (the Fb window of the OTHER axis folded
    // into this pass: the fused forward path keeps its prepared facets pre-windowed so that the
    // next kernel, K2, does not have to fetch a window value per sample)
    const double* lw;
    SW_HD cplx load(int64_t line, int q) const {
        int k = wrap_add(q, shift_in, n);
        if (k >= fs) return mk(0.0, 0.0);
        int64_t row = rm_m ? (int64_t)wrap_add(rm_base, wrap_sub((int)line, rm_s_m, rm_m), rm_mod)
                           : line;
        return cscale(ld_stream(g.in + row * g.in_ls + (int64_t)k * g.in_es), ldg_d(fb + k));
    }
    SW_HD void store(int64_t line, int p, cplx v) const {
        int pc = wrap_add(p, n / 2, n);
        const double f = lw ? scale * ldg_d(lw + line) : scale;
        st_stream(g.out + line * g.out_ls + (int64_t)pc * g.out_es, cscale(v, f));
    }
    SW_HD void prefetch(int64_t line, int q) const {
        int k = wrap_add(q, shift_in, n);
        if (k >= fs) return;
        int64_t row = rm_m ? (int64_t)wrap_add(rm_base, wrap_sub((int)line, rm_s_m, rm_m), rm_mod)
                           : line;
        prefetch_l2(g.in + row * g.in_ls + (int64_t)k * g.in_es);
    }
};

// prepare_facet of a REAL facet into half rows: the input samples are doubles (`rin`, strides
// g.in_ls / g.in_es counted in doubles; no row map) and only the outputs at natural index
// p <= n/2 are stored, at row p.  A real sample x enters as (x * Fb, 0 * Fb), the product the
// complex op forms on the promoted sample, so the stored rows are bitwise those of PrepareFacetOp.
struct PrepareFacetRealHalfOp : PrepareFacetOp {
    const double* rin;
    SW_HD cplx load(int64_t line, int q) const {
        int k = wrap_add(q, shift_in, n);
        if (k >= fs) return mk(0.0, 0.0);
        const double f = ldg_d(fb + k);
        return mk(ld_stream_d(rin + line * g.in_ls + (int64_t)k * g.in_es) * f, 0.0 * f);
    }
    SW_HD void store(int64_t line, int p, cplx v) const {
        if (p > n / 2) return;
        const double f = lw ? scale * ldg_d(lw + line) : scale;
        st_stream(g.out + line * g.out_ls + (int64_t)p * g.out_es, cscale(v, f));
    }
    SW_HD void prefetch(int64_t line, int q) const {
        int k = wrap_add(q, shift_in, n);
        if (k < fs) prefetch_l2(rin + line * g.in_ls + (int64_t)k * g.in_es);
    }
};

// prepare_facet along the STRIDED axis (axis 0 of a C-ordered facet) as a two-pass
// ("four-step") transform so that every global access covers a run of adjacent columns:
//   n = n1 * n2,  j = j1 n2 + j2,  k = k1 + n1 k2,  w = exp(+2 pi i / n)
//   pass A (n1-point lines, one per (j2, column)):  T[k1 n2 + j2] = w^(j2 k1) sum_j1 z[j1 n2 + j2] w^(n2 j1 k1)
//   pass B (n2-point lines, one per (k1, column)):  X[k1 + n1 k2] = sum_j2 T[k1 n2 + j2] w^(n1 j2 k2)
// Line id = sub * ncols + column, and the line kernels run with LINE_FASTEST, so a warp touches
// 16 adjacent columns (256 contiguous bytes) of one row per request.  The single-pass kernel
// needs a whole 16384-point line per CTA and therefore one COLUMN per CTA: 16-byte accesses
// at a 128 KiB stride, which amplifies the DRAM writes.
struct PrepareFacetPassAOp {
    Lines g;  // g.in: facet (fs rows, ncols columns, row stride in_es); g.out: scratch T (n rows)
    const double* fb;
    const cplx* twf;  // exp(-2 pi i t / n), t < n/2
    int n, n1, n2, fs, shift_in, ncols;
    const double* lw;  // optional per-column weights (see PrepareFacetOp::lw): the transform is
                       // linear, so the weight of column c is applied to its INPUT samples --
                       // one table value per line instead of one per stored sample
    SW_HD cplx load(int64_t line, int q) const {
        const int j2 = (int)(line / ncols);
        const int c = (int)(line - (int64_t)j2 * ncols);
        int k = wrap_add(q * n2 + j2, shift_in, n);
        if (k >= fs) return mk(0.0, 0.0);
        double f = ldg_d(fb + k);
        if (lw) f *= ldg_d(lw + c);
        return cscale(ld_stream(g.in + (int64_t)k * g.in_es + c), f);
    }
    // The inter-pass twiddles w^(j2 k1) of a thread's outputs k1 = j0 + it * T + r * NS follow
    // by recurrence from three table values that depend on (j2, thread) only: prep() loads them
    // BEFORE the transform, together with the data, instead of one dependent table load per
    // output after it (round 1: a second exposed L2 round trip per line, long-scoreboard 6.4
    // warps per issue at 31 % of the DRAM bandwidth).
    struct Tw {
        cplx base, step_it, step_r;
    };
    SW_HD cplx root(int t) const {  // exp(+2 pi i t / n), 0 <= t < n  (inverse direction)
        const bool neg = t >= n / 2;
        cplx w = ldg_c(twf + (neg ? t - n / 2 : t));
        w.y = -w.y;
        return neg ? mk(-w.x, -w.y) : w;
    }
    SW_HD Tw prep(int64_t line, int j0, int T, int NS) const {
        const int j2 = (int)(line / ncols);
        Tw t;
        t.base = root(j2 * j0);        // all exponents < n1 * n2 = n
        t.step_it = root(j2 * T);
        t.step_r = root((j2 * NS) % n);
        return t;
    }
    SW_HD void store_w(int64_t line, int k1, cplx v, cplx w) const {
        const int j2 = (int)(line / ncols);
        const int c = (int)(line - (int64_t)j2 * ncols);
        g.out[((int64_t)k1 * n2 + j2) * ncols + c] = cmul(v, w);
    }
    SW_HD void store(int64_t line, int k1, cplx v) const {
        const int j2 = (int)(line / ncols);
        store_w(line, k1, v, root(j2 * k1));
    }
};
struct PrepareFacetPassBOp {
    Lines g;  // g.in: scratch T; g.out: prepared facet (n rows, row stride out_es)
    int n, n1, n2, ncols;
    double scale;
    SW_HD cplx load(int64_t line, int q) const {
        const int k1 = (int)(line / ncols);
        const int c = (int)(line - (int64_t)k1 * ncols);
        return g.in[((int64_t)k1 * n2 + q) * ncols + c];
    }
    SW_HD void store(int64_t line, int k2, cplx v) const {
        const int k1 = (int)(line / ncols);
        const int c = (int)(line - (int64_t)k1 * ncols);
        int pc = wrap_add(k1 + n1 * k2, n / 2, n);
        st_stream(g.out + (int64_t)pc * g.out_es + c, cscale(v, scale));
    }
};
// The two passes for a REAL facet into half rows: pass A reads doubles (`rin`, row stride
// g.in_es doubles) as PrepareFacetRealHalfOp does, the scratch T stays full size; pass B stores
// natural index d = k1 + n1 k2 at row d when d <= n/2 and drops the other rows.
struct PrepareFacetPassARealOp : PrepareFacetPassAOp {
    const double* rin;
    SW_HD cplx load(int64_t line, int q) const {
        const int j2 = (int)(line / ncols);
        const int c = (int)(line - (int64_t)j2 * ncols);
        int k = wrap_add(q * n2 + j2, shift_in, n);
        if (k >= fs) return mk(0.0, 0.0);
        double f = ldg_d(fb + k);
        if (lw) f *= ldg_d(lw + c);
        return mk(ld_stream_d(rin + (int64_t)k * g.in_es + c) * f, 0.0 * f);
    }
};
struct PrepareFacetPassBHalfOp : PrepareFacetPassBOp {
    SW_HD void store(int64_t line, int k2, cplx v) const {
        const int k1 = (int)(line / ncols);
        const int c = (int)(line - (int64_t)k1 * ncols);
        const int d = k1 + n1 * k2;
        if (d > n / 2) return;
        st_stream(g.out + (int64_t)d * g.out_es + c, cscale(v, scale));
    }
};

// Several prepare_facet jobs with a row map (extract_column of MANY facets, one launch):
// global line L = f * lines_per + l belongs to facet f; per-facet base pointers / shifts
// come from a table in the kernel parameters.
struct ColumnFacet {
    const cplx* in;   // BF_F of the facet (yN rows of fs samples)
    cplx* out;        // NMBF_BF of the facet (m rows of yN samples)
    int64_t in_ls, out_ls;
    int fs, shift_in, fb_off;
    int pad_;
};
#define SW_MAX_COLUMN_FACETS 64
struct ExtractColumnsOp {
    Lines g;           // only n_lines (= n_facets * lines_per) is used
    ColumnFacet fac[SW_MAX_COLUMN_FACETS];
    const double* fb;  // full Fb table, or null: the rows are already Fb weighted
    int n;             // yN
    int lines_per;     // m
    double scale;      // 1 / yN
    int rm_s_m, rm_base;  // row map: input row = (rm_base + ((l - rm_s_m) mod m)) mod yN
    int rows;  // (host side) rows of every bf_f: yN, or m for row rings (the TMA row maps)
    SW_HD cplx load(int64_t line, int q) const {
        const int f = (int)(line / lines_per);
        const int l = (int)(line - (int64_t)f * lines_per);
        const ColumnFacet& F = fac[f];
        int k = wrap_add(q, F.shift_in, n);
        if (k >= F.fs) return mk(0.0, 0.0);
        int64_t row = wrap_add(rm_base, wrap_sub(l, rm_s_m, lines_per), n);
        cplx x = ld_stream(F.in + row * F.in_ls + k);
        return fb ? cscale(x, ldg_d(fb + F.fb_off + k)) : x;
    }
    SW_HD void store(int64_t line, int p, cplx v) const {
        const int f = (int)(line / lines_per);
        const int l = (int)(line - (int64_t)f * lines_per);
        const ColumnFacet& F = fac[f];
        int pc = wrap_add(p, n / 2, n);
        st_stream(F.out + (int64_t)l * F.out_ls + pc, cscale(v, scale));
    }
    SW_HD void prefetch(int64_t line, int q) const {
        const int f = (int)(line / lines_per);
        const int l = (int)(line - (int64_t)f * lines_per);
        const ColumnFacet& F = fac[f];
        int k = wrap_add(q, F.shift_in, n);
        if (k >= F.fs) return;
        int64_t row = wrap_add(rm_base, wrap_sub(l, rm_s_m, lines_per), n);
        prefetch_l2(F.in + row * F.in_ls + k);
    }
};
// ExtractColumnsOp on half rows (rows = n/2 + 1): window row r is read from stored row
// half_row(r) and conjugated when that says so -- bitwise the load of the full Hermitian rows
struct ExtractColumnsHalfOp : ExtractColumnsOp {
    SW_HD cplx load(int64_t line, int q) const {
        const int f = (int)(line / lines_per);
        const int l = (int)(line - (int64_t)f * lines_per);
        const ColumnFacet& F = fac[f];
        int k = wrap_add(q, F.shift_in, n);
        if (k >= F.fs) return mk(0.0, 0.0);
        bool cj;
        const int64_t row = half_row(wrap_add(rm_base, wrap_sub(l, rm_s_m, lines_per), n), n, cj);
        cplx x = ld_stream(F.in + row * F.in_ls + k);
        if (fb) x = cscale(x, ldg_d(fb + F.fb_off + k));
        return cj ? cconj(x) : x;
    }
    SW_HD void prefetch(int64_t line, int q) const {
        const int f = (int)(line / lines_per);
        const int l = (int)(line - (int64_t)f * lines_per);
        const ColumnFacet& F = fac[f];
        int k = wrap_add(q, F.shift_in, n);
        if (k >= F.fs) return;
        bool cj;
        const int64_t row = half_row(wrap_add(rm_base, wrap_sub(l, rm_s_m, lines_per), n), n, cj);
        prefetch_l2(F.in + row * F.in_ls + k);
    }
};

// ------------------------------------------------------------------ fused backward ops
// One subgrid -> the column accumulators of ALL facets in one launch
// (api_helper.py:115-152 per facet: extract_from_subgrid(axis 1) then accumulate_column =
// add_to_facet(axis 1)).  Global line L = f * lines_per + t: row t of the (m, xM) block that
// extract_from_subgrid(axis 0) produced for facet f's off0; the m-point inverse transform of
// the Fn-weighted window is added at the subgrid's position of facet f's (m, yN) accumulator.
struct BackFacet {
    const cplx* in;  // (m, xM) block of the facet's row group
    cplx* out;       // (m, yN) column accumulator NAF_MNAF of the facet
    int64_t in_ls, out_ls;
    int sf_m, base_x;  // facet_off1 * xM // N mod m ; (xM/2 - m/2 + sf) mod xM
};
struct SubgridToFacetsOp {
    Lines g;  // only n_lines is used
    BackFacet fac[SW_MAX_COLUMN_FACETS];
    const double* fn;
    int m, xM, yN, lines_per;
    int s_m, base_y;  // subgrid_off1 * yN // N mod m ; (yN/2 - m/2 + s) mod yN
    double scale;     // 1 / m
    SW_HD cplx load(int64_t line, int q) const {
        const int f = (int)(line / lines_per);
        const int t = (int)(line - (int64_t)f * lines_per);
        const BackFacet& F = fac[f];
        int tc = wrap_add(q, m / 2, m);
        int u = wrap_sub(tc, F.sf_m, m);
        int pos = wrap_add(F.base_x, u, xM);
        return cscale(ld_stream(F.in + (int64_t)t * F.in_ls + pos), ldg_d(fn + u));
    }
    SW_HD void store(int64_t line, int p, cplx v) const {
        const int f = (int)(line / lines_per);
        const int t = (int)(line - (int64_t)f * lines_per);
        const BackFacet& F = fac[f];
        int pc = wrap_add(p, m / 2, m);
        int w = wrap_add(base_y, wrap_sub(pc, s_m, m), yN);
        cplx* o = F.out + (int64_t)t * F.out_ls + w;
        cplx a = *o;
        *o = mk(a.x + scale * v.x, a.y + scale * v.y);
    }
};

// Fold a finished subgrid column into ALL facets in one launch (api_helper.py:155-179 per
// facet: finish_facet(axis 1), mask, add_to_facet(axis 0)).  Line L = f * lines_per + t: row t
// of facet f's (m, yN) column accumulator; its yN-point forward transform, cut to the facet
// size and weighted with Fb (and the facet mask), is added to row
// (base0 + ((t - s0_m) mod m)) mod yN of the facet's (yN, fs) accumulator.
struct FoldFacet {
    const cplx* in;      // (m, yN) column accumulator
    cplx* out;           // (yN, fs) facet accumulator MNAF_BMNAF
    const double* mask;  // fs doubles or null
    int64_t in_ls, out_ls;
    int fs, start1, fb_off;
    int pad_;
};
struct FoldColumnOp {
    Lines g;  // only n_lines is used
    FoldFacet fac[SW_MAX_COLUMN_FACETS];
    const double* fb;
    int n, lines_per;   // yN, m
    int s0_m, base0;    // subgrid_off0 * yN // N mod m ; (yN/2 - m/2 + s0) mod yN
    SW_HD cplx load(int64_t line, int q) const {
        const int f = (int)(line / lines_per);
        const int t = (int)(line - (int64_t)f * lines_per);
        const FoldFacet& F = fac[f];
        int qc = wrap_add(q, n / 2, n);
        return ld_stream(F.in + (int64_t)t * F.in_ls + qc);
    }
    SW_HD void store(int64_t line, int p, cplx v) const {
        const int f = (int)(line / lines_per);
        const int t = (int)(line - (int64_t)f * lines_per);
        const FoldFacet& F = fac[f];
        int pc = wrap_add(p, n / 2, n);
        int k = wrap_sub(pc, F.start1, n);
        if (k >= F.fs) return;
        double w = ldg_d(fb + F.fb_off + k);
        if (F.mask) w *= ldg_d(F.mask + k);
        int64_t row = wrap_add(base0, wrap_sub(t, s0_m, lines_per), n);
        cplx* o = F.out + row * F.out_ls + k;
        cplx a = *o;
        *o = mk(a.x + w * v.x, a.y + w * v.y);
    }
};
// FoldColumnOp into half-row facet accumulators, for the run of window rows u in
// [u_lo, u_lo + lines_per) (u = (t - s0_m) mod m, t the column accumulator row).  Row
// base0 + u goes to stored row half_row(.): conj(w v) is added where that flags a conjugate,
// w v elsewhere.  The host cuts the window into runs whose rows have distinct targets.  The
// conjugated add rounds the product first (no fused multiply-add), so that one fold into zeroed
// accumulators is bitwise x[d] + conj(x[-d]) of the full-row fold x; the plain add is the
// full-row op's.
struct FoldColumnHalfOp : FoldColumnOp {
    int m, u_lo;
    SW_HD cplx load(int64_t line, int q) const {
        const int f = (int)(line / lines_per);
        const int j = (int)(line - (int64_t)f * lines_per);
        const FoldFacet& F = fac[f];
        const int t = wrap_add(u_lo + j, s0_m, m);
        int qc = wrap_add(q, n / 2, n);
        return ld_stream(F.in + (int64_t)t * F.in_ls + qc);
    }
    SW_HD void store(int64_t line, int p, cplx v) const {
        const int f = (int)(line / lines_per);
        const int j = (int)(line - (int64_t)f * lines_per);
        const FoldFacet& F = fac[f];
        int pc = wrap_add(p, n / 2, n);
        int k = wrap_sub(pc, F.start1, n);
        if (k >= F.fs) return;
        double w = ldg_d(fb + F.fb_off + k);
        if (F.mask) w *= ldg_d(F.mask + k);
        bool cj;
        const int64_t row = half_row(wrap_add(base0, u_lo + j, n), n, cj);
        cplx* o = F.out + row * F.out_ls + k;
        cplx a = *o;
        *o = cj ? mk(a.x + mul_rn(w, v.x), a.y - mul_rn(w, v.y))
                : mk(a.x + w * v.x, a.y + w * v.y);
    }
};

// finish_facet (core.py:452-484): out[k] = Fb_c[k] * fft_c(sum)[(yN/2 - fs//2 + k + off) mod yN]
struct FinishFacetOp {
    Lines g;
    const double* fb;
    int n, fs;
    int start;  // (yN/2 - fs//2 + facet_off) mod yN
    const double* mask;  // optional 0/1 facet mask along the axis (api_helper.py:175-176,195-196)
    SW_HD cplx load(int64_t line, int q) const {
        int qc = wrap_add(q, n / 2, n);
        return ld_stream(g.in + line * g.in_ls + (int64_t)qc * g.in_es);
    }
    SW_HD void prefetch(int64_t line, int q) const {
        int qc = wrap_add(q, n / 2, n);
        prefetch_l2(g.in + line * g.in_ls + (int64_t)qc * g.in_es);
    }
    SW_HD void store(int64_t line, int p, cplx v) const {
        int pc = wrap_add(p, n / 2, n);
        int k = wrap_sub(pc, start, n);
        if (k < fs) {
            double s = mask ? ldg_d(fb + k) * ldg_d(mask + k) : ldg_d(fb + k);
            st_stream(g.out + line * g.out_ls + (int64_t)k * g.out_es, cscale(v, s));
        }
    }
};

// finish_facet of a real image: out[k] = (Re(fft_c(sum))[...] * Fb_c[k]) * mask[k], written as
// doubles.  The product order is that of finish_facet followed by the driver's row mask
// (api_helper.py finish_facet), so the samples are bitwise Re of the complex facet's.  g.out and
// mask are unused; the output strides are counted in doubles.
struct FinishFacetRealOp : FinishFacetOp {
    double* rout;
    int64_t rout_ls, rout_es;
    const double* rmask;  // optional facet mask along the axis, or null
    SW_HD void store(int64_t line, int p, cplx v) const {
        int pc = wrap_add(p, n / 2, n);
        int k = wrap_sub(pc, start, n);
        if (k < fs) {
            double x = v.x * ldg_d(fb + k);
            if (rmask) x *= ldg_d(rmask + k);
            st_stream_d(rout + line * rout_ls + (int64_t)k * rout_es, x);
        }
    }
};

// FinishFacetRealOp reading half-row lines (n/2 + 1 samples, natural order): the loader forms the
// Hermitian part of the full line, whose transform has the same real part,
//   0.5 H[q] (0 < q < n/2),  0.5 conj(H[n - q]) (q > n/2),  (Re H[q], 0) (q = 0, n/2)
struct FinishFacetRealHalfOp : FinishFacetRealOp {
    SW_HD cplx load(int64_t line, int q) const {
        const cplx* p = g.in + line * g.in_ls;
        if (q == 0 || q == n / 2) return mk(ld_stream(p + (int64_t)q * g.in_es).x, 0.0);
        if (q < n / 2) return cscale(ld_stream(p + (int64_t)q * g.in_es), 0.5);
        const cplx x = ld_stream(p + (int64_t)(n - q) * g.in_es);
        return mk(0.5 * x.x, -(0.5 * x.y));
    }
    SW_HD void prefetch(int64_t line, int q) const {
        prefetch_l2(g.in + line * g.in_ls + (int64_t)(q <= n / 2 ? q : n - q) * g.in_es);
    }
};

// add_to_subgrid (core.py:255-285):
//   out[(xM/2 - m/2 + u + sf) mod xM] += Fn[u] * fft_c(contrib)[(u + sf) mod m]
struct AddToSubgridOp {
    Lines g;
    const double* fn;
    int m, xM;
    int sf_m;  // sf mod m
    int base;  // (xM/2 - m/2 + sf) mod xM
    SW_HD cplx load(int64_t line, int t) const {
        int tc = wrap_add(t, m / 2, m);
        return ld_stream(g.in + line * g.in_ls + (int64_t)tc * g.in_es);
    }
    SW_HD void store(int64_t line, int w, cplx v) const {
        int wc = wrap_add(w, m / 2, m);
        int u = wrap_sub(wc, sf_m, m);
        int pos = wrap_add(base, u, xM);
        cplx* o = g.out + line * g.out_ls + (int64_t)pos * g.out_es;
        cplx a = *o;
        double f = ldg_d(fn + u);
        *o = mk(a.x + f * v.x, a.y + f * v.y);
    }
};

// extract_from_subgrid (core.py:370-406):
//   w[(u + sf) mod m] = Fn[u] * FSi[(xM/2 - m/2 + u + sf) mod xM];  out = ifft_c(w)
struct ExtractFromSubgridOp {
    Lines g;
    const double* fn;
    int m, xM;
    int sf_m, base;
    double scale;  // 1 / m
    SW_HD cplx load(int64_t line, int t) const {
        int tc = wrap_add(t, m / 2, m);
        int u = wrap_sub(tc, sf_m, m);
        int pos = wrap_add(base, u, xM);
        return cscale(ld_stream(g.in + line * g.in_ls + (int64_t)pos * g.in_es), ldg_d(fn + u));
    }
    SW_HD void store(int64_t line, int p, cplx v) const {
        int pc = wrap_add(p, m / 2, m);
        st_stream(g.out + line * g.out_ls + (int64_t)pc * g.out_es, cscale(v, scale));
    }
};

// finish_subgrid, one axis (core.py:287-325):
//   out[r] = ifft_c(summed)[(xM/2 - sz//2 + r + off) mod xM]
struct FinishSubgridOp {
    Lines g;
    int xM, sz;
    int start;  // (xM/2 - sz//2 + off) mod xM
    double scale;  // 1 / xM
    const double* mask;  // optional 0/1 mask along the axis (api_helper.py:107-111) or null
    SW_HD cplx load(int64_t line, int q) const {
        int qc = wrap_add(q, xM / 2, xM);
        return ld_stream(g.in + line * g.in_ls + (int64_t)qc * g.in_es);
    }
    SW_HD void store(int64_t line, int p, cplx v) const {
        int pc = wrap_add(p, xM / 2, xM);
        int r = wrap_sub(pc, start, xM);
        if (r < sz) {
            double s = mask ? scale * ldg_d(mask + r) : scale;
            st_stream(g.out + line * g.out_ls + (int64_t)r * g.out_es, cscale(v, s));
        }
    }
};

// prepare_subgrid, one axis (core.py:328-368):
//   out = fft_c(roll(pad_mid(subgrid, xM), off))
struct PrepareSubgridOp {
    Lines g;
    int xM, sz;
    int start;  // (xM/2 - sz//2 + off) mod xM
    SW_HD cplx load(int64_t line, int q) const {
        int qc = wrap_add(q, xM / 2, xM);
        int r = wrap_sub(qc, start, xM);
        if (r >= sz) return mk(0.0, 0.0);
        return ld_stream(g.in + line * g.in_ls + (int64_t)r * g.in_es);
    }
    SW_HD void store(int64_t line, int p, cplx v) const {
        int pc = wrap_add(p, xM / 2, xM);
        st_stream(g.out + line * g.out_ls + (int64_t)pc * g.out_es, v);
    }
};

// ops that derive per-output factors by recurrence (prep / store_w, see PrepareFacetPassAOp)
template <class Op, class = void>
struct HasTwiddlePrep : std::false_type {};
template <class Op>
struct HasTwiddlePrep<Op, std::void_t<typename Op::Tw>> : std::true_type {};

// ------------------------------------------------------------------ line kernels
// NFFT-point transform of a batch of lines; LPC lines per CTA, T = NFFT/16
// threads per line.  LINE_FASTEST selects which of (line, thread-in-line) varies
// fastest across the lanes of a warp: use it when lines are adjacent in memory
// (axis-0 transforms of C-ordered arrays) so that global accesses coalesce
// across lines instead of along them.
template <int NFFT, int DIR, int LPC, bool LINE_FASTEST, class Op>
struct LineKernel {
    static constexpr int T = FftCfg<NFFT>::T;
    static constexpr int THREADS = T * LPC;
    // odd slot stride between line buffers => lines land in different banks
    static constexpr int LSTRIDE = FftCfg<NFFT>::PADDED | 1;
    static constexpr size_t SMEM = (size_t)LSTRIDE * LPC * sizeof(double);
    Op op;
    const cplx* tw;

    template <class Ctx>
    SW_HD void operator()(Ctx& ctx) const {
        double* smem = (double*)ctx.smem;
        const int l = LINE_FASTEST ? (ctx.tid % LPC) : (ctx.tid / T);
        const int lt = LINE_FASTEST ? (ctx.tid / LPC) : (ctx.tid % T);
        double* sm = smem + (size_t)l * LSTRIDE;
        auto sync = [&]() { ctx.sync(); };
        for (int64_t line0 = (int64_t)ctx.bid * LPC; line0 < op.g.n_lines;
             line0 += (int64_t)ctx.nblocks * LPC) {
            const int64_t line = line0 + l;
            const bool active = line < op.g.n_lines;
            auto ld = [&](int q) { return active ? op.load(line, q) : mk(0.0, 0.0); };
            if constexpr (HasTwiddlePrep<Op>::value) {
                typedef LastPass<NFFT> LP;
                typename Op::Tw tws = op.prep(active ? line : 0, lt, T, LP::NS);
                cplx w_it = tws.base, w = tws.base;
                auto st = [&](int p, cplx v, int it, int r) {
                    if (r == 0) {
                        if (it > 0) w_it = cmul(w_it, tws.step_it);
                        w = w_it;
                    } else {
                        w = cmul(w, tws.step_r);
                    }
                    if (active) op.store_w(line, p, v, w);
                };
                line_fft<NFFT, DIR>(lt, sm, tw, ld, st, sync);
            } else {
                auto st = [&](int p, cplx v) {
                    if (active) op.store(line, p, v);
                };
                line_fft<NFFT, DIR>(lt, sm, tw, ld, st, sync);
            }
            ctx.sync();  // smem is reused by the next line
        }
    }
};

// 2*H-point transform as two H-point transforms (lines that do not fit shared memory,
// yN = 16384), decimation in time:
//   E = FFT_H(z[2j]),  O = FFT_H(z[2j+1]),  w = exp(DIR 2 pi i k / 2H)
//   X[k] = E[k] + w O[k],   X[k+H] = E[k] - w O[k]
// E is parked in a per-CTA global scratch line (H samples, L2 resident; every thread reads
// back exactly the samples it wrote, so no synchronisation is involved) while O is
// computed; both halves of the output are then written with unit stride.  (A
// decimation-in-frequency split needs no scratch but writes X[2k] and X[2k+1] in
// separate passes: 16-byte stores at 32-byte stride multiply the DRAM write traffic.)  tw2 is the table exp(-2 pi i t / 2H), t < H.
template <int H, int DIR, class Op>
struct SplitLineKernel {
    static constexpr int T = FftCfg<H>::T;
    static constexpr int THREADS = T;
    static constexpr size_t SMEM = (size_t)FftCfg<H>::PADDED * sizeof(double);
    Op op;
    const cplx* tw;   // compact table of the H-point plan
    const cplx* tw2;  // exp(-2 pi i t / 2H), t < H
    cplx* scratch;    // gridDim.x * H samples

    template <class Ctx>
    SW_HD void operator()(Ctx& ctx) const {
        double* sm = (double*)ctx.smem;
        cplx* stash = scratch + (size_t)ctx.bid * H;
        const int lt = ctx.tid;
        auto sync = [&]() { ctx.sync(); };
        for (int64_t line = ctx.bid; line < op.g.n_lines; line += ctx.nblocks) {
            {
                auto ld = [&](int q) { return op.load(line, 2 * q); };
                auto st = [&](int k, cplx v) { stash[k] = v; };
                line_fft<H, DIR>(lt, sm, tw, ld, st, sync);
            }
            ctx.sync();
            {
                auto ld = [&](int q) { return op.load(line, 2 * q + 1); };
                auto st = [&](int k, cplx o) {
                    cplx w = ldg_c(tw2 + k);
                    if (DIR > 0) w.y = -w.y;
                    cplx e = stash[k];
                    cplx wo = cmul(o, w);
                    op.store(line, k, cadd(e, wo));
                    op.store(line, k + H, csub(e, wo));
                };
                line_fft<H, DIR>(lt, sm, tw, ld, st, sync);
            }
            ctx.sync();
        }
    }
};

// N = F * M point transform for ANY small factor F <= 16 and power-of-two M (non power-of-two
// lengths of the parameter catalogue: yN, xM = {3, 5, 7, 9} * 2^k, and lengths above 16384):
// decimation in time by F,
//   E_q = FFT_M(z[F j + q]),  X[k + M s] = sum_q (w^(q k) E_q[k]) exp(DIR 2 pi i q s / F),
//   w = exp(DIR 2 pi i / N).
// E_0 .. E_{F-2} are parked in the per-CTA scratch (L2), E_{F-1} stays in registers; the
// combine is a dense F-point DFT per output index (F^2 complex multiplies per F outputs --
// these lengths are off the benchmark path, generality over speed).
// twf: exp(-2 pi i t / N), t < N/2 (N is even for every SwiFTly size); wf: exp(-2 pi i t / F).
#define SW_MAX_SPLIT_F 16
template <int M, int DIR, class Op>
struct SplitFKernel {
    static constexpr int T = FftCfg<M>::T;
    static constexpr int THREADS = T;
    static constexpr size_t SMEM = (size_t)FftCfg<M>::PADDED * sizeof(double);
    Op op;
    const cplx* tw;   // compact table of the M-point plan
    const cplx* twf;  // exp(-2 pi i t / N), t < N / 2
    cplx* scratch;    // gridDim.x * (F - 1) * M samples
    int F;
    cplx wf[SW_MAX_SPLIT_F];  // exp(-2 pi i t / F)

    SW_HD cplx root_n(int64_t t, int64_t n) const {  // exp(DIR 2 pi i t / n), 0 <= t < n
        const bool neg = t >= n / 2;
        cplx w = ldg_c(twf + (neg ? t - n / 2 : t));
        if (DIR > 0) w.y = -w.y;
        return neg ? mk(-w.x, -w.y) : w;
    }

    template <class Ctx>
    SW_HD void operator()(Ctx& ctx) const {
        double* sm = (double*)ctx.smem;
        cplx* stash = scratch + (size_t)ctx.bid * (size_t)(F - 1) * M;
        const int lt = ctx.tid;
        const int64_t n = (int64_t)F * M;
        auto sync = [&]() { ctx.sync(); };
        for (int64_t line = ctx.bid; line < op.g.n_lines; line += ctx.nblocks) {
            for (int q = 0; q < F; ++q) {
                auto ld = [&](int j) { return op.load(line, F * j + q); };
                if (q < F - 1) {
                    cplx* sq = stash + (size_t)q * M;
                    auto st = [&](int k, cplx v) { sq[k] = v; };
                    line_fft<M, DIR>(lt, sm, tw, ld, st, sync);
                } else {
                    auto st = [&](int k, cplx last) {
                        cplx e[SW_MAX_SPLIT_F];
                        for (int qq = 0; qq < F - 1; ++qq)
                            e[qq] = cmul(stash[(size_t)qq * M + k], root_n((int64_t)qq * k, n));
                        e[F - 1] = cmul(last, root_n((int64_t)(F - 1) * k, n));
                        for (int s = 0; s < F; ++s) {
                            cplx acc = e[0];
                            for (int qq = 1; qq < F; ++qq) {
                                cplx w = wf[(qq * s) % F];
                                if (DIR > 0) w.y = -w.y;
                                acc = cadd(acc, cmul(e[qq], w));
                            }
                            op.store(line, k + M * s, acc);
                        }
                    };
                    line_fft<M, DIR>(lt, sm, tw, ld, st, sync);
                }
                ctx.sync();
            }
        }
    }
};

// ------------------------------------------------------------------ gather / scatter kernels
// extract_from_facet (core.py:224-253):  out[t] = prep[(base + ((t - s_m) mod m)) mod yN]
// add_to_facet      (core.py:408-449):  out[(base + ((t - s_m) mod m)) mod yN] += contrib[t]
//   s = subgrid_off * yN // N, s_m = s mod m, base = (yN/2 - m/2 + s) mod yN
template <bool SCATTER_ADD>
struct WindowCopyKernel {
    static constexpr int THREADS = 256;
    static constexpr size_t SMEM = 0;
    Lines g;
    int m, yN, s_m, base;
    int line_fastest;  // lines adjacent in memory (axis 0): make `line` the fast index
    template <class Ctx>
    SW_HD void operator()(Ctx& ctx) const {
        const int64_t total = g.n_lines * (int64_t)m;
        for (int64_t i = (int64_t)ctx.bid * THREADS + ctx.tid; i < total;
             i += (int64_t)ctx.nblocks * THREADS) {
            int64_t line;
            int t;
            if (line_fastest) {
                line = i % g.n_lines;
                t = (int)(i / g.n_lines);
            } else {
                line = i / m;
                t = (int)(i % m);
            }
            int w = wrap_add(base, wrap_sub(t, s_m, m), yN);
            if (SCATTER_ADD) {
                cplx v = ld_stream(g.in + line * g.in_ls + (int64_t)t * g.in_es);
                cplx* o = g.out + line * g.out_ls + (int64_t)w * g.out_es;
                cplx a = *o;
                *o = cadd(a, v);
            } else {
                g.out[line * g.out_ls + (int64_t)t * g.out_es] =
                    ld_stream(g.in + line * g.in_ls + (int64_t)w * g.in_es);
            }
        }
    }
};


// ------------------------------------------------------------------ fused subgrid axis kernel
// One axis of "sum the contributions of several sources and finish":
//   for every output line l:
//     acc[0..xM) = 0
//     for every source g:  c = window of source line l   (extract_from_facet, core.py:224-253)
//                          acc[(pos_g + u) mod xM] += Fn[u] * fft_c(c)[(u + sf_g) mod m]
//                                                           (add_to_subgrid, core.py:255-285)
//     out[l, r] = mask[r] * ifft_c(acc)[(start + r) mod xM], r < sz
//                                                           (finish_subgrid, core.py:287-325)
// The padded accumulator lives in shared memory only: neither the (m) contributions nor the
// (xM) accumulators of the reference's sum_and_finish_subgrid (api_helper.py:73-112) ever
// touch HBM.  Used twice per subgrid: along axis 1 with the facets of one facet row as
// sources (windows of their NMBF_BF buffers), then along axis 0 with the per-row strips as
// sources.  Sources are processed CONC = xM/m at a time ("rounds"); the host orders them so
// that the windows inside one round do not overlap (plain read-modify-write on acc).
struct SgSource {
    const cplx* base;      // nullptr: empty slot
    int64_t ls, es;        // stride between task lines / between samples (complex elements)
    int wbase, s_m, wmod;  // sample index of centred contribution index tc:
                           //   (wbase + ((tc - s_m) mod m)) mod wmod
    int sf_m, pos_base;    // sf mod m ; (xM/2 - m/2 + sf) mod xM
};
#define SW_MAX_SOURCES 64
#define SW_MAX_GROUPS 16

// LINES = 2 processes two ADJACENT lines per CTA with the two lines interleaved across
// lanes (lane pairs touch 32 contiguous bytes): used when lines are adjacent in memory
// (axis-0 work on C-ordered arrays), where one line per CTA would fetch every 32-byte
// sector twice.
//
// m and xM may also be mixed-radix lengths (LineCfg<N, false> in fft_engine.cuh, the
// catalogue's 3, 5 and 7 * 2^k geometries); the transforms then go through line_fft_mixed,
// whose work area also holds the sub-transform outputs.
template <int M, int XM, int LINES>
struct SubgridAxisKernel {
    static constexpr int T_M = LineCfg<M>::T;
    static constexpr int T_X = LineCfg<XM>::T;
    static constexpr int THREADS = T_X * LINES;
    static constexpr int CONC = T_X / T_M;  // = XM / M concurrent m-point transforms per line
    // power of two: odd stride (the transforms' exchanges land in different banks); mixed
    // radix: even (the work area holds complex samples)
    static constexpr int WSTRIDE = (M & (M - 1)) == 0 ? (LineCfg<M>::SCRATCH | 1)
                                                      : ((LineCfg<M>::SCRATCH + 1) & ~1);
    // doubles: the CONC m-point work areas, which the xM-point transform reuses
    static constexpr int WORK0 = CONC * WSTRIDE >= LineCfg<XM>::SCRATCH ? CONC * WSTRIDE
                                                                         : LineCfg<XM>::SCRATCH;
    // per-line strides: the second line lands 8 bank pairs (64 B) away from the first
    static constexpr int WORK = LINES == 1 ? WORK0 : ((WORK0 + 15) / 16) * 16 + 8;
    static constexpr int ACCS = LINES == 1 ? XM : XM + 4;
    static constexpr size_t SMEM =
        ((size_t)ACCS * sizeof(cplx) + (size_t)WORK * sizeof(double)) * LINES;
    // register budget by allocated warps (MinBlocks, common.cuh) for the pairs added for the
    // catalogue whose CTAs are not whole warps: the mixed-radix lengths and m = xM = 256
    // (10..56 threads).  Counted by thread their budget was 64..96 registers and they spilled
    // 380..908 bytes.  The earlier power-of-two pairs keep the budget they were measured with.
    static constexpr bool WARP_BOUNDS = (M & (M - 1)) != 0 || (XM & (XM - 1)) != 0 || M == XM;

    // Several independent "groups" (e.g. the facet rows of one subgrid) share one launch:
    // group g uses source slots [g * n_slots, (g + 1) * n_slots), has n_lines lines and
    // writes to out + g * out_gs.
    SgSource src[SW_MAX_SOURCES];
    int n_slots;   // slots per group (multiple of CONC)
    int n_groups;
    const double* fn;
    const cplx* tw_m;
    const cplx* tw_x;
    int64_t n_lines;  // per group
    cplx* out;
    int64_t out_ls, out_es, out_gs;
    int sz;
    int start[SW_MAX_GROUPS];           // per group: (xM/2 - sz//2 + subgrid_off) mod xM
    const double* mask[SW_MAX_GROUPS];  // per group: sz doubles or null
    double scale;                       // 1 / xM
    // set by the host when, in EVERY group, the windows of the first round are pairwise
    // disjoint and tile the accumulator completely (the regular facet layouts): the first
    // round then stores instead of read-modify-write and the accumulator is not zeroed
    int first_round_tiles;
    // the launch is a later piece of a job with more sources than fit one launch: the
    // finished lines are ADDED to `out` (finishing is linear)
    int accumulate_out;
    cplx* out_g[SW_MAX_GROUPS];  // optional per-group output base (null: out + g * out_gs)

    template <class Ctx>
    SW_HD void operator()(Ctx& ctx) const {
        const int sub = ctx.tid % LINES;  // which of the CTA's lines
        const int t = ctx.tid / LINES;    // thread within the line
        cplx* acc = (cplx*)ctx.smem + (size_t)sub * ACCS;
        double* work = (double*)((cplx*)ctx.smem + (size_t)LINES * ACCS) + (size_t)sub * WORK;
        const int c = t / T_M;
        const int lt = t % T_M;
        auto sync = [&]() { ctx.sync(); };
        // The CONC concurrent m-point transforms only need to synchronise among their own
        // T_M * LINES threads: with one named barrier per transform the groups drift apart and
        // the exchange phases (LSU bound) of some overlap the butterfly phases (FP64 bound) of
        // others instead of the whole CTA alternating between the two.
        constexpr bool GROUP_BARRIERS = (T_M * LINES) % 32 == 0 && CONC > 1 && CONC <= 15;
        auto gsync = [&]() {
            if (GROUP_BARRIERS)
                ctx.group_sync(1 + c, T_M * LINES);
            else
                ctx.sync();
        };
        const int64_t lines_cta = (n_lines + LINES - 1) / LINES;  // line pairs per group
        const int64_t total = lines_cta * n_groups;
        for (int64_t gl = ctx.bid; gl < total; gl += ctx.nblocks) {
            const int grp = (int)(gl / lines_cta);
            const int64_t line = (gl - (int64_t)grp * lines_cta) * LINES + sub;
            const bool line_ok = line < n_lines;
            if (!first_round_tiles) {
                for (int i = t; i < XM; i += T_X) acc[i] = mk(0.0, 0.0);
                ctx.sync();
            }
            for (int slot0 = 0; slot0 < n_slots; slot0 += CONC) {
                const bool overwrite = first_round_tiles && slot0 == 0;
                const int slot = grp * n_slots + slot0 + c;
                const bool active = line_ok && slot0 + c < n_slots && src[slot].base != nullptr;
                // keep the descriptor in registers (kernel parameters live in constant memory)
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
                // prefetch what this thread will load next into L2: the next round of this
                // line, or -- in the last round -- the first round of the CTA's next line
                {
                    int pslot0 = slot0 + CONC, pgrp = grp;
                    int64_t pline = line;
                    if (pslot0 >= n_slots) {
                        pslot0 = 0;
                        const int64_t ngl = gl + ctx.nblocks;
                        pgrp = (int)(ngl / lines_cta);
                        pline = (ngl - (int64_t)pgrp * lines_cta) * LINES + sub;
                        if (ngl >= total || pline >= n_lines) pgrp = -1;
                    }
                    // (measured: helps contiguous lines, hurts the strided two-line variant)
                    if (LINES == 1 && pgrp >= 0 && pslot0 + c < n_slots) {
                        const SgSource& ps = src[pgrp * n_slots + pslot0 + c];
                        if (ps.base != nullptr) {
                            const cplx* pb = ps.base + pline * ps.ls;
#pragma unroll
                            for (int r = 0; r < 16; ++r) {
                                int tc = wrap_add(lt + r * T_M, M / 2, M);
                                int idx = wrap_add(ps.wbase, wrap_sub(tc, ps.s_m, M), ps.wmod);
                                prefetch_l2(pb + (int64_t)idx * ps.es);
                            }
                        }
                    }
                }
                line_fft_any<M, -1>(lt, work + (size_t)c * WSTRIDE, tw_m, ld, st, gsync);
                ctx.sync();
            }
            {
                cplx* o = (out_g[grp] ? out_g[grp] : out + (int64_t)grp * out_gs) + line * out_ls;
                const int gstart = start[grp];
                const double* gmask = mask[grp];
                auto ld = [&](int q) { return acc[wrap_add(q, XM / 2, XM)]; };
                auto st = [&](int p, cplx v) {
                    int pc = wrap_add(p, XM / 2, XM);
                    int r = wrap_sub(pc, gstart, XM);
                    if (line_ok && r < sz) {
                        double f = gmask ? scale * ldg_d(gmask + r) : scale;
                        cplx* dst = o + (int64_t)r * out_es;
                        if (accumulate_out) {
                            cplx a = *dst;
                            *dst = mk(a.x + f * v.x, a.y + f * v.y);
                        } else {
                            st_stream(dst, cscale(v, f));
                        }
                    }
                };
                line_fft_any<XM, +1>(t, work, tw_x, ld, st, sync);
            }
            ctx.sync();  // acc / work are reused by the next line
        }
    }
};

// ------------------------------------------------------------------ fused subgrid split kernel
// The adjoint of SubgridAxisKernel: one axis of "prepare a subgrid and cut it into the
// contributions of several facets":
//   for every input line l:
//     acc[0..xM) = fft_c(roll(pad_mid(in[l], xM), off))      (prepare_subgrid, core.py:328-368)
//     for every target j:  w[(u + sf_j) mod m] = Fn[u] * acc[(xM/2 - m/2 + u + sf_j) mod xM]
//                          c = ifft_c(w)                      (extract_from_subgrid, core.py:370-406)
//       store mode:  out_j[l, t] = c[t]
//       add mode:    out_j[l, (yN/2 - m/2 + s + ((t - s) mod m)) mod yN] += c[t],  s = off yN / N
//                                                           (add_to_facet, core.py:408-449)
// The prepared xM-point line lives in shared memory only.  The targets only READ it, so their
// windows may overlap or repeat: targets are processed CONC = xM/m at a time in the order given,
// and a round with fewer targets leaves its idle transform slots idle (no transform of zeros).
// A CTA takes a line (two adjacent lines with LINES = 2) and runs it through EVERY group of the
// launch in order, so every (target, line) is written by exactly one CTA even when targets of
// different groups share an accumulator (a batch of subgrids of one subgrid column): no
// atomics, and the sums are formed in group order.
struct SplitTarget {
    cplx* base;          // line 0, sample 0 of the target
    int64_t ls, es;      // line / sample stride (complex elements)
    int sf_m, pos_base;  // facet_off * xM // N mod m ; (xM/2 - m/2 + sf) mod xM
};
struct SplitGroup {
    const cplx* in;     // input lines (sz samples each)
    int64_t in_ls, in_es;
    int sz, start;      // subgrid size ; (xM/2 - sz//2 + subgrid_off) mod xM
    int s_m, base_y;    // add mode: subgrid_off * yN // N mod m ; (yN/2 - m/2 + s) mod yN
    int first, count;   // targets [first, first + count) of the launch's table
};

// CTA barrier that the threads of one warp may reach from DIFFERENT places in the code
// (barrier.sync without .aligned; __syncthreads is the aligned form, which requires the whole
// warp to execute the same barrier instruction)
template <class Ctx>
SW_HD void cta_sync_divergent(const Ctx& ctx) {
#if defined(__CUDA_ARCH__) && !defined(SWIFTLY_EMU)
    (void)ctx;
    asm volatile("barrier.sync 0;" ::: "memory");
#else
    ctx.sync();
#endif
}

template <int M, int XM, int LINES>
struct SubgridSplitAxisKernel {
    static constexpr int T_M = LineCfg<M>::T;
    static constexpr int T_X = LineCfg<XM>::T;
    static constexpr int THREADS = T_X * LINES;
    static constexpr int CONC = T_X / T_M;
    // shared memory layout as in SubgridAxisKernel
    static constexpr int WSTRIDE = SubgridAxisKernel<M, XM, LINES>::WSTRIDE;
    static constexpr int WORK = SubgridAxisKernel<M, XM, LINES>::WORK;
    static constexpr int ACCS = SubgridAxisKernel<M, XM, LINES>::ACCS;
    static constexpr size_t SMEM = SubgridAxisKernel<M, XM, LINES>::SMEM;
    static constexpr bool WARP_BOUNDS = SubgridAxisKernel<M, XM, LINES>::WARP_BOUNDS;
    // transforms of whole warps synchronise on a named barrier of their own; otherwise the
    // barrier is CTA-wide and the threads of an idle slot take part in it -- from another place
    // in the code than the transform's threads of the same warp, hence the non-aligned barrier
    static constexpr bool GROUP_BARRIERS = (T_M * LINES) % 32 == 0 && CONC > 1 && CONC <= 15;

    SplitTarget tgt[SW_MAX_SOURCES];
    SplitGroup grp[SW_MAX_GROUPS];
    int n_groups;
    int64_t n_lines;  // every group
    int add;          // 0: store mode, 1: add-to-facet mode
    int yN;
    const double* fn;
    const cplx* tw_m;
    const cplx* tw_x;
    double scale;  // 1 / m

    template <class Ctx>
    SW_HD void operator()(Ctx& ctx) const {
        const int sub = ctx.tid % LINES;
        const int t = ctx.tid / LINES;
        cplx* acc = (cplx*)ctx.smem + (size_t)sub * ACCS;
        double* work = (double*)((cplx*)ctx.smem + (size_t)LINES * ACCS) + (size_t)sub * WORK;
        const int c = t / T_M;
        const int lt = t % T_M;
        auto sync = [&]() { ctx.sync(); };
        auto gsync = [&]() {
            if (GROUP_BARRIERS)
                ctx.group_sync(1 + c, T_M * LINES);
            else
                cta_sync_divergent(ctx);
        };
        const int64_t lines_cta = (n_lines + LINES - 1) / LINES;
        for (int64_t wl = ctx.bid; wl < lines_cta; wl += ctx.nblocks) {
            const int64_t line = wl * LINES + sub;
            const bool line_ok = line < n_lines;
            for (int g = 0; g < n_groups; ++g) {
                const int count = grp[g].count;
                if (count == 0) continue;
                {
                    const cplx* in = grp[g].in + (line_ok ? line : 0) * grp[g].in_ls;
                    const int64_t in_es = grp[g].in_es;
                    const int sz = grp[g].sz, start = grp[g].start;
                    auto ld = [&](int q) {
                        int r = wrap_sub(wrap_add(q, XM / 2, XM), start, XM);
                        if (!line_ok || r >= sz) return mk(0.0, 0.0);
                        return ld_stream(in + (int64_t)r * in_es);
                    };
                    auto st = [&](int p, cplx v) { acc[wrap_add(p, XM / 2, XM)] = v; };
                    line_fft_any<XM, -1>(t, work, tw_x, ld, st, sync);
                }
                ctx.sync();  // acc complete; the work area is free for the m-point transforms
                const int s_m = grp[g].s_m, base_y = grp[g].base_y;
                for (int k0 = 0; k0 < count; k0 += CONC) {
                    if (k0 + c < count) {
                        const SplitTarget& T = tgt[grp[g].first + k0 + c];
                        cplx* base = T.base + (line_ok ? line : 0) * T.ls;
                        const int64_t es = T.es;
                        const int sf_m = T.sf_m, pos_base = T.pos_base;
                        auto ld = [&](int q) {
                            int u = wrap_sub(wrap_add(q, M / 2, M), sf_m, M);
                            return cscale(acc[wrap_add(pos_base, u, XM)], ldg_d(fn + u));
                        };
                        auto st = [&](int p, cplx v) {
                            if (!line_ok) return;
                            int pc = wrap_add(p, M / 2, M);
                            if (add) {
                                int w = wrap_add(base_y, wrap_sub(pc, s_m, M), yN);
                                cplx* o = base + (int64_t)w * es;
                                cplx a = *o;
                                *o = mk(a.x + scale * v.x, a.y + scale * v.y);
                            } else {
                                st_stream(base + (int64_t)pc * es, cscale(v, scale));
                            }
                        };
                        line_fft_any<M, +1>(lt, work + (size_t)c * WSTRIDE, tw_m, ld, st, gsync);
                    } else if constexpr (!GROUP_BARRIERS) {
                        for (int i = 0; i < LineBarriers<M>::V; ++i) cta_sync_divergent(ctx);
                    }
                    // work areas are reused by the next round / the next line
                    if constexpr (GROUP_BARRIERS)
                        ctx.sync();
                    else
                        cta_sync_divergent(ctx);
                }
            }
        }
    }
};

}  // namespace swiftly
