"""
The subgrid-side primitives (add_to_subgrid, extract_from_subgrid, finish_subgrid,
prepare_subgrid, subgrid_to_facets) and the window copies (extract_from_facet / add_to_facet) at
every subgrid-side FFT length the library runs, shared by the emulated and the GPU tests.

An ``m``-point line (m = xM_yN_size: add_to_subgrid, extract_from_subgrid, subgrid_to_facets) or
an ``xM``-point line (finish_subgrid, prepare_subgrid) runs through ``LineKernel`` (a power of two,
``LinesPerCta`` lines per CTA) or ``SplitFKernel<M>`` (any other ``F * M``), chosen by length as
for the facet lines (``dispatch.cuh``; ``length_cases.line_kernel`` restates it).  The window
copies run ``WindowCopyKernel``.  Every case asserts the launch it was written for
(``swiftly_b200_debug_last_launch``: kernel, lines per CTA or F, line-fastest flag, grid) against
the pinned :data:`FORMS`.

``m_plans()`` / ``xm_plans()`` derive the lengths from ``SWIFT_CONFIGS`` (which holds the
benchmark sets) and ``FUSED_FORWARD_PAIRS`` and pin them, so that a new catalogue entry or a
change of the dispatch fails loudly.  Each length gets two geometries: the smallest catalogue
entry that uses it, as ``pair_cases.core_plan`` picks it (the GPU tests), and a small plan of
the same pair, as ``pair_cases.small_plan`` picks it (the emulated tests); a library-only length
takes the library pair with the smallest other length.
"""

import contextlib

import numpy
import torch

from ska_sdp_distributed_fourier_transform_b200.swift_configs import (
    FUSED_FORWARD_PAIRS,
    SWIFT_CONFIGS,
)
from tests import catalogue_cases as cc
from tests import length_cases as lc
from tests import pair_cases as prc
from tests import parity_cases as pc

# kernels of swiftly_b200_debug_last_launch (plan.h)
LINE, SPLIT_LINE, SPLIT_F, WINDOW_COPY = 4, 5, 6, 7
NUM_SMS = 132  # plan.h
LINE_GRID_CAP = NUM_SMS * 32  # grid_for: a grid-stride loop covers the rest
WINDOW_GRID_CAP = NUM_SMS * 64  # capi.cu window_copy_grid
WINDOW_THREADS = 256
SPLIT_GRID = 296  # launch_split_f: persistent CTAs

PINNED_M_DIRECT = (32, 64, 128, 256, 512, 1024, 2048)
PINNED_M_SPLIT_F = frozenset([(32, 5), (32, 7), (64, 3)])  # (M, F): m = 160, 224, 192
PINNED_XM_DIRECT = (64, 128, 256, 512, 1024, 2048, 4096, 8192)
PINNED_XM_SPLIT_F = frozenset([(128, 3), (64, 5), (64, 7)])  # xM = 384, 320, 448

# The launch of an n-point subgrid line: (kernel, lines per CTA for LINE / F for SPLIT_F).
# LinesPerCta<n> = min(16, 256 / (n / 16)), at least 1.
FORMS = {
    32: (LINE, 16), 64: (LINE, 16), 128: (LINE, 16), 256: (LINE, 16), 512: (LINE, 8),
    1024: (LINE, 4), 2048: (LINE, 2), 4096: (LINE, 1), 8192: (LINE, 1),
    160: (SPLIT_F, 5), 192: (SPLIT_F, 3), 224: (SPLIT_F, 7),
    320: (SPLIT_F, 5), 384: (SPLIT_F, 3), 448: (SPLIT_F, 7),
}

# extract_from_facet / add_to_facet at the cfg4 geometry (m = 1024, yN = 16384)
CFG4 = "64k[1]-n16k-4k"


# ---------------------------------------------------------------------- plans
def _all_pairs():
    pairs = {(p["xM_size"] * p["yN_size"] // p["N"], p["xM_size"]) for p in SWIFT_CONFIGS.values()}
    return pairs | set(FUSED_FORWARD_PAIRS)


def _plans(which):
    """``which`` 0: m, 1: xM.  Plan id -> (n, plan, pair, gpu geometry, emulated geometry, xA)
    with geometries (W, N, xM, yN); xA is the catalogue entry's (None for a library-only
    length)."""
    reps = {}
    for name, p in SWIFT_CONFIGS.items():
        pair = (p["xM_size"] * p["yN_size"] // p["N"], p["xM_size"])
        key = (p["N"], p["yN_size"], name)
        n = pair[which]
        if n not in reps or key < reps[n][0]:
            reps[n] = (key, pair, (p["W"], p["N"], p["xM_size"], p["yN_size"]), p["xA_size"])
    for pair in sorted(_all_pairs(), key=lambda q: q[1 - which]):
        n = pair[which]
        if n not in reps:  # library-only length: the pair with the smallest other length
            reps[n] = (None, pair, prc.core_plan(pair), None)
    out = {}
    for n in sorted(reps):
        _, pair, gpu, xa = reps[n]
        plan = lc.line_kernel(n)
        out[f"{'m' if which == 0 else 'xM'}{n}-{lc.plan_id(plan)}"] = (
            n, plan, pair, gpu, prc.small_plan(pair), xa)
    return out


def m_plans():
    return _plans(0)


def xm_plans():
    return _plans(1)


def pinned_kinds(plans):
    """({direct lengths}, {(M, F) of the split-F lengths}) of a plan table."""
    direct = {p[1] for _, p, *_ in plans.values() if p[0] == "direct"}
    split_f = {p[1:] for _, p, *_ in plans.values() if p[0] == "splitf"}
    return direct, split_f


# ---------------------------------------------------------------------- launch record
def last_launch(core):
    return prc.last_launch(core)


def line_form(n, n_lines, adjacent, cap=0):
    """The launch record of an n-point line transform of ``n_lines`` lines."""
    kind, v = FORMS[n]
    if kind == LINE:
        grid = min(-(-n_lines // v), LINE_GRID_CAP)
        flag = int(adjacent and n_lines > 1 and v > 1)
    else:
        grid, flag = min(n_lines, SPLIT_GRID), 0
    return (kind, v, flag, min(grid, cap) if cap else grid)


def window_form(m, n_lines, adjacent, cap=0):
    grid = min(-(-(n_lines * m) // WINDOW_THREADS), WINDOW_GRID_CAP)
    return (WINDOW_COPY, 0, int(adjacent and n_lines > 1), min(grid, cap) if cap else grid)


def expect(core, want, what):
    got = last_launch(core)
    assert got == want, f"{what}: launched {got}, expected {want}"


@contextlib.contextmanager
def capped(core, cap):
    if not cap:
        yield
        return
    with prc.max_blocks(core, cap):
        yield


# ---------------------------------------------------------------------- helpers
_to = lc._to  # pylint: disable=protected-access
_check = lc._check  # pylint: disable=protected-access


def _lines(rng, axis, n_lines, size):
    return pc.rand_c(rng, n_lines, size) if axis == 1 else pc.rand_c(rng, size, n_lines)


def _np(t):
    return t.cpu().numpy() if isinstance(t, torch.Tensor) else numpy.asarray(t)


def facet_offsets(core):
    """Facet offsets 0, negative and >= N; the non-zero ones have sf = off xM / N with
    sf mod m != 0."""
    step = core.facet_off_step
    offs = [0, -3 * step, core.N + 5 * step]
    m = core.xM_yN_size
    assert all((o // step) % m for o in offs[1:])
    return offs


def subgrid_offsets(core):
    """Subgrid offsets below 0 and >= N."""
    step = core.subgrid_off_step
    return [-5 * step, core.N + 3 * step]


def sizes(core, xa):
    """Subgrid sizes xM, xM - 1, xM / 2 + 1 and the catalogue entry's xA."""
    xM = core.xM_size
    out = [xM, xM - 1, xM // 2 + 1]
    return out + ([xa] if xa and xa not in out else [])


def lpc_line_counts(n):
    """Line counts that leave the last CTA partly empty: LPC - 1, LPC + 1, 2 LPC + 3."""
    lpc = max(FORMS[n][1] if FORMS[n][0] == LINE else 1, 2)
    return [lpc - 1, lpc + 1, 2 * lpc + 3]


# ---------------------------------------------------------------------- against the oracle
def add_to_subgrid_vs_oracle(core, oracle, axis, n_lines, facet_off, accumulate, seed,
                             cap=0, rtol=1e-12):
    rng = numpy.random.default_rng(seed)
    m, xM = core.xM_yN_size, core.xM_size
    contrib = _lines(rng, axis, n_lines, m)
    out0 = _lines(rng, axis, n_lines, xM) if accumulate else None
    with capped(core, cap):
        got = core.add_to_subgrid(_to(core, contrib), facet_off, axis=axis,
                                  out=None if out0 is None else _to(core, out0))
    what = (f"add_to_subgrid m {m} axis {axis}, {n_lines} lines, off {facet_off}"
            f"{', into out' if accumulate else ''}{f', cap {cap}' if cap else ''}")
    expect(core, line_form(m, n_lines, axis == 0, cap), what)
    ref = oracle.add_to_subgrid(contrib, facet_off, axis=axis,
                                out=None if out0 is None else out0.copy())
    return _check(_np(got), ref, rtol, what)


def add_to_subgrid_2d_vs_oracle(core, oracle, off0, off1, seed, rtol=1e-12):
    rng = numpy.random.default_rng(seed)
    m, xM = core.xM_yN_size, core.xM_size
    contrib = pc.rand_c(rng, m, m)
    out0 = pc.rand_c(rng, xM, xM)
    got = core.add_to_subgrid_2d(_to(core, contrib), off0, off1, out=_to(core, out0))
    what = f"add_to_subgrid_2d m {m}, offs {off0}, {off1}"
    expect(core, line_form(m, xM, False), what)  # the last pass: axis 1, xM lines
    ref = oracle.add_to_subgrid(oracle.add_to_subgrid(contrib, off0, axis=0), off1, axis=1,
                                out=out0.copy())
    return _check(_np(got), ref, rtol, what)


def extract_from_subgrid_vs_oracle(core, oracle, axis, n_lines, facet_off, seed, cap=0,
                                   rtol=1e-12):
    rng = numpy.random.default_rng(seed)
    m, xM = core.xM_yN_size, core.xM_size
    fsi = _lines(rng, axis, n_lines, xM)
    with capped(core, cap):
        got = core.extract_from_subgrid(_to(core, fsi), facet_off, axis=axis)
    what = (f"extract_from_subgrid m {m} axis {axis}, {n_lines} lines, off {facet_off}"
            f"{f', cap {cap}' if cap else ''}")
    expect(core, line_form(m, n_lines, axis == 0, cap), what)
    return _check(_np(got), oracle.extract_from_subgrid(fsi, facet_off, axis=axis), rtol, what)


def finish_subgrid_vs_oracle(core, oracle, dims, sz, sg_offs, masked, seed, n_lines=1, cap=0,
                             rtol=1e-12):
    """1-D (``n_lines`` 1: a vector; more: the lines of an (n_lines, xM) array along axis 1 --
    the kernel a 1-D call runs) or 2-D (xM x xM, both axes), with a mask on every axis when
    ``masked``."""
    rng = numpy.random.default_rng(seed)
    xM = core.xM_size
    if dims == 2:
        summed = pc.rand_c(rng, xM, xM)
        masks = [(rng.random(sz) > 0.3).astype(float) for _ in range(2)] if masked else None
        got = core.finish_subgrid(_to(core, summed), list(sg_offs), sz,
                                  masks=None if masks is None else [_to(core, k) for k in masks])
        # the last pass: axis 0 of the (xM, sz) intermediate, sz adjacent lines
        form = line_form(xM, sz, True)
        ref = oracle.finish_subgrid(summed, list(sg_offs), sz)
        if masks is not None:
            ref = ref * masks[0][:, None] * masks[1][None, :]
    else:
        summed = pc.rand_c(rng, n_lines, xM)
        mask = (rng.random(sz) > 0.3).astype(float) if masked else None
        with capped(core, cap):
            if n_lines == 1:
                got = core.finish_subgrid(_to(core, summed[0]), sg_offs[0], sz,
                                          masks=None if mask is None else [_to(core, mask)])
            else:
                # pylint: disable=protected-access
                got = core._run("swiftly_b200_finish_subgrid", _to(core, summed), sz, 1, None,
                                sg_offs[0], mask=None if mask is None else _to(core, mask))
        form = line_form(xM, n_lines, False, cap)
        ref = numpy.array([oracle.finish_subgrid(line, sg_offs[0], sz) for line in summed])
        if n_lines == 1:
            ref = ref[0]
        if mask is not None:
            ref = ref * mask
    what = (f"finish_subgrid xM {xM} {dims}-D, {n_lines if dims == 1 else xM} lines, sz {sz}, "
            f"offs {list(sg_offs)}{', masked' if masked else ''}{f', cap {cap}' if cap else ''}")
    expect(core, form, what)
    return _check(_np(got), ref, rtol, what)


def prepare_subgrid_vs_oracle(core, oracle, dims, sz, sg_offs, seed, rtol=1e-12):
    rng = numpy.random.default_rng(seed)
    xM = core.xM_size
    if dims == 2:
        sub = pc.rand_c(rng, sz, sz)
        got = core.prepare_subgrid(_to(core, sub), tuple(sg_offs))
        form = line_form(xM, xM, False)  # the last pass: axis 1, xM lines
        ref = oracle.prepare_subgrid(sub, tuple(sg_offs))
    else:
        sub = pc.rand_c(rng, sz)
        got = core.prepare_subgrid(_to(core, sub), sg_offs[0])
        form = line_form(xM, 1, False)
        ref = oracle.prepare_subgrid(sub, sg_offs[0])
    what = f"prepare_subgrid xM {xM} {dims}-D, sz {sz}, offs {list(sg_offs)}"
    expect(core, form, what)
    return _check(_np(got), ref, rtol, what)


def prepare_subgrid_lines_vs_oracle(core, oracle, axis, n_lines, sz, sg_off, seed, cap=0,
                                    rtol=1e-12):
    """prepare_subgrid along one axis of an array of ``n_lines`` lines (the pass the 2-D call
    makes), against the oracle's 1-D transform per line."""
    rng = numpy.random.default_rng(seed)
    xM = core.xM_size
    sub = _lines(rng, axis, n_lines, sz)
    with capped(core, cap):
        # pylint: disable=protected-access
        got = core._run("swiftly_b200_prepare_subgrid", _to(core, sub), xM, axis, None, sg_off)
    what = (f"prepare_subgrid xM {xM} axis {axis}, {n_lines} lines, sz {sz}, off {sg_off}"
            f"{f', cap {cap}' if cap else ''}")
    expect(core, line_form(xM, n_lines, axis == 0, cap), what)
    rows = sub if axis == 1 else sub.T
    ref = numpy.array([oracle.prepare_subgrid(line, sg_off) for line in rows])
    return _check(_np(got), ref if axis == 1 else ref.T, rtol, what)


def subgrid_to_facets_vs_oracle(core, oracle, n_facets, sg_off1, seed, rtol=1e-12):
    """One subgrid's (m, xM) blocks into ``n_facets`` non-zero column accumulators with distinct
    facet offsets (more than 64: two launches) against the oracle's
    extract_from_subgrid(axis 1) -> add_to_facet(axis 1).  Facets share three blocks."""
    rng = numpy.random.default_rng(seed)
    m, xM, yN = core.xM_yN_size, core.xM_size, core.yN_size
    step = core.facet_off_step
    blocks = [pc.rand_c(rng, m, xM) for _ in range(3)]
    accs = [pc.rand_c(rng, m, yN) for _ in range(n_facets)]
    offs = [(f * 7 - 3 * n_facets) * step + (core.N if f % 5 == 4 else 0) for f in range(n_facets)]
    assert len(set(offs)) == n_facets
    d_blocks = [_to(core, b) for b in blocks]
    d_accs = [_to(core, a) for a in accs]
    core.subgrid_to_facets([d_blocks[f % 3] for f in range(n_facets)], d_accs, offs, sg_off1)
    last = n_facets - (n_facets - 1) // 64 * 64  # facets of the last launch
    what = f"subgrid_to_facets m {m}, {n_facets} facets, sg_off1 {sg_off1}"
    expect(core, line_form(m, last * m, False), what)
    worst = 0.0
    for f in range(n_facets):
        ext = oracle.extract_from_subgrid(blocks[f % 3], offs[f], axis=1)
        ref = oracle.add_to_facet(ext, sg_off1, axis=1, out=accs[f].copy())
        worst = max(worst, _check(_np(d_accs[f]), ref, rtol, f"{what}: facet {f}"))
    return worst


def window_copies_vs_oracle(core, oracle, seed, cap=0):
    """extract_from_facet and add_to_facet (into a random accumulator), bitwise: along axis 1,
    along axis 0 with adjacent lines (line-fastest) and along axis 0 with every other column
    (not line-fastest), at subgrid offsets whose window wraps around yN."""
    rng = numpy.random.default_rng(seed)
    m, yN, N = core.xM_yN_size, core.yN_size, core.N
    step = core.subgrid_off_step
    # sc = off yN / N: the window starts at yN/2 - m/2 + sc, so it wraps for sc > m/2 (mod yN)
    offs = [N // 2 + 3 * step, -(N // 2) - 5 * step, 0]
    for k, (axis, n_lines, every) in enumerate([(1, 5, 1), (0, 37, 1), (0, 9, 2)]):
        off = offs[k % len(offs)]
        shape = (n_lines * every, yN) if axis == 1 else (yN, n_lines * every)
        prep = pc.rand_c(rng, *shape)
        view = (slice(None), slice(None, None, every))
        src = prep[view]
        adjacent = axis == 0 and every == 1
        what = (f"extract_from_facet m {m} yN {yN} axis {axis}, {n_lines} lines, every {every},"
                f" off {off}{f', cap {cap}' if cap else ''}")
        cshape = (n_lines, m) if axis == 1 else (m, n_lines)
        # every other column: the output too, so that neither side has unit line stride
        out = None if every == 1 else _to(core, pc.rand_c(rng, m, 2 * n_lines))[view]
        with capped(core, cap):
            got = core.extract_from_facet(_to(core, prep)[view], off, axis=axis, out=out)
        expect(core, window_form(m, n_lines, adjacent, cap), what)
        ref = oracle.extract_from_facet(src, off, axis=axis)
        assert numpy.array_equal(_np(got), ref), what
        contrib = pc.rand_c(rng, *cshape)
        acc0 = pc.rand_c(rng, *shape)
        acc = _to(core, acc0)
        what = what.replace("extract_from_facet", "add_to_facet")
        d_contrib = _to(core, contrib)
        if every != 1:
            d_contrib = _to(core, pc.rand_c(rng, m, 2 * n_lines))[view]
            d_contrib[...] = _to(core, contrib)
        with capped(core, cap):
            core.add_to_facet(d_contrib, off, axis=axis, out=acc[view])
        expect(core, window_form(m, n_lines, adjacent, cap), what)
        ref = acc0.copy()
        oracle.add_to_facet(contrib, off, axis=axis, out=ref[view])
        assert numpy.array_equal(_np(acc), ref), what


def m_plan_vs_oracle(core, oracle, seed, n_facets=67, max_2d=8192):
    """Every m-point primitive of one plan against the oracle: add_to_subgrid and
    extract_from_subgrid along both axes (a partly empty last CTA along axis 0),
    add_to_subgrid_2d (m <= max_2d), subgrid_to_facets with ``n_facets`` facets and the window
    copies.  Returns the worst relative error per op."""
    m = core.xM_yN_size
    offs = facet_offsets(core)
    worst = {}

    def note(op, err):
        worst[op] = max(worst.get(op, 0.0), err)

    k = 0
    for off in offs:
        note("add_to_subgrid", add_to_subgrid_vs_oracle(core, oracle, 1, 3, off, False, seed + k))
        note("add_to_subgrid", add_to_subgrid_vs_oracle(core, oracle, 1, 2, off, True, seed + k + 1))
        note("extract_from_subgrid",
             extract_from_subgrid_vs_oracle(core, oracle, 1, 3, off, seed + k + 2))
        k += 3
    for j, n_lines in enumerate(lpc_line_counts(m)):
        off = offs[j % 3]
        note("add_to_subgrid",
             add_to_subgrid_vs_oracle(core, oracle, 0, n_lines, off, j % 2 == 1, seed + k))
        note("extract_from_subgrid",
             extract_from_subgrid_vs_oracle(core, oracle, 0, n_lines, off, seed + k + 1))
        k += 2
    if m <= max_2d:
        note("add_to_subgrid_2d",
             add_to_subgrid_2d_vs_oracle(core, oracle, offs[1], offs[2], seed + k))
    note("subgrid_to_facets",
         subgrid_to_facets_vs_oracle(core, oracle, n_facets, subgrid_offsets(core)[0], seed + k + 1))
    window_copies_vs_oracle(core, oracle, seed + k + 2)
    return worst


def xm_plan_vs_oracle(core, oracle, xa, seed, max_2d=8192):
    """finish_subgrid and prepare_subgrid of one xM plan against the oracle: 1-D at every size
    of :func:`sizes`, lines along both axes (partly empty last CTA), and 2-D (xM <= max_2d)
    with a mask on each axis."""
    xM = core.xM_size
    sgo = subgrid_offsets(core)
    worst = {}

    def note(op, err):
        worst[op] = max(worst.get(op, 0.0), err)

    k = 0
    for j, sz in enumerate(sizes(core, xa)):
        offs = [sgo[j % 2], sgo[(j + 1) % 2]]
        note("finish_subgrid",
             finish_subgrid_vs_oracle(core, oracle, 1, sz, offs, j % 2 == 0, seed + k))
        note("prepare_subgrid", prepare_subgrid_vs_oracle(core, oracle, 1, sz, offs, seed + k + 1))
        if xM <= max_2d and j in (1, 3):
            note("finish_subgrid",
                 finish_subgrid_vs_oracle(core, oracle, 2, sz, offs, True, seed + k + 2))
            note("prepare_subgrid",
                 prepare_subgrid_vs_oracle(core, oracle, 2, sz, offs, seed + k + 3))
        k += 4
    for j, n_lines in enumerate(lpc_line_counts(xM)):
        sz = sizes(core, xa)[j % 3]
        note("finish_subgrid", finish_subgrid_vs_oracle(
            core, oracle, 1, sz, [sgo[j % 2]], j % 2 == 1, seed + k, n_lines=n_lines))
        for axis in (0, 1):
            note("prepare_subgrid", prepare_subgrid_lines_vs_oracle(
                core, oracle, axis, n_lines, sz, sgo[(j + axis) % 2], seed + k + 1 + axis))
        k += 3
    return worst


def capped_vs_oracle(core, oracle, which, cap, seed, n_lines=37):
    """The grid capped at ``cap`` CTAs: ``n_lines`` lines walk the grid-stride loop.
    ``which`` "m": add_to_subgrid (axis 0 and 1), extract_from_subgrid and the window copies;
    "xM": finish_subgrid and prepare_subgrid."""
    if which == "m":
        off = facet_offsets(core)[1]
        return max(
            add_to_subgrid_vs_oracle(core, oracle, 0, n_lines, off, True, seed, cap=cap),
            add_to_subgrid_vs_oracle(core, oracle, 1, n_lines - 2, off, False, seed + 1, cap=cap),
            extract_from_subgrid_vs_oracle(core, oracle, 0, n_lines, off, seed + 2, cap=cap),
            window_copies_vs_oracle(core, oracle, seed + 3, cap=cap) or 0.0)
    sg = subgrid_offsets(core)
    return max(
        finish_subgrid_vs_oracle(core, oracle, 1, core.xM_size - 1, [sg[0]], True, seed,
                                 n_lines=n_lines, cap=cap),
        prepare_subgrid_lines_vs_oracle(core, oracle, 0, n_lines, core.xM_size // 2 + 1, sg[1],
                                        seed + 1, cap=cap),
        prepare_subgrid_lines_vs_oracle(core, oracle, 1, n_lines - 3, core.xM_size - 1, sg[0],
                                        seed + 2, cap=cap))


# ---------------------------------------------------------------------- host / device staging
def _sentinel_view(core, host, form, n_lines, size):
    """An (n_lines, size) output view inside a NaN-filled array, in one of ``stage_in``'s two
    forms: "slice" (a column slice of a wider array: unit element stride, line stride > size)
    or "transposed" (a transposed view: unit line stride).  Returns (base, view)."""
    if form == "slice":
        shape, sl = (n_lines, size + 7), (slice(None), slice(3, 3 + size))
    else:
        shape, sl = (size, n_lines + 5), (slice(None), slice(2, 2 + n_lines))
    if host:
        base = numpy.full(shape, complex(numpy.nan, numpy.nan))
    else:
        base = torch.full(shape, complex(numpy.nan, numpy.nan), dtype=torch.complex128,
                          device=lc._dev(core))  # pylint: disable=protected-access
    view = base[sl]
    return base, (view if form == "slice" else view.T)


def _outside_untouched(base, view_shape, form):
    b = _np(base)
    inside = numpy.zeros(b.shape, dtype=bool)
    if form == "slice":
        inside[:, 3:3 + view_shape[1]] = True
    else:
        inside[:, 2:2 + view_shape[0]] = True
    return bool(numpy.isnan(b[~inside]).all())


def staging_vs_oracle(core, oracle, host, seed, rtol=1e-12):
    """One case per primitive (add_to_subgrid, extract_from_subgrid, finish_subgrid with masks,
    prepare_subgrid, extract_from_facet, add_to_facet) with numpy arrays (``host``) or device
    tensors, writing into output views of both stage_in forms inside a NaN-filled array: the
    result matches the oracle and every sample outside the view is still NaN."""
    rng = numpy.random.default_rng(seed)
    m, xM, yN = core.xM_yN_size, core.xM_size, core.yN_size
    f_off, s_off = facet_offsets(core)[1], subgrid_offsets(core)[0]
    sz = xM - 3
    put = (lambda a: a) if host else (lambda a: _to(core, a))
    L = 6
    for form in ("slice", "transposed"):
        cases = []
        contrib = pc.rand_c(rng, L, m)
        acc0 = pc.rand_c(rng, L, xM)
        cases.append(("add_to_subgrid", (L, xM), acc0,
                      lambda o, c=contrib: core.add_to_subgrid(put(c), f_off, axis=1, out=o),
                      lambda c=contrib, a=acc0: oracle.add_to_subgrid(c, f_off, axis=1,
                                                                      out=a.copy())))
        fsi = pc.rand_c(rng, L, xM)
        cases.append(("extract_from_subgrid", (L, m), None,
                      lambda o, f=fsi: core.extract_from_subgrid(put(f), f_off, axis=1, out=o),
                      lambda f=fsi: oracle.extract_from_subgrid(f, f_off, axis=1)))
        summed = pc.rand_c(rng, xM, xM)
        masks = [(rng.random(sz) > 0.3).astype(float) for _ in range(2)]
        cases.append(("finish_subgrid", (sz, sz), None,
                      lambda o, s=summed, k=masks: core.finish_subgrid(
                          put(s), [s_off, -s_off], sz, out=o, masks=[put(x) for x in k]),
                      lambda s=summed, k=masks: oracle.finish_subgrid(s, [s_off, -s_off], sz)
                      * k[0][:, None] * k[1][None, :]))
        sub = pc.rand_c(rng, sz, sz)
        cases.append(("prepare_subgrid", (xM, xM), None,
                      lambda o, s=sub: core.prepare_subgrid(put(s), (s_off, -s_off), out=o),
                      lambda s=sub: oracle.prepare_subgrid(s, (s_off, -s_off))))
        prep = pc.rand_c(rng, L, yN)
        cases.append(("extract_from_facet", (L, m), None,
                      lambda o, p=prep: core.extract_from_facet(put(p), s_off, axis=1, out=o),
                      lambda p=prep: oracle.extract_from_facet(p, s_off, axis=1)))
        c2 = pc.rand_c(rng, L, m)
        accf0 = pc.rand_c(rng, L, yN)
        cases.append(("add_to_facet", (L, yN), accf0,
                      lambda o, c=c2: core.add_to_facet(put(c), s_off, axis=1, out=o),
                      lambda c=c2, a=accf0: oracle.add_to_facet(c, s_off, axis=1, out=a.copy())))
        for name, shape, init, run, ref in cases:
            what = f"{name} m {m} xM {xM}, {'host' if host else 'device'} {form} output view"
            base, view = _sentinel_view(core, host, form, *shape)
            if init is not None:
                view[...] = init if host else _to(core, init)
            got = run(view)
            assert got is view or _np(got).shape == shape, what
            want = ref()
            if name in ("extract_from_facet", "add_to_facet"):
                assert numpy.array_equal(_np(view), want), what
            else:
                _check(_np(view), want, rtol, what)
            assert _outside_untouched(base, shape, form), f"{what}: wrote outside the view"


# ---------------------------------------------------------------------- drop-in adapter
def sdp_func_adapter_vs_oracle(swiftly, oracle, yB, xA, lines=9, rtol=1e-12):
    """The ska_sdp_func-shaped adapter ``swiftly`` (``sdp_func_compat.Swiftly``: last-axis
    transforms on strided views, in-place prepare_subgrid) called the way the reference's
    SwiftlyCoreFunc calls it (core.py:577-630, 684-929), against the oracle.  ``lines``: the
    number of facet columns the chain along axis 0 transforms."""
    from oracle.swiftly_oracle import pad_mid  # pylint: disable=import-outside-toplevel

    N, xM, yN = oracle.N, oracle.xM_size, oracle.yN_size
    m = oracle.xM_yN_size
    rng = numpy.random.default_rng(31)
    f_off, s_off = 3 * oracle.facet_off_step, -3 * oracle.subgrid_off_step
    assert (N, yN, xM) == (swiftly.N, swiftly.yN_size, swiftly.xM_size)
    facet = pc.rand_c(rng, yB, lines)
    # axis 0 through transposed views
    out = numpy.empty((yN, lines), dtype=complex)
    swiftly.prepare_facet(facet.T, out.T, f_off)
    pc.close(out, oracle.prepare_facet(facet, f_off, axis=0), rtol, what="compat prepare_facet")
    contrib = numpy.empty((m, lines), dtype=complex)
    swiftly.extract_from_facet(out.T, contrib.T, s_off)
    assert numpy.array_equal(contrib, oracle.extract_from_facet(out, s_off, axis=0))
    acc = numpy.zeros((xM, lines), dtype=complex)
    swiftly.add_to_subgrid(contrib.T, acc.T, f_off)
    pc.close(acc, oracle.add_to_subgrid(contrib, f_off, axis=0), rtol,
             what="compat add_to_subgrid")
    # 2-D accumulate and finish like SwiftlyCoreFunc.finish_subgrid (core.py:803-812)
    c2 = pc.rand_c(rng, m, m)
    acc2 = numpy.zeros((xM, xM), dtype=complex)
    swiftly.add_to_subgrid_2d(c2, acc2, f_off, -f_off)
    oacc2 = oracle.add_to_subgrid(oracle.add_to_subgrid(c2, f_off, axis=0), -f_off, axis=1)
    pc.close(acc2, oacc2, rtol, what="compat add_to_subgrid_2d")
    out1 = numpy.empty((xM, xA), dtype=complex)
    swiftly.finish_subgrid(acc2, out1, s_off)
    sg = numpy.empty((xA, xA), dtype=complex)
    swiftly.finish_subgrid(out1.T, sg.T, -s_off)
    pc.close(sg, oracle.finish_subgrid(oacc2, [-s_off, s_off], xA), rtol,
             what="compat finish_subgrid")
    # in-place prepare_subgrid on the padded subgrid (core.py:842-853)
    sub = pc.rand_c(rng, xA, xA)
    padded = numpy.ascontiguousarray(pad_mid(pad_mid(sub, xM, 0), xM, 1))
    swiftly.prepare_subgrid_inplace_2d(padded, s_off, -s_off)
    opsg = oracle.prepare_subgrid(sub, (s_off, -s_off))
    pc.close(padded, opsg, rtol, what="compat prepare_subgrid")
    ext = numpy.empty((xM, m), dtype=complex)
    swiftly.extract_from_subgrid(padded, ext, f_off)
    pc.close(ext, oracle.extract_from_subgrid(padded, f_off, axis=1), rtol, what="compat extract")
    accf = numpy.zeros((xM, yN), dtype=complex)
    swiftly.add_to_facet(ext, accf, s_off)
    assert numpy.array_equal(accf, oracle.add_to_facet(ext, s_off, axis=1))
    fin = numpy.empty((xM, yB), dtype=complex)
    swiftly.finish_facet(accf, fin, f_off)
    pc.close(fin, oracle.finish_facet(accf, f_off, yB, axis=1), rtol, what="compat finish_facet")


# ---------------------------------------------------------------------- extended precision
# Bound of the spot checks in units of EPS * log2(n) of the line's RMS (n = m or xM), as for
# the facet lines (length_cases.SPOT_BOUND); the split-F plans, F = 7 included, need no bound of
# their own.  Observed with the test seeds (the worse of the two primitives per plan):
#   H100 80GB HBM3 (700 W), 2 lines per check: m direct 0.26 .. 0.68, m split-F 0.24 .. 0.28,
#     xM direct 0.30 .. 0.44, xM split-F 0.21 .. 0.30;
#   emulated kernels (host build without fused multiply-adds), 1 line per check: m direct
#     0.24 .. 0.59, m split-F 0.26 .. 0.34, xM direct 0.21 .. 0.44, xM split-F 0.21 .. 0.25.
# Worst error against the oracle on the H100, relative to the largest sample: 9.1e-17 .. 1.03e-15
# for the m plans, 3.9e-16 .. 1.69e-15 for the xM plans.
SPOT_BOUND = 1.5


def _sub_transforms(n):
    return lc.sub_transforms(lc.line_kernel(n))


def _centred_bins(n, rng):
    """Centred positions (array indices) of the natural-order bins of ``lc.spot_bins``."""
    M, F = _sub_transforms(n)
    return [(b + n // 2) % n for b in lc.spot_bins(M, F, n, rng)]


def _units(worst, n):
    return worst / (lc.EPS * numpy.log2(n))


def spot_check_add_to_subgrid(core, seed, n_lines=2):
    """add_to_subgrid (axis 1, fresh output): the m-point forward transform at the spectrum
    bins of ``spot_bins``, weighted with ``Fn`` and placed in the xM line; the ``Fn`` factor of
    each sample is divided out.  Units EPS * log2(m) of the spectrum's RMS."""
    rng = numpy.random.default_rng(seed)
    m, xM = core.xM_yN_size, core.xM_size
    off = 3 * core.facet_off_step
    sf = off * xM // core.N
    contrib = pc.rand_c(rng, n_lines, m)
    got = _np(core.add_to_subgrid(_to(core, contrib), off, axis=1))
    spec_pos = _centred_bins(m, rng)
    u = [(s - sf) % m for s in spec_pos]
    dest = [(xM // 2 - m // 2 + uu + sf) % xM for uu in u]
    fn = numpy.asarray(core._Fn, dtype=numpy.longdouble)[u]  # pylint: disable=protected-access
    worst = 0.0
    for line in range(n_lines):
        z = contrib[line].astype(numpy.clongdouble)
        exact = lc.centred_dft(z, spec_pos, -1)
        rms = numpy.sqrt((numpy.abs(z) ** 2).sum())
        err = numpy.abs(got[line, dest].astype(numpy.clongdouble) / fn - exact).max() / rms
        worst = max(worst, float(err))
    return _units(worst, m)


def spot_check_extract_from_subgrid(core, seed, n_lines=2):
    """extract_from_subgrid (axis 1): the m-point inverse transform of the Fn-weighted window
    at the bins of ``spot_bins``.  Units EPS * log2(m) of the output's RMS."""
    rng = numpy.random.default_rng(seed)
    m, xM = core.xM_yN_size, core.xM_size
    off = -5 * core.facet_off_step
    sf = off * xM // core.N
    fsi = pc.rand_c(rng, n_lines, xM)
    got = _np(core.extract_from_subgrid(_to(core, fsi), off, axis=1))
    pos = _centred_bins(m, rng)
    u = numpy.arange(m)
    fn = numpy.asarray(core._Fn, dtype=numpy.longdouble)  # pylint: disable=protected-access
    worst = 0.0
    for line in range(n_lines):
        w = numpy.zeros(m, dtype=numpy.clongdouble)
        w[(u + sf) % m] = fn * fsi[line, (xM // 2 - m // 2 + u + sf) % xM].astype(numpy.clongdouble)
        exact = lc.centred_dft(w, pos, +1) / m
        rms = numpy.sqrt((numpy.abs(w) ** 2).sum()) / m
        err = numpy.abs(got[line, pos].astype(numpy.clongdouble) - exact).max() / rms
        worst = max(worst, float(err))
    return _units(worst, m)


def spot_check_finish_subgrid(core, seed, n_lines=2):
    """finish_subgrid (1-D per line, sz = xM - 1): the xM-point inverse transform at the bins of
    ``spot_bins`` that fall in the subgrid.  Units EPS * log2(xM) of the output's RMS."""
    rng = numpy.random.default_rng(seed)
    xM = core.xM_size
    sz, off = xM - 1, 2 * core.subgrid_off_step
    start = (xM // 2 - sz // 2 + off) % xM
    pos = [c for c in _centred_bins(xM, rng) if (c - start) % xM < sz]
    r = [(c - start) % xM for c in pos]
    worst = 0.0
    for line in range(n_lines):
        z = pc.rand_c(rng, xM)
        got = _np(core.finish_subgrid(_to(core, z), off, sz))
        exact = lc.centred_dft(z.astype(numpy.clongdouble), pos, +1) / xM
        rms = numpy.sqrt((numpy.abs(z.astype(numpy.clongdouble)) ** 2).sum()) / xM
        err = numpy.abs(got[r].astype(numpy.clongdouble) - exact).max() / rms
        worst = max(worst, float(err))
    return _units(worst, xM)


def spot_check_prepare_subgrid(core, seed, n_lines=2):
    """prepare_subgrid (1-D per line, sz = xM - 1): the xM-point forward transform of the padded,
    rolled subgrid at the bins of ``spot_bins``.  Units EPS * log2(xM) of the output's RMS."""
    rng = numpy.random.default_rng(seed)
    xM = core.xM_size
    sz, off = xM - 1, -3 * core.subgrid_off_step
    dest = (xM // 2 - sz // 2 + off + numpy.arange(sz)) % xM
    pos = _centred_bins(xM, rng)
    worst = 0.0
    for line in range(n_lines):
        sub = pc.rand_c(rng, sz)
        got = _np(core.prepare_subgrid(_to(core, sub), off))
        z = numpy.zeros(xM, dtype=numpy.clongdouble)
        z[dest] = sub.astype(numpy.clongdouble)
        exact = lc.centred_dft(z, pos, -1)
        rms = numpy.sqrt((numpy.abs(z) ** 2).sum())
        err = numpy.abs(got[pos].astype(numpy.clongdouble) - exact).max() / rms
        worst = max(worst, float(err))
    return _units(worst, xM)


def spot_check_m(core, seed, n_lines=2):
    return max(spot_check_add_to_subgrid(core, seed, n_lines),
               spot_check_extract_from_subgrid(core, seed + 1, n_lines))


def spot_check_xm(core, seed, n_lines=2):
    return max(spot_check_finish_subgrid(core, seed, n_lines),
               spot_check_prepare_subgrid(core, seed + 1, n_lines))


def geometry_entry(name):
    p = SWIFT_CONFIGS[name]
    return (p["W"], p["N"], p["xM_size"], p["yN_size"])


def family_geometries():
    """(m, xM) -> {"gpu": (geometry, yB, xA), "emu": (geometry, yB, xA)} of every catalogue
    family: the smallest catalogue entry (pair_cases.core_plan) with yB = yN / 2, and the small
    plan of the pair (pair_cases.small_plan) with catalogue_cases.SMALL's yB or yN / 2; both
    with the entry's xA (the small plan has the same xM).  (At the entry's own yB / yN = 0.875
    of 16k[.75]-n2k-1k, Fb reaches a size at which finish_facet of the same input differs from
    the oracle by 4e-11 of the largest sample: the window's conditioning, which
    catalogue_cases.SMALL and test_gpu_subgrid_pairs.config also note.)"""
    out = {}
    for pair in sorted(prc.CATALOGUE):
        p = SWIFT_CONFIGS[prc.CATALOGUE[pair][1]]
        small = prc.small_plan(pair)
        yb = cc.SMALL[pair][2] if pair in cc.SMALL else small[3] // 2
        out[pair] = {"gpu": (prc.core_plan(pair), p["yN_size"] // 2, p["xA_size"]),
                     "emu": (small, yb, p["xA_size"])}
    return out
