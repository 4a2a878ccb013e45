"""
Cases of the fused subgrid kernels at every (m, xM) pair of the library, shared by the emulated
and the GPU tests: ``sum_finish_axis`` (K3 / K4 of the forward step) and
``split_subgrid_axis`` (K4T / K3T of the backward step) against the oracle, each case asserting
the kernel form it was written for (``swiftly_b200_debug_last_launch``), and an
extended-precision spot check of ``sum_finish_axis``.

``dispatch_subgrid_axis.cu`` picks the form per pair and per call: the two-group kernel
(``SubgridAxisKernelPP``) for strided lines at the power-of-two pairs whose thread groups are
whole warps and fit shared memory, otherwise the round-1 kernel (``SubgridAxisKernel``) with two
lines per CTA for adjacent lines where two fit.  The two-group kernel stages a finished line for
the TMA engine when ``ceil(sz / box) * box`` samples (box = min(sz, 256)) fit its work area.
"""

import contextlib
import ctypes

import numpy
import torch

from oracle.swiftly_oracle import OracleCore
from ska_sdp_distributed_fourier_transform_b200.swift_configs import (
    FUSED_FORWARD_PAIRS,
    SWIFT_CONFIGS,
)
from tests import catalogue_cases as cc
from tests import length_cases as lc
from tests import parity_cases as pc
from tests import subgrid_round_cases as rc

# kernels and output paths of swiftly_b200_debug_last_launch
ROUND1, TWO_GROUP, SPLIT = 1, 2, 3
DIRECT, TMA, TMA_PER_GROUP = 0, 1, 2


def _catalogue_pairs():
    """(m, xM) -> (catalogue entries, smallest entry by (N, yN, name))."""
    names = {}
    for name, p in SWIFT_CONFIGS.items():
        names.setdefault((p["xM_size"] * p["yN_size"] // p["N"], p["xM_size"]), []).append(name)
    return {pair: (len(v), min(v, key=lambda n: (SWIFT_CONFIGS[n]["N"],
                                                 SWIFT_CONFIGS[n]["yN_size"], n)))
            for pair, v in names.items()}


CATALOGUE = _catalogue_pairs()
# pairs of SW_SG_PAIRS no catalogue entry uses
LIBRARY_ONLY = sorted(set(FUSED_FORWARD_PAIRS) - set(CATALOGUE))
ALL_PAIRS = sorted(FUSED_FORWARD_PAIRS)

# Per pair, pinned: the forward form on strided lines and on adjacent lines (kernel, lines per
# CTA), the split kernel's lines per CTA on adjacent lines (one on strided lines), CONC and the
# largest sz that stages through the TMA engine (two-group pairs only).
FORMS = {
    #  (m, xM):       strided           adjacent      split  CONC  TMA sz
    (32, 64):     ((ROUND1, 1),    (ROUND1, 2),      2,    2,   None),
    (32, 128):    ((ROUND1, 1),    (ROUND1, 2),      2,    4,   None),
    (64, 128):    ((ROUND1, 1),    (ROUND1, 2),      2,    2,   None),
    (64, 256):    ((ROUND1, 1),    (ROUND1, 2),      2,    4,   None),
    (128, 256):   ((ROUND1, 1),    (ROUND1, 2),      2,    2,   None),
    (128, 384):   ((ROUND1, 1),    (ROUND1, 2),      2,    3,   None),
    (128, 512):   ((TWO_GROUP, 2), (ROUND1, 2),      2,    4,   256),
    (128, 1024):  ((ROUND1, 1),    (ROUND1, 2),      2,    8,   None),
    (160, 320):   ((ROUND1, 1),    (ROUND1, 2),      2,    2,   None),
    (192, 384):   ((ROUND1, 1),    (ROUND1, 2),      2,    2,   None),
    (224, 448):   ((ROUND1, 1),    (ROUND1, 2),      2,    2,   None),
    (256, 256):   ((ROUND1, 1),    (ROUND1, 2),      2,    1,   None),
    (256, 512):   ((TWO_GROUP, 2), (ROUND1, 2),      2,    2,   256),
    (256, 1024):  ((TWO_GROUP, 2), (ROUND1, 2),      2,    4,   512),
    (512, 1024):  ((TWO_GROUP, 2), (ROUND1, 2),      2,    2,   512),
    (512, 2048):  ((TWO_GROUP, 2), (ROUND1, 2),      2,    4,   1024),
    (1024, 2048): ((TWO_GROUP, 2), (ROUND1, 2),      2,    2,   1024),
    (1024, 4096): ((TWO_GROUP, 2), (ROUND1, 2),      2,    4,   2048),
    (2048, 4096): ((TWO_GROUP, 2), (ROUND1, 2),      2,    2,   2048),
    (2048, 8192): ((ROUND1, 1),    (ROUND1, 1),      1,    4,   None),
}
# two-group pairs whose transforms are whole warps: empty transform slots are skipped there
# (sg_variant 25 transforms zeros instead)
SKIP_PAIRS = [p for p in ALL_PAIRS if FORMS[p][0][0] == TWO_GROUP and p[0] // 16 % 32 == 0]


def pair_id(pair):
    return cc.pair_id(pair)


def core_plan(pair):
    """(W, N, xM, yN) of the smallest catalogue entry, or for a library-only pair N = 2 xM,
    yN = 2 m."""
    if pair in CATALOGUE:
        p = SWIFT_CONFIGS[CATALOGUE[pair][1]]
        return (p["W"], p["N"], p["xM_size"], p["yN_size"])
    m, xM = pair
    return (13.5625, 2 * xM, xM, 2 * m)


def small_plan(pair):
    """(W, N, xM, yN) of a small plan with the pair (the emulated tests): the kernels see m and
    xM only, the plan size sets the oracle's cost."""
    if pair in cc.SMALL:
        W, N, _, yN, _, xM = cc.SMALL[pair]
        return (W, N, xM, yN)
    m, xM = pair
    return (13.5625, 2 * xM, xM, 2 * m)


# ---------------------------------------------------------------------- test hooks
def last_launch(core):
    """(kernel, lines per CTA, output path, grid) of the last fused subgrid launch."""
    lib = core._lib
    lib.swiftly_b200_debug_last_launch.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int)]
    out = (ctypes.c_int * 4)()
    lib.swiftly_b200_debug_last_launch(core._plan, out)
    return tuple(out)


@contextlib.contextmanager
def max_blocks(core, n):
    """Cap the grid of the fused subgrid kernels (0: no cap)."""
    core._lib.swiftly_b200_debug_max_blocks.argtypes = [ctypes.c_void_p, ctypes.c_int]
    core._lib.swiftly_b200_debug_max_blocks(core._plan, int(n))
    try:
        yield
    finally:
        core._lib.swiftly_b200_debug_max_blocks(core._plan, 0)


@contextlib.contextmanager
def variant(core, v):
    rc.set_variant(core, v)
    try:
        yield
    finally:
        rc.set_variant(core, 0)


def expect_form(core, kernel, lines, out_path=None, grid=None, what=""):
    got = last_launch(core)
    want = (kernel, lines,
            got[2] if out_path is None else out_path, got[3] if grid is None else grid)
    assert got == want, f"{what}: launched {got}, expected {want}"
    return got


def forward_form(pair, adjacent):
    return FORMS[pair][1 if adjacent else 0]


# ---------------------------------------------------------------------- forward (K3 / K4)
def _view(core, a, axis, adjacent):
    """Lines-first array ``a`` as a device tensor with the transformed axis ``axis``: strided
    lines are stored line after line, adjacent lines sample after sample (unit line stride)."""
    dev = rc.device(core)
    if adjacent:
        t = torch.from_numpy(numpy.ascontiguousarray(a.T)).to(dev)  # (samples, lines)
        return t if axis == 0 else t.T
    t = torch.from_numpy(numpy.ascontiguousarray(a)).to(dev)  # (lines, samples)
    return t if axis == 1 else t.T


def _out(core, groups, lines, sz, axis, adjacent):
    dev = rc.device(core)
    shape = (groups, sz, lines) if adjacent else (groups, lines, sz)
    t = torch.empty(shape, dtype=torch.complex128, device=dev)
    return t if (axis == 0) == adjacent else t.transpose(1, 2)


def _lines_first(t, axis):
    a = t.cpu().numpy()
    return a if axis == 1 else a.T


def sum_finish_job(core, groups, sz, axis, *, mode="single", adjacent=False, lines=3,
                   sg_offs=None, masked=False, contrib_sized=False, seed=0, rtol=1e-12,
                   what=""):
    """One ``sum_finish_axis`` job against the oracle.

    :param groups: per group the facet offsets in units of yN / 2 (None: a group without
        sources); ``mode`` "single" takes one group through ``sum_finish_axis``, "grouped",
        "batched" and "scattered" go through ``sum_finish_axis_grouped``
    :param sg_offs: subgrid offset per group (grouped: the first one for all)
    Returns the outputs (lines-first numpy arrays, one per group) and the worst error relative
    to the largest reference sample.
    """
    oracle = oracle_of(core)
    rng = numpy.random.default_rng(seed)
    size = core.xM_yN_size if contrib_sized else core.yN_size
    ng = len(groups)
    if sg_offs is None:
        sg_offs = [(2 * g - 3) * core.subgrid_off_step for g in range(ng)]
    if mode in ("single", "grouped"):
        sg_offs = [sg_offs[0]] * ng
    offs = [[k * (core.yN_size // 2) for k in (grp or [])] for grp in groups]
    srcs = [[pc.rand_c(rng, lines, size) for _ in o] for o in offs]
    masks = [(rng.random(sz) > 0.3).astype(float) if masked else None for _ in range(ng)]
    if mode in ("single", "grouped"):
        masks = [masks[0]] * ng
    dev_groups = [[(_view(core, s, axis, adjacent), o) for s, o in zip(ss, oo)]
                  for ss, oo in zip(srcs, offs)]
    t_masks = [None if mk is None else torch.from_numpy(mk).to(rc.device(core)) for mk in masks]
    if mode == "single":
        assert ng == 1
        out = _out(core, 1, lines, sz, axis, adjacent)[0]
        core.sum_finish_axis(dev_groups[0], out, axis=axis, subgrid_off=sg_offs[0],
                             mask=t_masks[0])
        outs = [out]
    elif mode == "grouped":
        out = _out(core, ng, lines, sz, axis, adjacent)
        core.sum_finish_axis_grouped(dev_groups, out, axis=axis, subgrid_off=sg_offs[0],
                                     mask=t_masks[0])
        outs = list(out)
    elif mode == "batched":
        out = _out(core, ng, lines, sz, axis, adjacent)
        core.sum_finish_axis_grouped(dev_groups, out, axis=axis, subgrid_off=list(sg_offs),
                                     mask=t_masks)
        outs = list(out)
    else:
        outs = [_out(core, 1, lines, sz, axis, adjacent)[0] for _ in range(ng)]
        core.sum_finish_axis_grouped(dev_groups, outs, axis=axis, subgrid_off=list(sg_offs),
                                     mask=t_masks)
    got = [_lines_first(o, axis) for o in outs]
    worst = 0.0
    for g in range(ng):
        ref = rc.reference(oracle, srcs[g], offs[g], sg_offs[g], sz, 1, contrib_sized, lines,
                           mask=masks[g])
        pc.close(got[g], ref, rtol=rtol, what=f"{what} group {g}")
        scale = max(numpy.abs(ref).max(), 1e-300)
        worst = max(worst, float(numpy.abs(got[g] - ref).max() / scale))
    return got, worst


_oracles = {}


def oracle_of(core):
    key = (core.W, core.N, core.xM_size, core.yN_size)
    if key not in _oracles:
        _oracles.clear()
        _oracles[key] = OracleCore(*key)
    return _oracles[key]


def tma_sizes(pair):
    """sz at the TMA threshold, threshold - 37 (a partial last box where the threshold is
    512 or more), 200 (one box narrower than 256) and threshold + 1 (direct stores)."""
    t = FORMS[pair][4]
    return [(t, TMA), (t - 37, TMA), (200, TMA), (t + 1, DIRECT)]


# ---------------------------------------------------------------------- extended precision
def spot_positions(sz, rng, n_random=4):
    pos = {0, 1, sz // 2 - 1, sz // 2, sz - 2, sz - 1}
    pos |= {int(p) for p in rng.integers(0, sz, n_random)}
    return sorted(p for p in pos if 0 <= p < sz)


def exact_sum_finish(core, line_srcs, facet_offs, sg_off, sz, positions, mask=None):
    """``sum_finish_axis`` of ONE line in ``numpy.longdouble`` at the output samples
    ``positions``: the window gather of every prepared facet line, its m-point centred DFT,
    the roll by the facet offset and the ``Fn`` weight (the core's double table, promoted), the
    sum in the xM accumulator, then the inverse xM-point centred DFT at the chosen samples and
    ``1 / xM``.  Returns (values, RMS of the exact output line)."""
    m, xM, N = core.xM_yN_size, core.xM_size, core.N
    oracle = oracle_of(core)
    fn = numpy.asarray(core._Fn, dtype=numpy.longdouble)
    acc = numpy.zeros(xM, dtype=numpy.clongdouble)
    u = numpy.arange(m)
    win = oracle._facet_window(sg_off)
    for s, off in zip(line_srcs, facet_offs):
        c = s[win] if len(s) != m else s
        spec = lc.centred_dft(numpy.asarray(c, dtype=complex), range(m), -1)
        sf = off * xM // N
        acc[(xM // 2 - m // 2 + u + sf) % xM] += fn * spec[(u + sf) % m]
    src = (xM // 2 - sz // 2 + sg_off + numpy.asarray(positions)) % xM
    vals = lc.centred_dft(acc, src, +1) / xM
    if mask is not None:
        vals = vals * numpy.asarray(mask, dtype=numpy.longdouble)[positions]
    rms = numpy.sqrt((numpy.abs(acc) ** 2).sum()) / xM  # Parseval
    return vals, rms


def spot_check_sum_finish(core, facet_steps, sz, seed, lines=2, adjacent=False):
    """Two lines of ``sum_finish_axis`` (axis 1) at the positions of :func:`spot_positions`
    against :func:`exact_sum_finish`.  Returns the worst ``|got - exact|`` relative to the RMS
    of the exact output line, in units of ``EPS * (log2 m + log2 xM)``."""
    rng = numpy.random.default_rng(seed)
    m, xM, yN = core.xM_yN_size, core.xM_size, core.yN_size
    offs = [k * (yN // 2) for k in facet_steps]
    srcs = [pc.rand_c(rng, lines, yN) for _ in offs]
    sg_off = 3 * core.subgrid_off_step
    out = _out(core, 1, lines, sz, 1, adjacent)[0]
    core.sum_finish_axis([(_view(core, s, 1, adjacent), o) for s, o in zip(srcs, offs)], out,
                         axis=1, subgrid_off=sg_off)
    got = _lines_first(out, 1)
    pos = spot_positions(sz, rng)
    worst = 0.0
    for line in range(lines):
        exact, rms = exact_sum_finish(core, [s[line] for s in srcs], offs, sg_off, sz, pos)
        err = numpy.abs(got[line, pos].astype(numpy.clongdouble) - exact).max() / rms
        worst = max(worst, float(err))
    return worst / (lc.EPS * (numpy.log2(m) + numpy.log2(xM)))


# Bound of the spot check, in units of EPS * (log2 m + log2 xM) of the line RMS (see the GPU and
# emulated tests for the ratios observed)
SPOT_BOUND = 1.5


# ---------------------------------------------------------------------- cases
def _facet_far(core):
    """Facet offsets (units of yN / 2) below zero and at or above N."""
    return [-3, 0, 2 * core.N // core.yN_size + 1]


def _sg_far(core):
    """Subgrid offsets below zero and at or above N."""
    return [-5 * core.subgrid_off_step, core.N + 3 * core.subgrid_off_step]


def case_layouts(core, pair, axis, adjacent, lines=3, seed=0):
    """Every layout of subgrid_round_cases.LAYOUTS in the pair's strided / adjacent form; on
    strided lines of a two-group pair at the TMA threshold, elsewhere at xM - 3 (direct)."""
    kernel, lpc = forward_form(pair, adjacent)
    tma = FORMS[pair][4] if kernel == TWO_GROUP else None
    sz = tma or core.xM_size - 3
    worst = 0.0
    for k, layout in enumerate(sorted(rc.LAYOUTS)):
        what = f"{pair} layout {layout} axis {axis} adjacent {adjacent}"
        _, err = sum_finish_job(core, [rc.LAYOUTS[layout]], sz, axis, adjacent=adjacent,
                                lines=lines, contrib_sized=axis == 0, seed=seed + k, what=what)
        expect_form(core, kernel, lpc, TMA if tma else DIRECT, what=what)
        worst = max(worst, err)
    return worst


def case_sizes(core, pair, seed=0, lines=3):
    """Sizes around the TMA threshold (two-group pairs) with masks, facet and subgrid offsets
    below zero and at or above N; round-1 pairs: odd sizes, direct stores."""
    kernel, lpc = forward_form(pair, False)
    if kernel == TWO_GROUP:
        sizes = tma_sizes(pair)
    else:
        sizes = [(core.xM_size - 3, DIRECT), (core.xM_size // 2 + 1, DIRECT)]
    worst = 0.0
    for k, (sz, path) in enumerate(sizes):
        for j, sg in enumerate(_sg_far(core)):
            what = f"{pair} sz {sz} sg_off {sg}"
            _, err = sum_finish_job(core, [_facet_far(core)], sz, 1, lines=lines, sg_offs=[sg],
                                    masked=True, seed=seed + 2 * k + j, what=what)
            expect_form(core, kernel, lpc, path, what=what)
            worst = max(worst, err)
    return worst


def entry_sizes(pair, core):
    if FORMS[pair][0][0] == TWO_GROUP:
        return [(FORMS[pair][4], True), (FORMS[pair][4] + 1, False)]
    return [(core.xM_size // 2 + 1, False)]


def case_entry_points(core, pair, mode, seed=0, lines=3):
    """grouped / batched / scattered with groups of different round counts (and an empty
    group), at a TMA size and a direct size: scattered outputs take one tensor map per group."""
    kernel, lpc = forward_form(pair, False)
    layouts = ["5_three_plus_two", "1", None, "3_disjoint"]
    groups = [rc.LAYOUTS[lay] if lay else None for lay in layouts]
    worst = 0.0
    for k, (sz, tma) in enumerate(entry_sizes(pair, core)):
        path = (TMA_PER_GROUP if mode == "scattered" else TMA) if tma else DIRECT
        what = f"{pair} {mode} sz {sz}"
        _, err = sum_finish_job(core, groups, sz, 1, mode=mode, lines=lines, masked=True,
                                sg_offs=[(3 * g - 4) * core.subgrid_off_step for g in range(4)],
                                seed=seed + k, what=what)
        expect_form(core, kernel, lpc, path, what=what)
        worst = max(worst, err)
    return worst


def case_many_rounds(core, pair, seed=0, lines=3):
    """64 // CONC + 3 clashing sources: more rounds than one launch carries, so the library
    cuts the job and the later launch ADDS its finished lines to the output."""
    kernel, lpc = forward_form(pair, False)
    n = 64 // FORMS[pair][3] + 3
    what = f"{pair} {n} clashing sources"
    _, err = sum_finish_job(core, [[0] * n], core.xM_size // 2, 1, lines=lines, masked=True,
                            seed=seed, what=what)
    expect_form(core, kernel, lpc, DIRECT, what=what)
    return err


def case_capped_grid(core, pair, cap, seed=0, lines=5):
    """Four groups with the grid capped at ``cap`` CTAs: every CTA walks several lines (pairs)
    and groups."""
    kernel, lpc = forward_form(pair, False)
    groups = [rc.LAYOUTS["8_tiled"], rc.LAYOUTS["1"], None, rc.LAYOUTS["5_three_plus_two"]]
    sz = FORMS[pair][4] or core.xM_size - 3
    what = f"{pair} grid capped at {cap}"
    with max_blocks(core, cap):
        _, err = sum_finish_job(core, groups, sz, 1, mode="grouped", lines=lines, seed=seed,
                                what=what)
    expect_form(core, kernel, lpc, grid=cap, what=what)
    return err


def case_variant_bitwise(core, pair, v, seed=0, lines=3):
    """sg_variant ``v`` (5: direct stores; 25: empty transform slots transform zeros) gives the
    same bits as the default, on every layout (and a TMA size for 5)."""
    sz = FORMS[pair][4]
    for k, layout in enumerate(sorted(rc.LAYOUTS)):
        what = f"{pair} layout {layout}"
        new, _ = sum_finish_job(core, [rc.LAYOUTS[layout]], sz, 1, lines=lines, masked=True,
                                seed=seed + k, what=what)
        expect_form(core, TWO_GROUP, 2, TMA, what=what)
        with variant(core, v):
            old, _ = sum_finish_job(core, [rc.LAYOUTS[layout]], sz, 1, lines=lines, masked=True,
                                    seed=seed + k, what=what + f", sg_variant {v}")
        expect_form(core, TWO_GROUP, 2, DIRECT if v == 5 else TMA, what=what)
        assert numpy.array_equal(new[0], old[0]), f"{what}: sg_variant {v} differs"


def case_split_capped(core, pair, axis, mode, cap=2, lines=7, seed=0):
    """split_subgrid_axis with the grid capped: along axis 0 the lines are adjacent (the
    two-line form where two fit), along axis 1 one line per CTA."""
    from tests import split_cases as sc  # pylint: disable=import-outside-toplevel

    fs, ss, N = core.facet_off_step, core.subgrid_off_step, core.N
    conc = FORMS[pair][3]
    f_offs = [(k % 5 - 2) * fs + (N if k % 3 == 2 else 0) for k in range(conc + 1)]
    with max_blocks(core, cap):
        err = sc.split_vs_oracle(core, axis, mode, core.xM_size - 5, lines, [-3 * ss, N + ss],
                                 [f_offs, [fs]], seed=seed)
    lpc = FORMS[pair][2] if axis == 0 else 1
    expect_form(core, SPLIT, lpc, DIRECT, grid=cap, what=f"{pair} split axis {axis}")
    return err
