"""
``extract_columns`` (K2) in every launch form the dispatch picks, shared by the emulated and the
GPU tests.

``csrc/dispatch_extract_columns.cu`` chooses the kernel from ``yN``, the facet sizes, the row
strides and a shared-memory budget, and how the facet rows reach shared memory: by swizzled
tensor loads (every facet has ``fs % 8 == 0`` and a row stride of at least ``fs``, and the
staging buffer rounded up to whole boxes fits 227 KiB) or by linear bulk copies.  :func:`form`
restates that choice; every case asserts the launch it was written for through
``swiftly_b200_debug_last_launch`` (kernel, chunks per tensor load or 0, capacity of the staging
buffer, grid) and then compares with ``OracleCore``.

``catalogue_rows()`` derives the distinct ``(yN, yB)`` of ``SWIFT_CONFIGS``; :data:`PINNED_TMA`
and :data:`PINNED_GENERIC` pin the form of each for a launch as ``SwiftlyForward`` makes it
(contiguous rows, every facet ``yB`` wide), with the number of catalogue entries behind each row,
so that a new entry or a change of the dispatch fails a test.  At ``yN = 16384`` only ``yB =
8192`` (2 of 16 entries) runs the tuned 4 x 4096 kernel: a staged row may hold 8192 samples
swizzled and 10174 linear, and the catalogue's other rows (``yB >= 11264``) run
``SplitLineKernel<8192>``.

Extended-precision spot check (:func:`spot_check`), worst ``|got - exact|`` in units of
``eps log2(yN)`` of the line's RMS per form, with the test seeds:

* H100 80GB HBM3 (700 W power limit), two lines per form: tma 0.25 .. 0.37 (yN = 1024 .. 8192),
  tma-4xQ 0.36 .. 0.60, tma-2xH 0.50, dif 0.54, park-dif 0.60, park-dif-long 0.58,
  park-dit 0.49, park-skew 0.47 (yN = 16384); against the oracle every form stays below
  1.4e-15 of the largest sample;
* emulated kernels (host build without fused multiply-adds), one line per form: tma
  0.23 .. 0.77, tma-4xQ 0.33 .. 0.54, tma-2xH 0.38 (yN = 16384), dif and park-dif 0.24,
  park-dit and park-skew 0.19 (yN = 512).
"""

import contextlib
import ctypes

import numpy
import torch

from ska_sdp_distributed_fourier_transform_b200.swift_configs import SWIFT_CONFIGS
from tests import length_cases as lc
from tests import pair_cases as prc
from tests import parity_cases as pc
from tests import subgrid_round_cases as rc

# kernel codes of swiftly_b200_debug_last_launch (plan.h)
LINE, SPLIT_LINE, SPLIT_F = 4, 5, 6
TMA, TMA_SPLIT, TMA4, DIF, PARK_DIF, PARK_DIF2, PARK_DIT, PARK_SKEW = range(8, 16)
KERNEL_NAMES = {LINE: "line", SPLIT_LINE: "split-line", SPLIT_F: "split-F", TMA: "tma",
                TMA_SPLIT: "tma-2xH", TMA4: "tma-4xQ", DIF: "dif", PARK_DIF: "park-dif",
                PARK_DIF2: "park-dif-long", PARK_DIT: "park-dit", PARK_SKEW: "park-skew"}

NUM_SMS = 132  # plan.h
SMEM = 227 * 1024  # shared memory of one SM that a CTA may take
MAX_BOX = 256  # chunks of 128 bytes (8 samples) per tensor load
MAX_LAUNCH_FACETS = 64  # core.extract_columns: facets per launch
SPLIT_GRID = 296  # launch_split / launch_split_f: persistent CTAs
LINE_GRID_CAP = NUM_SMS * 32
TMA_LENGTHS = (1024, 2048, 4096, 8192)  # ExtractColumnsTmaKernel<yN, false>
EMU_TMA_LENGTHS = (128, 512)  # instantiated for the emulated library only
# sg_variant at yN = 16384 -> force_split of the same form at yN = 512 (emulated library only)
FORCE_SPLIT_TWIN = {7: 1, 15: 3, 17: 4, 18: 5, 19: 6, 0: 2}


# ---------------------------------------------------------------------- the dispatch, restated
def _padded(h):
    return h + h // 16  # FftCfg<h>::PADDED doubles


def _smem_tma(h, in_cap):  # ExtractColumnsTmaKernel<h, *>::smem_bytes
    return in_cap * 16 + _padded(h) * 8 + 16


def _smem_two_groups(q, in_cap):  # the 4 x q kernels: two exchange buffers
    return in_cap * 16 + 2 * ((_padded(q) + 1) & ~1) * 8 + 32


def staging(sizes, smem, rows_ok=True, variant=0):
    """``(box_chunks, boxes, in_cap)`` of the staging buffer; box_chunks 0: linear bulk copies.
    ``rows_ok``: every row stride is at least the facet size and every base 16-byte aligned."""
    max_fs = max(sizes)
    linear = (0, 0, (max_fs + 1) & ~1)
    if variant == 6 or not rows_ok or any(fs % 8 for fs in sizes):
        return linear
    chunks = max_fs // 8
    box = MAX_BOX if chunks >= MAX_BOX else chunks & ~7
    if box < 8:
        return linear
    boxes = -(-chunks // box)
    if smem(boxes * box * 8) > SMEM:
        return linear
    return (box, boxes, boxes * box * 8)


def generic_form(yN, n_lines, cap=0, variant=0):
    """The launch record of the generic line kernels for ``n_lines`` lines of ``yN`` samples."""
    if variant == 3 and yN == 16384:
        kernel, v, grid = SPLIT_F, 4, min(n_lines, SPLIT_GRID)
    else:
        plan = lc.line_kernel(yN)
        if plan[0] == "direct":
            t = yN // 16
            v = 1 if t >= 256 else min(16, 256 // t)
            kernel, grid = LINE, min(-(-n_lines // v), LINE_GRID_CAP)
        elif plan[0] == "split":
            kernel, v, grid = SPLIT_LINE, 2, min(n_lines, SPLIT_GRID)
        else:
            kernel, v, grid = SPLIT_F, plan[2], min(n_lines, SPLIT_GRID)
    return (kernel, v, 0, min(grid, cap) if cap else grid)


def form(yN, sizes, n_lines, *, rows_ok=True, variant=0, force_split=0, cap=0, emulated=False,
         pair_ok=True):
    """The launch record ``(kernel, box_chunks, in_cap, grid)`` of one ``extract_columns`` launch
    (``(kernel, lines per CTA or F, 0, grid)`` when it leaves the TMA-staged kernels), and the
    number of boxes per row: ``(record, boxes)``.  ``pair_ok``: every output has an even line
    stride and starts on a 32-byte boundary (the pair stores of sg_variant 17)."""
    max_fs = max(sizes)
    split = yN > lc.MAX_DIRECT_FFT or bool(force_split)
    hh = yN // 2 if split else yN
    kernel = None
    if variant not in (3, 4) and ((max_fs + 1) & ~1) * 16 + _padded(hh) * 8 + 16 <= SMEM:
        if split:
            quad = yN == 16384 or (emulated and yN == 512)
            if quad and variant != 7 and force_split != 1:
                sel = variant if yN == 16384 else {4: 17, 5: 18, 6: 19, 3: 15}.get(force_split, 0)
                if sel == 17 and pair_ok:
                    kernel = PARK_DIF if max_fs <= yN // 2 else PARK_DIF2
                else:
                    kernel = {18: PARK_DIT, 19: PARK_SKEW, 15: DIF}.get(sel, TMA4)
                q = yN // 4
                smem, threads = (lambda cap_: _smem_two_groups(q, cap_)), 2 * q // 16
            elif quad:
                kernel = TMA_SPLIT
                smem, threads = (lambda cap_: _smem_tma(yN // 2, cap_)), yN // 32
        elif yN in TMA_LENGTHS or (emulated and yN in EMU_TMA_LENGTHS):
            kernel = TMA
            smem, threads = (lambda cap_: _smem_tma(yN, cap_)), yN // 16
    if kernel is None:
        return generic_form(yN, n_lines, cap, variant), 0
    box, boxes, in_cap = staging(sizes, smem, rows_ok, variant)
    per_sm = max(1, min(SMEM // smem(in_cap), 512 // threads))
    grid = min(NUM_SMS * per_sm, n_lines)
    return (kernel, box, in_cap, min(grid, cap) if cap else grid), boxes


# ---------------------------------------------------------------------- the catalogue
def catalogue_rows():
    """``(yN, yB)`` -> (number of catalogue entries, geometry ``(W, N, xM, yN)`` of the smallest
    one by (m, N, name))."""
    rows = {}
    for name, p in SWIFT_CONFIGS.items():
        key = (p["yN_size"], p["yB_size"])
        m = p["xM_size"] * p["yN_size"] // p["N"]
        rep = (m, p["N"], name, (p["W"], p["N"], p["xM_size"], p["yN_size"]))
        n, best = rows.get(key, (0, rep))
        rows[key] = (n + 1, min(best, rep))
    return {k: (n, rep[3]) for k, (n, rep) in sorted(rows.items())}


def row_form(yN, yB, emulated=False):
    """``(kernel, box_chunks, boxes, in_cap)`` of a launch whose facets are all ``yB`` wide with
    contiguous rows; for the generic kernels ``(kernel, lines per CTA or F, 0, 0)``."""
    (kernel, box, in_cap, _), boxes = form(yN, [yB], 1, emulated=emulated)
    return (kernel, box, boxes, in_cap) if kernel >= TMA else (kernel, box, 0, 0)


# (yN, yB): (kernel, chunks per tensor load, boxes per row, staging capacity, catalogue entries)
PINNED_TMA = {
    (1024, 512): (TMA, 64, 1, 512, 1),
    (1024, 704): (TMA, 88, 1, 704, 2),
    (1024, 768): (TMA, 96, 1, 768, 1),
    (1024, 832): (TMA, 104, 1, 832, 1),
    (2048, 1024): (TMA, 128, 1, 1024, 1),
    (2048, 1408): (TMA, 176, 1, 1408, 2),
    (2048, 1536): (TMA, 192, 1, 1536, 1),
    (2048, 1664): (TMA, 208, 1, 1664, 2),
    (2048, 1792): (TMA, 224, 1, 1792, 2),
    (2048, 1824): (TMA, 224, 2, 3584, 1),
    (4096, 2048): (TMA, 256, 1, 2048, 2),
    (4096, 2816): (TMA, 256, 2, 4096, 2),
    (4096, 3072): (TMA, 256, 2, 4096, 2),
    (4096, 3328): (TMA, 256, 2, 4096, 4),
    (4096, 3584): (TMA, 256, 2, 4096, 3),
    (4096, 3648): (TMA, 256, 2, 4096, 1),
    (8192, 4096): (TMA, 256, 2, 4096, 2),
    (8192, 5632): (TMA, 256, 3, 6144, 3),
    (8192, 6144): (TMA, 256, 3, 6144, 2),
    (8192, 6656): (TMA, 256, 4, 8192, 5),
    (8192, 7168): (TMA, 256, 4, 8192, 4),
    (8192, 7296): (TMA, 256, 4, 8192, 1),
    (16384, 8192): (TMA4, 256, 4, 8192, 2),
}
# yN: (generic kernel, lines per CTA or F, distinct yB, catalogue entries); at yN = 16384 the
# rows whose facets do not fit the staging buffer
PINNED_GENERIC = {
    256: (LINE, 16, 1, 1), 512: (LINE, 8, 3, 4),
    384: (SPLIT_F, 3, 1, 1), 640: (SPLIT_F, 5, 3, 3), 768: (SPLIT_F, 3, 3, 4),
    896: (SPLIT_F, 7, 3, 3), 1280: (SPLIT_F, 5, 4, 5), 1536: (SPLIT_F, 3, 4, 5),
    1792: (SPLIT_F, 7, 4, 5), 2560: (SPLIT_F, 5, 6, 9), 3072: (SPLIT_F, 3, 6, 9),
    3584: (SPLIT_F, 7, 6, 9), 5120: (SPLIT_F, 5, 7, 12), 6144: (SPLIT_F, 3, 7, 12),
    7168: (SPLIT_F, 7, 7, 12), 10240: (SPLIT_F, 5, 6, 13), 12288: (SPLIT_F, 3, 6, 13),
    14336: (SPLIT_F, 7, 6, 13), 16384: (SPLIT_LINE, 2, 5, 14),
    20480: (SPLIT_F, 5, 4, 8), 24576: (SPLIT_F, 3, 4, 8), 28672: (SPLIT_F, 7, 4, 8),
    32768: (SPLIT_F, 4, 4, 9), 36864: (SPLIT_F, 9, 1, 1), 40960: (SPLIT_F, 5, 4, 4),
    49152: (SPLIT_F, 6, 4, 5), 57344: (SPLIT_F, 7, 4, 5), 65536: (SPLIT_F, 8, 4, 5),
}
# the staging limits at yN = 16384: the largest facet staged swizzled, the largest staged at all
MAX_SWIZZLED_16384 = 8192
MAX_STAGED_16384 = 10174


def derived_tables():
    """``(tma, generic)`` in the layout of :data:`PINNED_TMA` / :data:`PINNED_GENERIC`, from
    ``SWIFT_CONFIGS`` and :func:`form`."""
    tma, generic = {}, {}
    for (yN, yB), (n, _) in catalogue_rows().items():
        f = row_form(yN, yB)
        if f[0] >= TMA:
            tma[(yN, yB)] = f + (n,)
        else:
            k, v, rows, entries = generic.get(yN, (f[0], f[1], 0, 0))
            assert (k, v) == f[:2]
            generic[yN] = (k, v, rows + 1, entries + n)
    return tma, generic


# ---------------------------------------------------------------------- hooks
def last_launch(core):
    return prc.last_launch(core)


@contextlib.contextmanager
def hooks(core, variant=0, cap=0, force_split=0):
    """Select a kernel form (``sg_variant``; ``force_split``, emulated library) and cap the
    persistent grid for the launches inside."""
    lib = core._lib
    lib.swiftly_b200_debug_force_split.argtypes = [ctypes.c_void_p, ctypes.c_int]
    lib.swiftly_b200_debug_max_blocks.argtypes = [ctypes.c_void_p, ctypes.c_int]
    rc.set_variant(core, variant)
    lib.swiftly_b200_debug_max_blocks(core._plan, int(cap))
    lib.swiftly_b200_debug_force_split(core._plan, int(force_split))
    try:
        yield
    finally:
        rc.set_variant(core, 0)
        lib.swiftly_b200_debug_max_blocks(core._plan, 0)
        lib.swiftly_b200_debug_force_split(core._plan, 0)


def is_emulated(core):
    return getattr(core, "tensor_device", None) is not None


_dev = lc._dev  # pylint: disable=protected-access
_to = lc._to  # pylint: disable=protected-access
NAN = complex(numpy.nan, numpy.nan)


# ---------------------------------------------------------------------- one launch
def make_input(core, rows, blk, layout):
    """A prepared facet ``(yN, fs)`` on the device whose rows ``rows`` hold ``blk`` and whose
    other rows are never written.  ``layout``: "contiguous" (row stride fs); "slice" (columns
    3 .. 3 + fs of an array 24 samples wider: row stride > fs, base 16- but not 128-byte
    aligned); "overlap" (rows ``lc.ROW_STEP`` samples apart, row stride < fs)."""
    yN, fs = core.yN_size, blk.shape[1]
    dev = _dev(core)
    idx = torch.from_numpy(numpy.asarray(rows)).to(dev)
    if layout == "overlap":
        # rows overlap: row r holds buf[8 r : 8 r + fs]; fill it from the rows' own values where
        # they do not collide -- so build the buffer on the host from the LAST writer
        buf = numpy.zeros((yN - 1) * lc.ROW_STEP + fs, dtype=complex)
        view = numpy.lib.stride_tricks.as_strided(
            buf, (yN, fs), (lc.ROW_STEP * buf.itemsize, buf.itemsize))
        for r, line in zip(rows, blk):
            view[r] = line
        return _to(core, buf).as_strided((yN, fs), (lc.ROW_STEP, 1)), view[numpy.asarray(rows)]
    if layout == "slice":
        wide = torch.zeros((yN, fs + 24), dtype=torch.complex128, device=dev)
        bf = wide[:, 3:3 + fs]
        assert bf.data_ptr() % 16 == 0 and (is_emulated(core) or bf.data_ptr() % 128 == 48)
    else:
        assert layout == "contiguous"
        bf = torch.zeros((yN, fs), dtype=torch.complex128, device=dev)
    bf[idx] = _to(core, blk)
    return bf, blk


def make_outputs(core, n, out_layout):
    """``n`` outputs ``(m, yN)`` filled with NaN, and the arrays they live in.  ``out_layout``:
    "own"; "wide" (row slices of an array 6 samples wider, the line starts 32-byte aligned);
    "odd" (line stride yN + 1); "shifted" (line stride even, lines start 16 bytes off a 32-byte
    boundary)."""
    yN, m = core.yN_size, core.xM_yN_size
    extra, lo = {"own": (0, 0), "wide": (6, 2), "odd": (1, 0), "shifted": (2, 1)}[out_layout]
    homes = [torch.full((m, yN + extra), NAN, dtype=torch.complex128, device=_dev(core))
             for _ in range(n)]
    return [h[:, lo:lo + yN] for h in homes], homes


def run(core, oracle, sizes, offs, sg_off0, *, want=None, prewindowed=False,
        layout="contiguous", out_layout="own", variant=0, cap=0, force_split=0, seed=0,
        outs=None, shared_input=False, rtol=1e-12, what=""):
    """One ``extract_columns`` call against ``prepare_facet(extract_from_facet(BF, sg_off0,
    axis 0), off1, axis 1)`` of the oracle.  Asserts the launch record against ``want`` (default:
    :func:`form` of the call's last launch), that every output sample was written and that the
    samples around a "wide" output are untouched.  Returns ``(outputs as numpy arrays, worst
    error relative to the largest reference sample, launch record)``."""
    rng = numpy.random.default_rng(seed)
    yN, m = core.yN_size, core.xM_yN_size
    emulated = is_emulated(core)
    rows = oracle._facet_window(sg_off0)  # pylint: disable=protected-access
    assert len(set(rows.tolist())) == m
    bfs, refs = [], []
    for j, (fs, off) in enumerate(zip(sizes, offs)):
        if shared_input and j:
            assert fs == sizes[0]
            bf = bfs[0]
        else:
            bf, blk = make_input(core, rows, pc.rand_c(rng, m, fs), layout)
        bfs.append(bf)
        data = blk / oracle._fb_window(fs)[None, :] if prewindowed else blk  # pylint: disable=protected-access
        refs.append(oracle.prepare_facet(data, off, axis=1))
    homes = None
    if outs is None:
        outs, homes = make_outputs(core, len(sizes), out_layout)
    with hooks(core, variant, cap, force_split):
        core.extract_columns(bfs, sg_off0, list(offs), outs=outs, prewindowed=prewindowed)
        got = last_launch(core)
    tail = (len(sizes) - 1) % MAX_LAUNCH_FACETS + 1  # facets of the call's last launch
    if want is None:
        pair_ok = all(o.stride(0) % 2 == 0 and (emulated or o.data_ptr() % 32 == 0) for o in outs)
        want, _ = form(yN, sizes[-tail:], tail * m, rows_ok=layout != "overlap", variant=variant,
                       force_split=force_split, cap=cap, emulated=emulated, pair_ok=pair_ok)
    label = (f"{what or 'extract_columns'} (yN {yN}, m {m}, sizes {list(sizes)[:4]}, "
             f"sg_off0 {sg_off0}, {layout}{', prewindowed' if prewindowed else ''})")
    assert got == want, f"{label}: launched {got}, expected {want}"
    res = [o.cpu().numpy() for o in outs]
    err = max(lc._check(o, r, rtol, f"{label} facet {j} (fs {fs}, off1 {off})")  # pylint: disable=protected-access
              for j, (o, r, fs, off) in enumerate(zip(res, refs, sizes, offs)))
    if homes is not None and out_layout != "own":
        for h, o in zip(homes, outs):
            lo = o.storage_offset() - h.storage_offset()
            outside = torch.cat([h[:, :lo], h[:, lo + yN:]], dim=1)
            assert bool(torch.isnan(outside.real).all()), f"{label}: wrote outside the output lines"
    return res, err, got


# ---------------------------------------------------------------------- offsets
def facet_offsets(core):
    """Facet offsets 0, negative and >= N."""
    step = core.facet_off_step
    return [0, -3 * step, core.N + 5 * step]


def subgrid_offsets(core):
    """Subgrid offsets whose m-row window wraps around yN (one negative, one >= N), an ordinary
    one and 0."""
    N, yN, m = core.N, core.yN_size, core.xM_yN_size
    step = core.subgrid_off_step
    # window rows start at yN / 2 - m / 2 + s, s = off yN / N: s = yN / 2 puts the middle of the
    # window on the seam
    wrap = (yN // 2) * step
    return [-wrap, N + wrap + step, 3 * step, 0]


def window_wraps(core, oracle, sg_off0):
    rows = oracle._facet_window(sg_off0)  # pylint: disable=protected-access
    return bool(rows.min() == 0 and rows.max() == core.yN_size - 1)


# ---------------------------------------------------------------------- the cases
def catalogue_row_case(core, oracle, yB, n_facets=3, seed=0):
    """A launch as ``SwiftlyForward`` makes it: ``n_facets`` contiguous facets of ``yB`` samples,
    raw and prewindowed.  Returns the worst error and the launch record."""
    yN = core.yN_size
    offs = facet_offsets(core)[:n_facets]
    sg = subgrid_offsets(core)
    want = row_form(yN, yB, is_emulated(core))
    worst = 0.0
    for k, prewindowed in enumerate([False, True]):
        _, err, got = run(core, oracle, [yB] * n_facets, offs, sg[k], prewindowed=prewindowed,
                          seed=seed + k, what=f"catalogue row ({yN}, {yB})")
        assert got[:2] == want[:2] and (got[0] < TMA or got[2] == want[3]), (got, want)
        worst = max(worst, err)
    return worst, got


def box_layouts(yN):
    """Facet sizes with one box below 256 chunks, exactly 256 chunks, 256 plus a short tail,
    several boxes plus a tail, 228 chunks (box 224 plus a tail of 4), the smallest swizzled row
    (64 samples) and the sizes 56 and 8 that go linear -- those that fit ``yN``."""
    sizes = [8, 56, 64, 88 * 8, 228 * 8, 256 * 8, 260 * 8, 352 * 8, 912 * 8, 1024 * 8]
    return [fs for fs in sizes if fs < yN]


def box_layout_case(core, oracle, fs, seed=0):
    """One facet size: the default staging, then ``sg_variant`` 6 (linear staging of the same
    rows) and a grid capped at 2 CTAs must give the same bits."""
    yN, m = core.yN_size, core.xM_yN_size
    offs = facet_offsets(core)[1:]
    sg = subgrid_offsets(core)[2]
    (record, boxes) = form(yN, [fs, fs], 2 * m, emulated=is_emulated(core))
    chunks = fs // 8
    if fs >= 64:
        assert record[1] == min(MAX_BOX, chunks & ~7) and boxes == -(-chunks // record[1])
    else:
        assert record[1] == 0
    base, err, _ = run(core, oracle, [fs, fs], offs, sg, seed=seed, what=f"box layout fs {fs}")
    lin, _, got = run(core, oracle, [fs, fs], offs, sg, seed=seed, variant=6,
                      what=f"box layout fs {fs}, linear staging")
    assert got[1] == 0
    few, _, _ = run(core, oracle, [fs, fs], offs, sg, seed=seed, cap=2,
                    what=f"box layout fs {fs}, 2 CTAs")
    for a, b, c in zip(base, lin, few):
        assert numpy.array_equal(a, b), f"fs {fs}: linear staging changes the bits"
        assert numpy.array_equal(a, c), f"fs {fs}: a capped grid changes the bits"
    return err, record, boxes


def mixed_sizes(yN):
    """[large, small, large] with every size a multiple of 8, the small facet shorter than one
    box of the large ones (large: 11/16 yN; yN / 2 where longer rows are not staged swizzled)."""
    large = (yN * 11 // 16) & ~7 if yN <= lc.MAX_DIRECT_FFT else yN // 2
    box = min(MAX_BOX, (large // 8) & ~7)
    small = max(64, (box * 8 // 3) & ~7)
    assert small < box * 8
    return [large, small, large - 64]


def mixed_case(core, oracle, cap=0, seed=0):
    """[large, small, large] in one launch (swizzled, the box taken from the largest facet, so
    the small facet's tensor is narrower than one box and the stale tail of the long row before
    it stays in the staging buffer), and the same with one odd size (the whole launch linear)."""
    yN = core.yN_size
    sizes = mixed_sizes(yN)
    offs = facet_offsets(core)
    sg = subgrid_offsets(core)
    _, e1, got = run(core, oracle, sizes, offs, sg[0], cap=cap, seed=seed, what="mixed sizes")
    assert got[1] == min(MAX_BOX, (sizes[0] // 8) & ~7) and got[1] * 8 > sizes[1]
    odd = [sizes[0], sizes[1] + 1, sizes[2]]
    _, e2, got = run(core, oracle, odd, offs, sg[1], cap=cap, prewindowed=True, seed=seed + 1,
                     what="mixed sizes, one odd")
    assert got[1] == 0 and got[2] == sizes[0]
    return max(e1, e2)


def stride_case(core, oracle, fs, seed=0):
    """Row stride equal to fs, larger (a column slice at a base that is 16- but not 128-byte
    aligned: still swizzled) and smaller (overlapping rows: linear)."""
    offs = facet_offsets(core)[:2]
    sg = subgrid_offsets(core)[2]
    worst = 0.0
    for k, (layout, swizzled) in enumerate([("contiguous", True), ("slice", True),
                                            ("overlap", False)]):
        _, err, got = run(core, oracle, [fs, fs], offs, sg, layout=layout, seed=seed + k,
                          prewindowed=k == 1, what=f"row stride ({layout})")
        assert (got[1] != 0) == swizzled, (layout, got)
        worst = max(worst, err)
    return worst


def output_case(core, oracle, fs, seed=0):
    """Outputs that are row slices of a wider NaN-filled array; and one set of outputs reused by
    two calls with different offsets, as the LRU of SwiftlyForward reuses its column buffers."""
    offs = facet_offsets(core)
    sg = subgrid_offsets(core)
    _, e1, _ = run(core, oracle, [fs, fs - 8, fs], offs, sg[0], out_layout="wide", seed=seed,
                   what="wide outputs")
    outs, _ = make_outputs(core, 2, "own")
    _, e2, _ = run(core, oracle, [fs, fs], offs[:2], sg[1], outs=outs, seed=seed + 1,
                   what="reused outputs, first call")
    _, e3, _ = run(core, oracle, [fs, fs], offs[1:], sg[2], outs=outs, seed=seed + 2,
                   prewindowed=True, what="reused outputs, second call")
    return max(e1, e2, e3)


def offset_case(core, oracle, fs, seed=0):
    """Every subgrid offset of :func:`subgrid_offsets` (two of them wrap the row window around
    yN) with facet offsets 0, negative and >= N."""
    offs = facet_offsets(core)
    sgs = subgrid_offsets(core)
    assert window_wraps(core, oracle, sgs[0]) and window_wraps(core, oracle, sgs[1])
    assert sgs[0] < 0 and sgs[1] >= core.N
    return max(run(core, oracle, [fs, fs - 1 if k % 2 else fs, fs], offs, sg, seed=seed + k,
                   what=f"offsets, sg_off0 {sg}")[1] for k, sg in enumerate(sgs))


def many_lines_case(core, oracle, fs, n_facets=MAX_LAUNCH_FACETS, seed=0):
    """``n_facets`` facets sharing one small input buffer, a different ``off1`` each: with 64
    facets more lines than the persistent grid has CTAs; with more than 64 two launches, of
    which the record shows the last."""
    yN, m = core.yN_size, core.xM_yN_size
    step = core.facet_off_step
    offs = [(k - 5) * step for k in range(n_facets)]
    _, err, got = run(core, oracle, [fs] * n_facets, offs, subgrid_offsets(core)[2],
                      shared_input=True, seed=seed, what=f"{n_facets} facets")
    tail = (n_facets - 1) % MAX_LAUNCH_FACETS + 1
    if n_facets > MAX_LAUNCH_FACETS:
        assert got[3] == tail * m, got
    else:
        assert got[3] < n_facets * m, f"grid {got[3]} covers all {n_facets * m} lines"
    return err, got


def boundary_sizes_16384():
    """Facet sizes next to the staging limits at yN = 16384 and the form each must run:
    ``fs -> (kernel, box_chunks, in_cap)``."""
    return {8192: (TMA4, 256, 8192), 8200: (TMA4, 0, 8200), 10168: (TMA4, 0, 10168),
            10174: (TMA4, 0, 10174), 10175: (SPLIT_LINE, 2, 0), 11264: (SPLIT_LINE, 2, 0)}


def boundary_case(core, oracle, fs, seed=0):
    assert core.yN_size == 16384
    want = boundary_sizes_16384()[fs]
    (record, _) = form(16384, [fs], core.xM_yN_size, emulated=is_emulated(core))
    assert record[:3] == want, (fs, record, want)
    _, err, got = run(core, oracle, [fs], [core.facet_off_step], subgrid_offsets(core)[2],
                      seed=seed, what=f"staging boundary fs {fs}")
    assert got[:3] == want
    return err


# sg_variant -> kernel at facets of at most yN / 2, at longer ones
VARIANT_KERNELS = {0: (TMA4, TMA4), 7: (TMA_SPLIT, TMA_SPLIT), 15: (DIF, DIF),
                   17: (PARK_DIF, PARK_DIF2), 18: (PARK_DIT, PARK_DIT),
                   19: (PARK_SKEW, PARK_SKEW), 20: (TMA4, TMA4)}


def variant_case(core, oracle, variant, seed=0):
    """One selectable K2 form at the 4 x Q lengths (``sg_variant`` at yN = 16384; its
    ``force_split`` twin at yN = 512 on the emulated library): rows staged by swizzled tensor
    loads, by linear bulk copies (an odd size), rows longer than yN / 2, several lines per CTA,
    each asserting the recorded kernel; for 17 also the fall-back to the default form when an
    output line stride is odd or (GPU) an output is not 32-byte aligned."""
    yN, m = core.yN_size, core.xM_yN_size
    emulated = is_emulated(core)
    if yN == 16384:
        sel = dict(variant=variant)
    else:
        assert emulated and yN == 512 and variant in FORCE_SPLIT_TWIN
        sel = dict(force_split=FORCE_SPLIT_TWIN[variant])
    short, longer = VARIANT_KERNELS[variant]
    step, sg = core.facet_off_step, subgrid_offsets(core)[2]
    half = yN // 2
    worst = 0.0
    for k, (sizes, kernel, swizzled) in enumerate([
            ([half, half], short, True),
            ([half - 1, half + half // 8 + 8], longer, False),
            # (at yN = 16384 rows longer than yN / 2 do not fit the buffer in whole boxes)
            ([half + half // 8, half - 8], longer, yN != 16384)]):
        _, err, got = run(core, oracle, sizes, [step, -2 * step], sg, seed=seed + k,
                          cap=3 if k == 2 else 0, what=f"sg_variant {variant}", **sel)
        assert got[0] == kernel and (got[1] != 0) == swizzled, (variant, sizes, got)
        worst = max(worst, err)
    if variant == 17:
        for out_layout in ["odd"] + ([] if emulated else ["shifted"]):
            _, err, got = run(core, oracle, [half, half], [0, step], sg, seed=seed + 5,
                              out_layout=out_layout, what=f"sg_variant 17, {out_layout} outputs",
                              **sel)
            assert got[0] == TMA4, got
            worst = max(worst, err)
    return worst


# ---------------------------------------------------------------------- extended precision
def sub_transforms(kernel, yN):
    """``(M, F)``: the kernel computes the line as F transforms of M points."""
    if kernel == TMA:
        return yN, 1
    if kernel == TMA_SPLIT:
        return yN // 2, 2
    assert kernel >= TMA4
    return yN // 4, 4


def spot_check(core, fs, seed, *, variant=0, force_split=0, layout="contiguous", n_lines=2):
    """K2 of one facet at the bins of ``length_cases.spot_bins`` (the sub-transform boundaries
    ``M s - 1, M s, M s + 1``, the centre, random bins) of its first ``n_lines`` lines against
    ``length_cases.centred_dft`` of the exactly weighted, padded and rolled row.  Returns the
    launch record and the worst ``|got - exact|`` relative to the RMS of the exact line, in
    units of ``EPS * log2(yN)``."""
    rng = numpy.random.default_rng(seed)
    yN, m = core.yN_size, core.xM_yN_size
    off, sg_off0 = 3 * core.facet_off_step, 2 * core.subgrid_off_step
    s = sg_off0 * yN // core.N
    rows = numpy.mod(yN // 2 - m // 2 + numpy.mod(numpy.arange(m) - s, m) + s, yN)
    blk = pc.rand_c(rng, m, fs)
    bf, blk = make_input(core, rows, blk, layout)
    outs, _ = make_outputs(core, 1, "own")
    with hooks(core, variant, 0, force_split):
        core.extract_columns([bf], sg_off0, [off], outs=outs)
        got = last_launch(core)
    res = outs[0].cpu().numpy()
    M, F = sub_transforms(got[0], yN)
    pos = [(p + yN // 2) % yN for p in lc.spot_bins(M, F, yN, rng)]
    dest = (yN // 2 - fs // 2 + off + numpy.arange(fs)) % yN
    fb = lc._window_of(core, fs)  # pylint: disable=protected-access
    worst = 0.0
    for line in range(n_lines):
        z = numpy.zeros(yN, dtype=numpy.clongdouble)
        z[dest] = blk[line].astype(numpy.clongdouble) * fb
        exact = lc.centred_dft(z, pos, +1) / yN
        rms = numpy.sqrt((numpy.abs(z) ** 2).sum()) / yN  # Parseval
        err = numpy.abs(res[line, pos].astype(numpy.clongdouble) - exact).max() / rms
        worst = max(worst, float(err))
    return got, worst / (lc.EPS * numpy.log2(yN))
