"""
Shared checks of the real-image backward transform, run by tests/test_emu_real_backward.py on the
host-emulated kernels and by tests/test_gpu_real_backward.py on the H100.

ABI level: ``merge_mirror_subgrid`` exactly against numpy (one complex add where both terms
exist), and as the adjoint of ``mirror_subgrid``; ``finish_facet_real`` bitwise against the real
part of ``finish_facet`` times the mask, with the same launch form.  API level:
``SwiftlyBackward(real_image=True)`` without pairs bitwise ``Re`` of the default mode; with pairs
(``add_subgrid_tasks``) against the analytic facets and the default mode, and the work it saves
(subgrid sides, merge calls, folded columns) counted.
"""

import contextlib
import ctypes

import numpy
import pytest
import torch

from ska_sdp_distributed_fourier_transform_b200 import (
    SwiftlyBackward,
    SwiftlyForward,
    _lib,
    api,
    make_facet,
)
from ska_sdp_distributed_fourier_transform_b200.api_helper import check_facet
from ska_sdp_distributed_fourier_transform_b200.fourier_algorithm import make_subgrid_from_sources
from tests import k2_cases as kc
from tests import real_image_cases as rc

MERGE = 17  # kernel code of swiftly_b200_debug_last_launch (plan.h)
NAN = complex(numpy.nan, numpy.nan)


# ---------------------------------------------------------------------- merge_mirror_subgrid
def expected_merge(sg, mirror):
    """numpy: ``sg + conj(mirror[2h - r, 2h - c])`` on the ``S x S`` grid, each term where it
    exists (adding 0 elsewhere keeps the other term's bits)."""
    sz = sg.shape[0]
    S = rc.source_size(sz)
    a = numpy.zeros((S, S), dtype=complex)
    b = numpy.zeros((S, S), dtype=complex)
    a[:sz, :sz] = sg
    b[:sz, :sz] = mirror
    return a + numpy.conj(b[::-1, ::-1])


def _merge_outputs(core, S, layout):
    dev = kc._dev(core)
    if layout == "own":
        return None, None
    if layout == "wide":
        wide = torch.full((S + 5, S + 9), NAN, dtype=torch.complex128, device=dev)
        return wide[2:2 + S, 3:3 + S], wide
    assert layout == "transposed"
    return torch.full((S, S), NAN, dtype=torch.complex128, device=dev).t(), None


def merge_case(core, sz, *, layout="own", transposed_inputs=False, cap=0, seed=0):
    """One ``merge_mirror_subgrid`` call on random inputs: exactly numpy's samples, nothing
    written outside the output view, the launch recorded as ``MergeMirrorSubgridKernel`` with
    one CTA per output row up to the cap."""
    rng = numpy.random.default_rng(seed)
    S = rc.source_size(sz)
    sg, mirror = (rng.standard_normal((sz, sz)) + 1j * rng.standard_normal((sz, sz))
                  for _ in range(2))
    if transposed_inputs:
        dsg, dmir = (kc._to(core, numpy.ascontiguousarray(x.T)).t() for x in (sg, mirror))
    else:
        dsg, dmir = kc._to(core, sg), kc._to(core, mirror)
    out, wide = _merge_outputs(core, S, layout)
    with kc.hooks(core, 0, cap, 0):
        got = core.merge_mirror_subgrid(dsg, dmir, out=out)
        rec = kc.last_launch(core)
    assert tuple(got.shape) == (S, S)
    g = got.cpu().numpy()
    want = expected_merge(sg, mirror)
    assert numpy.array_equal(g, want), f"max diff {numpy.nanmax(numpy.abs(g - want)):.3e}"
    if wide is not None:
        outside = torch.isnan(wide.real).cpu().numpy()
        outside[2:2 + S, 3:3 + S] = ~outside[2:2 + S, 3:3 + S]
        assert outside.all(), "a sample outside the view was written"
    assert tuple(rec) == (MERGE, 0, 0, min(cap, S) if cap else S), rec
    return rec


def _raw_merge(core, sg, mirror, out, locations=(_lib.DEVICE,) * 3, null=None):
    """The C entry point (no Python checks); ``null``: index of a descriptor passed as NULL."""
    # pylint: disable=protected-access
    descs = [core._describe(t, 1) for t in (sg, mirror, out)]
    for d, loc in zip(descs, locations):
        d.location = loc
    args = [None if k == null else ctypes.byref(d) for k, d in enumerate(descs)]
    rc_ = core._lib.swiftly_b200_merge_mirror_subgrid(core._plan, *args, ctypes.c_void_p(0))
    _lib.check(core._lib, rc_)


def merge_rejects(core):
    """``EINVAL`` (``ValueError``): NULL arguments, host arrays, inputs not both ``sz x sz``, an
    output not ``S x S``."""
    dev = kc._dev(core)

    def z(*shape):
        return torch.zeros(shape, dtype=torch.complex128, device=dev)

    for sz in (8, 9):
        S = rc.source_size(sz)
        for k in range(3):
            with pytest.raises(ValueError, match="NULL"):
                _raw_merge(core, z(sz, sz), z(sz, sz), z(S, S), null=k)
            locs = [_lib.DEVICE] * 3
            locs[k] = _lib.HOST
            with pytest.raises(ValueError, match="device arrays only"):
                _raw_merge(core, z(sz, sz), z(sz, sz), z(S, S), locs)
        for sg, mirror in ((z(sz, sz - 1), z(sz, sz)), (z(sz - 1, sz), z(sz, sz)),
                           (z(sz, sz), z(sz, sz + 1)), (z(sz, sz), z(sz + 1, sz))):
            with pytest.raises(ValueError, match="sg and mirror"):
                _raw_merge(core, sg, mirror, z(S, S))
            with pytest.raises(ValueError):
                core.merge_mirror_subgrid(sg, mirror)
        for out in (z(S - 1, S), z(S, S + 1), z(S + 1, S + 1)):
            with pytest.raises(ValueError, match="out is"):
                _raw_merge(core, z(sz, sz), z(sz, sz), out)
            with pytest.raises(ValueError):
                core.merge_mirror_subgrid(z(sz, sz), z(sz, sz), out=out)


def adjoint_case(core, sz, seed=0):
    """``Re<mirror_subgrid(x), (a, b)> = Re<x[:S, :S], merge(a, b)>`` (unmasked), to rounding."""
    rng = numpy.random.default_rng(seed)
    S = rc.source_size(sz)

    def rand(*shape):
        return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)

    x, a, b = rand(S, S), rand(sz, sz), rand(sz, sz)
    u, v = (t.cpu().numpy() for t in core.mirror_subgrid(kc._to(core, x), sz))
    c = core.merge_mirror_subgrid(kc._to(core, a), kc._to(core, b)).cpu().numpy()
    lhs = numpy.vdot(u, a).real + numpy.vdot(v, b).real
    rhs = numpy.vdot(x, c).real
    scale = numpy.abs(x).sum() * max(numpy.abs(a).max(), numpy.abs(b).max())
    assert abs(lhs - rhs) <= 1e-13 * scale, (lhs, rhs)


# ---------------------------------------------------------------------- finish_facet_real
def finish_real_case(core, fs, axis, *, n_lines=6, masked=True, layout="own", force_split=0,
                     cap=0, seed=0):
    """``finish_facet_real`` bitwise ``finish_facet(mask=None).real * mask`` along ``axis``, into
    an own, a wide (NaN-prefilled) or a transposed output; the same launch record as
    ``finish_facet``.  Returns the record."""
    rng = numpy.random.default_rng(seed)
    yN = core.yN_size
    shape_in = (yN, n_lines) if axis == 0 else (n_lines, yN)
    acc = kc._to(core, rng.standard_normal(shape_in) + 1j * rng.standard_normal(shape_in))
    shape = list(shape_in)
    shape[axis] = fs
    shape = tuple(shape)
    mask = (rng.random(fs) > 0.3).astype(float) if masked else None
    dmask = None if mask is None else torch.from_numpy(mask).to(acc.device)
    dev = kc._dev(core)
    wide = None
    if layout == "own":
        out = None
    elif layout == "wide":
        wide = torch.full((shape[0] + 3, shape[1] + 7), numpy.nan, dtype=torch.float64,
                          device=dev)
        out = wide[1:1 + shape[0], 5:5 + shape[1]]
    else:
        assert layout == "transposed"
        out = torch.full(shape[::-1], numpy.nan, dtype=torch.float64, device=dev).t()
    off = int(rng.integers(-3, 4)) * core.facet_off_step
    with kc.hooks(core, 0, cap, force_split):
        ref = core.finish_facet(acc, off, fs, axis)
        rec_ref = kc.last_launch(core)
        got = core.finish_facet_real(acc, off, fs, axis, out=out, mask=dmask)
        rec = kc.last_launch(core)
    assert got.dtype == torch.float64 and tuple(got.shape) == shape
    want = ref.real.cpu().numpy()
    if mask is not None:
        want = want * (mask[:, None] if axis == 0 else mask[None, :])
    g = got.cpu().numpy()
    assert numpy.array_equal(g, want), f"max diff {numpy.nanmax(numpy.abs(g - want)):.3e}"
    if wide is not None:
        outside = torch.isnan(wide).cpu().numpy()
        outside[1:1 + shape[0], 5:5 + shape[1]] = ~outside[1:1 + shape[0], 5:5 + shape[1]]
        assert outside.all(), "a sample outside the view was written"
    assert rec == rec_ref, (rec, rec_ref)
    return rec


def finish_real_rejects(core):
    """Host arrays, wrong dtypes and shapes, and masks of the wrong size are rejected."""
    dev = kc._dev(core)
    yN = core.yN_size
    acc = torch.zeros((yN, 4), dtype=torch.complex128, device=dev)
    out = torch.zeros((8, 4), dtype=torch.float64, device=dev)
    # pylint: disable=protected-access
    din, dout = core._describe(acc, 0), _lib.Lines(out.data_ptr(), 4, 8, 1, 4, _lib.DEVICE)
    for d in (din, dout):
        loc = d.location
        d.location = _lib.HOST
        with pytest.raises(ValueError, match="device arrays only"):
            _lib.check(core._lib, core._lib.swiftly_b200_finish_facet_real(
                core._plan, ctypes.byref(din), ctypes.byref(dout), 0, None, ctypes.c_void_p(0)))
        d.location = loc
    with pytest.raises(ValueError):
        core.finish_facet_real(acc, 0, 8, 0, out=out.to(torch.complex128))
    with pytest.raises(ValueError):
        core.finish_facet_real(acc, 0, 9, 0, out=out)
    with pytest.raises(ValueError):
        core.finish_facet_real(acc.to(torch.complex64), 0, 8, 0)
    with pytest.raises(ValueError):
        core.finish_facet_real(acc, 0, 8, 0, mask=torch.ones(7, dtype=torch.float64, device=dev))


# ---------------------------------------------------------------------- API level
def hermitian_subgrids(cfg, sg_cfgs, sources):
    """Subgrids of real point sources (the analytic DFT, with the configs' masks)."""
    N = cfg.image_size
    return [make_subgrid_from_sources(sources, N, sg.size, [sg.off0, sg.off1],
                                      [sg.mask0, sg.mask1]) for sg in sg_cfgs]


def _facets(bwd):
    return [numpy.asarray(t.result()) for t in bwd.finish()]


def unpaired_bitwise(cfg, facet_cfgs, sg_cfgs, subgrids, *, lru=1, budget=None):
    """Real mode fed through ``add_new_subgrid_task`` only: bitwise ``Re`` of the default mode
    (float64 facets); the default mode's ``add_subgrid_tasks`` bitwise its own loop."""
    res = {}
    for real in (False, True):
        bwd = SwiftlyBackward(cfg, facet_cfgs, lru_backward=lru, queue_size=4,
                              device_budget=budget, real_image=real)
        assert bwd.host_tier == (budget is not None)
        for sg, data in zip(sg_cfgs, subgrids):
            bwd.add_new_subgrid_task(sg, data)
        res[real] = _facets(bwd)
    bwd = SwiftlyBackward(cfg, facet_cfgs, lru_backward=lru, queue_size=4, device_budget=budget)
    assert bwd.add_subgrid_tasks(sg_cfgs, subgrids) == [(i, None) for i in range(len(sg_cfgs))]
    looped = _facets(bwd)
    for j, (a, b, c) in enumerate(zip(res[False], res[True], looped)):
        assert b.dtype == numpy.float64 and b.shape == a.shape
        assert numpy.array_equal(b, a.real), f"facet {j}: real mode is not Re of the default"
        assert numpy.array_equal(c, a), f"facet {j}: add_subgrid_tasks differs from the loop"
    return res[True]


class Work:
    """What a backward transform ran: subgrid sides (K4T launches, or ``prepare_subgrid`` on the
    unsplit fused path), ``merge_mirror_subgrid`` calls, and the subgrid columns folded
    (``fold_column``, one entry per call)."""

    def __init__(self):
        self.sides = 0
        self.merge = 0
        self.folds = []


@contextlib.contextmanager
def counting(core):
    """Count the work of ``core``'s callers into a :class:`Work` (test-local wrappers)."""
    work = Work()
    orig = {name: getattr(core, name) for name in
            ("split_subgrid_axis", "prepare_subgrid", "merge_mirror_subgrid", "fold_column")}

    def split(groups, axis, *a, **k):
        if axis == 0:
            work.sides += 1
        return orig["split_subgrid_axis"](groups, axis, *a, **k)

    def prepare(*a, **k):
        work.sides += 1
        return orig["prepare_subgrid"](*a, **k)

    def merge(*a, **k):
        work.merge += 1
        return orig["merge_mirror_subgrid"](*a, **k)

    def fold(accs, facet_accs, facet_off1s, masks1, subgrid_off0):
        work.folds.append(subgrid_off0 % core.N)
        return orig["fold_column"](accs, facet_accs, facet_off1s, masks1, subgrid_off0)

    core.split_subgrid_axis, core.prepare_subgrid = split, prepare
    core.merge_mirror_subgrid, core.fold_column = merge, fold
    try:
        yield work
    finally:
        for name in orig:
            delattr(core, name)


def paired_case(cfg, facet_cfgs, sg_cfgs, sources, *, subgrids=None, lru=1, budget=None,
                agree=1e-7):
    """Real mode through ``add_subgrid_tasks`` against the default mode on Hermitian subgrids of
    ``sources``: the real facets at most twice the default mode's error against the analytic
    facets, and within ``agree`` (relative to the largest true sample) of ``Re`` of the default
    facets.  With ``sources=None``, on the given ``subgrids``: the agreement only, relative to the
    largest default sample.  The work: one subgrid side per pair or unpaired config, one merge
    per pair.  Returns ``(plan, work, real facets, errors)``."""
    N = cfg.image_size
    if subgrids is None:
        subgrids = hermitian_subgrids(cfg, sg_cfgs, sources)
    ref = SwiftlyBackward(cfg, facet_cfgs, lru_backward=lru, queue_size=4)
    for sg, data in zip(sg_cfgs, subgrids):
        ref.add_new_subgrid_task(sg, data)
    default = _facets(ref)
    bwd = SwiftlyBackward(cfg, facet_cfgs, lru_backward=lru, queue_size=4, device_budget=budget,
                          real_image=True)
    assert bwd.host_tier == (budget is not None)
    with counting(cfg.core) as work:
        plan = bwd.add_subgrid_tasks(sg_cfgs, subgrids)
        real = _facets(bwd)
    assert plan == api.mirror_pairs(sg_cfgs, N, cfg.internal_subgrid_size)
    n_pairs = sum(j is not None for _, j in plan)
    assert (work.sides, work.merge) == (len(plan), n_pairs), (work.sides, work.merge)
    assert all(r.dtype == numpy.float64 for r in real)
    errs = {}
    if sources is None:
        scale = max(numpy.abs(d).max() for d in default)
    else:
        truth = [make_facet(N, fc, sources) for fc in facet_cfgs]
        scale = max(numpy.abs(t).max() for t in truth)
        errs["real"] = max(numpy.abs(r - t).max() for r, t in zip(real, truth)) / scale
        errs["default"] = max(numpy.abs(d - t).max() for d, t in zip(default, truth)) / scale
        assert errs["real"] <= 2 * errs["default"], errs
    errs["agree"] = max(numpy.abs(r - d.real).max() for r, d in zip(real, default)) / scale
    assert errs["agree"] <= agree, errs
    return plan, work, real, errs


def full_cover_work(n):
    """A full ``n x n`` cover in cover order: subgrid sides (``n^2/2 + 2``: one per pair plus the
    four self-mirrored subgrids), merges, and columns folded (``n/2 + 1``)."""
    sides = n * n // 2 + 2
    return sides, sides - 4, n // 2 + 1


def round_trip(cfg, facet_cfgs, sg_cfgs, sources):
    """Forward then backward on real point-source facets, default and real mode (both
    directions); the worst facet RMS error of each against the sources."""
    facets = [make_facet(cfg.image_size, fc, sources).real for fc in facet_cfgs]
    errs = {}
    for real in (False, True):
        fwd = SwiftlyForward(cfg, list(zip(facet_cfgs, facets)), queue_size=100, real_image=real)
        subgrids = [None] * len(sg_cfgs)
        for idx, task in fwd.iter_subgrid_tasks(sg_cfgs):
            subgrids[idx] = task
        bwd = SwiftlyBackward(cfg, facet_cfgs, queue_size=100, real_image=real)
        bwd.add_subgrid_tasks(sg_cfgs, subgrids)
        errs[real] = max(check_facet(cfg.image_size, fc, t.result(), sources)
                         for fc, t in zip(facet_cfgs, bwd.finish()))
    if errs[False] < 3e-10:
        assert errs[True] < 3e-10, errs
    return errs
