"""
Shared checks of the half-row layout of real images (include/swiftly_b200.h, "Half rows"), run by
tests/test_emu_half_rows.py on the host-emulated kernels and by tests/test_gpu_half_rows.py on the
H100.

Kernel level, bitwise: ``prepare_facet_real_half`` against the rows ``d <= yN/2`` of
``prepare_facet(window_lines=True)`` on the promoted facet; ``extract_columns`` on half rows
against the call on their full Hermitian extension, in the same launch form; ``fold_column`` into
half accumulators against the host fold of the full-row result, with its runs checked for
distinct targets; ``finish_facet_real_half`` against ``finish_facet_real`` of the extension.
API level: ``half_rows=True`` against ``real_image=True`` alone, the analytic DFT and a round trip.
"""

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
from tests import k2_cases as kc
from tests import real_backward_cases as rb
from tests import real_image_cases as rc

NAN = complex(numpy.nan, numpy.nan)

# relative bound of half_rows=True against real_image=True alone (DESIGN section 4.10): the two
# differ by the rounding of K1's mirrored rows only
AGREE = 1e-12


def centred(yN, d):
    """Centred row held by stored row ``d``."""
    return (yN // 2 + d) % yN


def half_row(r, yN):
    """``(stored row, conj)`` of centred row ``r``."""
    d = (r - yN // 2) % yN
    return (d, False) if d <= yN // 2 else (yN - d, True)


def hermitian_full(H, yN):
    """The full ``yN``-row Hermitian extension of half rows ``H`` (stored rows 0 and yN/2 made
    real in both), rows in centred order."""
    H = H.copy()
    H[0] = H[0].real
    H[yN // 2] = H[yN // 2].real
    full = numpy.empty((yN,) + H.shape[1:], dtype=complex)
    for d in range(yN // 2 + 1):
        full[centred(yN, d)] = H[d]
        if 0 < d < yN // 2:
            full[centred(yN, -d)] = numpy.conj(H[d])
    return H, full


def _rand(rng, shape):
    return rng.standard_normal(shape) + 1j * rng.standard_normal(shape)


# ---------------------------------------------------------------------- K1
def k1_case(core, fs, n_lines, *, axis=0, off=0, wide=False, variant=0, force_split=0, seed=0):
    """``prepare_facet_real_half`` bitwise the half rows of ``prepare_facet(window_lines=True)``
    on the facet promoted to complex, in the same launch form.  Returns the record."""
    rng = numpy.random.default_rng(seed)
    yN, half = core.yN_size, core.half_rows
    shape = (fs, n_lines) if axis == 0 else (n_lines, fs)
    facet = kc._to(core, rng.standard_normal(shape))
    oshape = (half, n_lines) if axis == 0 else (n_lines, half)
    home = None
    out = None
    if wide:
        home = torch.full((oshape[0] + 3, oshape[1] + 5), NAN, dtype=torch.complex128,
                          device=facet.device)
        out = home[1:1 + oshape[0], 2:2 + oshape[1]]
    with kc.hooks(core, variant, 0, force_split):
        ref = core.prepare_facet(facet.to(torch.complex128), off, axis, window_lines=True)
        rec_ref = kc.last_launch(core)
        got = core.prepare_facet_real_half(facet, off, axis, out=out)
        rec = kc.last_launch(core)
    rows = [centred(yN, d) for d in range(half)]
    want = ref.cpu().numpy()
    want = want[rows] if axis == 0 else want[:, rows]
    g = got.cpu().numpy()
    assert g.shape == oshape
    assert numpy.array_equal(g, want), f"max diff {numpy.nanmax(numpy.abs(g - want)):.3e}"
    if home is not None:
        outside = torch.isnan(torch.view_as_real(home)).all(-1).cpu().numpy()
        outside[1:1 + oshape[0], 2:2 + oshape[1]] ^= True
        assert outside.all(), "a sample outside the view was written"
    assert rec == rec_ref, (rec, rec_ref)
    return rec


# ---------------------------------------------------------------------- K2
def k2_case(core, sizes, offs, sg_off0, *, prewindowed=True, variant=0, force_split=0, cap=0,
            seed=0, ref_hooks=None):
    """``extract_columns`` on half rows bitwise the call on their full Hermitian extension (under
    ``ref_hooks = (variant, force_split)``, by default the half call's).  Returns ``(half
    record, half cluster, full record, full cluster)``."""
    rng = numpy.random.default_rng(seed)
    yN, half = core.yN_size, core.half_rows
    halves, fulls = [], []
    for fs in sizes:
        H, full = hermitian_full(_rand(rng, (half, fs)), yN)
        halves.append(kc._to(core, H))
        fulls.append(kc._to(core, full))
    cluster = core._lib.swiftly_b200_debug_last_cluster
    cluster.argtypes = [ctypes.c_void_p]
    with kc.hooks(core, variant, cap, force_split):
        got = core.extract_columns(halves, sg_off0, offs, prewindowed=prewindowed)
        rec, cl = kc.last_launch(core), cluster(core._plan)
    ref_variant, ref_split = ref_hooks or (variant, force_split)
    with kc.hooks(core, ref_variant, cap, ref_split):
        want = core.extract_columns(fulls, sg_off0, offs, prewindowed=prewindowed)
        rec_ref, cl_ref = kc.last_launch(core), cluster(core._plan)
    for j, (g, w) in enumerate(zip(got, want)):
        g, w = g.cpu().numpy(), w.cpu().numpy()
        assert numpy.array_equal(g, w), f"facet {j}: max diff {numpy.abs(g - w).max():.3e}"
    return rec, cl, rec_ref, cl_ref


def window_kinds(core):
    """Subgrid off0 of columns whose window straddles centred offset 0, straddles yN/2, and
    neither."""
    N = core.N
    return {"zero": 0, "nyquist": N // 2, "neither": N // 4 + core.subgrid_off_step}


# ---------------------------------------------------------------------- fold
def fold_runs(core):
    fn = core._lib.swiftly_b200_debug_fold_runs
    fn.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int)]
    fn.restype = ctypes.c_int
    buf = (ctypes.c_int * 24)()
    n = fn(core._plan, buf)
    return [tuple(buf[3 * i:3 * i + 3]) for i in range(n)]


def fold_case(core, sizes, offs, sg_off0, *, masked=(), force_split=0, cap=0, seed=0):
    """One ``fold_column`` into zeroed half accumulators bitwise the host fold of the full-row
    result, ``H[d] = x[d] + conj(x[-d])`` (``H = x`` on the self-conjugate rows).  The runs of
    the call: every window row once, pass 1 before pass 2, and no run with two lines of one
    target.  Returns the runs."""
    rng = numpy.random.default_rng(seed)
    yN, m, half = core.yN_size, core.xM_yN_size, core.half_rows
    accs = [kc._to(core, _rand(rng, (m, yN))) for _ in sizes]
    masks = [kc._to(core, (rng.random(fs) > 0.3).astype(float)) if j in masked else None
             for j, fs in enumerate(sizes)]
    dev = accs[0].device
    full = [torch.zeros((yN, fs), dtype=torch.complex128, device=dev) for fs in sizes]
    halves = [torch.zeros((half, fs), dtype=torch.complex128, device=dev) for fs in sizes]
    with kc.hooks(core, 0, cap, force_split):
        core.fold_column(accs, full, offs, masks, sg_off0)
        core.fold_column(accs, halves, offs, masks, sg_off0)
    runs = fold_runs(core)
    for j, (x, g) in enumerate(zip(full, halves)):
        x, g = x.cpu().numpy(), g.cpu().numpy()
        want = numpy.empty_like(g)
        for d in range(half):
            want[d] = x[centred(yN, d)]
            if 0 < d < yN // 2:
                want[d] = want[d] + numpy.conj(x[centred(yN, -d)])
        assert numpy.array_equal(g, want), f"facet {j}: max diff {numpy.abs(g - want).max():.3e}"
    base0 = api.window_start(core, sg_off0)
    seen = []
    for u_lo, cnt, pas in runs:
        targets = [half_row((base0 + u) % yN, yN)[0] for u in range(u_lo, u_lo + cnt)]
        assert len(set(targets)) == cnt, f"run {(u_lo, cnt, pas)} has a shared target"
        seen += range(u_lo, u_lo + cnt)
    assert sorted(seen) == list(range(m)), runs
    passes = [p for _, _, p in runs]
    assert passes == sorted(passes), runs
    return runs


def straddles(core, sg_off0):
    """True when the column's window holds two rows of one half-row target."""
    yN, m = core.yN_size, core.xM_yN_size
    base0 = api.window_start(core, sg_off0)
    targets = [half_row((base0 + u) % yN, yN)[0] for u in range(m)]
    return len(set(targets)) < m


# ---------------------------------------------------------------------- finish
def finish_case(core, fs, *, n_lines=5, masked=True, force_split=0, seed=0):
    """``finish_facet_real_half`` bitwise ``finish_facet_real`` of the full line built on the host
    from its Hermitian part, along axis 0, in the same launch form."""
    rng = numpy.random.default_rng(seed)
    yN, half = core.yN_size, core.half_rows
    H = _rand(rng, (half, n_lines))
    nat = numpy.empty((yN, n_lines), dtype=complex)
    nat[0] = H[0].real
    nat[yN // 2] = H[yN // 2].real
    nat[1:yN // 2] = 0.5 * H[1:yN // 2]
    nat[yN // 2 + 1:] = numpy.conj(0.5 * H[1:yN // 2])[::-1]
    full = numpy.roll(nat, yN // 2, axis=0)  # natural index q at centred q + yN/2
    mask = kc._to(core, (rng.random(fs) > 0.3).astype(float)) if masked else None
    off = int(rng.integers(-3, 4)) * core.facet_off_step
    with kc.hooks(core, 0, 0, force_split):
        want = core.finish_facet_real(kc._to(core, full), off, fs, 0, mask=mask)
        rec_ref = kc.last_launch(core)
        got = core.finish_facet_real_half(kc._to(core, H), off, fs, 0, mask=mask)
        rec = kc.last_launch(core)
    g, w = got.cpu().numpy(), want.cpu().numpy()
    assert numpy.array_equal(g, w), f"max diff {numpy.abs(g - w).max():.3e}"
    assert rec == rec_ref, (rec, rec_ref)
    return rec


def finish_rejects(core):
    """Wrong line length and host arrays are EINVAL (ValueError)."""
    dev = kc._dev(core)
    yN, half = core.yN_size, core.half_rows
    with pytest.raises(ValueError, match="line length"):
        core.finish_facet_real_half(torch.zeros((yN, 3), dtype=torch.complex128, device=dev),
                                    0, 8, 0)
    acc = numpy.zeros((half, 3), dtype=complex)
    out = numpy.zeros((8, 3))
    din = _lib.Lines(acc.ctypes.data, 3, half, 1, 3, _lib.HOST)
    dout = _lib.Lines(out.ctypes.data, 3, 8, 1, 3, _lib.HOST)
    rc_ = core._lib.swiftly_b200_finish_facet_real_half(
        core._plan, ctypes.byref(din), ctypes.byref(dout), 0, None, None)
    assert rc_ == _lib.EINVAL and "device arrays only" in _lib.last_error(core._lib)


def odd_rejects(core):
    """A plan with odd yN rejects every half-row entry point."""
    dev = kc._dev(core)
    yN = core.yN_size
    assert yN % 2 == 1
    with pytest.raises(ValueError, match="even"):
        core.finish_facet_real_half(torch.zeros((yN // 2 + 1, 2), dtype=torch.complex128,
                                                device=dev), 0, 1, 0)
    with pytest.raises(ValueError, match="even"):
        core.prepare_facet_real_half(torch.zeros((1, 2), dtype=torch.float64, device=dev), 0)


# ---------------------------------------------------------------------- API
def forward_case(cfg, facet_cfgs, sg_cfgs, sources, *, lru=1):
    """``SwiftlyForward(real_image=True, half_rows=True)`` against ``real_image=True`` alone
    (within AGREE of the largest sample) and against the analytic DFT (at most twice the
    full-row error, plus the agreement bound).  Returns the errors."""
    N = cfg.image_size
    facets = [make_facet(N, fc, sources).real for fc in facet_cfgs]
    res = {}
    for half in (False, True):
        fwd = SwiftlyForward(cfg, list(zip(facet_cfgs, facets)), lru_forward=lru,
                             queue_size=100, real_image=True, half_rows=half)
        if half:
            assert all(b.shape == (cfg.core.half_rows, fc.size)
                       for b, fc in zip(fwd._get_BF_Fs(), facet_cfgs))
        got = [None] * len(sg_cfgs)
        for idx, task in fwd.iter_subgrid_tasks(sg_cfgs):
            got[idx] = torch.from_numpy(numpy.array(task.result()))
        res[half] = got
    scale = max(float(numpy.abs(g.cpu().numpy()).max()) for g in res[False])
    agree = max(float(numpy.abs((a - b).cpu().numpy()).max())
                for a, b in zip(res[False], res[True])) / scale
    errs = {"agree": agree, "full": 0.0, "half": 0.0}
    for k in range(0, len(sg_cfgs), max(1, len(sg_cfgs) // 6)):
        e_full, e_half = rc.rel_errs(N, sg_cfgs[k], [res[False][k], res[True][k]], sources)
        errs["full"] = max(errs["full"], e_full)
        errs["half"] = max(errs["half"], e_half)
    assert agree <= AGREE, errs
    assert errs["half"] <= 2 * errs["full"] + AGREE, errs
    return errs


def forward_lockstep(cfg, facet_cfgs, facets, sg_cfgs, sources, *, n_checked=3):
    """Both forward modes side by side, subgrid by subgrid (a large cover never holds all its
    subgrids): agreement within AGREE of each subgrid's largest sample, and ``n_checked``
    subgrids against the analytic DFT.  Returns the errors."""
    N = cfg.image_size
    fwds = [SwiftlyForward(cfg, list(zip(facet_cfgs, facets)), queue_size=4, real_image=True,
                           half_rows=half) for half in (False, True)]
    checked = set(range(0, len(sg_cfgs), max(1, len(sg_cfgs) // n_checked)))
    errs = {"agree": 0.0, "full": 0.0, "half": 0.0}
    for (i, a), (j, b) in zip(*(f.iter_subgrid_tasks(sg_cfgs) for f in fwds)):
        assert i == j
        a, b = (torch.as_tensor(t.result()) for t in (a, b))
        scale = float(a.abs().max())
        errs["agree"] = max(errs["agree"], float((a - b).abs().max()) / scale)
        if i in checked:
            e_full, e_half = rc.rel_errs(N, sg_cfgs[i], [a, b], sources)
            errs["full"] = max(errs["full"], e_full)
            errs["half"] = max(errs["half"], e_half)
    assert errs["agree"] <= AGREE, errs
    assert errs["half"] <= 2 * errs["full"] + AGREE, errs
    return errs


def backward_case(cfg, facet_cfgs, sg_cfgs, sources, *, lru=1, subgrids=None):
    """``SwiftlyBackward(real_image=True, half_rows=True)`` against ``real_image=True`` alone and
    (with ``sources``) against the analytic facets.  Returns the errors."""
    N = cfg.image_size
    if subgrids is None:
        subgrids = rb.hermitian_subgrids(cfg, sg_cfgs, sources)
    res = {}
    for half in (False, True):
        bwd = SwiftlyBackward(cfg, facet_cfgs, lru_backward=lru, queue_size=100,
                              real_image=True, half_rows=half)
        bwd.add_subgrid_tasks(sg_cfgs, subgrids)
        if half:
            assert all(a is None or a.shape[0] == cfg.core.half_rows
                       for a in bwd.MNAF_BMNAFs_persist)
        res[half] = [numpy.asarray(t.result()) for t in bwd.finish()]
    assert all(r.dtype == numpy.float64 for r in res[True])
    if sources is None:
        scale = max(numpy.abs(a).max() for a in res[False])
        errs = {"agree": max(numpy.abs(a - b).max() for a, b in zip(res[False], res[True])) / scale}
        assert errs["agree"] <= AGREE, errs
        return errs
    truth = [make_facet(N, fc, sources) for fc in facet_cfgs]
    scale = max(numpy.abs(t).max() for t in truth)
    errs = {
        "agree": max(numpy.abs(a - b).max() for a, b in zip(res[False], res[True])) / scale,
        "full": max(numpy.abs(a - t).max() for a, t in zip(res[False], truth)) / scale,
        "half": max(numpy.abs(b - t).max() for b, t in zip(res[True], truth)) / scale,
    }
    assert errs["agree"] <= AGREE, errs
    assert errs["half"] <= 2 * errs["full"] + AGREE, errs
    return errs


def round_trip(cfg, facet_cfgs, sg_cfgs, sources):
    """Forward then backward, both with half rows: the facets within the reference's 3e-10 RMS
    of the sources (when full-row real mode is)."""
    facets = [make_facet(cfg.image_size, fc, sources).real for fc in facet_cfgs]
    errs = {}
    for half in (False, True):
        fwd = SwiftlyForward(cfg, list(zip(facet_cfgs, facets)), queue_size=100,
                             real_image=True, half_rows=half)
        subgrids = [None] * len(sg_cfgs)
        for idx, task in fwd.iter_subgrid_tasks(sg_cfgs):
            subgrids[idx] = task
        bwd = SwiftlyBackward(cfg, facet_cfgs, queue_size=100, real_image=True, half_rows=half)
        bwd.add_subgrid_tasks(sg_cfgs, subgrids)
        errs[half] = max(check_facet(cfg.image_size, fc, t.result(), sources)
                         for fc, t in zip(facet_cfgs, bwd.finish()))
    if errs[False] < 3e-10:
        assert errs[True] < 3e-10, errs
    return errs


def api_rejects(cfg, facet_cfgs, sources):
    """half_rows without real_image, bf_f_buffers of the wrong shape (ValueError), a budget below
    the half-row estimate (NotImplementedError, both directions)."""
    N = cfg.image_size
    core = cfg.core
    facets = [make_facet(N, fc, sources).real for fc in facet_cfgs]
    tasks = list(zip(facet_cfgs, facets))
    with pytest.raises(ValueError, match="real_image"):
        SwiftlyForward(cfg, tasks, half_rows=True)
    with pytest.raises(ValueError, match="real_image"):
        SwiftlyBackward(cfg, facet_cfgs, half_rows=True)
    dev = kc._dev(core)
    bad = [torch.empty((core.yN_size, fc.size), dtype=torch.complex128, device=dev)
           for fc in facet_cfgs]
    with pytest.raises(ValueError, match="bf_f_buffers"):
        SwiftlyForward(cfg, tasks, real_image=True, half_rows=True, bf_f_buffers=bad)
    with pytest.raises(NotImplementedError, match="budget"):
        SwiftlyForward(cfg, tasks, real_image=True, half_rows=True, device_budget=1)
    with pytest.raises(NotImplementedError, match="budget"):
        SwiftlyBackward(cfg, facet_cfgs, real_image=True, half_rows=True, device_budget=1)
    # the device-tier estimate counts yN // 2 + 1 rows for the facet arrays
    yN, m = core.yN_size, core.xM_yN_size
    sizes = [fc.size for fc in facet_cfgs]
    for direction in ("forward", "backward"):
        full = api.device_tier_bytes(direction, yN, m, sizes, 1, 2, 8)
        half = api.device_tier_bytes(direction, yN, m, sizes, 1, 2, 8, half_rows=True)
        assert full - half == 16 * (yN - yN // 2 - 1) * sum(sizes)
