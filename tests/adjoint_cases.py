"""
The backward transform as the adjoint of the forward transform, shared by the emulated and the
GPU tests.

Per axis every forward primitive is the adjoint of its backward twin up to a constant,
``<y, A x> = c <A^T y, x>`` with ``<a, b> = sum conj(a) b``:

============================  ==================================  ===========
forward ``A``                 backward ``A^T``                    ``c``
============================  ==================================  ===========
``prepare_facet``             ``finish_facet``                    ``1 / yN``
``extract_from_facet``        ``add_to_facet``                    ``1``
``add_to_subgrid``            ``extract_from_subgrid``            ``m``
``finish_subgrid``            ``prepare_subgrid``                 ``1 / xM``
============================  ==================================  ===========

(the numpy FFTs of the oracle: the inverse transform carries ``1 / n``).  The product per axis is
``m / (yN xM) = 1 / N``, so over both axes ``N^2 sum_i <S_i, fwd(F)_i> = sum_j <bwd(S)_j, F_j>``.

A fused kernel is a chain of these, so each fused pair has the product of its links' constants
(:func:`constants`): K2 (``extract_columns``) and ``fold_column`` ``1 / yN``, K3 / K4
(``sum_finish_axis``) and ``split_subgrid_axis`` ``m / xM``, ``subgrid_to_facets`` ``m``.  The
forward twins are tied to the oracle and to extended precision elsewhere, so the identity checks
every backward kernel at any size, with no oracle evaluation.

Two kinds of probe: random complex operands check the whole operator; a delta probe (a single
unit sample in ``y`` or in ``x``) makes the identity an element-wise check of one output sample
of the other side, which an error confined to that sample cannot hide from.

Masks: the forward transform masks subgrids, the backward transform masks facets (and the fused
backward kernels mask facet columns).  A mask ``M`` on one side is moved onto the other side's
input: ``<y, A x> = c <M A^T y, x> = c <A^T y, M x>``, so the forward operand is multiplied by
the masks the backward side applies, and the backward operand by those the forward side applies.

Real images: for a real operand the identity holds with the real inner product ``Re <a, b>``;
the half-row forms store ``yN / 2 + 1`` rows whose other rows are the conjugates, which is the
adjoint pair ``E`` (extend) / ``E^T`` (fold the conjugate of the mirrored row onto its twin) of
that inner product.
"""

import contextlib
import ctypes
import gc
import random

import numpy
import torch

from ska_sdp_distributed_fourier_transform_b200 import (
    SwiftlyBackward,
    SwiftlyForward,
)
from ska_sdp_distributed_fourier_transform_b200.api import mirror_pairs
from tests import k2_cases as kc
from tests import length_cases as lc
from tests import pair_cases as prc
from tests import parity_cases as pc
from tests import subgrid_line_cases as slc

EPS = lc.EPS

# Bound of one kernel pair, in units of EPS * log2(n) of the norm product (n: the longest
# transform of the pair).  See DESIGN.md section 6 for the residuals measured per form.
PAIR_BOUND = 1.0
# Bound of the driver chains (SwiftlyForward <-> SwiftlyBackward), relative to the norm product,
# where the facet window is mild (see chain_bound)
CHAIN_BOUND = 1e-12


def pair_bound(n):
    return PAIR_BOUND * EPS * numpy.log2(n)


def window_gain(core, facet_size):
    """``max / min`` of the facet window ``Fb`` over ``facet_size`` samples: 16 at cfg2 and cfg4
    (yB / yN = 0.5), 4.9e3 at yB / yN = 0.8125, 1.7e6 at 16k[1]-n2k-1k (0.89)."""
    w = fb_window(core, facet_size)
    return float(w.max() / w.min())


def chain_bound(cfg):
    """Bound of a driver chain: :data:`CHAIN_BOUND`, or ``8 eps`` times the facet window's gain
    where that is larger.  The window does inflate the residual relative to the norm product:
    the rounding of the samples it weights most is not weighted down again, so at
    16k[1]-n2k-1k (gain 1.7e6) the H100 measures 3.2e-11 where the yB / yN = 0.5 geometries stay
    below 1e-18; the oracle's chain shows the same growth (2.4e-13 at gain 6.4e4)."""
    return max(CHAIN_BOUND, 8 * EPS * window_gain(cfg.core, cfg.max_facet_size))


# ---------------------------------------------------------------------- the identity
def _host(a):
    if isinstance(a, torch.Tensor):
        a = a.detach().cpu().numpy()
    return numpy.asarray(a)


def _parts(a):
    return list(a) if isinstance(a, (list, tuple)) else [a]


def _ld(a):
    return _host(a).astype(numpy.clongdouble).ravel()


def inner(a, b, real=False):
    """``<a, b> = sum conj(a) b`` over every part of ``a`` / ``b`` (arrays, tensors or lists of
    them), accumulated in ``numpy.longdouble`` on the host; ``real``: its real part."""
    pa, pb = _parts(a), _parts(b)
    assert len(pa) == len(pb), (len(pa), len(pb))
    tot = numpy.clongdouble(0)
    for p, q in zip(pa, pb):
        p, q = _ld(p), _ld(q)
        assert p.shape == q.shape, (p.shape, q.shape)
        tot += numpy.dot(numpy.conj(p), q)
    return tot.real if real else tot


def norm(a):
    tot = numpy.longdouble(0)
    for p in _parts(a):
        p = _ld(p)
        tot += (p.real * p.real + p.imag * p.imag).sum()
    return numpy.sqrt(tot)


def adjoint_residual(y, Ax, ATy, x, c, real=False):
    """``|<y, Ax> - c <ATy, x>| / (|y| |Ax| + |c| |ATy| |x|)``, in ``numpy.longdouble`` on the
    host (``real``: the real inner product)."""
    c = numpy.longdouble(c)
    lhs = inner(y, Ax, real)
    rhs = inner(ATy, x, real)
    den = norm(y) * norm(Ax) + abs(c) * norm(ATy) * norm(x)
    assert den > 0
    return float(abs(lhs - c * rhs) / den)


def constants(core):
    """The per-axis constants of the table above, from the plan's sizes."""
    yN, m, xM = core.yN_size, core.xM_yN_size, core.xM_size
    return {"facet": 1.0 / yN, "window": 1.0, "subgrid": float(m), "finish": 1.0 / xM}


def chain_constant(core, links):
    c = 1.0
    for link in links:
        c *= constants(core)[link]
    return c


K1 = ("facet",)
K2 = ("window", "facet")  # extract_from_facet(axis 0) -> prepare_facet(axis 1)
K34 = ("window", "subgrid", "finish")  # sum_finish_axis on prepared facet lines
K34_CONTRIB = ("subgrid", "finish")  # sum_finish_axis on contributions
TO_FACETS = ("window", "subgrid")  # subgrid_to_facets: extract_from_subgrid -> add_to_facet
AXIS = ("facet", "window", "subgrid", "finish")


# ---------------------------------------------------------------------- probes
def rand_c(rng, shape):
    return pc.rand_c(rng, *shape)


def delta(shape, index):
    """A unit sample at ``index`` (a tuple, negative entries count from the end)."""
    a = numpy.zeros(shape, dtype=complex)
    a[tuple(index)] = 1.0
    return a


def _dev(core):
    return lc._dev(core)  # pylint: disable=protected-access


def _to(core, a):
    return lc._to(core, a)  # pylint: disable=protected-access


def _lines(a, axis):
    """Lines-first array ``a`` ``(lines, samples)`` as an array with samples along ``axis``."""
    return numpy.ascontiguousarray(a if axis == 1 else a.T)


def is_emulated(core):
    return kc.is_emulated(core)


def fb_window(core, n):
    """The kernels' ``extract_mid(Fb, n)`` as float64."""
    return numpy.asarray(lc._window_of(core, n), dtype=float)  # pylint: disable=protected-access


# ---------------------------------------------------------------------- the oracle
def oracle_pairs(oracle, seed=0):
    """Every primitive pair of the oracle at odd sizes and offsets past +-N: returns
    ``{name: residual}``; each pair's constant comes from :func:`constants`."""
    rng = numpy.random.default_rng(seed)
    N, yN, m, xM = oracle.N, oracle.yN_size, oracle.xM_yN_size, oracle.xM_size
    c = constants(oracle)
    fs, sz = yN - 1 if yN % 2 == 0 else yN, xM - 3
    fo, so = oracle.facet_off_step, oracle.subgrid_off_step
    out = {}
    for k, (foff, soff) in enumerate([(0, 0), (-N - 3 * fo, N + 5 * so), (N + fo, -2 * N - so)]):
        x, y = rand_c(rng, (fs,)), rand_c(rng, (yN,))
        out[f"facet {k}"] = adjoint_residual(
            y, oracle.prepare_facet(x, foff, 0), oracle.finish_facet(y, foff, fs, 0), x,
            c["facet"])
        x, y = rand_c(rng, (yN,)), rand_c(rng, (m,))
        out[f"window {k}"] = adjoint_residual(
            y, oracle.extract_from_facet(x, soff, 0), oracle.add_to_facet(y, soff, 0), x,
            c["window"])
        x, y = rand_c(rng, (m,)), rand_c(rng, (xM,))
        out[f"subgrid {k}"] = adjoint_residual(
            y, oracle.add_to_subgrid(x, foff, 0), oracle.extract_from_subgrid(y, foff, 0), x,
            c["subgrid"])
        x, y = rand_c(rng, (xM,)), rand_c(rng, (sz,))
        out[f"finish {k}"] = adjoint_residual(
            y, oracle.finish_subgrid(x, soff, sz), oracle.prepare_subgrid(y, soff), x,
            c["finish"])
    return out


def oracle_drivers(oracle, facet_offs, fs, subgrid_offs, sz, seed=0):
    """``forward_reference_order`` against ``backward_reference_order`` with the constant of
    both axes' chains: the residual."""
    from oracle.swiftly_oracle import (  # pylint: disable=import-outside-toplevel
        backward_reference_order,
        forward_reference_order,
    )

    rng = numpy.random.default_rng(seed)
    facets = [rand_c(rng, (fs, fs)) for _ in facet_offs]
    subgrids = [rand_c(rng, (sz, sz)) for _ in subgrid_offs]
    fwd = forward_reference_order(oracle, facets, facet_offs, subgrid_offs, sz)
    bwd = backward_reference_order(oracle, subgrids, subgrid_offs, facet_offs, fs)
    return adjoint_residual(subgrids, fwd, bwd, facets, chain_constant(oracle, AXIS) ** 2)


# ---------------------------------------------------------------------- hooks
@contextlib.contextmanager
def hooks(core, variant=0, cap=0, force_split=0):
    with kc.hooks(core, variant, cap, force_split):
        yield


def last_launch(core):
    return prc.last_launch(core)


def last_cluster(core):
    fn = core._lib.swiftly_b200_debug_last_cluster  # pylint: disable=protected-access
    fn.argtypes, fn.restype = [ctypes.c_void_p], ctypes.c_int
    return fn(core._plan)  # pylint: disable=protected-access


def line_record(n, n_lines, adjacent, cap=0):
    """Launch record of an ``n``-point facet or subgrid line transform of ``n_lines`` lines:
    ``(kernel, lines per CTA or F, line-fastest flag, grid)``."""
    rec = kc.generic_form(n, n_lines, cap)
    if rec[0] == kc.LINE:
        rec = (rec[0], rec[1], int(adjacent and n_lines > 1 and rec[1] > 1), rec[3])
    return rec


def _expect(got, want, what):
    assert tuple(got) == tuple(want), f"{what}: launched {got}, expected {want}"


# ---------------------------------------------------------------------- K1 <-> finish_facet
def facet_pair(core, axis, n_lines, fs, off, *, masked=False, probe=None, two_pass=False,
               cap=0, seed=0):
    """``prepare_facet`` (``fs`` samples along ``axis`` into ``yN``) against ``finish_facet``
    (``mask`` on the finish side moved onto ``x``).  ``probe``: None (random operands),
    ``("y", line, sample)`` or ``("x", line, sample)`` (a delta in that operand, indices
    lines-first).  Asserts both launches; returns the residual."""
    rng = numpy.random.default_rng(seed)
    yN = core.yN_size
    x = rand_c(rng, (n_lines, fs))
    y = rand_c(rng, (n_lines, yN))
    if probe is not None:
        which, line, sample = probe
        if which == "y":
            y = delta((n_lines, yN), (line, sample))
        else:
            x = delta((n_lines, fs), (line, sample))
    mask = (rng.random(fs) > 0.3).astype(float) if masked else None
    xm = x if mask is None else x * mask[None, :]
    what = f"yN {yN} axis {axis}, {n_lines} lines, fs {fs}, off {off}"
    with hooks(core, cap=cap):
        Ax = core.prepare_facet(_to(core, _lines(xm, axis)), off, axis=axis)
        rec_a = last_launch(core)
        ATy = core.finish_facet(_to(core, _lines(y, axis)), off, fs, axis=axis,
                                mask=None if mask is None else _to(core, mask))
        rec_b = last_launch(core)
    want = line_record(yN, n_lines, axis == 0, cap)
    if two_pass:  # the record of pass B: n1 * lines transforms of n2 = yN / n1 points, adjacent
        n1 = 1 << (int(numpy.log2(yN)) + 1) // 2
        _expect(rec_a, line_record(yN // n1, n1 * n_lines, True, cap),
                f"two-pass prepare_facet, {what}")
    else:
        _expect(rec_a, want, f"prepare_facet, {what}")
    _expect(rec_b, want, f"finish_facet, {what}")
    Ax, ATy = _host(Ax), _host(ATy)
    if axis == 0:
        Ax, ATy = Ax.T, ATy.T
    return adjoint_residual(y, Ax, ATy, x, chain_constant(core, K1))


def facet_plan_cases(core, plan, seed=0):
    """The identity of one facet-line plan (``length_cases.yn_plans``) on random and delta
    probes: both axes, odd and even facet sizes, offsets at and beyond +-N, a mask.  Returns the
    worst residual."""
    yN, N, step = core.yN_size, core.N, core.facet_off_step
    odd, even, full = lc.facet_sizes(yN)
    worst = 0.0
    if plan[0] == "twopass":
        n = lc.TWO_PASS_COLUMNS
        cases = [(0, n, full, N + 2 * step, False, None),
                 (0, n + 3, odd, -N, True, None),
                 (0, n, odd, -3 * step, False, ("x", n - 1, 0)),
                 (0, n, odd, 5 * step, False, ("x", 0, odd - 1))]
        for k, (axis, lines, fs, off, masked, probe) in enumerate(cases):
            worst = max(worst, facet_pair(core, axis, lines, fs, off, masked=masked,
                                          probe=probe, two_pass=True, seed=seed + k))
        return worst
    cases = [(1, 3, full, N + 2 * step, False, None),
             (0, 5, odd, -3 * step, True, None),
             (1, 2, even, -N, True, None),
             (0, 4, full, N, False, None),
             # delta probes: first and last sample of an odd facet, first and last line
             (1, 3, odd, -2 * step, False, ("x", 0, 0)),
             (0, 5, odd, N + step, False, ("x", 4, odd - 1)),
             # a single output sample of prepare_facet: the centre and the last bin
             (1, 2, odd, 3 * step, False, ("y", 1, yN // 2)),
             (0, 3, even, -step, False, ("y", 2, yN - 1))]
    for k, (axis, lines, fs, off, masked, probe) in enumerate(cases):
        worst = max(worst, facet_pair(core, axis, lines, fs, off, masked=masked, probe=probe,
                                      seed=seed + k))
    return worst


def finish_real_pair(core, axis, n_lines, fs, off, *, masked=False, probe=None, seed=0):
    """``prepare_facet`` of a real facet against ``finish_facet_real`` (real inner product)."""
    rng = numpy.random.default_rng(seed)
    yN = core.yN_size
    x = rng.standard_normal((n_lines, fs))
    y = rand_c(rng, (n_lines, yN))
    if probe is not None:
        x = numpy.zeros_like(x)
        x[probe] = 1.0
    mask = (rng.random(fs) > 0.3).astype(float) if masked else None
    xm = x if mask is None else x * mask[None, :]
    Ax = core.prepare_facet(_to(core, _lines(xm, axis)).to(torch.complex128), off, axis=axis)
    rec_a = last_launch(core)
    ATy = core.finish_facet_real(_to(core, _lines(y, axis)), off, fs, axis,
                                 mask=None if mask is None else _to(core, mask))
    rec_b = last_launch(core)
    want = line_record(yN, n_lines, axis == 0)
    _expect(rec_a, want, "prepare_facet (real facet)")
    _expect(rec_b, want, "finish_facet_real")
    Ax, ATy = _host(Ax), _host(ATy)
    if axis == 0:
        Ax, ATy = Ax.T, ATy.T
    return adjoint_residual(y, Ax, ATy, x, chain_constant(core, K1), real=True)


def half_rows_of(yN, d):
    """Centred row held by stored half row ``d``."""
    return (yN // 2 + d) % yN


def finish_half_pair(core, axis, n_lines, fs, off, *, masked=False, probe=None, seed=0):
    """``prepare_facet_real_half`` (real facet, ``yN / 2 + 1`` rows, every output line weighted
    with ``Fb`` of the other axis) against ``finish_facet_real_half``, real inner product: the
    half rows are the adjoint of the Hermitian line's real part.  ``probe``: None,
    ``("y", line, stored row)`` or ``("x", line, sample)``."""
    rng = numpy.random.default_rng(seed)
    half = core.half_rows
    x = rng.standard_normal((n_lines, fs))
    y = rand_c(rng, (n_lines, half))
    if probe is not None:
        which, line, sample = probe
        if which == "y":
            y = delta((n_lines, half), (line, sample))
        else:
            x = numpy.zeros_like(x)
            x[line, sample] = 1.0
    mask = (rng.random(fs) > 0.3).astype(float) if masked else None
    xm = x if mask is None else x * mask[None, :]
    Ax = core.prepare_facet_real_half(_to(core, _lines(xm, axis)), off, axis)
    rec_a = last_launch(core)
    ATy = core.finish_facet_real_half(_to(core, _lines(y, axis)), off, fs, axis,
                                      mask=None if mask is None else _to(core, mask))
    rec_b = last_launch(core)
    assert rec_a[0] == rec_b[0] == line_record(core.yN_size, n_lines, axis == 0)[0], \
        (rec_a, rec_b)
    Ax, ATy = _host(Ax), _host(ATy)
    if axis == 0:
        Ax, ATy = Ax.T, ATy.T
    # window_lines: output line l carries Fb(n_lines)[l]; it moves onto the finished side
    ATy = ATy * fb_window(core, n_lines)[:, None]
    return adjoint_residual(y, Ax, ATy, x, chain_constant(core, K1), real=True)


def real_facet_cases(core, seed=0):
    """finish_facet_real and finish_facet_real_half against their forward twins, both axes,
    masked, with delta probes on stored rows 0 and yN / 2, a conjugated pair and the first and
    last sample of an odd facet.  Returns the worst residual."""
    yN, N, step = core.yN_size, core.N, core.facet_off_step
    odd, even, _ = lc.facet_sizes(yN)
    half = core.half_rows
    worst = 0.0
    for k, (axis, lines, fs, off, masked, probe) in enumerate([
            (0, 3, odd, N + step, True, None), (1, 4, even, -2 * step, False, None),
            (0, 2, odd, 0, False, (1, odd - 1)), (1, 2, odd, -N, False, (0, 0))]):
        worst = max(worst, finish_real_pair(core, axis, lines, fs, off, masked=masked,
                                            probe=probe, seed=seed + k))
    for k, (axis, lines, fs, off, masked, probe) in enumerate([
            (0, 5, odd, -3 * step, True, None), (1, 3, even, N + 2 * step, False, None),
            (0, 3, odd, step, False, ("y", 0, 0)), (0, 3, odd, step, False, ("y", 2, half - 1)),
            (1, 2, even, -step, False, ("y", 1, 1)), (1, 2, even, -step, False, ("y", 0, half - 2)),
            (0, 3, odd, 2 * step, False, ("x", 0, 0)), (0, 3, odd, 2 * step, False, ("x", 2, odd - 1))]):
        worst = max(worst, finish_half_pair(core, axis, lines, fs, off, masked=masked,
                                            probe=probe, seed=seed + 10 + k))
    return worst


# ---------------------------------------------------------------------- K2 <-> fold_column
def window_rows(core, sg_off0):
    """Facet rows of the column's ``m``-row window (``OracleCore._facet_window``)."""
    yN, m, N = core.yN_size, core.xM_yN_size, core.N
    s = sg_off0 * yN // N
    t = numpy.arange(m)
    return numpy.mod(yN // 2 - m // 2 + numpy.mod(t - s, m) + s, yN)


def column_pair(core, sizes, offs, sg_off0, *, layout="full", prewindowed=False, masked=(),
                probe=None, variant=0, force_split=0, cap=0, seed=0):
    """``extract_columns`` against ``fold_column`` (zeroed facet accumulators), constant
    ``1 / yN``.  ``layout``: "full" (``(yN, fs)`` prepared facets / accumulators), "ring" (the
    ``m``-row rings: window row ``r`` at line ``r mod m``) or "half" (``yN / 2 + 1`` half rows of
    a real image, real inner product).  ``prewindowed``: K2 takes its rows as weighted with
    ``Fb`` already, so the fold's result is divided by it.  ``masked``: indices of the facets
    whose fold has a mask (moved onto K2's input).  ``probe``: None, ``("y", facet, line,
    sample)`` (a delta in a column accumulator) or ``("x", facet, row, sample)``.

    Returns ``(residual, K2 record, K2 cluster, fold record)``."""
    rng = numpy.random.default_rng(seed)
    yN, m, half = core.yN_size, core.xM_yN_size, core.half_rows
    rows = {"full": yN, "ring": m, "half": half}[layout]
    xs = [rand_c(rng, (rows, fs)) for fs in sizes]
    ys = [rand_c(rng, (m, yN)) for _ in sizes]
    if probe is not None:
        which, j, a, b = probe
        if which == "y":
            ys = [numpy.zeros_like(v) for v in ys]
            ys[j][a, b] = 1.0
        else:
            xs = [numpy.zeros_like(v) for v in xs]
            xs[j][a, b] = 1.0
    if layout == "half":  # self-conjugate rows of a Hermitian array are real
        for v in xs:
            v[0] = v[0].real
            v[yN // 2] = v[yN // 2].real
    masks = [(rng.random(fs) > 0.3).astype(float) if j in masked else None
             for j, fs in enumerate(sizes)]
    xin = [x if mk is None else x * mk[None, :] for x, mk in zip(xs, masks)]
    dev = _dev(core)
    with hooks(core, variant, cap, force_split):
        Ax = core.extract_columns([_to(core, x) for x in xin], sg_off0, list(offs),
                                  prewindowed=prewindowed)
        rec_k2, cl_k2 = last_launch(core), last_cluster(core)
        faccs = [torch.zeros((rows, fs), dtype=torch.complex128, device=dev) for fs in sizes]
        core.fold_column([_to(core, y) for y in ys], faccs, list(offs),
                         [None if mk is None else _to(core, mk) for mk in masks], sg_off0)
        rec_fold = last_launch(core)
    ATy = [_host(f) for f in faccs]
    if prewindowed:
        ATy = [a / fb_window(core, fs)[None, :] for a, fs in zip(ATy, sizes)]
    res = adjoint_residual(ys, [_host(a) for a in Ax], ATy, xs, chain_constant(core, K2),
                           real=layout == "half")
    return res, rec_k2, cl_k2, rec_fold


def expected_k2(core, sizes, variant=0, force_split=0, cap=0):
    """:func:`k2_cases.form` of the call's last launch."""
    tail = (len(sizes) - 1) % kc.MAX_LAUNCH_FACETS + 1
    rec, _ = kc.form(core.yN_size, sizes[-tail:], tail * core.xM_yN_size, variant=variant,
                     force_split=force_split, cap=cap, emulated=is_emulated(core))
    return rec, tail


def column_case(core, sizes, offs, sg_off0, *, what="", **kw):
    """:func:`column_pair` asserting the K2 form of :func:`k2_cases.form` and the fold's line
    kernel; returns the residual."""
    res, rec_k2, _, rec_fold = column_pair(core, sizes, offs, sg_off0, **kw)
    want, tail = expected_k2(core, sizes, kw.get("variant", 0), kw.get("force_split", 0),
                             kw.get("cap", 0))
    _expect(rec_k2, want, f"extract_columns {what}")
    fold = line_record(core.yN_size, tail * core.xM_yN_size, False, kw.get("cap", 0))
    if kw.get("layout") == "half":  # the fold's second pass covers the rows of one half only
        _expect(rec_fold[:2], fold[:2], f"fold_column {what}")
    else:
        _expect(rec_fold, fold, f"fold_column {what}")
    return res


def window_offsets(core):
    """Column offsets whose window wraps around yN (below 0 and >= N), straddles centred rows 0
    and yN / 2, and an ordinary one."""
    N, step = core.N, core.subgrid_off_step
    wrap = kc.subgrid_offsets(core)
    return {"wrap-": wrap[0], "wrap+": wrap[1], "zero": 0, "nyquist": N // 2,
            "plain": N // 4 + step}


def column_row_cases(core, yB, seed=0):
    """One catalogue row ``(yN, yB)``: three facets of ``yB`` (two at yN * yB > 2^26) in full
    rows and rings, raw and prewindowed, a mask, windows that wrap and straddle; delta probes
    at the wrap of the row window and on the first and last sample of the facet.  Where whole
    facets would exceed 2^24 samples only the rings (the window's rows) run.  Returns the worst
    residual."""
    yN, m = core.yN_size, core.xM_yN_size
    n = 3 if yN * yB <= 1 << 26 else 2
    full = "full" if n * yN * yB <= 1 << 24 else "ring"
    offs = kc.facet_offsets(core)[:n]
    win = window_offsets(core)
    sizes = [yB] * n
    worst = 0.0
    for k, (layout, sg, pre, masked) in enumerate([
            (full, win["wrap-"], False, (0,)), ("ring", win["wrap+"], True, ()),
            (full, win["nyquist"], True, (n - 1,)), ("ring", win["plain"], False, (1,))]):
        worst = max(worst, column_case(core, sizes, offs, sg, layout=layout, prewindowed=pre,
                                       masked=masked, seed=seed + k,
                                       what=f"row ({yN}, {yB}) {layout}"))
    rows = window_rows(core, win["wrap-"])
    seam = int(numpy.flatnonzero(rows == 0)[0])  # window line that holds facet row 0
    at = (lambda r: int(r)) if full == "full" else (lambda r: int(r) % m)
    for k, probe in enumerate([("y", 0, seam, 0), ("y", n - 1, max(seam - 1, 0), yN - 1),
                               ("x", 0, at(rows[0]), 0), ("x", n - 1, at(rows[-1]), yB - 1)]):
        worst = max(worst, column_case(core, sizes, offs, win["wrap-"], probe=probe,
                                       layout=full, prewindowed=True, seed=seed + 10 + k,
                                       what=f"row ({yN}, {yB}) delta {probe}"))
    return worst


def column_half_cases(core, sizes, seed=0):
    """Half rows: windows straddling centred rows 0 and yN / 2 (the fold's two passes) and
    neither, masked, with delta probes on stored rows 0 and yN / 2 and on a conjugated pair."""
    yN, half = core.yN_size, core.half_rows
    offs = kc.facet_offsets(core)[:len(sizes)]
    win = window_offsets(core)
    worst = 0.0
    for k, key in enumerate(["zero", "nyquist", "plain", "wrap-"]):
        worst = max(worst, column_case(core, sizes, offs, win[key], layout="half",
                                       prewindowed=True, masked=(0,), seed=seed + k,
                                       what=f"half rows, window {key}"))
    # stored row d: centred row (yN/2 + d); row 0 and yN / 2 are self-conjugate; in the window
    # at "zero" stored rows d and yN - d ... are a conjugated pair
    rows_zero = window_rows(core, win["zero"])
    line_of = {int(r): u for u, r in enumerate(rows_zero)}
    r0 = half_rows_of(yN, 0)
    pair_d = 1
    for k, probe in enumerate([
            ("x", 0, 0, 0), ("x", 0, half - 1, sizes[0] - 1), ("x", len(sizes) - 1, pair_d, 1),
            ("y", 0, line_of.get(r0, 0), yN // 2),
            ("y", 0, line_of.get(half_rows_of(yN, pair_d), 0), 3),
            ("y", 0, line_of.get(half_rows_of(yN, -pair_d), 0), 3)]):
        key = "zero" if k != 1 else "nyquist"
        worst = max(worst, column_case(core, sizes, offs, win[key], layout="half",
                                       prewindowed=True, probe=probe, seed=seed + 10 + k,
                                       what=f"half rows, delta {probe}"))
    return worst


def column_many_case(core, fs, n_facets=67, seed=0):
    """``n_facets`` facets (more than 64: two launches of each kernel) with distinct offsets."""
    step = core.facet_off_step
    offs = [(k - 5) * step + (core.N if k % 7 == 6 else 0) for k in range(n_facets)]
    return column_case(core, [fs] * n_facets, offs, kc.subgrid_offsets(core)[2],
                       masked=(3, n_facets - 1), seed=seed, what=f"{n_facets} facets")


# ---------------------------------------------------------------------- K3 / K4 <-> split
def _sources(core, rng, n, lines, size, axis, adjacent):
    """``n`` random source arrays of ``lines`` lines of ``size`` samples along ``axis``
    (lines-first numpy, device tensor in the pair's layout)."""
    srcs = [rand_c(rng, (lines, size)) for _ in range(n)]
    # pylint: disable=protected-access
    return srcs, [prc._view(core, s, axis, adjacent) for s in srcs]


def subgrid_pair(core, groups, sz, axis, *, mode="add", entry="single", adjacent=None,
                 lines=3, sg_offs=None, masked=False, probe=None, cap=0, seed=0):
    """``sum_finish_axis`` (``entry`` "single", "grouped", "batched") against
    ``split_subgrid_axis`` into zeroed targets, constant ``m / xM`` (``mode`` "add": prepared
    facet lines of ``yN`` samples / facet accumulators; "store": contributions of ``m``).
    ``groups``: per group the facet offsets in units of ``yN / 2``.  ``adjacent`` (default: along
    axis 0): lines adjacent in memory, the split kernel's two-lines-per-CTA form.  ``probe``:
    None, ``("y", group, line, sample)`` or ``("x", group, target, line, sample)``.  Returns
    ``(residual, forward record, split record)``."""
    rng = numpy.random.default_rng(seed)
    m, yN = core.xM_yN_size, core.yN_size
    if adjacent is None:
        adjacent = axis == 0
    size = yN if mode == "add" else m
    ng = len(groups)
    if sg_offs is None:
        sg_offs = [(2 * g - 3) * core.subgrid_off_step for g in range(ng)]
    if entry in ("single", "grouped"):
        sg_offs = [sg_offs[0]] * ng
    offs = [[k * (yN // 2) for k in grp] for grp in groups]
    xs = [[rand_c(rng, (lines, size)) for _ in o] for o in offs]
    ys = [rand_c(rng, (lines, sz)) for _ in range(ng)]
    if probe is not None:
        if probe[0] == "y":
            _, g, line, s = probe
            ys = [numpy.zeros_like(v) for v in ys]
            ys[g][line, s] = 1.0
        else:
            _, g, t, line, s = probe
            xs = [[numpy.zeros_like(v) for v in grp] for grp in xs]
            xs[g][t][line, s] = 1.0
    masks = [(rng.random(sz) > 0.3).astype(float) if masked else None for _ in range(ng)]
    if entry in ("single", "grouped"):
        masks = [masks[0]] * ng
    dev = _dev(core)
    # pylint: disable=protected-access
    t_groups = [[(prc._view(core, s, axis, adjacent), o) for s, o in zip(ss, oo)]
                for ss, oo in zip(xs, offs)]
    t_masks = [None if mk is None else torch.from_numpy(mk).to(dev) for mk in masks]
    with prc.max_blocks(core, cap):
        if entry == "single":
            assert ng == 1
            out = prc._out(core, 1, lines, sz, axis, adjacent)
            core.sum_finish_axis(t_groups[0], out[0], axis=axis, subgrid_off=sg_offs[0],
                                 mask=t_masks[0])
        elif entry == "grouped":
            out = prc._out(core, ng, lines, sz, axis, adjacent)
            core.sum_finish_axis_grouped(t_groups, out, axis=axis, subgrid_off=sg_offs[0],
                                         mask=t_masks[0])
        else:
            out = prc._out(core, ng, lines, sz, axis, adjacent)
            core.sum_finish_axis_grouped(t_groups, out, axis=axis, subgrid_off=list(sg_offs),
                                         mask=t_masks)
        rec_fwd = last_launch(core)
        Ax = [prc._lines_first(o, axis) for o in out]
        # split: the mask of the forward side moves onto its input
        ins = [prc._view(core, y if mk is None else y * mk[None, :], axis, adjacent)
               for y, mk in zip(ys, masks)]
        tgts = [[(prc._view(core, numpy.zeros((lines, size), dtype=complex), axis, adjacent), o)
                 for o in oo] for oo in offs]
        groups_in = [i for i, oo in zip(ins, offs) if oo]
        keep = [g for g, oo in enumerate(offs) if oo]
        core.split_subgrid_axis(groups_in, axis, [sg_offs[g] for g in keep],
                                [tgts[g] for g in keep], mode)
        rec_split = last_launch(core)
    ATy = [prc._lines_first(t, axis) for grp in tgts for t, _ in grp]
    x_flat = [x for grp in xs for x in grp]
    links = K34 if mode == "add" else K34_CONTRIB
    return (adjoint_residual(ys, Ax, ATy, x_flat, chain_constant(core, links)),
            rec_fwd, rec_split)


def subgrid_pair_cases(core, pair, seed=0):
    """One ``(m, xM)`` pair: both axes, add and store, the three entry points, a partial last
    round of the split kernel (targets not a multiple of CONC), the grid capped; random and
    delta probes (first and last line of a CTA, the last line of the partial round, the first
    and last sample of an odd subgrid).  Each case asserts the forward form of
    :data:`pair_cases.FORMS` and the split kernel's lines per CTA.  Returns the worst residual."""
    _, _, split_lpc, conc, tma_sz = prc.FORMS[pair]
    xM = core.xM_size
    sz = xM - 3 if (xM - 3) % 2 else xM - 4
    sz = sz if sz % 2 else sz - 1  # odd
    far = [-3, 0, 2 * core.N // core.yN_size + 1]
    n_part = conc + 1  # a full round and a partial one
    part = [far[k % 3] + (k // 3) for k in range(n_part)]
    worst = 0.0

    def note(res, rec_fwd, rec_split, axis, adjacent, cap=0, what=""):
        nonlocal worst
        fk, fl = prc.forward_form(pair, adjacent)
        assert rec_fwd[:2] == (fk, fl), f"{pair} {what}: forward launched {rec_fwd}"
        lpc = split_lpc if axis == 0 else 1
        assert rec_split[:2] == (prc.SPLIT, lpc), f"{pair} {what}: split launched {rec_split}"
        if cap:
            assert rec_fwd[3] == cap and rec_split[3] == cap, (rec_fwd, rec_split)
        worst = max(worst, res)

    lines = {0: 2 * split_lpc + 1, 1: 3}  # axis 0: a CTA with a single line at the end
    for k, (axis, mode) in enumerate([(0, "add"), (1, "add"), (0, "store"), (1, "store")]):
        note(*subgrid_pair(core, [part], sz, axis, mode=mode, lines=lines[axis], masked=k % 2 == 0,
                           seed=seed + k), axis, axis == 0, what=f"axis {axis} {mode}")
    for k, entry in enumerate(["grouped", "batched"]):
        groups = [part, [far[1]], [far[0], far[2]]]
        note(*subgrid_pair(core, groups, sz, 1, entry=entry, masked=True, seed=seed + 10 + k),
             1, False, what=entry)
    note(*subgrid_pair(core, [part, [0]], sz, 0, entry="batched", lines=7, cap=2,
                       seed=seed + 20), 0, True, cap=2, what="capped grid")
    if tma_sz:  # two-group forward form with TMA stores
        note(*subgrid_pair(core, [part], tma_sz, 1, mode="store", adjacent=False,
                           seed=seed + 21), 1, False, what="two-group TMA size")
    # delta probes
    lastl = lines[0] - 1
    for k, probe in enumerate([
            ("y", 0, 0, 0), ("y", 0, lastl, sz - 1),
            ("x", 0, n_part - 1, lastl, 0), ("x", 0, n_part - 1, 0, core.yN_size - 1),
            ("x", 0, 0, 1, core.yN_size // 2)]):
        note(*subgrid_pair(core, [part], sz, 0, lines=lines[0], probe=probe, seed=seed + 30 + k),
             0, True, what=f"delta {probe}")
    return worst


# ---------------------------------------------------------------------- primitive subgrid side
def subgrid_line_pair(core, which, axis, n_lines, off, *, sz=None, probe=None, seed=0):
    """One primitive pair along ``axis``: ``which`` "subgrid" (``add_to_subgrid`` <->
    ``extract_from_subgrid``, ``off`` a facet offset) or "finish" (``finish_subgrid`` <->
    ``prepare_subgrid`` at size ``sz``, ``off`` a subgrid offset).  Asserts both launches."""
    rng = numpy.random.default_rng(seed)
    m, xM = core.xM_yN_size, core.xM_size
    n_in, n_out = (m, xM) if which == "subgrid" else (xM, sz)
    x, y = rand_c(rng, (n_lines, n_in)), rand_c(rng, (n_lines, n_out))
    if probe is not None:
        if probe[0] == "y":
            y = delta(y.shape, probe[1:])
        else:
            x = delta(x.shape, probe[1:])
    xin, yin = _to(core, _lines(x, axis)), _to(core, _lines(y, axis))
    # pylint: disable=protected-access
    if which == "subgrid":
        Ax = core.add_to_subgrid(xin, off, axis=axis)
        rec_a = last_launch(core)
        ATy = core.extract_from_subgrid(yin, off, axis=axis)
        rec_b = last_launch(core)
        want = slc.line_form(m, n_lines, axis == 0)
    else:
        Ax = core._run("swiftly_b200_finish_subgrid", xin, sz, axis, None, off)
        rec_a = last_launch(core)
        ATy = core._run("swiftly_b200_prepare_subgrid", yin, xM, axis, None, off)
        rec_b = last_launch(core)
        want = slc.line_form(xM, n_lines, axis == 0)
    _expect(rec_a, want, f"{which} forward, axis {axis}")
    _expect(rec_b, want, f"{which} backward, axis {axis}")
    Ax, ATy = _host(Ax), _host(ATy)
    if axis == 0:
        Ax, ATy = Ax.T, ATy.T
    return adjoint_residual(y, Ax, ATy, x, constants(core)[which])


def subgrid_2d_pair(core, sz, sg_offs, seed=0):
    """``finish_subgrid`` <-> ``prepare_subgrid`` in 2-D, constant ``1 / xM^2``."""
    rng = numpy.random.default_rng(seed)
    xM = core.xM_size
    x, y = rand_c(rng, (xM, xM)), rand_c(rng, (sz, sz))
    Ax = core.finish_subgrid(_to(core, x), list(sg_offs), sz)
    ATy = core.prepare_subgrid(_to(core, y), tuple(sg_offs))
    return adjoint_residual(y, Ax, ATy, x, constants(core)["finish"] ** 2)


def to_facets_pair(core, n_facets, sg_off1, probe=None, seed=0):
    """``subgrid_to_facets`` (zeroed column accumulators) against its forward twin,
    ``extract_from_facet(axis 1) -> add_to_subgrid(axis 1)`` of the primitives (the latter
    pinned to the oracle), constant ``m``."""
    rng = numpy.random.default_rng(seed)
    m, xM, yN = core.xM_yN_size, core.xM_size, core.yN_size
    step = core.facet_off_step
    offs = [(f * 7 - 3 * n_facets) * step + (core.N if f % 5 == 4 else 0) for f in range(n_facets)]
    ys = [rand_c(rng, (m, xM)) for _ in range(n_facets)]
    xs = [rand_c(rng, (m, yN)) for _ in range(n_facets)]
    if probe is not None:
        f, a, b = probe
        ys = [numpy.zeros_like(v) for v in ys]
        ys[f][a, b] = 1.0
    Ax = []
    for x, off in zip(xs, offs):
        c = core.extract_from_facet(_to(core, x), sg_off1, axis=1)
        Ax.append(_host(core.add_to_subgrid(c, off, axis=1)))
    accs = [torch.zeros((m, yN), dtype=torch.complex128, device=_dev(core)) for _ in offs]
    core.subgrid_to_facets([_to(core, y) for y in ys], accs, offs, sg_off1)
    last = n_facets - (n_facets - 1) // 64 * 64
    _expect(last_launch(core), slc.line_form(m, last * m, False), "subgrid_to_facets")
    return adjoint_residual(ys, Ax, [_host(a) for a in accs], xs,
                            chain_constant(core, TO_FACETS))


def subgrid_side_cases(core, which, xa=None, seed=0):
    """The primitive subgrid side of one ``m`` plan (``which`` "m": add_to_subgrid <->
    extract_from_subgrid along both axes, subgrid_to_facets over 67 facets) or ``xM`` plan
    ("xM": finish_subgrid <-> prepare_subgrid at odd and catalogue sizes, both axes and 2-D),
    random and delta probes.  Returns the worst residual."""
    m, xM = core.xM_yN_size, core.xM_size
    fo = slc.facet_offsets(core)
    so = slc.subgrid_offsets(core)
    worst = 0.0
    if which == "m":
        counts = slc.lpc_line_counts(m)
        for k, (axis, n, off, probe) in enumerate([
                (0, counts[0], fo[1], None), (1, counts[1], fo[2], None), (0, counts[2], fo[0], None),
                (0, counts[2], fo[1], ("y", counts[2] - 1, xM - 1)),
                (1, counts[1], fo[2], ("x", 0, 0)), (1, counts[1], fo[2], ("x", counts[1] - 1, m - 1))]):
            worst = max(worst, subgrid_line_pair(core, "subgrid", axis, n, off, probe=probe,
                                                 seed=seed + k))
        # 67 facets (two launches) where their accumulators stay small
        many = 67 if 67 * m * core.yN_size <= 1 << 22 else 3
        worst = max(worst, to_facets_pair(core, many, so[0], seed=seed + 10),
                    to_facets_pair(core, 5, so[1], probe=(4, m - 1, xM - 1), seed=seed + 11))
        return worst
    sizes = [s for s in slc.sizes(core, xa) if s % 2] + [xM // 2 + 1]
    for k, sz in enumerate(sizes):
        for axis in (0, 1):
            worst = max(worst, subgrid_line_pair(core, "finish", axis, 3 + axis, so[k % 2],
                                                 sz=sz, seed=seed + 2 * k + axis))
        worst = max(worst, subgrid_line_pair(core, "finish", 0, 3, so[1], sz=sz,
                                             probe=("y", 2, sz - 1), seed=seed + 20 + k),
                    subgrid_line_pair(core, "finish", 1, 2, so[0], sz=sz,
                                      probe=("y", 0, 0), seed=seed + 30 + k))
    if xM <= 2048:
        worst = max(worst, subgrid_2d_pair(core, sizes[0], so, seed=seed + 40))
    return worst


# ---------------------------------------------------------------------- drivers
def subgrid_probe(core, index, size, seed, real=False):
    """The backward operand of subgrid ``index``: complex normal samples from a device generator
    seeded with ``seed`` and ``index``, so that no subgrid set is ever stored."""
    dev = _dev(core)
    gen = torch.Generator(device=dev)
    gen.manual_seed(seed * 1000003 + index)
    return torch.randn((size, size), dtype=torch.complex128, device=dev, generator=gen)


class _Lazy:
    """A subgrid handle for :meth:`SwiftlyBackward.add_subgrid_tasks`, made when resolved."""

    def __init__(self, make):
        self._make = make

    def result(self):
        return self._make()


def mask_2d(cfg_):
    """The 0/1 product of a facet or subgrid config's two masks (ones where a mask is None)."""
    m0, m1 = (numpy.ones(cfg_.size) if mk is None else numpy.asarray(mk, dtype=float)
              for mk in (cfg_.mask0, cfg_.mask1))
    return m0[:, None] * m1[None, :]


def _mask_2d(cfg_, like):
    """:func:`mask_2d` on the device of ``like``, built there from the two 1-D masks."""
    m0, m1 = (torch.ones(cfg_.size, dtype=torch.float64, device=like.device) if mk is None
              else torch.as_tensor(numpy.asarray(mk, dtype=float), device=like.device)
              for mk in (cfg_.mask0, cfg_.mask1))
    return m0[:, None] * m1[None, :]


def _release(dev):
    """Free what a dropped driver held: the drivers keep reference cycles, so their device
    arrays go only with a collection."""
    gc.collect()
    if dev.type == "cuda":
        torch.cuda.empty_cache()


def facet_probe(core, index, size, seed, real=False):
    """The forward operand of facet ``index``: normal samples (complex unless ``real``) from a
    device generator seeded with ``seed`` and ``index``."""
    dev = _dev(core)
    gen = torch.Generator(device=dev)
    gen.manual_seed(seed * 1000003 + 500009 + index)
    dtype = torch.float64 if real else torch.complex128
    return torch.randn((size, size), dtype=dtype, device=dev, generator=gen)


DEVICE_CHUNK = 1 << 16


def _chunk_sums(t):
    """Sums of ``DEVICE_CHUNK`` consecutive samples of a flat device tensor (the last partial)."""
    n = t.numel()
    k = n // DEVICE_CHUNK
    parts = [t[:k * DEVICE_CHUNK].view(k, DEVICE_CHUNK).sum(1)] if k else []
    if n > k * DEVICE_CHUNK:
        parts.append(t[k * DEVICE_CHUNK:].sum().reshape(1))
    return numpy.asarray(torch.cat(parts).cpu().numpy()).astype(numpy.clongdouble)


def _dot_norms(a, b):
    """``(<a, b>, |a|^2, |b|^2)``, summed in ``numpy.longdouble`` on the host.  Device tensors of
    2^20 samples or more (cfg4's subgrids and facets) are reduced on the device in chunks of
    ``DEVICE_CHUNK`` samples first: each chunk's sum carries a rounding of at most
    ``log2(DEVICE_CHUNK) eps = 3.6e-15`` of its norm product, far below :data:`CHAIN_BOUND`,
    and the host never holds a subgrid set."""
    if isinstance(a, torch.Tensor) and a.is_cuda and a.numel() >= 1 << 20:
        a, b = a.reshape(-1), b.reshape(-1)
        d = _chunk_sums(a.conj() * b).sum()
        na = _chunk_sums(a.real * a.real + (a.imag * a.imag if a.is_complex() else 0)).sum()
        nb = _chunk_sums(b.real * b.real + (b.imag * b.imag if b.is_complex() else 0)).sum()
        return d, na.real, nb.real
    p, q = _ld(a), _ld(b)
    return (numpy.dot(numpy.conj(p), q), (p.real * p.real + p.imag * p.imag).sum(),
            (q.real * q.real + q.imag * q.imag).sum())


def driver_case(cfg, facet_cfgs, sg_cfgs, *, lru=1, shuffle=False, budget=None, real=False,
                half_rows=False, seed=0, log=None):
    """``SwiftlyForward`` against ``SwiftlyBackward``: ``N^2 sum_i <S_i, fwd(F)_i> =
    sum_j <bwd(S)_j, F_j>`` (``real``: the real part on the left, real facets, the backward
    transform's real mode through ``add_subgrid_tasks``, the merge path).

    Masks move across: the forward operand is the facets times their facet masks (what the
    backward transform applies), the backward operand the subgrid probes times their subgrid
    masks (what the forward transform applies).  Facets and subgrids come from seeded device
    generators and are made when used; ``<S_i, fwd(F)_i>`` is accumulated as each subgrid is
    yielded and the subgrid dropped, and the forward transform is freed before the backward one
    runs.  ``budget``: the ``device_budget`` of both (1: the host tier); ``log``: called with a
    progress message every 256 subgrids.  Returns ``(residual,
    forward in the host tier, backward in the host tier)``."""
    core = cfg.core
    dev = _dev(core)
    sg_cfgs = list(sg_cfgs)
    if shuffle:
        random.Random(seed).shuffle(sg_cfgs)
    N = cfg.image_size

    def facet(j, masked):
        f = facet_probe(core, j, facet_cfgs[j].size, seed, real)
        return f * _mask_2d(facet_cfgs[j], f) if masked else f

    def probe(i):
        s = subgrid_probe(core, i, sg_cfgs[i].size, seed)
        return s * _mask_2d(sg_cfgs[i], s)

    lhs = numpy.clongdouble(0)
    n_y = n_ax = numpy.longdouble(0)
    # the real-image mode resolves every facet when it is built (to check its dtype) and uploads
    # them one by one: hand it host copies, so that the facets never all sit on the device
    fwd = SwiftlyForward(cfg, [(fc, _Lazy(lambda j=j: facet(j, True).cpu() if real
                                          else facet(j, True)))
                               for j, fc in enumerate(facet_cfgs)],
                         lru_forward=lru, queue_size=4, device_budget=budget, real_image=real,
                         half_rows=half_rows)
    fwd_host = fwd.host_tier
    seen = 0
    for i, task in fwd.iter_subgrid_tasks(sg_cfgs):
        d, a, b = _dot_norms(probe(i), task.wait().tensor)
        lhs, n_y, n_ax = lhs + d, n_y + a, n_ax + b
        seen += 1
        if log is not None and seen % 256 == 0:
            log(f"forward: {seen} subgrids")
        del task
    assert seen == len(sg_cfgs)
    del fwd
    _release(dev)
    bwd = SwiftlyBackward(cfg, facet_cfgs, lru_backward=lru, queue_size=4, device_budget=budget,
                          real_image=real, half_rows=half_rows)
    bwd_host = bwd.host_tier
    bwd.add_subgrid_tasks(sg_cfgs, [_Lazy(lambda i=i: probe(i)) for i in range(len(sg_cfgs))])
    tasks = bwd.finish()
    del bwd
    _release(dev)
    if log is not None:
        log("backward finished")
    rhs = numpy.clongdouble(0)
    n_b = n_f = numpy.longdouble(0)
    for j, t in enumerate(tasks):
        d, a, b = _dot_norms(t.wait().tensor, facet(j, False))
        rhs, n_b, n_f = rhs + d, n_b + a, n_f + b
        tasks[j] = None
    c = numpy.longdouble(N) ** 2
    if real:
        lhs, rhs = lhs.real, rhs.real
    den = c * numpy.sqrt(n_y * n_ax) + numpy.sqrt(n_b * n_f)
    return float(abs(c * lhs - rhs) / den), fwd_host, bwd_host


def self_mirrored_and_unpaired(sg_cfgs, N, xM):
    """A subgrid list with self-mirrored configs and configs whose mirror is missing: ``sg_cfgs``
    without the second member of every other Hermitian pair."""
    pairs = [j for _, j in mirror_pairs(sg_cfgs, N, xM) if j is not None]
    drop = set(pairs[::2])
    kept = [c for k, c in enumerate(sg_cfgs) if k not in drop]
    plan = mirror_pairs(kept, N, xM)
    assert drop and any(j is not None for _, j in plan), plan
    return kept
