"""
The facet-side line transforms at every facet length ``yN`` of the parameter catalogue, shared
by the emulated and the GPU tests.

A transform along a facet axis picks its kernel by length (``csrc/dispatch_*.cu`` and
``capi.cu::prepare_facet_impl``):

* a power of two <= 8192: ``LineKernel``, one transform per CTA in shared memory;
* 16384: ``SplitLineKernel<8192>`` (``extract_columns`` also has the K2 forms of
  ``extract_tma.cuh`` / ``extract_park.cuh``);
* any other ``F * M``: ``SplitFKernel<M>``, with ``M`` the largest power of two <= 8192 dividing
  ``yN`` and ``2 <= F <= 16`` -- powers of two above 16384 included;
* ``prepare_facet`` along axis 0 with at least 16 adjacent columns and a power-of-two ``yN`` in
  256 .. 65536: the two-pass transform (``PrepareFacetPassA/BOp``).

``yn_plans()`` derives the distinct plans from ``SWIFT_CONFIGS`` and pins them, so that a new
catalogue entry or a change of the dispatch fails loudly instead of going untested.  The check
functions run the facet-side ops of one plan against ``OracleCore``; ``spot_check_*`` compares
``prepare_facet`` / ``finish_facet`` with a DFT evaluated in extended precision at chosen bins,
which bounds the kernels' rounding absolutely rather than relative to another fp64 FFT.
"""

import numpy
import torch

from ska_sdp_distributed_fourier_transform_b200.swift_configs import SWIFT_CONFIGS
from tests import parity_cases as pc

MAX_DIRECT_FFT = 8192  # plan.h
MIN_FFT = 16
MAX_SPLIT_F = 16  # SW_MAX_SPLIT_F, kernels.cuh
TWO_PASS_COLUMNS = 16  # prepare_facet_impl: two-pass from this many adjacent columns on
TWO_PASS_LENGTHS = tuple(2**k for k in range(8, 17))  # 256 .. 65536

# (M, F) of every catalogue yN that runs through SplitFKernel
PINNED_SPLIT_F = frozenset(
    [(M, F) for M in (128, 256, 512, 1024, 2048) for F in (3, 5, 7)]
    + [(4096, F) for F in (3, 5, 7, 9)]
    + [(8192, F) for F in (3, 4, 5, 6, 7, 8)]
)
PINNED_DIRECT = (256, 512, 1024, 2048, 4096, 8192)
PINNED_TWO_PASS = TWO_PASS_LENGTHS

# Rows of the prepared facets handed to extract_columns start this many samples apart: the rows
# of a (yN, fs) view overlap, so fs = yN - 1 at yN = 65536 takes 8 MiB instead of 64 GiB, and
# every row still holds different values in every column.
ROW_STEP = 8


def split_f_plan(n):
    """``(M, F)`` of ``SplitFKernel`` for an ``n``-point line, or None (``dispatch.cuh``)."""
    if n < 2 * MIN_FFT or n % 2:
        return None
    m = 1
    while n % (2 * m) == 0 and 2 * m <= MAX_DIRECT_FFT:
        m *= 2
    f = n // m
    while f < 2 and m > MIN_FFT:
        m //= 2
        f = n // m
    if m < MIN_FFT or f < 2 or f > MAX_SPLIT_F:
        return None
    return m, f


def line_kernel(n):
    """The kernel of an ``n``-point facet line: ("direct", n), ("split", n) or
    ("splitf", M, F)."""
    if n <= MAX_DIRECT_FFT and n & (n - 1) == 0:
        return ("direct", n)
    if n == 2 * MAX_DIRECT_FFT:
        return ("split", n)
    mf = split_f_plan(n)
    if mf is None:
        raise ValueError(f"no facet line kernel for yN = {n}")
    return ("splitf",) + mf


def plan_id(plan):
    if plan[0] == "splitf":
        return f"splitf-{plan[1]}x{plan[2]}"
    return f"{plan[0]}-{plan[1]}"


def sub_transforms(plan):
    """``(M, F)``: the line is F transforms of M points combined (F = 1: one transform)."""
    if plan[0] == "splitf":
        return plan[1], plan[2]
    if plan[0] == "split":
        return plan[1] // 2, 2
    return plan[1], 1


def yn_plans():
    """Plan id -> ``(plan, (name, W, N, xM, yN))``: every facet-line plan of the catalogue
    (the line kernel of every ``yN``, and the two-pass transform of every power-of-two
    ``yN >= 256``), each with the smallest catalogue entry that uses it (smallest N, then xM)."""
    reps = {}
    for name, p in SWIFT_CONFIGS.items():
        yN = p["yN_size"]
        plans = [line_kernel(yN)]
        if yN in TWO_PASS_LENGTHS:
            plans.append(("twopass", yN))
        rep = (p["N"], p["xM_size"], name)
        for plan in plans:
            if plan not in reps or rep < reps[plan][0]:
                reps[plan] = (rep, (name, p["W"], p["N"], p["xM_size"], yN))
    order = {"direct": 0, "split": 1, "splitf": 2, "twopass": 3}
    return {plan_id(plan): (plan, reps[plan][1])
            for plan in sorted(reps, key=lambda q: (order[q[0]],) + q[1:])}


def line_plans():
    return {k: v for k, v in yn_plans().items() if v[0][0] != "twopass"}


def two_pass_plans():
    return {k: v for k, v in yn_plans().items() if v[0][0] == "twopass"}


# ---------------------------------------------------------------------- against the oracle
def _dev(core):
    return getattr(core, "tensor_device", None) or torch.device("cuda", core.device)


def _to(core, a):
    # clone: on the emulated (CPU) device .to() would alias the numpy array
    return torch.from_numpy(numpy.ascontiguousarray(a)).clone().to(_dev(core))


def _along(v, axis):
    """A vector along ``axis`` of a 2-D array (broadcast over the other axis)."""
    return v[None, :] if axis == 1 else v[:, None]


def _check(got, ref, rtol, what):
    """max|got - ref| <= rtol max|ref|; returns the relative error."""
    got = numpy.asarray(got)
    assert got.shape == ref.shape, f"{what}: shape {got.shape} vs {ref.shape}"
    err = float(numpy.abs(got - ref).max() / max(numpy.abs(ref).max(), 1e-300))
    assert err <= rtol, f"{what}: max err {err:.3e} of the maximum (bound {rtol:.0e})"
    return err


def prepare_facet_vs_oracle(core, oracle, axis, n_lines, fs, facet_off, windowed, seed,
                            rtol=1e-12):
    """``prepare_facet`` of ``n_lines`` lines of ``fs`` samples along ``axis``; with
    ``windowed`` (``window_lines=True``) output line ``l`` is also weighted with
    ``extract_mid(Fb, n_lines)[l]`` of the other axis (``capi.cu::prepare_facet_impl``)."""
    rng = numpy.random.default_rng(seed)
    facet = pc.rand_c(rng, n_lines, fs) if axis == 1 else pc.rand_c(rng, fs, n_lines)
    got = core.prepare_facet(_to(core, facet), facet_off, axis=axis, window_lines=windowed)
    ref = oracle.prepare_facet(facet, facet_off, axis=axis)
    if windowed:
        ref = ref * _along(oracle._fb_window(n_lines), 1 - axis)
    return _check(got.cpu().numpy(), ref, rtol,
                  f"prepare_facet axis {axis}, {n_lines} lines, fs {fs}, off {facet_off}"
                  f"{', windowed' if windowed else ''}")


def finish_facet_vs_oracle(core, oracle, axis, n_lines, fs, facet_off, masked, seed,
                           rtol=1e-12):
    rng = numpy.random.default_rng(seed)
    yN = core.yN_size
    acc = pc.rand_c(rng, n_lines, yN) if axis == 1 else pc.rand_c(rng, yN, n_lines)
    mask = (rng.random(fs) > 0.3).astype(float) if masked else None
    got = core.finish_facet(_to(core, acc), facet_off, fs, axis=axis,
                            mask=None if mask is None else _to(core, mask))
    ref = oracle.finish_facet(acc, facet_off, fs, axis=axis)
    if masked:
        ref = ref * _along(mask, axis)
    return _check(got.cpu().numpy(), ref, rtol,
                  f"finish_facet axis {axis}, {n_lines} lines, fs {fs}, off {facet_off}"
                  f"{', masked' if masked else ''}")


def extract_columns_vs_oracle(core, oracle, sizes, facet_offs, sg_off0, prewindowed, seed,
                              rtol=1e-12):
    """K2 for ``len(sizes)`` prepared facets in one launch against
    ``extract_from_facet(axis 0) -> prepare_facet(axis 1)`` of the oracle.  The prepared facets
    are ``(yN, fs)`` views whose rows start ``ROW_STEP`` samples apart.  ``prewindowed``: the
    kernel takes the rows as already weighted with ``Fb`` along axis 1 (what
    ``prepare_facet(..., window_lines=True)`` hands it), so the oracle gets them divided by it."""
    rng = numpy.random.default_rng(seed)
    yN, m = core.yN_size, core.xM_yN_size
    bfs, refs = [], []
    for fs, off in zip(sizes, facet_offs):
        buf = pc.rand_c(rng, (yN - 1) * ROW_STEP + fs)
        full = numpy.lib.stride_tricks.as_strided(
            buf, (yN, fs), (ROW_STEP * buf.itemsize, buf.itemsize), writeable=False)
        rows = oracle.extract_from_facet(full, sg_off0, axis=0)  # the m rows the subgrid takes
        if prewindowed:
            rows = rows / oracle._fb_window(fs)[None, :]
        refs.append(oracle.prepare_facet(rows, off, axis=1))
        bfs.append(_to(core, buf).as_strided((yN, fs), (ROW_STEP, 1)))
    outs = [torch.full((m, yN), complex(numpy.nan, numpy.nan), dtype=torch.complex128,
                       device=_dev(core)) for _ in sizes]
    core.extract_columns(bfs, sg_off0, list(facet_offs), outs=outs, prewindowed=prewindowed)
    return max(_check(o.cpu().numpy(), r, rtol,
                      f"extract_columns facet {j} (fs {fs}, off1 {off}, sg_off0 {sg_off0}"
                      f"{', prewindowed' if prewindowed else ''})")
               for j, (o, r, fs, off) in enumerate(zip(outs, refs, sizes, facet_offs)))


def fold_column_vs_oracle(core, oracle, sizes, facet_offs, sg_off0, masked, seed, rtol=1e-12):
    """``fold_column`` of ``len(sizes)`` column accumulators into non-zero facet accumulators
    against the oracle's ``finish_facet(axis 1)`` -> mask -> ``add_to_facet(axis 0)``.
    ``masked``: indices of the facets that get a mask.  ``add_to_facet`` is applied to the m rows
    of the subgrid's window only (it adds nothing elsewhere), on the device, so that facet
    accumulators of cfg4 size need no host copy; every other row must stay as it was."""
    rng = numpy.random.default_rng(seed)
    dev = _dev(core)
    yN, m = core.yN_size, core.xM_yN_size
    accs = [pc.rand_c(rng, m, yN) for _ in sizes]
    masks = [(rng.random(fs) > 0.2).astype(float) if j in masked else None
             for j, fs in enumerate(sizes)]
    gen = torch.Generator(device=dev)
    gen.manual_seed(seed)
    faccs = [torch.randn((yN, fs), dtype=torch.complex128, device=dev, generator=gen)
             for fs in sizes]
    want = [f.clone() for f in faccs]
    core.fold_column([_to(core, a) for a in accs], faccs, list(facet_offs),
                     [None if mk is None else _to(core, mk) for mk in masks], sg_off0)
    rows = torch.from_numpy(oracle._facet_window(sg_off0)).to(dev)
    assert len(set(rows.tolist())) == m
    worst = 0.0
    for j, (fs, off) in enumerate(zip(sizes, facet_offs)):
        part = oracle.finish_facet(accs[j], off, fs, axis=1)
        if masks[j] is not None:
            part = part * masks[j][None, :]
        want[j][rows] += torch.from_numpy(part).to(dev)
        err = float((faccs[j] - want[j]).abs().max()) / float(want[j].abs().max())
        assert err <= rtol, (f"fold_column facet {j} (fs {fs}, off1 {off}, sg_off0 {sg_off0}"
                             f"{', masked' if masks[j] is not None else ''}): max err "
                             f"{err:.3e} of the maximum (bound {rtol:.0e})")
        worst = max(worst, err)
    return worst


def facet_sizes(yN):
    """Odd, even and the largest facet size: (yN * 11 // 16) | 1, yN / 2 + 8, yN - 1."""
    return [(yN * 11 // 16) | 1, yN // 2 + 8, yN - 1]


def fold_sizes(yN, budget=1 << 22):
    """Three different facet sizes whose ``(yN, fs)`` accumulators hold at most ``budget``
    samples each (64 MiB): the full yN - 1 up to yN = 2048, 64 samples at yN = 65536."""
    s = min(yN - 1, budget // yN)
    return [s, s - 1, s // 2 + 1]


def line_plan_vs_oracle(core, oracle, seed, fold_budget=1 << 22):
    """Every facet-side op of one line-kernel plan against the oracle; returns the worst
    relative error per op.  Facet offsets 0, negative and >= N in units of
    ``facet_off_step``, subgrid offsets likewise in units of ``subgrid_off_step``."""
    yN, N = core.yN_size, core.N
    fs_step, sg_step = core.facet_off_step, core.subgrid_off_step
    odd, even, full = facet_sizes(yN)
    offs = [0, -3 * fs_step, N + 2 * fs_step]
    worst = {}

    def note(op, err):
        worst[op] = max(worst.get(op, 0.0), err)

    # prepare_facet: along axis 1, and along axis 0 with 5 adjacent columns (below the two-pass
    # threshold, so power-of-two yN run the line kernel with lines fastest)
    for k, (axis, n_lines, fs, windowed) in enumerate([
            (1, 3, full, False), (1, 4, odd, True), (0, 5, even, False), (0, 5, odd, True)]):
        note("prepare_facet", prepare_facet_vs_oracle(core, oracle, axis, n_lines, fs,
                                                      offs[k % 3], windowed, seed + k))
    for k, (axis, n_lines, fs, masked) in enumerate([
            (1, 3, full, False), (1, 2, odd, True), (0, 5, even, True), (0, 4, full, False)]):
        note("finish_facet", finish_facet_vs_oracle(core, oracle, axis, n_lines, fs,
                                                    offs[(k + 1) % 3], masked, seed + 10 + k))
    # K2: three facets (odd, even, yN - 1) in one launch, raw and prewindowed
    for k, prewindowed in enumerate([False, True]):
        note("extract_columns", extract_columns_vs_oracle(
            core, oracle, [odd, even, full], offs, [-5 * sg_step, N + 3 * sg_step][k],
            prewindowed, seed + 20 + k))
    note("fold_column", fold_column_vs_oracle(
        core, oracle, fold_sizes(yN, fold_budget), [offs[1], offs[0], offs[2]],
        -N - 2 * sg_step, masked=[1], seed=seed + 30))
    if yN <= 2 * MAX_DIRECT_FFT:
        # without yN - 1 the K2 launch fits the TMA-staged forms
        note("extract_columns", extract_columns_vs_oracle(
            core, oracle, [odd, even], [fs_step, -fs_step], 0, True, seed + 22))
        note("fold_column", fold_column_vs_oracle(
            core, oracle, fold_sizes(yN, fold_budget)[::-1], offs, 7 * sg_step,
            masked=[0, 2], seed=seed + 31))
    return worst


def two_pass_vs_oracle(core, oracle, seed):
    """prepare_facet along axis 0 with >= 16 adjacent columns (the two-pass transform), plain
    and windowed; returns the worst relative error."""
    yN, N, fs_step = core.yN_size, core.N, core.facet_off_step
    odd, even, full = facet_sizes(yN)
    n = TWO_PASS_COLUMNS
    cases = [(n, full, 0, False), (n + 3, odd, -5 * fs_step, True), (n, even, N + fs_step, True),
             (n + 5, full, 2 * fs_step, False)]
    return max(prepare_facet_vs_oracle(core, oracle, 0, n, fs, off, windowed, seed + k)
               for k, (n, fs, off, windowed) in enumerate(cases))


# ---------------------------------------------------------------------- extended precision
EPS = float(numpy.finfo(numpy.float64).eps)  # 2.2e-16
TWO_PI_L = 8 * numpy.arctan(numpy.longdouble(1))

# Bound of the spot checks in units of EPS * log2(yN) of the line's RMS: about twice the worst
# the direct power-of-two kernels reach.  Observed with the test seeds, prepare_facet and
# finish_facet alike:
#   H100 80GB HBM3 (700 W), 2 lines per check: direct 0.15 .. 0.59, split-16384 0.31 .. 0.50,
#     split-F 0.16 .. 0.51;
#   emulated kernels (host build without fused multiply-adds), 1 line per check: direct
#     0.20 .. 0.65, split-16384 0.32 .. 0.42, split-F 0.19 .. 0.76.
SPOT_BOUND = 1.5


def spot_bins(M, F, n, rng, n_random=4):
    """Natural-order output bins of an ``n = F M``-point line: the sub-transform boundaries
    ``M s - 1, M s, M s + 1`` (s = 0 .. F, mod n), the centre ``n/2 - 1 .. n/2 + 1`` and a few
    random bins."""
    bins = {(M * s + d) % n for s in range(F + 1) for d in (-1, 0, 1)}
    bins |= {n // 2 + d for d in (-1, 0, 1)}
    bins |= {int(b) for b in rng.integers(0, n, n_random)}
    return sorted(bins)


def centred_dft(z, positions, sign):
    """``sum_j z[j] exp(sign 2 pi i (j - n/2)(p - n/2) / n)`` -- the centred transform of
    ``fourier_algorithm.py`` without normalisation -- at the centred output positions ``p``,
    in ``numpy.longdouble``.  The exponent is reduced as the exact integer
    ``((j - n/2)(p - n/2)) mod n`` before it is scaled, so the angle is accurate to the extended
    precision whatever n."""
    assert numpy.finfo(numpy.longdouble).eps < 1e-18, "needs an extended-precision longdouble"
    n = len(z)
    a = TWO_PI_L * numpy.arange(n, dtype=numpy.longdouble) / n
    roots = numpy.cos(a) + sign * 1j * numpy.sin(a)  # exp(sign 2 pi i r / n), r < n
    j = numpy.flatnonzero(z)
    zl = z[j].astype(numpy.clongdouble)
    jc = j.astype(numpy.int64) - n // 2
    return numpy.array([(zl * roots[(jc * (int(p) - n // 2)) % n]).sum() for p in positions],
                       dtype=numpy.clongdouble)


def _window_of(core, fs):
    """The kernels' own ``extract_mid(Fb, fs)`` (``capi.cu``: ``d_Fb + (yN-1)/2 - fs/2``)."""
    lo = (core.yN_size - 1) // 2 - fs // 2
    return numpy.asarray(core._Fb[lo:lo + fs], dtype=numpy.longdouble)


def spot_check_prepare_facet(core, plan, seed, n_lines=2):
    """``prepare_facet`` (axis 1, fs = yN - 1) at the bins of ``spot_bins`` against
    ``centred_dft`` of the exactly weighted, padded and rolled line.  Returns the worst
    ``|got - exact|`` relative to the RMS of the exact output line, in units of
    ``EPS * log2(yN)``."""
    rng = numpy.random.default_rng(seed)
    yN = core.yN_size
    M, F = sub_transforms(plan)
    fs, off = yN - 1, 3 * core.facet_off_step
    facet = pc.rand_c(rng, n_lines, fs)
    got = core.prepare_facet(_to(core, facet), off, axis=1).cpu().numpy()
    pos = [(p + yN // 2) % yN for p in spot_bins(M, F, yN, rng)]
    dest = (yN // 2 - fs // 2 + off + numpy.arange(fs)) % yN
    fb = _window_of(core, fs)
    worst = 0.0
    for line in range(n_lines):
        z = numpy.zeros(yN, dtype=numpy.clongdouble)
        z[dest] = facet[line].astype(numpy.clongdouble) * fb
        exact = centred_dft(z, pos, +1) / yN
        rms = numpy.sqrt((numpy.abs(z) ** 2).sum()) / yN  # Parseval
        err = numpy.abs(got[line, pos].astype(numpy.clongdouble) - exact).max() / rms
        worst = max(worst, float(err))
    return worst / (EPS * numpy.log2(yN))


def spot_check_finish_facet(core, plan, seed, n_lines=2):
    """``finish_facet`` (axis 1, fs = yN - 1) at the bins of ``spot_bins`` against
    ``centred_dft`` of the line; the window factor of each output sample is divided out.  Same
    units as :func:`spot_check_prepare_facet`."""
    rng = numpy.random.default_rng(seed)
    yN = core.yN_size
    M, F = sub_transforms(plan)
    fs, off = yN - 1, -2 * core.facet_off_step
    acc = pc.rand_c(rng, n_lines, yN)
    got = core.finish_facet(_to(core, acc), off, fs, axis=1).cpu().numpy()
    start = (yN // 2 - fs // 2 + off) % yN
    pos = [(p + yN // 2) % yN for p in spot_bins(M, F, yN, rng)]
    pos = [p for p in pos if (p - start) % yN < fs]
    k = [(p - start) % yN for p in pos]
    fb = _window_of(core, fs)[k]
    worst = 0.0
    for line in range(n_lines):
        z = acc[line].astype(numpy.clongdouble)
        exact = centred_dft(z, pos, -1)
        rms = numpy.sqrt((numpy.abs(z) ** 2).sum())  # Parseval: RMS of the output line
        err = numpy.abs(got[line, k].astype(numpy.clongdouble) / fb - exact).max() / rms
        worst = max(worst, float(err))
    return worst / (EPS * numpy.log2(yN))
