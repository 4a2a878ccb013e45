"""
Shared checks of the argument handling of ``SwiftlyCoreB200``, run by
tests/test_emu_core_arguments.py on the host-emulated kernels and by
tests/test_gpu_core_arguments.py on the H100.

Agreement: every way of launching one grouped ``sum_finish_axis`` job -- ``sum_finish_axis`` per
group, ``sum_finish_axis_grouped`` with one offset, with per-group offsets into a stacked output
and into a list of outputs, and ``prepare_sum_finish(...).launch`` with ``out=``, ``outs=`` and
``out_ptrs=`` -- writes the same bits, and so do numpy, float32 and float64 tensor masks of the
same 0/1 samples.  Rejection (emulated kernels only: without the checks these calls read past
the end of a mask or write past an output): masks of the wrong length and outputs of the wrong
shape or strides raise ``ValueError`` before anything is launched.
"""

import numpy
import pytest
import torch

from tests import length_cases as lc

MASK_KINDS = ("numpy", "float32", "float64")
NAN = complex(numpy.nan, numpy.nan)


def _dev(core):
    return lc._dev(core)  # pylint: disable=protected-access


def _mask(core, m, kind):
    """The 0/1 numpy mask ``m`` (or None) as a ``kind`` mask."""
    if m is None:
        return None
    if kind == "numpy":
        return m.copy()
    dtype = torch.float32 if kind == "float32" else torch.float64
    return torch.from_numpy(m).to(_dev(core), dtype)


class Job:
    """Seeded sources, subgrid offsets and masks of ``n_groups`` groups of ``per_group`` sources
    each, whose outputs have ``lines`` lines of ``sz`` samples along ``axis``.  Groups 0 and 3
    share one mask object (as the drivers pass ``[mask] * n``), group 1 has none."""

    def __init__(self, core, axis, sz, *, lines=3, n_groups=4, per_group=2, seed=0):
        rng = numpy.random.default_rng(seed)
        self.core, self.axis, self.sz, self.lines, self.n = core, axis, sz, lines, n_groups
        yN = core.yN_size
        self.groups = []
        for _ in range(n_groups):
            grp = []
            for _ in range(per_group):
                a = rng.standard_normal((lines, yN)) + 1j * rng.standard_normal((lines, yN))
                t = lc._to(core, a)  # pylint: disable=protected-access
                grp.append((t if axis == 1 else t.T, int(rng.integers(-2, 3)) * (yN // 2)))
            self.groups.append(grp)
        self.offs = [(2 * g - 3) * core.subgrid_off_step for g in range(n_groups)]
        a, b = ((rng.random(sz) > 0.3).astype(float) for _ in range(2))
        self.masks = [a, None, b, a][:n_groups] + [b] * max(0, n_groups - 4)

    def outs(self):
        """One NaN-filled output per group (lines along the other axis)."""
        shape = (self.lines, self.sz) if self.axis == 1 else (self.sz, self.lines)
        return [torch.full(shape, NAN, dtype=torch.complex128, device=_dev(self.core))
                for _ in range(self.n)]

    def stacked(self):
        shape = (self.n, self.lines, self.sz) if self.axis == 1 else (self.n, self.sz, self.lines)
        return torch.full(shape, NAN, dtype=torch.complex128, device=_dev(self.core))

    def masks_as(self, kind):
        """The masks as ``kind``, one converted object per distinct numpy mask."""
        conv = {}
        for m in self.masks:
            if id(m) not in conv:
                conv[id(m)] = _mask(self.core, m, kind)
        return [conv[id(m)] for m in self.masks]

    def block(self):
        o = self.outs()[0]
        strides = (o.stride(1 - self.axis), o.stride(self.axis))
        return self.core.prepare_sum_finish(self.groups, self.axis, self.lines, self.sz, strides)


def _bits(t):
    return t.cpu().numpy()


def _same(got, want, what):
    for g, (a, b) in enumerate(zip(got, want)):
        a, b = _bits(a), _bits(b)
        assert not numpy.isnan(a).any(), f"{what}: group {g} not fully written"
        assert numpy.array_equal(a, b), f"{what}: group {g} max diff {numpy.abs(a - b).max():.3e}"


def agreement_case(core, axis, sz, *, kinds=MASK_KINDS, launch_kinds=MASK_KINDS, seed=0):
    """Every launch form and every mask kind against ``sum_finish_axis`` per group with float64
    device masks, bitwise.  ``launch_kinds``: the mask kinds handed to ``launch``."""
    job = Job(core, axis, sz, seed=seed)
    ref = []
    for g, grp in enumerate(job.groups):
        out = job.outs()[0]
        core.sum_finish_axis(grp, out, axis, job.offs[g],
                             mask=_mask(core, job.masks[g], "float64"))
        ref.append(out)
    # one subgrid offset and mask for every group
    ref0 = []
    for grp in job.groups:
        out = job.outs()[0]
        core.sum_finish_axis(grp, out, axis, job.offs[0],
                             mask=_mask(core, job.masks[0], "float64"))
        ref0.append(out)
    assert not numpy.array_equal(_bits(ref[1]), _bits(ref0[1]))
    for kind in kinds:
        masks = job.masks_as(kind)
        for g, grp in enumerate(job.groups):
            out = job.outs()[0]
            core.sum_finish_axis(grp, out, axis, job.offs[g], mask=masks[g])
            _same([out], [ref[g]], f"sum_finish_axis group {g}, {kind} mask")
        out = job.stacked()
        core.sum_finish_axis_grouped(job.groups, out, axis, job.offs[0], mask=masks[0])
        _same(list(out), ref0, f"grouped, one offset, {kind} mask")
        out = job.stacked()
        core.sum_finish_axis_grouped(job.groups, out, axis, list(job.offs), mask=masks)
        _same(list(out), ref, f"grouped, stacked out, {kind} masks")
        outs = job.outs()
        got = core.sum_finish_axis_grouped(job.groups, outs, axis, list(job.offs), mask=masks)
        _same(got, ref, f"grouped, list of outs, {kind} masks")
    block = job.block()
    for kind in launch_kinds:
        masks = job.masks_as(kind)
        out = job.stacked()
        block.launch(job.offs, masks, out=out, out_group_stride=out.stride(0))
        _same(list(out), ref, f"launch out=, {kind} masks")
        outs = job.outs()
        block.launch(job.offs, masks, outs=outs)
        _same(outs, ref, f"launch outs=, {kind} masks")
        outs = job.outs()
        block.launch(job.offs, masks, out_ptrs=[o.data_ptr() for o in outs], stream_of=outs[0])
        _same(outs, ref, f"launch out_ptrs=, {kind} masks")
    # the first groups only, and one group into a 2-D out
    outs = job.outs()
    block.launch(job.offs, job.masks_as("numpy"), outs=outs, n_groups=2)
    _same(outs[:2], ref[:2], "launch outs=, n_groups=2")
    assert all(numpy.isnan(_bits(o)).all() for o in outs[2:])
    out = job.outs()[0]
    block.launch(job.offs, job.masks_as("numpy"), out=out, n_groups=1)
    _same([out], ref[:1], "launch 2-D out, n_groups=1")


# ---------------------------------------------------------------------- rejection
def launch_rejects(core, axis, sz):
    """``launch`` checks its masks and its ``out`` / ``outs`` against the block."""
    job = Job(core, axis, sz)
    block = job.block()
    short = numpy.ones(sz - 1)
    for kind in MASK_KINDS[::-1]:
        with pytest.raises(ValueError, match="mask must have the subgrid size"):
            out = job.stacked()
            block.launch(job.offs, [None, None, _mask(core, short, kind), None], out=out,
                         out_group_stride=out.stride(0))
    longer = numpy.ones(sz + 1)
    with pytest.raises(ValueError, match="mask must have the subgrid size"):
        block.launch(job.offs, [None, None, longer, None], outs=job.outs())
    with pytest.raises(ValueError, match="mask must have the subgrid size"):
        outs = job.outs()
        block.launch(job.offs, [longer] * 4, out_ptrs=[o.data_ptr() for o in outs],
                     stream_of=outs[0])

    dev = _dev(core)
    stacked = job.stacked()
    n, lines = job.n, job.lines
    bad_outs = {
        "one sample more": torch.zeros(
            (n, lines, sz + 1) if axis == 1 else (n, sz + 1, lines), dtype=torch.complex128,
            device=dev),
        "one line fewer": torch.zeros(
            (n, lines - 1, sz) if axis == 1 else (n, sz, lines - 1), dtype=torch.complex128,
            device=dev),
        # the same shape, the other memory order
        "transposed": torch.zeros((n,) + tuple(stacked.shape[:0:-1]), dtype=torch.complex128,
                                  device=dev).transpose(1, 2),
        "strided": torch.zeros((n,) + tuple(2 * s for s in stacked.shape[1:]),
                               dtype=torch.complex128, device=dev)[:, ::2, ::2],
        "complex64": stacked.to(torch.complex64),
        "fewer groups": stacked[:n - 1],
    }
    for what, out in bad_outs.items():
        with pytest.raises(ValueError):
            block.launch(job.offs, None, out=out, out_group_stride=out.stride(0))
            pytest.fail(f"out {what} was launched")
        outs = list(out)
        with pytest.raises(ValueError):
            block.launch(job.offs, None, outs=outs)
            pytest.fail(f"outs {what} were launched")
    with pytest.raises(ValueError):  # a stacked out whose groups lie at another stride
        block.launch(job.offs, None, out=stacked, out_group_stride=stacked.stride(0) // 2)
    with pytest.raises(ValueError):  # a 2-D out holds one group
        block.launch(job.offs, None, out=stacked[0], out_group_stride=stacked.stride(0))
    with pytest.raises(ValueError):  # one of the outs differs
        outs = job.outs()
        outs[2] = outs[2].t().contiguous().t()
        block.launch(job.offs, None, outs=outs)


def finish_mask_rejects(core):
    """``finish_facet`` / ``finish_subgrid`` on numpy arrays and on tensors, and the other
    entries that take masks, with masks of the wrong length."""
    rng = numpy.random.default_rng(3)
    yN, xM, m = core.yN_size, core.xM_size, core.xM_yN_size
    fs, sgs = yN // 2, xM // 2
    facet = rng.standard_normal((yN, 5)) + 1j * rng.standard_normal((yN, 5))
    contrib = rng.standard_normal((xM, xM)) + 1j * rng.standard_normal((xM, xM))
    for host in (True, False):
        f = facet if host else lc._to(core, facet)  # pylint: disable=protected-access
        c = contrib if host else lc._to(core, contrib)  # pylint: disable=protected-access
        for mask in (numpy.ones(fs - 1), numpy.ones(fs + 1), torch.ones(fs - 1)):
            with pytest.raises(ValueError, match="mask must have the facet size"):
                core.finish_facet(f, 0, fs, 0, mask=mask)
        for mask in (numpy.ones(sgs - 1), torch.ones(sgs + 1, dtype=torch.float64)):
            with pytest.raises(ValueError, match="mask must have the subgrid size"):
                core.finish_subgrid(c[:, 0], 0, sgs, masks=[mask])
            for masks in ([None, mask], [mask, None]):
                with pytest.raises(ValueError, match="mask must have the subgrid size"):
                    core.finish_subgrid(c, [0, 0], sgs, masks=masks)
        # the right lengths pass
        core.finish_facet(f, 0, fs, 0, mask=numpy.ones(fs))
        core.finish_subgrid(c[:, 0], 0, sgs, masks=[numpy.ones(sgs)])
    dev = _dev(core)
    acc = lc._to(core, facet)  # pylint: disable=protected-access
    with pytest.raises(ValueError, match="mask must have the facet size"):
        core.finish_facet_real(acc, 0, fs, 0, mask=numpy.ones(fs - 1))
    accs = [torch.zeros((m, yN), dtype=torch.complex128, device=dev) for _ in range(2)]
    faccs = [torch.zeros((yN, fs), dtype=torch.complex128, device=dev) for _ in range(2)]
    with pytest.raises(ValueError, match="mask must have the facet size"):
        core.fold_column(accs, faccs, [0, 0], [None, torch.ones(fs - 1, device=dev)], 0)
    src = torch.zeros((9, 9), dtype=torch.complex128, device=dev)
    with pytest.raises(ValueError, match="mask must have the subgrid size"):
        core.mirror_subgrid(src, 8, masks=(None, numpy.ones(7)))
    with pytest.raises(ValueError, match="mask must have the subgrid size"):
        core.mirror_subgrid(src, 8, mirror_masks=(torch.ones(9, device=dev), None))
