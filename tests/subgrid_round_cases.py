"""
Fused subgrid kernel (two-group form) with partly empty rounds, shared by the emulated and the
GPU tests.  The kernel adds the m-point transforms of a line's sources into an xM accumulator
in rounds of up to CONC = xM / m transforms whose windows are pairwise disjoint.  Sparse
source sets leave slots of a round without a source; those slots skip their transform, and in
the first round they clear what the round's windows do not cover.  The layouts below produce
every shape of round: one source, two clashing sources (two rounds of one), three disjoint
sources, the 3 + 2 rounds of the benchmark's 5 x 5 facet block, 3 + 3 and the tiling 4 + 4.
"""

import ctypes

import numpy
import torch

from tests import parity_cases as pc

# facet offsets in units of yN / 2, which moves a source's window by m / 2 in the accumulator
LAYOUTS = {
    "1": [0],
    "2_clashing": [0, 1],
    "3_disjoint": [0, 2, 4],
    "5_three_plus_two": [0, 1, 2, 6, 7],  # cfg4's central 5 x 5 block (bench.SPARSE_BLOCKS)
    "6": [0, 1, 2, 3, 4, 5],
    "8_tiled": [0, 1, 2, 3, 4, 5, 6, 7],
}
LEGACY_VARIANT = 25  # empty slots transform zeros, accumulator cleared ahead of the rounds


def set_variant(core, v):
    core._lib.swiftly_b200_debug_sg_variant.argtypes = [ctypes.c_void_p, ctypes.c_int]
    core._lib.swiftly_b200_debug_sg_variant(core._plan, int(v))


def offsets(core, layout):
    return [k * (core.yN_size // 2) for k in LAYOUTS[layout]]


def make_sources(core, rng, n, lines, axis, contrib_sized):
    """Sources with a line stride other than 1 (the layout that selects the two-group kernel):
    rows of prepared facets along axis 1, transposed contribution strips along axis 0."""
    size = core.xM_yN_size if contrib_sized else core.yN_size
    srcs = [pc.rand_c(rng, lines, size) for _ in range(n)]
    return [s if axis == 1 else s.T for s in srcs]


def reference(oracle, srcs, offs, sg_off, sz, axis, contrib_sized, lines, mask=None):
    acc = None
    for s, o in zip(srcs, offs):
        c = s if contrib_sized else oracle.extract_from_facet(s, sg_off, axis=axis)
        acc = oracle.add_to_subgrid(c, o, axis=axis, out=acc)
    if acc is None:
        return numpy.zeros((lines, sz) if axis == 1 else (sz, lines), dtype=complex)
    fin = numpy.array([oracle.finish_subgrid(line, sg_off, sz)
                       for line in (acc if axis == 1 else acc.T)])
    if mask is not None:
        fin = fin * mask[None, :]
    return fin if axis == 1 else fin.T


def device(core):
    return getattr(core, "tensor_device", None) or torch.device("cuda", 0)


def to_dev(core, a):
    # (keeps the strides: the transposed sources stay transposed)
    return torch.from_numpy(a).to(device(core))


def out_tensor(core, lines, sz, axis, n_groups=None):
    """Contiguous output: rows of the subgrid along axis 1 (line stride = size), columns along
    axis 0 (unit line stride, like the per-subgrid axis-0 kernel's output)."""
    dev = device(core)
    shape = (lines, sz) if axis == 1 else (sz, lines)
    if n_groups is None:
        return torch.empty(shape, dtype=torch.complex128, device=dev)
    return torch.empty((n_groups,) + shape, dtype=torch.complex128, device=dev)


def check_single(core, oracle, layout, axis, contrib_sized, variant, lines=5, seed=0,
                 sg_step=3, rtol=1e-11):
    """sum_finish_axis with one source group."""
    rng = numpy.random.default_rng(seed)
    sg_off = sg_step * core.subgrid_off_step
    sz = core.xM_size - 3
    offs = offsets(core, layout)
    srcs = make_sources(core, rng, len(offs), lines, axis, contrib_sized)
    out = out_tensor(core, lines, sz, axis)
    set_variant(core, variant)
    try:
        core.sum_finish_axis([(to_dev(core, s), o) for s, o in zip(srcs, offs)], out, axis=axis,
                             subgrid_off=sg_off)
    finally:
        set_variant(core, 0)
    ref = reference(oracle, srcs, offs, sg_off, sz, axis, contrib_sized, lines)
    pc.close(out.cpu().numpy(), ref, rtol=rtol, what=f"layout {layout}, axis {axis}")
    return out


def grouped_layouts():
    # groups with different round counts in one launch: trailing rounds of the shorter groups
    # and the whole of the empty group have no source at all
    return ["5_three_plus_two", "1", "8_tiled", None, "2_clashing", "3_disjoint", "6"]


def check_grouped(core, oracle, variant, mode, lines=5, seed=1, layouts=None, rtol=1e-11,
                  axis=1):
    """The grouped (one subgrid offset), batched (one offset per group) and scattered (one
    output buffer per group) entry points, prepared facet rows along axis 1 / contribution
    strips along axis 0."""
    rng = numpy.random.default_rng(seed)
    layouts = layouts or grouped_layouts()
    ng = len(layouts)
    sz = core.xM_size // 2 + 1
    contrib_sized = axis == 0
    groups_np = []
    for lay in layouts:
        offs = offsets(core, lay) if lay else []
        groups_np.append((make_sources(core, rng, len(offs), lines, axis, contrib_sized), offs))
    sg_offs = [(2 * g - 5) * core.subgrid_off_step for g in range(ng)]
    if mode == "grouped":
        sg_offs = [sg_offs[0]] * ng
    groups = [[(to_dev(core, s), o) for s, o in zip(srcs, offs)] for srcs, offs in groups_np]
    set_variant(core, variant)
    try:
        if mode == "grouped":
            out = out_tensor(core, lines, sz, axis, ng)
            core.sum_finish_axis_grouped(groups, out, axis=axis, subgrid_off=sg_offs[0])
            outs = list(out)
        elif mode == "batched":
            out = out_tensor(core, lines, sz, axis, ng)
            core.sum_finish_axis_grouped(groups, out, axis=axis, subgrid_off=sg_offs)
            outs = list(out)
        else:
            outs = [out_tensor(core, lines, sz, axis) for _ in range(ng)]
            core.sum_finish_axis_grouped(groups, outs, axis=axis, subgrid_off=sg_offs)
    finally:
        set_variant(core, 0)
    for g, ((srcs, offs), o) in enumerate(zip(groups_np, outs)):
        ref = reference(oracle, srcs, offs, sg_offs[g], sz, axis, contrib_sized, lines)
        pc.close(o.cpu().numpy(), ref, rtol=rtol, what=f"{mode}, group {g} ({layouts[g]})")
    return [o.clone() for o in outs]
