"""
Cases of the fused subgrid split kernel (``swiftly_b200_split_subgrid_axis``, the subgrid side
of the backward transform), shared by the emulated and the GPU tests: the kernel through the C
ABI against the oracle's prepare_subgrid -> extract_from_subgrid (-> add_to_facet), and
SwiftlyBackward against the oracle's serial driver.
"""

import numpy
import torch

from oracle.swiftly_oracle import OracleCore, backward_reference_order
from ska_sdp_distributed_fourier_transform_b200 import FacetConfig, SwiftlyBackward
from ska_sdp_distributed_fourier_transform_b200.api import make_full_facet_cover
from ska_sdp_distributed_fourier_transform_b200.api import make_full_subgrid_cover
from tests import parity_cases as pc


def oracle_of(core):
    return OracleCore(core.W, core.N, core.xM_size, core.yN_size)


def _dev(core):
    return getattr(core, "tensor_device", None) or torch.device("cuda", core.device)


def _lines_first(a, axis):
    """(lines, samples) view of a 2-D array whose samples run along ``axis``."""
    return a if axis == 1 else a.T


def split_vs_oracle(core, axis, mode, sz, n_lines, sg_offs, facet_offs, seed,
                    nonzero_acc=True, rtol=1e-12, check_lines=None):
    """One ``split_subgrid_axis`` call against the oracle, line by line.

    :param sg_offs: one subgrid offset per group
    :param facet_offs: per group the list of target facet offsets (may repeat)
    :param check_lines: line indices to compare (default: all)
    Inputs and targets are C-ordered with the lines along the OTHER axis, so along axis 0 the
    lines are adjacent in memory (the two-line kernel form).
    """
    oracle = oracle_of(core)
    dev = _dev(core)
    rng = numpy.random.default_rng(seed)
    m, yN = core.xM_yN_size, core.yN_size
    size = yN if mode == "add" else m
    ins, targets, init = [], [], []
    for facets in facet_offs:
        a = pc.rand_c(rng, n_lines, sz)
        ins.append(numpy.ascontiguousarray(a if axis == 1 else a.T))
        grp = []
        for _ in facets:
            t0 = pc.rand_c(rng, n_lines, size) if (mode == "add" and nonzero_acc) else \
                numpy.zeros((n_lines, size), dtype=complex)
            init.append(t0)
            grp.append(numpy.ascontiguousarray(t0 if axis == 1 else t0.T))
        targets.append(grp)
    t_ins = [torch.from_numpy(a).to(dev) for a in ins]
    t_tgts = [[(torch.from_numpy(t.copy()).to(dev), off) for t, off in zip(grp, offs)]
              for grp, offs in zip(targets, facet_offs)]
    if mode == "store":  # the kernel must overwrite whatever is there
        for grp in t_tgts:
            for t, _ in grp:
                t.fill_(complex(numpy.nan, numpy.nan))
    core.split_subgrid_axis(t_ins, axis, sg_offs, t_tgts, mode)
    lines = range(n_lines) if check_lines is None else check_lines
    k = 0
    worst = 0.0
    for g, offs in enumerate(facet_offs):
        src = _lines_first(ins[g], axis)
        for j, off in enumerate(offs):
            got = _lines_first(t_tgts[g][j][0].cpu().numpy(), axis)
            ref = init[k].copy()
            k += 1
            # targets of several groups may share memory only in add mode, where the
            # caller passes the same initial values (see shared_accumulator_case)
            for line in lines:
                prep = oracle.prepare_subgrid(src[line], sg_offs[g])
                c = oracle.extract_from_subgrid(prep, off, axis=0)
                if mode == "add":
                    ref[line] = oracle.add_to_facet(c, sg_offs[g], axis=0, out=ref[line].copy())
                else:
                    ref[line] = c
            sel = list(lines)
            pc.close(got[sel], ref[sel], rtol=rtol,
                     what=f"axis {axis} {mode} group {g} target {j} (facet_off {off})")
            worst = max(worst, float(numpy.abs(got[sel] - ref[sel]).max()))
    return worst


def shared_accumulator_case(core, axis, seed, n_groups=3, n_lines=5):
    """Add mode, several groups (subgrids) adding into the SAME accumulators: the groups of a
    launch are applied in order by one CTA per line, so the result is the oracle's sum."""
    oracle = oracle_of(core)
    dev = _dev(core)
    rng = numpy.random.default_rng(seed)
    yN, xM = core.yN_size, core.xM_size
    step = core.subgrid_off_step
    sz = xM // 2 + 1
    facet_offs = [0, core.facet_off_step * 3, -core.facet_off_step * 5]
    accs0 = [pc.rand_c(rng, n_lines, yN) for _ in facet_offs]
    accs = [torch.from_numpy(numpy.array(a if axis == 1 else a.T, order="C")).to(dev)
            for a in accs0]
    ins0 = [pc.rand_c(rng, n_lines, sz) for _ in range(n_groups)]
    ins = [torch.from_numpy(numpy.ascontiguousarray(a if axis == 1 else a.T)).to(dev)
           for a in ins0]
    sg_offs = [(3 * g - 4) * step for g in range(n_groups)]
    core.split_subgrid_axis(ins, axis, sg_offs,
                            [[(a, f) for a, f in zip(accs, facet_offs)]] * n_groups, "add")
    for j, f in enumerate(facet_offs):
        ref = accs0[j].copy()
        for g in range(n_groups):
            for line in range(n_lines):
                c = oracle.extract_from_subgrid(oracle.prepare_subgrid(ins0[g][line], sg_offs[g]),
                                                f, axis=0)
                ref[line] = oracle.add_to_facet(c, sg_offs[g], axis=0, out=ref[line].copy())
        got = _lines_first(accs[j].cpu().numpy(), axis)
        pc.close(got, ref, rtol=1e-12, what=f"shared accumulator {j}, axis {axis}")


def chained_2d_vs_oracle(core, sz, sg_off, facet_offs, seed):
    """Both axes chained as SwiftlyBackward runs them (axis 0 into strips, axis 1 into column
    accumulators) against oracle.prepare_subgrid (2-D) + extract_from_subgrid x 2 +
    add_to_facet(axis 1)."""
    oracle = oracle_of(core)
    dev = _dev(core)
    rng = numpy.random.default_rng(seed)
    m, yN = core.xM_yN_size, core.yN_size
    sub = pc.rand_c(rng, sz, sz)
    rows = sorted({f0 for f0, _ in facet_offs})
    strips = torch.empty((len(rows), m, sz), dtype=torch.complex128, device=dev)
    t_sub = torch.from_numpy(sub).to(dev)
    core.split_subgrid_axis([t_sub], 0, [sg_off[0]], [[(strips[r], f0) for r, f0 in enumerate(rows)]],
                            "store")
    accs0 = [pc.rand_c(rng, m, yN) for _ in facet_offs]
    accs = [torch.from_numpy(a.copy()).to(dev) for a in accs0]
    groups, tg = [], []
    for r, f0 in enumerate(rows):
        groups.append(strips[r])
        tg.append([(accs[j], f1) for j, (a0, f1) in enumerate(facet_offs) if a0 == f0])
    core.split_subgrid_axis(groups, 1, [sg_off[1]] * len(rows), tg, "add")
    prep = oracle.prepare_subgrid(sub, (sg_off[0], sg_off[1]))
    for j, (f0, f1) in enumerate(facet_offs):
        c = oracle.extract_from_subgrid(oracle.extract_from_subgrid(prep, f0, axis=0), f1, axis=1)
        ref = oracle.add_to_facet(c, sg_off[1], axis=1, out=accs0[j].copy())
        pc.close(accs[j].cpu().numpy(), ref, rtol=1e-12, what=f"2-D chain, facet {j}")


def backward_inputs(cfg, sparse, n_subgrids, seed, shuffle=True, n_facets=4):
    """Facet configs (full cover or a sparse set) and subgrid configs / data for a backward
    transform; the subgrid order is shuffled so that subgrid columns interleave."""
    rng = numpy.random.default_rng(seed)
    core = cfg.core
    yB, xA = cfg.max_facet_size, cfg.max_subgrid_size
    if sparse:
        step = core.facet_off_step
        n_steps = core.N // step
        facet_cfgs = [FacetConfig(((3 * i) % n_steps - n_steps // 2) * step,
                                  ((5 * i + 1) % n_steps - n_steps // 2) * step, yB)
                      for i in range(n_facets)]
    else:
        facet_cfgs = make_full_facet_cover(cfg)
    sgs = make_full_subgrid_cover(cfg)
    sgs = [sgs[(7 * i) % len(sgs)] for i in range(min(n_subgrids, len(sgs)))]
    if shuffle:
        sgs = [sgs[i] for i in rng.permutation(len(sgs))]
    data = [pc.rand_c(rng, xA, xA) for _ in sgs]
    return facet_cfgs, sgs, data


def backward_vs_oracle(cfg, facet_cfgs, sgs, data, lru_backward=1, tol=1e-11):
    """SwiftlyBackward against backward_reference_order; returns the worst relative error
    (the primitive chain and the split kernels both land at 4e-12 .. 8e-12 of the largest facet
    sample at the small test geometries: the whole backward transform's rounding)."""
    core = cfg.core
    bwd = SwiftlyBackward(cfg, facet_cfgs, lru_backward=lru_backward)
    for sg, d in zip(sgs, data):
        bwd.add_new_subgrid_task(sg, torch.from_numpy(d).to(_dev(core)))
    got = [t.result() for t in bwd.finish()]
    ref = backward_reference_order(
        oracle_of(core), data, [(s.off0, s.off1) for s in sgs],
        [(c.off0, c.off1) for c in facet_cfgs], cfg.max_facet_size,
        facet_masks=[(c.mask0, c.mask1) for c in facet_cfgs])
    scale = max(numpy.abs(r).max() for r in ref)
    worst = max(numpy.abs(a - b).max() for a, b in zip(got, ref)) / scale
    assert worst <= tol, f"backward: max rel err {worst:.3e}"
    return worst
