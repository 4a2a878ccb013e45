"""
The fused subgrid split kernel (the subgrid side of the backward transform) on an H100: the
kernel at the benchmark's cfg4 shapes against the oracle, the new subgrid side against the
primitive chain it replaces at cfg2 and cfg4 sizes, and SwiftlyBackward at the smallest entry of
every catalogue family against the oracle.
"""

import numpy
import pytest
import torch

from ska_sdp_distributed_fourier_transform_b200 import SwiftlyBackward
from ska_sdp_distributed_fourier_transform_b200.core import SwiftlyCoreB200
from ska_sdp_distributed_fourier_transform_b200.swift_configs import SWIFT_CONFIGS
from tests import catalogue_cases as cc
from tests import split_cases as sc

pytestmark = pytest.mark.gpu

CFG4 = "64k[1]-n16k-4k"  # m = 1024, xM = 4096, xA = 2048
CFG2 = "8k[1]-n4k-2k"
_cores = {}


def core_of(name):
    if name not in _cores:
        p = SWIFT_CONFIGS[name]
        _cores[name] = SwiftlyCoreB200(p["W"], p["N"], p["xM_size"], p["yN_size"], device=0)
    return _cores[name]


@pytest.mark.parametrize("axis", [1, 0])
@pytest.mark.parametrize("mode", ["store", "add"])
def test_gpu_split_kernel_cfg4(axis, mode):
    """cfg4 shapes (odd and even subgrid sizes, offsets below zero and beyond N, a partial
    round of five targets at CONC 4, repeated windows), sampled lines against the oracle."""
    core = core_of(CFG4)
    assert core.split_axis_supported()
    N, fs, ss = core.N, core.facet_off_step, core.subgrid_off_step
    f_offs = [0, 8192, 8192, -16384, N + 49152]
    lines = [0, 1, 2, 77, 128, 200, 254, 255]
    sc.split_vs_oracle(core, axis, mode, 2048, 256, [-3 * ss, N + 5 * ss],
                       [f_offs, [16 * fs]], seed=axis, check_lines=lines)
    sc.split_vs_oracle(core, axis, mode, 2047, 256, [2048], [[-8192, 24576, 0]], seed=4,
                       check_lines=lines)


def _old_vs_new(core, xA, rows, fcs, sg_off, seed):
    dev = torch.device("cuda", 0)
    rng = numpy.random.default_rng(seed)
    x = torch.from_numpy(rng.standard_normal((xA, xA)) + 1j * rng.standard_normal((xA, xA))).to(dev)
    m, yN = core.xM_yN_size, core.yN_size
    new = [torch.zeros((m, yN), dtype=torch.complex128, device=dev) for _ in fcs]
    old = [torch.zeros((m, yN), dtype=torch.complex128, device=dev) for _ in fcs]
    strips = torch.empty((len(rows), m, xA), dtype=torch.complex128, device=dev)
    core.split_subgrid_axis([x], 0, [sg_off[0]], [[(strips[r], o) for r, o in enumerate(rows)]],
                            "store")
    core.split_subgrid_axis([strips[r] for r in range(len(rows))], 1, [sg_off[1]] * len(rows),
                            [[(new[j], f1) for j, (f0, f1) in enumerate(fcs) if f0 == o]
                             for o in rows], "add")
    prepared = core.prepare_subgrid(x, sg_off)
    blocks = {o: core.extract_from_subgrid(prepared, o, axis=0) for o in rows}
    core.subgrid_to_facets([blocks[f0] for f0, _ in fcs], old, [f1 for _, f1 in fcs], sg_off[1])
    scale = max(float(a.abs().max()) for a in old)
    err = max(float((a - b).abs().max()) for a, b in zip(new, old))
    assert err <= 1e-12 * scale, f"split vs primitive chain: {err:.3e} ({scale:.3e})"


def test_gpu_split_vs_primitive_chain_cfg4():
    core = core_of(CFG4)
    block = [0, 8192, 16384, 49152, 57344]
    fcs = [(a, b) for a in block for b in block]
    _old_vs_new(core, 2048, block, fcs, (3 * 2048 - 32768, 2048 * 5), seed=1)


def test_gpu_split_vs_primitive_chain_cfg2():
    core = core_of(CFG2)
    step = core.facet_off_step * (SWIFT_CONFIGS[CFG2]["yB_size"] // core.facet_off_step)
    offs = [k * step for k in range(core.N // step)]
    fcs = [(a, b) for a in offs for b in offs]
    _old_vs_new(core, SWIFT_CONFIGS[CFG2]["xA_size"], offs, fcs, (-1024, 2048), seed=2)


@pytest.mark.parametrize("pair", sorted(cc.SMALLEST), ids=cc.pair_id)
def test_gpu_backward_smallest_catalogue_entries(pair):
    """SwiftlyBackward on the split kernels at the smallest entry of each family, against the
    oracle; the primitive chain on the same inputs sets the bar where both are above 1e-11."""
    cfg = cc.make_config(SwiftlyCoreB200, cc.catalogue_plan(cc.SMALLEST[pair]))
    facet_cfgs, sgs, data = sc.backward_inputs(cfg, True, 4, seed=pair[0])
    assert SwiftlyBackward(cfg, facet_cfgs)._split
    cfg.core.split_axis_supported = lambda: False
    old = sc.backward_vs_oracle(cfg, facet_cfgs, sgs, data, tol=1.0)
    del cfg.core.split_axis_supported
    new = sc.backward_vs_oracle(cfg, facet_cfgs, sgs, data, tol=max(1e-11, 2 * old))
    print(f"{cc.SMALLEST[pair]}: backward max rel err split {new:.2e}, primitive chain {old:.2e}")


def test_gpu_sharded_backward_world_one_uses_split():
    """SwiftlyBackwardSharded without a process group (world size 1) runs the split kernels."""
    from ska_sdp_distributed_fourier_transform_b200.distributed import SwiftlyBackwardSharded

    cfg = cc.make_config(SwiftlyCoreB200, cc.catalogue_plan(cc.SMALLEST[(160, 320)]))
    facet_cfgs, sgs, data = sc.backward_inputs(cfg, True, 4, seed=3)
    bwd = SwiftlyBackwardSharded(cfg, facet_cfgs)
    assert bwd._split
    bwd.add_subgrid_tasks(sgs, data)
    got = [t.result() for _, t in sorted(bwd.finish().items())]
    ref = SwiftlyBackward(cfg, facet_cfgs)
    ref._split = False
    for s, d in zip(sgs, data):
        ref.add_new_subgrid_task(s, d)
    want = [t.result() for t in ref.finish()]
    scale = max(numpy.abs(w).max() for w in want)
    assert max(numpy.abs(a - b).max() for a, b in zip(got, want)) <= 1e-11 * scale
