"""
The host tier on the H100 (``tests/host_tier_cases.py``): ``SwiftlyForward`` /
``SwiftlyBackward`` with the facet arrays in pinned host memory are bitwise equal to the device
tier at cfg2 (full cover), a 3 x 3 block of cfg3 and a 2 x 2 block of cfg4, where the rings run
the same K2 kernel as whole facets (``ExtractColumnsTma4Kernel``); the reference round trip in
the host tier; and the device memory the host tier holds does not grow with the facet arrays.
"""

import numpy
import pytest
import torch

from ska_sdp_distributed_fourier_transform_b200 import (
    SwiftlyBackward,
    SwiftlyForward,
    check_facet,
    check_subgrid,
    make_facet,
    make_full_facet_cover,
    make_full_subgrid_cover,
)
from ska_sdp_distributed_fourier_transform_b200.core import SwiftlyCoreB200
from tests import host_tier_cases as hc
from tests import k2_cases as kc

pytestmark = pytest.mark.gpu

make_config = hc.config_factory(SwiftlyCoreB200)


def _facets(cfg, facet_cfgs, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    out = []
    for fc in facet_cfgs:
        f = torch.empty((fc.size, fc.size), dtype=torch.complex128, device="cuda")
        torch.view_as_real(f).normal_(generator=gen)
        out.append(f)
    return out


@pytest.mark.parametrize("name,block,columns", [("8k[1]-n4k-2k", None, None),
                                                ("32k[1]-n8k-4k", 3, None),
                                                ("64k[1]-n16k-4k", 2, 3)])
def test_gpu_host_tier_equals_device_tier(name, block, columns):
    """Forward and backward, subgrids in cover order (at cfg4 the first ``columns`` subgrid
    columns), lru 1: the host tier gives the device tier's bits and moves the cover-order rows."""
    cfg = make_config(**hc.params(name))
    core = cfg.core
    facet_cfgs = hc.facet_configs(cfg, name, block)
    facets = _facets(cfg, facet_cfgs, 7)
    sg_cfgs = make_full_subgrid_cover(cfg)
    if columns:
        keep = sorted({s.off0 for s in sg_cfgs})[:columns]
        sg_cfgs = [s for s in sg_cfgs if s.off0 in keep]
    fwds = [SwiftlyForward(cfg, list(zip(facet_cfgs, facets)), lru_forward=1, queue_size=4,
                           device_budget=budget) for budget in (None, 1)]
    assert [f.host_tier for f in fwds] == [False, True]
    bwds = [SwiftlyBackward(cfg, facet_cfgs, lru_backward=1, queue_size=4, device_budget=budget)
            for budget in (None, 1)]
    assert [b.host_tier for b in bwds] == [False, True]
    checked_k2 = False
    for i, sg in enumerate(sg_cfgs):
        if name.startswith("64k") and not checked_k2 and fwds[1].lru.get(sg.off0) is None:
            fwds[1].get_NMBF_BFs_off0(sg.off0, fwds[1]._get_BF_Fs())  # pylint: disable=protected-access
            assert kc.last_launch(core)[0] == kc.TMA4  # the rings run ExtractColumnsTma4Kernel
            checked_k2 = True
        a = fwds[0].get_subgrid_task(sg).tensor
        b = fwds[1].get_subgrid_task(sg).tensor
        assert torch.equal(a, b), f"subgrid {i}: host tier differs from the device tier"
        for bwd in bwds:
            bwd.add_new_subgrid_task(sg, a)
    assert checked_k2 or not name.startswith("64k")
    got = [[t.tensor for t in bwd.finish()] for bwd in bwds]
    for j, (a, b) in enumerate(zip(*got)):
        assert a.is_cuda and not b.is_cuda
        assert torch.equal(a.cpu(), b), f"facet {j}: host tier differs from the device tier"
    rows = hc.cover_rows(core, sg_cfgs)
    assert fwds[1].h2d_rows == rows
    assert bwds[1].d2h_rows == rows and bwds[1].h2d_rows + bwds[1].zeroed_rows == rows


def test_gpu_host_tier_round_trip():
    """The reference's round trip (unit source, facet error < 3e-10) in the host tier."""
    cfg = make_config(**hc.params("1k[1]-n512-256"))
    sources = [(1, 1, 0)]
    facet_cfgs = make_full_facet_cover(cfg)
    fwd = SwiftlyForward(cfg, [(fc, make_facet(cfg.image_size, fc, sources)) for fc in facet_cfgs],
                         lru_forward=1, queue_size=100, device_budget=1)
    bwd = SwiftlyBackward(cfg, facet_cfgs, lru_backward=1, queue_size=100, device_budget=1)
    assert fwd.host_tier and bwd.host_tier
    worst = 0.0
    for sg in make_full_subgrid_cover(cfg):
        task = fwd.get_subgrid_task(sg)
        worst = max(worst, check_subgrid(cfg.image_size, sg, task.tensor, sources))
        bwd.add_new_subgrid_task(sg, task)
    assert worst < 1e-13
    for fc, task in zip(facet_cfgs, bwd.finish()):
        assert check_facet(cfg.image_size, fc, task.result(), sources) < 3e-10


def test_gpu_host_tier_device_memory():
    """Peak torch allocation of a cfg3 3 x 3 host-tier forward + backward stays under rings +
    columns + strips + staging buffers + facets in flight, well below the facet arrays."""
    name = "32k[1]-n8k-4k"
    p = hc.params(name)
    cfg = make_config(**p)
    core = cfg.core
    m, yN, yB, xA = core.xM_yN_size, p["yN"], p["yB"], p["xA"]
    facet_cfgs = hc.facet_configs(cfg, name, 3)
    F, rows = len(facet_cfgs), 3
    rng = numpy.random.default_rng(1)
    facets = [rng.standard_normal((yB, yB)) + 0j for _ in facet_cfgs]
    sg_cfgs = make_full_subgrid_cover(cfg)
    sg_cfgs = [s for s in sg_cfgs if s.off0 in sorted({s.off0 for s in sg_cfgs})[:4]]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fwd = SwiftlyForward(cfg, list(zip(facet_cfgs, facets)), lru_forward=1, queue_size=4,
                         device_budget=1)
    bwd = SwiftlyBackward(cfg, facet_cfgs, lru_backward=1, queue_size=4, device_budget=1)
    for sg in sg_cfgs:
        bwd.add_new_subgrid_task(sg, fwd.get_subgrid_task(sg))
    bwd.finish()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    bound = 16 * (2 * F * m * yB            # forward and backward rings
                  + 2 * F * m * yN          # one column of each direction
                  + rows * m * xA           # subgrid strips
                  + 2 * yN * yB + yN * yB   # stage-1 buffers, the finish buffer
                  + 2 * yB * yB             # facets in flight (upload, finished facet)
                  + 8 * xA * xA) + (64 << 20)
    print(f"\npeak {peak / 2**30:.3f} GiB, bound {bound / 2**30:.3f} GiB, "
          f"facet arrays {16 * F * yN * yB / 2**30:.3f} GiB")
    assert peak <= bound
    assert bound < 2 * 16 * F * yN * yB  # the device tier holds BF_F and the accumulators
