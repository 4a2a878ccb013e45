"""
The real-image backward transform on the H100 (``tests/real_backward_cases.py``):
``merge_mirror_subgrid`` exactly against numpy and as the adjoint of ``mirror_subgrid``,
``finish_facet_real`` bitwise against ``finish_facet`` at the catalogue's facet lengths (the
2 x 8192 split at yN = 16384 included), and ``SwiftlyBackward(real_image=True)`` at the full cfg2
cover and a 2 x 2 facet block of cfg4 over all 32 x 32 subgrids, against the analytic facets and
the default mode, with the work it saves counted.
"""

import random

import pytest
import torch

from ska_sdp_distributed_fourier_transform_b200 import SwiftlyBackward, make_full_subgrid_cover
from ska_sdp_distributed_fourier_transform_b200.core import SwiftlyCoreB200
from tests import host_tier_cases as hc
from tests import real_backward_cases as rb
from tests import real_image_cases as rc

pytestmark = pytest.mark.gpu

make_config = hc.config_factory(SwiftlyCoreB200)
CFG2 = "8k[1]-n4k-2k"
CFG4 = "64k[1]-n16k-4k"


def _core(name=CFG2):
    return make_config(**hc.params(name)).core


@pytest.mark.parametrize("sz", [8, 9, 160, 161, 2048])
def test_gpu_merge_mirror_subgrid(sz):
    rb.merge_case(_core(), sz, seed=sz)


@pytest.mark.parametrize("layout,transposed_inputs,cap", [
    ("wide", False, 0), ("transposed", False, 0), ("own", True, 0), ("wide", True, 1),
    ("own", False, 2), ("transposed", True, 3)])
def test_gpu_merge_mirror_subgrid_layouts(layout, transposed_inputs, cap):
    core = _core()
    for sz in (10, 13, 2048):
        rb.merge_case(core, sz, layout=layout, transposed_inputs=transposed_inputs, cap=cap,
                      seed=sz)


def test_gpu_merge_mirror_subgrid_rejects():
    rb.merge_rejects(_core())


@pytest.mark.parametrize("sz", [8, 9, 1024, 1025])
def test_gpu_merge_is_adjoint_of_mirror(sz):
    rb.adjoint_case(_core(), sz, seed=sz)


@pytest.mark.parametrize("name", [CFG2, "1280[1]-n640-256", CFG4])
@pytest.mark.parametrize("axis", [0, 1])
def test_gpu_finish_facet_real(name, axis):
    """Direct (4096), split-F (640) and the 2 x 8192 split (16384), with and without a mask,
    into own, wide and transposed outputs; a capped grid."""
    core = _core(name)
    fs = hc.params(name)["yB"]
    n_lines = 3 if name == CFG4 else 6
    for k, (masked, layout, cap) in enumerate([(True, "own", 0), (False, "wide", 0),
                                               (True, "transposed", 2)]):
        rb.finish_real_case(core, fs, axis, n_lines=n_lines, masked=masked, layout=layout,
                            cap=cap, seed=k)


def test_gpu_finish_facet_real_rejects():
    rb.finish_real_rejects(_core())


def test_gpu_unpaired_is_re_of_default():
    """Real mode through add_new_subgrid_task only: bitwise Re of the default, both tiers."""
    cfg = make_config(**hc.params(CFG2))
    facet_cfgs = hc.facet_configs(cfg, CFG2)
    sources = rc.point_sources(cfg.image_size, facet_cfgs, 8, 29)
    sg_cfgs = make_full_subgrid_cover(cfg)[::5]
    subgrids = rb.hermitian_subgrids(cfg, sg_cfgs, sources)
    for budget in (None, 1):
        rb.unpaired_bitwise(cfg, facet_cfgs, sg_cfgs, subgrids, budget=budget)


def test_gpu_cfg2_cover():
    """The full cfg2 cover: 34 of 64 subgrid sides, 30 merges, 5 of 8 columns folded; against the
    analytic facets and the default mode."""
    cfg = make_config(**hc.params(CFG2))
    facet_cfgs = hc.facet_configs(cfg, CFG2)
    sources = rc.point_sources(cfg.image_size, facet_cfgs, 8, 17)
    sg_cfgs = make_full_subgrid_cover(cfg)
    _, work, _, errs = rb.paired_case(cfg, facet_cfgs, sg_cfgs, sources)
    sides, merges, columns = rb.full_cover_work(8)
    assert (work.sides, work.merge, len(set(work.folds))) == (sides, merges, columns)
    print(f"\n{CFG2}: errors {errs}")


def test_gpu_cfg2_host_tier_shuffled():
    """cfg2 in the host tier, shuffled, lru 2: against the analytic facets and the default."""
    cfg = make_config(**hc.params(CFG2))
    facet_cfgs = hc.facet_configs(cfg, CFG2)
    sources = rc.point_sources(cfg.image_size, facet_cfgs, 8, 23)
    sg_cfgs = make_full_subgrid_cover(cfg)
    random.Random(2).shuffle(sg_cfgs)
    rb.paired_case(cfg, facet_cfgs, sg_cfgs, sources, lru=2, budget=1)


def test_gpu_cfg4_block():
    """A 2 x 2 cfg4 facet block over all 32 x 32 subgrids: 514 subgrid sides, 510 merges, 17 of
    32 columns folded; against the default mode."""
    cfg = make_config(**hc.params(CFG4))
    facet_cfgs = hc.facet_configs(cfg, CFG4, 2)
    sg_cfgs = make_full_subgrid_cover(cfg)
    assert len(sg_cfgs) == 1024
    # 1024 analytic subgrids would take 64 GiB: 16 random device subgrids fed cyclically (the
    # identity holds for any subgrid data)
    gen = torch.Generator(device="cuda").manual_seed(31)
    inputs = [torch.randn((2048, 2048), dtype=torch.complex128, device="cuda", generator=gen)
              for _ in range(16)]
    _, work, _, errs = rb.paired_case(cfg, facet_cfgs, sg_cfgs, None,
                                      subgrids=[inputs[i % 16] for i in range(1024)], agree=1e-6)
    sides, merges, columns = rb.full_cover_work(32)
    assert (work.sides, work.merge, len(work.folds), len(set(work.folds))) == (
        sides, merges, columns, columns)
    print(f"\n{CFG4} 2 x 2: errors {errs}")


def test_gpu_round_trip():
    cfg = make_config(**hc.params(CFG2))
    facet_cfgs = hc.facet_configs(cfg, CFG2)
    errs = rb.round_trip(cfg, facet_cfgs, make_full_subgrid_cover(cfg), [(1, 1, 0), (1, -37, 52)])
    print(f"\nround trip RMS: {errs}")


def test_gpu_rejects():
    cfg = make_config(**hc.params(CFG2))
    facet_cfgs = hc.facet_configs(cfg, CFG2)[:2]
    with pytest.raises(ValueError):
        SwiftlyBackward(cfg, facet_cfgs, real_image=True).add_subgrid_tasks(
            make_full_subgrid_cover(cfg)[:2], [None])
