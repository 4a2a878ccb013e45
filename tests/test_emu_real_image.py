"""
The real-image forward transform on the host-emulated kernels (``tests/real_image_cases.py``):
``mirror_subgrid`` exactly against numpy, and ``SwiftlyForward(real_image=True)`` bitwise against
the default mode at a full cover, a sparse facet list with shuffled subgrids, ``lru_forward=2``,
the host tier and an odd subgrid size, with the work it saves counted.
"""

import random

import pytest

from ska_sdp_distributed_fourier_transform_b200 import (
    SwiftlyForward,
    make_facet,
    make_full_facet_cover,
    make_full_subgrid_cover,
)
from tests import host_tier_cases as hc
from tests import real_image_cases as rc
from tests.emu_support import emu_core_class

make_config = hc.config_factory(lambda W, N, xM, yN: emu_core_class()(W, N, xM, yN))

# N = 1280, xA = 160: an 8 x 8 cover; yN = 640 runs the mixed-radix K2 forms
COVER = "1280[1]-n640-256"
# (192, 384) family, odd xA = 345 (its cover is broken for odd sizes: explicit configs)
ODD = "1536[1]-n768-384"


def _core():
    return make_config(**hc.params(COVER)).core


@pytest.mark.parametrize("sz", [8, 9, 160, 161])
@pytest.mark.parametrize("masked", [(), (1, 2), (0, 1, 2, 3)], ids=["none", "some", "all"])
def test_emu_mirror_subgrid(sz, masked):
    rc.mirror_case(_core(), sz, masked=masked, seed=sz)


@pytest.mark.parametrize("layout,extra,cap", [("wide", 0, 0), ("transposed", 3, 0),
                                              ("wide", 2, 1), ("own", 0, 2), ("transposed", 0, 3)])
def test_emu_mirror_subgrid_layouts(layout, extra, cap):
    """Outputs inside wider arrays and transposed, a source larger than ``2h + 1``, capped
    grids (every CTA walks several rows)."""
    core = _core()
    for sz in (10, 13):
        rc.mirror_case(core, sz, extra=extra, masked=(0, 3), layout=layout, cap=cap, seed=sz)


def test_emu_mirror_subgrid_cfg4_size():
    """cfg4's subgrid size: sz = 2048 from a 2049 x 2049 source, every mask."""
    rc.mirror_case(_core(), 2048, masked=(0, 1, 2, 3), layout="wide")


def test_emu_mirror_subgrid_rejects():
    rc.mirror_rejects(_core())


def _cover_setup(facet_offs=None, seed=3):
    cfg = make_config(**hc.params(COVER))
    facet_cfgs = (make_full_facet_cover(cfg) if facet_offs is None
                  else rc.facet_block(cfg, facet_offs))
    sources = rc.point_sources(cfg.image_size, facet_cfgs, 6, seed)
    facets = [make_facet(cfg.image_size, fc, sources).real for fc in facet_cfgs]
    return cfg, facet_cfgs, facets, sources


def test_emu_full_cover():
    """8 x 8 cover in cover order: 34 of 64 subgrids computed, K2 for 5 of 8 columns, every
    subgrid bitwise equal to the default mode's and as accurate against the analytic DFT."""
    cfg, facet_cfgs, facets, sources = _cover_setup()
    sg_cfgs = make_full_subgrid_cover(cfg)
    assert len(sg_cfgs) == 64
    pairs, work, _ = rc.driver_case(cfg, facet_cfgs, facets, sg_cfgs, sources=sources)
    columns, computed, prepared = rc.full_cover_counts(8)
    assert (len(pairs), len(work.k2_columns), work.sum_finish, work.prepared) == (
        computed, columns, 2 * computed, prepared)
    assert len(rc.self_mirrored(cfg, sg_cfgs)) == 4


@pytest.mark.parametrize("lru,budget", [(1, None), (2, None), (3, 1)],
                         ids=["device", "lru2", "host-tier-lru3"])
def test_emu_sparse_shuffled(lru, budget):
    """A sparse facet list and the cover shuffled; device and host tier, lru 1 to 3."""
    cfg, facet_cfgs, facets, sources = _cover_setup(
        [(0, 0), (0, 440), (440, -440), (-440, 440), (-440, 0)], seed=5)
    sg_cfgs = make_full_subgrid_cover(cfg)
    random.Random(lru).shuffle(sg_cfgs)
    pairs, _, _ = rc.driver_case(cfg, facet_cfgs, facets, sg_cfgs, lru=lru, budget=budget,
                                 sources=sources if lru == 1 else None)
    assert len(pairs) == 34


def test_emu_host_tier_equals_device_tier():
    """Real mode in the host tier gives the device tier's bits."""
    cfg, facet_cfgs, facets, _ = _cover_setup()
    sg_cfgs = make_full_subgrid_cover(cfg)[:24]
    res = {}
    for budget in (None, 1):
        fwd = SwiftlyForward(cfg, list(zip(facet_cfgs, facets)), device_budget=budget,
                             real_image=True)
        assert fwd.host_tier == (budget is not None)
        res[budget] = {i: t.result() for i, t in fwd.iter_subgrid_tasks(sg_cfgs)}
    assert sorted(res[None]) == list(range(24))
    for i, a in res[None].items():
        assert (a == res[1][i]).all(), f"subgrid {i}: host tier differs from the device tier"


def test_emu_odd_size_and_unpaired():
    """Odd xA = 345 (S = sz) with unmasked explicit configs: pairs, a self-mirrored config, a
    config whose mirror is missing, and a duplicate pair."""
    cfg = make_config(**hc.params(ODD))
    N = cfg.image_size
    facet_cfgs = rc.facet_block(cfg, [(0, 0), (0, 512), (512, -512), (-512, 0)])
    sources = rc.point_sources(N, facet_cfgs, 5, 11)
    facets = [make_facet(N, fc, sources).real for fc in facet_cfgs]
    offs = [(0, 0), (192, 384), (-384, 96), (768, 0), (-192, -384), (384, -96), (96, 96),
            (192, 384), (-192, -384), (-96, 768), (96, -768), (768, 768)]
    sg_cfgs = rc.explicit_configs(cfg, offs)
    pairs, _, _ = rc.driver_case(cfg, facet_cfgs, facets, sg_cfgs, sources=sources)
    assert pairs == [(0, None), (1, 4), (2, 5), (3, None), (6, None), (7, 8), (9, 10),
                     (11, None)]


def test_emu_rejects():
    """Complex facets raise ValueError naming the facet; a core without the fused forward kernels
    raises NotImplementedError."""
    cfg, facet_cfgs, facets, _ = _cover_setup()
    rc.rejects_complex(cfg, facet_cfgs, facets)
    cfg.core.fused_forward_supported = lambda: False
    with pytest.raises(NotImplementedError):
        SwiftlyForward(cfg, list(zip(facet_cfgs, facets)), real_image=True)
    SwiftlyForward(cfg, list(zip(facet_cfgs, facets)))  # the default mode is unaffected
