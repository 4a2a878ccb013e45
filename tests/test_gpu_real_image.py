"""
The real-image forward transform on the H100 (``tests/real_image_cases.py``): ``mirror_subgrid``
exactly against numpy, and ``SwiftlyForward(real_image=True)`` bitwise against the default mode at
the full cfg2 cover (34 of 64 subgrids computed) and a 2 x 2 facet block of cfg4 over all 32 x 32
subgrids (514 computed), with the mirrored subgrids as accurate as the default path against the
analytic DFT and the work it saves counted.
"""

import random

import pytest
import torch

from ska_sdp_distributed_fourier_transform_b200 import (
    SwiftlyForward,
    make_facet_device,
    make_full_subgrid_cover,
)
from ska_sdp_distributed_fourier_transform_b200.core import SwiftlyCoreB200
from tests import host_tier_cases as hc
from tests import real_image_cases as rc

pytestmark = pytest.mark.gpu

make_config = hc.config_factory(SwiftlyCoreB200)


def _core():
    return make_config(**hc.params("8k[1]-n4k-2k")).core


@pytest.mark.parametrize("sz", [8, 9, 1024, 1025, 2048])
@pytest.mark.parametrize("masked", [(), (1, 2), (0, 1, 2, 3)], ids=["none", "some", "all"])
def test_gpu_mirror_subgrid(sz, masked):
    rc.mirror_case(_core(), sz, masked=masked, seed=sz)


@pytest.mark.parametrize("layout,extra,cap", [("wide", 0, 0), ("transposed", 3, 0),
                                              ("wide", 2, 1), ("own", 0, 2), ("transposed", 0, 3)])
def test_gpu_mirror_subgrid_layouts(layout, extra, cap):
    core = _core()
    for sz in (10, 13, 2048):
        rc.mirror_case(core, sz, extra=extra, masked=(0, 3), layout=layout, cap=cap, seed=sz)


def test_gpu_mirror_subgrid_rejects():
    rc.mirror_rejects(_core())


def _real_facets(cfg, facet_cfgs, sources):
    return [make_facet_device(cfg.image_size, fc, sources, torch.device("cuda")).real.contiguous()
            for fc in facet_cfgs]


@pytest.mark.parametrize("name,block,n", [("8k[1]-n4k-2k", None, 8), ("64k[1]-n16k-4k", 2, 32)])
def test_gpu_real_image_cover(name, block, n):
    """Every subgrid of the cover bitwise against the default mode; K2 for n/2 + 1 columns,
    n^2/2 + 2 subgrids computed; 3 pairs and the self-mirrored subgrids against the DFT."""
    cfg = make_config(**hc.params(name))
    facet_cfgs = hc.facet_configs(cfg, name, block)
    sources = rc.point_sources(cfg.image_size, facet_cfgs, 8, 17)
    facets = _real_facets(cfg, facet_cfgs, sources)
    sg_cfgs = make_full_subgrid_cover(cfg)
    assert len(sg_cfgs) == n * n
    pairs = rc.api.mirror_pairs(sg_cfgs, cfg.image_size, cfg.internal_subgrid_size)
    accuracy = rc.accuracy_set(cfg, sg_cfgs, pairs)
    pairs, work, errors = rc.driver_case(cfg, facet_cfgs, facets, sg_cfgs, sources=sources,
                                         accuracy=accuracy)
    columns, computed, prepared = rc.full_cover_counts(n)
    assert (len(pairs), len(work.k2_columns), work.sum_finish, work.prepared) == (
        computed, columns, 2 * computed, prepared)
    print(f"\n{name}: {computed} of {n * n} subgrids computed, K2 for {columns} of {n} columns; "
          f"max rel err real {max(errors['real'].values()):.2e}, "
          f"default {max(errors['default'].values()):.2e}")


def test_gpu_real_image_host_tier():
    """cfg2 in the host tier (``device_budget=1``), shuffled, lru 2: bitwise against the default
    device tier."""
    name = "8k[1]-n4k-2k"
    cfg = make_config(**hc.params(name))
    facet_cfgs = hc.facet_configs(cfg, name)
    sources = rc.point_sources(cfg.image_size, facet_cfgs, 8, 23)
    facets = _real_facets(cfg, facet_cfgs, sources)
    sg_cfgs = make_full_subgrid_cover(cfg)
    random.Random(2).shuffle(sg_cfgs)
    rc.driver_case(cfg, facet_cfgs, facets, sg_cfgs, lru=2, budget=1)


def test_gpu_real_image_rejects():
    cfg = make_config(**hc.params("8k[1]-n4k-2k"))
    facet_cfgs = hc.facet_configs(cfg, "8k[1]-n4k-2k")[:2]
    facets = [torch.zeros((fc.size, fc.size), dtype=torch.float64) for fc in facet_cfgs]
    rc.rejects_complex(cfg, facet_cfgs, [f.numpy() for f in facets])
    SwiftlyForward(cfg, list(zip(facet_cfgs, facets)), real_image=True)
