"""
Fused subgrid kernel with partly empty rounds on the GPU, at the cfg4 geometry of bench.py
(N = 65536, xM = 4096, yN = 16384, m = 1024: four 1024-point transforms per round).  The
benchmark's central 5 x 5 facet block gives every line 5 sources in rounds of 3 + 2; the
default kernel (empty slots skipped, first round stored) is compared with the oracle and with
the former scheme (sg_variant 25: empty slots transform zeros), which must agree bit for bit.
"""

import numpy
import pytest

from oracle.swiftly_oracle import OracleCore
from tests import subgrid_round_cases as rc

pytestmark = pytest.mark.gpu

CFG4 = (13.5625, 65536, 4096, 16384)  # W, N, xM, yN
_cores = {}


def cores():
    if "cfg4" not in _cores:
        from ska_sdp_distributed_fourier_transform_b200 import SwiftlyCoreB200

        _cores["cfg4"] = (SwiftlyCoreB200(*CFG4, device=0), OracleCore(*CFG4))
    return _cores["cfg4"]


@pytest.mark.parametrize("variant", [0, 5])
def test_gpu_rounds_cfg4_k3_5x5(variant):
    """K3 as the step launches it: one group per facet row, 5 rows of 5 prepared facets; 135
    line pairs, so some CTAs walk two.  The former scheme gives the same bits."""
    core, oracle = cores()
    layouts = ["5_three_plus_two"] * 5
    new = rc.check_grouped(core, oracle, variant, "grouped", lines=54, layouts=layouts, seed=3)
    old = rc.check_grouped(core, oracle, rc.LEGACY_VARIANT if variant == 0 else variant,
                           "grouped", lines=54, layouts=layouts, seed=3)
    for a, b in zip(new, old):
        assert numpy.array_equal(a.cpu().numpy(), b.cpu().numpy())


def test_gpu_rounds_cfg4_k4_5x5():
    """K4: the 5 strips of a subgrid (contribution-sized, transposed) along axis 0."""
    core, oracle = cores()
    new = rc.check_single(core, oracle, "5_three_plus_two", axis=0, contrib_sized=True,
                          variant=0, lines=300, seed=5)
    old = rc.check_single(core, oracle, "5_three_plus_two", axis=0, contrib_sized=True,
                          variant=rc.LEGACY_VARIANT, lines=300, seed=5)
    assert numpy.array_equal(new.cpu().numpy(), old.cpu().numpy())


@pytest.mark.parametrize("layout", sorted(rc.LAYOUTS))
def test_gpu_rounds_cfg4_layouts(layout):
    core, oracle = cores()
    rc.check_single(core, oracle, layout, axis=1, contrib_sized=False, variant=0, lines=8)
    rc.check_single(core, oracle, layout, axis=0, contrib_sized=True, variant=0, lines=8)


@pytest.mark.parametrize("mode", ["grouped", "batched", "scattered"])
def test_gpu_rounds_cfg4_entry_points(mode):
    core, oracle = cores()
    rc.check_grouped(core, oracle, 0, mode, lines=6)
