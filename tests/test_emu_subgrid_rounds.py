"""
Fused subgrid kernel with partly empty rounds on the host-emulated kernels (every CUDA thread
a fibre, named barriers with the hardware's counting semantics): slots without a source skip
their transform, the first round stores and its empty slots clear the rest of the
accumulator.  An unbalanced barrier shows up as the emulator's deadlock report, a position
left uncleared as the poison the emulator fills shared memory with.  m = 512 and 1024 make a
transform whole warps (the form in which empty slots are skipped); CONC = 4 and 2.
"""

import numpy
import pytest

from oracle.swiftly_oracle import OracleCore
from tests import subgrid_round_cases as rc
from tests.emu_support import emu_core_class

# (N, xM, yN): m = xM * yN / N
GEOMETRIES = {"conc4": (8192, 2048, 2048), "conc2": (4096, 2048, 2048)}
_cores = {}


def cores(name):
    if name not in _cores:
        N, xM, yN = GEOMETRIES[name]
        _cores[name] = (emu_core_class()(13.5625, N, xM, yN), OracleCore(13.5625, N, xM, yN))
    return _cores[name]


@pytest.mark.parametrize("variant", [0, 5])
@pytest.mark.parametrize("layout", sorted(rc.LAYOUTS))
def test_emu_rounds_axis1_facet_rows(layout, variant):
    core, oracle = cores("conc4")
    rc.check_single(core, oracle, layout, axis=1, contrib_sized=False, variant=variant)


@pytest.mark.parametrize("layout", sorted(rc.LAYOUTS))
def test_emu_rounds_axis0_strips(layout):
    core, oracle = cores("conc4")
    rc.check_single(core, oracle, layout, axis=0, contrib_sized=True, variant=0)


@pytest.mark.parametrize("layout", ["1", "2_clashing", "3_disjoint", "5_three_plus_two"])
def test_emu_rounds_two_per_round(layout):
    core, oracle = cores("conc2")
    rc.check_single(core, oracle, layout, axis=1, contrib_sized=False, variant=0)


@pytest.mark.parametrize("variant", [0, 5])
@pytest.mark.parametrize("mode", ["grouped", "batched", "scattered"])
def test_emu_rounds_entry_points(mode, variant):
    core, oracle = cores("conc4")
    rc.check_grouped(core, oracle, variant, mode)


def test_emu_rounds_legacy_variant_bit_identical():
    """Storing the first round's products instead of adding them to zeros changes nothing."""
    core, oracle = cores("conc4")
    for layout in sorted(rc.LAYOUTS):
        new = rc.check_single(core, oracle, layout, 1, False, 0, seed=4)
        old = rc.check_single(core, oracle, layout, 1, False, rc.LEGACY_VARIANT, seed=4)
        assert numpy.array_equal(new.numpy(), old.numpy()), layout


def test_emu_rounds_many_lines_per_cta():
    """More line pairs than CTAs (132): CTAs walk several lines, so the TMA staging wait, the
    prefetch of the next line's windows and the round-0 stores run line after line.  The
    CTAs that walk two line pairs meet the 3 + 2 rounds after a tiled line: an accumulator
    position left uncleared would still hold that line's xM exchange."""
    core, oracle = cores("conc4")
    layouts = ["8_tiled", "1", None, "5_three_plus_two"]
    rc.check_grouped(core, oracle, 0, "grouped", lines=71, layouts=layouts, seed=9)
