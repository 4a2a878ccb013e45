"""
The fused subgrid kernels at every (m, xM) pair of the library on the host-emulated kernels, in
the forms the H100 runs (the emulated build dispatches like the GPU build): ``sum_finish_axis``
(the round-1 and the two-group kernel, direct stores and TMA staging) and ``split_subgrid_axis``
against the oracle, every case asserting the kernel form it was written for
(``swiftly_b200_debug_last_launch``, tests/pair_cases.py), and the extended-precision spot check.
The emulator reports a named barrier with a thread count that is not whole warps as a protocol
error, so a barrier scheme that only the emulator could run fails here.
"""

import pytest

from ska_sdp_distributed_fourier_transform_b200.swift_configs import (
    FUSED_FORWARD_PAIRS,
    SWIFT_CONFIGS,
)
from tests import pair_cases as prc
from tests.emu_support import emu_core_class

PAIRS = prc.ALL_PAIRS
TWO_GROUP_PAIRS = [p for p in PAIRS if prc.FORMS[p][0][0] == prc.TWO_GROUP]
_cores = {}


def core(pair):
    if pair not in _cores:
        _cores.clear()
        _cores[pair] = emu_core_class()(*prc.small_plan(pair))
    return _cores[pair]


def test_pair_table_covers_the_catalogue_and_the_library():
    """The catalogue's 13 pairs (with their entry counts) and the 7 library-only pairs are
    exactly the pairs of the pinned table; CONC is what the library reports."""
    assert {p: n for p, (n, _) in prc.CATALOGUE.items()} == {
        (128, 256): 17, (128, 512): 17, (256, 512): 21, (256, 1024): 52, (512, 1024): 52,
        (1024, 2048): 1, (1024, 4096): 2, (128, 1024): 52, (256, 256): 17, (128, 384): 4,
        (160, 320): 4, (192, 384): 4, (224, 448): 4}
    assert sum(n for n, _ in prc.CATALOGUE.values()) == len(SWIFT_CONFIGS) == 247
    assert prc.LIBRARY_ONLY == [(32, 64), (32, 128), (64, 128), (64, 256), (512, 2048),
                                (2048, 4096), (2048, 8192)]
    assert set(prc.FORMS) == set(FUSED_FORWARD_PAIRS) == set(prc.CATALOGUE) | set(prc.LIBRARY_ONLY)
    lib = core((32, 64))._lib
    for (m, xM), form in prc.FORMS.items():
        c = emu_core_class()(*prc.small_plan((m, xM)))
        assert (c.xM_yN_size, c.xM_size) == (m, xM)
        assert lib.swiftly_b200_sum_finish_axis_supported(c._plan) == form[3], (m, xM)
        # the TMA threshold: ceil(sz / box) * box samples (box = min(sz, 256)) in the work area
        if form[4] is not None:
            assert form[4] == xM // 2 and form[4] % min(form[4], 256) == 0


@pytest.mark.parametrize("pair", PAIRS, ids=prc.pair_id)
@pytest.mark.parametrize("axis", [1, 0])
@pytest.mark.parametrize("adjacent", [False, True], ids=["strided", "adjacent"])
def test_emu_pair_layouts(pair, axis, adjacent):
    """Every round shape of subgrid_round_cases.LAYOUTS; adjacent lines with an odd count."""
    prc.case_layouts(core(pair), pair, axis, adjacent, lines=5 if adjacent else 3)


@pytest.mark.parametrize("pair", PAIRS, ids=prc.pair_id)
def test_emu_pair_sizes_and_offsets(pair):
    prc.case_sizes(core(pair), pair)


@pytest.mark.parametrize("pair", PAIRS, ids=prc.pair_id)
@pytest.mark.parametrize("mode", ["grouped", "batched", "scattered"])
def test_emu_pair_entry_points(pair, mode):
    prc.case_entry_points(core(pair), pair, mode)


@pytest.mark.parametrize("pair", PAIRS, ids=prc.pair_id)
def test_emu_pair_more_rounds_than_one_launch(pair):
    prc.case_many_rounds(core(pair), pair)


@pytest.mark.parametrize("pair", PAIRS, ids=prc.pair_id)
@pytest.mark.parametrize("cap", [1, 3])
def test_emu_pair_capped_grid(pair, cap):
    prc.case_capped_grid(core(pair), pair, cap)


@pytest.mark.parametrize("pair", TWO_GROUP_PAIRS, ids=prc.pair_id)
def test_emu_pair_direct_stores_bitwise(pair):
    """sg_variant 5 (direct stores) gives the bits of the TMA-staged run."""
    prc.case_variant_bitwise(core(pair), pair, 5)


@pytest.mark.parametrize("pair", prc.SKIP_PAIRS, ids=prc.pair_id)
def test_emu_pair_skip_path_bitwise(pair):
    """sg_variant 25 (empty slots transform zeros) gives the bits of the default."""
    prc.case_variant_bitwise(core(pair), pair, prc.rc.LEGACY_VARIANT)


@pytest.mark.parametrize("pair", PAIRS, ids=prc.pair_id)
@pytest.mark.parametrize("axis", [1, 0])
def test_emu_pair_split_capped(pair, axis):
    """K4T / K3T with the grid capped at 2 CTAs, in both lines-per-CTA forms."""
    prc.case_split_capped(core(pair), pair, axis, "add" if axis else "store")


@pytest.mark.parametrize("pair", PAIRS, ids=prc.pair_id)
def test_emu_pair_extended_precision(pair):
    """sum_finish_axis against the longdouble chain (see tests/test_gpu_subgrid_pairs.py for
    the bound)."""
    c = core(pair)
    ratio = prc.spot_check_sum_finish(c, [0, 1, 2, 6, 7], prc.FORMS[pair][4] or c.xM_size - 3,
                                      seed=pair[1])
    print(f"{pair}: extended-precision ratio {ratio:.3f}")
    assert ratio <= prc.SPOT_BOUND, ratio
