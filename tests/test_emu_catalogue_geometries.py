"""
The fused forward kernels at the catalogue's (m, xM) pairs outside xM / m in {2, 4}, on the
host-emulated kernels: (128, 1024) with eight transforms per round, (256, 256) with one, and
the mixed-radix pairs (128, 384), (160, 320), (192, 384), (224, 448).  ``sum_finish_axis``
along both axes and every entry point against the oracle's extract_from_facet ->
add_to_subgrid -> finish_subgrid, then SwiftlyForward against the oracle's serial driver.
"""

import numpy
import pytest

from oracle.swiftly_oracle import OracleCore
from ska_sdp_distributed_fourier_transform_b200.swift_configs import (
    _BASELINE,
    FUSED_FORWARD_PAIRS,
    SWIFT_CONFIGS,
    fused_forward,
)
from tests import catalogue_cases as cc
from tests import subgrid_round_cases as rc
from tests.emu_support import emu_core_class

PAIRS = sorted(cc.SMALL)
_cfgs = {}


def config(pair):
    if pair not in _cfgs:
        _cfgs[pair] = cc.make_config(emu_core_class(), cc.SMALL[pair])
    return _cfgs[pair]


def oracle_of(cfg):
    return OracleCore(cfg.core.W, cfg.core.N, cfg.core.xM_size, cfg.core.yN_size)


def test_fused_forward_for_every_catalogue_entry():
    assert len(SWIFT_CONFIGS) >= 244
    for name, params in list(SWIFT_CONFIGS.items()) + list(_BASELINE.items()):
        assert fused_forward(params), name


def test_fused_forward_pairs_match_the_library():
    """``swift_configs.FUSED_FORWARD_PAIRS`` is the list of pairs the C library instantiates
    (SW_SG_PAIRS in dispatch_subgrid_axis.cu), in full, and the library reports a kernel for
    each of them."""
    import os
    import re

    src = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                       "ska_sdp_distributed_fourier_transform_b200", "csrc",
                       "dispatch_subgrid_axis.cu")
    with open(src) as f:
        text = f.read()
    macro = re.search(r"#define SW_SG_PAIRS\(X\)((?:.*\\\n)*.*\n)", text).group(1)
    c_pairs = {(int(a), int(b)) for a, b in re.findall(r"X\((\d+),\s*(\d+)\)", macro)}
    assert c_pairs == set(FUSED_FORWARD_PAIRS)
    core_cls = emu_core_class()
    for m, xM in sorted(c_pairs):
        # N = 2 xM, yN = 2 m passes check_params for every pair
        core = core_cls(13.5625, 2 * xM, xM, 2 * m)
        assert core._lib.swiftly_b200_sum_finish_axis_supported(core._plan) == xM // m, (m, xM)


def test_every_catalogue_pair_has_a_fused_kernel():
    core_cls = emu_core_class()
    pairs = {}
    for params in SWIFT_CONFIGS.values():
        m = params["xM_size"] * params["yN_size"] // params["N"]
        pairs.setdefault((m, params["xM_size"]), params)
    for (m, xM), p in sorted(pairs.items()):
        # the smallest plan with this (m, xM): N = 2 xM, yN = 2 m
        core = core_cls(p["W"], 2 * xM, xM, 2 * m)
        assert core.xM_yN_size == m
        assert core._lib.swiftly_b200_sum_finish_axis_supported(core._plan) == max(1, xM // m), (m, xM)
        assert core.fused_forward_supported()


@pytest.mark.parametrize("pair", PAIRS, ids=cc.pair_id)
@pytest.mark.parametrize("axis", [1, 0])
def test_emu_catalogue_sum_finish_layouts(pair, axis):
    """Every round shape (one source, clashing windows, disjoint windows, 3 + 2, tiled),
    prepared facet rows along axis 1, contribution strips along axis 0."""
    cfg = config(pair)
    for layout in sorted(rc.LAYOUTS):
        rc.check_single(cfg.core, oracle_of(cfg), layout, axis=axis, contrib_sized=axis == 0,
                        variant=0, rtol=1e-12)


@pytest.mark.parametrize("pair", PAIRS, ids=cc.pair_id)
def test_emu_catalogue_sum_finish_offsets_masks_sizes(pair):
    """Both source kinds along both axes, masks, odd and even subgrid sizes, subgrid offsets
    below zero and at or above N."""
    cfg = config(pair)
    step, xM, N = cfg.core.subgrid_off_step, cfg.core.xM_size, cfg.core.N
    cases = [
        (1, False, [0, 1, 3], -5 * step, xM - 1, True),
        (1, True, [0, 2], N + 3 * step, xM // 2, False),
        (0, False, [1, 2, -1], N - step, xM // 2 + 1, True),
        (0, True, [0, 1, 2, 3], -N - 2 * step, xM, False),
    ]
    for i, (axis, contrib, steps, sg_off, sz, masked) in enumerate(cases):
        cc.sum_finish_vs_oracle(cfg, axis, contrib, steps, sg_off, sz, masked, seed=10 + i)


@pytest.mark.parametrize("pair", PAIRS, ids=cc.pair_id)
@pytest.mark.parametrize("mode", ["grouped", "batched", "scattered"])
def test_emu_catalogue_entry_points(pair, mode):
    cfg = config(pair)
    rc.check_grouped(cfg.core, oracle_of(cfg), 0, mode, rtol=1e-12)
    rc.check_grouped(cfg.core, oracle_of(cfg), 0, mode, rtol=1e-12, axis=0, seed=3)


@pytest.mark.parametrize("pair", PAIRS, ids=cc.pair_id)
def test_emu_catalogue_more_sources_than_one_launch(pair):
    """One job with more rounds than one launch carries: later launches add their finished
    lines to the output.  A launch carries 64 source slots, 64 // CONC rounds.  All sources sit
    at the same facet offset, so every window clashes with every other one and each source takes
    a round of its own: 64 // CONC + 3 sources need two launches at every CONC."""
    cfg = config(pair)
    conc = max(1, cfg.core.xM_size // cfg.core.xM_yN_size)
    assert cfg.core._lib.swiftly_b200_sum_finish_axis_supported(cfg.core._plan) == conc
    n_src = 64 // conc + 3
    steps = [0] * n_src
    cc.sum_finish_vs_oracle(cfg, 1, True, steps, 2 * cfg.core.subgrid_off_step,
                            cfg.core.xM_size - 5, True, seed=21, lines=3)


@pytest.mark.parametrize("pair", PAIRS, ids=cc.pair_id)
def test_emu_catalogue_many_lines_per_cta(pair):
    """More lines than CTAs (the emulated grid is capped at 3 CTAs): every CTA walks several
    lines, so an accumulator left uncleared between lines would show."""
    import ctypes

    cfg = config(pair)
    lib = cfg.core._lib
    lib.swiftly_b200_debug_max_blocks.argtypes = [ctypes.c_void_p, ctypes.c_int]
    lib.swiftly_b200_debug_max_blocks(cfg.core._plan, 3)
    try:
        layouts = ["8_tiled", "1", None, "5_three_plus_two"]
        rc.check_grouped(cfg.core, oracle_of(cfg), 0, "grouped", lines=11, layouts=layouts,
                         seed=9, rtol=1e-12)
    finally:
        lib.swiftly_b200_debug_max_blocks(cfg.core._plan, 0)


@pytest.mark.parametrize("pair", PAIRS, ids=cc.pair_id)
def test_emu_catalogue_swiftly_forward(pair):
    """SwiftlyForward takes the fused path and matches the oracle's serial driver."""
    cc.forward_vs_oracle(config(pair), n_facets=4, n_subgrids=4, seed=pair[1])
