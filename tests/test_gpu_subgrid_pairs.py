"""
The fused subgrid kernels at every (m, xM) pair of the library on the GPU: the cases of
tests/pair_cases.py (``sum_finish_axis`` in every form of the pinned table, ``split_subgrid_axis``
in both lines-per-CTA forms, each asserting the form it ran) on cores at the smallest catalogue
entry of each of the 13 catalogue pairs and at the 7 library-only pairs; jobs with more line
pairs than the H100 has SMs; SwiftlyForward / SwiftlyBackward against the oracle and the round
trip at the power-of-two families whose smallest entry is not a benchmark geometry
((1024, 2048) and (1024, 4096) are cfg2 / cfg3 / cfg4, tests/test_gpu_api.py and
tests/test_gpu_subgrid_rounds.py); and the extended-precision spot check of ``sum_finish_axis``
at every catalogue pair.

Extended precision: worst ``|got - exact|`` over the line RMS, in units of
``EPS * (log2 m + log2 xM)``, bound 1.5 (pair_cases.SPOT_BOUND).  Observed with the test seeds:
emulated kernels (host build without fused multiply-adds) 0.14 .. 0.44 over the 20 pairs;
one H100 80GB HBM3 0.14 .. 0.27 over the 13 catalogue pairs.
"""

import pytest
import torch

from ska_sdp_distributed_fourier_transform_b200 import (
    SwiftlyBackward,
    SwiftlyCoreB200,
    SwiftlyForward,
    check_facet,
    make_facet,
    make_full_facet_cover,
    make_full_subgrid_cover,
)
from tests import catalogue_cases as cc
from tests import pair_cases as prc
from tests import split_cases as sc

pytestmark = pytest.mark.gpu

PAIRS = prc.ALL_PAIRS
CATALOGUE_PAIRS = sorted(prc.CATALOGUE)
TWO_GROUP_PAIRS = [p for p in PAIRS if prc.FORMS[p][0][0] == prc.TWO_GROUP]
# power-of-two families whose smallest entry is not a benchmark geometry
API_PAIRS = [(128, 256), (128, 512), (256, 512), (256, 1024), (512, 1024)]
_cores = {}


def core(pair):
    """One core at a time (the largest plans hold yN = 8192 tables and their transforms)."""
    if pair not in _cores:
        _cores.clear()
        torch.cuda.empty_cache()
        _cores[pair] = SwiftlyCoreB200(*prc.core_plan(pair), device=0)
    return _cores[pair]


def config(pair, half_facets=False):
    """The smallest catalogue entry of the pair; ``half_facets``: with yB = yN / 2.  (The
    oracle comparisons use yB = yN / 2.  At the entry's own yB / yN = 0.81 of 1k[1]-n512-256
    and 1k[1]-n256-512, SwiftlyForward / SwiftlyBackward differ from the oracle by 3e-11 / 6e-10
    of the largest sample, beyond the 1e-12 / 1e-11 bounds, while their kernels pass the cases
    above at 1e-12: the window's conditioning at that ratio (DESIGN.md section 6), which
    catalogue_cases.SMALL also notes for 16k[1]-n2k-1k.  The round trip runs at the entry
    itself.)"""
    W, N, yB, yN, xA, xM = cc.catalogue_plan(prc.CATALOGUE[pair][1])
    key = ("cfg", pair, half_facets)
    if key not in _cores:
        _cores.clear()
        torch.cuda.empty_cache()
        _cores[key] = cc.make_config(SwiftlyCoreB200,
                                     (W, N, yN // 2 if half_facets else yB, yN, xA, xM))
    return _cores[key]


@pytest.mark.parametrize("pair", PAIRS, ids=prc.pair_id)
def test_gpu_pair_forward_forms(pair):
    """Every layout on strided and adjacent lines along both axes, sizes around the TMA
    threshold with masks and far offsets, the three grouped entry points, a job cut over two
    launches and grids capped at 1 and 3 CTAs."""
    c = core(pair)
    worst = 0.0
    for axis in (1, 0):
        for adjacent in (False, True):
            worst = max(worst, prc.case_layouts(c, pair, axis, adjacent,
                                                lines=5 if adjacent else 3))
    worst = max(worst, prc.case_sizes(c, pair))
    for mode in ("grouped", "batched", "scattered"):
        worst = max(worst, prc.case_entry_points(c, pair, mode))
    worst = max(worst, prc.case_many_rounds(c, pair))
    for cap in (1, 3):
        worst = max(worst, prc.case_capped_grid(c, pair, cap))
    print(f"{pair}: sum_finish_axis worst error {worst:.2e} of the largest sample")


@pytest.mark.parametrize("pair", TWO_GROUP_PAIRS, ids=prc.pair_id)
def test_gpu_pair_variants_bitwise(pair):
    """Direct stores (sg_variant 5) and, where empty slots are skipped, the former round scheme
    (sg_variant 25) give the bits of the default."""
    c = core(pair)
    prc.case_variant_bitwise(c, pair, 5)
    if pair in prc.SKIP_PAIRS:
        prc.case_variant_bitwise(c, pair, prc.rc.LEGACY_VARIANT)


@pytest.mark.parametrize("pair", PAIRS, ids=prc.pair_id)
def test_gpu_pair_split(pair):
    """K4T / K3T with the grid capped at 2 CTAs, in both lines-per-CTA forms."""
    c = core(pair)
    worst = max(prc.case_split_capped(c, pair, 0, "store"),
                prc.case_split_capped(c, pair, 1, "add"))
    print(f"{pair}: split worst error {worst:.2e}")


@pytest.mark.parametrize("pair", [(256, 1024), (512, 1024)], ids=prc.pair_id)
def test_gpu_pair_more_line_pairs_than_sms(pair):
    """An uncapped grouped job with 270 line pairs (132 SMs): persistent CTAs walk two or
    three line pairs, at a TMA size."""
    c = core(pair)
    sz = prc.FORMS[pair][4]
    groups = [prc.rc.LAYOUTS["5_three_plus_two"], prc.rc.LAYOUTS["3_disjoint"]]
    prc.sum_finish_job(c, groups, sz, 1, mode="grouped", lines=270, seed=21,
                       what=f"{pair} 270 line pairs")
    prc.expect_form(c, prc.TWO_GROUP, 2, prc.TMA, grid=132, what=f"{pair} 270 line pairs")


@pytest.mark.parametrize("pair", CATALOGUE_PAIRS, ids=prc.pair_id)
def test_gpu_pair_extended_precision(pair):
    c = core(pair)
    ratio = prc.spot_check_sum_finish(c, [0, 1, 2, 6, 7], prc.FORMS[pair][4] or c.xM_size - 3,
                                      seed=pair[1])
    print(f"{pair}: extended-precision ratio {ratio:.3f}")
    assert ratio <= prc.SPOT_BOUND, ratio


@pytest.mark.parametrize("pair", API_PAIRS, ids=prc.pair_id)
def test_gpu_pair_forward_vs_oracle(pair):
    cc.forward_vs_oracle(config(pair, True), n_facets=3, n_subgrids=3, seed=pair[1])


@pytest.mark.parametrize("pair", API_PAIRS, ids=prc.pair_id)
def test_gpu_pair_backward_vs_oracle(pair):
    cfg = config(pair, True)
    facet_cfgs, sgs, data = sc.backward_inputs(cfg, True, 3, seed=pair[1], n_facets=2)
    assert SwiftlyBackward(cfg, facet_cfgs)._split
    err = sc.backward_vs_oracle(cfg, facet_cfgs, sgs, data)
    print(f"{pair}: backward worst error {err:.2e}")


def _round_trip(cfg, fused):
    N = cfg.image_size
    sources = [(1, 1, 0)]
    facet_cfgs = make_full_facet_cover(cfg)
    fwd = SwiftlyForward(cfg, [(fc, make_facet(N, fc, sources)) for fc in facet_cfgs],
                         lru_forward=1)
    assert fwd._fused
    fwd._fused = fused
    bwd = SwiftlyBackward(cfg, facet_cfgs, lru_backward=1)
    for sg in make_full_subgrid_cover(cfg):
        bwd.add_new_subgrid_task(sg, fwd.get_subgrid_task(sg))
    return max(check_facet(N, fc, task.result(), sources)
               for fc, task in zip(facet_cfgs, bwd.finish()))


@pytest.mark.parametrize("pair", API_PAIRS, ids=prc.pair_id)
def test_gpu_pair_round_trip(pair):
    """Forward then backward over the full covers with a unit source: facet RMSE below 3e-10,
    or no worse than the primitive forward path (tests/test_gpu_catalogue.py)."""
    cfg = config(pair)
    err = _round_trip(cfg, True)
    print(f"{pair}: round-trip facet RMSE {err:.3e}")
    if err >= 3e-10:
        prim = _round_trip(cfg, False)
        assert err <= 1.1 * prim, (err, prim)
