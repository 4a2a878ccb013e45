"""
The facet-side line transforms (prepare_facet, finish_facet, extract_columns, fold_column) on an
H100 at every facet length plan of the parameter catalogue (``tests/length_cases.py``), each at
its smallest catalogue entry, against the oracle and against an extended-precision DFT; and the
cfg4 backward hot path (fold_column at yN = 16384) against the oracle.

Every test prints its worst errors (run pytest with -s to see them).
"""

import ctypes

import pytest
import torch

from oracle.swiftly_oracle import OracleCore
from ska_sdp_distributed_fourier_transform_b200.core import SwiftlyCoreB200
from ska_sdp_distributed_fourier_transform_b200.swift_configs import SWIFT_CONFIGS
from tests import length_cases as lc

pytestmark = pytest.mark.gpu

PLANS = lc.yn_plans()
LINE_PLANS = sorted(lc.line_plans(), key=list(PLANS).index)
TWO_PASS_PLANS = sorted(lc.two_pass_plans(), key=list(PLANS).index)
_pairs = {}


def pair(geometry):
    """(core, oracle) of a geometry (W, N, xM, yN); one at a time, so that the scratch and
    tables of the previous plan are released before the next one is built."""
    if geometry not in _pairs:
        _pairs.clear()
        torch.cuda.empty_cache()
        _pairs[geometry] = (SwiftlyCoreB200(*geometry, device=0), OracleCore(*geometry))
    return _pairs[geometry]


def plan_pair(plan_id):
    _, (_, W, N, xM, yN) = PLANS[plan_id]
    return pair((W, N, xM, yN))


def _fmt(errs):
    return ", ".join(f"{k} {v:.2e}" for k, v in errs.items())


@pytest.mark.parametrize("plan_id", LINE_PLANS)
def test_gpu_line_plan(plan_id):
    core, oracle = plan_pair(plan_id)
    worst = lc.line_plan_vs_oracle(core, oracle, seed=len(plan_id))
    print(f"\n{plan_id} ({PLANS[plan_id][1][0]}): max rel err vs oracle: {_fmt(worst)}")


@pytest.mark.parametrize("plan_id", TWO_PASS_PLANS)
def test_gpu_two_pass(plan_id):
    core, oracle = plan_pair(plan_id)
    worst = lc.two_pass_vs_oracle(core, oracle, seed=3)
    print(f"\n{plan_id} ({PLANS[plan_id][1][0]}): two-pass prepare_facet max rel err {worst:.2e}")


@pytest.mark.parametrize("plan_id", LINE_PLANS)
def test_gpu_extended_precision(plan_id):
    """prepare_facet and finish_facet at the sub-transform boundaries, the centre and random bins
    against a DFT in extended precision: error <= 1.5 eps log2(yN) of the line's RMS
    (eps = 2.2e-16).  On an H100 80GB HBM3 (700 W) the direct power-of-two plans reach
    0.15 .. 0.59, the split-F plans 0.16 .. 0.51."""
    plan = PLANS[plan_id][0]
    core, _ = plan_pair(plan_id)
    prep = lc.spot_check_prepare_facet(core, plan, seed=1)
    fin = lc.spot_check_finish_facet(core, plan, seed=2)
    print(f"\n{plan_id}: extended-precision spot check, in eps log2(yN): "
          f"prepare_facet {prep:.3f}, finish_facet {fin:.3f}")
    assert max(prep, fin) <= lc.SPOT_BOUND, (prep, fin)


CFG4 = "64k[1]-n16k-4k"  # yN = 16384, m = 1024, facets of 8192


def test_gpu_cfg4_fold_and_masked_finish():
    """The backward hot path at cfg4: fold_column of three column accumulators (3 x 1024 lines,
    SplitLineKernel<8192> on a grid-stride loop) into facet accumulators of the benchmark's size,
    one masked; and masked finish_facet over more lines than the persistent grid."""
    p = SWIFT_CONFIGS[CFG4]
    core, oracle = pair((p["W"], p["N"], p["xM_size"], p["yN_size"]))
    assert core.xM_yN_size == 1024
    N, yB = core.N, p["yB_size"]
    fs_step, sg_step = core.facet_off_step, core.subgrid_off_step
    fold = lc.fold_column_vs_oracle(core, oracle, [yB, yB - 1, yB // 2 + 1],
                                    [0, -3 * fs_step, N + 5 * fs_step], -7 * sg_step,
                                    masked=[1], seed=1)
    fin = max(lc.finish_facet_vs_oracle(core, oracle, 1, 301, yB, 2 * fs_step, True, seed=2),
              lc.finish_facet_vs_oracle(core, oracle, 0, 300, yB - 1, -fs_step, True, seed=3))
    print(f"\ncfg4: fold_column max rel err {fold:.2e}, masked finish_facet {fin:.2e}")


MANY = "splitf-256x3"  # 1536[1]-n768-256: m = 128, so three facets fold 384 lines


@pytest.mark.parametrize("max_blocks", [0, 1, 3])
def test_gpu_many_lines_per_cta(max_blocks):
    """More lines than the persistent grid (296 CTAs) of SplitFKernel and SplitLineKernel, and
    the grid capped at 1 and 3 CTAs: every CTA walks many lines and reuses its scratch stash."""
    for plan_id in (MANY, "split-16384"):
        core, oracle = plan_pair(plan_id)
        yN, N = core.yN_size, core.N
        fs_step, sg_step = core.facet_off_step, core.subgrid_off_step
        lib = core._lib
        lib.swiftly_b200_debug_max_blocks.argtypes = [ctypes.c_void_p, ctypes.c_int]
        lib.swiftly_b200_debug_max_blocks(core._plan, max_blocks)
        try:
            errs = [
                lc.finish_facet_vs_oracle(core, oracle, 1, 301, yN - 1, -fs_step, True, seed=1),
                lc.finish_facet_vs_oracle(core, oracle, 0, 300, (yN * 11 // 16) | 1, N, False,
                                          seed=2),
                lc.prepare_facet_vs_oracle(core, oracle, 1, 299, yN - 1, 2 * fs_step, True,
                                           seed=3),
                lc.fold_column_vs_oracle(core, oracle, lc.fold_sizes(yN, 1 << 24),
                                         [0, -fs_step, N], 5 * sg_step, masked=[1], seed=4),
                lc.extract_columns_vs_oracle(core, oracle, [yN - 1, 300, 301], [N, 0, -fs_step],
                                             -3 * sg_step, False, seed=5),
            ]
        finally:
            lib.swiftly_b200_debug_max_blocks(core._plan, 0)
        print(f"\n{plan_id}, max_blocks {max_blocks}: max rel err {max(errs):.2e}")
