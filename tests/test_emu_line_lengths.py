"""
The facet-side line transforms (prepare_facet, finish_facet, extract_columns, fold_column) on the
host-emulated kernels at every facet length plan of the parameter catalogue
(``tests/length_cases.py``), against the oracle and against an extended-precision DFT.

The plans run at the catalogue's ``W`` and ``yN`` with a small subgrid (``xM = 32``,
``N = 2 yN``, so ``m = 16``): the line kernels depend on ``yN`` only, and few accumulator lines
keep the emulated K2 / fold launches short at ``yN = 65536``.
"""

import ctypes
import os
import re

import pytest

from oracle.swiftly_oracle import OracleCore
from tests import length_cases as lc
from tests.emu_support import emu_core_class

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "ska_sdp_distributed_fourier_transform_b200", "csrc")

PLANS = lc.yn_plans()
LINE_PLANS = sorted(lc.line_plans(), key=list(PLANS).index)
TWO_PASS_PLANS = sorted(lc.two_pass_plans(), key=list(PLANS).index)
_cores = {}


def pair(geometry):
    """(core, oracle) of a geometry (W, N, xM, yN), kept for the module: the PSWF windows at
    yN = 65536 take seconds to compute."""
    if geometry not in _cores:
        _cores[geometry] = (emu_core_class()(*geometry), OracleCore(*geometry))
    return _cores[geometry]


def small_pair(plan_id):
    _, (_, W, _, _, yN) = PLANS[plan_id]
    return pair((W, 2 * yN, 32, yN))


def test_plans_are_pinned():
    """The catalogue needs exactly the pinned plans: a new catalogue length, or a change of the
    restated dispatch, has to be added to the cases here and in the GPU tests."""
    kinds = {}
    for plan, _ in PLANS.values():
        kinds.setdefault(plan[0], set()).add(plan[1:])
    assert kinds.pop("splitf") == set(lc.PINNED_SPLIT_F)
    assert kinds.pop("direct") == {(n,) for n in lc.PINNED_DIRECT}
    assert kinds.pop("split") == {(16384,)}
    assert kinds.pop("twopass") == {(n,) for n in lc.PINNED_TWO_PASS}
    assert not kinds
    # the powers of two above 16384 are split-F lines (and two-pass along axis 0)
    assert lc.line_kernel(32768) == ("splitf", 8192, 4)
    assert lc.line_kernel(65536) == ("splitf", 8192, 8)
    # every representative is a catalogue entry with that yN
    for plan, (name, W, N, xM, yN) in PLANS.values():
        assert (plan[1] if plan[0] != "splitf" else plan[1] * plan[2]) == yN, (plan, name)


def test_split_f_cases_cover_the_plans():
    """Every pinned M has a case in the library's SW_SPLIT_F_CASES, and every pinned F fits
    SW_MAX_SPLIT_F."""
    with open(os.path.join(CSRC, "dispatch.cuh")) as f:
        text = f.read()
    body = re.search(r"#define SW_SPLIT_F_CASES\(.*\)((?:.*\\\n)*.*\n)", text).group(1)
    cases = {int(c) for c in re.findall(r"case (\d+): return launch_split_f<\1,", body)}
    assert {M for M, _ in lc.PINNED_SPLIT_F} <= cases
    with open(os.path.join(CSRC, "kernels.cuh")) as f:
        max_f = int(re.search(r"#define SW_MAX_SPLIT_F (\d+)", f.read()).group(1))
    assert max(F for _, F in lc.PINNED_SPLIT_F) <= max_f == lc.MAX_SPLIT_F
    for M, F in lc.PINNED_SPLIT_F:
        assert lc.split_f_plan(M * F) == (M, F)


@pytest.mark.parametrize("plan_id", LINE_PLANS)
def test_emu_line_plan(plan_id):
    core, oracle = small_pair(plan_id)
    lc.line_plan_vs_oracle(core, oracle, seed=len(plan_id), fold_budget=1 << 20)


@pytest.mark.parametrize("plan_id", TWO_PASS_PLANS)
def test_emu_two_pass(plan_id):
    core, oracle = small_pair(plan_id)
    lc.two_pass_vs_oracle(core, oracle, seed=3)


@pytest.mark.parametrize("plan_id", LINE_PLANS)
def test_emu_extended_precision(plan_id):
    """prepare_facet and finish_facet at the sub-transform boundaries, the centre and random bins
    against a DFT in extended precision: error <= 1.5 eps log2(yN) of the line's RMS
    (eps = 2.2e-16).  The emulated kernels reach 0.20 .. 0.65 at the direct power-of-two plans
    and 0.19 .. 0.76 at the split-F plans (lc.SPOT_BOUND has the H100 numbers)."""
    plan = PLANS[plan_id][0]
    core, _ = small_pair(plan_id)
    prep = lc.spot_check_prepare_facet(core, plan, seed=1, n_lines=1)
    fin = lc.spot_check_finish_facet(core, plan, seed=2, n_lines=1)
    assert max(prep, fin) <= lc.SPOT_BOUND, (prep, fin)


MANY = "splitf-256x3"  # 1536[1]-n768-256: m = 128, so three facets fold 384 lines


@pytest.mark.parametrize("max_blocks", [0, 1, 3])
def test_emu_many_lines_per_cta(max_blocks):
    """More lines than the persistent grid of SplitFKernel (296 CTAs), and the grid capped at 1
    and 3 CTAs: every CTA walks many lines and reuses its scratch stash.  The same capped grid
    for SplitLineKernel at 16384."""
    _, (_, W, N, xM, yN) = PLANS[MANY]
    core, oracle = pair((W, N, xM, yN))
    assert core.xM_yN_size * 3 > 296
    big, _ = small_pair("split-16384")
    lib = core._lib
    lib.swiftly_b200_debug_max_blocks.argtypes = [ctypes.c_void_p, ctypes.c_int]
    for c in (core, big):
        lib.swiftly_b200_debug_max_blocks(c._plan, max_blocks)
    try:
        fs_step, sg_step = core.facet_off_step, core.subgrid_off_step
        lc.finish_facet_vs_oracle(core, oracle, 1, 301, yN - 1, -fs_step, True, seed=1)
        lc.finish_facet_vs_oracle(core, oracle, 0, 300, (yN * 11 // 16) | 1, N, False, seed=2)
        lc.prepare_facet_vs_oracle(core, oracle, 1, 299, yN - 1, 2 * fs_step, True, seed=3)
        lc.fold_column_vs_oracle(core, oracle, lc.fold_sizes(yN, 1 << 24), [0, -fs_step, N],
                                 5 * sg_step, masked=[1], seed=4)
        lc.extract_columns_vs_oracle(core, oracle, [yN - 1, 300, 301], [N, 0, -fs_step],
                                     -3 * sg_step, False, seed=5)
        if max_blocks:
            big_oracle = small_pair("split-16384")[1]
            lc.finish_facet_vs_oracle(big, big_oracle, 1, 7, 16383, 0, True, seed=6)
            lc.prepare_facet_vs_oracle(big, big_oracle, 1, 5, 16383, big.facet_off_step,
                                       False, seed=7)
    finally:
        for c in (core, big):
            lib.swiftly_b200_debug_max_blocks(c._plan, 0)
