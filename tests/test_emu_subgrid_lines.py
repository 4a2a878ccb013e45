"""
The subgrid-side primitives and the window copies on the host-emulated kernels at every m and xM
length plan of the library (tests/subgrid_line_cases.py), each at a small plan of its pair,
against the oracle and against an extended-precision DFT; every case asserts the launch it was
written for.  Also: the grid capped at 1 and 3 CTAs, host and device staging into output views,
the window copies at cfg4 and the ska_sdp_func-shaped adapter at every catalogue family.
"""

import os
import re

import pytest

from oracle.swiftly_oracle import OracleCore
from ska_sdp_distributed_fourier_transform_b200 import _lib, sdp_func_compat
from tests import length_cases as lc
from tests import subgrid_line_cases as slc
from tests.emu_support import emu_core_class

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "ska_sdp_distributed_fourier_transform_b200", "csrc")

M_PLANS = slc.m_plans()
XM_PLANS = slc.xm_plans()
FAMILIES = slc.family_geometries()
_cores = {}


def pair(geometry):
    """(core, oracle) of a geometry (W, N, xM, yN), one at a time."""
    if geometry not in _cores:
        _cores.clear()
        _cores[geometry] = (emu_core_class()(*geometry), OracleCore(*geometry))
    return _cores[geometry]


def test_plans_are_pinned():
    """The catalogue and the library pairs need exactly the pinned m and xM plans, and every
    plan has a pinned launch form: a new length, or a change of the restated dispatch, has to
    be added to the cases here and in the GPU tests."""
    direct, split_f = slc.pinned_kinds(M_PLANS)
    assert direct == set(slc.PINNED_M_DIRECT), "m plans (direct)"
    assert split_f == set(slc.PINNED_M_SPLIT_F), "m plans (split-F)"
    direct, split_f = slc.pinned_kinds(XM_PLANS)
    assert direct == set(slc.PINNED_XM_DIRECT), "xM plans (direct)"
    assert split_f == set(slc.PINNED_XM_SPLIT_F), "xM plans (split-F)"
    for plans, which in ((M_PLANS, 0), (XM_PLANS, 1)):
        for plan_id, (n, plan, pair_, gpu, emu, _) in plans.items():
            assert pair_[which] == n, plan_id
            kind, v = slc.FORMS[n]
            assert (kind, v) == ((slc.LINE, min(16, max(1, 256 // (n // 16))))
                                 if plan[0] == "direct" else (slc.SPLIT_F, plan[2])), plan_id
            for W, N, xM, yN in (gpu, emu):
                assert ((xM * yN // N, xM)[which]) == n, (plan_id, gpu, emu)
    assert set(slc.FORMS) == {v[0] for v in M_PLANS.values()} | {v[0] for v in XM_PLANS.values()}


def test_split_f_cases_cover_the_plans():
    """Every pinned M of a subgrid-side split-F plan has a case in the library's
    SW_SPLIT_F_CASES; the failure names the plan."""
    with open(os.path.join(CSRC, "dispatch.cuh")) as f:
        text = f.read()
    body = re.search(r"#define SW_SPLIT_F_CASES\(.*\)((?:.*\\\n)*.*\n)", text).group(1)
    cases = {int(c) for c in re.findall(r"case (\d+): return launch_split_f<\1,", body)}
    for plan_id, (n, plan, *_) in list(M_PLANS.items()) + list(XM_PLANS.items()):
        if plan[0] == "splitf":
            assert plan[1] in cases, f"{plan_id}: no SW_SPLIT_F_CASES case for M = {plan[1]}"
            assert lc.split_f_plan(n) == plan[1:], plan_id


@pytest.mark.parametrize("plan_id", list(M_PLANS))
def test_emu_m_plan(plan_id):
    n, _, _, _, emu, _ = M_PLANS[plan_id]
    core, oracle = pair(emu)
    assert core.xM_yN_size == n
    # two subgrid_to_facets launches (67 facets) up to m = 256; the 2-D pass up to m = 512
    slc.m_plan_vs_oracle(core, oracle, seed=n, n_facets=67 if n <= 256 else 3, max_2d=512)


@pytest.mark.parametrize("plan_id", list(XM_PLANS))
def test_emu_xm_plan(plan_id):
    n, _, _, _, emu, xa = XM_PLANS[plan_id]
    core, oracle = pair(emu)
    assert core.xM_size == n
    slc.xm_plan_vs_oracle(core, oracle, xa, seed=n, max_2d=1024)


@pytest.mark.parametrize("plan_id", list(M_PLANS) + list(XM_PLANS))
def test_emu_extended_precision(plan_id):
    """The m-point (add_to_subgrid, extract_from_subgrid) or xM-point (finish_subgrid,
    prepare_subgrid) transform at the sub-transform boundaries, the centre and random bins
    against a DFT in extended precision: error <= 1.5 eps log2(n) of the line's RMS."""
    if plan_id in M_PLANS:
        core, _ = pair(M_PLANS[plan_id][4])
        got = slc.spot_check_m(core, seed=1, n_lines=1)
    else:
        core, _ = pair(XM_PLANS[plan_id][4])
        got = slc.spot_check_xm(core, seed=1, n_lines=1)
    print(f"\n{plan_id}: extended-precision spot check {got:.3f} eps log2(n)")
    assert got <= slc.SPOT_BOUND, got


CAPPED = ["m128-direct-128", "m192-splitf-64x3", "xM256-direct-256", "xM448-splitf-64x7"]


@pytest.mark.parametrize("cap", [1, 3])
@pytest.mark.parametrize("plan_id", CAPPED)
def test_emu_capped_grid(plan_id, cap):
    """The grid capped at 1 and 3 CTAs: a few dozen lines walk the grid-stride loop of
    LineKernel / SplitFKernel and WindowCopyKernel."""
    plans = M_PLANS if plan_id in M_PLANS else XM_PLANS
    core, oracle = pair(plans[plan_id][4])
    slc.capped_vs_oracle(core, oracle, "m" if plans is M_PLANS else "xM", cap, seed=cap)


@pytest.mark.parametrize("host", [True, False], ids=["host", "device"])
@pytest.mark.parametrize("plan_id", ["m32-direct-32", "m192-splitf-64x3"])
def test_emu_staging(plan_id, host):
    core, oracle = pair(M_PLANS[plan_id][4])
    slc.staging_vs_oracle(core, oracle, host, seed=5)


def test_emu_window_copies_cfg4():
    core, oracle = pair(slc.geometry_entry(slc.CFG4))
    slc.window_copies_vs_oracle(core, oracle, seed=7)


# (1024, 4096): the adapter's xM x xM passes take half a minute on the emulator; the GPU tests
# run that family
ADAPTER_FAMILIES = [f for f in sorted(FAMILIES) if f[1] <= 2048]


@pytest.mark.parametrize("family", ADAPTER_FAMILIES, ids=lambda p: f"{p[0]}_{p[1]}")
def test_emu_sdp_func_adapter(family):
    (geometry, yB, xA) = FAMILIES[family]["emu"]
    core, oracle = pair(geometry)
    W, N, xM, yN = geometry
    real_load = _lib.load
    _lib.load = lambda path=None: core._lib  # pylint: disable=protected-access
    try:
        sw = sdp_func_compat.Swiftly(N, yN, xM, W)
    finally:
        _lib.load = real_load
    slc.sdp_func_adapter_vs_oracle(sw, oracle, yB, xA)
