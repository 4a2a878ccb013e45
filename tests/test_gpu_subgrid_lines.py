"""
The subgrid-side primitives and the window copies on an H100 at every m and xM length plan of
the library (tests/subgrid_line_cases.py), each at the smallest catalogue entry that uses the
length, against the oracle and against an extended-precision DFT; every case asserts the launch
it was written for.  Also: the grid capped at 1 and 3 CTAs, host and device staging into output
views, the window copies at cfg4 and the ska_sdp_func-shaped adapter at every catalogue family.

Every test prints its worst errors (run pytest with -s to see them).
"""

import pytest
import torch

from oracle.swiftly_oracle import OracleCore
from ska_sdp_distributed_fourier_transform_b200.core import SwiftlyCoreB200
from ska_sdp_distributed_fourier_transform_b200.sdp_func_compat import Swiftly
from tests import subgrid_line_cases as slc

pytestmark = pytest.mark.gpu

M_PLANS = slc.m_plans()
XM_PLANS = slc.xm_plans()
FAMILIES = slc.family_geometries()
_pairs = {}


def pair(geometry):
    """(core, oracle) of a geometry (W, N, xM, yN); one at a time."""
    if geometry not in _pairs:
        _pairs.clear()
        torch.cuda.empty_cache()
        _pairs[geometry] = (SwiftlyCoreB200(*geometry, device=0), OracleCore(*geometry))
    return _pairs[geometry]


def _fmt(errs):
    return ", ".join(f"{k} {v:.2e}" for k, v in errs.items())


@pytest.mark.parametrize("plan_id", list(M_PLANS))
def test_gpu_m_plan(plan_id):
    n, _, _, gpu, _, _ = M_PLANS[plan_id]
    core, oracle = pair(gpu)
    assert core.xM_yN_size == n
    # 67 facets (two subgrid_to_facets launches) while their accumulators stay below 1 GiB
    n_facets = 67 if 67 * n * core.yN_size * 16 <= 1 << 30 else 3
    worst = slc.m_plan_vs_oracle(core, oracle, seed=n, n_facets=n_facets, max_2d=2048)
    print(f"\n{plan_id} {gpu}: max rel err vs oracle: {_fmt(worst)}")


@pytest.mark.parametrize("plan_id", list(XM_PLANS))
def test_gpu_xm_plan(plan_id):
    n, _, _, gpu, _, xa = XM_PLANS[plan_id]
    core, oracle = pair(gpu)
    assert core.xM_size == n
    worst = slc.xm_plan_vs_oracle(core, oracle, xa, seed=n, max_2d=4096)
    print(f"\n{plan_id} {gpu}: max rel err vs oracle: {_fmt(worst)}")


@pytest.mark.parametrize("plan_id", list(M_PLANS) + list(XM_PLANS))
def test_gpu_extended_precision(plan_id):
    """The m-point (add_to_subgrid, extract_from_subgrid) or xM-point (finish_subgrid,
    prepare_subgrid) transform at the sub-transform boundaries, the centre and random bins
    against a DFT in extended precision: error <= 1.5 eps log2(n) of the line's RMS."""
    if plan_id in M_PLANS:
        core, _ = pair(M_PLANS[plan_id][3])
        got = slc.spot_check_m(core, seed=1)
    else:
        core, _ = pair(XM_PLANS[plan_id][3])
        got = slc.spot_check_xm(core, seed=1)
    print(f"\n{plan_id}: extended-precision spot check {got:.3f} eps log2(n)")
    assert got <= slc.SPOT_BOUND, got


CAPPED = ["m128-direct-128", "m224-splitf-32x7", "xM256-direct-256", "xM384-splitf-128x3"]


@pytest.mark.parametrize("cap", [1, 3])
@pytest.mark.parametrize("plan_id", CAPPED)
def test_gpu_capped_grid(plan_id, cap):
    """The grid capped at 1 and 3 CTAs: a few dozen lines walk the grid-stride loop of
    LineKernel / SplitFKernel and WindowCopyKernel."""
    plans = M_PLANS if plan_id in M_PLANS else XM_PLANS
    core, oracle = pair(plans[plan_id][3])
    err = slc.capped_vs_oracle(core, oracle, "m" if plans is M_PLANS else "xM", cap, seed=cap)
    print(f"\n{plan_id}, grid capped at {cap}: max rel err {err:.2e}")


@pytest.mark.parametrize("host", [True, False], ids=["host", "device"])
@pytest.mark.parametrize("plan_id", ["m128-direct-128", "m192-splitf-64x3"])
def test_gpu_staging(plan_id, host):
    core, oracle = pair(M_PLANS[plan_id][3])
    slc.staging_vs_oracle(core, oracle, host, seed=5)


def test_gpu_window_copies_cfg4():
    core, oracle = pair(slc.geometry_entry(slc.CFG4))
    assert (core.xM_yN_size, core.yN_size) == (1024, 16384)
    slc.window_copies_vs_oracle(core, oracle, seed=7)


@pytest.mark.parametrize("family", sorted(FAMILIES), ids=lambda p: f"{p[0]}_{p[1]}")
def test_gpu_sdp_func_adapter(family):
    (geometry, yB, xA) = FAMILIES[family]["gpu"]
    W, N, xM, yN = geometry
    _pairs.clear()
    torch.cuda.empty_cache()
    slc.sdp_func_adapter_vs_oracle(Swiftly(N, yN, xM, W), OracleCore(*geometry), yB, xA)
