"""
The backward transform as the adjoint of the forward transform (``tests/adjoint_cases.py``) on an
H100: every kernel pair at the catalogue geometries, and the drivers end to end up to cfg4's
central 5 x 5 facet block over all 32 x 32 subgrids.  The forms covered are those of the table in
``tests/test_emu_adjoint.py``, here at the sizes the catalogue runs; every test prints its worst
residual (run pytest with -s to see them).
"""

import gc
import time

import pytest
import torch

from ska_sdp_distributed_fourier_transform_b200 import (
    SwiftlyConfig,
    make_full_facet_cover,
    make_full_subgrid_cover,
)
from ska_sdp_distributed_fourier_transform_b200.api import device_tier_bytes
from ska_sdp_distributed_fourier_transform_b200.core import SwiftlyCoreB200
from ska_sdp_distributed_fourier_transform_b200.swift_configs import SWIFT_CONFIGS
from tests import adjoint_cases as ac
from tests import catalogue_cases as cc
from tests import host_tier_cases as hc
from tests import k2_cases as kc
from tests import length_cases as lc
from tests import pair_cases as prc
from tests import subgrid_line_cases as slc

pytestmark = pytest.mark.gpu

_cores = {}


def core_of(geometry):
    """Core of a geometry (W, N, xM, yN); one at a time, so that the scratch and tables of the
    previous plan are released before the next one is built."""
    if geometry not in _cores:
        _cores.clear()
        torch.cuda.empty_cache()
        _cores[geometry] = SwiftlyCoreB200(*geometry, device=0)
    return _cores[geometry]


def _units(res, n):
    return res / (ac.EPS * (n.bit_length() - 1))


def _report(what, res, n):
    print(f"\n{what}: residual {res:.2e} ({_units(res, n):.4f} eps log2 n)")
    assert res <= ac.pair_bound(n), (what, res)


# ---------------------------------------------------------------------- K1 <-> finish_facet
PLANS = lc.yn_plans()


@pytest.mark.parametrize("plan_id", list(PLANS))
def test_gpu_facet_plan(plan_id):
    plan, (_, W, N, xM, yN) = PLANS[plan_id]
    core = core_of((W, N, xM, yN))
    _report(plan_id, ac.facet_plan_cases(core, plan, seed=len(plan_id)), yN)


@pytest.mark.parametrize("plan_id", ["direct-512", "splitf-256x5", "split-16384",
                                     "splitf-8192x8"])
def test_gpu_real_facets(plan_id):
    _, (_, W, N, xM, yN) = PLANS[plan_id]
    core = core_of((W, N, xM, yN))
    _report(f"real {plan_id}", ac.real_facet_cases(core, seed=yN), yN)


# ---------------------------------------------------------------------- K2 <-> fold_column
ROWS = kc.catalogue_rows()
# every (yN, yB) staged by the TMA kernels, one row of every generic kernel kind and the
# yN = 16384 rows that miss the staging buffer; sorted by geometry so plans are built once
GPU_ROWS = sorted(
    list(kc.PINNED_TMA) + [(256, 208), (512, 416), (768, 528), (16384, 11264)],
    key=lambda r: (r[0], ROWS[r][1]))


@pytest.mark.parametrize("row", GPU_ROWS, ids=lambda r: f"{r[0]}-{r[1]}")
def test_gpu_column_row(row):
    yN, yB = row
    core = core_of(ROWS[row][1])
    _report(f"K2 / fold row {row}, m {core.xM_yN_size}", ac.column_row_cases(core, yB, seed=yB),
            yN)


CFG4 = "64k[1]-n16k-4k"


def _cfg4_core():
    p = SWIFT_CONFIGS[CFG4]
    return core_of((p["W"], p["N"], p["xM_size"], p["yN_size"]))


def test_gpu_column_cfg4_cluster_half_rows():
    """cfg4 (yN = 16384, m = 1024): K2 in its two-CTA cluster form (the default) and in the
    single-CTA form, half rows with both fold passes."""
    core = _cfg4_core()
    offs = kc.facet_offsets(core)[:2]
    sg = ac.window_offsets(core)["wrap+"]
    worst = 0.0
    for variant, cluster in [(0, 2), (26, 1)]:
        # rings: the window's rows only, so that the host's longdouble sums stay short
        res, rec, cl, _ = ac.column_pair(core, [8192, 8191], offs, sg, layout="ring",
                                         variant=variant, masked=(1,), prewindowed=True,
                                         seed=variant)
        assert rec[0] == kc.TMA4 and cl == cluster, (rec, cl)
        worst = max(worst, res)
    worst = max(worst, ac.column_half_cases(core, [2049, 1024], seed=5))
    _report("cfg4 K2 / fold: cluster and single-CTA forms, half rows", worst, 16384)


def test_gpu_column_many():
    """67 facets at yN = 1024: two launches of K2 and of the fold, more lines than CTAs."""
    core = core_of(ROWS[(1024, 704)][1])
    _report("K2 / fold, 67 facets", ac.column_many_case(core, 512, seed=6), 1024)


# ---------------------------------------------------------------------- K3 / K4 <-> split
@pytest.mark.parametrize("pair", prc.ALL_PAIRS, ids=prc.pair_id)
def test_gpu_subgrid_pair(pair):
    core = core_of(prc.core_plan(pair))
    _report(f"K3/K4 / split {pair}", ac.subgrid_pair_cases(core, pair, seed=pair[0]), pair[1])


# ---------------------------------------------------------------------- primitive subgrid side
M_PLANS = slc.m_plans()
XM_PLANS = slc.xm_plans()


@pytest.mark.parametrize("plan_id", list(M_PLANS))
def test_gpu_subgrid_side_m(plan_id):
    n, _, _, geometry, _, _ = M_PLANS[plan_id]
    core = core_of(geometry)
    _report(plan_id, ac.subgrid_side_cases(core, "m", seed=n), core.xM_size)


@pytest.mark.parametrize("plan_id", list(XM_PLANS))
def test_gpu_subgrid_side_xm(plan_id):
    n, _, _, geometry, _, xa = XM_PLANS[plan_id]
    core = core_of(geometry)
    _report(plan_id, ac.subgrid_side_cases(core, "xM", xa=xa, seed=n), n)


# ---------------------------------------------------------------------- drivers
def _config(name):
    p = hc.params(name)
    _cores.clear()
    gc.collect()  # the previous test's drivers and facets
    torch.cuda.empty_cache()
    return SwiftlyConfig(W=p["W"], fov=1.0, N=p["N"], yB_size=p["yB"], yN_size=p["yN"],
                         xA_size=p["xA"], xM_size=p["xM"],
                         core=SwiftlyCoreB200(p["W"], p["N"], p["xM"], p["yN"], device=0))


def _driver(what, *args, **kw):
    res, fwd_host, bwd_host = ac.driver_case(*args, **kw)
    bound = ac.chain_bound(args[0])
    print(f"\n{what}: residual {res:.2e} (bound {bound:.1e})")
    assert res <= bound, (what, res)
    return fwd_host, bwd_host


CFG2 = "8k[1]-n4k-2k"


@pytest.mark.parametrize("mode", ["lru1", "lru2-shuffled", "host-tier", "real", "real-half"])
def test_gpu_driver_cfg2(mode):
    """The full cfg2 cover (4 x 4 facets, 8 x 8 subgrids)."""
    cfg = _config(CFG2)
    facet_cfgs, sg_cfgs = make_full_facet_cover(cfg), make_full_subgrid_cover(cfg)
    kw = {"lru1": {}, "lru2-shuffled": dict(lru=2, shuffle=True), "host-tier": dict(budget=1),
          "real": dict(real=True, shuffle=True),
          "real-half": dict(real=True, half_rows=True, lru=2)}[mode]
    hosts = _driver(f"cfg2 {mode}", cfg, facet_cfgs, sg_cfgs, seed=len(mode), **kw)
    assert hosts == ((True, True) if mode == "host-tier" else (False, False))


@pytest.mark.parametrize("pair", sorted(cc.SMALLEST), ids=cc.pair_id)
def test_gpu_driver_families(pair):
    """The smallest catalogue entry of each family outside xM / m in {2, 4}, full cover."""
    cfg = _config(cc.SMALLEST[pair])
    _driver(f"{cc.SMALLEST[pair]}", cfg, make_full_facet_cover(cfg),
            make_full_subgrid_cover(cfg), seed=pair[0])


def _progress():
    """A logger of elapsed time and a message."""
    t0 = time.time()
    return lambda msg: print(f"  {time.time() - t0:7.1f} s  {msg}", flush=True)


def _cfg4_block(block):
    cfg = _config(CFG4)
    return cfg, hc.facet_configs(cfg, CFG4, block), make_full_subgrid_cover(cfg)


def test_gpu_driver_cfg4_block():
    """cfg4's central 5 x 5 facet block over all 32 x 32 subgrids (the benchmark's workload)."""
    cfg, facet_cfgs, sg_cfgs = _cfg4_block(5)
    assert len(facet_cfgs) == 25 and len(sg_cfgs) == 1024
    torch.cuda.reset_peak_memory_stats()
    _driver("cfg4 5 x 5", cfg, facet_cfgs, sg_cfgs, log=_progress())
    print(f"peak device memory {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")


def test_gpu_driver_cfg4_block_real_half_rows():
    """cfg4's central 7 x 7 block of a real image, which fits the device with half rows only."""
    cfg, facet_cfgs, sg_cfgs = _cfg4_block(7)
    assert len(facet_cfgs) == 49
    core = cfg.core
    need = device_tier_bytes("forward", core.yN_size, core.xM_yN_size,
                             [fc.size for fc in facet_cfgs], 1, 7, cfg.max_subgrid_size,
                             half_rows=True)
    free, total = torch.cuda.mem_get_info()
    print(f"\ndevice memory: {free / 1e9:.1f} of {total / 1e9:.1f} GB free, "
          f"{torch.cuda.memory_reserved() / 1e9:.1f} GB reserved here; the forward transform "
          f"needs {need / 1e9:.1f} GB")
    if need > free:
        pytest.skip(f"the 7 x 7 block needs {need / 1e9:.1f} GB of device memory, "
                    f"{free / 1e9:.1f} GB are free")
    _driver("cfg4 7 x 7 real, half rows", cfg, facet_cfgs, sg_cfgs, real=True, half_rows=True,
            log=_progress())
