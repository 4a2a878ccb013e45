"""
The backward transform as the adjoint of the forward transform (``tests/adjoint_cases.py``) on
the host-emulated kernels: the constants on the oracle, every kernel pair in the forms the H100
runs, and the drivers end to end (device and host tier, LRU columns, real images, sharded on
gloo ranks).

Forms covered (each case asserts its launches through ``swiftly_b200_debug_last_launch``):

==========================================  ================================================
pair                                        forms
==========================================  ================================================
prepare_facet <-> finish_facet              every yN plan: line (direct), split 2 x 8192,
                                            split-F M x F, two-pass (axis 0, >= 16 columns)
prepare_facet <-> finish_facet_real         line, split-F, split
prepare_facet_real_half <->                 line, split-F, split
finish_facet_real_half
extract_columns (K2) <-> fold_column        TMA-staged and generic rows, full rows, rings,
                                            half rows (both fold passes), cluster form,
                                            67 facets (two launches), masks
sum_finish_axis <-> split_subgrid_axis      all 20 (m, xM) pairs: round-1 and two-group
                                            forward forms, 1 and 2 lines per CTA, store and
                                            add, single / grouped / batched, partial last
                                            round, capped grid
add_to_subgrid <-> extract_from_subgrid,    every m and xM of subgrid_line_cases: line and
finish_subgrid <-> prepare_subgrid,         split-F kernels, partial last CTA
subgrid_to_facets
SwiftlyForward <-> SwiftlyBackward          device / host tier, lru 1 / 2 shuffled, real
                                            images (merge, self-mirrored, unpaired, half
                                            rows), SwiftlyForward/BackwardSharded on 2 and 3
                                            gloo ranks
==========================================  ================================================
"""

import os
import socket

import numpy
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle.swiftly_oracle import OracleCore
from ska_sdp_distributed_fourier_transform_b200 import (
    FacetConfig,
    make_full_facet_cover,
    make_full_subgrid_cover,
)
from tests import adjoint_cases as ac
from tests import catalogue_cases as cc
from tests import host_tier_cases as hc
from tests import k2_cases as kc
from tests import length_cases as lc
from tests import pair_cases as prc
from tests import real_image_cases as ric
from tests import subgrid_line_cases as slc
from tests.emu_support import emu_core_class

_cores = {}


def core_of(geometry):
    """Emulated core of a geometry (W, N, xM, yN), kept for the module."""
    if geometry not in _cores:
        _cores[geometry] = emu_core_class()(*geometry)
    return _cores[geometry]


make_config = hc.config_factory(lambda W, N, xM, yN: emu_core_class()(W, N, xM, yN))


def _units(res, n):
    return res / (ac.EPS * numpy.log2(n))


# ---------------------------------------------------------------------- the oracle
@pytest.mark.parametrize("geometry, fs, sz", [((13.5625, 256, 64, 128), 95, 51),
                                              ((11.125, 1280, 320, 640), 447, 279)],
                         ids=["n256", "n1280"])
def test_constants_on_oracle(geometry, fs, sz):
    """Every primitive pair of the table and the 2-D drivers on the oracle, offsets that wrap
    past +-N, odd facet and subgrid sizes (yB, xA): residual <= 1e-14; the product per axis is
    1 / N; a constant off by a factor of two fails."""
    oracle = OracleCore(*geometry)
    N = oracle.N
    assert ac.chain_constant(oracle, ac.AXIS) == pytest.approx(1.0 / N, rel=1e-15)
    res = ac.oracle_pairs(oracle, seed=1)
    assert max(res.values()) <= 1e-14, res
    fo, so = oracle.facet_off_step, oracle.subgrid_off_step
    facet_offs = [(0, 0), (-3 * fo, N + 2 * fo), (N + fo, -N - 5 * fo)]
    subgrid_offs = [(0, 0), (3 * so, -N - so), (-2 * N + so, 2 * so), (N, N - 7 * so)]
    assert ac.oracle_drivers(oracle, facet_offs, fs, subgrid_offs, sz) <= 1e-14
    rng = numpy.random.default_rng(0)
    x, y = ac.rand_c(rng, (fs,)), ac.rand_c(rng, (oracle.yN_size,))
    Ax, ATy = oracle.prepare_facet(x, fo, 0), oracle.finish_facet(y, fo, fs, 0)
    assert ac.adjoint_residual(y, Ax, ATy, x, 2 * ac.constants(oracle)["facet"]) > 0.01


# ---------------------------------------------------------------------- K1 <-> finish_facet
PLANS = lc.yn_plans()


@pytest.mark.parametrize("plan_id", list(PLANS))
def test_emu_facet_plan(plan_id):
    """prepare_facet <-> finish_facet at the plan's yN (N = 2 yN, xM = 32): both axes, odd
    facets, offsets at and past +-N, a mask, delta probes."""
    plan, (_, W, _, _, yN) = PLANS[plan_id]
    core = core_of((W, 2 * yN, 32, yN))
    assert ac.facet_plan_cases(core, plan, seed=len(plan_id)) <= ac.pair_bound(yN)


@pytest.mark.parametrize("yN", [512, 640, 16384])
def test_emu_real_facets(yN):
    """finish_facet_real and finish_facet_real_half against their forward twins (real inner
    product), with delta probes on stored rows 0, yN / 2 and a conjugated pair."""
    core = core_of((11.0, 2 * yN, 32, yN))
    assert ac.real_facet_cases(core, seed=yN) <= ac.pair_bound(yN)


# ---------------------------------------------------------------------- K2 <-> fold_column
ROWS = kc.catalogue_rows()
EMU_ROWS = [(1024, 704), (256, 208), (768, 528)]


@pytest.mark.parametrize("row", EMU_ROWS, ids=lambda r: f"{r[0]}-{r[1]}")
def test_emu_column_row(row):
    """A catalogue row (TMA-staged at 1024, the line and split-F kernels at 256 and 768) with
    m = 16: full rows and rings, raw and prewindowed, masks, windows that wrap and straddle,
    delta probes at the window's wrap and on the first and last facet sample."""
    yN, yB = row
    core = core_of((ROWS[row][1][0], 2 * yN, 32, yN))
    assert ac.column_row_cases(core, yB, seed=yB) <= ac.pair_bound(yN)


def test_emu_column_cluster_and_many():
    """yN = 512 (the emulated 4 x Q length): the two-CTA cluster form (force_split 2) and the
    single-CTA form (7) of K2 against the fold; 67 facets: two launches of each side."""
    core = core_of((11.0, 1024, 32, 512))
    offs = kc.facet_offsets(core)
    sg = ac.window_offsets(core)["wrap+"]
    for fsplit, cluster in [(2, 2), (7, 1)]:
        res, rec, cl, _ = ac.column_pair(core, [256, 255, 300], offs, sg, force_split=fsplit,
                                         masked=(1,), prewindowed=True, seed=fsplit)
        assert rec[0] == kc.TMA4 and cl == cluster, (rec, cl)
        assert res <= ac.pair_bound(512)
    assert ac.column_many_case(core, 200, seed=3) <= ac.pair_bound(512)


@pytest.mark.parametrize("yN", [512, 640])
def test_emu_column_half_rows(yN):
    """Half rows (real inner product): the fold's two passes where the window straddles
    centred row 0 or yN / 2, with delta probes on stored rows 0 and yN / 2 and a conjugated
    pair."""
    core = core_of((11.0, 2 * yN, 32, yN))
    assert ac.column_half_cases(core, [yN // 2 + 1, yN // 4], seed=yN) <= ac.pair_bound(yN)


# ---------------------------------------------------------------------- K3 / K4 <-> split
@pytest.mark.parametrize("pair", prc.ALL_PAIRS, ids=prc.pair_id)
def test_emu_subgrid_pair(pair):
    """sum_finish_axis <-> split_subgrid_axis at one (m, xM) pair in every form its dispatch
    selects."""
    core = core_of(prc.small_plan(pair))
    assert ac.subgrid_pair_cases(core, pair, seed=pair[0]) <= ac.pair_bound(pair[1])


# ---------------------------------------------------------------------- primitive subgrid side
# m <= 512 here (the longer m run on the H100: their column accumulators take minutes on the host)
M_PLANS = {k: v for k, v in slc.m_plans().items() if v[0] <= 512}
XM_PLANS = slc.xm_plans()


@pytest.mark.parametrize("plan_id", list(M_PLANS))
def test_emu_subgrid_side_m(plan_id):
    n, _, _, _, geometry, _ = M_PLANS[plan_id]
    core = core_of(geometry)
    assert ac.subgrid_side_cases(core, "m", seed=n) <= ac.pair_bound(core.xM_size)


@pytest.mark.parametrize("plan_id", list(XM_PLANS))
def test_emu_subgrid_side_xm(plan_id):
    n, _, _, _, geometry, xa = XM_PLANS[plan_id]
    core = core_of(geometry)
    assert ac.subgrid_side_cases(core, "xM", xa=xa, seed=n) <= ac.pair_bound(n)


# ---------------------------------------------------------------------- drivers
def _cover(name, block=None):
    cfg = make_config(**hc.params(name))
    return cfg, hc.facet_configs(cfg, name, block), make_full_subgrid_cover(cfg)


@pytest.mark.parametrize("mode", ["lru1", "lru2-shuffled", "host-tier", "host-tier-lru2"])
def test_emu_driver(mode):
    """SwiftlyForward <-> SwiftlyBackward over the full 1k[1]-n512-256 cover (3 x 3 facets,
    5 x 5 subgrids with masks): N^2 sum <S_i, fwd(F)_i> = sum <bwd(S)_j, F_j> to 1e-12."""
    cfg, facet_cfgs, sg_cfgs = _cover("1k[1]-n512-256")
    lru = 2 if "lru2" in mode else 1
    budget = 1 if mode.startswith("host") else None
    res, fwd_host, bwd_host = ac.driver_case(cfg, facet_cfgs, sg_cfgs, lru=lru,
                                             shuffle=lru == 2, budget=budget, seed=lru)
    assert fwd_host == bwd_host == (budget is not None)
    assert res <= ac.chain_bound(cfg), res


@pytest.mark.parametrize("pair", sorted(cc.SMALLEST), ids=cc.pair_id)
def test_emu_driver_families(pair):
    """The smallest geometry of each catalogue family outside xM / m in {2, 4}: a sparse facet
    set over every third subgrid of the cover."""
    cfg = cc.make_config(emu_core_class(), cc.SMALL[pair])
    facet_cfgs = make_full_facet_cover(cfg)[:4]
    sg_cfgs = make_full_subgrid_cover(cfg)[::3]
    res, _, _ = ac.driver_case(cfg, facet_cfgs, sg_cfgs, seed=pair[0])
    assert res <= ac.chain_bound(cfg), res


REAL_COVER = "1280[1]-n640-256"  # 8 x 8 subgrid cover: 30 Hermitian pairs


@pytest.mark.parametrize("half_rows", [False, True], ids=["full-rows", "half-rows"])
def test_emu_driver_real(half_rows):
    """Real images, N^2 Re sum <S_i, fwd(F)_i> = sum <bwd_real(S)_j, F_j>: the forward transform
    mirrors, the backward transform merges each pair (add_subgrid_tasks); the cover shuffled,
    and the cover without every other pair's second subgrid (unpaired configs)."""
    cfg, _, sg_cfgs = _cover(REAL_COVER)
    facet_cfgs = [FacetConfig(a, b, cfg.max_facet_size)
                  for a, b in [(0, 0), (0, 440), (440, -440), (-440, 0)]]
    N, xM = cfg.image_size, cfg.internal_subgrid_size
    assert sum(j is not None for _, j in ac.mirror_pairs(sg_cfgs, N, xM)) == 30
    kept = ac.self_mirrored_and_unpaired(sg_cfgs, N, xM)
    for k, sgs in enumerate([sg_cfgs, kept]):
        res, _, _ = ac.driver_case(cfg, facet_cfgs, sgs, shuffle=k == 0, real=True,
                                   half_rows=half_rows, seed=k)
        assert res <= ac.chain_bound(cfg), res


def test_emu_driver_real_odd_explicit():
    """Odd xA = 345: explicit unmasked configs with pairs, a self-mirrored config, a config
    whose mirror is missing and a duplicate pair; real mode, half rows, lru 2."""
    cfg = make_config(**hc.params("1536[1]-n768-384"))
    facet_cfgs = [FacetConfig(a, b, cfg.max_facet_size)
                  for a, b in [(0, 0), (0, 512), (512, -512), (-512, 0)]]
    offs = [(0, 0), (192, 384), (-384, 96), (768, 0), (-192, -384), (384, -96), (96, 96),
            (192, 384), (-192, -384), (-96, 768), (96, -768), (768, 768)]
    sg_cfgs = ric.explicit_configs(cfg, offs)
    res, _, _ = ac.driver_case(cfg, facet_cfgs, sg_cfgs, lru=2, real=True, half_rows=True)
    assert res <= ac.chain_bound(cfg), res


# ---------------------------------------------------------------------- sharded, gloo
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _sharded_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank),
                      WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        # pylint: disable=import-outside-toplevel
        from ska_sdp_distributed_fourier_transform_b200 import SwiftlyConfig
        from ska_sdp_distributed_fourier_transform_b200.distributed import (
            SwiftlyBackwardSharded, SwiftlyForwardSharded, partition_facets)

        W, N, yB, yN, xA, xM = 13.5625, 256, 96, 128, 52, 64
        core = emu_core_class()(W, N, xM, yN)
        cfg = SwiftlyConfig(W=W, fov=1.0, N=N, yB_size=yB, yN_size=yN, xA_size=xA,
                            xM_size=xM, core=core)
        facet_cfgs = make_full_facet_cover(cfg)
        sgs = make_full_subgrid_cover(cfg)[:7]  # ragged last batch at two and three ranks
        rng = numpy.random.default_rng(42)
        facets = [ac.rand_c(rng, (yB, yB)) for _ in facet_cfgs]  # same on every rank
        masked = [f * ac.mask_2d(c) for f, c in zip(facets, facet_cfgs)]
        owner = partition_facets(facet_cfgs, world)
        local = {i: masked[i] for i, o in enumerate(owner) if o == rank}

        def probe(i):
            s = ac.subgrid_probe(core, i, xA, 7)
            return s * ac._mask_2d(sgs[i], s)  # pylint: disable=protected-access

        lhs = [numpy.clongdouble(0)]
        fwd = SwiftlyForwardSharded(cfg, facet_cfgs, local, lru_forward=1)

        den = [numpy.longdouble(0)]

        def consume(i, _cfg, t):
            s = probe(i)
            lhs[0] += ac.inner(s, t)
            den[0] += ac.norm(s) * ac.norm(t) * N ** 2

        fwd.get_subgrid_tasks(sgs, consumer=consume)
        del fwd
        bwd = SwiftlyBackwardSharded(cfg, facet_cfgs, lru_backward=1)
        bwd.add_subgrid_tasks(sgs, [probe(i) if i % world == rank else None
                                    for i in range(len(sgs))])
        mine = bwd.finish()
        rhs = sum((ac.inner(t.result(), facets[i]) for i, t in mine.items()),
                  numpy.clongdouble(0))
        den[0] += sum(ac.norm(t.result()) * ac.norm(facets[i]) for i, t in mine.items())
        # every rank: its share of both sides (subgrids it owns, facets it owns)
        q.put((rank, complex(lhs[0]), complex(rhs), float(den[0])))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_gloo_adjoint(world):
    """SwiftlyForwardSharded <-> SwiftlyBackwardSharded (split kernels, strip exchange) on
    ``world`` gloo ranks: the ranks' shares of both sides sum to the identity."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_sharded_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=600)
        assert p.exitcode == 0
    got = sorted(q.get(timeout=10) for _ in range(world))
    assert [g[0] for g in got] == list(range(world))
    lhs = sum(g[1] for g in got) * 256.0 ** 2
    rhs = sum(g[2] for g in got)
    # Cauchy-Schwarz per rank: the sum of the ranks' norm products bounds the residual's scale
    den = sum(g[3] for g in got)
    assert abs(lhs - rhs) / den <= ac.CHAIN_BOUND, (lhs, rhs, den)
