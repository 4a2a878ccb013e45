"""
SwiftlyForwardSharded / SwiftlyBackwardSharded on two ``gloo`` ranks (see
tests/test_dist_gloo.py) at catalogue geometries whose fused subgrid kernel is the round-1
form: (m, xM) = (128, 1024), eight transforms per round, and the mixed-radix (160, 320).
Kernels on the host-emulated library; checked against the single-process oracle.
"""

import os
import socket

import numpy
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from tests import catalogue_cases as cc
from tests import parity_cases as pc


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, world, port, pair, sparse, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank),
                      WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from oracle.swiftly_oracle import OracleCore, backward_reference_order, forward_reference_order
        from ska_sdp_distributed_fourier_transform_b200 import make_full_facet_cover
        from ska_sdp_distributed_fourier_transform_b200.distributed import (
            SwiftlyBackwardSharded, SwiftlyForwardSharded, partition_facets)
        from tests.emu_support import emu_core_class

        cfg = cc.make_config(emu_core_class(), cc.SMALL[pair])
        core = cfg.core
        yB, xA = cfg.max_facet_size, cfg.max_subgrid_size
        if sparse:
            facet_cfgs, _, sgs = cc.facets_and_subgrids(cfg, 5, 7, seed=0)
        else:
            facet_cfgs = make_full_facet_cover(cfg)
            _, _, sgs = cc.facets_and_subgrids(cfg, 0, 7, seed=0)
        rng = numpy.random.default_rng(42)
        facets = [pc.rand_c(rng, yB, yB) for _ in facet_cfgs]  # same on every rank
        owner = partition_facets(facet_cfgs, world)
        local = {i: facets[i] for i, o in enumerate(owner) if o == rank}
        fwd = SwiftlyForwardSharded(cfg, facet_cfgs, local, lru_forward=1)
        tasks = fwd.get_subgrid_tasks(sgs)
        assert sorted(tasks) == [i for i in range(len(sgs)) if i % world == rank]
        oracle = OracleCore(core.W, core.N, core.xM_size, core.yN_size)
        ref = forward_reference_order(
            oracle, facets, [(c.off0, c.off1) for c in facet_cfgs],
            [(s.off0, s.off1) for s in sgs], xA,
            subgrid_masks=[(s.mask0, s.mask1) for s in sgs])
        scale = max(numpy.abs(r).max() for r in ref)
        worst = 0.0
        for i, t in tasks.items():
            worst = max(worst, numpy.abs(t.result() - ref[i]).max() / scale)
        bwd = SwiftlyBackwardSharded(cfg, facet_cfgs, lru_backward=1)
        bwd.add_subgrid_tasks(sgs, [tasks.get(i) for i in range(len(sgs))])
        mine = bwd.finish()
        assert sorted(mine) == [i for i, o in enumerate(owner) if o == rank]
        back_ref = backward_reference_order(
            oracle, ref, [(s.off0, s.off1) for s in sgs],
            [(c.off0, c.off1) for c in facet_cfgs], yB,
            facet_masks=[(c.mask0, c.mask1) for c in facet_cfgs])
        bscale = max(numpy.abs(b).max() for b in back_ref)
        for i, t in mine.items():
            worst = max(worst, numpy.abs(t.result() - back_ref[i]).max() / bscale)
        q.put((rank, worst, len(tasks)))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("sparse", [False, True], ids=["full", "sparse"])
@pytest.mark.parametrize("pair", [(128, 1024), (160, 320)], ids=cc.pair_id)
def test_sharded_catalogue_two_ranks_gloo(pair, sparse):
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, pair, sparse, q))
             for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=600)
        assert p.exitcode == 0
    got = sorted(q.get(timeout=10) for _ in range(world))
    assert [g[0] for g in got] == [0, 1]
    assert sum(g[2] for g in got) == 7
    for _, worst, _ in got:
        assert worst <= 1e-11
