"""
SwiftlyBackwardSharded on the split kernels, two and three ``gloo`` ranks, kernels on the
host-emulated library: the supplier of each subgrid cuts it into strips for every rank's facet
rows, one ``all_to_all`` per batch moves only those strips, and each rank adds them to its
facets.  Checked against the single-process oracle; the collective calls are recorded to check
what moves.
"""

import os
import socket

import numpy
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from tests import parity_cases as pc

W, N, yB, yN, xA, xM = 13.5625, 256, 96, 128, 52, 64
N_SUBGRIDS = 7  # ragged last batch at two and at three ranks


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, world, port, sparse, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank),
                      WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from oracle.swiftly_oracle import OracleCore, backward_reference_order
        from ska_sdp_distributed_fourier_transform_b200 import (
            FacetConfig, SwiftlyConfig, make_full_facet_cover, make_full_subgrid_cover)
        from ska_sdp_distributed_fourier_transform_b200.distributed import (
            SwiftlyBackwardSharded, partition_facets)
        from tests.emu_support import emu_core_class

        core = emu_core_class()(W, N, xM, yN)
        cfg = SwiftlyConfig(W=W, fov=1.0, N=N, yB_size=yB, yN_size=yN, xA_size=xA,
                            xM_size=xM, core=core)
        if sparse:
            offs = [(0, 0), (0, 96), (96, 0), (-96, 192), (192, 192)]
            facet_cfgs = [FacetConfig(a, b, yB) for a, b in offs]
        else:
            facet_cfgs = make_full_facet_cover(cfg)
        cover = make_full_subgrid_cover(cfg)
        sgs = [cover[(5 * i) % len(cover)] for i in range(N_SUBGRIDS)]
        rng = numpy.random.default_rng(42)
        data = [pc.rand_c(rng, xA, xA) for _ in sgs]  # same on every rank
        owner = partition_facets(facet_cfgs, world)

        calls = {"all_to_all_single": [], "all_gather_into_tensor": 0}
        real_a2a = dist.all_to_all_single

        def a2a(output, input, *a, **k):  # pylint: disable=redefined-builtin
            calls["all_to_all_single"].append(input.numel() // 2)  # complex samples
            return real_a2a(output, input, *a, **k)

        def gather(*_a, **_k):
            calls["all_gather_into_tensor"] += 1
            raise AssertionError("the split backward must not replicate subgrids")

        dist.all_to_all_single = a2a
        dist.all_gather_into_tensor = gather

        bwd = SwiftlyBackwardSharded(cfg, facet_cfgs, lru_backward=1)
        assert bwd._split
        rows = [{facet_cfgs[i].off0 for i, o in enumerate(owner) if o == r} for r in range(world)]
        bwd.add_subgrid_tasks(sgs, [data[i] if i % world == rank else None
                                    for i in range(len(sgs))])
        mine = bwd.finish()
        assert sorted(mine) == [i for i, o in enumerate(owner) if o == rank]
        m = core.xM_yN_size
        rows_max = max(len(r) for r in rows)
        n_batches = (len(sgs) + world - 1) // world
        assert calls["all_to_all_single"] == [world * rows_max * m * xA] * n_batches
        assert calls["all_gather_into_tensor"] == 0
        ref = backward_reference_order(
            OracleCore(W, N, xM, yN), data, [(s.off0, s.off1) for s in sgs],
            [(c.off0, c.off1) for c in facet_cfgs], yB,
            facet_masks=[(c.mask0, c.mask1) for c in facet_cfgs])
        scale = max(numpy.abs(b).max() for b in ref)
        worst = 0.0
        for i, t in mine.items():
            worst = max(worst, numpy.abs(t.result() - ref[i]).max() / scale)
        shared_rows = sum(1 for r in range(world) for s in range(r)
                          if rows[r] & rows[s])
        q.put((rank, worst, len(mine), shared_rows))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("sparse", [False, True], ids=["full", "sparse"])
@pytest.mark.parametrize("world", [2, 3])
def test_sharded_backward_split_gloo(world, sparse):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, sparse, q))
             for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=600)
        assert p.exitcode == 0
    got = sorted(q.get(timeout=10) for _ in range(world))
    assert [g[0] for g in got] == list(range(world))
    assert sum(g[2] for g in got) == (5 if sparse else 9)
    if (world, sparse) in ((2, False), (3, True)):
        # the partition splits a facet row over two ranks: its strips are cut for both
        assert got[0][3] >= 1
    for _, worst, _, _ in got:
        assert worst <= 1e-11
