"""
Shared checks of the host tier (facet arrays in host memory, an ``m``-row ring per facet on the
device) run by tests/test_emu_host_tier.py on the host-emulated kernels and by
tests/test_gpu_host_tier.py on the H100.

ABI level: ``extract_columns`` and ``fold_column`` on row rings against the same call on whole
facet arrays -- bitwise, with the same launch form.  API level: ``SwiftlyForward`` /
``SwiftlyBackward`` in the host tier (``device_budget=1``) against the device tier -- bitwise, and
the rows the host tier moves against the count for subgrids in cover order.  Every sample goes
through the same arithmetic in the same order in both forms, so any difference is a bug.
"""

import contextlib
import random

import numpy
import pytest
import torch

from ska_sdp_distributed_fourier_transform_b200 import (
    FacetConfig,
    SwiftlyBackward,
    SwiftlyConfig,
    SwiftlyForward,
    make_full_facet_cover,
    make_full_subgrid_cover,
)
from ska_sdp_distributed_fourier_transform_b200 import api
from ska_sdp_distributed_fourier_transform_b200.swift_configs import SWIFT_CONFIGS
from tests import k2_cases as kc
from tests import parity_cases as pc

NAN = complex(numpy.nan, numpy.nan)


# ---------------------------------------------------------------------- ABI level
def window_rows(oracle, sg_off0):
    return [int(r) for r in oracle._facet_window(sg_off0)]  # pylint: disable=protected-access


def make_ring(core, oracle, full, sg_off0, prev_off0=None):
    """NaN-prefilled ``(m, size)`` ring holding the window rows of ``sg_off0`` of ``full`` at line
    ``r mod m``.  With ``prev_off0`` the ring first holds that column's window and then receives
    only the rows the new window adds (a slid ring: rows that stay keep their line)."""
    m = core.xM_yN_size
    ring = torch.full((m, full.shape[1]), NAN, dtype=torch.complex128, device=full.device)
    have = set()
    for off in ([] if prev_off0 is None else [prev_off0]) + [sg_off0]:
        rows = [r for r in window_rows(oracle, off) if r not in have]
        if rows:
            ring[torch.tensor([r % m for r in rows], device=full.device)] = \
                full[torch.tensor(rows, device=full.device)]
        have = set(window_rows(oracle, off))
    return ring


def check_window_start(core, oracle, sg_off0):
    """The driver's window start gives the oracle's window rows."""
    start = api.window_start(core, sg_off0)
    yN, m = core.yN_size, core.xM_yN_size
    assert sorted(window_rows(oracle, sg_off0)) == sorted((start + u) % yN for u in range(m))


def k2_ring_case(core, oracle, sizes, offs, sg_off0, *, prev_off0=None, variant=0, cap=0,
                 force_split=0, seed=0):
    """``extract_columns`` (prewindowed, as the driver runs it) on rings and on whole facets:
    the same launch record and the same bits.  Returns the record."""
    rng = numpy.random.default_rng(seed)
    yN = core.yN_size
    check_window_start(core, oracle, sg_off0)
    fulls = [kc._to(core, pc.rand_c(rng, yN, fs)) for fs in sizes]
    rings = [make_ring(core, oracle, f, sg_off0, prev_off0) for f in fulls]
    out_full, _ = kc.make_outputs(core, len(sizes), "own")
    out_ring, _ = kc.make_outputs(core, len(sizes), "own")
    with kc.hooks(core, variant, cap, force_split):
        core.extract_columns(fulls, sg_off0, list(offs), outs=out_full, prewindowed=True)
        got_full = kc.last_launch(core)
        core.extract_columns(rings, sg_off0, list(offs), outs=out_ring, prewindowed=True)
        got_ring = kc.last_launch(core)
    assert got_ring == got_full, (got_ring, got_full)
    for j, (a, b) in enumerate(zip(out_full, out_ring)):
        assert not bool(torch.isnan(a.real).any()), f"facet {j}: output not written"
        assert torch.equal(a, b), f"facet {j}: ring differs from the whole facet"
    return got_ring


def fold_ring_case(core, oracle, sizes, offs, sg_off0, *, prev_off0=None, cap=0, force_split=0,
                   seed=0):
    """``fold_column`` into rings and into whole facet accumulators: the same launch record and,
    on every window row, the same bits.  Returns the record."""
    rng = numpy.random.default_rng(seed)
    yN, m = core.yN_size, core.xM_yN_size
    check_window_start(core, oracle, sg_off0)
    cols = [kc._to(core, pc.rand_c(rng, m, yN)) for _ in sizes]
    fulls = [kc._to(core, pc.rand_c(rng, yN, fs)) for fs in sizes]
    rings = [make_ring(core, oracle, f, sg_off0, prev_off0) for f in fulls]
    masks = [None if j % 2 == 0 else kc._to(core, (rng.random(fs) > 0.3).astype(float))
             for j, fs in enumerate(sizes)]
    with kc.hooks(core, 0, cap, force_split):
        core.fold_column(cols, fulls, list(offs), masks, sg_off0)
        got_full = kc.last_launch(core)
        core.fold_column(cols, rings, list(offs), masks, sg_off0)
        got_ring = kc.last_launch(core)
    assert got_ring == got_full, (got_ring, got_full)
    rows = window_rows(oracle, sg_off0)
    idx = torch.tensor(rows, device=fulls[0].device)
    lines = torch.tensor([r % m for r in rows], device=fulls[0].device)
    for j, (f, r) in enumerate(zip(fulls, rings)):
        assert torch.equal(f[idx], r[lines]), f"facet {j}: ring differs from the whole accumulator"
    return got_ring


def ring_rejects(core, oracle):
    """Row counts other than yN and m, and rings mixed with whole facets, are rejected."""
    yN, m = core.yN_size, core.xM_yN_size
    dev = kc._dev(core)
    out, _ = kc.make_outputs(core, 2, "own")
    full = torch.zeros((yN, 8), dtype=torch.complex128, device=dev)
    ring = torch.zeros((m, 8), dtype=torch.complex128, device=dev)
    bad = torch.zeros((m + 1, 8), dtype=torch.complex128, device=dev)
    for bfs in ([bad], [full, ring], [ring, full]):
        with pytest.raises(ValueError):
            core.extract_columns(bfs, 0, [0] * len(bfs), outs=out[:len(bfs)], prewindowed=True)
    cols = [torch.zeros((m, yN), dtype=torch.complex128, device=dev) for _ in range(2)]
    for accs in ([bad], [full, ring]):
        with pytest.raises(ValueError):
            core.fold_column(cols[:len(accs)], accs, [0] * len(accs), [None] * len(accs), 0)


# ---------------------------------------------------------------------- API level
GEOMETRIES = {
    "1k[1]-n512-256": None,        # full cover
    "1280[1]-n640-320": None,      # mixed radix (split-F kernels)
    "1k[1]-n512-256-sparse": [(0, 0), (0, 416), (416, -416), (-416, 416), (-416, 0)],
}


def params(name):
    p = SWIFT_CONFIGS[name.replace("-sparse", "")]
    return dict(W=p["W"], N=p["N"], yB=p["yB_size"], yN=p["yN_size"], xA=p["xA_size"],
                xM=p["xM_size"])


def facet_configs(cfg, name, block=None):
    """Full cover, the sparse list of GEOMETRIES, or the central ``block x block`` of the cover."""
    if GEOMETRIES.get(name):
        return [FacetConfig(a, b, cfg.max_facet_size) for a, b in GEOMETRIES[name]]
    cover = make_full_facet_cover(cfg)
    if block is None:
        return cover
    offs = sorted({c.off0 for c in cover})
    n = len(offs)
    keep = set(offs[(n - block) // 2:(n - block) // 2 + block])
    return [c for c in cover if c.off0 in keep and c.off1 in keep]


@contextlib.contextmanager
def ring_batch(batch):
    old = api.RING_BATCH
    api.RING_BATCH = batch
    try:
        yield
    finally:
        api.RING_BATCH = old


def cover_rows(core, sg_cfgs):
    """Rows of the ``m``-row window that enter the rings over a transform in cover order:
    ``m`` for the first subgrid column, the column step for every further one."""
    cols = sorted({s.off0 for s in sg_cfgs})
    step = (cols[1] - cols[0]) * core.yN_size // core.N if len(cols) > 1 else 0
    assert step <= core.xM_yN_size
    return core.xM_yN_size + (len(cols) - 1) * step


def forward_tiers(cfg, facet_cfgs, facets, sg_cfgs, lru, batch):
    """Subgrids of the device tier and of the host tier (bitwise equal) and the host driver."""
    res = {}
    for host in (False, True):
        with ring_batch(batch):
            fwd = SwiftlyForward(cfg, list(zip(facet_cfgs, facets)), lru_forward=lru,
                                 queue_size=4, device_budget=1 if host else None)
            assert fwd.host_tier == host
            res[host] = [fwd.get_subgrid_task(sg).result() for sg in sg_cfgs]
            if host:
                host_fwd = fwd
    for i, (a, b) in enumerate(zip(res[False], res[True])):
        assert numpy.array_equal(a, b), f"subgrid {i}: host tier differs from the device tier"
    return res[True], host_fwd


def backward_tiers(cfg, facet_cfgs, subgrids, sg_cfgs, lru):
    """Facets of the device tier and of the host tier (bitwise equal) and the host driver."""
    res = {}
    for host in (False, True):
        bwd = SwiftlyBackward(cfg, facet_cfgs, lru_backward=lru, queue_size=4,
                              device_budget=1 if host else None)
        assert bwd.host_tier == host
        for sg, data in zip(sg_cfgs, subgrids):
            bwd.add_new_subgrid_task(sg, data)
        tasks = bwd.finish()
        res[host] = [numpy.asarray(t.result()) for t in tasks]
        if host:
            host_bwd = bwd
            assert all(t.tensor.device.type == "cpu" for t in tasks)
    for j, (a, b) in enumerate(zip(res[False], res[True])):
        assert numpy.array_equal(a, b), f"facet {j}: host tier differs from the device tier"
    return res[True], host_bwd


def case_tiers(make_config, name, *, shuffle, lru, batch, block=None, seed=0):
    """Forward and backward: host tier bitwise equal to the device tier; in cover order the rows
    moved match :func:`cover_rows`."""
    p = params(name)
    cfg = make_config(**p)
    core = cfg.core
    rng = numpy.random.default_rng(seed)
    facet_cfgs = facet_configs(cfg, name, block)
    facets = [pc.rand_c(rng, fc.size, fc.size) for fc in facet_cfgs]
    sg_cfgs = make_full_subgrid_cover(cfg)
    if shuffle:
        random.Random(seed).shuffle(sg_cfgs)
    subgrids, fwd = forward_tiers(cfg, facet_cfgs, facets, sg_cfgs, lru, batch)
    _, bwd = backward_tiers(cfg, facet_cfgs, subgrids, sg_cfgs, lru)
    if not shuffle:
        rows = cover_rows(core, sg_cfgs)
        assert fwd.h2d_rows == rows
        assert bwd.h2d_rows + bwd.zeroed_rows == rows
        assert bwd.d2h_rows == rows
        assert bwd.h2d_rows == max(0, rows - core.yN_size)
        yB = sum(fc.size for fc in facet_cfgs)
        assert fwd.copied_bytes == (16 * rows * yB, 16 * core.yN_size * yB)
    return cfg, fwd, bwd


def config_factory(core_factory):
    def make_config(W, N, yB, yN, xA, xM):
        return SwiftlyConfig(W=W, fov=1.0, N=N, yB_size=yB, yN_size=yN, xA_size=xA, xM_size=xM,
                             core=core_factory(W, N, xM, yN))
    return make_config
