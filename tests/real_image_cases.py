"""
Shared checks of the real-image forward transform, run by tests/test_emu_real_image.py on the
host-emulated kernels and by tests/test_gpu_real_image.py on the H100.

ABI level: ``mirror_subgrid`` against numpy, exactly (one product of two mask samples and one of
the source sample per output sample).  API level: ``SwiftlyForward(real_image=True)`` against the
default mode on the same real facets -- every source output equals the default subgrid, every
mirror the masked conjugate reversal of the default subgrid at the source size ``S`` (bitwise:
the covers' masks are 0/1, so masking after the transforms gives the samples masking inside K3 /
K4 gives); the mirrors as accurate as the default path against the analytic DFT; the work done
(distinct K2 columns, K3 / K4 and mirror calls).
"""

import contextlib
import ctypes

import numpy
import pytest
import torch

from ska_sdp_distributed_fourier_transform_b200 import (
    FacetConfig,
    SubgridConfig,
    SwiftlyForward,
    _lib,
    api,
)
from ska_sdp_distributed_fourier_transform_b200.fourier_algorithm import make_subgrid_from_sources
from tests import k2_cases as kc

MIRROR = 16  # kernel code of swiftly_b200_debug_last_launch (plan.h)
NAN = complex(numpy.nan, numpy.nan)


def source_size(sz):
    return 2 * (sz // 2) + 1


# ---------------------------------------------------------------------- ABI level
def _weights(sz, pair):
    m0, m1 = (numpy.ones(sz) if m is None else m for m in (pair or (None, None)))
    return m0[:, None] * m1[None, :]


def _scaled(z, w):
    out = numpy.empty(z.shape, dtype=complex)
    out.real = z.real * w
    out.imag = z.imag * w
    return out


def expected(src, sz, masks=None, mirror_masks=None):
    """numpy: ``(out, mirror)`` of ``mirror_subgrid``."""
    h = sz // 2
    out = _scaled(src[:sz, :sz], _weights(sz, masks))
    mirror = _scaled(numpy.conj(src[2 * h::-1, 2 * h::-1][:sz, :sz]), _weights(sz, mirror_masks))
    return out, mirror


def _outputs(core, sz, layout):
    """``(out, mirror, wide arrays or None)``: fresh tensors, NaN-prefilled views inside wider
    arrays, or NaN-prefilled transposed views."""
    dev = kc._dev(core)
    if layout == "own":
        return None, None, None
    if layout == "wide":
        wides = [torch.full((sz + 5, sz + 9), NAN, dtype=torch.complex128, device=dev)
                 for _ in range(2)]
        return wides[0][2:2 + sz, 3:3 + sz], wides[1][4:4 + sz, 1:1 + sz], wides
    assert layout == "transposed"
    ts = [torch.full((sz, sz), NAN, dtype=torch.complex128, device=dev).t() for _ in range(2)]
    return ts[0], ts[1], None


def mirror_case(core, sz, *, extra=0, masked=(), layout="own", cap=0, seed=0):
    """One ``mirror_subgrid`` call: a random source of ``S + extra`` rows and columns, the masks
    with index in ``masked`` (0, 1: the subgrid's, 2, 3: the mirror's) random, the others None.
    Exact equality with numpy; the launch recorded as ``MirrorSubgridKernel``."""
    rng = numpy.random.default_rng(seed)
    n = source_size(sz) + extra
    src = rng.standard_normal((n, n)) + 1j * rng.standard_normal((n, n))
    masks = [rng.random(sz) if k in masked else None for k in range(4)]
    dmasks = [None if mk is None else kc._to(core, mk) for mk in masks]
    out, mirror, wides = _outputs(core, sz, layout)
    with kc.hooks(core, 0, cap, 0):
        got = core.mirror_subgrid(kc._to(core, src), sz, out=out, mirror=mirror,
                                  masks=dmasks[:2], mirror_masks=dmasks[2:])
        rec = kc.last_launch(core)
    want = expected(src, sz, masks[:2], masks[2:])
    for name, g, w in zip(("out", "mirror"), got, want):
        g = g.cpu().numpy()
        assert numpy.array_equal(g, w), f"{name}: max diff {numpy.abs(g - w).max():.3e}"
    if wides is not None:
        for k, (wide, (r0, c0)) in enumerate(zip(wides, ((2, 3), (4, 1)))):
            outside = torch.isnan(wide.real).cpu().numpy()
            outside[r0:r0 + sz, c0:c0 + sz] = ~outside[r0:r0 + sz, c0:c0 + sz]
            assert outside.all(), f"output {k}: a sample outside the view was written"
    grid = source_size(sz) if not cap else min(cap, source_size(sz))
    assert tuple(rec) == (MIRROR, 0, 0, grid), rec
    return rec


def _raw(core, src, out, mirror, locations=(_lib.DEVICE,) * 3):
    """The C entry point on tensors described with the given locations (no Python checks)."""
    # pylint: disable=protected-access
    descs = [core._describe(t, 1) for t in (src, out, mirror)]
    for d, loc in zip(descs, locations):
        d.location = loc
    rc = core._lib.swiftly_b200_mirror_subgrid(
        core._plan, *[ctypes.byref(d) for d in descs], None, None, None, None, ctypes.c_void_p(0))
    _lib.check(core._lib, rc)


def mirror_rejects(core):
    """``EINVAL`` (``ValueError``): a source smaller than ``2h + 1`` in either dimension, output
    shapes that disagree, and host arrays."""
    dev = kc._dev(core)

    def z(*shape):
        return torch.zeros(shape, dtype=torch.complex128, device=dev)

    for sz in (8, 9):
        n = source_size(sz)
        for src in (z(n - 1, n), z(n, n - 1)):
            with pytest.raises(ValueError, match="source"):
                _raw(core, src, z(sz, sz), z(sz, sz))
            with pytest.raises(ValueError):
                core.mirror_subgrid(src, sz)
        for out, mirror in ((z(sz, sz - 1), z(sz, sz)), (z(sz - 1, sz), z(sz, sz)),
                            (z(sz, sz), z(sz, sz + 1)), (z(sz, sz), z(sz + 1, sz))):
            with pytest.raises(ValueError, match="out and mirror"):
                _raw(core, z(n, n), out, mirror)
            with pytest.raises(ValueError):
                core.mirror_subgrid(z(n, n), sz, out=out, mirror=mirror)
        for k in range(3):
            locs = [_lib.DEVICE] * 3
            locs[k] = _lib.HOST
            with pytest.raises(ValueError, match="device arrays only"):
                _raw(core, z(n, n), z(sz, sz), z(sz, sz), locs)


# ---------------------------------------------------------------------- API level
def point_sources(N, facet_cfgs, n, seed):
    """``n`` point sources of intensity 0.5 ... 1.5 inside the facets (which may be sparse)."""
    rng = numpy.random.default_rng(seed)
    out = []
    for _ in range(n):
        fc = facet_cfgs[int(rng.integers(len(facet_cfgs)))]
        pos = [(off + int(rng.integers(-(fc.size // 2), fc.size // 2)) + N // 2) % N - N // 2
               for off in (fc.off0, fc.off1)]
        out.append((float(rng.random()) + 0.5, pos[0], pos[1]))
    return out


class Work:
    """What a forward transform ran while ``active``: the subgrid columns K2 (``extract_columns``)
    ran for, the K3 / K4 blocks it prepared (``prepare_sum_finish``) and calls it made
    (``PreparedSumFinish.launch``), and the ``mirror_subgrid`` calls."""

    def __init__(self):
        self.active = False
        self.k2_columns = set()
        self.prepared = 0
        self.sum_finish = 0
        self.mirror = 0


@contextlib.contextmanager
def counting(core):
    """Count the work of ``core``'s callers into a :class:`Work` (test-local wrappers)."""
    work = Work()
    orig_k2, orig_prep, orig_mirror = (core.extract_columns, core.prepare_sum_finish,
                                       core.mirror_subgrid)

    def k2(BF_Fs, subgrid_off0, *a, **k):
        if work.active:
            work.k2_columns.add(subgrid_off0 % core.N)
        return orig_k2(BF_Fs, subgrid_off0, *a, **k)

    def prep(*a, **k):
        if work.active:
            work.prepared += 1
        block = orig_prep(*a, **k)
        launch = block.launch

        def counted(*la, **lk):
            if work.active:
                work.sum_finish += 1
            return launch(*la, **lk)

        block.launch = counted
        return block

    def mirror(*a, **k):
        if work.active:
            work.mirror += 1
        return orig_mirror(*a, **k)

    core.extract_columns, core.prepare_sum_finish, core.mirror_subgrid = k2, prep, mirror
    try:
        yield work
    finally:
        del core.extract_columns, core.prepare_sum_finish, core.mirror_subgrid


def _masked(z, sg):
    """``z`` (a device tensor) times the subgrid's masks, one product per sample like the
    kernel (``z`` is multiplied by ``mask0[r] * mask1[c]``)."""
    w = torch.from_numpy(_weights(sg.size, (sg.mask0, sg.mask1))).to(z.device)
    return torch.view_as_complex(torch.view_as_real(z.resolve_conj().contiguous()) * w[..., None])


def rel_errs(N, sg, gots, sources):
    """``max|got - truth| / max|truth|`` of each of ``gots`` against the analytic DFT."""
    truth = make_subgrid_from_sources(sources, N, sg.size, [sg.off0, sg.off1],
                                      [sg.mask0, sg.mask1])
    scale = numpy.abs(truth).max()
    return [float(numpy.abs(g.cpu().numpy() - truth).max() / scale) for g in gots]


def driver_case(cfg, facet_cfgs, facets, sg_cfgs, *, lru=1, budget=None, sources=None,
                accuracy=None):
    """``SwiftlyForward(real_image=True).iter_subgrid_tasks`` against the default mode on the
    same facets, bitwise, on every config; the order of the yielded tasks; the work done.  With
    ``sources``: the relative error against the analytic DFT of the configs in ``accuracy`` (all
    when None), real mode against default mode.  Returns ``(pairs, work, errors)``."""
    core, N = cfg.core, cfg.image_size
    tasks = list(zip(facet_cfgs, facets))
    ref = SwiftlyForward(cfg, tasks, lru_forward=lru, queue_size=4)
    fwd = SwiftlyForward(cfg, tasks, lru_forward=lru, queue_size=4, device_budget=budget,
                         real_image=True)
    if budget is not None:
        assert fwd.host_tier
    pairs = api.mirror_pairs(sg_cfgs, N, cfg.internal_subgrid_size)
    source_of = {j: i for i, j in pairs if j is not None}
    order = [k for i, j in pairs for k in ((i,) if j is None else (i, j))]
    assert sorted(order) == list(range(len(sg_cfgs)))
    errors = {"real": {}, "default": {}}
    got_order = []
    with counting(core) as work:
        it = fwd.iter_subgrid_tasks(sg_cfgs)
        while True:
            work.active = True
            try:
                idx, task = next(it)
            except StopIteration:
                break
            finally:
                work.active = False
            got_order.append(idx)
            sg = sg_cfgs[idx]
            direct = ref.get_subgrid_task(sg).tensor
            if idx in source_of:
                src = sg_cfgs[source_of[idx]]
                T = ref.get_subgrid_task(
                    SubgridConfig(src.off0, src.off1, source_size(src.size))).tensor
                want = _masked(T.flip(0, 1)[:sg.size, :sg.size].conj(), sg)
            else:
                want = direct
            assert torch.equal(task.tensor, want), (
                f"subgrid {idx} {sg} ({'mirror' if idx in source_of else 'computed'}): max diff "
                f"{(task.tensor - want).abs().max().item():.3e}")
            if sources is not None and (accuracy is None or idx in accuracy):
                errors["real"][idx], errors["default"][idx] = rel_errs(
                    N, sg, (task.tensor, direct), sources)
    assert got_order == order
    assert work.mirror == len(source_of)
    assert work.sum_finish == 2 * len(pairs)  # one K3 and one K4 call per computed subgrid
    assert work.k2_columns == {sg_cfgs[i].off0 % N for i, _ in pairs}
    if sources is not None:
        mirrored = [errors["real"][k] for k in errors["real"] if k in source_of]
        assert mirrored, "no mirrored subgrid checked against the analytic DFT"
        assert max(mirrored) <= 2 * max(errors["default"].values()), errors
    return pairs, work, errors


def full_cover_counts(n):
    """A full cover of ``n x n`` subgrids (``n`` even) in cover order: K2 columns, subgrids
    computed, and K3 / K4 blocks prepared -- K3 once per column and size (columns 0 and n/2 hold
    the self-mirrored subgrids: sizes S and xA), K4 once per size."""
    return n // 2 + 1, n * n // 2 + 2, n // 2 + 3 + 2


def self_mirrored(cfg, sg_cfgs):
    N = cfg.image_size
    return [k for k, sg in enumerate(sg_cfgs) if (2 * sg.off0) % N == 0 and (2 * sg.off1) % N == 0]


def accuracy_set(cfg, sg_cfgs, pairs, n_pairs=3):
    """The first, middle and last of the pairs (both members) and the self-mirrored subgrids."""
    both = [p for p in pairs if p[1] is not None]
    pick = [both[0], both[len(both) // 2], both[-1]][:n_pairs]
    return {k for p in pick for k in p} | set(self_mirrored(cfg, sg_cfgs))


def rejects_complex(cfg, facet_cfgs, facets):
    """Complex facets (numpy or tensor) raise ``ValueError`` naming the facet."""
    tasks = [(fc, f) for fc, f in zip(facet_cfgs, facets)]
    k = len(tasks) - 1
    for bad in (numpy.asarray(facets[k], dtype=complex),
                torch.from_numpy(numpy.asarray(facets[k], dtype=complex))):
        with pytest.raises(ValueError, match=f"facet {k} "):
            SwiftlyForward(cfg, tasks[:k] + [(tasks[k][0], bad)], real_image=True)
    # real numpy / tensor facets of any floating width are accepted
    SwiftlyForward(cfg, [(tasks[0][0], numpy.asarray(facets[0], dtype=numpy.float32))],
                   real_image=True)
    SwiftlyForward(cfg, [(tasks[0][0], torch.from_numpy(numpy.asarray(facets[0])))],
                   real_image=True)


def explicit_configs(cfg, offsets):
    """Unmasked subgrid configs of the maximum subgrid size at the given offsets."""
    return [SubgridConfig(a, b, cfg.max_subgrid_size) for a, b in offsets]


def facet_block(cfg, offs):
    return [FacetConfig(a, b, cfg.max_facet_size) for a, b in offs]
