"""
The catalogue geometries whose (m, xM) pair lies outside xM / m in {2, 4}, shared by the
emulated, the gloo and the GPU tests.  Their fused subgrid kernel is the round-1 form
(SubgridAxisKernel): CONC = 8 at (128, 1024), CONC = 1 at (256, 256), and mixed-radix
transforms (3, 5, 7 * 2^k points, line_fft_mixed) at the other four pairs.
"""

import numpy
import torch

from oracle.swiftly_oracle import OracleCore, forward_reference_order
from ska_sdp_distributed_fourier_transform_b200 import (
    FacetConfig,
    SwiftlyConfig,
    SwiftlyForward,
    make_full_subgrid_cover,
)
from ska_sdp_distributed_fourier_transform_b200.swift_configs import SWIFT_CONFIGS
from tests import parity_cases as pc

# (m, xM) -> smallest catalogue entry
SMALLEST = {
    (128, 1024): "16k[1]-n2k-1k",
    (256, 256): "1k[1]-n1k-256",
    (128, 384): "1536[1]-n512-384",
    (160, 320): "1280[1]-n640-320",
    (192, 384): "1536[1]-n768-384",
    (224, 448): "1792[1]-n896-448",
}

# (m, xM) -> small plan (W, N, yB, yN, xA, xM) for the emulated kernels: the catalogue entry
# itself, or (for 16k[1]-n2k-1k) a plan with the same (m, xM) and an eighth of the image size
# (with yB = yN / 2: at the catalogue's yB / yN = 0.89 and this small yN the window amplifies
# rounding beyond the 1e-12 bound on the fused and the primitive path alike)
SMALL = {
    (128, 1024): (13.5625, 2048, 128, 256, 512, 1024),
    (256, 256): (9.25, 1024, 512, 1024, 236, 256),
    (128, 384): (12.0, 1536, 384, 512, 296, 384),
    (160, 320): (11.125, 1280, 448, 640, 280, 320),
    (192, 384): (10.75, 1536, 512, 768, 345, 384),
    (224, 448): (10.875, 1792, 608, 896, 392, 448),
}


def pair_id(pair):
    return f"{pair[0]}_{pair[1]}"


def catalogue_plan(name):
    p = SWIFT_CONFIGS[name]
    return (p["W"], p["N"], p["yB_size"], p["yN_size"], p["xA_size"], p["xM_size"])


def make_config(core_cls, plan):
    W, N, yB, yN, xA, xM = plan
    core = core_cls(W, N, xM, yN)
    return SwiftlyConfig(W=W, fov=1.0, N=N, yB_size=yB, yN_size=yN, xA_size=xA, xM_size=xM,
                         core=core)


def device(cfg):
    return getattr(cfg.core, "tensor_device", None) or torch.device("cuda", 0)


def to_dev(cfg, a):
    return torch.from_numpy(numpy.ascontiguousarray(a)).clone().to(device(cfg))


def sum_finish_vs_oracle(cfg, axis, contrib_sized, facet_steps, sg_off, sz, masked, seed,
                         lines=7):
    """One ``sum_finish_axis`` call against extract_from_facet -> add_to_subgrid ->
    finish_subgrid of the oracle; facet offsets in units of yN / 2 (the window moves by m / 2)."""
    core = cfg.core
    oracle = OracleCore(cfg.core.W, cfg.core.N, cfg.core.xM_size, cfg.core.yN_size)
    rng = numpy.random.default_rng(seed)
    size = core.xM_yN_size if contrib_sized else core.yN_size
    offs = [k * (core.yN_size // 2) for k in facet_steps]
    srcs = [pc.rand_c(rng, lines, size) for _ in offs]
    if axis == 0:
        srcs = [s.T for s in srcs]
    mask = (rng.random(sz) > 0.3).astype(float) if masked else None
    shape = (lines, sz) if axis == 1 else (sz, lines)
    out = torch.empty(shape, dtype=torch.complex128, device=device(cfg))
    core.sum_finish_axis([(torch.from_numpy(s).to(device(cfg)), o) for s, o in zip(srcs, offs)],
                         out, axis=axis, subgrid_off=sg_off,
                         mask=None if mask is None else to_dev(cfg, mask))
    acc = None
    for s, o in zip(srcs, offs):
        c = s if contrib_sized else oracle.extract_from_facet(s, sg_off, axis=axis)
        acc = oracle.add_to_subgrid(c, o, axis=axis, out=acc)
    fin = numpy.array([oracle.finish_subgrid(line, sg_off, sz)
                       for line in (acc if axis == 1 else acc.T)])
    if mask is not None:
        fin = fin * mask[None, :]
    ref = fin if axis == 1 else fin.T
    pc.close(out.cpu().numpy(), ref, rtol=1e-12,
             what=f"axis {axis}, facets {facet_steps}, sg_off {sg_off}, sz {sz}")


def facets_and_subgrids(cfg, n_facets, n_subgrids, seed):
    """A sparse facet set (facet offsets spread over the image, odd facet sizes included) and
    the first subgrids of the full cover."""
    rng = numpy.random.default_rng(seed)
    step = cfg.core.facet_off_step
    yB = cfg.max_facet_size
    n_steps = cfg.core.N // step
    facet_cfgs, facets = [], []
    for i in range(n_facets):
        off0 = ((3 * i) % n_steps - n_steps // 2) * step
        off1 = ((5 * i + 1) % n_steps - n_steps // 2) * step
        facet_cfgs.append(FacetConfig(off0, off1, yB))
        facets.append(pc.rand_c(rng, yB, yB))
    sgs = make_full_subgrid_cover(cfg)
    sgs = [sgs[(7 * i) % len(sgs)] for i in range(n_subgrids)]
    return facet_cfgs, facets, sgs


def dft_subgrids(cfg):
    """First, middle and last subgrid of the full cover among those whose masks are not empty
    (make_full_cover_config, like the reference's, gives every chunk but the first an empty mask
    when the chunk size is odd: 1536[1]-n768-384, xA = 345, see DESIGN.md section 7)."""
    def nonempty(mask):
        return mask is None or numpy.asarray(mask).any()

    sgs = [s for s in make_full_subgrid_cover(cfg) if nonempty(s.mask0) and nonempty(s.mask1)]
    return [sgs[0], sgs[len(sgs) // 2], sgs[-1]]


def forward_vs_oracle(cfg, n_facets=5, n_subgrids=5, seed=0, fused=True):
    """SwiftlyForward over a sparse facet set against the oracle's serial driver; returns
    (subgrid configs, results, reference)."""
    oracle = OracleCore(cfg.core.W, cfg.core.N, cfg.core.xM_size, cfg.core.yN_size)
    facet_cfgs, facets, sgs = facets_and_subgrids(cfg, n_facets, n_subgrids, seed)
    fwd = SwiftlyForward(cfg, list(zip(facet_cfgs, facets)), lru_forward=2)
    if fused:
        assert fwd._fused
    else:
        fwd._fused = False
    got = [fwd.get_subgrid_task(sg).result() for sg in sgs]
    ref = forward_reference_order(
        oracle, facets, [(c.off0, c.off1) for c in facet_cfgs], [(s.off0, s.off1) for s in sgs],
        cfg.max_subgrid_size, subgrid_masks=[(s.mask0, s.mask1) for s in sgs])
    scale = max(numpy.abs(r).max() for r in ref)
    for i, (a, b) in enumerate(zip(got, ref)):
        err = numpy.abs(a - b).max()
        assert err <= 1e-12 * scale, f"subgrid {i}: max err {err:.3e} vs scale {scale:.3e}"
    return sgs, got, ref
