"""
GPU API parity: SwiftlyForward / SwiftlyBackward and the fused kernels on the B200
against the reference-generated golden fixture, the oracle and the reference's
round-trip criterion (tests/test_api.py:125, facet RMSE < 3e-10), plus the BASELINE
cfg2 geometry (N=8192) checked stage by stage against the oracle and -- for point
sources -- against the analytic DFT.
"""

import numpy
import pytest
import torch

from oracle.swiftly_oracle import OracleCore, forward_reference_order
from ska_sdp_distributed_fourier_transform_b200 import (
    FacetConfig,
    SubgridConfig,
    SwiftlyConfig,
    SwiftlyForward,
    check_subgrid,
    make_facet,
    make_full_facet_cover,
    make_full_subgrid_cover,
)
from tests import api_cases
from tests import parity_cases as pc

pytestmark = pytest.mark.gpu


def make_config(W, N, yB, yN, xA, xM, **kw):
    return SwiftlyConfig(W=W, fov=1.0, N=N, yB_size=yB, yN_size=yN, xA_size=xA, xM_size=xM)


def test_fused_ops_vs_oracle():
    api_cases.case_fused_ops_vs_oracle(make_config)


def test_fused_backward_ops_vs_oracle():
    api_cases.case_fused_backward_ops_vs_oracle(make_config)
    api_cases.case_fused_backward_ops_vs_oracle(make_config, W=11.0, N=1280, yB=440, yN=640,
                                                xA=280, xM=320)
    api_cases.case_fused_backward_ops_vs_oracle(make_config, N=8192, yB=2048, yN=4096, xA=1024,
                                                xM=2048)


@pytest.mark.parametrize("sg_variant", [0, 1, 2, 5, 16])
def test_forward_backward_vs_oracle_kernel_variants(sg_variant):
    """Every variant of the fused subgrid kernel against the oracle (N=2048, xA/xM = 0.5)."""
    api_cases.case_forward_backward_vs_oracle(make_config, sg_variant=sg_variant)


def test_many_sources():
    """More sources / groups than one fused launch carries (10 x 10 facets and beyond)."""
    api_cases.case_many_sources(make_config)


def test_forward_backward_vs_reference_golden(golden_2d):
    api_cases.case_forward_backward_vs_reference_golden(make_config, golden_2d)


def test_sparse_facets_shuffled_subgrids():
    api_cases.case_sparse_facets_shuffled_subgrids(make_config)


@pytest.mark.parametrize(
    "lru_forward,lru_backward,shuffle",
    [(1, 1, False), (2, 1, False), (1, 2, False), (1, 1, True), (2, 1, True), (1, 2, True)],
)
def test_api_round_trip(lru_forward, lru_backward, shuffle):
    api_cases.case_api_round_trip(make_config, lru_forward, lru_backward, shuffle)


def test_cfg2_forward_vs_oracle_and_dft():
    """BASELINE cfg2 (N=8192, m=1024, xM=2048): fused GPU pipeline vs the oracle on dense
    random facets (two facets, three subgrids) and vs the analytic DFT for point sources."""
    W, N, yB, yN, xA, xM = 13.5625, 8192, 2048, 4096, 1024, 2048
    cfg = make_config(W, N, yB, yN, xA, xM)
    oracle = OracleCore(W, N, xM, yN)
    rng = numpy.random.default_rng(123456789)
    offs = [(0, 0), (0, 2048)]
    facets = [pc.rand_c(rng, yB, yB) for _ in offs]
    sgs = [SubgridConfig(1024, 3072, xA), SubgridConfig(1024, 0, xA), SubgridConfig(-2048, 1024, xA)]
    fwd = SwiftlyForward(cfg, [(FacetConfig(o0, o1, yB), f) for (o0, o1), f in zip(offs, facets)])
    got = [fwd.get_subgrid_task(sg).result() for sg in sgs]
    ref = forward_reference_order(oracle, facets, offs, [(s.off0, s.off1) for s in sgs], xA)
    for a, b in zip(got, ref):
        assert numpy.abs(a - b).max() <= 1e-11 * numpy.abs(b).max()
    # point sources, full facet cover, a few subgrids: analytic truth
    sources = [(float(rng.random()), int(rng.integers(-N // 2, N // 2)),
                int(rng.integers(-N // 2, N // 2))) for _ in range(8)]
    facet_cfgs = make_full_facet_cover(cfg)
    fwd = SwiftlyForward(cfg, [(fc, make_facet(N, fc, sources)) for fc in facet_cfgs])
    sg_cfgs = make_full_subgrid_cover(cfg)
    for sg in (sg_cfgs[0], sg_cfgs[9], sg_cfgs[-1]):
        err = check_subgrid(N, sg, fwd.get_subgrid_task(sg).tensor, sources)
        assert err < 1e-13, err


def test_cfg3_forward_vs_oracle():
    """BASELINE cfg3 (N=32768, yN=8192: K2 as the direct 8192-point line kernel, m=1024,
    xM=4096) in 2-D: two dense facets x three subgrids through SwiftlyForward vs the oracle in
    the reference's call order, and point sources vs the analytic DFT."""
    W, N, yB, yN, xA, xM = 13.5625, 32768, 4096, 8192, 2048, 4096
    cfg = make_config(W, N, yB, yN, xA, xM)
    oracle = OracleCore(W, N, xM, yN)
    rng = numpy.random.default_rng(32768)
    offs = [(0, 4096), (-8192, 4096 * 5)]
    facets = [pc.rand_c(rng, yB, yB) for _ in offs]
    sgs = [SubgridConfig(2048, 6144, xA), SubgridConfig(2048, 0, xA),
           SubgridConfig(-4096, 2048 * 7, xA)]
    fwd = SwiftlyForward(cfg, [(FacetConfig(o0, o1, yB), f) for (o0, o1), f in zip(offs, facets)])
    got = [fwd.get_subgrid_task(sg).result() for sg in sgs]
    del fwd
    ref = forward_reference_order(oracle, facets, offs, [(s.off0, s.off1) for s in sgs], xA)
    for a, b in zip(got, ref):
        assert numpy.abs(a - b).max() <= 1e-11 * numpy.abs(b).max()
    del facets, ref, got
    torch.cuda.empty_cache()
    fcs = [FacetConfig(4096, 0, yB), FacetConfig(4096 * 3, 4096 * 6, yB)]
    sources = []
    for fc in fcs:
        for _ in range(5):
            l = (fc.off0 + int(rng.integers(-yB // 2, yB // 2)) + N // 2) % N - N // 2
            m_ = (fc.off1 + int(rng.integers(-yB // 2, yB // 2)) + N // 2) % N - N // 2
            sources.append((float(rng.random()) + 0.5, l, m_))
    fwd = SwiftlyForward(cfg, [(fc, make_facet(N, fc, sources)) for fc in fcs])
    sg_cfgs = make_full_subgrid_cover(cfg)
    scale = sum(s[0] for s in sources) / N**2
    for sg in (sg_cfgs[0], sg_cfgs[100], sg_cfgs[-1]):
        err = check_subgrid(N, sg, fwd.get_subgrid_task(sg).tensor, sources)
        assert err / scale < 1e-9, (err, scale)


def _sources_inside(rng, fcs, N, yB, per_facet):
    sources = []
    for fc in fcs:
        for _ in range(per_facet):
            l = (fc.off0 + int(rng.integers(-yB // 2, yB // 2)) + N // 2) % N - N // 2
            m_ = (fc.off1 + int(rng.integers(-yB // 2, yB // 2)) + N // 2) % N - N // 2
            sources.append((float(rng.random()) + 0.5, l, m_))
    return sources


def test_cfg5_sparse_facets_full_size():
    """BASELINE cfg5: the cfg4 geometry (N=65536) with 25 % of the facets -- the central 4 x 4
    block, offsets {0, 8192, 49152, 57344}^2 (SURVEY 8d) -- and the 7-facet disc cover the
    reference's demo builds (scripts/demo_sparse_facet.py:106-134).  Point sources inside the
    covered facets: every subgrid must equal the analytic DFT."""
    import os
    import sys

    W, N, yB, yN, xA, xM = 13.5625, 65536, 8192, 16384, 2048, 4096
    cfg = make_config(W, N, yB, yN, xA, xM)
    rng = numpy.random.default_rng(5)
    block = [0, 8192, 49152, 57344]
    fcs = [FacetConfig(a, b, yB) for a in block for b in block]
    sources = _sources_inside(rng, fcs[::3], N, yB, 2)
    scale = sum(s[0] for s in sources) / N**2
    # facets are built on demand (one 1 GiB host array at a time)
    fwd = SwiftlyForward(cfg, [(fc, (lambda fc=fc: make_facet(N, fc, sources))) for fc in fcs])
    sg_cfgs = make_full_subgrid_cover(cfg)
    for sg in (sg_cfgs[0], sg_cfgs[517], sg_cfgs[-1]):
        err = check_subgrid(N, sg, fwd.get_subgrid_task(sg).tensor, sources)
        assert err / scale < 1e-9, (err, scale)
    del fwd
    torch.cuda.empty_cache()
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                    "scripts"))
    from demo_sparse_facet import disc_cover_offsets  # pylint: disable=import-error

    offsets = disc_cover_offsets(N, yB, 2.12 * yB)
    assert len(offsets) == 7
    assert all(o0 % cfg.facet_off_step == 0 and o1 % cfg.facet_off_step == 0 for o0, o1 in offsets)
    fcs = [FacetConfig(o0, o1, yB) for o0, o1 in offsets]
    sources = _sources_inside(rng, fcs[:3], N, yB, 2)
    scale = sum(s[0] for s in sources) / N**2
    fwd = SwiftlyForward(cfg, [(fc, (lambda fc=fc: make_facet(N, fc, sources))) for fc in fcs])
    for sg in (sg_cfgs[31], sg_cfgs[600]):
        err = check_subgrid(N, sg, fwd.get_subgrid_task(sg).tensor, sources)
        assert err / scale < 1e-9, (err, scale)


def test_catalogue_config_round_trip():
    """A runnable entry of the reference catalogue through the full API (forward vs analytic
    DFT, backward vs the source list), and a non-power-of-two entry failing loudly."""
    from ska_sdp_distributed_fourier_transform_b200 import (
        SWIFT_CONFIGS, SwiftlyBackward, check_facet)
    from ska_sdp_distributed_fourier_transform_b200.swift_configs import runnable

    name = "4k[1]-n2k-512"
    params = SWIFT_CONFIGS[name]
    assert runnable(params)
    cfg = SwiftlyConfig(**params)
    N = cfg.image_size
    sources = [(1, 1, 0), (0.5, -200, 333)]
    facet_cfgs = make_full_facet_cover(cfg)
    sg_cfgs = make_full_subgrid_cover(cfg)
    fwd = SwiftlyForward(cfg, [(fc, make_facet(N, fc, sources)) for fc in facet_cfgs])
    bwd = SwiftlyBackward(cfg, facet_cfgs)
    for sg in sg_cfgs:
        task = fwd.get_subgrid_task(sg)
        assert check_subgrid(N, sg, task.tensor, sources) < 1e-12
        bwd.add_new_subgrid_task(sg, task)
    for fc, task in zip(facet_cfgs, bwd.finish()):
        assert check_facet(N, fc, task.result(), sources) < 1e-8
    assert all(runnable(c) for c in SWIFT_CONFIGS.values())
    # a non-power-of-two catalogue entry (yN = 3 * 256): unfused GPU path, analytic check
    params = SWIFT_CONFIGS["1536[1]-n768-512"]
    cfg3 = SwiftlyConfig(**params)
    N3 = cfg3.image_size
    facet_cfgs = make_full_facet_cover(cfg3)
    fwd = SwiftlyForward(cfg3, [(fc, make_facet(N3, fc, sources)) for fc in facet_cfgs])
    sgs = make_full_subgrid_cover(cfg3)
    for sg in (sgs[0], sgs[5], sgs[-1]):
        assert check_subgrid(N3, sg, fwd.get_subgrid_task(sg).tensor, sources) < 1e-12
    # a length this build has no kernel for (17 * 16) fails loudly
    from ska_sdp_distributed_fourier_transform_b200 import SwiftlyCoreB200
    bad = SwiftlyCoreB200(11.0, 544, 272, 272)
    with pytest.raises(NotImplementedError):
        bad.prepare_facet(numpy.zeros(100), 0, axis=0)


@pytest.mark.parametrize("sg_variant", [0, 17, 18, 19, 20, 15, 7])
def test_k2_kernel_forms_yN16384(sg_variant):
    """Every form of K2 at yN = 16384 against the oracle (prepare_facet(extract_from_facet)):
    0 / 20 = default (4 x 4096 with the L2 scratch and a CTA-wide combine), 19 = results parked
    per thread in L2-resident scratch, DIT within and across the two thread groups, store phases
    half a line apart, 18 = without the skew, 17 = DIF across the groups with 32-byte pair
    stores, 15 = DIF / DIT with the L2 scratch, 7 = 2 x 8192.  Rows staged by swizzled tensor loads (fs = 8192),
    by linear bulk copies (odd fs), rows longer than yN / 2, several lines per CTA; each launch
    asserts the kernel it recorded (tests/k2_cases.py::variant_case)."""
    from oracle.swiftly_oracle import OracleCore
    from tests import k2_cases

    W, N, yN, xM = 13.5625, 65536, 16384, 4096
    cfg = make_config(W, N, 8192, yN, 2048, xM)
    k2_cases.variant_case(cfg.core, OracleCore(W, N, xM, yN), sg_variant, seed=16384 + sg_variant)


def test_cfg4_full_size_properties():
    """BASELINE cfg4 geometry (N=65536, yN=16384 split kernels, m=1024, xM=4096) at full
    size through the fused pipeline: (1) point sources inside two facets -> the subgrids equal
    the analytic DFT (all other facets are empty, so the two-facet sum is the exact answer);
    (2) linearity of the whole transform on dense random facets."""
    W, N, yB, yN, xA, xM = 13.5625, 65536, 8192, 16384, 2048, 4096
    cfg = make_config(W, N, yB, yN, xA, xM)
    rng = numpy.random.default_rng(65536)
    fcs = [FacetConfig(0, 8192, yB), FacetConfig(57344, 8192, yB)]  # rows 0 and 7, column 1
    sources = []
    for fc in fcs:
        for _ in range(6):
            l = (fc.off0 + int(rng.integers(-yB // 2, yB // 2)) + N // 2) % N - N // 2
            m_ = (fc.off1 + int(rng.integers(-yB // 2, yB // 2)) + N // 2) % N - N // 2
            sources.append((float(rng.random()) + 0.5, l, m_))
    facets = [make_facet(N, fc, sources) for fc in fcs]
    assert abs(sum(f.sum() for f in facets) - sum(s[0] for s in sources)) < 1e-9
    fwd = SwiftlyForward(cfg, list(zip(fcs, facets)))
    sg_cfgs = make_full_subgrid_cover(cfg)
    for sg in (sg_cfgs[0], sg_cfgs[33], sg_cfgs[-1]):
        got = fwd.get_subgrid_task(sg).tensor
        err = check_subgrid(N, sg, got, sources)
        scale = sum(s[0] for s in sources) / N**2  # magnitude of the subgrid samples
        assert err / scale < 1e-9, (err, scale)
    del fwd
    torch.cuda.empty_cache()
    # linearity
    a, b = 0.75, -1.25 + 0.5j
    F1 = [pc.rand_c(rng, yB, yB) for _ in fcs]
    F2 = [pc.rand_c(rng, yB, yB) for _ in fcs]
    sg = sg_cfgs[40]

    def run(data):
        f = SwiftlyForward(cfg, list(zip(fcs, data)))
        out = f.get_subgrid_task(sg).tensor.clone()
        del f
        return out

    s1, s2 = run(F1), run(F2)
    s12 = run([a * x + b * y for x, y in zip(F1, F2)])
    ref = a * s1 + b * s2
    assert float((s12 - ref).abs().max() / ref.abs().max()) < 1e-12
