"""
Half rows of real images on the H100 (``tests/half_rows_cases.py``): K1, K2, the fold and the
finish bitwise against their full-row twins at the lengths the H100 runs (the TMA-staged K2 forms
at 1024 ... 8192 and the two-CTA cluster form at 16384 included), and ``half_rows=True`` of both
transforms against ``real_image=True`` alone at the full cfg2 cover and a 2 x 2 facet block of
cfg4 over all 32 x 32 subgrids.
"""

import pytest
import torch

from ska_sdp_distributed_fourier_transform_b200 import (
    make_facet,
    make_full_facet_cover,
    make_full_subgrid_cover,
)
from ska_sdp_distributed_fourier_transform_b200.core import SwiftlyCoreB200
from tests import half_rows_cases as hr
from tests import host_tier_cases as hc
from tests import k2_cases as kc
from tests import real_image_cases as rc

pytestmark = pytest.mark.gpu

make_config = hc.config_factory(SwiftlyCoreB200)
CFG2 = "8k[1]-n4k-2k"
CFG4 = "64k[1]-n16k-4k"
_cores = {}


def small(yN, m=64):
    if yN not in _cores:
        _cores[yN] = SwiftlyCoreB200(11.0, 2 * yN, 2 * m, yN)
    return _cores[yN]


@pytest.mark.parametrize("yN,fs,n_lines,form", [
    (4096, 2049, 64, kc.LINE),      # two-pass
    (16384, 8191, 40, kc.LINE),     # two-pass
    (4096, 2049, 5, kc.LINE),       # single pass, direct
    (16384, 8191, 5, kc.SPLIT_LINE),  # single pass, 2 x 8192
    (640, 255, 7, kc.SPLIT_F),      # single pass, split-F
])
def test_gpu_k1(yN, fs, n_lines, form):
    core = small(yN)
    rec = hr.k1_case(core, fs, n_lines, off=-3 * core.facet_off_step, wide=True)
    assert rec[0] == form, rec


@pytest.mark.parametrize("yN,form,cluster", [
    (1024, kc.TMA, 1), (2048, kc.TMA, 1), (4096, kc.TMA, 1), (8192, kc.TMA, 1),
    (16384, kc.TMA4, 2), (640, kc.SPLIT_F, 1)])
@pytest.mark.parametrize("kind", ["zero", "nyquist", "neither"])
def test_gpu_k2_default_forms(yN, form, cluster, kind):
    core = small(yN)
    sg_off0 = hr.window_kinds(core)[kind]
    offs = [0, -3 * core.facet_off_step, core.N + 5 * core.facet_off_step]
    rec, cl, rec_ref, cl_ref = hr.k2_case(core, [yN // 2, yN // 2 - 3, 24], offs, sg_off0,
                                          seed=yN)
    assert (rec[0], cl) == (form, cluster) and (rec, cl) == (rec_ref, cl_ref), (rec, cl)


def test_gpu_k2_16384_staging_limit_and_fallback():
    """At yN = 16384: facets too long to stage run the generic 2 x 8192 line kernel; an odd
    capped grid cannot be paired and runs the single-CTA 4 x Q form."""
    core = small(16384)
    rec, _, rec_ref, _ = hr.k2_case(core, [16383, 100], [0, 3], 0)
    assert rec[0] == kc.SPLIT_LINE and rec == rec_ref, rec
    rec, cl, rec_ref, _ = hr.k2_case(core, [8192, 4000], [0, 3], core.N // 2, cap=5)
    assert (rec[0], cl, rec[3]) == (kc.TMA4, 1, 5) and rec == rec_ref, rec


@pytest.mark.parametrize("yN", [4096, 16384, 640])
def test_gpu_fold(yN):
    core = small(yN)
    N, step = core.N, core.subgrid_off_step
    for sg_off0 in (0, step, N // 2, N // 4 + step):
        runs = hr.fold_case(core, [yN // 2, yN - 1, 31], [0, -2 * core.facet_off_step, 5],
                            sg_off0, masked=(1,), seed=sg_off0)
        assert any(p == 2 for _, _, p in runs) == hr.straddles(core, sg_off0), runs


@pytest.mark.parametrize("yN,form", [(4096, kc.LINE), (16384, kc.SPLIT_LINE), (640, kc.SPLIT_F)])
@pytest.mark.parametrize("masked", [True, False])
def test_gpu_finish(yN, form, masked):
    rec = hr.finish_case(small(yN), yN // 2 + 3, masked=masked)
    assert rec[0] == form, rec


def test_gpu_finish_rejects():
    hr.finish_rejects(small(4096))


def test_gpu_cfg2_cover():
    cfg = make_config(**hc.params(CFG2))
    facet_cfgs = make_full_facet_cover(cfg)
    sources = rc.point_sources(cfg.image_size, facet_cfgs, 5, 3)
    sg_cfgs = make_full_subgrid_cover(cfg)
    print(f"\nforward {hr.forward_case(cfg, facet_cfgs, sg_cfgs, sources, lru=2)}")
    print(f"backward {hr.backward_case(cfg, facet_cfgs, sg_cfgs, sources, lru=2)}")
    print(f"round trip {hr.round_trip(cfg, facet_cfgs, sg_cfgs, sources)}")


def test_gpu_api_rejects():
    cfg = make_config(**hc.params(CFG2))
    facet_cfgs = make_full_facet_cover(cfg)[:2]
    sources = rc.point_sources(cfg.image_size, facet_cfgs, 2, 1)
    hr.api_rejects(cfg, facet_cfgs, sources)
    facets = [make_facet(cfg.image_size, fc, sources).real for fc in facet_cfgs]
    host = [torch.empty((cfg.core.half_rows, fc.size), dtype=torch.complex128)
            for fc in facet_cfgs]
    with pytest.raises(NotImplementedError, match="device tier"):
        hr.SwiftlyForward(cfg, list(zip(facet_cfgs, facets)), real_image=True, half_rows=True,
                          bf_f_buffers=host)


def test_gpu_cfg4_block():
    """A 2 x 2 cfg4 facet block over all 32 x 32 subgrids, both directions, against full-row
    real mode."""
    cfg = make_config(**hc.params(CFG4))
    facet_cfgs = hc.facet_configs(cfg, CFG4, 2)
    sources = rc.point_sources(cfg.image_size, facet_cfgs, 5, 7)
    facets = [make_facet(cfg.image_size, fc, sources).real for fc in facet_cfgs]
    sg_cfgs = make_full_subgrid_cover(cfg)
    assert len(sg_cfgs) == 1024
    print(f"\nforward {hr.forward_lockstep(cfg, facet_cfgs, facets, sg_cfgs, sources)}")
    del facets
    gen = torch.Generator(device="cuda").manual_seed(31)
    inputs = [torch.randn((2048, 2048), dtype=torch.complex128, device="cuda", generator=gen)
              for _ in range(16)]
    errs = hr.backward_case(cfg, facet_cfgs, sg_cfgs, None,
                            subgrids=[inputs[i % 16] for i in range(1024)])
    print(f"backward {errs}")
