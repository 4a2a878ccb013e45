"""
Half rows of real images on the host-emulated kernels (``tests/half_rows_cases.py``): K1, K2, the
fold and the finish bitwise against their full-row twins in every form the default dispatch
selects at the emulated lengths, and ``half_rows=True`` of both transforms against
``real_image=True`` alone.
"""

import random

import pytest

from ska_sdp_distributed_fourier_transform_b200 import (
    make_full_facet_cover,
    make_full_subgrid_cover,
)
from tests import half_rows_cases as hr
from tests import host_tier_cases as hc
from tests import k2_cases as kc
from tests import real_image_cases as rc
from tests.emu_support import emu_core_class

make_config = hc.config_factory(lambda W, N, xM, yN: emu_core_class()(W, N, xM, yN))

# N = 1280, yN = 640 (split-F line kernels, generic K2), an 8 x 8 cover with masks
COVER = "1280[1]-n640-256"
_cores = {}


def small(yN, m=16):
    """Emulated core with N = 2 yN, xM = 2 m."""
    if yN not in _cores:
        _cores[yN] = emu_core_class()(11.0, 2 * yN, 2 * m, yN)
    return _cores[yN]


# ---------------------------------------------------------------------- K1
@pytest.mark.parametrize("yN,fs,n_lines,variant,force_split,form", [
    (512, 301, 40, 0, 0, kc.LINE),      # two-pass
    (512, 300, 70, 10, 0, kc.LINE),     # two-pass, ragged column tiles (sg_variant 10)
    (128, 77, 6, 0, 0, kc.LINE),        # single pass, direct
    (512, 201, 5, 0, 1, kc.SPLIT_LINE),  # single pass, 2 x 256 (the 16384 split's twin)
    (640, 255, 7, 0, 0, kc.SPLIT_F),    # single pass, split-F
])
def test_emu_k1(yN, fs, n_lines, variant, force_split, form):
    core = small(yN)
    for off, wide in ((0, False), (-5 * core.facet_off_step, True),
                      (core.N + 3 * core.facet_off_step, False)):
        rec = hr.k1_case(core, fs, n_lines, off=off, wide=wide, variant=variant,
                         force_split=force_split, seed=fs + n_lines)
        assert rec[0] == form, rec


def test_emu_k1_axis1():
    rec = hr.k1_case(small(128), 77, 5, axis=1, off=3, wide=True)
    assert rec[0] == kc.LINE


# ---------------------------------------------------------------------- K2
@pytest.mark.parametrize("yN,force_split,form,cluster", [
    (128, 0, kc.TMA, 1),
    (512, 0, kc.TMA, 1),
    (512, 1, kc.TMA_SPLIT, 1),   # 2 x 256, the 2 x 8192 twin
    (512, 2, kc.TMA4, 2),        # 4 x 128 on two-CTA clusters, the default at 16384
    (512, 7, kc.TMA4, 1),        # its single-CTA fallback
    (640, 0, kc.SPLIT_F, 1),     # generic: SplitFKernel
])
@pytest.mark.parametrize("kind", ["zero", "nyquist", "neither"])
def test_emu_k2_forms(yN, force_split, form, cluster, kind):
    core = small(yN)
    sg_off0 = hr.window_kinds(core)[kind]
    offs = [0, -3 * core.facet_off_step, core.N + 5 * core.facet_off_step]
    for prewindowed in (True, False):
        rec, cl, rec_ref, cl_ref = hr.k2_case(core, [yN // 2, yN - 1, 24], offs, sg_off0,
                                              prewindowed=prewindowed, force_split=force_split,
                                              seed=yN + force_split)
        assert (rec[0], cl) == (form, cluster), (rec, cl)
        assert (rec, cl) == (rec_ref, cl_ref)


@pytest.mark.parametrize("force_split", [3, 4, 5, 6])
def test_emu_k2_ignores_debug_forms(force_split):
    """The debug-selectable forms have no half instantiation: the single-CTA 4 x Q form runs."""
    core = small(512)
    rec, cl, rec_ref, _ = hr.k2_case(core, [300, 200], [0, 7], 0, force_split=force_split,
                                     ref_hooks=(0, 7))
    assert (rec[0], cl) == (kc.TMA4, 1) and rec == rec_ref, rec


def test_emu_k2_linear_staging_and_cap():
    """Facets of no whole 128-byte chunks stage linearly; a capped grid walks several lines."""
    core = small(512)
    rec, _, rec_ref, _ = hr.k2_case(core, [301, 77], [0, 3], core.N // 2, cap=3)
    assert rec[0] == kc.TMA and rec[1] == 0 and rec[3] == 3, rec
    rec, _, _, _ = hr.k2_case(core, [304, 80], [0, 3], 0, cap=5)
    assert rec[0] == kc.TMA and rec[1] > 0 and rec[3] == 5, rec


def test_emu_k2_generic_line():
    """yN = 256 has no TMA instantiation on the emulator: LineKernel on the half op."""
    core = small(256)
    rec, _, rec_ref, _ = hr.k2_case(core, [100, 255], [0, 5], 0)
    assert rec[0] == kc.LINE and rec == rec_ref


def test_emu_k2_67_facets():
    """67 facets: two launches."""
    core = small(128)
    hr.k2_case(core, [60 + (j % 7) for j in range(67)], [j - 30 for j in range(67)], 0)


# ---------------------------------------------------------------------- fold
@pytest.mark.parametrize("yN,force_split", [(128, 0), (512, 0), (512, 1), (640, 0)])
def test_emu_fold(yN, force_split):
    core = small(yN)
    N, step = core.N, core.subgrid_off_step
    offs = [0, -2 * core.facet_off_step, 5]
    cases = {"central": 0, "next": step, "nyquist": N // 2, "far": N // 4 + step}
    for name, sg_off0 in cases.items():
        runs = hr.fold_case(core, [yN // 2, yN - 1, 31], offs, sg_off0, masked=(1,),
                            force_split=force_split, cap=7, seed=sg_off0)
        shared = hr.straddles(core, sg_off0)
        assert any(p == 2 for _, _, p in runs) == shared, (name, runs)
        if name in ("central", "nyquist"):
            assert shared, (name, runs)
        if name == "far":
            assert runs == [(0, core.xM_yN_size, 1)], runs


# ---------------------------------------------------------------------- finish
@pytest.mark.parametrize("yN,force_split,form", [
    (128, 0, kc.LINE), (512, 0, kc.LINE), (512, 1, kc.SPLIT_LINE), (640, 0, kc.SPLIT_F)])
@pytest.mark.parametrize("masked", [True, False])
def test_emu_finish(yN, force_split, form, masked):
    rec = hr.finish_case(small(yN), yN // 2 + 3, masked=masked, force_split=force_split)
    assert rec[0] == form, rec


def test_emu_finish_rejects():
    hr.finish_rejects(small(128))
    hr.odd_rejects(emu_core_class()(11.0, 1280, 256, 5))


# ---------------------------------------------------------------------- API
def _cover(facet_offs=None, n_sources=5, seed=3):
    cfg = make_config(**hc.params(COVER))
    facet_cfgs = (make_full_facet_cover(cfg) if facet_offs is None
                  else rc.facet_block(cfg, facet_offs))
    sources = rc.point_sources(cfg.image_size, facet_cfgs, n_sources, seed)
    return cfg, facet_cfgs, sources


def test_emu_api_full_cover():
    cfg, facet_cfgs, sources = _cover()
    sg_cfgs = make_full_subgrid_cover(cfg)
    errs = hr.forward_case(cfg, facet_cfgs, sg_cfgs, sources)
    print(f"\nforward: {errs}")
    errs = hr.backward_case(cfg, facet_cfgs, sg_cfgs, sources)
    print(f"backward: {errs}")


def test_emu_api_sparse_shuffled_lru2():
    cfg, facet_cfgs, sources = _cover(
        facet_offs=[(0, 0), (0, 440), (440, -440), (-440, 440), (-440, 0)], seed=5)
    sg_cfgs = make_full_subgrid_cover(cfg)
    random.Random(2).shuffle(sg_cfgs)
    hr.forward_case(cfg, facet_cfgs, sg_cfgs, sources, lru=2)
    hr.backward_case(cfg, facet_cfgs, sg_cfgs, sources, lru=2)


def test_emu_api_round_trip():
    cfg, facet_cfgs, sources = _cover()
    errs = hr.round_trip(cfg, facet_cfgs, make_full_subgrid_cover(cfg), sources)
    print(f"\nround trip: {errs}")


def test_emu_api_rejects():
    cfg, facet_cfgs, sources = _cover()
    hr.api_rejects(cfg, facet_cfgs, sources)
