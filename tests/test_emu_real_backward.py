"""
The real-image backward transform on the host-emulated kernels (``tests/real_backward_cases.py``):
``merge_mirror_subgrid`` exactly against numpy and as the adjoint of ``mirror_subgrid``,
``finish_facet_real`` bitwise against ``finish_facet``, and ``SwiftlyBackward(real_image=True)``
at a full cover, a sparse facet list with shuffled subgrids, ``lru_backward=2``, the host tier,
an odd subgrid size and a forward-backward round trip, with the work it saves counted.
"""

import random

import numpy
import pytest

from ska_sdp_distributed_fourier_transform_b200 import (
    SwiftlyBackward,
    make_full_facet_cover,
    make_full_subgrid_cover,
)
from tests import host_tier_cases as hc
from tests import real_backward_cases as rb
from tests import real_image_cases as rc
from tests.emu_support import emu_core_class

make_config = hc.config_factory(lambda W, N, xM, yN: emu_core_class()(W, N, xM, yN))

# N = 1280, xA = 160: an 8 x 8 cover with masks; yN = 640 runs the split-F line kernels
COVER = "1280[1]-n640-256"
# (192, 384) family, odd xA = 345 (explicit unmasked configs)
ODD = "1536[1]-n768-384"
# yN = 512: direct line kernels, and the 2 x 256 split through force_split
DIRECT = "1k[1]-n512-256"


def _core(name=COVER):
    return make_config(**hc.params(name)).core


@pytest.mark.parametrize("sz", [8, 9, 160, 161])
def test_emu_merge_mirror_subgrid(sz):
    rb.merge_case(_core(), sz, seed=sz)


@pytest.mark.parametrize("layout,transposed_inputs,cap", [
    ("wide", False, 0), ("transposed", False, 0), ("own", True, 0), ("wide", True, 1),
    ("own", False, 2), ("transposed", True, 3)])
def test_emu_merge_mirror_subgrid_layouts(layout, transposed_inputs, cap):
    """Outputs inside wider arrays and transposed, transposed inputs, capped grids."""
    core = _core()
    for sz in (10, 13):
        rb.merge_case(core, sz, layout=layout, transposed_inputs=transposed_inputs, cap=cap,
                      seed=sz)


def test_emu_merge_mirror_subgrid_cfg4_size():
    """cfg4's subgrid size: sz = 2048 into a 2049 x 2049 output."""
    rb.merge_case(_core(), 2048, layout="wide")


def test_emu_merge_mirror_subgrid_rejects():
    rb.merge_rejects(_core())


@pytest.mark.parametrize("sz", [8, 9, 24, 31])
def test_emu_merge_is_adjoint_of_mirror(sz):
    rb.adjoint_case(_core(), sz, seed=sz)


@pytest.mark.parametrize("name,force_split", [(COVER, 0), (DIRECT, 0), (DIRECT, 1)],
                         ids=["split-F-640", "direct-512", "split-2x256"])
@pytest.mark.parametrize("axis", [0, 1])
def test_emu_finish_facet_real(name, force_split, axis):
    """Every length form, with and without a mask, into own, wide and transposed outputs; a
    capped grid."""
    core = _core(name)
    fs = hc.params(name)["yB"]
    for k, (masked, layout, cap) in enumerate([(True, "own", 0), (False, "wide", 0),
                                               (True, "transposed", 2)]):
        rb.finish_real_case(core, fs, axis, masked=masked, layout=layout, cap=cap,
                            force_split=force_split, seed=k)


def test_emu_finish_facet_real_rejects():
    rb.finish_real_rejects(_core())


def _cover(name=COVER, facet_offs=None, n_sources=5, seed=3):
    cfg = make_config(**hc.params(name))
    facet_cfgs = (make_full_facet_cover(cfg) if facet_offs is None
                  else rc.facet_block(cfg, facet_offs))
    sources = rc.point_sources(cfg.image_size, facet_cfgs, n_sources, seed)
    return cfg, facet_cfgs, sources


@pytest.mark.parametrize("budget", [None, 1], ids=["device", "host-tier"])
def test_emu_unpaired_is_re_of_default(budget):
    """Real mode through add_new_subgrid_task only: bitwise Re of the default mode."""
    cfg, facet_cfgs, sources = _cover()
    sg_cfgs = make_full_subgrid_cover(cfg)[::3]
    rb.unpaired_bitwise(cfg, facet_cfgs, sg_cfgs, rb.hermitian_subgrids(cfg, sg_cfgs, sources),
                        budget=budget)


def test_emu_full_cover():
    """8 x 8 cover in cover order: 34 of 64 subgrid sides, 30 merges, fold_column for 5 of 8
    columns; as accurate as the default mode against the analytic facets."""
    cfg, facet_cfgs, sources = _cover()
    sg_cfgs = make_full_subgrid_cover(cfg)
    assert len(sg_cfgs) == 64
    _, work, _, errs = rb.paired_case(cfg, facet_cfgs, sg_cfgs, sources)
    sides, merges, columns = rb.full_cover_work(8)
    assert (work.sides, work.merge, len(work.folds), len(set(work.folds))) == (
        sides, merges, columns, columns), (work.sides, work.merge, work.folds)
    print(f"\n{COVER}: errors {errs}")


@pytest.mark.parametrize("lru", [1, 2])
def test_emu_sparse_shuffled(lru):
    """A sparse facet list and the cover shuffled, lru 1 and 2."""
    cfg, facet_cfgs, sources = _cover(
        facet_offs=[(0, 0), (0, 440), (440, -440), (-440, 440), (-440, 0)], seed=5)
    sg_cfgs = make_full_subgrid_cover(cfg)
    random.Random(lru).shuffle(sg_cfgs)
    plan, _, _, _ = rb.paired_case(cfg, facet_cfgs, sg_cfgs, sources, lru=lru)
    assert len(plan) == 34


def test_emu_host_tier_equals_device_tier():
    """Real mode in the host tier (float64 facets in the pinned arena) gives the device tier's
    bits, and moves half the facet bytes back."""
    cfg, facet_cfgs, sources = _cover()
    sg_cfgs = make_full_subgrid_cover(cfg)
    subgrids = rb.hermitian_subgrids(cfg, sg_cfgs, sources)
    res = {}
    for budget in (None, 1):
        bwd = SwiftlyBackward(cfg, facet_cfgs, device_budget=budget, real_image=True)
        assert bwd.host_tier == (budget is not None)
        bwd.add_subgrid_tasks(sg_cfgs, subgrids)
        res[budget] = [numpy.asarray(t.result()) for t in bwd.finish()]
    for j, (a, b) in enumerate(zip(res[None], res[1])):
        assert a.dtype == b.dtype == numpy.float64
        assert numpy.array_equal(a, b), f"facet {j}: host tier differs from the device tier"
    # device -> host: the complex rows the rings write back, then 8 bytes per facet sample
    yB = sum(fc.size for fc in facet_cfgs)
    assert bwd.copied_bytes[1] == 16 * bwd.d2h_rows * yB + 8 * sum(
        fc.size * fc.size for fc in facet_cfgs)


def test_emu_odd_size_and_unpaired():
    """Odd xA = 345 (S = sz) with unmasked explicit configs: pairs, a self-mirrored config, a
    config whose mirror is missing, and a duplicate pair."""
    cfg, facet_cfgs, sources = _cover(ODD, [(0, 0), (0, 512), (512, -512), (-512, 0)], 5, 11)
    offs = [(0, 0), (192, 384), (-384, 96), (768, 0), (-192, -384), (384, -96), (96, 96),
            (192, 384), (-192, -384), (-96, 768), (96, -768), (768, 768)]
    sg_cfgs = rc.explicit_configs(cfg, offs)
    plan, _, _, _ = rb.paired_case(cfg, facet_cfgs, sg_cfgs, sources)
    assert plan == [(0, None), (1, 4), (2, 5), (3, None), (6, None), (7, 8), (9, 10),
                    (11, None)]


def test_emu_round_trip():
    """Forward real_image=True then backward real_image=True on real point-source facets: within
    the reference's round-trip bound wherever the default path meets it."""
    cfg = make_config(**hc.params(COVER))
    facet_cfgs = make_full_facet_cover(cfg)
    errs = rb.round_trip(cfg, facet_cfgs, make_full_subgrid_cover(cfg), [(1, 1, 0), (1, -37, 52)])
    print(f"\nround trip RMS: {errs}")


def test_emu_rejects():
    """Length mismatch raises ValueError; a core without the fused backward kernels raises
    NotImplementedError in real mode only."""
    cfg, facet_cfgs, _ = _cover()
    sg_cfgs = make_full_subgrid_cover(cfg)[:3]
    for real in (False, True):
        bwd = SwiftlyBackward(cfg, facet_cfgs, real_image=real)
        with pytest.raises(ValueError, match="subgrid"):
            bwd.add_subgrid_tasks(sg_cfgs, [None] * 2)
    cfg.core.fused_backward_supported = lambda: False
    with pytest.raises(NotImplementedError):
        SwiftlyBackward(cfg, facet_cfgs, real_image=True)
    SwiftlyBackward(cfg, facet_cfgs)  # the default mode is unaffected
