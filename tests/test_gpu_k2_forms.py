"""
``extract_columns`` (K2) on an H100 in every launch form the dispatch picks
(``tests/k2_cases.py``): every catalogue ``(yN, yB)`` at its smallest entry's own geometry, the
box layouts of the swizzled tensor loads, mixed facet sizes, row and output strides, wrapped
offsets, capped and overfull persistent grids, more than 64 facets, the staging limits at
``yN = 16384``, the selectable forms there, and an extended-precision spot check per form.
Every case asserts the launch record before it compares with the oracle.

Every test prints its worst errors (run pytest with -s to see them).
"""

import pytest
import torch

from oracle.swiftly_oracle import OracleCore
from ska_sdp_distributed_fourier_transform_b200.core import SwiftlyCoreB200
from tests import k2_cases as kc
from tests import length_cases as lc

pytestmark = pytest.mark.gpu

ROWS = kc.catalogue_rows()
_pairs = {}


def pair(geometry):
    """(core, oracle) of a geometry (W, N, xM, yN); one at a time, so that the scratch and
    tables of the previous plan are released before the next one is built."""
    if geometry not in _pairs:
        _pairs.clear()
        torch.cuda.empty_cache()
        _pairs[geometry] = (SwiftlyCoreB200(*geometry, device=0), OracleCore(*geometry))
    return _pairs[geometry]


def length_pair(yN):
    """The smallest catalogue geometry (by m, then N) with that yN."""
    return pair(min((g for (n, _), (_, g) in ROWS.items() if n == yN),
                    key=lambda g: (g[2] * g[3] // g[1], g[1])))


# every (yN, yB) staged by the TMA kernels, and one row of every generic kernel kind plus the
# yN = 16384 rows that miss the staging buffer; sorted by geometry so plans are built once
GPU_ROWS = sorted(
    list(kc.PINNED_TMA) + [(256, 208), (512, 416), (768, 528), (16384, 11264)],
    key=lambda r: (r[0], ROWS[r][1]))


@pytest.mark.parametrize("row", GPU_ROWS, ids=lambda r: f"{r[0]}-{r[1]}")
def test_gpu_catalogue_row(row):
    yN, yB = row
    core, oracle = pair(ROWS[row][1])
    n_facets = 3 if yN * yB <= 1 << 26 else 2
    err, got = kc.catalogue_row_case(core, oracle, yB, n_facets=n_facets, seed=yB)
    if row in kc.PINNED_TMA:
        kernel, box, boxes, in_cap, _ = kc.PINNED_TMA[row]
        assert got[:3] == (kernel, box, in_cap) and in_cap == boxes * box * 8
    else:
        assert got[:2] == kc.PINNED_GENERIC[yN][:2]
    print(f"\n({yN}, {yB}) m {core.xM_yN_size}: {kc.KERNEL_NAMES[got[0]]} {got}, "
          f"max rel err {err:.2e}")
    torch.cuda.empty_cache()


@pytest.mark.parametrize("yN", [1024, 2048, 4096, 8192, 16384])
def test_gpu_box_layouts(yN):
    """Every box layout that fits yN: default staging against the oracle, and the same bits with
    linear staging (sg_variant 6) and with a capped grid."""
    core, oracle = length_pair(yN)
    worst = 0.0
    for fs in kc.box_layouts(yN):
        if yN > 2048 and fs < 2048:
            continue  # the small layouts run at 1024 and 2048
        err, record, boxes = kc.box_layout_case(core, oracle, fs, seed=fs)
        worst = max(worst, err)
        print(f"\nyN {yN} fs {fs}: box {record[1]} x {boxes}, max rel err {err:.2e}", end="")
    print(f"\nyN {yN}: worst {worst:.2e}")


@pytest.mark.parametrize("cap", [0, 1, 3])
def test_gpu_mixed_sizes(cap):
    """[large, small, large] in one launch, uncapped and on 1 and 3 CTAs, whose walk crosses
    from a long row to a short one and back."""
    for yN in (1024, 8192, 16384) if cap == 3 else (1024, 8192):
        core, oracle = length_pair(yN)
        err = kc.mixed_case(core, oracle, cap=cap, seed=cap)
        print(f"\nmixed sizes yN {yN}, max_blocks {cap}: max rel err {err:.2e}")


def test_gpu_strides_outputs_offsets():
    core, oracle = length_pair(1024)
    errs = [kc.stride_case(core, oracle, 704, seed=1), kc.output_case(core, oracle, 704, seed=2),
            kc.offset_case(core, oracle, 832, seed=3)]
    core, oracle = length_pair(2048)
    errs += [kc.stride_case(core, oracle, 1824, seed=4), kc.offset_case(core, oracle, 1824, seed=5)]
    core, oracle = length_pair(8192)
    errs += [kc.stride_case(core, oracle, 7296, seed=6), kc.output_case(core, oracle, 7296, seed=7),
             kc.offset_case(core, oracle, 5632, seed=8)]
    print(f"\nstrides / outputs / offsets: max rel err {max(errs):.2e}")


def test_gpu_many_lines_and_facets():
    """64 facets of 128 lines on the 1056 CTAs of the yN = 1024 kernel (8192 lines); 67 facets:
    two launches, the record shows the 3-facet one."""
    core, oracle = length_pair(1024)
    m = core.xM_yN_size
    assert m == 128
    e1, got = kc.many_lines_case(core, oracle, 64, n_facets=64, seed=1)
    assert got == (kc.TMA, 8, 64, 1056)
    e2, got = kc.many_lines_case(core, oracle, 704, n_facets=67, seed=2)
    assert got == (kc.TMA, 88, 704, 3 * m)
    print(f"\n64 facets: max rel err {e1:.2e}; 67 facets: {e2:.2e}")


@pytest.mark.parametrize("fs", sorted(kc.boundary_sizes_16384()))
def test_gpu_staging_boundaries_yN16384(fs):
    """The facet sizes next to the staging limits at yN = 16384 (8192 swizzled, 10174 linear)
    and the catalogue's 11264, one (yN, fs) input at a time."""
    core, oracle = length_pair(16384)
    err = kc.boundary_case(core, oracle, fs, seed=fs)
    print(f"\nyN 16384 fs {fs}: {kc.boundary_sizes_16384()[fs]}, max rel err {err:.2e}")
    torch.cuda.empty_cache()


@pytest.mark.parametrize("variant", sorted(kc.VARIANT_KERNELS))
def test_gpu_variant_forms_yN16384(variant):
    core, oracle = length_pair(16384)
    err = kc.variant_case(core, oracle, variant, seed=variant)
    print(f"\nsg_variant {variant}: max rel err {err:.2e}")
    torch.cuda.empty_cache()


SPOTS = [  # (yN, fs, variant, layout, kernel)
    (1024, 704, 0, "contiguous", kc.TMA), (1024, 703, 0, "contiguous", kc.TMA),
    (2048, 1824, 0, "slice", kc.TMA), (4096, 2816, 0, "contiguous", kc.TMA),
    (8192, 7296, 0, "contiguous", kc.TMA), (16384, 8192, 0, "contiguous", kc.TMA4),
    (16384, 10174, 0, "contiguous", kc.TMA4), (16384, 8192, 7, "contiguous", kc.TMA_SPLIT),
    (16384, 8192, 15, "contiguous", kc.DIF), (16384, 8192, 17, "contiguous", kc.PARK_DIF),
    (16384, 10168, 17, "contiguous", kc.PARK_DIF2), (16384, 8192, 18, "contiguous", kc.PARK_DIT),
    (16384, 8192, 19, "contiguous", kc.PARK_SKEW),
]


@pytest.mark.parametrize("spot", SPOTS, ids=lambda s: f"{s[0]}-{s[1]}-{kc.KERNEL_NAMES[s[4]]}")
def test_gpu_extended_precision(spot):
    """Two rows per form against the centred DFT in extended precision at the sub-transform
    boundaries, the centre and random bins: error <= 1.5 eps log2(yN) of the line's RMS.  On an
    H100 80GB HBM3 (700 W) the forms reach 0.25 .. 0.60 (``k2_cases`` lists them)."""
    yN, fs, variant, layout, kernel = spot
    core, _ = length_pair(yN)
    got, ratio = kc.spot_check(core, fs, seed=fs, variant=variant, layout=layout)
    print(f"\n{kc.KERNEL_NAMES[got[0]]} yN {yN} fs {fs}: {ratio:.3f} eps log2(yN)")
    assert got[0] == kernel and (got[1] != 0) == (fs % 8 == 0 and fs <= 8192), got
    assert ratio <= lc.SPOT_BOUND, ratio
    torch.cuda.empty_cache()
