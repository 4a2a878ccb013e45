"""
The host tier on the host-emulated kernels (``tests/host_tier_cases.py``): ``extract_columns``
(K2) and ``fold_column`` on ``m``-row rings, bitwise equal to the whole facet arrays in every K2
form the emulator reaches, and ``SwiftlyForward`` / ``SwiftlyBackward`` in the host tier bitwise
equal to the device tier; the tier chosen from the device budget.
"""

import pytest

from ska_sdp_distributed_fourier_transform_b200 import (
    SwiftlyBackward,
    SwiftlyForward,
    device_tier_bytes,
    make_full_facet_cover,
)
from ska_sdp_distributed_fourier_transform_b200.swift_configs import SWIFT_CONFIGS
from tests import host_tier_cases as hc
from tests import k2_cases as kc
from tests.emu_support import emu_core_class
from tests.test_emu_k2_forms import small_pair

make_config = hc.config_factory(lambda W, N, xM, yN: emu_core_class()(W, N, xM, yN))

# (yN, facet sizes, sg_variant, force_split, kernel of the launch)
K2_FORMS = [
    (256, [208, 200], 0, 0, kc.LINE),
    (640, [448, 440], 0, 0, kc.SPLIT_F),
    (1024, [704, 704], 0, 0, kc.TMA),       # swizzled tensor loads
    (1024, [703, 704], 0, 0, kc.TMA),       # linear bulk copies
    (1024, [704, 704], 6, 0, kc.TMA),       # linear staging selected
    (512, [256, 256], 0, 1, kc.TMA_SPLIT),  # the forced split forms at yN = 512
    (512, [256, 256], 0, 2, kc.TMA4),
    (512, [256, 256], 0, 3, kc.DIF),
    (512, [256, 256], 0, 4, kc.PARK_DIF),
    (512, [256, 256], 0, 5, kc.PARK_DIT),
    (512, [256, 256], 0, 6, kc.PARK_SKEW),
    (16384, [8192], 0, 0, kc.TMA4),
]


def _id(form):
    yN, sizes, variant, force_split, kernel = form
    return f"{yN}-{sizes[0]}-{sizes[-1]}-v{variant}-fs{force_split}-{kc.KERNEL_NAMES[kernel]}"


@pytest.mark.parametrize("form", K2_FORMS, ids=_id)
def test_emu_k2_ring_forms(form):
    """Wrapping windows, negative and >= N subgrid offsets, a ring slid by one column and, at
    yN = 1024, a capped grid: every call in the expected form, bitwise equal to the whole facets."""
    yN, sizes, variant, force_split, kernel = form
    core, oracle = small_pair(yN)
    offs = kc.facet_offsets(core)[:len(sizes)]
    sgs = kc.subgrid_offsets(core)
    assert kc.window_wraps(core, oracle, sgs[0]) and kc.window_wraps(core, oracle, sgs[1])
    step = (core.xM_yN_size // 2) * core.subgrid_off_step  # a column half a window wide
    cases = [dict(sg_off0=sgs[0]), dict(sg_off0=sgs[1]),
             dict(sg_off0=sgs[0] + step, prev_off0=sgs[0])]
    if yN == 1024 and variant == 0:
        cases.append(dict(sg_off0=sgs[2], cap=3))
    if yN == 16384:
        cases = cases[2:]
    for k, case in enumerate(cases):
        got = hc.k2_ring_case(core, oracle, sizes, offs, variant=variant, force_split=force_split,
                              seed=k, **case)
        assert got[0] == kernel, (case, got)


@pytest.mark.parametrize("yN,force_split", [(256, 0), (640, 0), (1024, 0), (512, 1)])
def test_emu_fold_ring(yN, force_split):
    core, oracle = small_pair(yN)
    sizes = [yN * 3 // 4, yN * 3 // 4 - 1]
    offs = kc.facet_offsets(core)[1:]
    sgs = kc.subgrid_offsets(core)
    step = (core.xM_yN_size // 2) * core.subgrid_off_step
    want = None
    for k, case in enumerate([dict(sg_off0=sgs[0]), dict(sg_off0=sgs[1]),
                              dict(sg_off0=sgs[0] + step, prev_off0=sgs[0]),
                              dict(sg_off0=sgs[2], cap=2)]):
        got = hc.fold_ring_case(core, oracle, sizes, offs, force_split=force_split, seed=k, **case)
        want = want or got[0]
        assert got[0] == want and got[0] in (kc.LINE, kc.SPLIT_LINE, kc.SPLIT_F), got


def test_emu_ring_rejects_other_row_counts():
    hc.ring_rejects(*small_pair(1024))


TIER_CASES = [  # (geometry, shuffled, lru, facets per K2 batch)
    ("1k[1]-n512-256", False, 1, 8),
    ("1k[1]-n512-256", True, 3, 4),
    ("1k[1]-n512-256", False, 3, 2),
    ("1280[1]-n640-320", False, 1, 4),
    ("1280[1]-n640-320", True, 3, 8),
    ("1k[1]-n512-256-sparse", False, 1, 2),
    ("1k[1]-n512-256-sparse", True, 3, 3),
]


@pytest.mark.parametrize("case", TIER_CASES,
                         ids=lambda c: f"{c[0]}-shuffle{int(c[1])}-lru{c[2]}-b{c[3]}")
def test_emu_host_tier_equals_device_tier(case):
    name, shuffle, lru, batch = case
    hc.case_tiers(make_config, name, shuffle=shuffle, lru=lru, batch=batch)


def test_emu_tier_selection():
    """A budget below the estimate selects the host tier, the default budget the device tier."""
    cfg = make_config(**hc.params("1k[1]-n512-256"))
    facet_cfgs = make_full_facet_cover(cfg)
    tasks = [(fc, None) for fc in facet_cfgs]
    need_f = device_tier_bytes("forward", 512, 128, [416] * 9, 1, 3, 228)
    need_b = device_tier_bytes("backward", 512, 128, [416] * 9, 1)
    assert not SwiftlyForward(cfg, tasks).host_tier
    assert not SwiftlyForward(cfg, tasks, device_budget=need_f).host_tier
    assert SwiftlyForward(cfg, tasks, device_budget=need_f - 1).host_tier
    assert not SwiftlyBackward(cfg, facet_cfgs).host_tier
    assert not SwiftlyBackward(cfg, facet_cfgs, device_budget=need_b).host_tier
    assert SwiftlyBackward(cfg, facet_cfgs, device_budget=need_b - 1).host_tier


GiB = 1 << 30


def _estimates(name, block=None, lru=1):
    p = SWIFT_CONFIGS[name]
    yN, yB, xA = p["yN_size"], p["yB_size"], p["xA_size"]
    m = p["xM_size"] * yN // p["N"]
    n = block or -(-p["N"] // yB)
    return (device_tier_bytes("forward", yN, m, [yB] * n * n, lru, n, xA),
            device_tier_bytes("backward", yN, m, [yB] * n * n, lru))


def test_device_tier_estimate_pinned():
    """The estimate at the benchmark's workloads: cfg1-cfg5 (cfg4 and cfg5 as the benchmark's
    central blocks) stay in the device tier of an 80 GB H100; the full 8 x 8 cfg4 cover does not
    (128 GiB of prepared facets)."""
    assert _estimates("1k[1]-n512-256") == (44916736, 40108032)
    assert _estimates("8k[1]-n4k-2k") == (3422552064, 3 * GiB)
    assert _estimates("32k[1]-n8k-4k") == (43754979328, 40 * GiB)
    assert _estimates("64k[1]-n16k-4k", block=5) == (62713233408, 60397977600)
    assert _estimates("64k[1]-n16k-4k", block=4) == (40936407040, 36 * GiB)
    full = _estimates("64k[1]-n16k-4k")
    assert full == (157034741760, 144 * GiB)
    for name, block in [("1k[1]-n512-256", None), ("8k[1]-n4k-2k", None),
                        ("32k[1]-n8k-4k", None), ("64k[1]-n16k-4k", 5),
                        ("64k[1]-n16k-4k", 4)]:
        assert max(_estimates(name, block)) < 70 * GiB
    assert min(full) > 80 * GiB
