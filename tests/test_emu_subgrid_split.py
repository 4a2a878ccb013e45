"""
The fused subgrid split kernel (``swiftly_b200_split_subgrid_axis``: prepare_subgrid along one
axis, extract_from_subgrid per target, optionally add_to_facet) on the host-emulated kernels,
against the oracle, at every (m, xM) pair of the library, and SwiftlyBackward on top of it.
"""

import ctypes
import os
import re

import pytest
import torch

from ska_sdp_distributed_fourier_transform_b200 import _lib, api, core as core_mod
from ska_sdp_distributed_fourier_transform_b200.swift_configs import FUSED_FORWARD_PAIRS
from tests import catalogue_cases as cc
from tests import split_cases as sc
from tests.emu_support import emu_core_class

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "ska_sdp_distributed_fourier_transform_b200", "csrc")

# the N = 256 test geometry of the other emulated tests: (m, xM) = (32, 64)
N256 = (13.5625, 256, 96, 128, 52, 64)
# (m, xM) -> small plan: the catalogue families (tests/catalogue_cases.py), N = 256, and for every
# other pair of the library the smallest plan with that pair (N = 2 xM, yN = 2 m, yB = yN / 2) with
# a small subgrid size, so that the K4T lines of the chained and backward tests stay few
PLANS = dict(cc.SMALL)
PLANS[(32, 64)] = N256
for _m, _xM in FUSED_FORWARD_PAIRS:
    if (_m, _xM) not in PLANS:
        PLANS[(_m, _xM)] = (13.5625, 2 * _xM, _m, 2 * _m, min(_xM // 2, 128), _xM)
_cfgs = {}


def config(pair):
    if pair not in _cfgs:
        _cfgs[pair] = cc.make_config(emu_core_class(), PLANS[pair])
    return _cfgs[pair]


def _pairs_of(name, macro):
    with open(os.path.join(CSRC, name)) as f:
        text = f.read()
    body = re.search(r"#define " + macro + r"\(X\)((?:.*\\\n)*.*\n)", text).group(1)
    return {(int(a), int(b)) for a, b in re.findall(r"X\((\d+),\s*(\d+)\)", body)}


def test_split_kernel_pairs_are_the_forward_pairs():
    """The split kernel exists for exactly the pairs of the fused forward kernel, and the
    library reports it for each of them (and for nothing else)."""
    pairs = _pairs_of("dispatch_subgrid_split.cu", "SW_SPLIT_PAIRS")
    assert pairs == _pairs_of("dispatch_subgrid_axis.cu", "SW_SG_PAIRS")
    assert pairs == set(FUSED_FORWARD_PAIRS)
    core_cls = emu_core_class()
    for m, xM in sorted(pairs):
        c = core_cls(13.5625, 2 * xM, xM, 2 * m)
        assert c._lib.swiftly_b200_split_axis_supported(c._plan) == max(1, xM // m), (m, xM)
        assert c.split_axis_supported()
    c = core_cls(8.0, 512, 128, 64)  # m = 16: no fused kernel
    assert c.xM_yN_size == 16 and not c.split_axis_supported()


def test_split_symbols_exported():
    from tests.test_abi import declared_symbols

    syms = declared_symbols()
    for name in ("swiftly_b200_split_subgrid_axis", "swiftly_b200_split_axis_supported"):
        assert name in syms
        assert name in _lib.SYMBOLS
    lib = config((32, 64)).core._lib  # the emulated build exports them as well
    assert hasattr(lib, "swiftly_b200_split_subgrid_axis")


@pytest.mark.parametrize("pair", sorted(PLANS), ids=cc.pair_id)
@pytest.mark.parametrize("axis", [1, 0])
@pytest.mark.parametrize("mode", ["store", "add"])
def test_emu_split_axis(pair, axis, mode):
    """Odd and even subgrid sizes, subgrid / facet offsets below zero and at or above N, target
    counts that leave a partial last round, repeated and overlapping windows, two groups."""
    core = config(pair).core
    N, xM = core.N, core.xM_size
    fs, ss = core.facet_off_step, core.subgrid_off_step
    conc = max(1, xM // core.xM_yN_size)
    n_t = conc + 1  # one full round and a partial one (a single round at CONC 1: two rounds)
    f_offs = [0, fs, fs, -3 * fs, N + 2 * fs, -N - fs, 5 * fs, 2 * fs][:n_t]
    f_offs2 = [-fs, 7 * fs, 0]
    sc.split_vs_oracle(core, axis, mode, xM - 3, 5, [-5 * ss, N + 3 * ss], [f_offs, f_offs2],
                       seed=pair[1] + axis)
    sc.split_vs_oracle(core, axis, mode, xM // 2, 4, [N - ss], [[2 * fs]], seed=7)


@pytest.mark.parametrize("pair", sorted(PLANS), ids=cc.pair_id)
@pytest.mark.parametrize("axis", [1, 0])
def test_emu_split_shared_accumulators(pair, axis):
    """Several groups adding into the same accumulators in one launch."""
    sc.shared_accumulator_case(config(pair).core, axis, seed=3)


@pytest.mark.parametrize("pair", sorted(PLANS), ids=cc.pair_id)
def test_emu_split_two_axes_chained(pair):
    """K4T (axis 0 into strips) then K3T (axis 1 into column accumulators) against the oracle's
    2-D prepare_subgrid, extract_from_subgrid on both axes and add_to_facet."""
    core = config(pair).core
    fs, ss, N = core.facet_off_step, core.subgrid_off_step, core.N
    facets = [(0, 0), (0, 3 * fs), (-2 * fs, fs), (-2 * fs, -fs), (N + fs, 0)]
    sc.chained_2d_vs_oracle(core, config(pair).max_subgrid_size, (3 * ss, -2 * ss), facets, seed=5)


@pytest.mark.parametrize("mode", ["store", "add"])
def test_emu_split_more_targets_and_groups_than_one_launch(mode):
    """70 targets in one group and 18 groups: the library splits the job over launches."""
    core = config((32, 64)).core
    fs, ss = core.facet_off_step, core.subgrid_off_step
    sc.split_vs_oracle(core, 1, mode, 41, 3, [2 * ss], [[(k % 9 - 4) * fs for k in range(70)]],
                       seed=11, check_lines=[0, 2])
    sc.split_vs_oracle(core, 0, mode, 40, 3, [(g - 9) * ss for g in range(18)],
                       [[g * fs, -g * fs] for g in range(18)], seed=12)


@pytest.mark.parametrize("pair", sorted(PLANS), ids=cc.pair_id)
def test_emu_split_many_lines_per_cta(pair):
    """The grid capped at 3 CTAs: every CTA walks many lines (and groups)."""
    core = config(pair).core
    lib = core._lib
    lib.swiftly_b200_debug_max_blocks.argtypes = [ctypes.c_void_p, ctypes.c_int]
    lib.swiftly_b200_debug_max_blocks(core._plan, 3)
    try:
        fs, ss = core.facet_off_step, core.subgrid_off_step
        conc = max(1, core.xM_size // core.xM_yN_size)
        for axis in (1, 0):
            sc.split_vs_oracle(core, axis, "add", core.xM_size - 1, 13, [ss, -ss],
                               [[k * fs for k in range(conc + 1)], [fs]], seed=13 + axis)
    finally:
        lib.swiftly_b200_debug_max_blocks(core._plan, 0)


def test_emu_split_validation():
    core = config((32, 64)).core
    m, yN, xM = core.xM_yN_size, core.yN_size, core.xM_size
    sub = torch.zeros((5, xM), dtype=torch.complex128)
    with pytest.raises(ValueError, match="samples per line"):
        core.split_subgrid_axis([sub], 1, [0], [[(torch.zeros((5, m + 1), dtype=torch.complex128),
                                                  0)]], "store")
    with pytest.raises(ValueError, match="lines"):
        core.split_subgrid_axis([sub], 1, [0], [[(torch.zeros((4, m), dtype=torch.complex128),
                                                  0)]], "store")
    big = torch.zeros((5, xM + 1), dtype=torch.complex128)
    with pytest.raises(ValueError, match="exceeds"):
        core.split_subgrid_axis([big], 1, [0], [[(torch.zeros((5, m), dtype=torch.complex128),
                                                  0)]], "store")
    acc = torch.zeros((5, yN), dtype=torch.complex128)
    with pytest.raises(ValueError, match="distinct"):
        core.split_subgrid_axis([sub], 1, [0], [[(acc, 0), (acc, 0)]], "add")
    with pytest.raises(ValueError, match="same number of lines"):
        core.split_subgrid_axis([sub, sub[:4]], 1, [0, 0], [[], []], "store")
    with pytest.raises(ValueError, match="mode"):
        core.split_subgrid_axis([sub], 1, [0], [[]], "scatter")
    # the C entry point itself: host memory is refused
    ins = (_lib.Lines * 1)(_lib.Lines(sub.data_ptr(), 5, xM, xM, 1, _lib.HOST))
    offs = (ctypes.c_int64 * 1)(0)
    sizes = (ctypes.c_int32 * 1)(0)
    rc = core._lib.swiftly_b200_split_subgrid_axis(core._plan, ins, 1, offs, None, sizes, 0, None)
    assert rc == _lib.EINVAL and "device" in _lib.last_error(core._lib)


# ---------------------------------------------------------------------- SwiftlyBackward
BACKWARD_PAIRS = [(32, 64), (160, 320), (128, 1024)]  # N = 256, mixed radix, CONC 8


@pytest.mark.parametrize("pair", BACKWARD_PAIRS, ids=cc.pair_id)
@pytest.mark.parametrize("sparse", [False, True], ids=["full", "sparse"])
@pytest.mark.parametrize("lru", [1, 2])
def test_emu_backward_split_path(pair, sparse, lru, monkeypatch):
    """SwiftlyBackward on the split kernels (the primitive subgrid side is never called) against
    the oracle's serial driver, subgrids in shuffled order."""
    cfg = config(pair)
    for name in ("prepare_subgrid", "extract_from_subgrid", "subgrid_to_facets"):
        monkeypatch.setattr(type(cfg.core), name, _refuse(name))
    facet_cfgs, sgs, data = sc.backward_inputs(cfg, sparse, 6, seed=pair[1] + lru)
    assert api.SwiftlyBackward(cfg, facet_cfgs)._split
    sc.backward_vs_oracle(cfg, facet_cfgs, sgs, data, lru_backward=lru)


def _refuse(name):
    def fn(*_a, **_k):
        raise AssertionError(f"{name} called on the split backward path")

    return fn


@pytest.mark.parametrize("pair", sorted(PLANS), ids=cc.pair_id)
def test_emu_backward_split_every_pair(pair, monkeypatch):
    cfg = config(pair)
    for name in ("prepare_subgrid", "extract_from_subgrid", "subgrid_to_facets"):
        monkeypatch.setattr(type(cfg.core), name, _refuse(name))
    # (two subgrids, two facets: the oracle's 2-D prepare_subgrid at xM = 8192 and the emulated
    # fold of 2048 accumulator lines dominate; test_emu_backward_split_path varies the rest)
    facet_cfgs, sgs, data = sc.backward_inputs(cfg, True, 2, seed=1, n_facets=2)
    assert api.SwiftlyBackward(cfg, facet_cfgs)._split
    sc.backward_vs_oracle(cfg, facet_cfgs, sgs, data)


def test_emu_backward_unsupported_pair_keeps_the_primitive_chain(monkeypatch):
    """(m, xM) = (16, 128) has no split kernel: SwiftlyBackward runs prepare_subgrid /
    extract_from_subgrid / subgrid_to_facets as before."""
    plan = (8.0, 512, 48, 64, 80, 128)
    cfg = cc.make_config(emu_core_class(), plan)
    assert cfg.core.xM_yN_size == 16 and not cfg.core.split_axis_supported()
    calls = []
    real = core_mod.SwiftlyCoreB200.subgrid_to_facets

    def counting(self, *a, **k):
        calls.append(1)
        return real(self, *a, **k)

    monkeypatch.setattr(type(cfg.core), "subgrid_to_facets", counting)
    bwd = api.SwiftlyBackward(cfg, [])
    assert bwd._fused and not bwd._split
    facet_cfgs, sgs, data = sc.backward_inputs(cfg, True, 3, seed=2)
    sc.backward_vs_oracle(cfg, facet_cfgs, sgs, data)
    assert len(calls) == len(sgs)


def test_emu_split_null_targets_refused():
    """A NULL target table with targets in a group is an argument error, not a crash."""
    core = config((32, 64)).core
    sub = torch.zeros((5, 64), dtype=torch.complex128)
    ins = (_lib.Lines * 1)(_lib.Lines(sub.data_ptr(), 5, 64, 64, 1, _lib.DEVICE))
    offs = (ctypes.c_int64 * 1)(0)
    sizes = (ctypes.c_int32 * 1)(2)
    rc = core._lib.swiftly_b200_split_subgrid_axis(core._plan, ins, 1, offs, None, sizes, 0, None)
    assert rc == _lib.EINVAL and "NULL" in _lib.last_error(core._lib)


def test_split_launch_count():
    """split_launches (the benchmark's launch count) follows the library's packing: pieces of at
    most 64 targets, at most 16 pieces and 64 targets per launch."""
    assert core_mod.split_launches([5]) == 1
    assert core_mod.split_launches([70]) == 2
    assert core_mod.split_launches([2] * 18) == 2
    assert core_mod.split_launches([5] * 40) == 4  # 8 subgrids x 5 facet rows of 5 facets
    assert core_mod.split_launches([0, 3]) == 1


def test_emu_sharded_backward_split_world_one_queue():
    """SwiftlyBackwardSharded without a process group runs the split kernels, matches
    SwiftlyBackward, and its results pass through the task queue (queue_size bounds them)."""
    from ska_sdp_distributed_fourier_transform_b200.distributed import SwiftlyBackwardSharded

    cfg = config((32, 64))
    facet_cfgs, sgs, data = sc.backward_inputs(cfg, False, 5, seed=4)
    bwd = SwiftlyBackwardSharded(cfg, facet_cfgs, queue_size=3)
    assert bwd._split
    seen = []
    real = bwd._local.task_queue.process
    bwd._local.task_queue.process = lambda tasks: (seen.append(len(tasks)), real(tasks))
    bwd.add_subgrid_tasks(sgs, [torch.from_numpy(d) for d in data])
    assert len(seen) == len(sgs) and len(bwd._local.task_queue.pending) <= 3
    got = [t.result() for _, t in sorted(bwd.finish().items())]
    ref = api.SwiftlyBackward(cfg, facet_cfgs)
    for s, d in zip(sgs, data):
        ref.add_new_subgrid_task(s, torch.from_numpy(d))
    want = [t.result() for t in ref.finish()]
    for a, b in zip(got, want):
        assert abs(a - b).max() <= 1e-12 * abs(b).max()
