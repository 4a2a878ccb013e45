"""
GPU parity (the real gate): every primitive of ``SwiftlyCoreB200`` -- hand-written
CUDA behind the C ABI -- against the CPU oracle on seeded inputs, 1-D and 2-D,
both axes, odd sizes, negative / >= N offsets, host (numpy) and device (torch)
array modes, plus the reference-generated golden fixtures.
Tolerance: max|gpu - ref| <= 1e-12 * max|ref| (required: 1e-9).
"""

import numpy
import pytest

from tests import parity_cases as pc

pytestmark = pytest.mark.gpu

SMALL = dict(W=13.5625, N=256, xM=64, yN=128)
TESTP = dict(W=13.5625, N=1024, xM=256, yN=512)
CFG2 = dict(W=13.5625, N=8192, xM=2048, yN=4096)      # m = 1024
CFG3 = dict(W=13.5625, N=32768, xM=4096, yN=8192)     # m = 1024
CFG4 = dict(W=13.5625, N=65536, xM=4096, yN=16384)    # m = 1024, yN via 2 x 8192 split


@pytest.fixture(scope="module")
def core_cls():
    import torch

    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from ska_sdp_distributed_fourier_transform_b200 import SwiftlyCoreB200, _lib

    info = _lib.load().swiftly_b200_build_info()
    assert b"cuda sm_90a" in info and b"EMULATED" not in info
    return SwiftlyCoreB200


@pytest.mark.parametrize("p,yB,xA", [
    (SMALL, 96, 52), (SMALL, 95, 51), (TESTP, 416, 228), (TESTP, 415, 227),
    (CFG2, 2048, 1024), (CFG3, 4096, 2048), (CFG4, 8192, 2048), (CFG4, 8191, 2047),
])
def test_1d_chain(core_cls, p, yB, xA):
    core, oracle = pc.make_pair(core_cls, **p)
    rng = numpy.random.default_rng(7)
    Nx, Ny = core.subgrid_off_step, core.facet_off_step
    for f_off, s_off in [(0, 0), (3 * Ny, 5 * Nx), (-7 * Ny, -2 * Nx), (p["N"], p["N"] + Nx)]:
        pc.check_1d_chain(core, oracle, yB, xA, f_off, s_off, rng)


@pytest.mark.parametrize("axis", [0, 1])
@pytest.mark.parametrize("p,yB,other", [(SMALL, 95, 19), (TESTP, 416, 37), (CFG2, 2048, 9)])
def test_2d_axes(core_cls, p, yB, other, axis):
    core, oracle = pc.make_pair(core_cls, **p)
    rng = numpy.random.default_rng(8)
    Nx, Ny = core.subgrid_off_step, core.facet_off_step
    pc.check_2d_axis(core, oracle, yB, axis, other, 5 * Ny, -3 * Nx, rng)


def test_2d_subgrid_ops(core_cls):
    for p, xA in ((SMALL, 51), (TESTP, 228), (CFG2, 1024)):
        core, oracle = pc.make_pair(core_cls, **p)
        rng = numpy.random.default_rng(9)
        Nx = core.subgrid_off_step
        pc.check_2d_subgrid_ops(core, oracle, xA, (2 * Nx, -Nx), rng)


def test_errors(core_cls):
    core, _ = pc.make_pair(core_cls, **SMALL)
    pc.check_errors(core)
    with pytest.raises(ValueError):
        core_cls(13.5625, 1050, 256, 512)


def test_device_tensor_mode(core_cls):
    """torch CUDA tensors in/out (the fast path) give the same numbers as host mode."""
    import torch

    core, oracle = pc.make_pair(core_cls, **TESTP)
    rng = numpy.random.default_rng(11)
    Nx, Ny = core.subgrid_off_step, core.facet_off_step
    facet = pc.rand_c(rng, 416, 416)
    d_facet = torch.from_numpy(facet).cuda()
    f0, f1, s0, s1 = 2 * Ny, -3 * Ny, 5 * Nx, -4 * Nx
    d = core.prepare_facet(d_facet, f0, axis=0)
    assert isinstance(d, torch.Tensor) and d.is_cuda
    d = core.extract_from_facet(d, s0, axis=0)
    d = core.prepare_facet(d, f1, axis=1)
    d = core.extract_from_facet(d, s1, axis=1)
    acc = core.add_to_subgrid(d, f0, axis=0)
    acc = core.add_to_subgrid(acc, f1, axis=1)
    sg = core.finish_subgrid(acc, [s0, s1], 228)
    o = oracle.prepare_facet(facet, f0, axis=0)
    o = oracle.extract_from_facet(o, s0, axis=0)
    o = oracle.prepare_facet(o, f1, axis=1)
    o = oracle.extract_from_facet(o, s1, axis=1)
    oacc = oracle.add_to_subgrid(oracle.add_to_subgrid(o, f0, axis=0), f1, axis=1)
    osg = oracle.finish_subgrid(oacc, [s0, s1], 228)
    pc.close(acc.cpu().numpy(), oacc, what="device chain acc")
    pc.close(sg.cpu().numpy(), osg, rtol=1e-10, what="device chain subgrid")
    # backward on device.  At yB/yN = 0.8125 the chain amplifies fp64 rounding by ~4e6
    # (Fb reaches 4.9e3 per axis; a 1e-16 relative perturbation of the contribution moves
    # the facet by 4e-10), so the strict chain check uses the well-conditioned yB = 256
    # (the BASELINE geometries have yB/yN = 0.5) and the TEST_PARAMS round trip is judged
    # by the reference's own criterion in tests/test_gpu_api.py.
    yB = 256
    psg = core.prepare_subgrid(torch.from_numpy(osg).cuda(), (s0, s1))
    e = core.extract_from_subgrid(core.extract_from_subgrid(psg, f0, axis=0), f1, axis=1)
    a = core.add_to_facet(core.add_to_facet(e, s0, axis=0), s1, axis=1)
    fin = core.finish_facet(core.finish_facet(a, f0, yB, axis=0), f1, yB, axis=1)
    opsg = oracle.prepare_subgrid(osg, (s0, s1))
    oe = oracle.extract_from_subgrid(oracle.extract_from_subgrid(opsg, f0, axis=0), f1, axis=1)
    oa = oracle.add_to_facet(oracle.add_to_facet(oe, s0, axis=0), s1, axis=1)
    ofin = oracle.finish_facet(oracle.finish_facet(oa, f0, yB, axis=0), f1, yB, axis=1)
    pc.close(e.cpu().numpy(), oe, rtol=1e-11, what="device backward contribution")
    pc.close(fin.cpu().numpy(), ofin, rtol=1e-10, what="device backward chain")


def test_golden_1d(core_cls, golden_1d):
    g = golden_1d
    core, _ = pc.make_pair(core_cls, **TESTP)
    for idx, (yB, xA, f_off, s_off) in enumerate(g["cases"]):
        yB, xA, f_off, s_off = int(yB), int(xA), int(f_off), int(s_off)
        k = lambda name: g[f"c{idx}_{name}"]  # noqa: E731
        pc.close(core.prepare_facet(k("facet"), f_off, axis=0), k("prep"))
        assert numpy.array_equal(core.extract_from_facet(k("prep"), s_off, axis=0), k("contrib"))
        pc.close(core.add_to_subgrid(k("contrib"), f_off, axis=0), k("acc"))
        pc.close(core.finish_subgrid(k("acc"), s_off, xA), k("sg"))
        pc.close(core.prepare_subgrid(k("subgrid"), s_off), k("psg"))
        pc.close(core.extract_from_subgrid(k("psg"), f_off, axis=0), k("ext"))
        assert numpy.array_equal(core.add_to_facet(k("ext"), s_off, axis=0), k("accf"))
        pc.close(core.finish_facet(k("accf"), f_off, yB, axis=0), k("fin"))


def test_golden_2d(core_cls, golden_2d):
    g = golden_2d
    W, N, xM, yN, yB, xA = g["params"]
    core, _ = pc.make_pair(core_cls, float(W), int(N), int(xM), int(yN))
    yB, xA = int(yB), int(xA)
    f_off, s_off = (int(v) for v in g["prim_offs"])
    for axis in (0, 1):
        k = lambda name: g[f"ax{axis}_{name}"]  # noqa: E731
        pc.close(core.prepare_facet(k("facet"), f_off, axis=axis), k("prep"))
        assert numpy.array_equal(core.extract_from_facet(k("prep"), s_off, axis=axis), k("contrib"))
        pc.close(core.add_to_subgrid(k("contrib"), f_off, axis=axis, out=k("acc0").copy()), k("acc"))
        pc.close(core.finish_facet(k("prep"), f_off, yB - 1, axis=axis), k("fin"))
        pc.close(core.extract_from_subgrid(k("acc"), f_off, axis=axis), k("ext"))
        pc.close(core.add_to_facet(k("ext"), s_off, axis=axis, out=k("accf0").copy()), k("accf"))
    Nx = core.subgrid_off_step
    pc.close(core.finish_subgrid(g["fs_in"], [2 * Nx, -Nx], xA - 1), g["fs_out"])
    pc.close(core.prepare_subgrid(g["ps_in"], (2 * Nx, -Nx)), g["ps_out"])


NONPOW2 = [
    dict(W=11.0, N=1536, xM=512, yN=768),
    dict(W=9.25, N=1792, xM=256, yN=1792),
    dict(W=11.0, N=1280, xM=320, yN=640),
    dict(W=11.0, N=2304, xM=576, yN=1152),
    dict(W=11.0, N=114688, xM=512, yN=57344),   # catalogue 112k[1]-n56k-512: yN = 7 * 8192
]


@pytest.mark.parametrize("p", NONPOW2)
def test_non_power_of_two_lengths(core_cls, p):
    """F * 2^k FFT lengths (F = 3, 5, 7, 9) through the generic split-F kernel."""
    core, oracle = pc.make_pair(core_cls, **p)
    rng = numpy.random.default_rng(13)
    Nx, Ny = core.subgrid_off_step, core.facet_off_step
    yB = (p["yN"] * 11 // 16) | 1
    xA = (p["xM"] * 7 // 8) & ~1
    pc.check_1d_chain(core, oracle, yB, xA, 3 * Ny, -5 * Nx, rng)
    pc.check_1d_chain(core, oracle, yB - 1, xA - 1, -2 * Ny, 4 * Nx, rng)
    if p["yN"] < 4096:
        pc.check_2d_axis(core, oracle, yB, 0, 17, Ny, -Nx, rng)
        pc.check_2d_axis(core, oracle, yB, 1, 5, Ny, -Nx, rng)


def test_sdp_func_compat_adapter():
    """The ska_sdp_func-shaped adapter (last-axis transforms on strided views, in-place
    prepare_subgrid) called the way the reference's SwiftlyCoreFunc calls it
    (core.py:577-630, 684-929), against the oracle."""
    from ska_sdp_distributed_fourier_transform_b200.sdp_func_compat import Swiftly
    from oracle.swiftly_oracle import OracleCore
    from tests import subgrid_line_cases as slc

    W, N, xM, yN, yB, xA = 13.5625, 1024, 256, 512, 416, 228
    slc.sdp_func_adapter_vs_oracle(Swiftly(N, yN, xM, W), OracleCore(W, N, xM, yN), yB, xA)
