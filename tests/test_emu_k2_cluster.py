"""
``extract_columns`` (K2) at ``yN = 4 Q`` on two-CTA clusters (``ExtractColumnsClusterKernel``,
the default form at ``yN = 16384``; ``force_split`` 2 at ``yN = 512`` on the emulated library)
against the single-CTA form (``ExtractColumnsTma4Kernel``, ``sg_variant`` 26 / ``force_split`` 7).
Both record launch code 10 on the same grid; ``swiftly_b200_debug_last_cluster`` tells them apart.
The same bits on every case, raw and pre-windowed, on capped grids (an even cap pairs, an odd one
runs the single-CTA form), over more facets than one launch takes, at the staging limits, and in
extended precision.

The emulator co-schedules the CTAs of a cluster, maps the partner's shared memory, provides the
cluster barrier and delivers a multicast to each CTA's bulk-copy barrier
(``tests/emu/emu_cluster.h``); ``test_cluster_protocol_reports_misuse`` checks its protocol errors.
"""

import ctypes
import os
import subprocess

import numpy
import pytest

from tests import k2_cases as kc
from tests import length_cases as lc
from tests.test_emu_k2_forms import small_pair

HERE = os.path.dirname(os.path.abspath(__file__))
TMA4_VARIANT = 26  # sg_variant: ExtractColumnsTma4Kernel, the single-CTA form


def last_cluster(core):
    """CTAs per cluster of the last recorded launch."""
    fn = core._lib.swiftly_b200_debug_last_cluster  # pylint: disable=protected-access
    fn.argtypes, fn.restype = [ctypes.c_void_p], ctypes.c_int
    return fn(core._plan)  # pylint: disable=protected-access


def _both(core, oracle, sizes, offs, sg, *, yN, cap=0, **kw):
    """The cluster form and the single-CTA form on the same call: same bits.  Returns the two
    launch records."""
    twin = dict(force_split=2) if yN == 512 else {}
    single = dict(force_split=7) if yN == 512 else dict(variant=TMA4_VARIANT)
    a, _, got_a = kc.run(core, oracle, sizes, offs, sg, cap=cap, what="cluster form", **twin, **kw)
    cluster = last_cluster(core)
    b, _, got_b = kc.run(core, oracle, sizes, offs, sg, cap=cap, what="single-CTA form",
                         **single, **kw)
    assert got_b == got_a and got_b[0] == kc.TMA4 and last_cluster(core) == 1, got_b
    for x, y in zip(a, b):
        assert numpy.array_equal(x, y), "the cluster form changes the bits"
    return got_a, cluster


@pytest.mark.parametrize("yN", [512, 16384])
def test_emu_cluster_bitwise(yN):
    """Raw and pre-windowed rows, swizzled and linear staging (an odd size), uncapped, on capped
    grids of 2 CTAs (one cluster) and of 1 and 3 CTAs (odd: the single-CTA form)."""
    core, oracle = small_pair(yN)
    m, half = core.xM_yN_size, yN // 2
    step, sg = core.facet_off_step, kc.subgrid_offsets(core)
    for k, (sizes, prewindowed, cap) in enumerate([
            ([half, half], False, 0), ([half, half - 64], True, 0), ([half - 1, half + 8], False, 3),
            ([half, half], True, 2), ([half, half], False, 1)]):
        got, cluster = _both(core, oracle, sizes, [step, -2 * step], sg[k % len(sg)], yN=yN,
                             cap=cap, prewindowed=prewindowed, seed=k)
        assert got[3] == min(2 * m, cap or kc.NUM_SMS), got
        assert cluster == (1 if cap % 2 else 2), (cap, cluster)
        assert (got[1] != 0) == all(fs % 8 == 0 for fs in sizes), got


def test_emu_cluster_many_facets():
    """67 facets at yN = 512: two launches, more lines than clusters in the first."""
    core, oracle = small_pair(512)
    step = core.facet_off_step
    offs = [(k - 5) * step for k in range(67)]
    got, cluster = _both(core, oracle, [248] * 67, offs, kc.subgrid_offsets(core)[2], yN=512,
                         shared_input=True, seed=3)
    assert got[0] == kc.TMA4 and got[3] == 3 * core.xM_yN_size and cluster == 2, got


@pytest.mark.parametrize("fs", [8192, 10174])
def test_emu_cluster_staging_boundaries_yN16384(fs):
    core, oracle = small_pair(16384)
    got, cluster = _both(core, oracle, [fs], [core.facet_off_step], kc.subgrid_offsets(core)[2],
                         yN=16384, seed=fs)
    assert got[:3] == kc.boundary_sizes_16384()[fs] and cluster == 2


@pytest.mark.parametrize("spot", [(512, 256, 2)], ids=lambda s: f"{s[0]}-{s[1]}")
def test_emu_extended_precision(spot):
    """One row against the centred DFT in extended precision: error <= 1.5 eps log2(yN) of the
    line's RMS (0.33 .. 0.54 as the single-CTA form)."""
    yN, fs, force_split = spot
    core, _ = small_pair(yN)
    got, ratio = kc.spot_check(core, fs, seed=fs, force_split=force_split, n_lines=1)
    print(f"\n{kc.KERNEL_NAMES[got[0]]} on clusters, yN {yN} fs {fs}: {ratio:.3f} eps log2(yN)")
    assert got[0] == kc.TMA4 and last_cluster(core) == 2 and got[1] != 0, got
    assert ratio <= lc.SPOT_BOUND, ratio


# ---------------------------------------------------------------------- the protocol itself
MISUSE = r"""
#include "emu_cluster.h"
using namespace swiftly;
struct Body {
    static constexpr int THREADS = 32;
    static constexpr int CLUSTER = 2;
    struct Maps {};
    int mode;
    const char* src;
    void operator()(ClusterHostCtx& ctx) const {
        const int rank = ctx.cluster_rank();
        double2* buf = (double2*)ctx.smem;
        uint64_t* bar = (uint64_t*)(ctx.smem + 1024);
        if (ctx.tid == 0) ctx.tx_init(bar);
        ctx.cluster_sync();
        if (rank == 0 && ctx.tid == 0) {
            ctx.tx_expect_peer(bar, 0, 128);
            if (mode != 3) ctx.tx_expect_peer(bar, 1, mode == 4 ? 64 : 128);  // 3: unarmed, 4: short
            ctx.tx_copy_mc(buf, src, 128, bar, 3);
        }
        ctx.tx_wait(bar, 0);
        ctx.peer_st(buf + 8 + ctx.tid, 1 - rank, buf[ctx.tid]);
        if (mode == 1 && rank == 1) return;  // 1: leaves the cluster barrier short
        ctx.cluster_sync();
        if (mode == 2 && rank == 0) return;  // 2: exits while the partner still writes into it
        if (mode == 2) ctx.sync();
        if (mode != 2) ctx.cluster_sync();
        if (mode == 2 && rank == 1) ctx.peer_st(buf + ctx.tid, 0, buf[8 + ctx.tid]);
    }
};
int main(int argc, char** argv) {
    static char src[128];
    Body b{atoi(argv[1]), src};
    Body::Maps maps;
    if (launch_body_maps_cluster(b, maps, 3, 2048, nullptr, nullptr) == cudaSuccess) return 1;
    launch_body_maps_cluster(b, maps, 4, 2048, nullptr, nullptr);
    puts("done");
    return 0;
}
"""
MISUSE_MODES = {1: "cluster barrier that cannot complete", 2: "which has exited",
                3: "not armed", 4: "more bytes than tx_expect announced"}


def test_cluster_protocol_reports_misuse(tmp_path):
    """A correct cluster walk passes (and a grid that is not whole clusters is refused); each
    slip of the cluster protocol ends the run with the protocol error that names it."""
    src = tmp_path / "misuse.cpp"
    src.write_text(MISUSE)
    exe = tmp_path / "misuse"
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(HERE, "emu"),
                           str(src), "-o", str(exe)])
    ok = subprocess.run([str(exe), "0"], capture_output=True, text=True, check=False)
    assert ok.returncode == 0 and ok.stdout == "done\n", ok.stderr
    for mode, message in MISUSE_MODES.items():
        bad = subprocess.run([str(exe), str(mode)], capture_output=True, text=True, check=False)
        assert bad.returncode != 0, mode
        assert "PROTOCOL error" in bad.stderr and message in bad.stderr, (mode, bad.stderr)
