"""
``extract_columns`` (K2) on the host-emulated kernels in every launch form the dispatch picks
(``tests/k2_cases.py``): the pinned form of every catalogue ``(yN, yB)``, the box layouts of the
swizzled tensor loads, mixed facet sizes, row and output strides, wrapped offsets, capped and
overfull persistent grids, more than 64 facets, the staging limits at ``yN = 16384``, the
selectable 4 x Q forms, and an extended-precision spot check per form.

The emulator accounts for the bulk-copy barrier of the TMA-staged kernels
(``tests/emu/emu_runtime.h``): a transaction count that disagrees with the bytes delivered, a
wait on the wrong phase parity or a copy into a barrier that was not re-armed ends the test with
a protocol error instead of passing; ``test_barrier_accounting_reports_misuse`` checks that
accounting itself.

The cases run at the catalogue's ``W`` and ``yN`` with a small subgrid (``xM = 32``,
``N = 2 yN``, so ``m = 16``): the kernels' staging depends on ``yN`` and the facet sizes only.

Extended-precision spot check on the emulated kernels (host build without fused multiply-adds,
one line per form), in ``eps log2(yN)`` of the line's RMS: tma 0.23 .. 0.77, tma-2xH 0.38,
tma-4xQ 0.33 .. 0.54, dif 0.24, park-dif 0.24, park-dit 0.19, park-skew 0.19
(``k2_cases`` has the H100 numbers).
"""

import os
import subprocess

import pytest

from oracle.swiftly_oracle import OracleCore
from tests import k2_cases as kc
from tests import length_cases as lc
from tests.emu_support import emu_core_class

HERE = os.path.dirname(os.path.abspath(__file__))
ROWS = kc.catalogue_rows()
_cores = {}


def pair(geometry):
    if geometry not in _cores:
        _cores[geometry] = (emu_core_class()(*geometry), OracleCore(*geometry))
    return _cores[geometry]


def small_pair(yN, m=16):
    """(core, oracle) at the W of the smallest catalogue entry with that yN (11.0 for a length
    the catalogue does not have), N = 2 yN and xM = 2 m."""
    W = min((g for (n, _), (_, g) in ROWS.items() if n == yN), key=lambda g: g[1],
            default=(11.0,))[0]
    return pair((W, 2 * yN, 2 * m, yN))


# the rows the emulator runs: all of yN = 1024 and 2048, one each at 4096, 8192 and 16384, and
# one generic row of each kind
EMU_ROWS = [r for r in ROWS if r[0] in (1024, 2048)] + [
    (4096, 2816), (8192, 7296), (16384, 8192), (256, 208), (768, 528)]


def test_forms_are_pinned():
    """The catalogue needs exactly the pinned forms: a new (yN, yB), a changed number of entries
    behind a row or a change of the restated dispatch has to be looked at here and on the GPU."""
    tma, generic = kc.derived_tables()
    assert tma == kc.PINNED_TMA
    assert generic == kc.PINNED_GENERIC
    assert sum(v[-1] for v in tma.values()) + sum(v[-1] for v in generic.values()) \
        == len(kc.SWIFT_CONFIGS) == 247
    assert set(EMU_ROWS) <= set(ROWS)
    # yN = 16384: 2 of 16 entries run the tuned kernel, 14 SplitLineKernel<8192>
    assert kc.PINNED_TMA[(16384, 8192)][-1] == 2 and kc.PINNED_GENERIC[16384][-1] == 14
    assert min(yB for (yN, yB) in ROWS if yN == 16384 and yB > 8192) == 11264


def test_staging_limits_yN16384():
    """The staging limits at yN = 16384 from the kernels' shared-memory formulas: 8192 samples
    swizzled (whole boxes of 2048), 10174 linear, SplitLineKernel<8192> beyond."""
    records = {fs: kc.form(16384, [fs], 1)[0] for fs in range(8, 16384, 8)}
    swizzled = [fs for fs, r in records.items() if r[0] == kc.TMA4 and r[1]]
    assert max(swizzled) == kc.MAX_SWIZZLED_16384
    staged = [fs for fs in range(1, 16384) if kc.form(16384, [fs], 1)[0][0] == kc.TMA4]
    assert staged == list(range(1, kc.MAX_STAGED_16384 + 1))
    assert kc.form(16384, [kc.MAX_STAGED_16384 + 1], 1)[0][:2] == (kc.SPLIT_LINE, 2)
    for fs, want in kc.boundary_sizes_16384().items():
        assert kc.form(16384, [fs], 1)[0][:3] == want


@pytest.mark.parametrize("row", EMU_ROWS, ids=lambda r: f"{r[0]}-{r[1]}")
def test_emu_catalogue_row(row):
    yN, yB = row
    core, oracle = small_pair(yN)
    _, got = kc.catalogue_row_case(core, oracle, yB, n_facets=2, seed=yB)
    if row in kc.PINNED_TMA:
        kernel, box, boxes, in_cap, _ = kc.PINNED_TMA[row]
        assert got[:3] == (kernel, box, in_cap) and in_cap == boxes * box * 8
    else:
        assert got[:2] == kc.PINNED_GENERIC[yN][:2]


@pytest.mark.parametrize("yN", [1024, 2048, 4096, 8192])
def test_emu_box_layouts(yN):
    """Every box layout that fits yN: default staging against the oracle, and the same bits with
    linear staging (sg_variant 6) and with a capped grid."""
    core, oracle = small_pair(yN)
    seen = {}
    for fs in kc.box_layouts(yN):
        if yN > 2048 and fs < 2048:
            continue  # the small layouts run at 1024 and 2048
        _, record, boxes = kc.box_layout_case(core, oracle, fs, seed=fs)
        seen[fs] = (record[1], boxes)
    want = {1024: {8: (0, 0), 56: (0, 0), 64: (8, 1), 704: (88, 1)},
            2048: {8: (0, 0), 56: (0, 0), 64: (8, 1), 704: (88, 1), 1824: (224, 2)},
            4096: {2048: (256, 1), 2080: (256, 2), 2816: (256, 2)},
            8192: {2048: (256, 1), 2080: (256, 2), 2816: (256, 2), 7296: (256, 4)}}[yN]
    assert seen == want


@pytest.mark.parametrize("cap", [0, 1, 3])
def test_emu_mixed_sizes(cap):
    """[large, small, large] in one launch, uncapped (fewer lines than CTAs) and on 1 and 3
    CTAs, whose walk crosses from a long row to a short one and back."""
    for yN in (1024, 16384) if cap == 3 else (1024,):
        core, oracle = small_pair(yN)
        kc.mixed_case(core, oracle, cap=cap, seed=cap)


def test_emu_strides_outputs_offsets():
    core, oracle = small_pair(1024)
    kc.stride_case(core, oracle, 704, seed=1)
    kc.output_case(core, oracle, 704, seed=2)
    kc.offset_case(core, oracle, 832, seed=3)
    core, oracle = small_pair(2048)
    kc.stride_case(core, oracle, 1824, seed=4)
    kc.offset_case(core, oracle, 1824, seed=5)


def test_emu_many_lines_and_facets():
    """64 facets of 32 lines on the 1056 CTAs of the yN = 1024 kernel; 67 facets: two launches,
    the record shows the 3-facet one."""
    core, oracle = small_pair(1024, m=32)
    _, got = kc.many_lines_case(core, oracle, 64, n_facets=64, seed=1)
    assert got == (kc.TMA, 8, 64, 1056)
    core, oracle = small_pair(1024)
    _, got = kc.many_lines_case(core, oracle, 72, n_facets=67, seed=2)
    assert got == (kc.TMA, 8, 128, 48)


@pytest.mark.parametrize("fs", [8192, 8200, 10174, 10175])
def test_emu_staging_boundaries_yN16384(fs):
    core, oracle = small_pair(16384)
    kc.boundary_case(core, oracle, fs, seed=fs)


@pytest.mark.parametrize("variant", [0, 7, 15, 17, 18, 19])
def test_emu_variant_forms_yN512(variant):
    """The selectable 4 x Q forms through their force_split twins at yN = 512."""
    core, oracle = small_pair(512)
    kc.variant_case(core, oracle, variant, seed=variant)


SPOTS = [  # (yN, fs, variant, force_split, layout, kernel)
    (1024, 704, 0, 0, "contiguous", kc.TMA), (1024, 703, 0, 0, "contiguous", kc.TMA),
    (2048, 1824, 0, 0, "slice", kc.TMA), (4096, 2816, 0, 0, "contiguous", kc.TMA),
    (8192, 7296, 0, 0, "contiguous", kc.TMA), (16384, 8192, 0, 0, "contiguous", kc.TMA4),
    (16384, 10174, 0, 0, "contiguous", kc.TMA4), (16384, 8192, 7, 0, "contiguous", kc.TMA_SPLIT),
    (512, 256, 0, 3, "contiguous", kc.DIF), (512, 256, 0, 4, "contiguous", kc.PARK_DIF),
    (512, 256, 0, 5, "contiguous", kc.PARK_DIT), (512, 256, 0, 6, "contiguous", kc.PARK_SKEW),
]


@pytest.mark.parametrize("spot", SPOTS, ids=lambda s: f"{s[0]}-{s[1]}-{kc.KERNEL_NAMES[s[5]]}")
def test_emu_extended_precision(spot):
    """One row per form against the centred DFT in extended precision at the sub-transform
    boundaries, the centre and random bins: error <= 1.5 eps log2(yN) of the line's RMS."""
    yN, fs, variant, force_split, layout, kernel = spot
    core, _ = small_pair(yN)
    got, ratio = kc.spot_check(core, fs, seed=fs, variant=variant, force_split=force_split,
                               layout=layout, n_lines=1)
    print(f"\n{kc.KERNEL_NAMES[got[0]]} yN {yN} fs {fs}: {ratio:.3f} eps log2(yN)")
    assert got[0] == kernel and (got[1] != 0) == (fs % 8 == 0 and fs <= 8192), got
    assert ratio <= lc.SPOT_BOUND, ratio


# ---------------------------------------------------------------------- the accounting itself
MISUSE = r"""
#include "emu_runtime.h"
using namespace swiftly;
struct Body {
    static constexpr int THREADS = 32;
    int mode;
    const char* src;
    void operator()(HostCtx& ctx) const {
        char* dst = ctx.smem;
        uint64_t* bar = (uint64_t*)(ctx.smem + 256);
        auto issue = [&](uint32_t expect, uint32_t copy) {
            ctx.tx_expect(bar, expect);
            ctx.tx_copy(dst, src, copy, bar);
        };
        if (ctx.tid == 0) {
            if (mode != 6) ctx.tx_init(bar);
            issue(mode == 1 ? 64 : 128, mode == 2 ? 64 : 128);  // 1: overshoot, 2: short
        }
        ctx.sync();
        uint32_t parity = 0;
        for (int line = 0; line < 3; ++line) {
            ctx.tx_wait(bar, parity);
            if (mode != 3) parity ^= 1;  // 3: no parity flip
            if (mode != 7) ctx.sync();   // 7: refill before every thread has waited
            if (ctx.tid == 0 && line < 2) {
                if (mode == 4) ctx.tx_copy(dst, src, 128, bar);  // 4: copy without tx_expect
                else issue(128, 128);
                if (mode == 5 && line == 0) ctx.tx_expect(bar, 128);  // 5: armed twice
            }
            ctx.sync();
        }
    }
};
int main(int argc, char** argv) {
    static char src[128];
    Body b{atoi(argv[1]), src};
    launch_body(b, 2, 512, nullptr);
    puts("done");
    return 0;
}
"""
MISUSE_MODES = {1: "more bytes than tx_expect announced", 2: "phase that cannot complete",
                3: "parity of the wrong phase", 4: "not armed", 5: "already armed",
                6: "before tx_init", 7: "before every thread waited"}


def test_barrier_accounting_reports_misuse(tmp_path):
    """A correct walk of three phases passes; each slip of the bulk-copy barrier protocol ends
    the run with the protocol error that names it."""
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
        assert "bulk-copy barrier PROTOCOL error" in bad.stderr and message in bad.stderr, \
            (mode, bad.stderr)
