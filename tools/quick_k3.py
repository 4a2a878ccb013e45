"""Fused subgrid kernel at the cfg4 geometry for a list of sg_variant values (dev tool):

    python tools/quick_k3.py [--cover 8x8|5x5] [--reps R] 0 25 0 25

K3 is the axis-1 kernel (all facet rows of a subgrid, one group per row, transposed strips),
K4 the axis-0 kernel (the strips of one subgrid).  --cover 8x8 (default) runs the full cover:
8 sources per line.  --cover 5x5 runs the central 5x5 block that bench.py times for cfg4
(bench.SPARSE_BLOCKS): 5 facet rows of 5 facets, 5 sources per line, scheduled as rounds of
3 + 2 windows.  Per kernel: min and median over R launches, HBM fraction of the min, the
time per line of one thread group (132 SMs x 2 groups) and max|diff| against the first
variant timed."""
import argparse
import ctypes
import statistics
import sys

import torch

sys.path.insert(0, ".")
from ska_sdp_distributed_fourier_transform_b200 import SwiftlyCoreB200  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--cover", default="8x8", choices=["8x8", "5x5"])
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("variants", type=int, nargs="*")
args = ap.parse_args()

W, N, yB, yN, xA, xM = 13.5625, 65536, 8192, 16384, 2048, 4096
core = SwiftlyCoreB200(W, N, xM, yN)
m = core.xM_yN_size
dev = torch.device("cuda")
HBM = 3.35e12  # H100 SXM data sheet
THREAD_GROUPS = 132 * 2
core._lib.swiftly_b200_debug_sg_variant.argtypes = [ctypes.c_void_p, ctypes.c_int]
variants = args.variants or [0]
# facet offsets along either axis (cfg4's SPARSE_BLOCKS in bench.py for the 5x5 block)
offs = [i * yB for i in range(8)] if args.cover == "8x8" else [0, 8192, 16384, 49152, 57344]
nf = len(offs)
props = torch.cuda.get_device_properties(0)
print(f"# {props.name}, cover {args.cover}: {nf} facet rows x {nf} sources per line", flush=True)


def timeit(fn, reps):
    fn()
    fn()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
    ev[0].record()
    for i in range(reps):
        fn()
        ev[i + 1].record()
    torch.cuda.synchronize()
    ts = [ev[i].elapsed_time(ev[i + 1]) for i in range(reps)]
    return min(ts), statistics.median(ts)


def report(name, v, t, tmed, by, lines, out, ref):
    msg = (f"{name} variant {v}: min {t:.4f} ms  median {tmed:.4f} ms  frac {by/t*1e3/HBM:.3f}"
           f"  {t * 1e3 / (lines / THREAD_GROUPS):.2f} us/group-line")
    if ref is not None:
        msg += f"  max|diff| {(out - ref).abs().max().item():.2e}"
    print(msg, flush=True)


g = torch.Generator(device=dev)
g.manual_seed(1)
big = [[torch.randn(m, yN, dtype=torch.complex128, device=dev, generator=g) for _ in range(nf)]
       for _ in range(nf)]
groups = [[(big[r][i], offs[i]) for i in range(nf)] for r in range(nf)]
strips_t = torch.empty(nf, xA, m, dtype=torch.complex128, device=dev).transpose(1, 2)
out = torch.empty(xA, xA, dtype=torch.complex128, device=dev)
ref3 = ref4 = None
for v in variants:
    core._lib.swiftly_b200_debug_sg_variant(core._plan, v)
    t, tm = timeit(lambda: core.sum_finish_axis_grouped(groups, strips_t, axis=1,
                                                        subgrid_off=2048), args.reps)
    report("K3", v, t, tm, 16 * nf * (nf * m * m + m * xA), nf * m, strips_t, ref3)
    if ref3 is None:
        ref3 = strips_t.clone()
    srcs0t = [(strips_t[i], offs[i]) for i in range(nf)]
    t, tm = timeit(lambda: core.sum_finish_axis(srcs0t, out, axis=0, subgrid_off=4096), args.reps)
    report("K4", v, t, tm, 16 * (nf * m * xA + xA * xA), xA, out, ref4)
    if ref4 is None:
        ref4 = out.clone()

    # K3 then K4 back to back, as in a step
    def both():
        core.sum_finish_axis_grouped(groups, strips_t, axis=1, subgrid_off=2048)
        core.sum_finish_axis(srcs0t, out, axis=0, subgrid_off=4096)
    t, tm = timeit(both, args.reps)
    print(f"K3+K4 variant {v}: min {t:.4f} ms  median {tm:.4f} ms", flush=True)
core._lib.swiftly_b200_debug_sg_variant(core._plan, 0)
