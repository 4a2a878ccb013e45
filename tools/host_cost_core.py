"""
Host cost of the argument marshalling in ``core.py``: microseconds per call of
``PreparedSumFinish.launch`` (the per-subgrid K3 / K4 launches of ``SwiftlyForward`` and of the
sharded forward), ``extract_columns`` and ``fold_column``, with every C entry replaced by a stub
that returns 0, so that only the Python side is timed.  No GPU and no built library are needed:
the tensors are CPU tensors standing in for device tensors.

The calls run at the catalogue's largest facet count, 10 x 10 facets (e.g. 96k[.875]-n12k-1k):
ten facet rows of ten facets per K3 launch, 100 facets (two chunks) per K2 / fold call, a
float64 mask per group and per facet.  The host cost depends on these counts, not on the array
sizes, so a small plan holds the arrays.

    python tools/host_cost_core.py [--reps 2000] [--repeats 7]
"""

import argparse
import ctypes
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ska_sdp_distributed_fourier_transform_b200.core import SwiftlyCoreB200  # noqa: E402

NF = 10  # facets per row and facet rows


class _StubLib:
    """Every ``swiftly_b200_*`` entry returns 0 (success) at once."""

    def __getattr__(self, name):
        return lambda *args: 0


class StubCore(SwiftlyCoreB200):
    """``SwiftlyCoreB200`` without a plan or a library, on CPU tensors."""

    def __init__(self, W, N, xM_size, yN_size):  # pylint: disable=super-init-not-called
        self.W, self.N, self.xM_size, self.yN_size = W, N, xM_size, yN_size
        self.xM_yN_size = xM_size * yN_size // N
        self.device = 0
        self._lib = _StubLib()
        self._plan = ctypes.c_void_p(1)

    def _check_tensor(self, t):
        # the attribute reads of the real check, without its CUDA requirement
        if t.is_cuda and t.device.index != self.device:
            raise ValueError("wrong device")


def per_call_us(fn, reps, repeats):
    """Median and minimum over ``repeats`` of the mean time of ``reps`` calls, in us."""
    for _ in range(reps // 10 + 1):
        fn()
    times = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        times.append((time.perf_counter() - t0) / reps * 1e6)
    return statistics.median(times), min(times)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--reps", type=int, default=2000)
    ap.add_argument("--repeats", type=int, default=7)
    args = ap.parse_args()
    torch.set_num_threads(1)
    core = StubCore(13.5625, 1024, 256, 512)
    m, yN, fs, xA = core.xM_yN_size, core.yN_size, 8, 160
    c128 = dict(dtype=torch.complex128)
    n = NF * NF
    bfs = [torch.zeros((yN, fs), **c128) for _ in range(n)]
    cols = [torch.zeros((m, yN), **c128) for _ in range(n)]
    faccs = [torch.zeros((yN, fs), **c128) for _ in range(n)]
    fmasks = [torch.ones(fs, dtype=torch.float64) for _ in range(n)]
    off1s = [0] * n
    sg_mask = torch.ones(xA, dtype=torch.float64)

    # K3 / K4 as SwiftlyForward._gen_subgrid launches them
    strips = torch.zeros((NF, xA, m), **c128).transpose(1, 2)
    groups = [[(cols[r * NF + j], 0) for j in range(NF)] for r in range(NF)]
    prep1 = core.prepare_sum_finish(groups, 1, m, xA, (strips.stride(1), strips.stride(2)))
    out = torch.zeros((xA, xA), **c128)
    prep0 = core.prepare_sum_finish([[(strips[r], 0) for r in range(NF)]], 0, xA, xA,
                                    (out.stride(1), out.stride(0)))
    ptrs = [strips[r].data_ptr() for r in range(NF)]
    cases = {
        "launch K3 (out=, 10 groups x 10 sources)": lambda: prep1.launch(
            [0] * NF, [sg_mask] * NF, out=strips, out_group_stride=strips.stride(0)),
        "launch K4 (out=, 1 group x 10 sources)": lambda: prep0.launch(
            [0], [sg_mask], out=out),
        "launch K3 (out_ptrs=, 10 groups)": lambda: prep1.launch(
            [0] * NF, [sg_mask] * NF, out_ptrs=ptrs, stream_of=strips),
        "extract_columns (100 facets)": lambda: core.extract_columns(
            bfs, 0, off1s, outs=cols, prewindowed=True),
        "fold_column (100 facets, masks)": lambda: core.fold_column(
            cols, faccs, off1s, fmasks, 0),
    }
    for name, fn in cases.items():
        med, best = per_call_us(fn, args.reps if "launch" in name else args.reps // 10,
                                args.repeats)
        print(f"{name:45s} {med:9.1f} us/call (median)  {best:9.1f} (min)")


if __name__ == "__main__":
    main()
