"""K2 (extract_columns) variants at the cfg4 geometry: time per 8 facets and difference to the
default kernel on identical data (dev tool; run under `timeout`)."""
import ctypes
import sys

import torch

sys.path.insert(0, ".")
from ska_sdp_distributed_fourier_transform_b200 import SwiftlyCoreB200  # noqa: E402

W, N, yB, yN, xA, xM = 13.5625, 65536, 8192, 16384, 2048, 4096
core = SwiftlyCoreB200(W, N, xM, yN)
m = core.xM_yN_size
dev = torch.device("cuda")
nf = 8
HBM = 3.35e12  # H100 SXM data sheet
REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 8
core._lib.swiftly_b200_debug_sg_variant.argtypes = [ctypes.c_void_p, ctypes.c_int]
core._lib.swiftly_b200_debug_last_cluster.argtypes = [ctypes.c_void_p]


def timeit(fn, reps=REPS):
    """Minimum and spread (max - min) of `reps` timed calls, in ms."""
    fn()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
    ev[0].record()
    for i in range(reps):
        fn()
        ev[i + 1].record()
    torch.cuda.synchronize()
    ts = [ev[i].elapsed_time(ev[i + 1]) for i in range(reps)]
    return min(ts), max(ts) - min(ts)


# distinct prepared facets (8 x 2 GiB): no L2 reuse between facets, as in a step
bfs = [torch.randn(yN, yB, dtype=torch.complex128, device=dev) for _ in range(nf)]
nmbf = [torch.empty(m, yN, dtype=torch.complex128, device=dev) for _ in range(nf)]
offs = [yB * i for i in range(nf)]
by = 16 * (m * yB + m * yN) * nf
VARIANTS = ((0, "4 x 4096, two-CTA clusters, combine through distributed shared memory (default)"),
            (26, "4 x 4096, two groups, CTA-wide combine, L2 scratch"),
            (18, "DIT across / DIT within, L2 parking + swap, unit-stride stores"),
            (19, "DIT / DIT, L2 parking + swap, group 1 stores half a line later"),
            (15, "DIF across / DIT within, L2 scratch, 16-byte stores at 32-byte stride"),
            (17, "DIF across / DIT within, L2 parking + swap, 32-byte pair stores"),
            )
for pre in (False, True):
    keep = None
    for variant, name in VARIANTS:
        core._lib.swiftly_b200_debug_sg_variant(core._plan, variant)
        for o in nmbf:
            o.zero_()
        t, ta = timeit(lambda: core.extract_columns(bfs, 4096 + 2048, offs, outs=nmbf, prewindowed=pre))
        rec = (ctypes.c_int * 4)()
        core._lib.swiftly_b200_debug_last_launch(core._plan, rec)
        cluster = core._lib.swiftly_b200_debug_last_cluster(core._plan)
        print(f"K2 x{nf} prewindowed={int(pre)} [{variant}: {name}]: {t:.3f} ms (spread {ta:.3f}, "
              f"{REPS} runs, launch {list(rec)}, cluster {cluster})  "
              f"frac {by/t*1e3/HBM:.3f}", flush=True)
        if keep is None:
            keep = [o.clone() for o in (nmbf[0], nmbf[3], nmbf[7])]
        else:
            d = max((a - b).abs().max().item() for a, b in zip((nmbf[0], nmbf[3], nmbf[7]), keep))
            same = all(torch.equal(a, b) for a, b in zip((nmbf[0], nmbf[3], nmbf[7]), keep))
            print(f"   max |diff| vs the default kernel: {d:.3e} (max |ref| {keep[1].abs().max().item():.3e})"
                  f"{', bitwise equal' if same else ''}", flush=True)
core._lib.swiftly_b200_debug_sg_variant(core._plan, 0)
