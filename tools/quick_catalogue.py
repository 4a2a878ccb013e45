"""Fused forward path at the catalogue families outside xM / m in {2, 4} (dev tool):

    python tools/quick_catalogue.py [--reps R] [--fwd-reps F] [--only small|large] [NAME ...]

For each catalogue entry (default: the smallest entry of each of the six families and one
large entry, run with a sparse facet block):
  * K3 (axis 1, one group per facet row, transposed strips) and K4 (axis 0, the strips of one
    subgrid) alone: min and median over R launches (CUDA events), and the HBM fraction of the
    min, from the bytes the algorithm moves (DESIGN.md section 4.6: every source line's m-long
    window is read once, every finished line written once);
  * a forward transform over a fixed set of subgrid columns (every subgrid of the first two
    columns): min and median over F runs, wall clock around work that ends in a synchronise,
    once on the fused path and once on the primitive path (extract_from_facet,
    add_to_subgrid, finish_subgrid; forced with ``_fused = False``), and the max relative
    difference between the two.  Stage 1 (facet preparation) runs once, before the timing;
    the column cache is emptied before every run, so stage 2 (the columns) is timed too.
A build without the fused kernel for a family (the parent commit of this tool) prints "no
fused kernel" for K3 / K4 and the fused forward.
"""
import argparse
import statistics
import sys
import time

import torch

sys.path.insert(0, ".")
from ska_sdp_distributed_fourier_transform_b200 import (  # noqa: E402
    FacetConfig,
    SwiftlyConfig,
    SwiftlyForward,
    make_full_subgrid_cover,
)
from ska_sdp_distributed_fourier_transform_b200.swift_configs import SWIFT_CONFIGS  # noqa: E402

SMALL = ["16k[1]-n2k-1k", "1k[1]-n1k-256", "1536[1]-n512-384", "1280[1]-n640-320",
         "1536[1]-n768-384", "1792[1]-n896-448"]
# one large entry per family, with a block of BLOCK x BLOCK facets
LARGE = ["64k[1]-n8k-1k", "16k[1]-n16k-256", "12k[1]-n4k-384", "10k[1]-n5k-320",
         "12k[1]-n6k-384", "14k[1]-n7k-448"]
BLOCK_SMALL, BLOCK_LARGE = 3, 2
HBM = 3.35e12  # H100 SXM data sheet, bytes/s

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--fwd-reps", type=int, default=5)
ap.add_argument("--only", choices=["small", "large"])
ap.add_argument("names", nargs="*")
args = ap.parse_args()
names = args.names or ((SMALL if args.only != "large" else []) +
                       (LARGE if args.only != "small" else []))
dev = torch.device("cuda")
props = torch.cuda.get_device_properties(0)
print(f"# {props.name}", flush=True)


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


def run(name):
    p = SWIFT_CONFIGS[name]
    W, N, yB, yN, xA, xM = (p["W"], p["N"], p["yB_size"], p["yN_size"], p["xA_size"],
                            p["xM_size"])
    cfg = SwiftlyConfig(W=W, fov=1.0, N=N, yB_size=yB, yN_size=yN, xA_size=xA, xM_size=xM)
    core = cfg.core
    m = core.xM_yN_size
    nb = min(BLOCK_SMALL if name in SMALL else BLOCK_LARGE, N // yB)
    step = core.facet_off_step
    # the facet offsets: nb adjacent facet positions along either axis (multiples of the step)
    offs = [((i * yB + step - 1) // step) * step for i in range(nb)]
    print(f"{name}: N {N} yN {yN} m {m} xM {xM} xA {xA} yB {yB}, {nb}x{nb} facets", flush=True)

    # ---- K3 / K4 alone (random prepared facet rows, as stage 2 hands them on)
    g = torch.Generator(device=dev)
    g.manual_seed(1)
    rows = [[torch.randn(m, yN, dtype=torch.complex128, device=dev, generator=g)
             for _ in range(nb)] for _ in range(nb)]
    groups = [[(rows[r][i], offs[i]) for i in range(nb)] for r in range(nb)]
    strips_t = torch.empty(nb, xA, m, dtype=torch.complex128, device=dev).transpose(1, 2)
    out = torch.empty(xA, xA, dtype=torch.complex128, device=dev)
    srcs0 = [(strips_t[i], offs[i]) for i in range(nb)]
    for what, fn, by in (
            ("K3", lambda: core.sum_finish_axis_grouped(groups, strips_t, axis=1, subgrid_off=0),
             16 * nb * (nb * m * m + m * xA)),
            ("K4", lambda: core.sum_finish_axis(srcs0, out, axis=0, subgrid_off=0),
             16 * (nb * m * xA + xA * xA))):
        try:
            t, tm = timeit(fn, args.reps)
        except NotImplementedError:
            print(f"  {what}: no fused kernel", flush=True)
            continue
        print(f"  {what}: min {t:.4f} ms  median {tm:.4f} ms  HBM frac {by / (t * 1e-3) / HBM:.3f}",
              flush=True)
    del rows, groups, strips_t, out, srcs0

    # ---- forward transform over the first two subgrid columns
    facet_cfgs = [FacetConfig(a, b, yB) for a in offs for b in offs]
    facets = [torch.randn(yB, yB, dtype=torch.complex128, device=dev, generator=g)
              for _ in facet_cfgs]
    sgs = make_full_subgrid_cover(cfg)
    cols = sorted({s.off0 for s in sgs})[:2]
    sgs = [s for s in sgs if s.off0 in cols]
    results = {}
    for fused in (True, False):
        fwd = SwiftlyForward(cfg, list(zip(facet_cfgs, facets)), lru_forward=1)
        label = "fused" if fused else "primitive"
        if fused and not fwd._fused:
            print(f"  forward {label}: no fused kernel", flush=True)
            continue
        fwd._fused = fused

        def once(keep=False):
            fwd.lru.data.clear()
            outs = [fwd.get_subgrid_task(sg).tensor for sg in sgs]
            torch.cuda.synchronize()
            return outs if keep else None

        results[label] = once(keep=True)
        once()
        ts = []
        for _ in range(args.fwd_reps):
            t0 = time.perf_counter()
            once()
            ts.append((time.perf_counter() - t0) * 1e3)
        print(f"  forward {label}, {len(sgs)} subgrids in {len(cols)} columns: "
              f"min {min(ts):.2f} ms  median {statistics.median(ts):.2f} ms", flush=True)
        del fwd
    if len(results) == 2:
        scale = max(r.abs().max().item() for r in results["primitive"])
        diff = max((a - b).abs().max().item()
                   for a, b in zip(results["fused"], results["primitive"]))
        print(f"  fused vs primitive: max|diff| / max|primitive| = {diff / scale:.2e}", flush=True)
    del facets, results
    torch.cuda.empty_cache()


for n in names:
    run(n)
