"""Time the subgrid side of the backward transform, split kernels against the primitive chain.

    python tools/quick_split.py [cfg4|cfg3|cfg2] [--reps R] [--columns C]

On the same inputs: K4T (split_subgrid_axis along axis 0 into one strip per facet row) and K3T
(along axis 1, added to every facet's column accumulator) alone, the primitive chain they
replace (prepare_subgrid on both axes, extract_from_subgrid(axis 0) per facet row,
subgrid_to_facets), then SwiftlyBackward over the first C subgrid columns with either subgrid
side.  cfg4 is the central 5 x 5 facet block of the 64k[1]-n16k-4k cover (as bench.py runs it).
Min / median of R CUDA-event timings and the algorithmic bytes as a fraction of the HBM peak
(3.35 TB/s, H100 SXM5 nominal); max |new - old| / max |old| for the accumulators and facets.
"""
import argparse
import statistics
import sys

import numpy
import torch

sys.path.insert(0, ".")
from ska_sdp_distributed_fourier_transform_b200 import (  # noqa: E402
    SWIFT_CONFIGS, FacetConfig, SwiftlyBackward, SwiftlyConfig, make_full_facet_cover,
    make_full_subgrid_cover)

HBM = 3.35e12
NAMES = {"cfg4": "64k[1]-n16k-4k", "cfg3": "32k[1]-n8k-4k", "cfg2": "8k[1]-n4k-2k"}
BLOCK = [0, 8192, 16384, 49152, 57344]


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1))
    return min(out), statistics.median(out)


def report(what, t, nbytes):
    print(f"  {what:58s} min {t[0]:8.3f} ms  median {t[1]:8.3f} ms  "
          f"{nbytes / 2**20:9.1f} MiB  HBM {nbytes / (t[0] * 1e-3) / HBM:5.1%}", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workload", nargs="?", default="cfg4", choices=sorted(NAMES))
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--columns", type=int, default=2)
    args = ap.parse_args()
    params = SWIFT_CONFIGS[NAMES[args.workload]]
    cfg = SwiftlyConfig(**params)
    core = cfg.core
    m, xM, yN, xA = core.xM_yN_size, core.xM_size, core.yN_size, cfg.max_subgrid_size
    if args.workload == "cfg4":
        fcs = [FacetConfig(a, b, cfg.max_facet_size) for a in BLOCK for b in BLOCK]
    else:
        fcs = make_full_facet_cover(cfg)
    rows = sorted({f.off0 for f in fcs})
    F = len(fcs)
    sgs = make_full_subgrid_cover(cfg)
    sg = sgs[len(sgs) // 2 + 3]
    dev = torch.device("cuda")
    gen = torch.Generator(device=dev)
    gen.manual_seed(5)
    x = torch.empty((xA, xA), dtype=torch.complex128, device=dev)
    torch.view_as_real(x).normal_(generator=gen)
    print(f"{args.workload} ({NAMES[args.workload]}): m={m} xM={xM} yN={yN} xA={xA}, "
          f"{F} facets in {len(rows)} rows; split kernel: {core.split_axis_supported()}")

    # ---- new: K4T + K3T
    strips = torch.empty((len(rows), m, xA), dtype=torch.complex128, device=dev)
    accs_new = [torch.zeros((m, yN), dtype=torch.complex128, device=dev) for _ in fcs]
    k4 = lambda: core.split_subgrid_axis([x], 0, [sg.off0], [[(strips[r], o) for r, o in
                                                              enumerate(rows)]], "store")
    targets = [[(accs_new[j], f.off1) for j, f in enumerate(fcs) if f.off0 == o] for o in rows]
    k3 = lambda: core.split_subgrid_axis([strips[r] for r in range(len(rows))], 1,
                                         [sg.off1] * len(rows), targets, "add")
    b4 = 16.0 * (xA * xA + len(rows) * m * xA)
    b3 = 16.0 * (len(rows) * m * xA + 2 * F * m * m)
    report("K4T split axis 0 (strips)", timed(k4, args.reps), b4)
    report("K3T split axis 1 (add to column accumulators)", timed(k3, args.reps), b3)
    report("K4T + K3T", timed(lambda: (k4(), k3()), args.reps), b4 + b3)

    # ---- old: prepare_subgrid + extract_from_subgrid per row + subgrid_to_facets
    accs_old = [torch.zeros((m, yN), dtype=torch.complex128, device=dev) for _ in fcs]

    def old():
        prepared = core.prepare_subgrid(x, (sg.off0, sg.off1))
        blocks = {o: core.extract_from_subgrid(prepared, o, axis=0) for o in rows}
        core.subgrid_to_facets([blocks[f.off0] for f in fcs], accs_old, [f.off1 for f in fcs],
                               sg.off1)
    bo = 16.0 * (xA * xA + 2 * xM * xA + xM * xM + len(rows) * 2 * m * xM + F * 3 * m * m)
    report("primitive chain (prepare, extract x rows, subgrid_to_facets)", timed(old, args.reps), bo)
    for a in accs_new + accs_old:
        a.zero_()
    k4()
    k3()
    old()
    torch.cuda.synchronize()
    scale = max(float(a.abs().max()) for a in accs_old)
    diff = max(float((a - b).abs().max()) for a, b in zip(accs_new, accs_old))
    print(f"  column accumulators: max|new - old| / max|old| = {diff / scale:.2e}")
    del strips, accs_new, accs_old

    # ---- SwiftlyBackward over the first few subgrid columns
    cols = sorted({s.off0 for s in sgs})[:args.columns]
    run = [s for s in sgs if s.off0 in cols]
    facets = {}
    for split in (True, False):
        bwd = SwiftlyBackward(cfg, fcs, lru_backward=1, queue_size=8)
        bwd._split = bwd._split and split
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for s in run:
            bwd.add_new_subgrid_task(s, x)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        tasks = bwd.finish()
        facets[split] = [t.tensor[:256, :256].cpu().numpy() for t in tasks[:3]]
        print(f"  SwiftlyBackward, {len(run)} subgrids ({len(cols)} columns), "
              f"{'split kernels' if split else 'primitive chain'}: {ms:.1f} ms "
              f"({ms / len(run):.2f} ms per subgrid)", flush=True)
        del bwd, tasks
        torch.cuda.empty_cache()
    scale = max(numpy.abs(f).max() for f in facets[False])
    diff = max(numpy.abs(a - b).max() for a, b in zip(facets[True], facets[False]))
    print(f"  facets (256 x 256 corner of 3): max|new - old| / max|old| = {diff / scale:.2e}")


if __name__ == "__main__":
    main()
