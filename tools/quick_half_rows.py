"""
Half rows of real images (``half_rows=True``) at cfg4 (64k[1]-n16k-4k) on one GPU.

1. The benchmark's central 5 x 5 block of real (point-source) facets, all 32 x 32 subgrids:
   full-row real mode against ``half_rows``, alternated in one process.
   * whole forward and whole backward: wall clock from construction to the last result plus a
     device synchronise, min over ``--runs`` per mode after a warm-up, the tier each took, and
     ``torch.cuda.max_memory_allocated`` of each run.  With the facets held on the device, the
     full-row forward does not fit the device tier: it is timed only with ``--full-forward``;
   * per facet (CUDA events, mean over ``--reps``): K1 (the promotion of the real facet to
     complex128 plus ``prepare_facet(window_lines=True)``, and the K1 kernel alone, against
     ``prepare_facet_real_half``) and ``finish_facet_real`` against ``finish_facet_real_half``;
   * per launch: K2 (``extract_columns``) of 8 of the facets at one subgrid column, full against
     half rows.
   The backward is fed 16 random device subgrids cyclically; the values do not affect the timing.
2. A 7 x 7 block (49 facets in host memory, uploaded one at a time by the forward):
   ``half_rows`` in the device tier, forward and backward, wall clock and peak allocation; three
   subgrids against the analytic DFT and three facets holding a source (of a backward fed with
   the analytic subgrids, made on the device one at a time) against the point sources, relative
   to the brightest source.  The full-row
   device-tier estimate (``device_tier_bytes``) is reported beside the device's memory; its host
   tier is not run.

Prints one JSON object and writes it to ``--out``.

    python tools/quick_half_rows.py --out half_rows.json
"""

import argparse
import json
import os
import subprocess
import sys
import time

import numpy
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ska_sdp_distributed_fourier_transform_b200 import (  # noqa: E402
    FacetConfig,
    SwiftlyBackward,
    SwiftlyConfig,
    SwiftlyForward,
    make_full_subgrid_cover,
)
from ska_sdp_distributed_fourier_transform_b200.api import device_tier_bytes  # noqa: E402
from ska_sdp_distributed_fourier_transform_b200.api_helper import (  # noqa: E402
    make_facet,
    make_facet_device,
)
from ska_sdp_distributed_fourier_transform_b200.fourier_algorithm import (  # noqa: E402
    make_subgrid_from_sources,
)
from ska_sdp_distributed_fourier_transform_b200.swift_configs import SWIFT_CONFIGS  # noqa: E402
from tools.quick_real_image import NAME, SOURCES, event_ms, last_launch  # noqa: E402

BLOCK5 = [0, 8192, 16384, 49152, 57344]  # bench.py's cfg4 facet block (central 5 x 5)
BLOCK7 = [0, 8192, 16384, 24576, 40960, 49152, 57344]
K2_FACETS = 8
CHECKED_FACETS = (0, 7, 43)  # 7 x 7 facets holding a source: (0, 0), (8192, 0), (-8192, 8192)


def make_cfg(dev):
    p = SWIFT_CONFIGS[NAME]
    return SwiftlyConfig(W=p["W"], fov=1.0, N=p["N"], yB_size=p["yB_size"], yN_size=p["yN_size"],
                         xA_size=p["xA_size"], xM_size=p["xM_size"], device=dev.index)


def subgrid_device(N, sg, sources, dev):
    """``make_subgrid_from_sources`` (with the subgrid's masks) on the device: a sum of outer
    products per source."""
    coords = [torch.arange(off - sg.size // 2, off + (sg.size + 1) // 2, dtype=torch.float64,
                           device=dev) for off in (sg.off0, sg.off1)]
    out = torch.zeros((sg.size, sg.size), dtype=torch.complex128, device=dev)
    for intensity, x0, x1 in sources:
        e0 = torch.exp(1j * (2 * numpy.pi / N) * ((coords[0] * x0) % N))
        e1 = torch.exp(1j * (2 * numpy.pi / N) * ((coords[1] * x1) % N))
        out += (intensity / N ** 2) * torch.outer(e0, e1)
    for axis, mask in enumerate((sg.mask0, sg.mask1)):
        if mask is not None:
            m = torch.as_tensor(numpy.asarray(mask, dtype=float), device=dev)
            out *= m[:, None] if axis == 0 else m[None, :]
    return out


class LazySubgrid:
    def __init__(self, N, sg, dev):
        self.N, self.sg, self.dev = N, sg, dev

    def result(self):
        return subgrid_device(self.N, self.sg, SOURCES, self.dev)


def timed(dev, fn):
    # the transforms size their tier from the device's free memory, which the caching allocator's
    # reserve of the previous run would hide
    torch.cuda.empty_cache()
    torch.cuda.synchronize(dev)
    torch.cuda.reset_peak_memory_stats(dev)
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize(dev)
    return time.perf_counter() - t0, torch.cuda.max_memory_allocated(dev)


def block5(dev, runs, reps, progress, full_forward):
    cfg = make_cfg(dev)
    core = cfg.core
    yB = cfg.max_facet_size
    facet_cfgs = [FacetConfig(a, b, yB) for a in BLOCK5 for b in BLOCK5]
    sg_cfgs = make_full_subgrid_cover(cfg)
    facets = [make_facet_device(cfg.image_size, fc, SOURCES, dev).real.contiguous()
              for fc in facet_cfgs]
    inputs = []
    tiers = {}

    def forward(half):
        fwd = SwiftlyForward(cfg, list(zip(facet_cfgs, facets)), queue_size=4,
                             real_image=True, half_rows=half)
        tiers[("forward", half)] = fwd.host_tier
        for _ in fwd.iter_subgrid_tasks(sg_cfgs):
            pass

    def backward(half):
        bwd = SwiftlyBackward(cfg, facet_cfgs, queue_size=4, real_image=True, half_rows=half)
        tiers[("backward", half)] = bwd.host_tier
        bwd.add_subgrid_tasks(sg_cfgs, [inputs[i % 16] for i in range(len(sg_cfgs))])
        for t in bwd.finish():
            t.wait()

    res = {}
    # with the 25 real facets held on the device next to the transform, full-row real mode does
    # not fit the device tier and takes the host tier (tens of seconds a run): its forward is not
    # repeated here (``--full-forward`` runs it)
    for name, fn, modes in (("forward", forward, (True, False) if full_forward else (True,)),
                            ("backward", backward, (False, True))):
        if name == "backward":
            del facets[:]
            gen = torch.Generator(device=dev).manual_seed(31)
            inputs.extend(torch.randn((cfg.max_subgrid_size,) * 2, dtype=torch.complex128,
                                      device=dev, generator=gen) for _ in range(16))
        for half in modes:  # warm-up
            timed(dev, lambda: fn(half))
        times = {h: [] for h in modes}
        peaks = {h: 0 for h in modes}
        for _ in range(runs):
            for half in modes:
                t, peak = timed(dev, lambda: fn(half))
                times[half].append(t)
                peaks[half] = max(peaks[half], peak)
        res[name] = {("half_rows" if h else "full_rows"): {
            "min_s": min(times[h]), "all_s": times[h], "max_memory_allocated": peaks[h],
            "host_tier": tiers[(name, h)]} for h in modes}
        progress(res)
    del inputs[:]
    facets = [make_facet_device(cfg.image_size, fc, SOURCES, dev).real.contiguous()
              for fc in facet_cfgs]
    torch.cuda.empty_cache()

    # per facet: K1 and the finish
    fc, f = facet_cfgs[0], facets[0].contiguous()
    yN = core.yN_size
    bf = torch.empty((yN, yB), dtype=torch.complex128, device=dev)
    bh = torch.empty((core.half_rows, yB), dtype=torch.complex128, device=dev)
    fz = f.to(torch.complex128)
    per = {
        "k1_promote_and_full_ms": event_ms(lambda: core.prepare_facet(
            f.to(torch.complex128), fc.off0, 0, out=bf, window_lines=True), reps),
        "k1_full_kernel_ms": event_ms(lambda: core.prepare_facet(
            fz, fc.off0, 0, out=bf, window_lines=True), reps),
        "k1_half_ms": event_ms(lambda: core.prepare_facet_real_half(f, fc.off0, 0, out=bh), reps),
    }
    del fz
    out = torch.empty((yB, yB), dtype=torch.float64, device=dev)
    per["finish_real_ms"] = event_ms(lambda: core.finish_facet_real(bf, fc.off0, yB, 0, out=out),
                                     reps)
    per["finish_real_half_ms"] = event_ms(
        lambda: core.finish_facet_real_half(bh, fc.off0, yB, 0, out=out), reps)
    del bf, bh, out
    res["per_call"] = per
    progress(res)
    # per launch: K2 over the first K2_FACETS facets (the full-row arrays of all 25 would not fit
    # next to the facets)
    del facets[K2_FACETS:]
    torch.cuda.empty_cache()
    off1s = [c.off1 for c in facet_cfgs[:K2_FACETS]]
    outs = [torch.empty((core.xM_yN_size, yN), dtype=torch.complex128, device=dev)
            for _ in range(K2_FACETS)]
    for half in (False, True):
        bfs = [core.prepare_facet_real_half(x, c.off0) if half else
               core.prepare_facet(x.to(torch.complex128), c.off0, 0, window_lines=True)
               for c, x in zip(facet_cfgs, facets)]
        key = "half_rows" if half else "full_rows"
        per[f"k2_{key}_ms"] = event_ms(lambda: core.extract_columns(
            bfs, sg_cfgs[5].off0, off1s, outs=outs, prewindowed=True), reps)
        per[f"k2_{key}_form"] = last_launch(core)
        del bfs
        torch.cuda.empty_cache()
    res["per_call"] = per
    return res


def block7(dev, n_checked=3):
    cfg = make_cfg(dev)
    core = cfg.core
    N, yB = cfg.image_size, cfg.max_facet_size
    facet_cfgs = [FacetConfig(a, b, yB) for a in BLOCK7 for b in BLOCK7]
    sg_cfgs = make_full_subgrid_cover(cfg)
    free, total = torch.cuda.mem_get_info(dev)
    sizes = [fc.size for fc in facet_cfgs]
    est = {d: {half: device_tier_bytes(d, core.yN_size, core.xM_yN_size, sizes, 1,
                                       len(BLOCK7) if d == "forward" else 0,
                                       cfg.max_subgrid_size if d == "forward" else 0,
                                       half_rows=half)
               for half in (False, True)}
           for d in ("forward", "backward")}
    res = {"free_bytes": free, "total_bytes": total,
           "estimate_bytes": {d: {"full_rows": v[False], "half_rows": v[True]}
                              for d, v in est.items()},
           "full_rows_host_tier": "not run"}
    checked = list(range(0, len(sg_cfgs), len(sg_cfgs) // n_checked))[:n_checked]
    kept = []

    # host (numpy) facets: the forward uploads them one at a time, they never all sit on the device
    facets = [make_facet(N, fc, SOURCES).real for fc in facet_cfgs]

    def forward():
        fwd = SwiftlyForward(cfg, list(zip(facet_cfgs, facets)), queue_size=4, real_image=True,
                             half_rows=True)
        assert not fwd.host_tier
        for i, task in fwd.iter_subgrid_tasks(sg_cfgs):
            if i in checked:
                kept.append((i, task.result()))

    t, peak = timed(dev, forward)
    del facets
    errs = []  # relative to the subgrid's largest sample
    for i, got in kept:
        sg = sg_cfgs[i]
        truth = make_subgrid_from_sources(SOURCES, N, sg.size, [sg.off0, sg.off1],
                                          [sg.mask0, sg.mask1])
        errs.append(float(numpy.abs(got - truth).max() / numpy.abs(truth).max()))
    res["forward"] = {"s": t, "max_memory_allocated": peak, "subgrid_rel_errors": errs}
    torch.cuda.empty_cache()
    facets_out = []

    def backward():
        bwd = SwiftlyBackward(cfg, facet_cfgs, queue_size=4, real_image=True, half_rows=True)
        assert not bwd.host_tier
        bwd.add_subgrid_tasks(sg_cfgs, [LazySubgrid(N, sg, dev) for sg in sg_cfgs])
        for j, task in enumerate(bwd.finish()):
            if j in CHECKED_FACETS:
                facets_out.append((j, task.result()))

    t, peak = timed(dev, backward)
    ferrs = []
    scale = max(s[0] for s in SOURCES)
    for j, got in facets_out:
        truth = make_facet(N, facet_cfgs[j], SOURCES)
        ferrs.append(float(numpy.abs(got - truth.real).max() / scale))
    res["backward"] = {"s": t, "max_memory_allocated": peak, "facet_rel_errors": ferrs}
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--skip-block7", action="store_true")
    ap.add_argument("--full-forward", action="store_true",
                    help="also time the full-row forward (host tier at this block, slow)")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                          "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {"gpu": smi, "config": NAME}

    def emit():  # after every section, so that a partial run leaves its numbers
        text = json.dumps(res, indent=1, default=str)
        print(text, flush=True)
        if args.out:
            with open(args.out, "w", encoding="utf-8") as fh:
                fh.write(text)

    res["block5"] = block5(dev, args.runs, args.reps,
                           lambda part: (res.update(block5=part), emit()), args.full_forward)
    emit()
    torch.cuda.empty_cache()
    if not args.skip_block7:
        res["block7"] = block7(dev)
        emit()


if __name__ == "__main__":
    main()
