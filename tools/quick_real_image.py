"""
Real-image forward transform at cfg4 (64k[1]-n16k-4k), the benchmark's central 5 x 5 facet block,
all 32 x 32 subgrids, on one GPU: ``SwiftlyForward(real_image=True)`` (514 subgrids computed, 510
mirrored) against the default mode, run alternately in one process on the same real facets (the
benchmark's seeds, standard-normal real samples).

* whole forward: wall clock from construction to a device synchronise after the last subgrid,
  min over ``--runs`` runs per mode;
* per launch (CUDA events, mean over ``--reps``): K3 (axis 1) and K4 (axis 0) at the source size
  S = xA + 1 and at xA, with the output path each ran; ``mirror_subgrid`` and its share of the
  H100's 3.35 TB/s for its 16 (S^2 + 2 xA^2) bytes;
* agreement: the largest difference against the default mode of the sources (expected 0) and of
  the mirrors (expected: the approximation level), over 4096 sampled positions of every subgrid;
  then, with point-source facets, the error of 3 pairs against the analytic DFT in both modes.

Prints one JSON object and writes it to ``--out``.

    python tools/quick_real_image.py --out real_image.json
"""

import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ska_sdp_distributed_fourier_transform_b200 import (  # noqa: E402
    SWIFT_CONFIGS,
    FacetConfig,
    SubgridConfig,
    SwiftlyConfig,
    SwiftlyForward,
    make_facet_device,
    make_full_subgrid_cover,
)
from ska_sdp_distributed_fourier_transform_b200.api import mirror_pairs  # noqa: E402
from ska_sdp_distributed_fourier_transform_b200.fourier_algorithm import (  # noqa: E402
    make_subgrid_from_sources,
)

NAME = "64k[1]-n16k-4k"
BLOCK = [0, 8192, 16384, 49152, 57344]  # bench.py's cfg4 facet block (central 5 x 5)
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
SOURCES = [(1.0, 1, 0), (0.5, -7000, 5001), (0.25, 9011, -3777), (0.75, 12000, 11999)]


class Workload:
    """The 5 x 5 block with its real facets inside the prepared-facet arena (as bench.py lays out
    its complex facets: facet k is read before BF_F[k] overwrites it)."""

    def __init__(self, dev):
        p = SWIFT_CONFIGS[NAME]
        self.cfg = SwiftlyConfig(W=p["W"], fov=1.0, N=p["N"], yB_size=p["yB_size"],
                                 yN_size=p["yN_size"], xA_size=p["xA_size"],
                                 xM_size=p["xM_size"], device=dev.index)
        self.dev = dev
        yB, yN = p["yB_size"], p["yN_size"]
        self.facet_cfgs = [FacetConfig(a, b, yB) for a in BLOCK for b in BLOCK]
        self.sg_cfgs = make_full_subgrid_cover(self.cfg)
        F, b, u = len(self.facet_cfgs), yN * yB, yB * yB
        self.arena = torch.empty(F * b, dtype=torch.complex128, device=dev)
        self.bf = [self.arena[k * b:(k + 1) * b].view(yN, yB) for k in range(F)]
        reals = torch.view_as_real(self.arena[F * b - F * u // 2:]).reshape(-1)
        self.facets = [reals[k * u:(k + 1) * u].view(yB, yB) for k in range(F)]
        self.gen = torch.Generator(device=dev)

    def random_facets(self):
        for k, f in enumerate(self.facets):
            self.gen.manual_seed(123456789 + k)
            f.normal_(generator=self.gen)

    def point_facets(self):
        for fc, f in zip(self.facet_cfgs, self.facets):
            f.copy_(make_facet_device(self.cfg.image_size, fc, SOURCES, self.dev).real)

    def forward(self, real):
        return SwiftlyForward(self.cfg, list(zip(self.facet_cfgs, self.facets)), lru_forward=1,
                              queue_size=4, bf_f_buffers=self.bf, real_image=real)

    def run(self, real, consumer=None):
        """One whole forward; returns seconds (construction to the final synchronise)."""
        torch.cuda.synchronize(self.dev)
        t0 = time.perf_counter()
        fwd = self.forward(real)
        if real:
            for i, task in fwd.iter_subgrid_tasks(self.sg_cfgs):
                if consumer is not None:
                    consumer(i, task.tensor)
        else:
            for i, sg in enumerate(self.sg_cfgs):
                task = fwd.get_subgrid_task(sg)
                if consumer is not None:
                    consumer(i, task.tensor)
        torch.cuda.synchronize(self.dev)
        return time.perf_counter() - t0


def last_launch(core):
    lib = core._lib  # pylint: disable=protected-access
    lib.swiftly_b200_debug_last_launch.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int)]
    out = (ctypes.c_int * 4)()
    lib.swiftly_b200_debug_last_launch(core._plan, out)  # pylint: disable=protected-access
    return list(out)


def event_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def per_launch(w, reps):
    """K3 and K4 at S and xA, and mirror_subgrid, on the prepared blocks of a real forward."""
    # pylint: disable=protected-access
    w.random_facets()
    fwd = w.forward(True)
    core = fwd.core
    xA = w.cfg.max_subgrid_size
    S = 2 * (xA // 2) + 1
    sg = w.sg_cfgs[len(w.sg_cfgs) // 2 + 5]
    cols = fwd.get_NMBF_BFs_off0(sg.off0, fwd._get_BF_Fs())
    res = {}
    for size in (S, xA):
        fwd._gen_subgrid(SubgridConfig(sg.off0, sg.off1, size), cols)
        st = fwd._size_state(size)
        nrows = len(fwd._rows)
        out = torch.empty((size, size), dtype=torch.complex128, device=w.dev)

        def k3():
            st["prep1"][1].launch([sg.off1] * nrows, [None] * nrows, out=st["strips"],
                                  out_group_stride=st["strips"].stride(0))

        def k4():
            st["prep0"].launch([sg.off0], [None], out=out)

        k3_ms = event_ms(k3, reps)
        k3_rec = last_launch(core)
        k4_ms = event_ms(k4, reps)
        k4_rec = last_launch(core)
        res[f"size_{size}"] = {"K3_ms": k3_ms, "K4_ms": k4_ms,
                               "K3_launch": k3_rec, "K4_launch": k4_rec,
                               "K3_output_path": ["direct", "tma", "tma-per-group"][k3_rec[2]],
                               "K4_output_path": ["direct", "tma", "tma-per-group"][k4_rec[2]]}
    src = torch.empty((S, S), dtype=torch.complex128, device=w.dev)
    torch.view_as_real(src).normal_()
    outs = (torch.empty((xA, xA), dtype=torch.complex128, device=w.dev),
            torch.empty((xA, xA), dtype=torch.complex128, device=w.dev))
    mask = torch.ones(xA, dtype=torch.float64, device=w.dev)
    ms = event_ms(lambda: core.mirror_subgrid(src, xA, out=outs[0], mirror=outs[1],
                                              masks=(mask, mask), mirror_masks=(mask, mask)),
                  reps)
    nbytes = 16 * (S * S + 2 * xA * xA)
    res["mirror_subgrid"] = {"ms": ms, "bytes": nbytes, "GB_per_s": nbytes / ms / 1e6,
                             "hbm_fraction": nbytes / (ms * 1e-3) / HBM_BYTES_PER_S,
                             "launch": last_launch(core)}
    del fwd, cols
    return res


def agreement(w):
    """Sampled positions of every subgrid, default against real mode, random facets."""
    pairs = mirror_pairs(w.sg_cfgs, w.cfg.image_size, w.cfg.internal_subgrid_size)
    mirrors = {j for _, j in pairs if j is not None}
    xA = w.cfg.max_subgrid_size
    rng = numpy.random.default_rng(20261017)
    pos = torch.from_numpy(rng.choice(xA * xA, 4096, replace=False)).to(w.dev)
    kept = {}
    for real in (False, True):
        w.random_facets()
        store = kept.setdefault(real, {})
        w.run(real, lambda i, t, store=store: store.__setitem__(i, t.reshape(-1)[pos].clone()))
    diff = {"sources": 0.0, "mirrors": 0.0}
    scale = max(float(v.abs().max()) for v in kept[False].values())
    for i, v in kept[True].items():
        d = float((v - kept[False][i]).abs().max())
        key = "mirrors" if i in mirrors else "sources"
        diff[key] = max(diff[key], d)
    return {"max_abs_diff_sources": diff["sources"], "max_abs_diff_mirrors": diff["mirrors"],
            "max_abs_sample": scale, "positions_per_subgrid": 4096,
            "subgrids": len(kept[True])}


def accuracy(w):
    """Point-source facets: 3 pairs against the analytic DFT in both modes."""
    pairs = [p for p in mirror_pairs(w.sg_cfgs, w.cfg.image_size, w.cfg.internal_subgrid_size)
             if p[1] is not None]
    pick = {k for p in (pairs[0], pairs[len(pairs) // 2], pairs[-1]) for k in p}
    res = {}
    for real in (False, True):
        w.point_facets()
        kept = {}
        w.run(real, lambda i, t: kept.__setitem__(i, t.cpu().numpy()) if i in pick else None)
        errs = {}
        for i in sorted(pick):
            sg = w.sg_cfgs[i]
            truth = make_subgrid_from_sources(SOURCES, w.cfg.image_size, sg.size,
                                              [sg.off0, sg.off1], [sg.mask0, sg.mask1])
            errs[f"{sg.off0},{sg.off1}"] = float(numpy.abs(kept[i] - truth).max()
                                                 / numpy.abs(truth).max())
        res["real" if real else "default"] = errs
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--runs", type=int, default=3, help="whole forwards per mode")
    ap.add_argument("--reps", type=int, default=20, help="launches per kernel timing")
    ap.add_argument("--out", default="real_image.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("quick_real_image needs a CUDA device")
    dev = torch.device("cuda", 0)
    result = {"workload": NAME, "facets": f"{len(BLOCK)} x {len(BLOCK)} block {BLOCK}",
              "device": torch.cuda.get_device_name(dev)}
    try:
        result["power_limit_max_sm_clock"] = subprocess.run(
            ["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
            capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        result["power_limit_max_sm_clock"] = "unknown"
    w = Workload(dev)
    pairs = mirror_pairs(w.sg_cfgs, w.cfg.image_size, w.cfg.internal_subgrid_size)
    result["subgrids"] = len(w.sg_cfgs)
    result["computed_real"] = len(pairs)
    result["k2_columns_real"] = len({w.sg_cfgs[i].off0 for i, _ in pairs})
    times = {False: [], True: []}
    for k in range(args.runs + 1):  # the first pair warms both modes up
        for real in (False, True):
            w.random_facets()
            t = w.run(real)
            if k:
                times[real].append(t)
            print(f"run {k} {'real' if real else 'default'}: {t * 1e3:.1f} ms", file=sys.stderr)
    result["forward_ms"] = {"default": [t * 1e3 for t in times[False]],
                            "real": [t * 1e3 for t in times[True]],
                            "default_min": min(times[False]) * 1e3,
                            "real_min": min(times[True]) * 1e3,
                            "speedup_min": min(times[False]) / min(times[True])}
    result["per_launch"] = per_launch(w, args.reps)
    result["agreement"] = agreement(w)
    result["accuracy_vs_dft"] = accuracy(w)
    text = json.dumps(result, indent=1)
    print(text)
    with open(args.out, "w", encoding="ascii") as f:
        f.write(text + "\n")


if __name__ == "__main__":
    main()
