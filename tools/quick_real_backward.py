"""
Real-image backward transform at cfg4 (64k[1]-n16k-4k), the benchmark's central 5 x 5 facet block,
all 32 x 32 subgrids, on one GPU: ``SwiftlyBackward(real_image=True).add_subgrid_tasks`` (514
subgrid sides, 510 merges, 17 of 32 columns folded) against the default mode, run alternately in
one process on the same subgrids.

The 1024 subgrids of a cover take 64 GiB, which does not fit next to the 50 GiB of facet
accumulators, so -- as in ``bench.py --direction backward`` -- 32 distinct subgrids, the outputs
of ``SwiftlyForward(real_image=True)`` on the benchmark's real facets (the first 32 it yields),
are fed cyclically.  The identity the real mode rests on holds for any subgrid data, and the
values do not affect the timing.

* whole backward: wall clock from construction to ``finish()`` plus a device synchronise, min over
  ``--runs`` runs per mode after a warm-up pair;
* per launch (CUDA events, mean over ``--reps``): ``merge_mirror_subgrid`` and its share of the
  H100's 3.35 TB/s for its 16 (2 xA^2 + S^2) bytes; K4T (axis 0) and K3T (axis 1) at S = xA + 1
  and at xA; ``finish_facet_real`` against ``finish_facet`` on one facet accumulator;
* agreement: the largest difference between the real-mode facets and Re of the default-mode
  facets over 65536 sampled positions of every facet, relative to the largest sampled value.

Prints one JSON object and writes it to ``--out``.

    python tools/quick_real_backward.py --out real_backward.json
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

from ska_sdp_distributed_fourier_transform_b200 import SwiftlyBackward  # noqa: E402
from ska_sdp_distributed_fourier_transform_b200.api import mirror_pairs  # noqa: E402
from tools.quick_real_image import (  # noqa: E402
    HBM_BYTES_PER_S,
    NAME,
    Workload,
    event_ms,
    last_launch,
)

N_INPUTS = 32
N_SAMPLES = 65536


class BackwardWorkload:
    """The forward workload's configs, and ``N_INPUTS`` subgrids of its real forward."""

    def __init__(self, dev):
        fw = Workload(dev)
        self.cfg, self.dev = fw.cfg, dev
        self.facet_cfgs, self.sg_cfgs = fw.facet_cfgs, fw.sg_cfgs
        fw.random_facets()
        fwd = fw.forward(True)
        self.inputs = []
        for _, task in fwd.iter_subgrid_tasks(self.sg_cfgs):
            self.inputs.append(task.tensor.clone())
            if len(self.inputs) == N_INPUTS:
                break
        del fwd, fw
        torch.cuda.synchronize(dev)
        torch.cuda.empty_cache()
        self.data = [self.inputs[i % N_INPUTS] for i in range(len(self.sg_cfgs))]

    def backward(self, real):
        return SwiftlyBackward(self.cfg, self.facet_cfgs, lru_backward=1, queue_size=8,
                               real_image=real)

    def run(self, real, consumer=None):
        """One whole backward; returns seconds (construction to ``finish()`` and a synchronise).
        ``consumer(j, facet tensor)`` sees every facet after the clock stops."""
        torch.cuda.synchronize(self.dev)
        t0 = time.perf_counter()
        bwd = self.backward(real)
        if real:
            bwd.add_subgrid_tasks(self.sg_cfgs, self.data)
        else:
            for sg, data in zip(self.sg_cfgs, self.data):
                bwd.add_new_subgrid_task(sg, data)
        tasks = bwd.finish()
        torch.cuda.synchronize(self.dev)
        t = time.perf_counter() - t0
        if consumer is not None:
            for j, task in enumerate(tasks):
                consumer(j, task.tensor)
        del bwd, tasks
        torch.cuda.empty_cache()
        return t


def per_launch(w, reps):
    """merge, K4T / K3T at S and xA, finish_facet_real against finish_facet."""
    # pylint: disable=protected-access
    core = w.cfg.core
    xA = w.cfg.max_subgrid_size
    S = 2 * (xA // 2) + 1
    res = {}
    out = torch.empty((S, S), dtype=torch.complex128, device=w.dev)
    ms = event_ms(lambda: core.merge_mirror_subgrid(w.inputs[0], w.inputs[1], out=out), reps)
    nbytes = 16 * (2 * xA * xA + S * S)
    res["merge_mirror_subgrid"] = {"ms": ms, "bytes": nbytes, "GB_per_s": nbytes / ms / 1e6,
                                   "hbm_fraction": nbytes / (ms * 1e-3) / HBM_BYTES_PER_S,
                                   "launch": last_launch(core)}
    # a backward of only the first facet row's column: K4T / K3T as the driver runs them
    bwd = w.backward(True)
    sg = w.sg_cfgs[len(w.sg_cfgs) // 2 + 5]
    for size, data in ((S, out), (xA, w.inputs[0])):
        bwd._add_subgrid(data, sg.off0, sg.off1)
        strips = bwd._strips[size]
        rows = [(strips[r], row) for r, (row, _) in enumerate(bwd._rows)]

        def k4t(data=data, rows=rows):
            core.split_subgrid_axis([data], 0, [sg.off0], [rows], "store")

        column = bwd._column_for(sg.off0)
        groups, offs, targets = [], [], []
        for r, (row, members) in enumerate(bwd._rows):
            groups.append(strips[r])
            offs.append(sg.off1)
            targets.append([(column[j], w.facet_cfgs[j].off1) for j in members])

        def k3t(groups=groups, offs=offs, targets=targets):
            core.split_subgrid_axis(groups, 1, offs, targets, "add")

        k4_ms = event_ms(k4t, reps)
        k4_rec = last_launch(core)
        k3_ms = event_ms(k3t, reps)
        k3_rec = last_launch(core)
        res[f"size_{size}"] = {"K4T_ms": k4_ms, "K3T_ms": k3_ms, "K4T_launch": k4_rec,
                               "K3T_launch": k3_rec}
    del bwd, column, groups, targets
    torch.cuda.empty_cache()
    yN, yB = w.cfg.internal_facet_size, w.cfg.max_facet_size
    acc = torch.empty((yN, yB), dtype=torch.complex128, device=w.dev)
    torch.view_as_real(acc).normal_()
    fc = w.facet_cfgs[0]
    mask = torch.ones(yB, dtype=torch.float64, device=w.dev)
    fout = torch.empty((yB, yB), dtype=torch.complex128, device=w.dev)
    rout = torch.empty((yB, yB), dtype=torch.float64, device=w.dev)
    ms_c = event_ms(lambda: core.finish_facet(acc, fc.off0, yB, 0, out=fout), reps)
    rec_c = last_launch(core)
    ms_r = event_ms(lambda: core.finish_facet_real(acc, fc.off0, yB, 0, out=rout, mask=mask),
                    reps)
    rec_r = last_launch(core)
    res["finish_facet"] = {"ms": ms_c, "launch": rec_c}
    res["finish_facet_real"] = {"ms": ms_r, "launch": rec_r}
    return res


def agreement(w):
    yB = w.cfg.max_facet_size
    rng = numpy.random.default_rng(20261017)
    pos = torch.from_numpy(rng.choice(yB * yB, N_SAMPLES, replace=False)).to(w.dev)
    kept = {}
    for real in (False, True):
        store = kept.setdefault(real, {})
        w.run(real, lambda j, t, store=store: store.__setitem__(
            j, t.reshape(-1)[pos].real.clone()))
    scale = max(float(v.abs().max()) for v in kept[False].values())
    diff = max(float((kept[True][j] - kept[False][j]).abs().max()) for j in kept[False])
    return {"max_abs_diff": diff, "max_abs_sample": scale, "rel": diff / scale,
            "positions_per_facet": N_SAMPLES, "facets": len(kept[True])}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--runs", type=int, default=3, help="whole backwards per mode")
    ap.add_argument("--reps", type=int, default=20, help="launches per kernel timing")
    ap.add_argument("--out", default="real_backward.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("quick_real_backward needs a CUDA device")
    dev = torch.device("cuda", 0)
    result = {"workload": NAME,
              "device": torch.cuda.get_device_name(dev)}
    w = BackwardWorkload(dev)
    result["facets"] = len(w.facet_cfgs)
    pairs = mirror_pairs(w.sg_cfgs, w.cfg.image_size, w.cfg.internal_subgrid_size)
    result["subgrids"] = len(w.sg_cfgs)
    result["subgrid_sides_real"] = len(pairs)
    result["merges_real"] = sum(j is not None for _, j in pairs)
    result["columns_folded_real"] = len({w.sg_cfgs[i].off0 for i, _ in pairs})
    times = {False: [], True: []}
    for k in range(args.runs + 1):  # the first pair warms both modes up
        for real in (False, True):
            t = w.run(real)
            if k:
                times[real].append(t)
            print(f"run {k} {'real' if real else 'default'}: {t * 1e3:.1f} ms", file=sys.stderr)
    result["backward_ms"] = {"default": [t * 1e3 for t in times[False]],
                             "real": [t * 1e3 for t in times[True]],
                             "default_min": min(times[False]) * 1e3,
                             "real_min": min(times[True]) * 1e3,
                             "speedup_min": min(times[False]) / min(times[True])}
    try:  # right after the timed runs: the SM clock is still the loaded one
        result["power_limit_sm_clock_max_sm_clock"] = subprocess.run(
            ["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm",
             "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        result["power_limit_sm_clock_max_sm_clock"] = "unknown"
    result["per_launch"] = per_launch(w, args.reps)
    result["agreement"] = agreement(w)
    text = json.dumps(result, indent=1)
    print(text)
    with open(args.out, "w", encoding="ascii") as f:
        f.write(text + "\n")


if __name__ == "__main__":
    main()
