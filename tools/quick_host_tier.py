"""
Host tier at cfg4 (64k[1]-n16k-4k) on one GPU: the prepared facets (forward) or the facet
accumulators (backward) in pinned host memory, the m-row window of each on the device.

Runs the full 8 x 8 facet cover when pinning its facet arrays (128 GiB) stays under half of the
host's MemAvailable, else the largest centred n x n block (n >= 6) that does not fit the device
tier and whose arrays do fit that limit.  On a host with less memory than that it runs the largest
block that fits the limit (the forward's pinned arena passed as ``bf_f_buffers`` selects the host
tier, the backward gets a device budget of 1 byte).  The JSON says which.
Facets are painted on the device from point sources; subgrids (forward) and facets (backward) are
checked against the point-source truth.  Writes one JSON file.

    python tools/quick_host_tier.py --direction both --out host_tier.json
"""

import argparse
import json
import os
import sys
import time

import numpy
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ska_sdp_distributed_fourier_transform_b200 import (  # noqa: E402
    SWIFT_CONFIGS,
    PinnedArena,
    SwiftlyBackward,
    SwiftlyConfig,
    SwiftlyForward,
    check_facet,
    device_tier_bytes,
    make_facet_device,
    make_full_facet_cover,
    make_full_subgrid_cover,
    make_subgrid,
)

NAME = "64k[1]-n16k-4k"
# inside the facets of every centred block (image coordinates within +-12288 of the centre)
SOURCES = [(1.0, 1, 0), (0.5, -7000, 5001), (0.25, 9011, -3777)]


def mem_available():
    with open("/proc/meminfo", encoding="ascii") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    raise RuntimeError("no MemAvailable in /proc/meminfo")


def choose_block(p, host_avail, dev_free):
    """``(n, bytes of the facet arrays, device budget)``: the full cover, else the largest centred
    block that does not fit the device tier; on a host with too little memory for either, the
    largest block that fits, with a budget of 1 byte so that it still runs the host tier."""
    yN, yB, n_full = p["yN_size"], p["yB_size"], p["N"] // p["yB_size"]
    m = p["xM_size"] * yN // p["N"]
    for n in range(n_full, 0, -1):
        arrays = 16 * n * n * yN * yB
        need = device_tier_bytes("forward", yN, m, [yB] * n * n, 1, n, p["xA_size"])
        if arrays < host_avail // 2 and (n == n_full or need > dev_free):
            return n, arrays, None
    for n in range(n_full, 0, -1):
        arrays = 16 * n * n * yN * yB
        if arrays < host_avail // 2:
            return n, arrays, 1
    return None, 0, None


def block_cover(cfg, n):
    """The n x n facets nearest the image centre (facet offset 0, offsets taken mod N)."""
    N = cfg.image_size
    cover = make_full_facet_cover(cfg)
    offs = sorted({c.off0 for c in cover}, key=lambda o: (min(o, N - o), o))
    keep = set(offs[:n])
    return [c for c in cover if c.off0 in keep and c.off1 in keep]


def copy_rate(nbytes, dev):
    """GB/s of one pinned host -> device and one device -> host copy of ``nbytes``."""
    host = PinnedArena([(nbytes // 16, 1)], dev)
    d = torch.empty(nbytes // 16, dtype=torch.complex128, device=dev)
    h = host.views[0].view(-1)
    out = []
    for dst, src in ((d, h), (h, d)):
        dst.copy_(src, non_blocking=True)
        a = ev()
        dst.copy_(src, non_blocking=True)
        b = ev()
        b.synchronize()
        out.append(nbytes / (a.elapsed_time(b) / 1e3) / 1e9)
    host.release()
    return out


def rel_err(approx, truth):
    return float(numpy.abs(approx - truth).max() / max(numpy.abs(truth).max(), 1e-300))


def elapsed(pairs):
    return sum(a.elapsed_time(b) for a, b in pairs) / 1e3


def ev():
    e = torch.cuda.Event(enable_timing=True)
    e.record()
    return e


def run_forward(cfg, facet_cfgs, sg_cfgs, dev):
    N = cfg.image_size
    tasks = [(fc, (lambda fc=fc: make_facet_device(N, fc, SOURCES, dev))) for fc in facet_cfgs]
    # the pinned arena is passed in (as a caller reusing it across transforms would), so that
    # stage 1 is timed without the pinning
    arena = PinnedArena([(cfg.internal_facet_size, fc.size) for fc in facet_cfgs], dev)
    fwd = SwiftlyForward(cfg, tasks, lru_forward=1, queue_size=4, bf_f_buffers=arena.views)
    assert fwd.host_tier, "the device tier was selected"
    e0 = ev()
    bf = fwd._get_BF_Fs()  # pylint: disable=protected-access
    s1 = [(e0, ev())]
    s2, s3, check = [], [], {}
    probe = {0, len(sg_cfgs) // 2, len(sg_cfgs) - 1}
    for i, sg in enumerate(sg_cfgs):
        a = ev()
        cols = fwd.get_NMBF_BFs_off0(sg.off0, bf)
        b = ev()
        out = fwd._gen_subgrid(sg, cols)  # pylint: disable=protected-access
        c = ev()
        s2.append((a, b))
        s3.append((b, c))
        if i in probe:
            check[i] = (sg, out.cpu().numpy())
    torch.cuda.synchronize()
    h2d, d2h = fwd.copied_bytes
    t2 = elapsed(s2)
    res = {
        "pin_s": arena.seconds, "stage1_s": elapsed(s1), "stage2_s_on_compute_stream": t2,
        "stage3_s": elapsed(s3), "h2d_bytes": h2d, "d2h_bytes_stage1": d2h,
        "d2h_GBps_over_stage1": d2h / elapsed(s1) / 1e9,
        "h2d_rows_per_facet": fwd.h2d_rows,
        "subgrid_max_rel_err": max(rel_err(out, make_subgrid(N, sg, SOURCES))
                                   for sg, out in check.values()),
        "peak_device_GiB": torch.cuda.max_memory_allocated() / 2**30,
    }
    arena.release()
    return res


def subgrid_device(N, sg, dev):
    """``make_subgrid`` of SOURCES computed on the device (separable phases, reduced mod N)."""
    size = sg.size
    out = torch.zeros((size, size), dtype=torch.complex128, device=dev)
    c0 = torch.arange(sg.off0 - size // 2, sg.off0 + (size + 1) // 2, device=dev)
    c1 = torch.arange(sg.off1 - size // 2, sg.off1 + (size + 1) // 2, device=dev)
    for intensity, x0, x1 in SOURCES:
        e0 = torch.exp(2j * numpy.pi / N * torch.remainder(c0 * x0, N).to(torch.float64))
        e1 = torch.exp(2j * numpy.pi / N * torch.remainder(c1 * x1, N).to(torch.float64))
        out += (intensity / N**2) * torch.outer(e0, e1)
    for axis, mask in enumerate([sg.mask0, sg.mask1]):
        if mask is not None:
            m = torch.as_tensor(numpy.asarray(mask, dtype=float), device=dev)
            out *= m[:, None] if axis == 0 else m[None, :]
    return out


def run_backward(cfg, facet_cfgs, sg_cfgs, budget):
    N = cfg.image_size
    bwd = SwiftlyBackward(cfg, facet_cfgs, lru_backward=1, queue_size=4, device_budget=budget)
    assert bwd.host_tier, "the device tier was selected"
    gen, fold = [], []
    for sg in sg_cfgs:
        t0 = time.perf_counter()
        data = subgrid_device(N, sg, torch.device("cuda", 0))
        gen.append(time.perf_counter() - t0)
        a = ev()
        bwd.add_new_subgrid_task(sg, data)
        fold.append((a, ev()))
    a = ev()
    tasks = bwd.finish()
    fin = [(a, ev())]
    torch.cuda.synchronize()
    h2d, d2h = bwd.copied_bytes
    probe = [0, len(facet_cfgs) // 2, len(facet_cfgs) - 1]
    res = {
        "pin_s": bwd.arena.seconds, "subgrid_gen_enqueue_s": sum(gen),
        "add_subgrids_s_incl_pin": elapsed(fold), "finish_s": elapsed(fin),
        "h2d_bytes": h2d, "d2h_bytes": d2h,
        "h2d_rows_per_facet": bwd.h2d_rows, "zeroed_rows_per_facet": bwd.zeroed_rows,
        "d2h_rows_per_facet": bwd.d2h_rows,
        "facet_rms_err": max(check_facet(N, facet_cfgs[j], tasks[j].result(), SOURCES)
                             for j in probe),
        "peak_device_GiB": torch.cuda.max_memory_allocated() / 2**30,
    }
    bwd.arena.release()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n", maxsplit=1)[0])
    ap.add_argument("--direction", choices=["forward", "backward", "both"], default="both")
    ap.add_argument("--out", default="host_tier.json", help="JSON file to write")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("quick_host_tier needs a CUDA device")
    dev = torch.device("cuda", 0)
    p = SWIFT_CONFIGS[NAME]
    host_avail = mem_available()
    dev_free, dev_total = torch.cuda.mem_get_info(dev)
    n, arrays, budget = choose_block(p, host_avail, dev_free)
    props = torch.cuda.get_device_properties(dev)
    result = {"workload": NAME, "gpu": props.name, "host_MemAvailable_GiB": host_avail / 2**30,
              "device_free_GiB": dev_free / 2**30, "device_total_GiB": dev_total / 2**30}
    try:
        import subprocess  # pylint: disable=import-outside-toplevel
        result["power_limit"] = subprocess.run(
            ["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
            capture_output=True, text=True, check=False).stdout.strip()
    except OSError:
        result["power_limit"] = "unknown"
    if n is None:
        result["error"] = "not even one facet array fits half of MemAvailable"
    else:
        result["facet_block"] = f"{n}x{n}" + (
            " (full cover)" if n == p["N"] // p["yB_size"]
            else " (centred block; the full cover does not fit half of MemAvailable)"
            if budget is None else
            " (centred block; no block beyond the device tier fits half of MemAvailable, so the "
            "host tier is selected with device_budget=1)")
        result["pinned_GiB_per_direction"] = arrays / 2**30
        cfg = SwiftlyConfig(W=p["W"], fov=1.0, N=p["N"], yB_size=p["yB_size"],
                            yN_size=p["yN_size"], xA_size=p["xA_size"], xM_size=p["xM_size"])
        facet_cfgs = block_cover(cfg, n)
        sg_cfgs = make_full_subgrid_cover(cfg)
        result["subgrids"] = len(sg_cfgs)
        result["facets"] = len(facet_cfgs)
        result["pinned_copy_GBps_h2d_d2h_1GiB"] = copy_rate(1 << 30, dev)
        if args.direction in ("forward", "both"):
            result["forward"] = run_forward(cfg, facet_cfgs, sg_cfgs, dev)
            write(args.out, result)
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        if args.direction in ("backward", "both"):
            result["backward"] = run_backward(cfg, facet_cfgs, sg_cfgs, budget)
    write(args.out, result)
    print(json.dumps(result))


def write(path, result):
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "w", encoding="utf-8") as f:
        json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
