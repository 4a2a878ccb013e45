"""Register and spill budget of the two-group fused subgrid kernel (SubgridAxisKernelPP).

Two thread groups of 256 threads share the 64 K-register file at 128 registers per thread, and
the kernel's 209 KiB of shared memory leave about 28 KB of L1 per SM: whatever ptxas spills
goes out to L2 and is reloaded inside the latency-bound transform passes.  These tests compile
``dispatch_subgrid_axis.cu`` for sm_90a with ``-Xptxas -v`` (CUDA 12.9) and pin the spill
bytes: none at (m, xM) = (1024, 4096), the kernel the cfg4 step spends most of its time in, and
no more than today's figures for the other instantiations.
"""

import os
import re
import subprocess

import pytest

from ska_sdp_distributed_fourier_transform_b200 import build

# (m, xM, TOKENS) -> most spill store bytes, most spill load bytes
SPILL_BUDGET = {
    (1024, 4096, False): (0, 0),
    (2048, 4096, False): (0, 0),
    (1024, 2048, False): (0, 0),
    (512, 2048, False): (28, 72),
    (512, 1024, False): (38, 88),
    (256, 1024, False): (0, 0),
    (256, 512, False): (0, 0),
    (128, 512, False): (0, 0),
    # with the LSU token between the groups (sg_variant 2)
    (1024, 4096, True): (0, 0),
    (2048, 4096, True): (0, 0),
    (1024, 2048, True): (0, 0),
    (512, 2048, True): (24, 64),
    (512, 1024, True): (34, 84),
    (256, 1024, True): (0, 0),
    (256, 512, True): (0, 0),
    (128, 512, True): (0, 0),
}

_ENTRY = re.compile(r"Compiling entry function '(\S+)'")
_KERNEL = re.compile(r"SubgridAxisKernelPPILi(\d+)ELi(\d+)ELb([01])E")
_SPILL = re.compile(r"(\d+) bytes spill stores, (\d+) bytes spill loads")
_REGS = re.compile(r"Used (\d+) registers")


@pytest.fixture(scope="module")
def ptxas_report(tmp_path_factory):
    try:
        nvcc = build.nvcc()
    except RuntimeError:
        pytest.skip("nvcc not available")
    src = os.path.join(build.CSRC, "dispatch_subgrid_axis.cu")
    obj = str(tmp_path_factory.mktemp("ptxas") / "dispatch_subgrid_axis.o")
    p = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", obj],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, check=False)
    assert p.returncode == 0, p.stdout
    report = {}
    key = None
    for line in p.stdout.splitlines():
        m = _ENTRY.search(line)
        if m:
            k = _KERNEL.search(m.group(1))
            key = (int(k.group(1)), int(k.group(2)), k.group(3) == "1") if k else None
            continue
        if key is None:
            continue
        m = _SPILL.search(line)
        if m:
            report.setdefault(key, {})["spill"] = (int(m.group(1)), int(m.group(2)))
        m = _REGS.search(line)
        if m:
            report.setdefault(key, {})["regs"] = int(m.group(1))
    return report


@pytest.mark.parametrize("key", sorted(SPILL_BUDGET),
                         ids=lambda k: "m%d_xM%d%s" % (k[0], k[1], "_token" if k[2] else ""))
def test_two_group_kernel_spills(ptxas_report, key):
    assert key in ptxas_report, "no ptxas report for SubgridAxisKernelPP<%d, %d>" % key[:2]
    got = ptxas_report[key]
    stores, loads = got["spill"]
    max_st, max_ld = SPILL_BUDGET[key]
    assert stores <= max_st and loads <= max_ld, (
        "SubgridAxisKernelPP<%d, %d, %s>: %d bytes spill stores, %d bytes spill loads "
        "(budget %d / %d)" % (key + (stores, loads, max_st, max_ld)))
    assert got["regs"] <= 128
