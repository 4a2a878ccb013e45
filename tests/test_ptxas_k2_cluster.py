"""Register and spill budget of K2's cluster form (ExtractColumnsClusterKernel<4096>, the default at
yN = 16384).

Two thread groups of 256 threads take the 64 K-register file at 128 registers per thread.  The
kernel keeps each thread's half of its sub-transform outputs in registers across the CTA and
cluster barriers of the combine; ptxas spills 4 bytes (one loop-invariant shared-memory address,
reloaded once per line).  This test compiles ``dispatch_extract_columns.cu`` for sm_90a with
``-Xptxas -v`` (CUDA 12.9) and pins that figure, beside the single-CTA form's (no spills).
"""

import os
import re
import subprocess

import pytest

from ska_sdp_distributed_fourier_transform_b200 import build

# kernel -> most spill store bytes, most spill load bytes
SPILL_BUDGET = {"ExtractColumnsClusterKernelILi4096E": (4, 4),
                "ExtractColumnsTma4KernelILi4096E": (0, 0)}

_ENTRY = re.compile(r"Compiling entry function '(\S+)'")
_SPILL = re.compile(r"(\d+) bytes spill stores, (\d+) bytes spill loads")
_REGS = re.compile(r"Used (\d+) registers")


@pytest.fixture(scope="module")
def ptxas_report(tmp_path_factory):
    try:
        nvcc = build.nvcc()
    except RuntimeError:
        pytest.skip("nvcc not available")
    src = os.path.join(build.CSRC, "dispatch_extract_columns.cu")
    obj = str(tmp_path_factory.mktemp("ptxas") / "dispatch_extract_columns.o")
    p = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", obj],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, check=False)
    assert p.returncode == 0, p.stdout
    report = {}
    key = None
    for line in p.stdout.splitlines():
        m = _ENTRY.search(line)
        if m:
            key = next((k for k in SPILL_BUDGET if k in m.group(1)), None)
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


@pytest.mark.parametrize("kernel", sorted(SPILL_BUDGET))
def test_k2_4xq_spills(ptxas_report, kernel):
    assert kernel in ptxas_report, f"no ptxas report for {kernel}"
    got = ptxas_report[kernel]
    stores, loads = got["spill"]
    max_st, max_ld = SPILL_BUDGET[kernel]
    assert stores <= max_st and loads <= max_ld, (
        f"{kernel}: {stores} bytes spill stores, {loads} bytes spill loads "
        f"(budget {max_st} / {max_ld})")
    assert got["regs"] <= 128
