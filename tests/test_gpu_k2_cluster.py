"""
``extract_columns`` (K2) at ``yN = 16384`` on an H100 in the cluster form
(``ExtractColumnsClusterKernel``, the default) against the single-CTA form
(``ExtractColumnsTma4Kernel``, ``sg_variant`` 26).  Both record launch code 10 on the same grid;
``swiftly_b200_debug_last_cluster`` tells them apart.  The same bits on the pinned catalogue row
raw and pre-windowed, at the staging limits, on capped grids (an even cap pairs, an odd one runs
the single-CTA form) and over 67 facets; and the extended-precision spot check on clusters.
"""

import ctypes

import numpy
import pytest
import torch

from tests import k2_cases as kc
from tests import length_cases as lc
from tests.test_gpu_k2_forms import length_pair

pytestmark = pytest.mark.gpu
TMA4_VARIANT = 26  # sg_variant: ExtractColumnsTma4Kernel, the single-CTA form


def last_cluster(core):
    """CTAs per cluster of the last recorded launch."""
    fn = core._lib.swiftly_b200_debug_last_cluster  # pylint: disable=protected-access
    fn.argtypes, fn.restype = [ctypes.c_void_p], ctypes.c_int
    return fn(core._plan)  # pylint: disable=protected-access


def _both(core, oracle, sizes, offs, sg, cap=0, **kw):
    a, e, got = kc.run(core, oracle, sizes, offs, sg, cap=cap, what="cluster form", **kw)
    cluster = last_cluster(core)
    b, _, single = kc.run(core, oracle, sizes, offs, sg, cap=cap, variant=TMA4_VARIANT,
                          what="single-CTA form", **kw)
    assert single == got and last_cluster(core) == 1, single
    for x, y in zip(a, b):
        assert numpy.array_equal(x, y), "the cluster form changes the bits"
    return got, cluster, e


@pytest.mark.parametrize("case", ["row", "boundaries", "caps", "67-facets"])
def test_gpu_cluster_bitwise(case):
    core, oracle = length_pair(16384)
    m, step, sg = core.xM_yN_size, core.facet_off_step, kc.subgrid_offsets(core)
    worst = 0.0
    if case == "row":
        for k, pre in enumerate([False, True]):
            got, cluster, e = _both(core, oracle, [8192] * 2, kc.facet_offsets(core)[:2], sg[k],
                                    prewindowed=pre, seed=k)
            assert got[:3] == (kc.TMA4, 256, 8192) and cluster == 2, (got, cluster)
            worst = max(worst, e)
    elif case == "boundaries":
        for fs in (8192, 8200, 10174):
            got, cluster, e = _both(core, oracle, [fs], [step], sg[2], seed=fs)
            assert got[:3] == kc.boundary_sizes_16384()[fs] and cluster == 2, (got, cluster)
            worst = max(worst, e)
    elif case == "caps":
        for k, cap in enumerate([1, 2, 3, 8]):
            got, cluster, e = _both(core, oracle, [8192, 8192 - 64], [step, -2 * step], sg[2],
                                    cap=cap, prewindowed=k % 2 == 1, seed=cap)
            assert got[3] == cap and cluster == (1 if cap % 2 else 2), (got, cluster)
            worst = max(worst, e)
    else:
        offs = [(k - 5) * step for k in range(67)]
        got, cluster, worst = _both(core, oracle, [2048] * 67, offs, sg[2], shared_input=True,
                                    seed=5)
        assert got[0] == kc.TMA4 and cluster == 2, (got, cluster)
    print(f"\ncluster form, {case}: bitwise equal to the single-CTA form, max rel err {worst:.2e}")
    torch.cuda.empty_cache()


@pytest.mark.parametrize("fs", [8192, 10174])
def test_gpu_extended_precision(fs):
    """Two rows against the centred DFT in extended precision: error <= 1.5 eps log2(yN) of the
    line's RMS."""
    core, _ = length_pair(16384)
    got, ratio = kc.spot_check(core, fs, seed=fs)
    print(f"\n{kc.KERNEL_NAMES[got[0]]} on clusters, yN 16384 fs {fs}: {ratio:.3f} eps log2(yN)")
    assert got[0] == kc.TMA4 and last_cluster(core) == 2 and (got[1] != 0) == (fs <= 8192), got
    assert ratio <= lc.SPOT_BOUND, ratio
    torch.cuda.empty_cache()
