"""
The argument handling of ``SwiftlyCoreB200`` on the H100 (``tests/core_argument_cases.py``):
every launch form of one grouped ``sum_finish_axis`` job and every mask kind give the same bits,
at a direct and a TMA-staged subgrid size.  ``launch`` gets numpy and float64 device masks only.
"""

import pytest
import torch

from ska_sdp_distributed_fourier_transform_b200.core import SwiftlyCoreB200
from tests import core_argument_cases as ca
from tests import pair_cases as prc

pytestmark = pytest.mark.gpu

PAIRS = [(256, 512), (1024, 4096)]
_cores = {}


def core(pair):
    if pair not in _cores:
        _cores.clear()
        torch.cuda.empty_cache()
        _cores[pair] = SwiftlyCoreB200(*prc.core_plan(pair), device=0)
    return _cores[pair]


@pytest.mark.parametrize("pair", PAIRS, ids=prc.pair_id)
@pytest.mark.parametrize("axis", [1, 0])
@pytest.mark.parametrize("sz", ["tma", "direct"])
def test_gpu_sum_finish_forms_agree(pair, axis, sz):
    size = prc.tma_sizes(pair)[0 if sz == "tma" else 3][0]  # the TMA threshold, and one more
    ca.agreement_case(core(pair), axis, size, launch_kinds=("numpy", "float64"), seed=axis)
