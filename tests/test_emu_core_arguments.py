"""
The argument handling of ``SwiftlyCoreB200`` on the host-emulated kernels
(``tests/core_argument_cases.py``): every launch form of one grouped ``sum_finish_axis`` job and
every mask kind give the same bits; masks of the wrong length and ``launch`` outputs of the wrong
shape or strides raise ``ValueError``.
"""

import pytest

from tests import core_argument_cases as ca
from tests import pair_cases as prc
from tests.emu_support import emu_core_class

PAIR = (256, 512)  # TMA-staged stores up to 256 samples, direct stores above
_cores = {}


def core(pair):
    if pair not in _cores:
        _cores.clear()
        _cores[pair] = emu_core_class()(*prc.small_plan(pair))
    return _cores[pair]


@pytest.mark.parametrize("axis", [1, 0])
@pytest.mark.parametrize("sz", [256, 257], ids=["tma", "direct"])
def test_emu_sum_finish_forms_agree(axis, sz):
    ca.agreement_case(core(PAIR), axis, sz, seed=axis)


@pytest.mark.parametrize("axis", [1, 0])
def test_emu_launch_rejects(axis):
    ca.launch_rejects(core(PAIR), axis, 100)


def test_emu_finish_mask_rejects():
    ca.finish_mask_rejects(core(PAIR))
