"""
Named SwiFTly parameter sets (``SWIFT_CONFIGS[name]`` -> ``SwiftlyConfig`` keyword dict).

* the four BASELINE benchmark sets (none of which is in the reference catalogue, SURVEY.md
  section 8d) and the reference's unit-test set;
* the reference's own catalogue (244 entries, ``swift_configs.py`` there), carried as a data
  table ``swift_configs.json`` exported by ``tools/make_catalogue.py`` -- same names, same
  keys (``W, fov, N, Nx, yB_size, yN_size, yP_size, xA_size, xM_size``).

``runnable(params)`` tells whether this build can transform a set: every FFT length
(``yN_size``, ``xM_size``, ``xM_size*yN_size/N``) must be ``F * 2^k`` with ``F <= 16`` and
``16 <= 2^k <= 8192`` -- true for all 244 catalogue entries (factors 3, 5, 7, 9 and lengths up
to 65536 go through the generic split-F kernel).  Anything else raises
``NotImplementedError`` when a transform is requested.

``fused_forward(params)`` tells whether the fused forward kernels (``sum_finish_axis``) exist
for the set's ``(m, xM)`` pair, ``m = xM_size * yN_size / N``.  They do for every catalogue
entry: power-of-two pairs with ``xM / m`` in {1, 2, 4, 8}, and the mixed-radix pairs
(128, 384), (160, 320), (192, 384), (224, 448).  Other runnable sets take the forward path
primitive by primitive.
"""

import json
import os

_BASELINE = {
    # reference tests/test_core.py:20-27, tests/test_api.py:32-40
    "1k[1]-n512-256": dict(W=13.5625, fov=1.0, N=1024, yB_size=416, yN_size=512,
                           xA_size=228, xM_size=256),
    # BASELINE configs[1..3]
    "8k[1]-n4k-2k": dict(W=13.5625, fov=1.0, N=8192, yB_size=2048, yN_size=4096,
                         xA_size=1024, xM_size=2048),
    "32k[1]-n8k-4k": dict(W=13.5625, fov=1.0, N=32768, yB_size=4096, yN_size=8192,
                          xA_size=2048, xM_size=4096),
    "64k[1]-n16k-4k": dict(W=13.5625, fov=1.0, N=65536, yB_size=8192, yN_size=16384,
                           xA_size=2048, xM_size=4096),
}


def _load_catalogue():
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "swift_configs.json")
    out = {}
    if os.path.exists(path):
        with open(path) as f:
            table = json.load(f)
        cols = table["columns"][1:]
        for row in table["rows"]:
            out[row[0]] = {k: v for k, v in zip(cols, row[1:]) if v is not None}
    return out


SWIFT_CONFIGS = _load_catalogue()
SWIFT_CONFIGS.update(_BASELINE)


def fft_length_supported(n):
    """``n = F * 2^k`` with ``F <= 16`` and ``16 <= 2^k <= 8192`` (or a power of two <= 16384)."""
    if n < 16 or n % 2:
        return False
    m = 1
    while n % (2 * m) == 0 and 2 * m <= 8192:
        m *= 2
    return m >= 16 and n // m <= 16


def runnable(params):
    """True if this build has kernels for every FFT length of the parameter set."""
    N, yN, xM = params["N"], params["yN_size"], params["xM_size"]
    return all(fft_length_supported(s) for s in (yN, xM, xM * yN // N))


# (m, xM) pairs with a fused subgrid kernel: SW_SG_PAIRS in csrc/dispatch_subgrid_axis.cu
FUSED_FORWARD_PAIRS = frozenset([
    (32, 64), (32, 128), (64, 128), (64, 256), (128, 256), (128, 512), (256, 512), (256, 1024),
    (512, 1024), (512, 2048), (1024, 2048), (1024, 4096), (2048, 4096), (2048, 8192),
    (128, 1024), (256, 256), (128, 384), (160, 320), (192, 384), (224, 448),
])


def fused_forward(params):
    """True if the fused forward kernels exist for the set's ``(m, xM)`` pair (every catalogue
    entry; see the module docstring)."""
    N, yN, xM = params["N"], params["yN_size"], params["xM_size"]
    return (xM * yN // N, xM) in FUSED_FORWARD_PAIRS
