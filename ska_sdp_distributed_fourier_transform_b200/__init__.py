"""
B200-native SwiFTly facet<->subgrid distributed Fourier transform hot path.

Drop-in for the compute core of ``ska_sdp_exec_swiftly``: the same
``SwiftlyConfig`` / ``SwiftlyForward`` / ``SwiftlyBackward`` API surface and the
eight-primitive core interface, implemented as hand-written sm_90a CUDA kernels
behind a C ABI (``include/swiftly_b200.h``).  No CPU fallback.
"""

from .api import (  # noqa: F401
    FacetConfig,
    PinnedArena,
    SubgridConfig,
    SwiftlyBackward,
    SwiftlyConfig,
    SwiftlyForward,
    device_tier_bytes,
    make_full_facet_cover,
    make_full_subgrid_cover,
)
from .api_helper import (  # noqa: F401
    check_facet,
    check_subgrid,
    make_facet,
    make_facet_device,
    make_subgrid,
)
from .core import SwiftlyCoreB200  # noqa: F401
from .fourier_algorithm import make_facet_from_sources, make_subgrid_from_sources  # noqa: F401
from .swift_configs import SWIFT_CONFIGS  # noqa: F401

__all__ = [
    "FacetConfig",
    "PinnedArena",
    "SubgridConfig",
    "SwiftlyConfig",
    "SwiftlyForward",
    "SwiftlyBackward",
    "SwiftlyCoreB200",
    "SwiftlyForwardSharded",
    "SwiftlyBackwardSharded",
    "partition_facets",
    "SWIFT_CONFIGS",
    "device_tier_bytes",
    "check_facet",
    "check_subgrid",
    "make_subgrid",
    "make_facet",
    "make_facet_device",
    "make_full_facet_cover",
    "make_full_subgrid_cover",
    "make_facet_from_sources",
    "make_subgrid_from_sources",
]

__version__ = "0.2.0"

_SHARDED = ("SwiftlyBackwardSharded", "SwiftlyForwardSharded", "partition_facets")


def __getattr__(name):
    # the sharded drivers need torch.distributed; everything else (numpy-mode core,
    # sdp_func_compat) must import without it
    if name in _SHARDED:
        from . import distributed  # pylint: disable=import-outside-toplevel

        return getattr(distributed, name)
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")

