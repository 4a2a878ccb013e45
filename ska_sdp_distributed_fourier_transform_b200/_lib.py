"""
ctypes binding of ``libswiftly_b200.so`` (C ABI: ``include/swiftly_b200.h``).

The shared library is built in-tree by ``build.py`` (nvcc, sm_90a) next to this
file.  There is no CPU fallback: if the library is missing, importing the binding
raises ``RuntimeError`` with the build command.
"""

import ctypes
import os
import threading

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_NAME = "libswiftly_b200.so"
LIB_PATH = os.path.join(HERE, LIB_NAME)

OK = 0
EINVAL = -1
ECUDA = -2
EUNSUPPORTED = -3

DEVICE = 0
HOST = 1


class Lines(ctypes.Structure):
    """``swiftly_b200_lines``: a batch of strided 1-D lines of complex128 samples."""

    _fields_ = [
        ("data", ctypes.c_void_p),
        ("n_lines", ctypes.c_int64),
        ("size", ctypes.c_int64),
        ("line_stride", ctypes.c_int64),
        ("elem_stride", ctypes.c_int64),
        ("location", ctypes.c_int32),
    ]


class Source(ctypes.Structure):
    """``swiftly_b200_source``: one input of the fused sum-and-finish kernel."""

    _fields_ = [
        ("data", ctypes.c_void_p),
        ("line_stride", ctypes.c_int64),
        ("elem_stride", ctypes.c_int64),
        ("size", ctypes.c_int64),
        ("facet_off", ctypes.c_int64),
    ]


class SplitTarget(ctypes.Structure):
    """``swiftly_b200_split_target``: one output of the fused subgrid split kernel."""

    _fields_ = [
        ("data", ctypes.c_void_p),
        ("n_lines", ctypes.c_int64),
        ("line_stride", ctypes.c_int64),
        ("elem_stride", ctypes.c_int64),
        ("facet_off", ctypes.c_int64),
    ]


SPLIT_STORE = 0
SPLIT_ADD = 1

_PLAN = ctypes.c_void_p
_LINES_P = ctypes.POINTER(Lines)
_D_P = ctypes.POINTER(ctypes.c_double)

# name -> (restype, argtypes); every symbol declared in include/swiftly_b200.h
SYMBOLS = {
    "swiftly_b200_create": (
        ctypes.c_int,
        [ctypes.c_double, ctypes.c_int64, ctypes.c_int64, ctypes.c_int64, _D_P, _D_P,
         ctypes.c_int, ctypes.POINTER(_PLAN)],
    ),
    "swiftly_b200_destroy": (None, [_PLAN]),
    "swiftly_b200_last_error": (ctypes.c_char_p, []),
    "swiftly_b200_build_info": (ctypes.c_char_p, []),
    "swiftly_b200_contribution_size": (ctypes.c_int64, [_PLAN]),
    "swiftly_b200_release_scratch": (None, [_PLAN]),
    "swiftly_b200_prepare_facet": (ctypes.c_int, [_PLAN, _LINES_P, _LINES_P, ctypes.c_int64, ctypes.c_void_p]),
    "swiftly_b200_prepare_facet_windowed": (ctypes.c_int, [_PLAN, _LINES_P, _LINES_P, ctypes.c_int64, ctypes.c_void_p]),
    "swiftly_b200_extract_from_facet": (ctypes.c_int, [_PLAN, _LINES_P, _LINES_P, ctypes.c_int64, ctypes.c_void_p]),
    "swiftly_b200_add_to_subgrid": (ctypes.c_int, [_PLAN, _LINES_P, _LINES_P, ctypes.c_int64, ctypes.c_void_p]),
    "swiftly_b200_finish_subgrid": (ctypes.c_int, [_PLAN, _LINES_P, _LINES_P, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p]),
    "swiftly_b200_prepare_subgrid": (ctypes.c_int, [_PLAN, _LINES_P, _LINES_P, ctypes.c_int64, ctypes.c_void_p]),
    "swiftly_b200_extract_from_subgrid": (ctypes.c_int, [_PLAN, _LINES_P, _LINES_P, ctypes.c_int64, ctypes.c_void_p]),
    "swiftly_b200_add_to_facet": (ctypes.c_int, [_PLAN, _LINES_P, _LINES_P, ctypes.c_int64, ctypes.c_void_p]),
    "swiftly_b200_finish_facet": (ctypes.c_int, [_PLAN, _LINES_P, _LINES_P, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p]),
    "swiftly_b200_finish_facet_real": (ctypes.c_int, [_PLAN, _LINES_P, _LINES_P, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p]),
    "swiftly_b200_finish_facet_real_half": (ctypes.c_int, [_PLAN, _LINES_P, _LINES_P, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p]),
    "swiftly_b200_prepare_facet_real_half": (ctypes.c_int, [_PLAN, _LINES_P, _LINES_P, ctypes.c_int64, ctypes.c_void_p]),
    "swiftly_b200_extract_column": (ctypes.c_int, [_PLAN, _LINES_P, _LINES_P, ctypes.c_int64, ctypes.c_int64, ctypes.c_void_p]),
    "swiftly_b200_sum_finish_axis": (ctypes.c_int, [_PLAN, ctypes.POINTER(Source), ctypes.c_int, _LINES_P, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p]),
    "swiftly_b200_sum_finish_axis_grouped": (ctypes.c_int, [_PLAN, ctypes.POINTER(Source), ctypes.POINTER(ctypes.c_int32), ctypes.c_int, _LINES_P, ctypes.c_int64, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p]),
    "swiftly_b200_sum_finish_axis_batched": (ctypes.c_int, [_PLAN, ctypes.POINTER(Source), ctypes.POINTER(ctypes.c_int32), ctypes.c_int, _LINES_P, ctypes.c_int64, ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_void_p), ctypes.c_void_p]),
    "swiftly_b200_sum_finish_axis_scattered": (ctypes.c_int, [_PLAN, ctypes.POINTER(Source), ctypes.POINTER(ctypes.c_int32), ctypes.c_int, _LINES_P, ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_void_p), ctypes.c_void_p]),
    "swiftly_b200_peer_signal": (ctypes.c_int, [_PLAN, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int64, ctypes.c_void_p]),
    "swiftly_b200_peer_wait": (ctypes.c_int, [_PLAN, ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_double, ctypes.c_void_p, ctypes.c_void_p]),
    "swiftly_b200_extract_columns": (ctypes.c_int, [_PLAN, ctypes.c_int, _LINES_P, _LINES_P, ctypes.c_int64, ctypes.POINTER(ctypes.c_int64), ctypes.c_void_p]),
    "swiftly_b200_extract_columns_windowed": (ctypes.c_int, [_PLAN, ctypes.c_int, _LINES_P, _LINES_P, ctypes.c_int64, ctypes.POINTER(ctypes.c_int64), ctypes.c_void_p]),
    "swiftly_b200_mirror_subgrid": (ctypes.c_int, [_PLAN, _LINES_P, _LINES_P, _LINES_P, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    "swiftly_b200_merge_mirror_subgrid": (ctypes.c_int, [_PLAN, _LINES_P, _LINES_P, _LINES_P, ctypes.c_void_p]),
    "swiftly_b200_subgrid_to_facets": (ctypes.c_int, [_PLAN, ctypes.c_int, _LINES_P, _LINES_P, ctypes.POINTER(ctypes.c_int64), ctypes.c_int64, ctypes.c_void_p]),
    "swiftly_b200_fold_column": (ctypes.c_int, [_PLAN, ctypes.c_int, _LINES_P, _LINES_P, ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_void_p), ctypes.c_int64, ctypes.c_void_p]),
    "swiftly_b200_sum_finish_axis_supported": (ctypes.c_int, [_PLAN]),
    "swiftly_b200_split_subgrid_axis": (ctypes.c_int, [_PLAN, _LINES_P, ctypes.c_int, ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(SplitTarget), ctypes.POINTER(ctypes.c_int32), ctypes.c_int, ctypes.c_void_p]),
    "swiftly_b200_split_axis_supported": (ctypes.c_int, [_PLAN]),
}

_lock = threading.Lock()
_lib = None


def load(path=None):
    """Load (once) and return the bound shared library."""
    global _lib  # pylint: disable=global-statement
    with _lock:
        if _lib is not None and path is None:
            return _lib
        p = path or LIB_PATH
        if not os.path.exists(p):
            raise RuntimeError(
                f"{p} not found: the CUDA extension is not built. Run "
                "`python -c 'import __graft_entry__ as g; g.build()'` (needs nvcc); "
                "there is no CPU fallback."
            )
        lib = ctypes.CDLL(p)
        for name, (restype, argtypes) in SYMBOLS.items():
            fn = getattr(lib, name)  # AttributeError if the ABI is incomplete
            fn.restype = restype
            fn.argtypes = argtypes
        if path is None:
            _lib = lib
        return lib


def last_error(lib):
    msg = lib.swiftly_b200_last_error()
    return msg.decode() if msg else ""


def check(lib, rc):
    """Translate a C status into the Python exception the reference would raise."""
    if rc == OK:
        return
    msg = last_error(lib)
    if rc == EINVAL:
        raise ValueError(msg)
    if rc == EUNSUPPORTED:
        raise NotImplementedError(msg)
    raise RuntimeError(msg)
