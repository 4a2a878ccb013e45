"""
``SwiftlyCoreB200`` -- the eight SwiFTly processing primitives on a B200.

Drop-in for the reference's core objects (``SwiftlyCore`` numpy backend,
``fourier_transform/core.py:20-484`` and ``SwiftlyCoreFunc`` native adapter,
``core.py:487-929``): same constructor ``(W, N, xM_size, yN_size)``, same
attributes and properties, same method names, argument meaning and error
behaviour.  Every method forwards to the hand-written CUDA kernels behind the C
ABI of ``include/swiftly_b200.h`` -- there is no numpy implementation in here
and no fallback.

Arrays may be
  * ``numpy.ndarray`` (host): the library stages them through device memory
    (H2D, kernel, D2H) -- this is the mode the reference's unit tests use; or
  * ``torch.Tensor`` on a CUDA device (complex128): used in place on the
    current torch stream, results are device tensors -- the fast path used by
    ``SwiftlyForward`` / ``SwiftlyBackward``.

Masks (0/1 sample weights, or None) may be numpy arrays or tensors of any float dtype on any
device: each is converted to a contiguous float64 array where the call's output lives, and must
have as many samples as the output has along the axis it masks (``ValueError`` otherwise).
"""

import ctypes

import numpy

from . import _lib
from .pswf import window_tables

try:  # torch is plumbing (device memory, streams); numpy mode works without it
    import torch
except ImportError:  # pragma: no cover
    torch = None


def _is_tensor(a):
    return torch is not None and isinstance(a, torch.Tensor)


def split_launches(group_sizes, max_groups=16, max_targets=64):
    """Kernel launches of one ``split_subgrid_axis`` call with these targets per group: the
    library cuts a group into pieces of at most 64 targets and packs pieces in order into
    launches of at most 16 pieces and 64 targets (capi_backward.cu)."""
    pieces = [min(max_targets, n - k) for n in group_sizes if n > 0
              for k in range(0, n, max_targets)]
    launches, groups, used = 0, 0, 0
    for p in pieces:
        if launches == 0 or groups == max_groups or used + p > max_targets:
            launches, groups, used = launches + 1, 0, 0
        groups, used = groups + 1, used + p
    return launches


class PreparedSumFinish:
    """Reusable argument block of a grouped ``sum_finish_axis`` launch (see
    :meth:`SwiftlyCoreB200.prepare_sum_finish`)."""

    # pylint: disable=too-many-instance-attributes,protected-access
    def __init__(self, core, groups, axis, n_lines, size, out_strides):
        if axis not in (0, 1):
            raise ValueError(f"Invalid axis {axis}")
        self.core = core
        self.axis = axis
        self.n_groups = len(groups)
        # (the sources must outlive the block)
        self._arr, self._sizes, self._keep = core._sources(groups, axis, n_lines)
        self._offs = (ctypes.c_int64 * self.n_groups)()
        self._mptrs = (ctypes.c_void_p * self.n_groups)()
        self._optrs = (ctypes.c_void_p * self.n_groups)()
        self._dout = _lib.Lines(0, int(n_lines), int(size), int(out_strides[0]),
                                int(out_strides[1]), _lib.DEVICE)
        # shape and strides of one group's output tensor, whose lines run along the other axis
        step = 1 if axis == 1 else -1
        self._shape = (int(n_lines), int(size))[::step]
        self._strides = (int(out_strides[0]), int(out_strides[1]))[::step]

    def _check_out(self, o, k=0):
        """``o`` (after its first ``k`` dimensions) must be a group's output."""
        self.core._check_tensor(o)
        shape, strides = tuple(o.shape)[k:], o.stride()[k:]
        if o.dtype != torch.complex128 or shape != self._shape or strides != self._strides:
            raise ValueError(f"output has shape {shape}, strides {strides} and dtype {o.dtype}; "
                             f"the block writes {self._shape}, strides {self._strides}, "
                             f"complex128")

    def launch(self, subgrid_offs, masks=None, out=None, out_group_stride=0, outs=None,
               n_groups=None, out_ptrs=None, stream_of=None):
        """Launch for the first ``n_groups`` groups (default: all).

        :param subgrid_offs: one offset per group
        :param masks: None or one mask / None per group of the block's ``size`` samples (a mask
            object repeated for consecutive groups is converted once)
        :param out, out_group_stride: group 0's output, or the outputs of all groups stacked
            along a leading axis of stride ``out_group_stride``, or
        :param outs: one output tensor per group (same shape / strides, different buffers), or
        :param out_ptrs: their device addresses (ints) with ``stream_of`` a tensor on the device.
            Raw addresses cannot be checked: each must hold a group's output with the shape and
            strides given to :meth:`SwiftlyCoreB200.prepare_sum_finish`
        """
        n = self.n_groups if n_groups is None else int(n_groups)
        core = self.core
        if out_ptrs is not None:
            core._check_tensor(stream_of)
            like = stream_of
        elif outs is not None:
            if len(outs) < n:
                raise ValueError(f"{len(outs)} outputs for {n} groups")
            for o in outs[:n]:
                self._check_out(o)
            like, out_ptrs = outs[0], [o.data_ptr() for o in outs]
        else:
            k = 1 if out.dim() == 3 else 0  # the outputs of all groups stacked
            if n > (out.shape[0] if k else 1) or (k and out.stride(0) != out_group_stride):
                raise ValueError(f"out of shape {tuple(out.shape)} and strides {out.stride()} "
                                 f"does not hold {n} groups {out_group_stride} samples apart")
            self._check_out(out, k)
            like = out
        keep, prev, ptr = [], (), None
        for g in range(n):
            self._offs[g] = int(subgrid_offs[g])
            mk = None if masks is None else masks[g]
            if mk is not prev:  # the drivers pass one mask object for many groups
                prev, ptr = mk, core._mask_ptr(mk, like, self._dout.size, keep)
            self._mptrs[g] = ptr
        if out is None:
            for g in range(n):
                self._optrs[g] = out_ptrs[g]
            rc = core._lib.swiftly_b200_sum_finish_axis_scattered(
                core._plan, self._arr, self._sizes, n, ctypes.byref(self._dout), self._optrs,
                self._offs, self._mptrs, core._stream(like))
        else:
            self._dout.data = out.data_ptr()
            rc = core._lib.swiftly_b200_sum_finish_axis_batched(
                core._plan, self._arr, self._sizes, n, ctypes.byref(self._dout),
                int(out_group_stride), self._offs, self._mptrs, core._stream(out))
        _lib.check(core._lib, rc)


class SwiftlyCoreB200:
    """Streaming distributed Fourier transform primitives, CUDA (sm_90a) backend.

    :param W: PSWF parameter (grid-space support)
    :param N: total image size
    :param xM_size: padded subgrid size
    :param yN_size: padded facet size
    :param device: CUDA device index (default: torch's current device, else 0)
    """

    # pylint: disable=too-many-public-methods

    def __init__(self, W, N, xM_size, yN_size, device=None):
        self.W = W
        self.N = N
        self.xM_size = xM_size
        self.yN_size = yN_size
        self.check_params()
        self.xM_yN_size = self.xM_size * self.yN_size // self.N
        if device is None:
            device = 0
            if torch is not None and torch.cuda.is_available():
                device = torch.cuda.current_device()
        self.device = int(device)
        self._lib = _lib.load()
        Fb, Fn = window_tables(W, N, xM_size, yN_size)
        self._Fb = Fb
        self._Fn = Fn
        plan = ctypes.c_void_p()
        rc = self._lib.swiftly_b200_create(
            float(W), int(N), int(xM_size), int(yN_size),
            Fb.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
            Fn.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
            self.device, ctypes.byref(plan),
        )
        _lib.check(self._lib, rc)
        self._plan = plan

    def __del__(self):
        plan = getattr(self, "_plan", None)
        if plan is not None and plan.value:
            try:
                self._lib.swiftly_b200_destroy(plan)
            except Exception:  # pylint: disable=broad-except
                pass
            self._plan = None

    # pickle support like SwiftlyCoreFunc (core.py:513-525): rebuild from parameters
    def __getstate__(self):
        return {"W": self.W, "N": self.N, "xM_size": self.xM_size,
                "yN_size": self.yN_size, "device": self.device}

    def __setstate__(self, state):
        self.__init__(**state)

    def check_params(self):
        """Validate parameters (core.py:55-74)."""
        if self.N % self.yN_size != 0:
            raise ValueError(
                f"Image size {self.N} not divisible by facet size {self.yN_size}!"
            )
        if self.N % self.xM_size != 0:
            raise ValueError(
                f"Image size {self.N} not divisible by subgrid size {self.xM_size}!"
            )
        if (self.xM_size * self.yN_size) % self.N != 0:
            raise ValueError(
                f"Contribution size not integer with image size {self.N}, "
                f"subgrid size {self.xM_size} and facet size {self.yN_size}!"
            )

    @property
    def subgrid_off_step(self):
        """All subgrid offsets must be divisible by this (core.py:76-83)."""
        return self.N // self.yN_size

    @property
    def facet_off_step(self):
        """All facet offsets must be divisible by this (core.py:85-92)."""
        return self.N // self.xM_size

    def __repr__(self):
        return (
            f"{self.__class__.__name__}(W={self.W}, N={self.N}, "
            f"xM_size={self.xM_size}, yN_size={self.yN_size})"
        )

    # ------------------------------------------------------------------ plumbing
    @staticmethod
    def _as_complex(a):
        """Promote input to complex128 (core.py:581-585 promotes real input)."""
        if _is_tensor(a):
            if a.dtype != torch.complex128:
                a = a.to(torch.complex128)
            return a
        a = numpy.asarray(a)
        if a.dtype != numpy.complex128 or not a.flags.c_contiguous:
            a = numpy.ascontiguousarray(a, dtype=numpy.complex128)
        return a

    @staticmethod
    def _new(like, shape, zero):
        if _is_tensor(like):
            fn = torch.zeros if zero else torch.empty
            return fn(tuple(shape), dtype=torch.complex128, device=like.device)
        fn = numpy.zeros if zero else numpy.empty
        return fn(tuple(shape), dtype=numpy.complex128)

    @staticmethod
    def _describe(a, axis):
        """``swiftly_b200_lines`` for the 1-D lines of ``a`` along ``axis``."""
        tensor = _is_tensor(a)
        if tensor:
            shape = tuple(a.shape)
            strides = tuple(a.stride())
            ptr = a.data_ptr()
            loc = _lib.DEVICE
        else:
            shape = a.shape
            if any(s % a.itemsize for s in a.strides):
                raise ValueError("array strides must be multiples of the item size")
            strides = tuple(s // a.itemsize for s in a.strides)
            ptr = a.ctypes.data
            loc = _lib.HOST
        if len(shape) == 1:
            return _lib.Lines(ptr, 1, shape[0], shape[0] * max(strides[0], 1), strides[0], loc)
        other = 1 - axis
        return _lib.Lines(ptr, shape[other], shape[axis], strides[other], strides[axis], loc)

    @staticmethod
    def _stream(a):
        if _is_tensor(a) and a.is_cuda:
            return ctypes.c_void_p(torch.cuda.current_stream(a.device).cuda_stream)
        return ctypes.c_void_p(0)

    def _check_tensor(self, t):
        """Device tensors must be complex128 on this plan's CUDA device."""
        if not t.is_cuda:
            raise ValueError(
                "tensors must live on a CUDA device (use numpy arrays for host data)"
            )
        if t.device.index != self.device:
            raise ValueError(
                f"tensor is on cuda:{t.device.index}, the plan on cuda:{self.device}"
            )

    @staticmethod
    def _mask_ptr(mask, like, size, keep, what="subgrid"):
        """Address of ``mask`` (None: NULL) converted to a contiguous float64 array living where
        ``like`` lives; it must have ``size`` samples.  The converted mask is appended to
        ``keep``, which the caller holds until the C call returns."""
        if mask is None:
            return None
        if _is_tensor(like):
            if not _is_tensor(mask):
                mask = torch.as_tensor(numpy.asarray(mask, dtype=float), device=like.device)
            mask = mask.to(like.device, torch.float64).contiguous()
            n, ptr = mask.numel(), mask.data_ptr()
        else:
            mask = numpy.ascontiguousarray(mask.cpu() if _is_tensor(mask) else mask, dtype=float)
            n, ptr = mask.size, mask.ctypes.data
        if n != size:
            raise ValueError(f"mask must have the {what} size")
        keep.append(mask)
        return ptr

    def _sources(self, groups, axis, n_lines):
        """``Source`` array, int32 group sizes and source tensors (to keep alive) of ``groups``,
        lists of ``(tensor, facet_off)`` read along ``axis`` into outputs of ``n_lines`` lines."""
        other = 1 - axis
        flat = [s for grp in groups for s in grp]
        arr = (_lib.Source * max(1, len(flat)))()
        for i, (t, facet_off) in enumerate(flat):
            self._check_tensor(t)
            if t.dtype != torch.complex128 or t.dim() != 2:
                raise ValueError("sources must be 2-D complex128 device tensors")
            if t.shape[other] != n_lines:
                raise ValueError(f"source has {t.shape[other]} lines, output {n_lines}")
            arr[i] = _lib.Source(t.data_ptr(), t.stride(other), t.stride(axis), t.shape[axis],
                                 int(facet_off))
        sizes = (ctypes.c_int32 * len(groups))(*[len(g) for g in groups])
        return arr, sizes, [t for t, _ in flat]

    def _run(self, fn_name, in_arr, out_size, axis, out, offset, accumulate=False, mask=None):
        """Shape handling shared by all primitives.

        Mirrors ``SwiftlyCoreFunc._auto_broadcast_create`` (core.py:577-630):
        1-D or 2-D input, the transformed axis changes length to ``out_size``,
        ``out`` is created (zeros for accumulating primitives, core.py:742-750)
        or shape-checked (``ValueError``).
        """
        in_arr = self._as_complex(in_arr)
        dims = len(in_arr.shape)
        if dims == 1:
            shape = (out_size,)
            axis = 0
        elif dims == 2:
            if axis not in (0, 1):
                raise ValueError(f"Invalid axis {axis} for shape {tuple(in_arr.shape)}!")
            shape = list(in_arr.shape)
            shape[axis] = out_size
            shape = tuple(shape)
        else:
            raise ValueError(
                f"Invalid number of dimensions in input array: {tuple(in_arr.shape)}"
            )
        if out is None:
            out = self._new(in_arr, shape, zero=accumulate)
        else:
            if tuple(out.shape) != shape:
                raise ValueError(
                    f"Output array has shape {tuple(out.shape)}, expected {shape}!"
                )
            if _is_tensor(out) != _is_tensor(in_arr):
                raise ValueError("input and output must both be numpy arrays or CUDA tensors")
            if _is_tensor(out):
                if out.dtype != torch.complex128:
                    raise ValueError("output tensor must be complex128")
            elif out.dtype != numpy.complex128:
                raise ValueError("output array must be complex128")
        if _is_tensor(in_arr):
            self._check_tensor(in_arr)
            self._check_tensor(out)
        din = self._describe(in_arr, axis)
        dout = self._describe(out, axis)
        keep = []
        args = [self._plan, ctypes.byref(din), ctypes.byref(dout), int(offset)]
        if fn_name in ("swiftly_b200_finish_subgrid", "swiftly_b200_finish_facet"):
            what = fn_name.rsplit("_", 1)[1]  # "subgrid" / "facet"
            args.append(self._mask_ptr(mask, out, shape[axis], keep, what))
        args.append(self._stream(in_arr))
        rc = getattr(self._lib, fn_name)(*args)
        _lib.check(self._lib, rc)
        return out

    # ------------------------------------------------------------------ facet -> subgrid
    def prepare_facet(self, facet, facet_off, axis, out=None, window_lines=False):
        """Prepare facet for extracting subgrid contributions (core.py:189-222).

        ``window_lines`` (fused forward path only, not part of the reference interface): every
        output line ``l`` (index along the OTHER axis) is additionally multiplied by the facet
        window ``Fb`` at ``l`` -- the factor ``prepare_facet`` along the other axis would apply
        -- so that :meth:`extract_columns` (``prewindowed=True``) need not fetch it per sample.
        """
        fn = "swiftly_b200_prepare_facet_windowed" if window_lines else "swiftly_b200_prepare_facet"
        return self._run(fn, facet, self.yN_size, axis, out, facet_off)

    @property
    def half_rows(self):
        """Rows of a half-row array of a real image: ``yN_size // 2 + 1`` (include/swiftly_b200.h,
        "Half rows"); stored row ``d`` holds centred row ``(yN_size // 2 + d) mod yN_size``."""
        return self.yN_size // 2 + 1

    def prepare_facet_real_half(self, facet, facet_off, axis=0, out=None):
        """``prepare_facet(facet, facet_off, axis, window_lines=True)`` of a REAL facet, keeping only
        the half rows: along ``axis`` ``yN_size // 2 + 1`` samples, sample ``d`` being the prepared
        facet's centred index ``(yN_size // 2 + d) mod yN_size``.  Bitwise those samples of the
        complex call on the promoted facet; the others are their conjugates.  ``facet``: 2-D
        float64 device tensor; ``out``: complex128 device tensor of the half shape or None.
        """
        if not _is_tensor(facet) or facet.dtype != torch.float64 or facet.dim() != 2:
            raise ValueError("prepare_facet_real_half needs a 2-D float64 device tensor")
        self._check_tensor(facet)
        if axis not in (0, 1):
            raise ValueError(f"Invalid axis {axis} for shape {tuple(facet.shape)}!")
        shape = list(facet.shape)
        shape[axis] = self.half_rows
        shape = tuple(shape)
        if out is None:
            out = torch.empty(shape, dtype=torch.complex128, device=facet.device)
        self._check_tensor(out)
        if out.dtype != torch.complex128 or tuple(out.shape) != shape:
            raise ValueError(f"Output array has shape {tuple(out.shape)} and dtype {out.dtype}, "
                             f"expected {shape} complex128!")
        other = 1 - axis
        din = _lib.Lines(facet.data_ptr(), facet.shape[other], facet.shape[axis],
                         facet.stride(other), facet.stride(axis), _lib.DEVICE)
        rc = self._lib.swiftly_b200_prepare_facet_real_half(
            self._plan, ctypes.byref(din), ctypes.byref(self._describe(out, axis)),
            int(facet_off), self._stream(facet))
        _lib.check(self._lib, rc)
        return out

    def extract_from_facet(self, prep_facet, subgrid_off, axis, out=None):
        """Extract the facet contribution to a subgrid (core.py:224-253)."""
        return self._run(
            "swiftly_b200_extract_from_facet", prep_facet, self.xM_yN_size, axis, out, subgrid_off
        )

    def add_to_subgrid(self, facet_contrib, facet_off, axis, out=None):
        """Transform a facet contribution and ADD it to ``out`` (core.py:255-285)."""
        return self._run(
            "swiftly_b200_add_to_subgrid", facet_contrib, self.xM_size, axis, out, facet_off,
            accumulate=True,
        )

    def add_to_subgrid_2d(self, facet_contrib, facet_off0, facet_off1, out=None):
        """Both axes of ``add_to_subgrid`` at once (SwiftlyCoreFunc, core.py:752-778)."""
        facet_contrib = self._as_complex(facet_contrib)
        if len(facet_contrib.shape) != 2:
            raise ValueError(
                f"Invalid number of dimensions in input array: {tuple(facet_contrib.shape)}"
            )
        shape = (self.xM_size, self.xM_size)
        if out is not None and tuple(out.shape) != shape:
            raise ValueError(f"Output array has shape {tuple(out.shape)}, expected {shape}!")
        tmp = self.add_to_subgrid(facet_contrib, facet_off0, axis=0)
        return self.add_to_subgrid(tmp, facet_off1, axis=1, out=out)

    def finish_subgrid(self, summed_contribs, subgrid_off, subgrid_size, out=None, masks=None):
        """Finish a subgrid on all axes (core.py:287-325).

        ``masks``: optional per-axis 0/1 vectors folded into the final store
        (what ``sum_and_finish_subgrid`` multiplies afterwards, api_helper.py:107-111).
        """
        dims = len(summed_contribs.shape)
        if not isinstance(subgrid_off, (list, tuple)):
            if dims != 1:
                raise ValueError("Subgrid offset must be given for every dimension!")
            subgrid_off = [subgrid_off]
        if len(subgrid_off) != dims:
            raise ValueError("Subgrid offset must be given for every dimension!")
        if masks is None:
            masks = [None] * dims
        fn = "swiftly_b200_finish_subgrid"
        if dims == 1:
            return self._run(fn, summed_contribs, subgrid_size, 0, out, subgrid_off[0],
                             mask=masks[0])
        if dims != 2:
            raise ValueError(f"Invalid shape {tuple(summed_contribs.shape)}!")
        # contiguous axis first on the big array, strided axis on the smaller result
        tmp = self._run(fn, summed_contribs, subgrid_size, 1, None, subgrid_off[1], mask=masks[1])
        return self._run(fn, tmp, subgrid_size, 0, out, subgrid_off[0], mask=masks[0])

    # ------------------------------------------------------------------ subgrid -> facet
    def prepare_subgrid(self, subgrid, subgrid_off, out=None):
        """Pad, align and Fourier transform a subgrid on all axes (core.py:328-368)."""
        dims = len(subgrid.shape)
        if dims == 1 and not isinstance(subgrid_off, (list, tuple)):
            subgrid_off = (subgrid_off,)
        if len(subgrid_off) != dims:
            raise ValueError("Dimensionality mismatch between subgrid and offsets!")
        fn = "swiftly_b200_prepare_subgrid"
        if dims == 1:
            return self._run(fn, subgrid, self.xM_size, 0, out, subgrid_off[0])
        if dims != 2:
            raise ValueError(f"Invalid shape {tuple(subgrid.shape)}!")
        tmp = self._run(fn, subgrid, self.xM_size, 0, None, subgrid_off[0])
        return self._run(fn, tmp, self.xM_size, 1, out, subgrid_off[1])

    def extract_from_subgrid(self, FSi, facet_off, axis, out=None):
        """Extract the contribution of a subgrid to a facet (core.py:370-406)."""
        return self._run(
            "swiftly_b200_extract_from_subgrid", FSi, self.xM_yN_size, axis, out, facet_off
        )

    def add_to_facet(self, subgrid_contrib, subgrid_off, axis, out=None):
        """ADD a subgrid contribution to a facet accumulator (core.py:408-449)."""
        return self._run(
            "swiftly_b200_add_to_facet", subgrid_contrib, self.yN_size, axis, out, subgrid_off,
            accumulate=True,
        )

    def finish_facet(self, MiNjSi_sum, facet_off, facet_size, axis, out=None, mask=None):
        """Finish a facet along one axis (core.py:452-484); optional 0/1 ``mask``."""
        return self._run(
            "swiftly_b200_finish_facet", MiNjSi_sum, facet_size, axis, out, facet_off, mask=mask
        )

    # ------------------------------------------------------------------ fused forward path
    def fused_forward_supported(self):
        """True if the fused subgrid kernels exist for this (xM_yN_size, xM_size) pair."""
        return self._lib.swiftly_b200_sum_finish_axis_supported(self._plan) > 0

    def fused_backward_supported(self):
        """True if the fused backward kernels can run this plan's FFT lengths."""
        from .swift_configs import fft_length_supported  # pylint: disable=import-outside-toplevel

        return fft_length_supported(self.xM_yN_size) and fft_length_supported(self.yN_size)

    def extract_column(self, BF_F, subgrid_off0, facet_off1, out=None):
        """``extract_column`` task of the reference (api_helper.py:200-210) as ONE kernel.

        ``extract_from_facet(BF_F, subgrid_off0, axis=0)`` then
        ``prepare_facet(., facet_off1, axis=1)``; device tensors only.
        ``BF_F``: ``(yN_size, facet_size)``; result ``(xM_yN_size, yN_size)``.
        """
        if not _is_tensor(BF_F) or BF_F.dtype != torch.complex128 or BF_F.dim() != 2:
            raise ValueError("extract_column needs a 2-D complex128 device tensor")
        self._check_tensor(BF_F)
        shape = (self.xM_yN_size, self.yN_size)
        if out is None:
            out = torch.empty(shape, dtype=torch.complex128, device=BF_F.device)
        elif tuple(out.shape) != shape:
            raise ValueError(f"Output array has shape {tuple(out.shape)}, expected {shape}!")
        din = self._describe(BF_F, 1)
        dout = self._describe(out, 1)
        rc = self._lib.swiftly_b200_extract_column(
            self._plan, ctypes.byref(din), ctypes.byref(dout), int(subgrid_off0),
            int(facet_off1), self._stream(BF_F),
        )
        _lib.check(self._lib, rc)
        return out

    def extract_columns(self, BF_Fs, subgrid_off0, facet_off1s, outs=None, prewindowed=False):
        """``extract_column`` for a list of facets in ONE kernel launch (<= 64 per launch).

        ``prewindowed``: the ``BF_Fs`` were made with ``prepare_facet(..., window_lines=True)``
        (or :meth:`prepare_facet_real_half`).  Every ``BF_F`` is a whole ``(yN_size, size)``
        prepared facet, or every one is an ``(xM_yN_size, size)`` row ring holding row ``r`` of the
        column's window at line ``r mod xM_yN_size`` (include/swiftly_b200.h, "Row rings"), or
        every one holds the ``yN_size // 2 + 1`` half rows of a real image ("Half rows").
        """
        shape = (self.xM_yN_size, self.yN_size)
        rows = (self.yN_size, self.xM_yN_size, self.half_rows)
        BF_Fs = list(BF_Fs)
        if outs is None:
            outs = [None] * len(BF_Fs)
        outs = [
            torch.empty(shape, dtype=torch.complex128, device=b.device) if o is None else o
            for b, o in zip(BF_Fs, outs)
        ]

        def chk_b(t):
            if t.shape[0] not in rows:
                raise ValueError(f"prepared facet has {t.shape[0]} rows, expected {rows[0]} "
                                 f"(or a ring of {rows[1]}, or {rows[2]} half rows)!")

        def chk_o(t):
            if tuple(t.shape) != shape:
                raise ValueError(f"Output array has shape {tuple(t.shape)}, expected {shape}!")

        entry = (self._lib.swiftly_b200_extract_columns_windowed if prewindowed
                 else self._lib.swiftly_b200_extract_columns)
        return self._per_facet(
            lambda n, din, dout, offs, _, stream: entry(
                self._plan, n, din, dout, int(subgrid_off0), offs, stream),
            BF_Fs, outs, facet_off1s, chk_b, chk_o)

    def sum_finish_axis_grouped(self, groups, out, axis, subgrid_off, mask=None):
        """:meth:`sum_finish_axis` for several source groups in ONE launch.

        :param groups: list of source lists ``[(tensor, facet_off), ...]``
        :param out: 3-D device tensor ``(n_groups, ...)``; ``out[g]`` receives group ``g``.
            With per-group ``subgrid_off`` it may also be a LIST of 2-D tensors of equal shape
            and strides, one per group, living in different buffers (e.g. peer memory)
        :param subgrid_off: one offset, or a list with one offset per group (groups of
            different subgrids, e.g. a batch of the multi-GPU driver)
        :param mask: one mask (or None), or a list with one mask / None per group
        """
        if axis not in (0, 1):
            raise ValueError(f"Invalid axis {axis}")
        per_group = isinstance(subgrid_off, (list, tuple))
        scattered = isinstance(out, (list, tuple))  # one output buffer per group
        if not scattered:
            self._check_tensor(out)
            if out.dim() != 3:
                raise ValueError("out must be (n_groups, lines, size) / (n_groups, size, lines)")
        if (len(out) != len(groups) or (per_group and len(subgrid_off) != len(groups))
                or (scattered and not per_group)):
            raise ValueError("out / subgrid_off must have one entry per group")
        dout = self._describe(out[0], axis)
        if per_group:
            block = PreparedSumFinish(self, groups, axis, dout.n_lines, dout.size,
                                      (dout.line_stride, dout.elem_stride))
            masks = [None] * len(groups) if mask is None else mask
            if scattered:
                block.launch(subgrid_off, masks, outs=out)
                return list(out)
            block.launch(subgrid_off, masks, out=out, out_group_stride=out.stride(0))
            return out
        arr, sizes, keep = self._sources(groups, axis, dout.n_lines)
        rc = self._lib.swiftly_b200_sum_finish_axis_grouped(
            self._plan, arr, sizes, len(groups), ctypes.byref(dout), int(out.stride(0)),
            int(subgrid_off), self._mask_ptr(mask, out, dout.size, keep), self._stream(out))
        _lib.check(self._lib, rc)
        return out

    def prepare_sum_finish(self, groups, axis, n_lines, size, out_strides):
        """Build the argument block of a grouped ``sum_finish_axis`` launch ONCE.

        The streaming drivers launch the same source groups for every subgrid of a subgrid
        column (only the subgrid offsets, masks and output buffers change); building the
        ctypes descriptors of 64 sources costs more host time than the kernel takes on several
        GPUs.  Returns a :class:`PreparedSumFinish`; ``launch(...)`` fills in the per-call values.

        :param groups: list of source lists ``[(tensor, facet_off), ...]``
        :param n_lines, size: lines and samples per line of ONE group's output
        :param out_strides: ``(line_stride, elem_stride)`` of a group's output (samples)
        """
        return PreparedSumFinish(self, groups, axis, n_lines, size, out_strides)

    def sum_finish_axis(self, sources, out, axis, subgrid_off, mask=None):
        """One axis of ``sum_and_finish_subgrid`` (api_helper.py:73-112) as ONE kernel.

        :param sources: list of ``(tensor, facet_off)``; every tensor is 2-D with the
            transformed ``axis`` of length ``yN_size`` (prepared facet lines: the
            contribution window for ``subgrid_off`` is cut on the fly) or
            ``xM_yN_size`` (already contributions)
        :param out: 2-D device tensor, ``axis`` of length subgrid size (overwritten)
        :param mask: optional mask of length subgrid size
        """
        if axis not in (0, 1):
            raise ValueError(f"Invalid axis {axis}")
        self._check_tensor(out)
        dout = self._describe(out, axis)
        arr, _, keep = self._sources([sources], axis, dout.n_lines)
        rc = self._lib.swiftly_b200_sum_finish_axis(
            self._plan, arr, len(sources), ctypes.byref(dout), int(subgrid_off),
            self._mask_ptr(mask, out, dout.size, keep), self._stream(out),
        )
        _lib.check(self._lib, rc)
        return out

    def mirror_subgrid(self, src, sz, out=None, mirror=None, masks=None, mirror_masks=None):
        """The two finished subgrids of a Hermitian pair (real image) from ONE unmasked source.

        ``src``: the subgrid at ``(off0, off1)`` of size ``S = 2 * (sz // 2) + 1`` or larger (only
        the first ``S x S`` samples are read), e.g. ``sum_finish_axis`` along both axes at size
        ``S`` without masks.  Returns ``(out, mirror)``, both ``(sz, sz)``:
        ``out[r, c] = m0[r] * m1[c] * src[r, c]`` is the subgrid of size ``sz`` at
        ``(off0, off1)``; ``mirror[r, c] = n0[r] * n1[c] * conj(src[2h - r, 2h - c])``,
        ``h = sz // 2``, the one at ``(-off0, -off1)``.  ``masks`` / ``mirror_masks``: None or
        ``(mask0, mask1)``, each None or a mask of ``sz`` samples.  ``out`` /
        ``mirror`` may be given (any strides, e.g. views into larger arrays); device tensors only.
        """
        self._check_tensor(src)
        if src.dtype != torch.complex128 or src.dim() != 2:
            raise ValueError("mirror_subgrid needs a 2-D complex128 device tensor")
        shape = (int(sz), int(sz))
        outs = []
        for t in (out, mirror):
            if t is None:
                t = torch.empty(shape, dtype=torch.complex128, device=src.device)
            self._check_tensor(t)
            if t.dtype != torch.complex128 or tuple(t.shape) != shape:
                raise ValueError(f"Output array has shape {tuple(t.shape)}, expected {shape}!")
            outs.append(t)
        keep = []
        ptrs = [self._mask_ptr(mk, outs[0], shape[0], keep)
                for pair in (masks, mirror_masks) for mk in ((None, None) if pair is None else pair)]
        din, dout, dmir = (self._describe(t, 1) for t in (src, outs[0], outs[1]))
        rc = self._lib.swiftly_b200_mirror_subgrid(
            self._plan, ctypes.byref(din), ctypes.byref(dout), ctypes.byref(dmir), *ptrs,
            self._stream(src))
        _lib.check(self._lib, rc)
        return outs[0], outs[1]

    def merge_mirror_subgrid(self, sg, mirror, out=None):
        """One subgrid in place of a Hermitian pair (real image), the adjoint of
        :meth:`mirror_subgrid`.

        ``sg`` / ``mirror``: the ``(sz, sz)`` subgrids at ``(off0, off1)`` and ``(-off0, -off1)``.
        Returns the ``(S, S)`` subgrid at ``(off0, off1)``, ``S = 2 * (sz // 2) + 1``,
        ``out[r, c] = sg[r, c] + conj(mirror[2h - r, 2h - c])`` (each term where its indices are
        below ``sz``, 0 where neither is), whose backward transform has the real part of the sum
        of the pair's.  ``out`` may be given (any strides); complex128 device tensors only.
        """
        for t in (sg, mirror):
            self._check_tensor(t)
            if t.dtype != torch.complex128 or t.dim() != 2:
                raise ValueError("merge_mirror_subgrid needs 2-D complex128 device tensors")
        sz = int(sg.shape[0])
        if tuple(sg.shape) != (sz, sz) or tuple(mirror.shape) != (sz, sz):
            raise ValueError(f"sg and mirror must both be square of one size, got "
                             f"{tuple(sg.shape)} and {tuple(mirror.shape)}")
        S = 2 * (sz // 2) + 1
        if out is None:
            out = torch.empty((S, S), dtype=torch.complex128, device=sg.device)
        self._check_tensor(out)
        if out.dtype != torch.complex128 or tuple(out.shape) != (S, S):
            raise ValueError(f"Output array has shape {tuple(out.shape)}, expected {(S, S)}!")
        dsg, dmir, dout = (self._describe(t, 1) for t in (sg, mirror, out))
        rc = self._lib.swiftly_b200_merge_mirror_subgrid(
            self._plan, ctypes.byref(dsg), ctypes.byref(dmir), ctypes.byref(dout),
            self._stream(sg))
        _lib.check(self._lib, rc)
        return out

    def finish_facet_real(self, MiNjSi_sum, facet_off, facet_size, axis, out=None, mask=None):
        """:meth:`finish_facet` of a real image: the real part only, float64.

        ``out[k] = (Re(finish_facet(...))[k]) * mask[k]`` bitwise (the window product first, the
        mask after, as ``finish_facet`` followed by a row mask).  ``MiNjSi_sum``: 2-D complex128
        device tensor; ``out``: float64 device tensor of the finished shape (any strides) or None;
        ``mask``: None or ``facet_size`` samples.
        """
        return self._finish_real(MiNjSi_sum, facet_off, facet_size, axis, out, mask, False)

    def _finish_real(self, acc, facet_off, facet_size, axis, out, mask, half):
        self._check_tensor(acc)
        if acc.dtype != torch.complex128 or acc.dim() != 2:
            raise ValueError("finish_facet_real needs a 2-D complex128 device tensor")
        if axis not in (0, 1):
            raise ValueError(f"Invalid axis {axis} for shape {tuple(acc.shape)}!")
        shape = list(acc.shape)
        shape[axis] = int(facet_size)
        shape = tuple(shape)
        if out is None:
            out = torch.empty(shape, dtype=torch.float64, device=acc.device)
        self._check_tensor(out)
        if out.dtype != torch.float64 or tuple(out.shape) != shape:
            raise ValueError(f"Output array has shape {tuple(out.shape)} and dtype {out.dtype}, "
                             f"expected {shape} float64!")
        keep = []
        mptr = self._mask_ptr(mask, out, shape[axis], keep, "facet")
        other = 1 - axis
        dout = _lib.Lines(out.data_ptr(), shape[other], shape[axis], out.stride(other),
                          out.stride(axis), _lib.DEVICE)
        entry = (self._lib.swiftly_b200_finish_facet_real_half if half
                 else self._lib.swiftly_b200_finish_facet_real)
        rc = entry(self._plan, ctypes.byref(self._describe(acc, axis)), ctypes.byref(dout),
                   int(facet_off), mptr, self._stream(acc))
        _lib.check(self._lib, rc)
        return out

    def finish_facet_real_half(self, MiNjSi_sum, facet_off, facet_size, axis, out=None,
                               mask=None):
        """:meth:`finish_facet_real` of an accumulator kept as half rows: ``yN_size // 2 + 1``
        samples along ``axis`` (include/swiftly_b200.h, "Half rows").  Bitwise
        :meth:`finish_facet_real` of the full line whose natural-order samples are ``0.5 H[q]``,
        ``0.5 conj(H[yN - q])`` and ``(Re H[q], 0)`` at ``q = 0, yN/2``.
        """
        return self._finish_real(MiNjSi_sum, facet_off, facet_size, axis, out, mask, True)

    def release_scratch(self):
        """Give the plan's scratch buffers (2 GiB after stage 1 at N = 65536) back to the device."""
        self._lib.swiftly_b200_release_scratch(self._plan)

    # ------------------------------------------------------------------ rank-to-rank ordering
    def peer_signal(self, flag_table, n_peers, my_rank, value, stream_of):
        """Store ``value`` into entry ``my_rank`` of every rank's flag array (peer_sync.cu).
        ``flag_table``: int64 device tensor holding this rank's mappings of the arrays."""
        rc = self._lib.swiftly_b200_peer_signal(
            self._plan, ctypes.c_void_p(flag_table.data_ptr()), int(n_peers), int(my_rank),
            int(value), self._stream(stream_of))
        _lib.check(self._lib, rc)

    def peer_wait(self, my_flags, n_peers, value, status, timeout_s=20.0):
        """Make the stream wait until all ``n_peers`` entries of ``my_flags`` are >= value."""
        rc = self._lib.swiftly_b200_peer_wait(
            self._plan, ctypes.c_void_p(my_flags.data_ptr()), int(n_peers), int(value),
            float(timeout_s), ctypes.c_void_p(status.data_ptr()), self._stream(my_flags))
        _lib.check(self._lib, rc)

    # ------------------------------------------------------------------ fused backward path
    def split_axis_supported(self):
        """True if the fused subgrid split kernel exists for this (xM_yN_size, xM_size) pair."""
        return self._lib.swiftly_b200_split_axis_supported(self._plan) > 0

    def split_subgrid_axis(self, groups, axis, subgrid_offs, targets, mode):
        """The subgrid side of the backward transform along ``axis``, ONE kernel per call.

        Per line of ``groups[g]``: ``prepare_subgrid`` along ``axis`` with ``subgrid_offs[g]``
        (core.py:328-368), then ``extract_from_subgrid(., facet_off, axis)`` (core.py:370-406)
        for every target of the group; the adjoint of :meth:`sum_finish_axis`.

        :param groups: 2-D complex128 device tensors, one per group; ``axis`` has the subgrid
            size, the other axis the same line count in every group
        :param subgrid_offs: one subgrid offset (along ``axis``) per group
        :param targets: per group a list of ``(tensor, facet_off)``; the tensors have the
            group's line count along the other axis and, along ``axis``,
            ``xM_yN_size`` samples (``mode="store"``: overwritten with the contribution) or
            ``yN_size`` samples (``mode="add"``: ``add_to_facet(., subgrid_off, axis)``,
            core.py:408-449, accumulates into it).  In add mode the targets of one group must be
            distinct tensors; different groups may share one (they are applied in order).
        """
        if axis not in (0, 1):
            raise ValueError(f"Invalid axis {axis}")
        if mode not in ("store", "add"):
            raise ValueError(f"mode must be 'store' or 'add', not {mode!r}")
        if len(subgrid_offs) != len(groups) or len(targets) != len(groups):
            raise ValueError("subgrid_offs / targets must have one entry per group")
        if not groups:
            return targets
        other = 1 - axis
        size = self.yN_size if mode == "add" else self.xM_yN_size
        ins = (_lib.Lines * len(groups))()
        for g, t in enumerate(groups):
            self._check_tensor(t)
            if t.dtype != torch.complex128 or t.dim() != 2:
                raise ValueError("subgrid inputs must be 2-D complex128 device tensors")
            ins[g] = self._describe(t, axis)
        flat = [tg for grp in targets for tg in grp]
        arr = (_lib.SplitTarget * max(1, len(flat)))()
        for i, (t, facet_off) in enumerate(flat):
            self._check_tensor(t)
            if t.dtype != torch.complex128 or t.dim() != 2:
                raise ValueError("targets must be 2-D complex128 device tensors")
            if t.shape[axis] != size:
                raise ValueError(f"target has {t.shape[axis]} samples per line, expected {size}")
            arr[i] = _lib.SplitTarget(t.data_ptr(), t.shape[other], t.stride(other),
                                      t.stride(axis), int(facet_off))
        sizes = (ctypes.c_int32 * len(groups))(*[len(grp) for grp in targets])
        offs = (ctypes.c_int64 * len(groups))(*[int(o) for o in subgrid_offs])
        rc = self._lib.swiftly_b200_split_subgrid_axis(
            self._plan, ins, len(groups), offs, arr, sizes,
            _lib.SPLIT_ADD if mode == "add" else _lib.SPLIT_STORE, self._stream(groups[0]))
        _lib.check(self._lib, rc)
        return targets

    def _lines_array(self, tensors, shape_check):
        arr = (_lib.Lines * len(tensors))()
        for k, t in enumerate(tensors):
            self._check_tensor(t)
            if t.dtype != torch.complex128 or t.dim() != 2 or t.stride(1) != 1:
                raise ValueError("need row-contiguous 2-D complex128 device tensors")
            shape_check(t)
            arr[k] = self._describe(t, 1)
        return arr

    def _per_facet(self, call, ins, outs, offs, chk_in, chk_out, masks=None):
        """``call(n, din, dout, offs, mptrs, stream)`` once per chunk of at most 64 facets
        (``SW_MAX_COLUMN_FACETS``): the ``Lines`` of the chunk's ``ins`` and ``outs`` (row-contiguous
        tensors checked by ``chk_in`` / ``chk_out``), its facet offsets and, with ``masks``, its
        facet masks of ``outs[f].shape[1]`` samples (else ``mptrs`` is None).  Returns ``outs``."""
        keep = []
        for lo in range(0, len(ins), 64):
            hi = min(lo + 64, len(ins))
            din = self._lines_array(ins[lo:hi], chk_in)
            dout = self._lines_array(outs[lo:hi], chk_out)
            offs_k = (ctypes.c_int64 * (hi - lo))(*[int(o) for o in offs[lo:hi]])
            mptrs = None if masks is None else (ctypes.c_void_p * (hi - lo))(*[
                self._mask_ptr(mk, t, t.shape[1], keep, "facet")
                for mk, t in zip(masks[lo:hi], outs[lo:hi])])
            rc = call(hi - lo, din, dout, offs_k, mptrs, self._stream(ins[lo]))
            _lib.check(self._lib, rc)
        return outs

    def subgrid_to_facets(self, blocks, accs, facet_off1s, subgrid_off1):
        """One subgrid into the column accumulators of many facets, ONE launch per <= 64 facets.

        Per facet: ``extract_from_subgrid(block, facet_off1, axis=1)`` and
        ``add_to_facet(., subgrid_off1, axis=1, out=acc)`` (api_helper.py:115-152).
        ``blocks[f]``: ``(xM_yN_size, xM_size)``; ``accs[f]``: ``(xM_yN_size, yN_size)``, added to.
        """
        m, xM, yN = self.xM_yN_size, self.xM_size, self.yN_size

        def chk_b(t):
            if tuple(t.shape) != (m, xM):
                raise ValueError(f"block has shape {tuple(t.shape)}, expected {(m, xM)}!")

        def chk_a(t):
            if tuple(t.shape) != (m, yN):
                raise ValueError(f"accumulator has shape {tuple(t.shape)}, expected {(m, yN)}!")

        return self._per_facet(
            lambda n, din, dout, offs, _, stream: self._lib.swiftly_b200_subgrid_to_facets(
                self._plan, n, din, dout, offs, int(subgrid_off1), stream),
            blocks, accs, facet_off1s, chk_b, chk_a)

    def fold_column(self, accs, facet_accs, facet_off1s, masks1, subgrid_off0):
        """Fold a finished subgrid column into many facet accumulators, ONE launch per <= 64.

        Per facet: ``finish_facet(acc, facet_off1, size, axis=1)``, mask, and
        ``add_to_facet(., subgrid_off0, axis=0, out=facet_acc)`` (api_helper.py:155-179).
        ``facet_accs[f]``: ``(yN_size, facet_size)``, added to; or, for every facet, an
        ``(xM_yN_size, facet_size)`` row ring holding row ``r`` of the column's window at line
        ``r mod xM_yN_size`` (include/swiftly_b200.h, "Row rings"), or every one holds the
        ``yN_size // 2 + 1`` half rows of a real image ("Half rows"); ``masks1[f]``: a mask of
        the facet size or None.
        """
        m, yN, half = self.xM_yN_size, self.yN_size, self.half_rows

        def chk_a(t):
            if tuple(t.shape) != (m, yN):
                raise ValueError(f"accumulator has shape {tuple(t.shape)}, expected {(m, yN)}!")

        def chk_f(t):
            if t.shape[0] not in (yN, m, half):
                raise ValueError(f"facet accumulator has {t.shape[0]} rows, expected {yN} "
                                 f"(or a ring of {m}, or {half} half rows)!")

        return self._per_facet(
            lambda n, din, dout, offs, mptrs, stream: self._lib.swiftly_b200_fold_column(
                self._plan, n, din, dout, offs, mptrs, int(subgrid_off0), stream),
            accs, facet_accs, facet_off1s, chk_a, chk_f, masks1)
