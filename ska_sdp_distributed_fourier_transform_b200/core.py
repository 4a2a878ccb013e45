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
        other = 1 - axis
        flat = [s for grp in groups for s in grp]
        self._keep = [t for t, _ in flat]  # the sources must outlive the block
        self._arr = (_lib.Source * max(1, len(flat)))()
        for i, (t, facet_off) in enumerate(flat):
            core._check_tensor(t)
            if t.dtype != torch.complex128 or t.dim() != 2:
                raise ValueError("sources must be 2-D complex128 device tensors")
            if t.shape[other] != n_lines:
                raise ValueError(f"source has {t.shape[other]} lines, output {n_lines}")
            self._arr[i] = _lib.Source(t.data_ptr(), t.stride(other), t.stride(axis),
                                       t.shape[axis], int(facet_off))
        self._sizes = (ctypes.c_int32 * self.n_groups)(*[len(g) for g in groups])
        self._offs = (ctypes.c_int64 * self.n_groups)()
        self._mptrs = (ctypes.c_void_p * self.n_groups)()
        self._optrs = (ctypes.c_void_p * self.n_groups)()
        self._dout = _lib.Lines(0, int(n_lines), int(size), int(out_strides[0]),
                                int(out_strides[1]), _lib.DEVICE)
        self._device = flat[0][0].device if flat else None

    def launch(self, subgrid_offs, masks=None, out=None, out_group_stride=0, outs=None,
               n_groups=None, out_ptrs=None, stream_of=None):
        """Launch for the first ``n_groups`` groups (default: all).

        :param subgrid_offs: one offset per group
        :param masks: None or one float64 device tensor / None per group
        :param out, out_group_stride: base tensor of group 0 and the stride between groups, or
        :param outs: one output tensor per group (same shape / strides, different buffers), or
        :param out_ptrs: their device addresses (ints) with ``stream_of`` a tensor on the device
        """
        n = self.n_groups if n_groups is None else int(n_groups)
        core = self.core
        for g in range(n):
            self._offs[g] = int(subgrid_offs[g])
            mk = None if masks is None else masks[g]
            self._mptrs[g] = None if mk is None else mk.data_ptr()
        if outs is not None or out_ptrs is not None:
            if out_ptrs is not None:
                for g in range(n):
                    self._optrs[g] = out_ptrs[g]
                stream = core._stream(stream_of)
            else:
                for g in range(n):
                    self._optrs[g] = outs[g].data_ptr()
                stream = core._stream(outs[0])
            rc = core._lib.swiftly_b200_sum_finish_axis_scattered(
                core._plan, self._arr, self._sizes, n, ctypes.byref(self._dout), self._optrs,
                self._offs, self._mptrs, stream)
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

    def _mask_ptr(self, mask, like, keep):
        """Pointer to a float64 mask living where ``like`` lives (or NULL)."""
        if mask is None:
            return ctypes.c_void_p(0)
        if _is_tensor(like):
            if not _is_tensor(mask):
                mask = torch.as_tensor(numpy.asarray(mask, dtype=float), device=like.device)
            mask = mask.to(torch.float64).contiguous()
            keep.append(mask)
            return ctypes.c_void_p(mask.data_ptr())
        mask = numpy.ascontiguousarray(mask, dtype=float)
        keep.append(mask)
        return ctypes.c_void_p(mask.ctypes.data)

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
            args.append(self._mask_ptr(mask, out, keep))
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
        for lo in range(0, len(BF_Fs), 64):
            chunk = range(lo, min(lo + 64, len(BF_Fs)))
            din = (_lib.Lines * len(chunk))()
            dout = (_lib.Lines * len(chunk))()
            offs = (ctypes.c_int64 * len(chunk))()
            for k, i in enumerate(chunk):
                b, o = BF_Fs[i], outs[i]
                self._check_tensor(b)
                self._check_tensor(o)
                if b.dtype != torch.complex128 or b.dim() != 2 or b.stride(1) != 1:
                    raise ValueError("extract_columns needs row-contiguous complex128 tensors")
                if b.shape[0] not in rows:
                    raise ValueError(f"prepared facet has {b.shape[0]} rows, expected {rows[0]} "
                                     f"(or a ring of {rows[1]}, or {rows[2]} half rows)!")
                if tuple(o.shape) != shape or o.stride(1) != 1:
                    raise ValueError(f"Output array has shape {tuple(o.shape)}, expected {shape}!")
                din[k] = self._describe(b, 1)
                dout[k] = self._describe(o, 1)
                offs[k] = int(facet_off1s[i])
            entry = (self._lib.swiftly_b200_extract_columns_windowed if prewindowed
                     else self._lib.swiftly_b200_extract_columns)
            rc = entry(self._plan, len(chunk), din, dout, int(subgrid_off0), offs,
                       self._stream(BF_Fs[lo]))
            _lib.check(self._lib, rc)
        return outs

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
        if isinstance(subgrid_off, (list, tuple)):
            return self._sum_finish_axis_batched(groups, out, axis, subgrid_off, mask)
        if axis not in (0, 1):
            raise ValueError(f"Invalid axis {axis}")
        self._check_tensor(out)
        if out.dim() != 3 or out.shape[0] != len(groups):
            raise ValueError("out must be (n_groups, lines, size) / (n_groups, size, lines)")
        flat = [s for grp in groups for s in grp]
        arr = (_lib.Source * max(1, len(flat)))()
        other = 1 - axis
        for i, (t, facet_off) in enumerate(flat):
            self._check_tensor(t)
            if t.dtype != torch.complex128 or t.dim() != 2:
                raise ValueError("sources must be 2-D complex128 device tensors")
            if t.shape[other] != out.shape[1 + other]:
                raise ValueError(
                    f"source has {t.shape[other]} lines, output {out.shape[1 + other]}")
            arr[i] = _lib.Source(t.data_ptr(), t.stride(other), t.stride(axis), t.shape[axis],
                                 int(facet_off))
        sizes = (ctypes.c_int32 * len(groups))(*[len(g) for g in groups])
        dout = self._describe(out[0], axis)
        mptr = ctypes.c_void_p(0)
        if mask is not None:
            if mask.dtype != torch.float64 or mask.numel() != out.shape[1 + axis]:
                raise ValueError("mask must be float64 of the subgrid size")
            mask = mask.contiguous()
            mptr = ctypes.c_void_p(mask.data_ptr())
        rc = self._lib.swiftly_b200_sum_finish_axis_grouped(
            self._plan, arr, sizes, len(groups), ctypes.byref(dout), int(out.stride(0)),
            int(subgrid_off), mptr, self._stream(out))
        _lib.check(self._lib, rc)
        return out

    def _sum_finish_axis_batched(self, groups, out, axis, subgrid_offs, masks):
        if axis not in (0, 1):
            raise ValueError(f"Invalid axis {axis}")
        scattered = isinstance(out, (list, tuple))  # one output buffer per group
        if scattered:
            outs = list(out)
            if len(outs) != len(groups) or len(subgrid_offs) != len(groups):
                raise ValueError("out / subgrid_off must have one entry per group")
            for o in outs:
                self._check_tensor(o)
                if (o.dim() != 2 or tuple(o.shape) != tuple(outs[0].shape)
                        or o.stride() != outs[0].stride() or o.dtype != torch.complex128):
                    raise ValueError("scattered outputs must share shape, strides and dtype")
            out = outs[0][None]
        self._check_tensor(out)
        if out.dim() != 3 or (not scattered and out.shape[0] != len(groups)) \
                or len(subgrid_offs) != len(groups):
            raise ValueError("out / subgrid_off must have one entry per group")
        if masks is None:
            masks = [None] * len(groups)
        flat = [s for grp in groups for s in grp]
        arr = (_lib.Source * max(1, len(flat)))()
        other = 1 - axis
        for i, (t, facet_off) in enumerate(flat):
            self._check_tensor(t)
            if t.dtype != torch.complex128 or t.dim() != 2:
                raise ValueError("sources must be 2-D complex128 device tensors")
            if t.shape[other] != out.shape[1 + other]:
                raise ValueError(
                    f"source has {t.shape[other]} lines, output {out.shape[1 + other]}")
            arr[i] = _lib.Source(t.data_ptr(), t.stride(other), t.stride(axis), t.shape[axis],
                                 int(facet_off))
        sizes = (ctypes.c_int32 * len(groups))(*[len(g) for g in groups])
        offs = (ctypes.c_int64 * len(groups))(*[int(o) for o in subgrid_offs])
        keep = []
        mptrs = (ctypes.c_void_p * len(groups))()
        for g, mk in enumerate(masks):
            if mk is None:
                mptrs[g] = None
            else:
                if mk.dtype != torch.float64 or mk.numel() != out.shape[1 + axis]:
                    raise ValueError("mask must be float64 of the subgrid size")
                mk = mk.contiguous()
                keep.append(mk)
                mptrs[g] = mk.data_ptr()
        dout = self._describe(out[0], axis)
        if scattered:
            ptrs = (ctypes.c_void_p * len(groups))(*[o.data_ptr() for o in outs])
            rc = self._lib.swiftly_b200_sum_finish_axis_scattered(
                self._plan, arr, sizes, len(groups), ctypes.byref(dout), ptrs, offs, mptrs,
                self._stream(outs[0]))
            _lib.check(self._lib, rc)
            return outs
        rc = self._lib.swiftly_b200_sum_finish_axis_batched(
            self._plan, arr, sizes, len(groups), ctypes.byref(dout), int(out.stride(0)),
            offs, mptrs, self._stream(out))
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
        :param mask: optional float64 device tensor of length subgrid size
        """
        if axis not in (0, 1):
            raise ValueError(f"Invalid axis {axis}")
        self._check_tensor(out)
        arr = (_lib.Source * len(sources))()
        other = 1 - axis
        for i, (t, facet_off) in enumerate(sources):
            self._check_tensor(t)
            if t.dtype != torch.complex128 or t.dim() != 2:
                raise ValueError("sources must be 2-D complex128 device tensors")
            if t.shape[other] != out.shape[other]:
                raise ValueError(
                    f"source has {t.shape[other]} lines, output {out.shape[other]}"
                )
            arr[i] = _lib.Source(t.data_ptr(), t.stride(other), t.stride(axis), t.shape[axis],
                                 int(facet_off))
        dout = self._describe(out, axis)
        mptr = ctypes.c_void_p(0)
        if mask is not None:
            if mask.dtype != torch.float64 or mask.numel() != out.shape[axis]:
                raise ValueError("mask must be float64 of the subgrid size")
            mask = mask.contiguous()
            mptr = ctypes.c_void_p(mask.data_ptr())
        rc = self._lib.swiftly_b200_sum_finish_axis(
            self._plan, arr, len(sources), ctypes.byref(dout), int(subgrid_off), mptr,
            self._stream(out),
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
        ``(mask0, mask1)``, each None or a float64 device tensor of ``sz`` samples.  ``out`` /
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
        ptrs = []
        for pair in (masks, mirror_masks):
            for mk in (None, None) if pair is None else pair:
                if mk is None:
                    ptrs.append(None)
                    continue
                mk = mk.to(torch.float64).contiguous()
                self._check_tensor(mk)
                if mk.numel() != shape[0]:
                    raise ValueError("mask must have the subgrid size")
                keep.append(mk)
                ptrs.append(mk.data_ptr())
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
        mptr = ctypes.c_void_p(0)
        if mask is not None:
            mptr = self._mask_ptr(mask, out, keep)
            if keep[0].numel() != shape[axis]:
                raise ValueError("mask must have the facet size")
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

        for lo in range(0, len(blocks), 64):
            hi = min(lo + 64, len(blocks))
            din = self._lines_array(blocks[lo:hi], chk_b)
            dout = self._lines_array(accs[lo:hi], chk_a)
            offs = (ctypes.c_int64 * (hi - lo))(*[int(o) for o in facet_off1s[lo:hi]])
            rc = self._lib.swiftly_b200_subgrid_to_facets(
                self._plan, hi - lo, din, dout, offs, int(subgrid_off1), self._stream(accs[lo]))
            _lib.check(self._lib, rc)
        return accs

    def fold_column(self, accs, facet_accs, facet_off1s, masks1, subgrid_off0):
        """Fold a finished subgrid column into many facet accumulators, ONE launch per <= 64.

        Per facet: ``finish_facet(acc, facet_off1, size, axis=1)``, mask, and
        ``add_to_facet(., subgrid_off0, axis=0, out=facet_acc)`` (api_helper.py:155-179).
        ``facet_accs[f]``: ``(yN_size, facet_size)``, added to; or, for every facet, an
        ``(xM_yN_size, facet_size)`` row ring holding row ``r`` of the column's window at line
        ``r mod xM_yN_size`` (include/swiftly_b200.h, "Row rings"), or every one holds the
        ``yN_size // 2 + 1`` half rows of a real image ("Half rows"); ``masks1[f]``: float64
        device tensor of the facet size or None.
        """
        m, yN, half = self.xM_yN_size, self.yN_size, self.half_rows

        def chk_a(t):
            if tuple(t.shape) != (m, yN):
                raise ValueError(f"accumulator has shape {tuple(t.shape)}, expected {(m, yN)}!")

        def chk_f(t):
            if t.shape[0] not in (yN, m, half):
                raise ValueError(f"facet accumulator has {t.shape[0]} rows, expected {yN} "
                                 f"(or a ring of {m}, or {half} half rows)!")

        keep = []
        for lo in range(0, len(accs), 64):
            hi = min(lo + 64, len(accs))
            din = self._lines_array(accs[lo:hi], chk_a)
            dout = (_lib.Lines * (hi - lo))()
            for k, t in enumerate(facet_accs[lo:hi]):
                self._check_tensor(t)
                if t.dtype != torch.complex128 or t.dim() != 2 or t.stride(1) != 1:
                    raise ValueError("need row-contiguous 2-D complex128 device tensors")
                chk_f(t)
                # lines = rows (yN of them), line length = facet size
                dout[k] = _lib.Lines(t.data_ptr(), t.shape[0], t.shape[1], t.stride(0), 1,
                                     _lib.DEVICE)
            offs = (ctypes.c_int64 * (hi - lo))(*[int(o) for o in facet_off1s[lo:hi]])
            mptrs = (ctypes.c_void_p * (hi - lo))()
            for k, mk in enumerate(masks1[lo:hi]):
                if mk is None:
                    mptrs[k] = None
                else:
                    mk = mk.to(torch.float64).contiguous()
                    if mk.numel() != facet_accs[lo + k].shape[1]:
                        raise ValueError("mask must have the facet size")
                    keep.append(mk)
                    mptrs[k] = mk.data_ptr()
            rc = self._lib.swiftly_b200_fold_column(
                self._plan, hi - lo, din, dout, offs, mptrs, int(subgrid_off0),
                self._stream(accs[lo]))
            _lib.check(self._lib, rc)
        return facet_accs
