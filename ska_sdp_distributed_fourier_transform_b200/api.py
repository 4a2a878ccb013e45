"""
Application programming interface of the B200 SwiFTly transform.

Same surface as the reference's ``api.py`` (``FacetConfig`` :39-70,
``SubgridConfig`` :73-104, ``SwiftlyConfig`` :107-214, ``SwiftlyForward`` :217-324,
``SwiftlyBackward`` :327-463, ``make_full_subgrid_cover`` / ``make_full_facet_cover``
:593-612) -- constructor arguments, method names and properties are kept so a
driver written for ``ska_sdp_exec_swiftly`` only changes its import.  The
mechanism is different: instead of building a Dask task graph that is shipped to
CPU workers, every call enqueues hand-written CUDA kernels on the current CUDA
stream of one GPU; "tasks" are light handles around device tensors
(``.result()`` / ``.compute()`` copy to the host, ``.tensor`` stays on the GPU).
``lru_forward`` / ``lru_backward`` keep their meaning (number of subgrid columns
whose intermediates stay resident); ``queue_size`` bounds the number of results
in flight.  ``dask_client`` / ``client`` are accepted and ignored.
"""

import collections
import logging
import time

import numpy

from .api_helper import (
    accumulate_column,
    accumulate_facet,
    extract_column,
    finish_facet,
    make_full_cover_config,
    make_mask_from_slice,
    prepare_and_split_subgrid,
    sum_and_finish_subgrid,
)
from .core import SwiftlyCoreB200

try:
    import torch
except ImportError:  # pragma: no cover
    torch = None

__all__ = [
    "FacetConfig",
    "SubgridConfig",
    "SwiftlyConfig",
    "SwiftlyForward",
    "SwiftlyBackward",
    "PinnedArena",
    "device_tier_bytes",
    "make_full_facet_cover",
    "make_full_subgrid_cover",
]

log = logging.getLogger("fourier-logger")


class _ChunkConfig:
    """Offset, size and (lazily materialised) masks of a facet or subgrid."""

    def __init__(self, off0, off1, size, mask0=None, mask1=None):
        self.off0 = off0
        self.off1 = off1
        self.size = size
        self._mask0 = mask0
        self._mask1 = mask1

    @staticmethod
    def _materialise(mask):
        # a mask is either an array or ``[[slices], size]``
        if isinstance(mask, list):
            return make_mask_from_slice(mask[0], mask[1])
        return mask

    @property
    def mask0(self):
        """Mask along axis 0 (vertical)."""
        return self._materialise(self._mask0)

    @property
    def mask1(self):
        """Mask along axis 1 (horizontal)."""
        return self._materialise(self._mask1)

    def __repr__(self):
        return f"{self.__class__.__name__}(off0={self.off0}, off1={self.off1}, size={self.size})"


class FacetConfig(_ChunkConfig):
    """Facet configuration (offsets of the facet mid-point, size, masks)."""


class SubgridConfig(_ChunkConfig):
    """Subgrid configuration (offsets of the subgrid mid-point, size, masks)."""


class SwiftlyConfig:
    """SwiFTly configuration: sizes, window parameter and the processing core.

    :param W: PSWF parameter
    :param fov: field of view (kept for compatibility, unused like in the reference)
    :param N: image size
    :param yB_size: facet size
    :param yN_size: padded facet size
    :param xA_size: subgrid size
    :param xM_size: padded subgrid size
    :param dask_client: accepted for compatibility, ignored
    :param backend: ``"b200"`` (alias ``"cuda"``); the reference's backend names
        (``"numpy"``, ``"ska_sdp_func"``) are accepted and run on the same CUDA core
        (with a log warning) so that a reference driver only changes its import; any
        other name raises ``ValueError`` like the reference (api.py:137-143)
    :param device: CUDA device index (default: current device)
    :param core: optionally a ready-made object with the eight-primitive interface
    """

    # pylint: disable=too-many-arguments,too-many-instance-attributes
    def __init__(self, W, fov, N, yB_size, yN_size, xA_size, xM_size, dask_client=None,
                 backend="b200", device=None, core=None, **_other_args):
        self._W = W
        self._fov = fov
        self._N = N
        self._yB_size = yB_size
        self._yN_size = yN_size
        self._xA_size = xA_size
        self._xM_size = xM_size
        self.dask_client = dask_client
        if core is not None:
            self._core = core
        elif backend in ("b200", "cuda", "numpy", "ska_sdp_func"):
            if backend in ("numpy", "ska_sdp_func"):
                # a driver written for the reference passes its CPU backend names
                # (api.py:137-143); there is no CPU implementation here -- the same
                # primitives run on the GPU core
                log.warning("backend=%r requested: this package has no CPU backend, "
                            "using the B200 CUDA core", backend)
            self._core = SwiftlyCoreB200(W, N, xM_size, yN_size, device=device)
        else:
            raise ValueError(f"Unknown SwiFTly backend: {backend}")
        # the reference hands out a dask.delayed handle to the scattered core; here the
        # core itself plays that role (its methods run immediately on the GPU)
        self.core_task = self._core

    @property
    def core(self):
        """The processing core (eight SwiFTly primitives on the GPU)."""
        return self._core

    @property
    def image_size(self):
        """Size of the entire (virtual) image in pixels."""
        return self._N

    @property
    def max_facet_size(self):
        """Maximum size of a facet in pixels."""
        return self._yB_size

    @property
    def max_subgrid_size(self):
        """Maximum size of a subgrid in pixels."""
        return self._xA_size

    @property
    def pswf_parameter(self):
        """Parameter of the window function."""
        return self._W

    @property
    def internal_facet_size(self):
        """Padded facet size used internally."""
        return self._yN_size

    @property
    def internal_subgrid_size(self):
        """Padded subgrid size used internally."""
        return self._xM_size

    @property
    def facet_off_step(self):
        """All facet offsets must be divisible by this."""
        return self._core.facet_off_step

    @property
    def subgrid_off_step(self):
        """All subgrid offsets must be divisible by this."""
        return self._core.subgrid_off_step


def make_full_subgrid_cover(swiftlyconfig):
    """Subgrid configs covering the whole grid."""
    return make_full_cover_config(
        swiftlyconfig.image_size, swiftlyconfig.max_subgrid_size, SubgridConfig
    )


def make_full_facet_cover(swiftlyconfig):
    """Facet configs covering the whole image."""
    return make_full_cover_config(
        swiftlyconfig.image_size, swiftlyconfig.max_facet_size, FacetConfig
    )


# ---------------------------------------------------------------------- task handles
class DeviceTask:
    """Result handle: a device tensor plus the CUDA event that marks it complete.

    Stands in for the reference's dask futures / delayed objects.
    """

    def __init__(self, tensor):
        self.tensor = tensor
        self._event = None
        if torch is not None and hasattr(tensor, "is_cuda") and tensor.is_cuda:
            self._event = torch.cuda.Event()
            self._event.record(torch.cuda.current_stream(tensor.device))

    def done(self):
        """True once the GPU has produced the result."""
        return self._event is None or self._event.query()

    def wait(self):
        """Block until the result is complete."""
        if self._event is not None:
            self._event.synchronize()
        return self

    def result(self):
        """The result as a host numpy array."""
        self.wait()
        t = self.tensor
        return t.detach().cpu().numpy() if hasattr(t, "detach") else numpy.asarray(t)

    compute = result


def _resolve(data):
    """Turn whatever a caller passes as facet / subgrid data into an array or tensor."""
    if isinstance(data, DeviceTask):
        return data.tensor
    for attr in ("compute", "result"):
        if hasattr(data, attr) and not hasattr(data, "shape"):
            return getattr(data, attr)()
    if callable(data) and not hasattr(data, "shape"):
        return data()
    return data


class _TaskQueue:
    """Bound on the number of unfinished results (``queue_size`` of the reference)."""

    def __init__(self, max_task):
        self.max_task = max(1, int(max_task))
        self.pending = collections.deque()

    def process(self, tasks):
        for task in tasks:
            self.pending.append(task)
        while len(self.pending) > self.max_task:
            self.pending.popleft().wait()

    def wait_all_done(self):
        while self.pending:
            self.pending.popleft().wait()


class _LRU:
    """Least-recently-used cache keyed by subgrid column offset."""

    def __init__(self, size):
        self.size = max(1, int(size))
        self.data = collections.OrderedDict()

    def get(self, key):
        if key not in self.data:
            return None
        self.data.move_to_end(key)
        return self.data[key]

    def set(self, key, value):
        """Insert; returns the evicted ``(key, value)`` or ``(None, None)``."""
        self.data[key] = value
        self.data.move_to_end(key)
        if len(self.data) <= self.size:
            return None, None
        return self.data.popitem(last=False)

    def pop_all(self):
        while self.data:
            yield self.data.popitem(last=False)


def _device_of(core):
    dev = getattr(core, "tensor_device", None)
    if dev is not None:
        return dev
    return torch.device("cuda", core.device)


def _to_device(data, device, dtype=None):
    """complex128 tensor on ``device`` from a numpy array / tensor."""
    dtype = dtype or torch.complex128
    if isinstance(data, torch.Tensor):
        return data.to(device=device, dtype=dtype, non_blocking=True)
    arr = numpy.asarray(data)
    if dtype == torch.complex128 and arr.dtype != numpy.complex128:
        arr = arr.astype(numpy.complex128)
    return torch.from_numpy(numpy.ascontiguousarray(arr)).to(device, non_blocking=True)


def _upload_iter(datas, device, dtype=None):
    """Yield device tensors for ``datas`` in order.

    Host sources are uploaded on a side stream one item ahead of the consumer, so that the
    H2D copy of facet ``j + 1`` overlaps the kernels working on facet ``j`` (pinned host
    memory makes the copy asynchronous; pageable memory still works, without overlap).
    """
    datas = list(datas)
    use_side = device.type == "cuda"
    side = torch.cuda.Stream(device) if use_side else None

    def upload(data):
        data = _resolve(data)
        if isinstance(data, torch.Tensor) and data.device == device:
            return _to_device(data, device, dtype), None
        if not use_side:
            return _to_device(data, device, dtype), None
        with torch.cuda.stream(side):
            t = _to_device(data, device, dtype)
            ev = torch.cuda.Event()
            ev.record(side)
        return t, ev

    nxt = upload(datas[0]) if datas else None
    for j in range(len(datas)):
        cur = nxt
        nxt = upload(datas[j + 1]) if j + 1 < len(datas) else None
        t, ev = cur
        if ev is not None:
            torch.cuda.current_stream(device).wait_event(ev)
            t.record_stream(torch.cuda.current_stream(device))
        yield t


# ---------------------------------------------------------------------- host tier
def device_tier_bytes(direction, yN, m, facet_sizes, lru, n_rows=0, subgrid_size=0,
                      half_rows=False):
    """Bytes of device memory the device tier of a one-GPU transform holds at its peak.

    ``"forward"``: every prepared facet ``BF_F`` (``yN x size``), ``lru`` subgrid columns of
    ``NMBF_BF`` (``m x yN`` per facet), the subgrid strips (``n_rows x m x subgrid_size``) and the
    stage-1 scratch (one ``yN x size`` facet).  ``"backward"``: every facet accumulator
    (``yN x size``) and ``lru`` columns of accumulators (``m x yN`` per facet).  When this exceeds
    the device budget, :class:`SwiftlyForward` / :class:`SwiftlyBackward` keep those facet arrays
    in pinned host memory instead (the host tier).  ``half_rows``: the facet arrays have
    ``yN // 2 + 1`` rows (real images, ``half_rows=True`` of the transforms).
    """
    sizes = list(facet_sizes)
    facets = 16 * (yN // 2 + 1 if half_rows else yN) * sum(sizes)
    columns = 16 * max(1, int(lru)) * len(sizes) * m * yN
    if direction == "backward":
        return facets + columns
    if direction != "forward":
        raise ValueError(f"direction must be 'forward' or 'backward', not {direction!r}")
    return facets + columns + 16 * n_rows * m * subgrid_size + 16 * yN * max(sizes, default=0)


def _device_budget(device, device_budget):
    """``device_budget`` if given, else the free memory of ``device`` (no limit on the CPU
    "device" of the emulated library)."""
    if device_budget is not None:
        return int(device_budget)
    if device.type != "cuda":
        return float("inf")
    return torch.cuda.mem_get_info(device)[0]


def window_start(core, subgrid_off0):
    """First row of the ``m``-row window of the ``yN``-row facet arrays that subgrid column
    ``subgrid_off0`` reads (forward) or adds into (backward); the window wraps modulo ``yN``."""
    yN, m = core.yN_size, core.xM_yN_size
    return (yN // 2 - m // 2 + (subgrid_off0 * yN) // core.N) % yN


class _RowWindow:
    """The ``m``-row window of the ``yN``-row facet arrays that the device rings hold.  Facet row
    ``r`` lives at ring line ``r mod m`` (``m`` divides ``yN``), so rows that stay when the window
    slides keep their line and each new row takes the line of a row that left."""

    def __init__(self, yN, m):
        self.yN = yN
        self.m = m
        self.start = None

    def rows(self, start):
        return [(start + u) % self.yN for u in range(self.m)]

    def move(self, start):
        """Slide to the window at ``start``; returns ``(leaving, entering)`` rows."""
        old = [] if self.start is None else self.rows(self.start)
        new = self.rows(start)
        self.start = start
        old_set, new_set = set(old), set(new)
        return [r for r in old if r not in new_set], [r for r in new if r not in old_set]

    def runs(self, rows):
        """``(first row, count)`` of the runs of consecutive ``rows`` that are also consecutive ring
        lines: a run ends at every multiple of ``m``, so also at the wrap at ``yN``."""
        out = []
        for r in rows:
            if out and r == out[-1][0] + out[-1][1] and r % self.m:
                out[-1][1] += 1
            else:
                out.append([r, 1])
        return [(r, n) for r, n in out]


class _Copier:
    """Copies between host memory and the device on one copy stream, ordered against the compute
    stream by events.  On the emulated library's CPU "device" every copy runs at once."""

    def __init__(self, device):
        self.device = device
        self.stream = torch.cuda.Stream(device) if device.type == "cuda" else None
        self.h2d_bytes = 0
        self.d2h_bytes = 0

    def _compute(self):
        return torch.cuda.current_stream(self.device)

    def use(self, t):
        """``t`` (a device tensor) is used on the copy stream: keep its memory until then."""
        if self.stream is not None:
            t.record_stream(self.stream)
        return t

    def record(self, on_copy=True):
        """Event after the work queued so far on the copy (or compute) stream; None on the CPU."""
        if self.stream is None:
            return None
        ev = torch.cuda.Event()
        ev.record(self.stream if on_copy else self._compute())
        return ev

    def copy_waits(self, ev):
        if ev is not None:
            self.stream.wait_event(ev)

    def compute_waits(self, ev):
        if ev is not None:
            self._compute().wait_event(ev)

    def after_compute(self):
        """Later copies wait for everything queued so far on the compute stream."""
        self.copy_waits(self.record(on_copy=False))

    def copy(self, dst, src, to_host):
        """Queue ``dst.copy_(src)``: device -> host if ``to_host``, else host -> device."""
        nbytes = src.numel() * src.element_size()
        if to_host:
            self.d2h_bytes += nbytes
        else:
            self.h2d_bytes += nbytes
        if self.stream is None:
            dst.copy_(src)
            return
        with torch.cuda.stream(self.stream):
            dst.copy_(src, non_blocking=True)

    def zero(self, t):
        if self.stream is None:
            t.zero_()
            return
        with torch.cuda.stream(self.stream):
            t.zero_()

    def synchronize(self):
        if self.stream is not None:
            self.stream.synchronize()


class PinnedArena:
    """One page-locked host allocation, cut into ``(rows, size)`` complex128 views.

    The memory is a plain CPU tensor registered with ``cudaHostRegister`` (torch's caching host
    allocator would round the block size up).  On the emulated library's CPU "device" it stays
    pageable.  ``seconds`` is the time allocation and pinning took.  Views handed out stay valid
    after :meth:`release` (the memory is then pageable until the last view goes).
    """

    def __init__(self, shapes, device):
        t0 = time.perf_counter()
        self.shapes = [tuple(int(d) for d in s) for s in shapes]
        total = sum(a * b for a, b in self.shapes)
        self.tensor = torch.empty(max(1, total), dtype=torch.complex128)
        self.nbytes = self.tensor.numel() * 16
        self._registered = False
        if device.type == "cuda":
            with torch.cuda.device(device):
                torch.cuda.check_error(torch.cuda.cudart().cudaHostRegister(
                    self.tensor.data_ptr(), self.nbytes, 0))
            self._registered = True
        self.seconds = time.perf_counter() - t0
        self.views = []
        off = 0
        for a, b in self.shapes:
            self.views.append(self.tensor[off:off + a * b].view(a, b))
            off += a * b

    def release(self):
        """Unpin the memory (idempotent)."""
        if self._registered:
            self._registered = False
            torch.cuda.cudart().cudaHostUnregister(self.tensor.data_ptr())

    def __del__(self):
        try:
            self.release()
        except Exception:  # pylint: disable=broad-except
            pass


# facets per K2 launch of the forward host tier: the H2D copy of the next batch's new ring rows
# overlaps K2 of this batch
RING_BATCH = 8


def _device_mask(mask, device):
    """float64 device mask, or None when the mask is absent or all ones."""
    if mask is None:
        return None
    arr = numpy.asarray(mask, dtype=float)
    if arr.all() and (arr == 1).all():
        return None
    return torch.from_numpy(numpy.ascontiguousarray(arr)).to(device)


def _real_facet(idx, data):
    """``data`` resolved, after checking that it is real-valued (a real floating dtype)."""
    data = _resolve(data)
    if isinstance(data, torch.Tensor):
        real = data.is_floating_point()
    else:
        data = numpy.asarray(data)
        real = data.dtype.kind == "f"
    if not real:
        raise ValueError(f"real_image=True: facet {idx} has dtype {data.dtype}, expected a real "
                         "floating dtype")
    return data


def _half_rows_mode(half_rows, real_image):
    if half_rows and not real_image:
        raise ValueError("half_rows=True is valid only together with real_image=True")
    return bool(half_rows)


def _half_rows_budget(need, budget):
    """The half-row mode runs in the device tier only."""
    if need > budget:
        raise NotImplementedError(
            f"half_rows=True runs in the device tier only: it needs an estimated {need} bytes "
            f"of device memory, the budget is {budget} bytes")


def mirror_pairs(subgrid_configs, N, xM):
    """How the real-image forward transform covers ``subgrid_configs``: a list of
    ``(i, j)`` in the order of the sources ``i``, where ``j`` is the index of the config whose
    subgrid is mirrored from source ``i``, or None when ``i`` is computed alone.

    Configs pair greedily in list order: config ``i`` pairs with the first unpaired later config
    of the same size at offsets ``(-off0 mod N, -off1 mod N)``, provided the source size
    ``2 * (size // 2) + 1`` fits ``xM``.  Self-mirrored configs (``2 * off = 0 mod N`` on both
    axes) stay unpaired.
    """
    def key(sg, sign=1):
        return (sg.size, (sign * sg.off0) % N, (sign * sg.off1) % N)

    later = collections.defaultdict(collections.deque)  # key -> indices, in list order
    for idx, sg in enumerate(subgrid_configs):
        later[key(sg)].append(idx)
    paired = set()
    plan = []
    for i, sg in enumerate(subgrid_configs):
        if i in paired:
            continue
        j = None
        mkey = key(sg, -1)
        if mkey != key(sg) and 2 * (sg.size // 2) + 1 <= xM:
            queue = later[mkey]
            while queue and (queue[0] <= i or queue[0] in paired):
                queue.popleft()
            if queue:
                j = queue.popleft()
                paired.add(j)
        plan.append((i, j))
    return plan


# ---------------------------------------------------------------------- forward
class SwiftlyForward:
    """Facet -> subgrid streaming transform on one GPU.

    :param swiftly_config: ``SwiftlyConfig``
    :param facet_tasks: list of ``(FacetConfig, data)``; ``data`` is a numpy array, a
        (CUDA) tensor, or something with ``.compute()`` / ``.result()``
    :param lru_forward: number of subgrid columns whose prepared facet columns
        (``NMBF_BF``) stay resident
    :param queue_size: maximum number of unfinished subgrid results
    :param client: accepted for compatibility, ignored
    :param bf_f_buffers: optional preallocated ``(yN, size)`` tensors that receive the
        axis-0 prepared facets.  Device tensors may reuse storage of facets that were
        consumed earlier in the list (facets are processed in list order); host tensors
        (ideally pinned, e.g. the views of a :class:`PinnedArena`) select the host tier
    :param device_budget: bytes of device memory the transform may use (default: the
        device's free memory now).  When the device tier needs more
        (:func:`device_tier_bytes`), the prepared facets live in pinned host memory and
        each subgrid column brings only its ``m``-row window of them to the device (the
        host tier); the subgrids are the same bits either way
    :param real_image: the facets are real-valued (numpy arrays or tensors of a real floating
        dtype; ``ValueError`` otherwise).  The grid is then Hermitian, and
        :meth:`iter_subgrid_tasks` computes one subgrid of each pair at ``(off0, off1)`` /
        ``(-off0, -off1)`` and mirrors the other (:func:`mirror_pairs`).  Needs the fused
        kernels (``NotImplementedError`` otherwise).  :meth:`get_subgrid_task` is unchanged
    :param half_rows: with ``real_image`` only (``ValueError`` otherwise): every prepared facet
        is kept as its ``yN // 2 + 1`` half rows (``prepare_facet_real_half``; the other rows are
        their conjugates), half the device memory of the facet arrays.  The facets are uploaded
        as float64.  Device tier only: ``NotImplementedError`` when :func:`device_tier_bytes`
        with ``half_rows=True`` exceeds the budget or ``bf_f_buffers`` are host tensors;
        ``bf_f_buffers`` must have the half shape.  The subgrids differ from ``real_image`` alone
        by rounding only
    """

    # pylint: disable=too-many-arguments,too-many-instance-attributes
    def __init__(self, swiftly_config, facet_tasks, lru_forward=1, queue_size=20, client=None,
                 bf_f_buffers=None, device_budget=None, real_image=False, half_rows=False):
        self.config = swiftly_config
        self.facet_tasks = list(facet_tasks)
        self.core = swiftly_config.core
        self.device = _device_of(self.core)
        self.BF_Fs_persist = None
        self._bf_f_buffers = bf_f_buffers
        self.task_queue = _TaskQueue(queue_size)
        self.lru = _LRU(lru_forward)
        self._client = client
        # facets that share off0 form a "facet row": their contributions are combined
        # along axis 1 first, the rows then along axis 0
        rows = collections.OrderedDict()
        for idx, (cfg, _) in enumerate(self.facet_tasks):
            rows.setdefault(cfg.off0, []).append(idx)
        self._rows = list(rows.items())
        self._sizes = collections.OrderedDict()  # subgrid size -> strips, prepared K3 / K4
        self._masks = {}
        self._fused = bool(getattr(self.core, "fused_forward_supported", lambda: False)())
        self.real_image = bool(real_image)
        self.half_rows = _half_rows_mode(half_rows, self.real_image)
        if self.real_image:
            if not self._fused:
                raise NotImplementedError(
                    "real_image=True needs the fused forward kernels, which this core lacks")
            self.facet_tasks = [(cfg, _real_facet(idx, data))
                                for idx, (cfg, data) in enumerate(self.facet_tasks)]
        if self.half_rows and bf_f_buffers is not None:
            for (cfg, _), buf in zip(self.facet_tasks, bf_f_buffers):
                if buf.device != self.device:
                    raise NotImplementedError(
                        "half_rows=True runs in the device tier only: bf_f_buffers must be "
                        f"tensors on {self.device}")
                shape = (self.core.half_rows, cfg.size)
                if tuple(buf.shape) != shape or buf.dtype != torch.complex128:
                    raise ValueError(f"half_rows=True: bf_f_buffers entry of shape "
                                     f"{tuple(buf.shape)} and dtype {buf.dtype}, expected "
                                     f"{shape} complex128")
        self.host_tier = self._fused and self._select_host_tier(device_budget)
        self.arena = None
        self._rings = None
        self._ring_k2 = None
        self._window = None
        # rows of the m-row window copied host -> device in stage 2 (per facet)
        self.h2d_rows = 0
        self._copier = _Copier(self.device) if self.host_tier else None

    def _select_host_tier(self, device_budget):
        if self._bf_f_buffers is not None:
            return self._bf_f_buffers[0].device != self.device
        if not self.facet_tasks:
            return False
        core = self.core
        sizes = [cfg.size for cfg, _ in self.facet_tasks]
        need = device_tier_bytes("forward", core.yN_size, core.xM_yN_size, sizes, self.lru.size,
                                 len(self._rows), self.config.max_subgrid_size,
                                 half_rows=self.half_rows)
        budget = _device_budget(self.device, device_budget)
        if self.half_rows:
            _half_rows_budget(need, budget)
        return need > budget

    @property
    def copied_bytes(self):
        """``(host -> device, device -> host)`` bytes the host tier moved so far."""
        cp = self._copier
        return (cp.h2d_bytes, cp.d2h_bytes) if cp is not None else (0, 0)

    # -- stage 1: prepare every facet along axis 0 (once) --------------------------------
    def _stage1_host(self):
        """K1 into two device buffers in turn; the copy stream moves each finished buffer to the
        facet's host ``BF_F`` while K1 prepares the next facet.  K1 of facet ``j + 2`` waits for
        the copy of facet ``j``."""
        core, cp = self.core, self._copier
        yN = core.yN_size
        sizes = [cfg.size for cfg, _ in self.facet_tasks]
        if self._bf_f_buffers is not None:
            hosts = list(self._bf_f_buffers)
        else:
            self.arena = PinnedArena([(yN, s) for s in sizes], self.device)
            hosts = self.arena.views
        stage = cp.use(torch.empty((2, yN * max(sizes)), dtype=torch.complex128,
                                   device=self.device))
        copied = [None, None]
        uploads = _upload_iter([data for _, data in self.facet_tasks], self.device)
        for idx, ((cfg, _), facet) in enumerate(zip(self.facet_tasks, uploads)):
            slot = idx % 2
            cp.compute_waits(copied[slot])
            buf = stage[slot, :yN * cfg.size].view(yN, cfg.size)
            core.prepare_facet(facet, cfg.off0, axis=0, out=buf, window_lines=True)
            del facet
            cp.after_compute()
            cp.copy(hosts[idx], buf, True)
            copied[slot] = cp.record()
        return hosts

    def _get_BF_Fs(self):
        if self.BF_Fs_persist is None and self.host_tier:
            self.BF_Fs_persist = self._stage1_host()
            self.facet_tasks = [(cfg, None) for cfg, _ in self.facet_tasks]
        if self.BF_Fs_persist is None:
            out = []
            uploads = _upload_iter([data for _, data in self.facet_tasks], self.device,
                                   torch.float64 if self.half_rows else None)
            for idx, ((cfg, _), facet) in enumerate(zip(self.facet_tasks, uploads)):
                buf = None if self._bf_f_buffers is None else self._bf_f_buffers[idx]
                if self.half_rows:
                    # float64 with adjacent columns (a .real view of a complex facet has none),
                    # so that K1 takes its two-pass form
                    facet = facet.to(torch.float64).contiguous()
                    out.append(self.core.prepare_facet_real_half(facet, cfg.off0, axis=0,
                                                                 out=buf))
                elif self._fused:
                    # pre-windowed along axis 1 (the K2 kernel then skips its Fb multiply)
                    out.append(self.core.prepare_facet(facet, cfg.off0, axis=0, out=buf,
                                                       window_lines=True))
                else:
                    out.append(self.core.prepare_facet(facet, cfg.off0, axis=0, out=buf))
                del facet
            # facets are dead from here on: drop the references held by the task list
            self.facet_tasks = [(cfg, None) for cfg, _ in self.facet_tasks]
            self.BF_Fs_persist = out
            # (stage 1's scratch -- bounded at 2 GiB -- stays cached in the plan: freeing and
            # re-allocating it per transform cost 100-350 ms of cudaMalloc per step, measured.
            # ``core.release_scratch()`` gives it back explicitly.)
        return self.BF_Fs_persist

    # -- stage 2: per subgrid column ------------------------------------------------------
    def get_NMBF_BFs_off0(self, off0, BF_Fs):
        """Prepared facet columns for subgrid column ``off0`` (LRU cached)."""
        cached = self.lru.get(off0)
        if cached is None:
            reuse = None
            if len(self.lru.data) >= self.lru.size:
                # recycle the buffers of the column that is about to be evicted
                _, reuse = self.lru.data.popitem(last=False)
            if self.host_tier:
                cached = self._columns_from_rings(BF_Fs, off0, reuse)
            elif self._fused:
                cached = self.core.extract_columns(
                    BF_Fs, off0, [cfg.off1 for cfg, _ in self.facet_tasks], outs=reuse,
                    prewindowed=True)
            else:
                cached = [extract_column(self.core, BF_F, off0, cfg.off1)
                          for (cfg, _), BF_F in zip(self.facet_tasks, BF_Fs)]
            self.lru.set(off0, cached)
        return cached

    def _columns_from_rings(self, hosts, off0, outs):
        """K2 of the host tier: every facet has a device ring of ``m`` rows; the rows of the
        column's window that the rings lack are copied from the host ``BF_F`` (the copy of batch
        ``b + 1`` overlaps K2 of batch ``b``), then K2 reads the rings."""
        core, cp = self.core, self._copier
        m, yN = core.xM_yN_size, core.yN_size
        n = len(hosts)
        if self._rings is None:
            self._rings = [cp.use(torch.empty((m, h.shape[1]), dtype=torch.complex128,
                                              device=self.device)) for h in hosts]
            self._ring_k2 = [None] * len(range(0, n, RING_BATCH))
            self._window = _RowWindow(yN, m)
        _, entering = self._window.move(window_start(core, off0))
        runs = self._window.runs(entering)
        self.h2d_rows += len(entering)
        if outs is None:
            outs = [torch.empty((m, yN), dtype=torch.complex128, device=self.device)
                    for _ in hosts]
        off1s = [cfg.off1 for cfg, _ in self.facet_tasks]
        for b, lo in enumerate(range(0, n, RING_BATCH)):
            hi = min(lo + RING_BATCH, n)
            # the ring lines about to be overwritten were last read by K2 of this batch
            cp.copy_waits(self._ring_k2[b])
            for j in range(lo, hi):
                for r0, cnt in runs:
                    cp.copy(self._rings[j][r0 % m:r0 % m + cnt], hosts[j][r0:r0 + cnt], False)
            cp.compute_waits(cp.record())
            core.extract_columns(self._rings[lo:hi], off0, off1s[lo:hi], outs=outs[lo:hi],
                                 prewindowed=True)
            self._ring_k2[b] = cp.record(on_copy=False)
        return outs

    # -- stage 3: per subgrid ---------------------------------------------------------------
    def _gen_subgrid(self, subgrid_config, NMBF_BFs):
        core = self.core
        sg = subgrid_config
        if not self._fused:
            contribs = [core.extract_from_facet(nb, sg.off1, axis=1) for nb in NMBF_BFs]
            return sum_and_finish_subgrid(
                core, contribs, [cfg for cfg, _ in self.facet_tasks], sg
            )
        m = core.xM_yN_size
        st = self._size_state(sg.size)
        strips = st["strips"]
        mask0 = self._mask(sg, 0)
        mask1 = self._mask(sg, 1)
        # the argument blocks are built once per subgrid column (axis 1) / once per transform
        # (axis 0) and subgrid size, and reused: per subgrid only offsets, masks and the output
        # pointer change
        key = id(NMBF_BFs)
        if st["prep1"] is None or st["prep1"][0] != key:
            for other in self._sizes.values():  # no block keeps an earlier column alive
                if other["prep1"] is not None and other["prep1"][0] != key:
                    other["prep1"] = None
            groups =[[(NMBF_BFs[j], self.facet_tasks[j][0].off1) for j in members]
                      for _, members in self._rows]
            st["prep1"] = (key, core.prepare_sum_finish(
                groups, 1, m, sg.size, (strips.stride(1), strips.stride(2))), NMBF_BFs)
        nrows = len(self._rows)
        st["prep1"][1].launch([sg.off1] * nrows, [mask1] * nrows, out=strips,
                              out_group_stride=strips.stride(0))
        out = torch.empty((sg.size, sg.size), dtype=torch.complex128, device=self.device)
        if st["prep0"] is None:
            sources = [[(strips[r], off0) for r, (off0, _) in enumerate(self._rows)]]
            st["prep0"] = core.prepare_sum_finish(
                sources, 0, sg.size, sg.size, (out.stride(1), out.stride(0)))
        st["prep0"].launch([sg.off0], [mask0], out=out)
        return out

    def _size_state(self, size):
        """Subgrid strips and prepared K3 / K4 blocks of one subgrid size.  The two sizes used
        last are kept: the real-image mode alternates a column's source size ``S`` and its
        subgrid size when the column holds self-mirrored subgrids."""
        st = self._sizes.get(size)
        if st is None:
            # strips stored TRANSPOSED -- (row, xA, m), contribution index contiguous -- so that
            # the axis-0 kernel reads unit-stride lines; the axis-1 kernel's finished lines are
            # scattered into this layout by the TMA engine (bulk tensor stores)
            strips = torch.empty((len(self._rows), size, self.core.xM_yN_size),
                                 dtype=torch.complex128, device=self.device).transpose(1, 2)
            st = {"strips": strips, "prep1": None, "prep0": None}
            if len(self._sizes) >= 2:
                self._sizes.popitem(last=False)
            self._sizes[size] = st
        self._sizes.move_to_end(size)
        return st

    def _mask(self, sg, axis):
        """Device mask of a subgrid along ``axis`` (None when absent or all ones), cached by
        (axis, offset, size): a cover has only a few distinct masks per axis."""
        off = sg.off0 if axis == 0 else sg.off1
        key = (axis, off, sg.size)
        if key not in self._masks:
            self._masks[key] = _device_mask(sg.mask0 if axis == 0 else sg.mask1, self.device)
        return self._masks[key]

    def get_subgrid_task(self, subgrid_config):
        """Enqueue the computation of one subgrid and return its handle."""
        BF_Fs = self._get_BF_Fs()
        NMBF_BFs = self.get_NMBF_BFs_off0(subgrid_config.off0, BF_Fs)
        task = DeviceTask(self._gen_subgrid(subgrid_config, NMBF_BFs))
        self.task_queue.process([task])
        return task

    def iter_subgrid_tasks(self, subgrid_configs):
        """Enqueue every subgrid of ``subgrid_configs``; yields ``(index, task)`` once per config.

        Default: :meth:`get_subgrid_task` in list order.  With ``real_image``, configs pair as
        :func:`mirror_pairs` says.  A pair's source is computed once, without masks, at the odd
        size ``S = 2 * (size // 2) + 1`` (K2 for its column, K3 and K4 at ``S``); one
        ``mirror_subgrid`` launch then writes both subgrids with their own masks.  The source's
        task is yielded first, its mirror's right after.  Unpaired configs run
        :meth:`get_subgrid_task`.
        """
        configs = list(subgrid_configs)
        if not self.real_image:
            for i, sg in enumerate(configs):
                yield i, self.get_subgrid_task(sg)
            return
        for i, j in mirror_pairs(configs, self.config.image_size,
                                 self.config.internal_subgrid_size):
            if j is None:
                yield i, self.get_subgrid_task(configs[i])
                continue
            sg, mg = configs[i], configs[j]
            BF_Fs = self._get_BF_Fs()
            NMBF_BFs = self.get_NMBF_BFs_off0(sg.off0, BF_Fs)
            size = 2 * (sg.size // 2) + 1
            src = self._gen_subgrid(SubgridConfig(sg.off0, sg.off1, size), NMBF_BFs)
            out, mirror = self.core.mirror_subgrid(
                src, sg.size, masks=(self._mask(sg, 0), self._mask(sg, 1)),
                mirror_masks=(self._mask(mg, 0), self._mask(mg, 1)))
            del src
            tasks = [DeviceTask(out), DeviceTask(mirror)]
            self.task_queue.process(tasks)
            yield i, tasks[0]
            yield j, tasks[1]


# ---------------------------------------------------------------------- backward
class SwiftlyBackward:
    """Subgrid -> facet streaming accumulation on one GPU.

    :param swiftly_config: ``SwiftlyConfig``
    :param facets_config_list: facets to produce
    :param lru_backward: number of subgrid columns whose facet column accumulators
        (``NAF_MNAF``) stay resident before they are folded into the facets
    :param queue_size: maximum number of unfinished results
    :param client: accepted for compatibility, ignored
    :param device_budget: bytes of device memory the transform may use (default: the
        device's free memory now).  When the device tier needs more
        (:func:`device_tier_bytes`), the facet accumulators live in pinned host memory and
        the device holds only the ``m``-row window the current column adds into (the host
        tier); ``finish()`` then returns the facets in pinned host memory, the same bits
    :param real_image: the image is real-valued: ``finish()`` returns the real part of the
        facets as float64 (``finish_facet_real``), and :meth:`add_subgrid_tasks` merges each
        Hermitian pair of subgrids at ``(off0, off1)`` / ``(-off0, -off1)`` into one subgrid
        (``merge_mirror_subgrid``) before the subgrid side, which then runs once per pair.
        Needs the fused kernels (``NotImplementedError`` otherwise).
        :meth:`add_new_subgrid_task` is unchanged.  The sharded backward transform
        (``SwiftlyBackwardSharded``) has no real-image mode
    :param half_rows: with ``real_image`` only (``ValueError`` otherwise): the facet accumulators
        hold ``yN // 2 + 1`` half rows (``fold_column`` adds the conjugate of the rows it
        mirrors, ``finish_facet_real_half`` finishes them), half their device memory.  Device
        tier only: ``NotImplementedError`` when :func:`device_tier_bytes` with
        ``half_rows=True`` exceeds the budget.  The facets differ from ``real_image`` alone by
        rounding only
    """

    # pylint: disable=too-many-arguments,too-many-instance-attributes
    def __init__(self, swiftly_config, facets_config_list, lru_backward=1, queue_size=20,
                 client=None, device_budget=None, real_image=False, half_rows=False):
        self.config = swiftly_config
        self.core = swiftly_config.core
        self.device = _device_of(self.core)
        self.facets_config_list = list(facets_config_list)
        self.MNAF_BMNAFs_persist = [None for _ in self.facets_config_list]
        self.task_queue = _TaskQueue(queue_size)
        self.lru = _LRU(lru_backward)
        self._client = client
        # fused kernels: one launch per subgrid for all facets (extract axis 1 + accumulate
        # column), one launch per finished column for all facets (finish axis 1 + mask + add
        # axis 0); otherwise the reference's task bodies run primitive by primitive
        self._fused = bool(hasattr(self.core, "subgrid_to_facets")
                           and getattr(self.core, "fused_backward_supported", lambda: False)())
        # the subgrid side as two split kernels per subgrid (K4T along axis 0 into one strip
        # per facet row, K3T along axis 1 into the column accumulators); the prepared subgrid
        # and the (m, xM) blocks of the primitive chain never exist
        self._split = self._fused and bool(
            getattr(self.core, "split_axis_supported", lambda: False)())
        rows = collections.OrderedDict()
        for idx, cfg in enumerate(self.facets_config_list):
            rows.setdefault(cfg.off0, []).append(idx)
        self._rows = list(rows.items())
        self._row_members = dict(self._rows)
        # K4T strip buffers of the last two subgrid widths: real-image columns that hold
        # self-mirrored subgrids alternate the merged width S and the subgrid width
        self._strips = collections.OrderedDict()
        self._masks1 = None
        self.real_image = bool(real_image)
        self.half_rows = _half_rows_mode(half_rows, self.real_image)
        if self.real_image and not self._fused:
            raise NotImplementedError(
                "real_image=True needs the fused backward kernels, which this core lacks")
        need = device_tier_bytes(
            "backward", self.core.yN_size, self.core.xM_yN_size,
            [cfg.size for cfg in self.facets_config_list], self.lru.size,
            half_rows=self.half_rows)
        budget = _device_budget(self.device, device_budget)
        if self.half_rows and self.facets_config_list:
            _half_rows_budget(need, budget)
        self.host_tier = self._fused and bool(self.facets_config_list) and need > budget
        self.arena = None
        self._rings = None
        self._window = None
        self._touched = None  # per facet row: written back to the host accumulators yet
        # rows of the m-row window moved per facet: host -> device, device -> host, zero-filled
        self.h2d_rows = 0
        self.d2h_rows = 0
        self.zeroed_rows = 0
        self._copier = _Copier(self.device) if self.host_tier else None

    @property
    def copied_bytes(self):
        """``(host -> device, device -> host)`` bytes the host tier moved so far."""
        cp = self._copier
        return (cp.h2d_bytes, cp.d2h_bytes) if cp is not None else (0, 0)

    def _write_back(self, rows):
        """Queue the D2H copy of ``rows`` (held by the rings) to the host accumulators."""
        cp, m = self._copier, self.core.xM_yN_size
        for r0, cnt in self._window.runs(rows):
            for ring, host in zip(self._rings, self.arena.views):
                cp.copy(host[r0:r0 + cnt], ring[r0 % m:r0 % m + cnt], True)
        self._touched[rows] = True
        self.d2h_rows += len(rows)

    def _load_rows(self, rows, targets, line_of):
        """Queue the rows of the host accumulators into ``targets`` (line ``line_of(r)`` for row
        ``r``): copied if a column wrote them back before, zero-filled otherwise."""
        cp = self._copier
        touched = [r for r in rows if self._touched[r]]
        fresh = [r for r in rows if not self._touched[r]]
        for r0, cnt in self._window.runs(touched):
            for t, host in zip(targets, self.arena.views):
                cp.copy(t[line_of(r0):line_of(r0) + cnt], host[r0:r0 + cnt], False)
        for r0, cnt in self._window.runs(fresh):
            for t in targets:
                cp.zero(t[line_of(r0):line_of(r0) + cnt])
        self.h2d_rows += len(touched)
        self.zeroed_rows += len(fresh)

    def _slide_rings(self, off0):
        """Make the rings hold the window of subgrid column ``off0``: rows that leave go back to
        the host after the folds queued so far, then rows that enter are loaded, all on one copy
        stream (a row written back is never read back before it lands)."""
        core, cp = self.core, self._copier
        m, yN = core.xM_yN_size, core.yN_size
        if self._rings is None:
            self.arena = PinnedArena([(yN, cfg.size) for cfg in self.facets_config_list],
                                     self.device)
            self._rings = [cp.use(torch.empty((m, cfg.size), dtype=torch.complex128,
                                              device=self.device))
                           for cfg in self.facets_config_list]
            self._window = _RowWindow(yN, m)
            self._touched = numpy.zeros(yN, dtype=bool)
        start = window_start(core, off0)
        if start == self._window.start:
            return
        leaving, entering = self._window.move(start)
        cp.after_compute()
        if leaving:
            self._write_back(leaving)
        self._load_rows(entering, self._rings, lambda r: r % m)
        cp.compute_waits(cp.record())

    def _finish_host(self):
        """Flush the rings, then per facet: the accumulator into one reused ``yN x size`` device
        buffer, ``finish_facet`` along axis 0, the facet back into pinned host memory (the start
        of the facet's own, no longer needed, accumulator)."""
        core, cp = self.core, self._copier
        yN = core.yN_size
        tasks = []
        if self._rings is None:  # no column was folded: every accumulator is zero
            self._slide_rings(0)
        cp.after_compute()
        self._write_back(self._window.rows(self._window.start))
        self._rings = None
        sizes = [cfg.size for cfg in self.facets_config_list]
        buf = cp.use(torch.empty(yN * max(sizes), dtype=torch.complex128, device=self.device))
        touched = self._window.runs([r for r in range(yN) if self._touched[r]])
        fresh = self._window.runs([r for r in range(yN) if not self._touched[r]])
        for j, cfg in enumerate(self.facets_config_list):
            acc = buf[:yN * cfg.size].view(yN, cfg.size)
            host = self.arena.views[j]
            cp.after_compute()  # the previous facet's finish_facet has read the buffer
            for r0, cnt in touched:
                cp.copy(acc[r0:r0 + cnt], host[r0:r0 + cnt], False)
            for r0, cnt in fresh:
                cp.zero(acc[r0:r0 + cnt])
            cp.compute_waits(cp.record())
            if self.real_image:
                # float64 facet in the first half of the accumulator's bytes: half the D2H
                facet = self._finish_real(acc, cfg)
                out = host.reshape(-1).view(torch.float64)[:cfg.size * cfg.size]
            else:
                facet = finish_facet(core, acc, cfg)
                out = host.reshape(-1)[:cfg.size * cfg.size]
            out = out.view(cfg.size, cfg.size)
            cp.after_compute()
            cp.copy(out, cp.use(facet), True)
            tasks.append(DeviceTask(out))
        cp.synchronize()
        return tasks

    def add_new_subgrid_task(self, subgrid_config, new_subgrid_task):
        """Fold one subgrid into the facet accumulators."""
        subgrid = _to_device(_resolve(new_subgrid_task), self.device)
        return self._add_subgrid(subgrid, subgrid_config.off0, subgrid_config.off1)

    def _add_subgrid(self, subgrid, off0, off1):
        if self._split:
            done = self._add_subgrid_split(subgrid, off0, off1)
        elif self._fused:
            done = self._add_subgrid_fused(subgrid, off0, off1)
        else:
            pieces = prepare_and_split_subgrid(
                self.core, subgrid, [off0, off1], self.facets_config_list
            )
            done = self.update_off0_NAF_MNAFs(off0, off1, pieces)
        self.task_queue.process(done)
        return done

    def add_subgrid_tasks(self, subgrid_configs, subgrid_tasks):
        """Fold every subgrid of ``subgrid_configs`` (data in ``subgrid_tasks``, the same length;
        arrays, tensors or lazy handles, resolved when used) into the facet accumulators.
        Returns the :func:`mirror_pairs` plan it followed.

        Default: :meth:`add_new_subgrid_task` in list order, plan ``[(i, None), ...]``.  With
        ``real_image``, each pair ``(i, j)`` is merged (``merge_mirror_subgrid``) into one subgrid
        of size ``S = 2 * (size // 2) + 1`` at config ``i``'s offsets, which then runs the subgrid
        side once; the facets' real part is the same.  Unpaired and self-mirrored configs are
        added as they are.
        """
        configs = list(subgrid_configs)
        datas = list(subgrid_tasks)
        if len(configs) != len(datas):
            raise ValueError(f"{len(configs)} subgrid configs but {len(datas)} subgrids")
        if not self.real_image:
            for sg, data in zip(configs, datas):
                self.add_new_subgrid_task(sg, data)
            return [(i, None) for i in range(len(configs))]
        plan = mirror_pairs(configs, self.config.image_size, self.config.internal_subgrid_size)
        for i, j in plan:
            if j is None:
                self.add_new_subgrid_task(configs[i], datas[i])
                continue
            sg, mirror = (_to_device(_resolve(datas[k]), self.device) for k in (i, j))
            merged = self.core.merge_mirror_subgrid(sg, mirror)
            del sg, mirror
            self._add_subgrid(merged, configs[i].off0, configs[i].off1)
        return plan

    def _column_for(self, off0):
        """Column accumulators of subgrid column ``off0`` (LRU).  When a column has to make
        room, it is folded into the facets first and its buffers are recycled."""
        column = self.lru.get(off0)
        if column is not None:
            return column
        reuse = None
        if len(self.lru.data) >= self.lru.size:
            # fold the column that is about to be evicted NOW and recycle its buffers:
            # allocating the new column first would hold two columns (2 x 16 GiB at N=65536)
            # next to the 128 GiB of facet accumulators
            old_off0, reuse = self.lru.data.popitem(last=False)
            self.update_MNAF_BMNAFs(old_off0, reuse)
        if reuse is not None:
            column = reuse
            for acc in column:
                acc.zero_()
        else:
            shape = (self.core.xM_yN_size, self.core.yN_size)
            column = [torch.zeros(shape, dtype=torch.complex128, device=self.device)
                      for _ in self.facets_config_list]
        self.lru.set(off0, column)
        return column

    def _add_subgrid_split(self, subgrid, off0, off1):
        # K4T: the subgrid along axis 0 into one (m, xA) strip per distinct facet off0, kept
        # C-ordered so that the axis-0 lines (columns) are adjacent in memory
        width = subgrid.shape[1]
        strips = self._strips.get(width)
        if strips is None:
            strips = torch.empty((len(self._rows), self.core.xM_yN_size, width),
                                 dtype=torch.complex128, device=self.device)
            if len(self._strips) >= 2:
                self._strips.popitem(last=False)
            self._strips[width] = strips
        self._strips.move_to_end(width)
        self.core.split_subgrid_axis(
            [subgrid], 0, [off0], [[(strips[r], row) for r, (row, _) in enumerate(self._rows)]],
            "store")
        return self.add_strips(off0, [(strips[r], row, off1)
                                      for r, (row, _) in enumerate(self._rows)])

    def add_strips(self, off0, strips):
        """K3T: add facet-row strips of subgrids of column ``off0`` to the facets' column
        accumulators, ONE launch (per 16 strips / 64 facets) for all of them, in order.

        :param strips: list of ``(strip, row_off0, subgrid_off1)``: an ``(m, subgrid size)``
            device tensor, the facet ``off0`` it was cut for (K4T) and the subgrid's ``off1``;
            strips of rows without a facet here are skipped
        """
        column = self._column_for(off0)
        groups, offs, targets = [], [], []
        for strip, row, off1 in strips:
            members = self._row_members.get(row)
            if not members:
                continue
            groups.append(strip)
            offs.append(off1)
            targets.append([(column[j], self.facets_config_list[j].off1) for j in members])
        if groups:
            self.core.split_subgrid_axis(groups, 1, offs, targets, "add")
        return [DeviceTask(column[-1])] if column else []

    def _add_subgrid_fused(self, subgrid, off0, off1):
        core = self.core
        prepared = core.prepare_subgrid(subgrid, (off0, off1))
        blocks = {}
        for cfg in self.facets_config_list:
            if cfg.off0 not in blocks:
                blocks[cfg.off0] = core.extract_from_subgrid(prepared, cfg.off0, axis=0)
        column = self._column_for(off0)
        core.subgrid_to_facets(
            [blocks[cfg.off0] for cfg in self.facets_config_list], column,
            [cfg.off1 for cfg in self.facets_config_list], off1)
        return [DeviceTask(column[-1])] if column else []

    def update_off0_NAF_MNAFs(self, off0, off1, new_NAF_NAF_tasks):
        """Accumulate along axis 1 into the column accumulators of column ``off0``."""
        column = self.lru.get(off0)
        if column is None:
            column = [None for _ in self.facets_config_list]
        column = [
            accumulate_column(self.core, piece, acc, off1)
            for piece, acc in zip(new_NAF_NAF_tasks, column)
        ]
        tasks = [DeviceTask(column[-1])] if column else []
        old_off0, old_column = self.lru.set(off0, column)
        if old_off0 is not None:
            self.update_MNAF_BMNAFs(old_off0, old_column)
        return tasks

    def update_MNAF_BMNAFs(self, off0, new_NAF_MNAFs):
        """Finish a subgrid column along axis 1 and fold it into the facets (axis 0)."""
        if self.host_tier:
            if self._masks1 is None:
                self._masks1 = [_device_mask(cfg.mask1, self.device)
                                for cfg in self.facets_config_list]
            self._slide_rings(off0)
            self.core.fold_column(new_NAF_MNAFs, self._rings,
                                  [cfg.off1 for cfg in self.facets_config_list], self._masks1,
                                  off0)
            return self._rings
        if self._fused:
            core = self.core
            for j, cfg in enumerate(self.facets_config_list):
                if self.MNAF_BMNAFs_persist[j] is None:
                    rows = core.half_rows if self.half_rows else core.yN_size
                    self.MNAF_BMNAFs_persist[j] = torch.zeros(
                        (rows, cfg.size), dtype=torch.complex128, device=self.device)
            if self._masks1 is None:
                self._masks1 = [_device_mask(cfg.mask1, self.device)
                                for cfg in self.facets_config_list]
            core.fold_column(new_NAF_MNAFs, self.MNAF_BMNAFs_persist,
                             [cfg.off1 for cfg in self.facets_config_list], self._masks1, off0)
            return self.MNAF_BMNAFs_persist
        self.MNAF_BMNAFs_persist = [
            accumulate_facet(self.core, col, acc, cfg, off0)
            for cfg, col, acc in zip(
                self.facets_config_list, new_NAF_MNAFs, self.MNAF_BMNAFs_persist
            )
        ]
        return self.MNAF_BMNAFs_persist

    def finish(self):
        """Flush all pending columns and finish the facets; returns result handles."""
        for old_off0, old_column in self.lru.pop_all():
            self.update_MNAF_BMNAFs(old_off0, old_column)
        if self.host_tier:
            return self._finish_host()
        tasks = []
        for j, cfg in enumerate(self.facets_config_list):
            # release every accumulator as soon as its facet is finished: (yN, size) goes,
            # (size, size) stays -- at N=65536 on one GPU the 128 GiB of accumulators and the
            # 64 GiB of finished facets never coexist
            acc = self.MNAF_BMNAFs_persist[j]
            self.MNAF_BMNAFs_persist[j] = None
            if self.real_image:
                facet = self._finish_real(acc, cfg)
            else:
                facet = finish_facet(self.core, acc, cfg)
            del acc
            tasks.append(DeviceTask(facet))
        self.task_queue.process(tasks)
        self.task_queue.wait_all_done()
        return tasks

    def _finish_real(self, acc, cfg):
        """The real facet (float64) of a facet accumulator, masked inside the kernel."""
        if acc is None:
            return numpy.zeros((cfg.size, cfg.size))
        finish = self.core.finish_facet_real_half if self.half_rows else self.core.finish_facet_real
        return finish(acc, cfg.off0, cfg.size, axis=0, mask=_device_mask(cfg.mask0, self.device))
