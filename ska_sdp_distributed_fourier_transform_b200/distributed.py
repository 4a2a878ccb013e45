"""
Multi-GPU facet -> subgrid transform: one process per GPU, facets sharded.

The reference distributes one task per facet over Dask workers and ships every
``(m, m)`` contribution over TCP to the worker that sums a subgrid
(``api.py:263-277``; SURVEY.md section 3.2).  Here the facets are partitioned over the ranks
of a ``torch.distributed`` process group (NCCL over NVLink on the B200 box); each
rank keeps its facets' ``BF_F`` / ``NMBF_BF`` resident and, per subgrid, reduces
its facets along axis 1 *locally* into compact strips (``(m, xA)`` per distinct
facet ``off0`` on the rank -- the fused ``sum_finish_axis`` kernel).  The only data
exchange is those strips: subgrids are processed in batches of ``world_size``,
subgrid ``b`` of a batch is owned by rank ``b``, one ``all_to_all`` per batch moves
every rank's strips to the owners, and each owner runs the axis-0 kernel over the
strips of all ranks.  Per subgrid a rank sends ``n_local_rows * m * xA * 16`` bytes
(32 MiB at cfg4 on 8 GPUs) -- half of what reducing finished partial subgrids would
move and without replicating the axis-0 work.  The exchange of batch ``k`` runs on
the communication stream while the compute stream produces the strips of batch
``k + 1`` and finishes the subgrids of batch ``k - 1``.

Three exchange mechanisms (all parity-checked on 2 and 4 B200, ``tests/multi_gpu_check.py``):

* ``exchange="copy"`` (what ``"auto"`` selects): the axis-1 kernel writes the strips of a batch
  into a local send buffer, a communication stream moves every owner's part into that owner's
  receive slot -- symmetric memory (``torch.distributed._symmetric_memory``), every rank maps
  its peers' slots -- with plain device-to-device copies: NVLink DMA by the copy engines, no SM
  involved, so the transfer really runs beside the kernels; ordering by device-side flags
  (``peer_signal`` / ``peer_wait``, ``csrc/peer_sync.cu``), software pipelined by one batch.
* ``exchange="p2p"``: the axis-1 kernel of a batch stores its strips DIRECTLY into the owners'
  slots over NVLink -- bulk tensor stores of the TMA engine on peer-mapped addresses, the transfer
  is the kernel's own epilogue, no copy and no collective; same flags and pipeline.
* ``exchange="nccl"``: one ``all_to_all`` per batch on the communication stream, double
  buffered.  This is also the path the CPU (gloo) tests exercise.

Measured at cfg4 on 2 B200 (round 2, 625 ms of kernels per step): copy 639 ms, nccl 866 ms, p2p
921 ms.  The NCCL kernels need SMs, which the persistent one-CTA-per-SM kernels of this library
(up to 209 KiB of shared memory) do not leave free, so the collective serialises with them; the
16-byte rows of the transposed strips make poor NVLink packets for the TMA variant.

Calls are collective (SPMD): every rank must call ``get_subgrid_tasks`` with the same
subgrid list.
"""

import collections

import torch
import torch.distributed as dist

from .api import DeviceTask, _device_mask, _device_of, _LRU, _upload_iter


def partition_facets(facet_configs, world_size):
    """Owner rank of every facet: facets sorted by (off0, off1), split contiguously.

    For a full cover with ``rows % world_size == 0`` a rank owns whole facet rows; for a
    sparse cover rows are split so that no rank idles (only the sum over facets matters).
    """
    order = sorted(range(len(facet_configs)),
                   key=lambda i: (facet_configs[i].off0, facet_configs[i].off1))
    owner = [0] * len(facet_configs)
    n = len(order)
    for pos, idx in enumerate(order):
        owner[idx] = min(world_size - 1, pos * world_size // max(n, 1))
    return owner


class SwiftlyForwardSharded:
    """Facet -> subgrid transform with facets sharded over a process group.

    :param swiftly_config: ``SwiftlyConfig`` (its core lives on this rank's GPU)
    :param facet_configs: ALL facet configs (identical on every rank)
    :param local_facets: ``{facet index: data}`` for the facets this rank owns
        (see :func:`partition_facets`)
    :param lru_forward: resident subgrid columns
    :param group: process group (default: world)
    :param bf_f_buffers: optional ``{facet index: (yN, size) tensor}`` outputs of stage 1
    """

    # pylint: disable=too-many-instance-attributes,too-many-arguments
    def __init__(self, swiftly_config, facet_configs, local_facets, lru_forward=1, group=None,
                 bf_f_buffers=None, exchange="auto"):
        self.config = swiftly_config
        self.core = swiftly_config.core
        self.device = _device_of(self.core)
        self.group = group
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.facet_configs = list(facet_configs)
        self.owner = partition_facets(self.facet_configs, self.world)
        self.local_idx = [i for i, o in enumerate(self.owner) if o == self.rank]
        missing = [i for i in self.local_idx if i not in local_facets]
        if missing:
            raise ValueError(f"rank {self.rank} owns facets {missing} but got no data for them")
        self._local_facets = dict(local_facets)
        self._bf_f_buffers = bf_f_buffers or {}
        self.lru = _LRU(lru_forward)
        self.BF_Fs = None
        # strip layout: for every rank the sorted distinct off0 of its facets
        self.rank_rows = []
        for r in range(self.world):
            offs = sorted({self.facet_configs[i].off0
                           for i, o in enumerate(self.owner) if o == r})
            self.rank_rows.append(offs)
        self.rows_max = max(1, max(len(r) for r in self.rank_rows))
        self.my_rows = self.rank_rows[self.rank]
        self._bufs = {}
        self._prep1 = None   # (column key, prepared axis-1 launch over a full batch)
        self._prep0 = {}     # receive buffer -> prepared axis-0 launch
        self._masks = {}
        self._ptrs = {}      # output pointer tables of the batched axis-1 launch
        self.launches = 0
        if exchange not in ("auto", "copy", "p2p", "nccl"):
            raise ValueError(f"unknown exchange mechanism {exchange!r}")
        self.exchange = "nccl"
        self._symm = None
        self._comm_stream = None
        want = "copy" if exchange == "auto" else exchange
        if want in ("p2p", "copy") and self.world > 1 and self.device.type == "cuda":
            try:
                self._setup_symmetric()
                self.exchange = want
            except Exception as exc:  # pylint: disable=broad-except
                if exchange != "auto":
                    raise
                self._symm = None
                self.exchange_fallback_reason = f"{type(exc).__name__}: {exc}"

    # ------------------------------------------------------------------ symmetric memory
    def _setup_symmetric(self):
        """Allocate the receive slots as symmetric memory and map every peer's copy."""
        import torch.distributed._symmetric_memory as symm_mem  # pylint: disable=import-outside-toplevel

        grp = self.group if self.group is not None else dist.group.WORLD
        try:
            symm_mem.enable_symm_mem_for_group(grp.group_name)
        except Exception:  # pylint: disable=broad-except
            pass  # newer torch enables it lazily
        key = (grp.group_name, self.device.index, self.world, self.rows_max,
               self.core.xM_yN_size)
        if key not in self._SYMM_CACHE:
            self._SYMM_CACHE[key] = {"mod": symm_mem, "group": grp, "slots": {}}
        self._symm = self._SYMM_CACHE[key]

    N_SLOTS = 4  # see _run_p2p: a slot is rewritten four batches later
    # symmetric buffers are expensive to set up (a rendezvous over the group) and identical
    # for every transform of a geometry: they are kept per (group, device) across instances
    _SYMM_CACHE = {}

    def _symm_slots(self, xA):
        """(handle, [per-rank views of all slots]) for subgrid size ``xA``."""
        st = self._symm
        if xA not in st["slots"]:
            m = self.core.xM_yN_size
            # strips transposed (contribution index contiguous), see api.py
            shape = (self.N_SLOTS, self.world, self.rows_max, xA, m)
            n = 1
            for d in shape:
                n *= d
            buf = st["mod"].empty(2 * n, dtype=torch.float64, device=self.device)
            buf.zero_()
            hdl = st["mod"].rendezvous(buf, group=st["group"])
            views = []
            for r in range(self.world):
                peer = hdl.get_buffer(r, (2 * n,), torch.float64, 0)
                views.append(torch.view_as_complex(peer.view(n, 2)).view(shape).transpose(3, 4))
            st["slots"][xA] = (hdl, views, buf)
            # untransposed (storage order) views: a rank's part of a slot is one contiguous block
            st["bases"] = st.get("bases", {})
            st["bases"][xA] = [v.transpose(3, 4) for v in views]
        return st["slots"][xA]

    def _symm_flags(self):
        """Per-rank flag arrays (int64[world]) in symmetric memory: (table of my mappings of
        every rank's array, my own array, status word)."""
        st = self._symm
        if "flags" not in st:
            buf = st["mod"].empty(self.world, dtype=torch.int64, device=self.device)
            buf.zero_()
            hdl = st["mod"].rendezvous(buf, group=st["group"])
            maps = [hdl.get_buffer(r, (self.world,), torch.int64, 0) for r in range(self.world)]
            table = torch.tensor([t.data_ptr() for t in maps], dtype=torch.int64,
                                 device=self.device)
            status = torch.zeros(1, dtype=torch.int32, device=self.device)
            if self.device.type == "cuda":
                torch.cuda.synchronize(self.device)
            hdl.barrier(channel=0)  # everybody's flags are zero before anybody signals
            st["flags"] = (hdl, maps, table, buf, status)
            st["seq"] = 0
        return st["flags"]

    # ------------------------------------------------------------------ local stages
    def _prepare(self):
        if self.BF_Fs is None:
            self.BF_Fs = {}
            uploads = _upload_iter([self._local_facets[i] for i in self.local_idx], self.device)
            for i, facet in zip(self.local_idx, uploads):
                cfg = self.facet_configs[i]
                self.BF_Fs[i] = self.core.prepare_facet(
                    facet, cfg.off0, axis=0, out=self._bf_f_buffers.get(i), window_lines=True)
                self.launches += 1
                del facet
            self._local_facets = {}
        return self.BF_Fs

    def _column(self, off0):
        cached = self.lru.get(off0)
        if cached is None:
            reuse = None
            if len(self.lru.data) >= self.lru.size:
                _, reuse = self.lru.data.popitem(last=False)
            outs = self.core.extract_columns(
                [self.BF_Fs[i] for i in self.local_idx], off0,
                [self.facet_configs[i].off1 for i in self.local_idx],
                outs=None if reuse is None else [reuse[i] for i in self.local_idx],
                prewindowed=True)
            cached = dict(zip(self.local_idx, outs))
            self.launches += 1
            self.lru.set(off0, cached)
        return cached

    def _buffers(self, slot, xA):
        key = (slot, xA)
        if key not in self._bufs:
            m = self.core.xM_yN_size
            # strips are stored transposed (contribution index contiguous, see api.py)
            shape = (self.world, self.rows_max, xA, m)
            send = torch.zeros(shape, dtype=torch.complex128, device=self.device)
            recv = torch.zeros(shape, dtype=torch.complex128, device=self.device)
            # (logical (world, row, m, xA) views for the kernels, flat storage for the exchange)
            self._bufs[key] = (send.transpose(2, 3), recv.transpose(2, 3), send, recv)
        return self._bufs[key]

    def _mask(self, sg, axis):
        off = sg.off0 if axis == 0 else sg.off1
        key = (axis, off, sg.size)
        if key not in self._masks:
            self._masks[key] = _device_mask(sg.mask0 if axis == 0 else sg.mask1, self.device)
        return self._masks[key]

    def _batch_launch(self, run, ptrs, like):
        """ONE axis-1 launch for the subgrids ``run`` (same subgrid column): groups = subgrid x
        local facet row, group ``(b, row)`` writing to address ``ptrs[b * nrows + row]``.  The
        argument block (sources of all local facets, for a full batch) is built once per
        subgrid column; per launch only offsets, masks and output addresses change."""
        nrows = len(self.my_rows)
        column = self._column(run[0].off0)
        key = (id(column), run[0].size)
        if self._prep1 is None or self._prep1[0] != key:
            rows = [[(column[i], self.facet_configs[i].off1) for i in self.local_idx
                     if self.facet_configs[i].off0 == off0] for off0 in self.my_rows]
            groups = [g for _ in range(self.world) for g in rows]
            m = self.core.xM_yN_size
            # a strip is stored transposed: line (row of the contribution) stride 1, sample stride m
            self._prep1 = (key, self.core.prepare_sum_finish(groups, 1, m, run[0].size, (1, m)),
                           column)
        offs = [sg.off1 for sg in run for _ in range(nrows)]
        masks = [self._mask(sg, 1) for sg in run for _ in range(nrows)]
        self._prep1[1].launch(offs, masks, out_ptrs=ptrs, stream_of=like,
                              n_groups=len(run) * nrows)
        self.launches += 1

    def _runs(self, batch):
        """Maximal runs of consecutive subgrids of a batch that share the subgrid column."""
        b = 0
        while b < len(batch):
            e = b + 1
            while (e < len(batch) and batch[e].off0 == batch[b].off0
                   and batch[e].size == batch[b].size):
                e += 1
            yield b, e
            b = e

    def _local_strips_batch(self, batch, out):
        """Axis-1 reduction for all subgrids of a batch: ``out[b, row]`` for subgrid ``b``."""
        if not self.my_rows:
            return
        nrows = len(self.my_rows)
        key = ("nccl", out.data_ptr())
        if key not in self._ptrs:
            self._ptrs[key] = [[out[b, k].data_ptr() for k in range(nrows)]
                               for b in range(out.shape[0])]
        table = self._ptrs[key]
        for b, e in self._runs(batch):
            ptrs = [p for k in range(b, e) for p in table[k]]
            self._batch_launch(batch[b:e], ptrs, out)

    def _finish(self, sg, recv):
        """Axis-0 reduction over the strips of all ranks (owner only)."""
        out = torch.empty((sg.size, sg.size), dtype=torch.complex128, device=self.device)
        key = (recv.data_ptr(), sg.size)
        if key not in self._prep0:
            sources = [[(recv[r, k], off0) for r in range(self.world)
                        for k, off0 in enumerate(self.rank_rows[r])]]
            self._prep0[key] = self.core.prepare_sum_finish(
                sources, 0, sg.size, sg.size, (out.stride(1), out.stride(0)))
        self._prep0[key].launch([sg.off0], [self._mask(sg, 0)], out=out)
        self.launches += 1
        return out

    # ------------------------------------------------------------------ collective driver
    def get_subgrid_tasks(self, subgrid_configs, consumer=None):
        """Transform all ``subgrid_configs`` (collective call).

        Returns ``{index in subgrid_configs: DeviceTask}`` for the subgrids this rank owns
        (subgrid ``i`` is owned by rank ``i % world_size``).  ``consumer(index, config,
        tensor)``, if given, is called for every owned subgrid instead of keeping it.
        """
        subgrid_configs = list(subgrid_configs)
        self._prepare()
        results = {}
        if not subgrid_configs:
            return results
        sizes = {sg.size for sg in subgrid_configs}
        if len(sizes) != 1:
            raise ValueError("all subgrids of one call must have the same size")
        xA = sizes.pop()
        batches = [subgrid_configs[i:i + self.world]
                   for i in range(0, len(subgrid_configs), self.world)]
        if self.exchange == "p2p":
            return self._run_p2p(batches, xA, consumer, results)
        if self.exchange == "copy":
            return self._run_copy(batches, xA, consumer, results)
        pending = None  # (batch index, work, recv buffer)

        def finish(bi, work, recv):
            if work is not None:
                work.wait()
            batch = batches[bi]
            if self.rank < len(batch):
                idx = bi * self.world + self.rank
                out = self._finish(batch[self.rank], recv)
                if consumer is not None:
                    consumer(idx, batch[self.rank], out)
                else:
                    results[idx] = DeviceTask(out)

        for bi, batch in enumerate(batches):
            send, recv, send_flat, recv_flat = self._buffers(bi % 2, xA)
            self._local_strips_batch(batch, send)
            work = None
            if self.world > 1:
                work = dist.all_to_all_single(
                    torch.view_as_real(recv_flat).view(self.world, -1),
                    torch.view_as_real(send_flat).view(self.world, -1),
                    group=self.group, async_op=True)
            else:
                recv = send
            if pending is not None:
                finish(*pending)
            pending = (bi, work, recv)
        finish(*pending)
        return results

    def _local_strips_batch_p2p(self, batch, views, slot):
        """Axis-1 reduction for all subgrids of a batch, the strips of subgrid ``b`` going
        straight into the receive slot of its owner (rank ``b``) over NVLink: ONE launch per run
        of subgrids that share the subgrid column, every group with its own output buffer."""
        if not self.my_rows:
            return
        nrows = len(self.my_rows)
        key = ("p2p", slot)
        if key not in self._ptrs:
            self._ptrs[key] = [[views[b][slot, self.rank, k].data_ptr() for k in range(nrows)]
                               for b in range(self.world)]
        table = self._ptrs[key]
        for b, e in self._runs(batch):
            ptrs = [p for k in range(b, e) for p in table[k]]
            self._batch_launch(batch[b:e], ptrs, views[self.rank])

    def _run_p2p(self, batches, xA, consumer, results):
        """Peer-memory exchange, software pipelined.

        Per batch ``k`` the stream carries: axis-1 kernel of batch ``k`` (its finished lines
        are scattered into the owners' slots by the TMA engine, over NVLink), ``signal(k)``,
        ``wait(k - 1)``, axis-0 kernel of batch ``k - 1``.  The wait for batch ``k - 1`` thus
        comes one whole axis-1 kernel after the signal: unless a rank lags by more than a batch
        nobody ever blocks, and no SM runs a communication kernel.  A slot is rewritten four
        batches later: by then every owner is known (through ``signal(k - 2)``, which follows
        its axis-0 kernel of batch ``k - 4`` on its stream) to have consumed it.
        """
        _, views, _ = self._symm_slots(xA)
        _, _, table, my_flags, status = self._symm_flags()
        base = self._symm["seq"]
        self._symm["seq"] = base + len(batches)

        def finish(bi):
            self.core.peer_wait(my_flags, self.world, base + bi + 1, status)
            batch = batches[bi]
            if self.rank < len(batch):
                idx = bi * self.world + self.rank
                out = self._finish(batch[self.rank], views[self.rank][bi % self.N_SLOTS])
                if consumer is not None:
                    consumer(idx, batch[self.rank], out)
                else:
                    results[idx] = DeviceTask(out)

        for bi, batch in enumerate(batches):
            self._local_strips_batch_p2p(batch, views, bi % self.N_SLOTS)
            self.core.peer_signal(table, self.world, self.rank, base + bi + 1, my_flags)
            if bi >= 1:
                finish(bi - 1)
        finish(len(batches) - 1)
        bad = int(status.item())
        if bad:
            raise RuntimeError(f"rank {self.rank}: rank {bad - 1} did not deliver its strips "
                               "(peer wait timed out)")
        return results


    def _run_copy(self, batches, xA, consumer, results):
        """Peer-memory exchange by the COPY ENGINES, software pipelined (``exchange="copy"``).

        The axis-1 kernel writes the strips of a batch into a local send buffer; a communication
        stream then moves every owner's part into that owner's receive slot with plain
        device-to-device copies on peer-mapped (symmetric) memory -- NVLink DMA, no SM involved,
        so the transfer really runs beside the kernels (an NCCL all_to_all needs SMs, which the
        persistent one-CTA-per-SM kernels of this library do not leave free: measured on 2 GPUs
        the NCCL exchange serialised with them, 866 ms per step for 625 ms of kernels; scattering
        the strips straight into peer memory with 16-byte TMA rows is slower still, 921 ms) --
        and signals the owners (``peer_signal`` on the communication stream).  Compute stream:
        ``K3(k)``, ``wait(k - 1)``, ``K4(k - 1)``.  Send buffers: two slots, ``K3(k + 2)`` waits
        for the copies of batch ``k``.  Receive slots: four, as in :meth:`_run_p2p`: my
        ``signal(k + 2)`` follows my copies of batch ``k + 2``, hence my ``K3(k + 2)``, hence (same
        stream) my ``K4(k)`` -- so whoever passes ``wait(k + 2)`` may overwrite slot ``k % 4``.
        """
        self._symm_slots(xA)
        bases = self._symm["bases"][xA]   # per rank: (slot, source rank, row, xA, m) storage
        views = self._symm["slots"][xA][1]
        _, _, table, my_flags, status = self._symm_flags()
        base = self._symm["seq"]
        self._symm["seq"] = base + len(batches)
        cuda = self.device.type == "cuda"  # (the host-emulated test build runs everything inline)
        if cuda and self._comm_stream is None:
            self._comm_stream = torch.cuda.Stream(self.device)
        comm = self._comm_stream
        compute = torch.cuda.current_stream(self.device) if cuda else None
        copied = {}

        def finish(bi):
            self.core.peer_wait(my_flags, self.world, base + bi + 1, status)
            batch = batches[bi]
            if self.rank < len(batch):
                idx = bi * self.world + self.rank
                out = self._finish(batch[self.rank], views[self.rank][bi % self.N_SLOTS])
                if consumer is not None:
                    consumer(idx, batch[self.rank], out)
                else:
                    results[idx] = DeviceTask(out)

        def move(bi, batch, send_flat):
            slot = bi % self.N_SLOTS
            for b in range(len(batch)):  # subgrid b of the batch is owned by rank b
                bases[b][slot, self.rank].copy_(send_flat[b], non_blocking=True)
            self.core.peer_signal(table, self.world, self.rank, base + bi + 1, my_flags)

        for bi, batch in enumerate(batches):
            send, _, send_flat, _ = self._buffers(bi % 2, xA)
            if cuda and bi >= 2:
                compute.wait_event(copied.pop(bi - 2))
            self._local_strips_batch(batch, send)
            if cuda:
                ready = torch.cuda.Event()
                ready.record(compute)
                with torch.cuda.stream(comm):
                    comm.wait_event(ready)
                    move(bi, batch, send_flat)
                    done = torch.cuda.Event()
                    done.record(comm)
                copied[bi] = done
            else:
                move(bi, batch, send_flat)
            if bi >= 1:
                finish(bi - 1)
        finish(len(batches) - 1)
        bad = int(status.item())
        if bad:
            raise RuntimeError(f"rank {self.rank}: rank {bad - 1} did not deliver its strips "
                               "(peer wait timed out)")
        if cuda:
            compute.wait_stream(comm)
        return results


class SwiftlyBackwardSharded:
    """Subgrid -> facet accumulation with the facets sharded over a process group.

    Mirror image of :class:`SwiftlyForwardSharded` (SURVEY.md section 8e): every facet
    accumulator lives on the rank that owns the facet (:func:`partition_facets`).  Subgrids are
    processed in batches of ``world_size``; subgrid ``b`` of a batch is supplied by rank ``b``
    (the rank that owns it after the forward transform).  That rank cuts it along axis 0 into
    strips, one ``(m, xA)`` strip per facet row of EVERY rank (the split kernel K4T, written
    straight into a ``(world, rows_max, m, xA)`` send buffer; a facet row split over two ranks
    is cut for both), one ``all_to_all`` per batch moves the strips to the facets' owners, and
    each rank adds the strips of the whole batch to its facets' column accumulators (K3T, one
    launch per run of subgrids of the same subgrid column, in subgrid order).  Per batch a rank
    receives ``world * rows_max * m * xA`` samples -- its own facet rows only -- and the subgrid
    side is computed once per subgrid, not once per rank.  Plans without the split kernel
    replicate every subgrid with one ``all_gather`` per batch instead and run the fused
    backward kernels of :class:`~.api.SwiftlyBackward` on every rank.

    Calls are collective: every rank calls :meth:`add_subgrid_tasks` with the same subgrid
    configs; ``tasks[i]`` must be given on rank ``i % world_size`` (others pass ``None``).
    """

    def __init__(self, swiftly_config, facets_config_list, lru_backward=1, queue_size=20,
                 group=None):
        from .api import SwiftlyBackward  # pylint: disable=import-outside-toplevel

        self.config = swiftly_config
        self.group = group
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.facets_config_list = list(facets_config_list)
        self.owner = partition_facets(self.facets_config_list, self.world)
        self.local_idx = [i for i, o in enumerate(self.owner) if o == self.rank]
        self.device = _device_of(swiftly_config.core)
        self._local = SwiftlyBackward(
            swiftly_config, [self.facets_config_list[i] for i in self.local_idx],
            lru_backward=lru_backward, queue_size=queue_size)
        self.core = swiftly_config.core
        # strip layout as in SwiftlyForwardSharded: per rank the sorted distinct off0 of its facets
        self.rank_rows = []
        for r in range(self.world):
            self.rank_rows.append(sorted({self.facets_config_list[i].off0
                                          for i, o in enumerate(self.owner) if o == r}))
        self.rows_max = max(1, max(len(r) for r in self.rank_rows))
        self.my_rows = self.rank_rows[self.rank]
        self._split = self._local._split
        self._bufs = {}

    def _strip_buffers(self, xA):
        """(send, recv) of shape ``(world, rows_max, m, xA)``; strip ``[r, k]`` is the strip of
        facet row ``rank_rows[r][k]``, C-ordered (the axis-0 lines of K4T are adjacent)."""
        if xA not in self._bufs:
            shape = (self.world, self.rows_max, self.core.xM_yN_size, xA)
            self._bufs[xA] = (torch.zeros(shape, dtype=torch.complex128, device=self.device),
                              torch.zeros(shape, dtype=torch.complex128, device=self.device))
        return self._bufs[xA]

    def _supplied(self, tasks, mine, xA):
        from .api import _resolve, _to_device  # pylint: disable=import-outside-toplevel

        data = tasks[mine]
        if data is None:
            raise ValueError(f"rank {self.rank} must supply subgrid {mine}")
        sub = _to_device(_resolve(data), self.device)
        if tuple(sub.shape) != (xA, xA):
            raise ValueError(f"subgrid {mine} has shape {tuple(sub.shape)}, expected {(xA, xA)}")
        return sub

    def _add_batch_split(self, batch, lo, tasks):
        """One batch on the split kernels: K4T of my subgrid into the send buffer, all_to_all,
        K3T of the received strips into my facets' column accumulators."""
        xA = batch[0].size
        send, recv = self._strip_buffers(xA)
        if self.rank < len(batch):
            sub = self._supplied(tasks, lo + self.rank, xA)
            sg = batch[self.rank]
            targets = [(send[r, k], off0) for r in range(self.world)
                       for k, off0 in enumerate(self.rank_rows[r])]
            self.core.split_subgrid_axis([sub], 0, [sg.off0], [targets], "store")
        if self.world > 1:
            dist.all_to_all_single(torch.view_as_real(recv).view(self.world, -1),
                                   torch.view_as_real(send).view(self.world, -1),
                                   group=self.group)
        else:
            recv = send
        if not self.my_rows:
            return
        b = 0
        while b < len(batch):  # runs of consecutive subgrids of the same subgrid column
            e = b + 1
            while e < len(batch) and batch[e].off0 == batch[b].off0:
                e += 1
            done = self._local.add_strips(batch[b].off0, [
                (recv[s, k], off0, batch[s].off1)
                for s in range(b, e) for k, off0 in enumerate(self.my_rows)])
            self._local.task_queue.process(done)  # queue_size bounds the results in flight
            b = e

    def add_subgrid_tasks(self, subgrid_configs, tasks):
        """Fold ``subgrid_configs`` into the local facets (collective call)."""
        subgrid_configs = list(subgrid_configs)
        tasks = list(tasks)
        if len(tasks) != len(subgrid_configs):
            raise ValueError("one task entry (or None) per subgrid config")
        sizes = {sg.size for sg in subgrid_configs}
        if len(sizes) > 1:
            raise ValueError("all subgrids of one call must have the same size")
        for lo in range(0, len(subgrid_configs), self.world):
            batch = subgrid_configs[lo:lo + self.world]
            if self._split:
                self._add_batch_split(batch, lo, tasks)
                continue
            mine = lo + self.rank
            xA = batch[0].size
            if self.rank < len(batch):
                data = tasks[mine]
                if data is None:
                    raise ValueError(f"rank {self.rank} must supply subgrid {mine}")
                from .api import _resolve, _to_device  # pylint: disable=import-outside-toplevel

                local = _to_device(_resolve(data), self.device).contiguous()
            else:
                local = torch.zeros((xA, xA), dtype=torch.complex128, device=self.device)
            if self.world > 1:
                gathered = torch.empty((self.world, xA, xA), dtype=torch.complex128,
                                       device=self.device)
                dist.all_gather_into_tensor(
                    torch.view_as_real(gathered).reshape(self.world, -1),
                    torch.view_as_real(local).reshape(1, -1), group=self.group)
            else:
                gathered = local[None]
            for b, sg in enumerate(batch):
                self._local.add_new_subgrid_task(sg, gathered[b])

    def finish(self):
        """Finish the local facets; returns ``{facet index: DeviceTask}`` for this rank."""
        tasks = self._local.finish()
        return dict(zip(self.local_idx, tasks))
