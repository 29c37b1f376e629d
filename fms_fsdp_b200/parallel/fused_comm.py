"""NVLink / NVSwitch collectives of the sharded runtime: our own peer-memory kernels, no NCCL on the
parameter / gradient paths (SURVEY.md §5.8).

* buffers that peers must reach (compute-dtype parameter shards, unsharded gradient buffers, HSDP gradient
  shards) are allocated from torch symmetric memory and rendezvoused once; we keep, per buffer, a device
  table of the W peer addresses;
* ``all_gather``      = pull kernel (``csrc/comm.cu::p2p_allgather_kernel``): every rank copies the 7 remote
  shards with 16-byte peer loads, rotated start so all inbound NVLink flows are busy;
* gradients of LLaMA-style blocks never exist unsharded: the wgrad GEMM epilogue PUSHES each tile into the owning
  rank's staging slot ``[src rank][shard]`` (``csrc/gemm_sm90.cu`` ``EPI_PUSH``); after ONE cross-rank flag round
  per unit the owner sums its ``world`` local slots in fp32, scales by 1/world, writes the fp32 shard and accumulates
  ||g||^2 in the same pass (``reduce_pushed``; K11 folded into N8) -- no NVLink traffic outside the GEMMs;
* ``reduce_scatter``  = one-shot pull-reduce for everything else (root unit, Mamba blocks): rank r sums slice r of all
  W gradient buffers;
* HSDP replica all-reduce / DDP all-reduce = two-phase (reduce own slice in place, barrier, gather slices);
* ordering = signal-pad flags (``st.release.sys`` / ``ld.acquire.sys``) enqueued on the same streams; the pad has
  32-slot channels so flag rounds of different streams never see each other's epochs;
* the grad-norm scalar = a one-shot all-reduce kernel over the same pads (``scalar_allreduce``).

Only checkpoint metadata and the report-interval statistics still travel through c10d.
"""
from __future__ import annotations

import os

from typing import Dict, Optional, Tuple

import torch
import torch.distributed as dist

from fms_fsdp_b200.ops import _ext
from fms_fsdp_b200.ops.functional import kernels_for
from fms_fsdp_b200.parallel.mesh import DPMesh


class _SymGroup:
    """Symmetric allocations + barrier state for one process group."""

    # signal-pad channels (32 slots each): 0 = step / stream-ordered barriers on the compute or gather stream,
    # 1 = reduce stream, 2 = replica all-reduce, UNIT_CH0 + i = "optimizer updated unit i" flags
    N_CHANNELS = 512
    CH_STEP, CH_REDUCE, CH_AUX, UNIT_CH0 = 0, 1, 2, 8

    def __init__(self, group, size: int, my_index: int, device: torch.device):
        import torch.distributed._symmetric_memory as symm_mem
        self.symm_mem = symm_mem
        self.group, self.size, self.index, self.device = group, size, my_index, device
        self.tables: Dict[int, Tuple[torch.Tensor, list]] = {}  # data_ptr -> (device ptr table, host ptr list)
        self.regions = []  # (base address, bytes, peer base addresses)
        self._keep = []
        self.epochs: Dict[int, int] = {}
        pad = self.alloc(32 * self.N_CHANNELS, torch.int32)
        pad.zero_()
        self.pad_table = self.tables[pad.data_ptr()][0]
        self._sar_buf = self.alloc(1024, torch.int32)   # scalar all-reduce slots (csrc/comm.cu: 2304 bytes)
        self._sar_buf.zero_()
        self._sar_epoch = 0
        torch.cuda.synchronize(device)
        dist.barrier(group=group)

    def alloc(self, numel: int, dtype: torch.dtype) -> torch.Tensor:
        t = self.symm_mem.empty(numel, dtype=dtype, device=self.device)
        hdl = self.symm_mem.rendezvous(t, self.group)
        ptrs = [int(p) for p in hdl.buffer_ptrs]
        table = torch.tensor(ptrs, dtype=torch.int64, device=self.device)
        self.tables[t.data_ptr()] = (table, ptrs)
        self.regions.append((t.data_ptr(), t.numel() * t.element_size(), ptrs))
        self._keep.append((t, hdl))
        return t

    def table_of(self, t: torch.Tensor, byte_offset_per_peer=None) -> torch.Tensor:
        """Device table of the W peer addresses of ``t`` (a registered buffer or a view into one; a view sits
        at the same byte offset on every peer).  ``byte_offset_per_peer(i)`` adds a per-peer displacement."""
        key = t.data_ptr()
        if byte_offset_per_peer is None and key in self.tables:
            return self.tables[key][0]
        for base, nbytes, ptrs in self.regions:
            if base <= key < base + nbytes:
                off = key - base
                break
        else:
            raise RuntimeError("tensor is not in the symmetric heap")
        if byte_offset_per_peer is None:
            host = [p + off for p in ptrs]
            tab = torch.tensor(host, dtype=torch.int64, device=self.device)
            self.tables[key] = (tab, host)
            return tab
        return torch.tensor([p + off + byte_offset_per_peer(i) for i, p in enumerate(ptrs)], dtype=torch.int64,
                            device=self.device)

    def barrier(self, C, anchor: torch.Tensor, channel: int = 0):
        """All ranks of the group have reached this point of the current stream (flag round on ``channel``)."""
        e = self.epochs.get(channel, 0) + 1
        self.epochs[channel] = e
        C.signal_barrier(self.pad_table, self.size, self.index, e, anchor, 32 * channel, 0)

    def post(self, C, anchor: torch.Tensor, channel: int, epoch: int):
        """One-sided: everything this rank enqueued before is visible to whoever ``wait``s for (channel, epoch)."""
        C.signal_barrier(self.pad_table, self.size, self.index, int(epoch), anchor, 32 * channel, 1)

    def wait(self, C, anchor: torch.Tensor, channel: int, epoch: int):
        C.signal_barrier(self.pad_table, self.size, self.index, int(epoch), anchor, 32 * channel, 2)

    def scalar_allreduce(self, C, t: torch.Tensor):
        """In-place sum of up to 8 fp32 scalars over the group: one tiny kernel, identical result on every rank."""
        assert int(C.scalar_allreduce_bytes()) <= self._sar_buf.numel() * 4
        self._sar_epoch += 1
        C.scalar_allreduce(self.tables[self._sar_buf.data_ptr()][0], self.size, self.index, self._sar_epoch, t)


class FusedCollectives:
    name = "fused"

    def __init__(self, mesh: DPMesh, device: torch.device, replica_impl: str = "fused"):
        self.mesh, self.device = mesh, device
        self.C = _ext.require()
        self.shard = _SymGroup(mesh.shard_group, mesh.shard_size, mesh.shard_rank, device) if mesh.shard_size > 1 else None
        # replica_impl="nccl": the replica group crosses nodes (multi-node HSDP, ``comm.plan_collectives``) -- its all-reduce of
        # the fp32 gradient shard goes through c10d/NCCL on the reduce stream, everything inside the node stays on NVLink
        self.replica = _SymGroup(mesh.replica_group, mesh.replica_size, mesh.replica_rank, device) \
            if (mesh.replica_size > 1 and replica_impl == "fused") else None
        self._replica_nccl = mesh.replica_group if (mesh.replica_size > 1 and replica_impl != "fused") else None
        self._anchor = torch.zeros(1, device=device)
        self._slice_tables: Dict[Tuple[int, int], torch.Tensor] = {}
        self._ag_state: Dict[int, list] = {}
        # CTA cap of the reduce kernels (csrc/comm.cu): by default two CTAs per SM of this GPU
        sms = torch.cuda.get_device_properties(device).multi_processor_count
        self.C.set_reduce_ctas(int(os.environ.get("FMS_B200_REDUCE_CTAS", str(2 * sms))))
        self._own_scalar = os.environ.get("FMS_B200_OWN_SCALAR_ALLREDUCE", "1") == "1"
        # CTA cap of the local slot sum (runs under the backward GEMMs; 0 = same as the pull kernels)
        self._slotsum_ctas = int(os.environ.get("FMS_B200_SLOTSUM_CTAS", "0"))
        self.last_reduce_done = None

    # ---- allocation ---------------------------------------------------------------------------
    def alloc_shard(self, numel: int, dtype: torch.dtype) -> torch.Tensor:
        if self.shard is None:
            return torch.zeros(numel, dtype=dtype, device=self.device)
        t = self.shard.alloc(numel, dtype)
        t.zero_()
        return t

    def alloc_full(self, numel: int, dtype: torch.dtype, symmetric: bool = True) -> torch.Tensor:
        """Unsharded gradient buffers must be peer-visible; gathered-parameter buffers are local."""
        if not symmetric:
            # NOT zero-filled: the fill would run on the caller's (compute) stream and race with the first
            # gather that writes this buffer on the gather stream
            return torch.empty(numel, dtype=dtype, device=self.device)
        g = self.shard if self.shard is not None else self.replica
        if g is None:
            return torch.zeros(numel, dtype=dtype, device=self.device)
        t = g.alloc(numel, dtype)
        t.zero_()
        return t

    def alloc_grad_shard(self, numel: int) -> torch.Tensor:
        if self.replica is not None and self.shard is not None:  # hsdp: replicas all-reduce the fp32 shard
            t = self.replica.alloc(numel, torch.float32)
            t.zero_()
            return t
        return torch.zeros(numel, dtype=torch.float32, device=self.device)

    # ---- parameter path -----------------------------------------------------------------------
    def begin_step(self):
        """All ranks' optimizer updates are visible before anyone gathers (enqueue on the gather stream)."""
        if self.shard is not None:
            self.shard.barrier(self.C, self._anchor, _SymGroup.CH_STEP)

    # per-unit optimizer flags (asynchronous sharded AdamW): rank r posts (unit, step) after updating its shard of the
    # unit; a gather of that unit waits until every shard rank has posted
    def post_unit_updated(self, unit_index: int, step: int):
        if self.shard is not None:
            self.shard.post(self.C, self._anchor, _SymGroup.UNIT_CH0 + unit_index, step)

    def wait_unit_updated(self, unit_index: int, step: int):
        if self.shard is not None:
            self.shard.wait(self.C, self._anchor, _SymGroup.UNIT_CH0 + unit_index, step)

    @property
    def max_units(self) -> int:
        return _SymGroup.N_CHANNELS - _SymGroup.UNIT_CH0

    def all_gather(self, shard: torch.Tensor, full: torch.Tensor):
        if self.shard is None:
            if full.data_ptr() != shard.data_ptr():
                full.copy_(shard)
            return
        g = self.shard
        self.C.p2p_allgather(g.table_of(shard), full, shard.numel() * shard.element_size(), g.size, g.index)

    # ---- fused gather (ag_gemm) ----------------------------------------------------------------
    AG_CHUNK = 65536

    def gather_range(self, shard: torch.Tensor, full: torch.Tensor, begin_bytes: int, end_bytes: int):
        g = self.shard
        self.C.p2p_gather_range(g.table_of(shard), full, shard.numel() * shard.element_size(), begin_bytes, end_bytes)

    def ag_request(self, shard: torch.Tensor, full: torch.Tensor, begin_bytes: int, end_bytes: int, dependent: bool):
        """Descriptor of 'gather bytes [begin, end) of this unit into `full`' for a GEMM to carry."""
        g = self.shard
        key = full.data_ptr()
        st = self._ag_state.get(key)
        total = full.numel() * full.element_size()
        if st is None:
            n_chunks = (total + self.AG_CHUNK - 1) // self.AG_CHUNK
            st = [torch.zeros(n_chunks, dtype=torch.int32, device=self.device), 0]
            self._ag_state[key] = st
        st[1] += 1
        return dict(table=g.table_of(shard), full=full, shard_bytes=shard.numel() * shard.element_size(),
                    begin=int(begin_bytes), end=int(end_bytes), world=g.size, rank=g.index, flags=st[0], epoch=st[1],
                    dependent=bool(dependent))

    # ---- gradient path ------------------------------------------------------------------------
    def reduce_scatter(self, full: torch.Tensor, shard32: torch.Tensor, scale: float, sumsq: Optional[torch.Tensor],
                       on_barrier=None, accumulate: bool = False, replica: bool = True):
        """``accumulate``: add into ``shard32`` instead of overwriting it; ``replica=False``: skip the HSDP replica
        all-reduce (gradient accumulation runs it once, on the last micro-step)."""
        g = self.shard
        g.barrier(self.C, self._anchor, _SymGroup.CH_REDUCE)  # every rank's wgrads for this unit are complete
        if on_barrier is not None:
            on_barrier()
        hsdp = self.replica is not None or self._replica_nccl is not None
        self.C.reduce_scatter(g.table_of(full), shard32, g.index * shard32.numel(), g.size, g.index,
                              full.dtype == torch.bfloat16, float(scale), None if hsdp else sumsq, 0, accumulate)
        if not hsdp:
            # results of this unit are final here; consumers need not wait for the trailing flag round
            self.last_reduce_done = torch.cuda.Event()
            self.last_reduce_done.record(torch.cuda.current_stream(self.device))
        g.barrier(self.C, self._anchor, _SymGroup.CH_REDUCE)  # peers are done reading my buffer before it is rewritten
        if hsdp:
            if replica:
                self._replica_allreduce(shard32, sumsq)
            self.last_reduce_done = None

    # ---- fused wgrad GEMM -> reduce-scatter (push) ----------------------------------------------------------------
    def push_table(self, staging: torch.Tensor) -> torch.Tensor:
        """Addresses of every shard-rank's copy of ``staging`` (layout [src_rank][shard elements])."""
        return self.shard.table_of(staging)

    def push_vectors(self, vec: torch.Tensor, staging: torch.Tensor):
        """The non-GEMM gradients of a unit (norm gains: flat elements [0, vec.numel())) -> the owners' slots."""
        g = self.shard
        self.C.push_range(vec, g.table_of(staging), staging.numel() // g.size, 0, g.index)

    def reduce_pushed(self, staging: torch.Tensor, shard32: torch.Tensor, scale: float, sumsq: Optional[torch.Tensor],
                      on_barrier=None, accumulate: bool = False, replica: bool = True):
        """After every rank pushed its wgrad tiles: ONE flag round (all tiles of all ranks have landed in my slots),
        then a LOCAL sum of the ``world`` slots.  There is no trailing barrier: a staging buffer is handed out again
        only after a LATER flag round on this stream has completed (``on_barrier`` lets the engine record that), which
        implies every rank has finished summing it.  ``accumulate`` / ``replica``: as in ``reduce_scatter``."""
        g = self.shard
        n = shard32.numel()
        g.barrier(self.C, self._anchor, _SymGroup.CH_REDUCE)
        if on_barrier is not None:
            on_barrier()
        key = ("slots", staging.data_ptr())
        tab = self._slice_tables.get(key)
        if tab is None:
            tab = torch.tensor([staging.data_ptr() + s_ * n * staging.element_size() for s_ in range(g.size)],
                               dtype=torch.int64, device=self.device)
            self._slice_tables[key] = tab
        hsdp = self.replica is not None or self._replica_nccl is not None
        self.C.reduce_scatter(tab, shard32, 0, g.size, 0, staging.dtype == torch.bfloat16, float(scale),
                              None if hsdp else sumsq, self._slotsum_ctas, accumulate)
        self.last_reduce_done = None
        if hsdp and replica:
            self._replica_allreduce(shard32, sumsq)

    def _replica_allreduce(self, shard32: torch.Tensor, sumsq: Optional[torch.Tensor]):
        """HSDP: sum the (already scaled) fp32 gradient shard over the replicas, then its squared norm."""
        if self.replica is not None:
            self._allreduce(self.replica, shard32, 1.0, sumsq)
            return
        # c10d orders the NCCL kernel after the work already enqueued on the current (reduce) stream and makes that stream
        # wait for it, so the sumsq kernel and the optimizer see the reduced shard
        dist.all_reduce(shard32, op=dist.ReduceOp.SUM, group=self._replica_nccl)
        if sumsq is not None:
            kernels_for(shard32).sumsq(shard32, out=sumsq)

    def all_reduce_full(self, full: torch.Tensor, scale: float, sumsq: Optional[torch.Tensor]):
        if self.replica is None:
            assert self._replica_nccl is None, "multi-node DDP takes TorchCollectives (comm.plan_collectives)"
            if sumsq is not None:
                kernels_for(full).sumsq(full, out=sumsq)
            return
        self._allreduce(self.replica, full, scale, sumsq)

    def _allreduce(self, g: _SymGroup, buf: torch.Tensor, scale: float, sumsq: Optional[torch.Tensor]):
        n = buf.numel()
        is_bf16 = buf.dtype == torch.bfloat16
        unit = g.size * (8 if is_bf16 else 4)
        if n % unit:
            raise RuntimeError(f"all-reduce buffer of {n} elements is not a multiple of {unit}")
        es = buf.element_size()
        slice_bytes = n // g.size * es
        ch = _SymGroup.CH_AUX
        g.barrier(self.C, self._anchor, ch)
        self.C.allreduce_inplace(g.table_of(buf), n, g.size, g.index, is_bf16, float(scale), None, self._anchor)
        g.barrier(self.C, self._anchor, ch)
        key = (buf.data_ptr(), g.size)
        tab = self._slice_tables.get(key)
        if tab is None:
            tab = g.table_of(buf, byte_offset_per_peer=lambda i: i * slice_bytes)
            self._slice_tables[key] = tab
        self.C.p2p_allgather(tab, buf, slice_bytes, g.size, g.index)
        g.barrier(self.C, self._anchor, ch)
        if sumsq is not None:
            kernels_for(buf).sumsq(buf, out=sumsq)

    def all_reduce_scalar(self, t: torch.Tensor, over: str = "shard"):
        """Sum of one fp32 scalar (the squared grad-norm) over the shard group -- one-shot kernel over the signal pads
        instead of an NCCL ring (SURVEY.md N11; measured 3.7 ms of launch + ring latency per step at 8 GPUs)."""
        m = self.mesh
        if over == "shard":
            if m.shard_size > 1:
                if self._own_scalar and t.dtype == torch.float32 and t.is_contiguous():
                    self.shard.scalar_allreduce(self.C, t.view(-1))
                else:
                    dist.all_reduce(t, group=m.shard_group)
        elif m.world > 1:
            dist.all_reduce(t)
        return t

    def barrier(self):
        if self.mesh.world > 1:
            dist.barrier()
