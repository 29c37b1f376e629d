"""Collective back-ends of the sharded runtime.

``TorchCollectives`` -- c10d (NCCL on GPU, gloo on CPU).  It is the *baseline/oracle* path
(SURVEY.md §5.8 item 6) and the CPU plumbing path (BASELINE config #1).
``FusedCollectives`` (``fused_comm.py``) -- symmetric-memory peer kernels over NVLink/NVSwitch;
same interface, selected with ``collective_impl=fused``.

Interface (all ops are enqueued on the *current* stream of ``device``):
  alloc_shard / alloc_full     buffers the collectives may need to register (symmetric heap)
  all_gather(shard, full)      full[r*n:(r+1)*n] = shard of shard-rank r
  reduce_scatter(full, shard32, scale, sumsq)  shard32 = scale * sum_ranks(full)[my chunk]  (fp32),
                               then replica all-reduce (HSDP), then sumsq += ||shard32||^2;
                               ``accumulate=True``: shard32 += ... (gradient accumulation), ``replica=False``: the HSDP
                               replica all-reduce is deferred to a later call (micro-steps before the last one)
  all_reduce_full(full, scale, sumsq)  NO_SHARD/DDP gradient path (in place on the full buffer)
"""
from __future__ import annotations

from typing import Optional

import os

import torch
import torch.distributed as dist

from fms_fsdp_b200.ops.functional import kernels_for
from fms_fsdp_b200.parallel.mesh import DPMesh


class TorchCollectives:
    name = "torch"

    def __init__(self, mesh: DPMesh, device: torch.device):
        self.mesh, self.device = mesh, device
        self._scratch = {}

    # ---- allocation
    def alloc_shard(self, numel: int, dtype: torch.dtype) -> torch.Tensor:
        return torch.zeros(numel, dtype=dtype, device=self.device)

    def alloc_full(self, numel: int, dtype: torch.dtype, symmetric: bool = True) -> torch.Tensor:
        if not symmetric:
            # gathered-parameter buffer: first written on the gather stream, so no fill kernel on this stream
            return torch.empty(numel, dtype=dtype, device=self.device)
        return torch.zeros(numel, dtype=dtype, device=self.device)

    def alloc_grad_shard(self, numel: int) -> torch.Tensor:
        return torch.zeros(numel, dtype=torch.float32, device=self.device)

    def begin_step(self):
        pass

    # ---- parameter path
    def all_gather(self, shard: torch.Tensor, full: torch.Tensor):
        if self.mesh.shard_size == 1:
            if full.data_ptr() != shard.data_ptr():
                full.copy_(shard)
            return
        dist.all_gather_into_tensor(full, shard, group=self.mesh.shard_group)

    # ---- gradient path
    def _tmp(self, numel, dtype):
        key = (numel, dtype)
        t = self._scratch.get(key)
        if t is None:
            t = torch.empty(numel, dtype=dtype, device=self.device)
            self._scratch[key] = t
        return t

    def reduce_scatter(self, full: torch.Tensor, shard32: torch.Tensor, scale: float,
                       sumsq: Optional[torch.Tensor], accumulate: bool = False, replica: bool = True):
        m = self.mesh
        tmp = self._tmp(shard32.numel(), full.dtype)
        dist.reduce_scatter_tensor(tmp, full, op=dist.ReduceOp.SUM, group=m.shard_group)
        if accumulate:
            shard32.add_(tmp.float(), alpha=scale)
        else:
            shard32.copy_(tmp)
        if replica and m.replica_size > 1:
            dist.all_reduce(shard32, op=dist.ReduceOp.SUM, group=m.replica_group)
        if not accumulate:
            shard32.mul_(scale)
        if sumsq is not None:
            kernels_for(shard32).sumsq(shard32, out=sumsq)

    def all_reduce_full(self, full: torch.Tensor, scale: float, sumsq: Optional[torch.Tensor]):
        m = self.mesh
        if m.replica_size > 1:
            dist.all_reduce(full, op=dist.ReduceOp.SUM, group=m.replica_group)
            full.mul_(scale)
        if sumsq is not None:
            kernels_for(full).sumsq(full, out=sumsq)

    def all_reduce_scalar(self, t: torch.Tensor, over: str = "shard"):
        m = self.mesh
        if over == "shard":
            if m.shard_size > 1:
                dist.all_reduce(t, group=m.shard_group)
        elif m.world > 1:
            dist.all_reduce(t)
        return t

    def barrier(self):
        if self.mesh.world > 1:
            dist.barrier()


def plan_collectives(impl: str, device_type: str, world: int, shard_size: int, local_world: int, rank: int = 0):
    """-> (implementation of the shard-group collectives, implementation of the replica-group all-reduce).

    The peer-memory kernels need all ranks of a GROUP on one NVSwitch domain (one node).  Ranks are numbered node by node and
    a shard group is ``shard_size`` consecutive ranks, so it sits inside a node iff ``shard_size`` divides ``local_world``:

    * single node                      -> ("fused", "fused")
    * multi-node HSDP, shards in-node  -> ("fused", "nccl"): all-gather inside the GEMMs, wgrad push and the flag protocol stay
      on NVLink; only the replica all-reduce of the fp32 gradient shard (1/shard_size of the model per rank) crosses nodes
      -- the reference's production layout (``docs/train_details.md``: shard within a node, replicate across nodes)
    * multi-node FSDP (shards span nodes) or DDP -> ("torch", "nccl")
    """
    impl = (impl or "auto").lower()
    if device_type != "cuda" or world == 1:
        if impl == "fused" and device_type != "cuda":
            raise ValueError("collective_impl=fused needs CUDA devices")
        return "torch", "nccl"
    local_world = max(1, min(local_world, world))
    multi_node = local_world < world
    shards_in_node = shard_size > 1 and local_world % shard_size == 0
    replica_size = world // shard_size
    if impl == "torch":
        return "torch", "nccl"
    if multi_node:
        if shards_in_node:
            return "fused", "nccl"
        if impl == "fused":
            what = "multi-node ddp has no in-node shard group" if shard_size == 1 else \
                f"shard groups of {shard_size} ranks do not fit inside a node of {local_world} GPUs"
            raise ValueError(f"collective_impl=fused: {what}; use hsdp with hsdp_shard_size dividing {local_world}, "
                             "or collective_impl=torch")
        if rank == 0:
            print(f"[fms_fsdp_b200] {world} ranks over {world // local_world} nodes with shard groups of {shard_size}: "
                  "collective_impl=torch (NCCL); the NVLink peer-memory collectives need each shard group inside one node "
                  "(sharding_strategy=hsdp)")
        return "torch", "nccl"
    if max(shard_size, replica_size) > 32:
        # the signal pads hold 32 ranks per channel (csrc/comm.cu); the reduce kernels themselves take any group size
        if rank == 0:
            print(f"[fms_fsdp_b200] group of {max(shard_size, replica_size)} ranks exceeds the 32-rank signal pad: "
                  "collective_impl=torch (NCCL)")
        return "torch", "nccl"
    return "fused", "fused"


def make_collectives(impl: str, mesh: DPMesh, device: torch.device):
    # FMS_B200_LOCAL_WORLD overrides torchrun's LOCAL_WORLD_SIZE: lets one 8-GPU box pretend to be two 4-GPU nodes so the
    # multi-node composition (fused shard group + NCCL replica all-reduce) can be exercised without a second node
    local_world = int(os.environ.get("FMS_B200_LOCAL_WORLD", os.environ.get("LOCAL_WORLD_SIZE", mesh.world)))
    shard_impl, replica_impl = plan_collectives(impl, device.type, mesh.world, mesh.shard_size, local_world, mesh.rank)
    if shard_impl == "fused":
        from fms_fsdp_b200.parallel.fused_comm import FusedCollectives
        return FusedCollectives(mesh, device, replica_impl=replica_impl)
    return TorchCollectives(mesh, device)
