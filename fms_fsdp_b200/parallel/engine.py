"""The sharded-parameter runtime (the engine that replaces torch FSDP1 for this framework).

What the reference delegates to ``FullyShardedDataParallel`` (SURVEY.md §2.4 E1, §3.2) and what
this file owns instead:

  * one flat buffer per *unit* (block / root), cut 1-D across the shard group; every rank keeps a
    fp32 master shard, AdamW moments, and a compute-dtype shard that is what travels over NVLink;
  * an explicit schedule instead of module hooks: forward walks the units with ``prefetch_depth``
    parameter gathers in flight on a side stream; backward walks them in reverse, re-gathers
    (prefetching the next unit) and launches each unit's gradient reduce-scatter on a third
    stream as soon as that unit's backward has been enqueued;
  * unit boundaries are autograd boundaries (inputs are detached leaves), so a unit's backward is
    one ``autograd.backward`` call the scheduler issues -- which is also where selective
    recomputation happens (re-run the unit forward with the weights already gathered);
  * weight gradients are written by the ops straight into the unit's flat gradient buffer; the
    reduce-scatter scales by 1/world, emits fp32 shards and accumulates the squared gradient norm,
    so ``clip_grad_norm_`` costs one scalar all-reduce and the clip factor is applied inside the
    fused AdamW (K11/K12 of SURVEY.md §2.5).

Sharding strategies (reference ``train_utils.py:227-234``): fsdp / hsdp / ddp via ``DPMesh``.
Collectives are pluggable (``comm.py``): c10d baseline or fused NVLink peer kernels.
"""
from __future__ import annotations

import hashlib
import os

import contextlib
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist
import torch.nn as nn

from fms_fsdp_b200.parallel.comm import make_collectives
from fms_fsdp_b200.parallel.layout import UnitLayout, build_layout
from fms_fsdp_b200.parallel.mesh import DPMesh, build_mesh
from fms_fsdp_b200.policies.ac_handler import is_checkpointed
from fms_fsdp_b200.policies.mixed_precision import MixedPrecision, fp32_policy


class _NullEvent:
    def record(self, stream=None):
        pass

    def wait(self, stream=None):
        pass

    def synchronize(self):
        pass


class _Buf:
    """A pooled flat buffer plus the event after which it may be overwritten."""

    def __init__(self, tensor, event):
        self.t = tensor
        self.free_event = event


class ShardUnit:
    def __init__(self, name: str, modules: Sequence[nn.Module], params: List[Tuple[str, nn.Parameter]],
                 layout: UnitLayout):
        self.name, self.modules, self.params, self.layout = name, list(modules), params, layout
        self.master = self.lowp = self.exp_avg = self.exp_avg_sq = self.grad_shard = None
        self.full: Optional[_Buf] = None        # gathered parameters
        self.full_grad: Optional[_Buf] = None   # unsharded gradient buffer
        self.ev_gathered = _NullEvent()
        self.recompute = False
        self.gather_pending = False

    def bind_params(self, flat: torch.Tensor):
        for (_, p), s in zip(self.params, self.layout.slots):
            p.data = flat[s.offset:s.offset + s.numel].view(s.shape)

    def unbind_params(self, placeholder: torch.Tensor):
        for _, p in self.params:
            p.data = placeholder

    def bind_grads(self, flat: torch.Tensor, accumulate: bool = False):
        """``accumulate``: the buffer already holds earlier micro-steps' gradients -- every producer adds to it."""
        for (_, p), s in zip(self.params, self.layout.slots):
            p._grad_buf = flat[s.offset:s.offset + s.numel].view(s.shape)
            p._grad_ready = accumulate
            p.grad = None

    def bind_grads_push(self, vec: torch.Tensor, make_target):
        """EXPERIMENTAL push path: 1-D parameters write into the local vector buffer ``vec`` (flat elements
        [0, matrix_begin)), weight matrices get a push target instead of a buffer view."""
        for (_, p), s in zip(self.params, self.layout.slots):
            p._grad_ready = False
            p.grad = None
            if len(s.shape) == 1:
                p._grad_buf, p._grad_push = vec[s.offset:s.offset + s.numel].view(s.shape), None
            else:
                p._grad_buf, p._grad_push = None, make_target(s)

    def collect_grads(self):
        """Fold autograd-produced .grad (ops that did not write into the buffer) and zero the slots
        of parameters that received no gradient at all."""
        for pname, p in self.params:
            if getattr(p, "_grad_push", None) is not None:
                if p.grad is not None or not p._grad_ready:
                    raise RuntimeError(f"push reduce-scatter ({self.name}): weight {pname} {tuple(p.shape)} must receive exactly "
                                       f"one wgrad GEMM (autograd .grad present: {p.grad is not None}, wgrad delivered: "
                                       f"{bool(p._grad_ready)}); set engine_push_wgrad = False on the block to use the pull path")
                continue
            buf = p._grad_buf
            if p.grad is not None:
                if p._grad_ready:
                    buf.copy_(buf + p.grad.view_as(buf))     # in the wider dtype, rounded once
                else:
                    buf.copy_(p.grad.view_as(buf))
                p._grad_ready = True
                p.grad = None
            elif not p._grad_ready:
                buf.zero_()

    def unbind_grads(self):
        for _, p in self.params:
            p._grad_buf = None
            p._grad_push = None
            p._grad_ready = False


class ShardedModel(nn.Module):
    """Wrap a model exposing the engine protocol (``engine_units/engine_embed/engine_head``)."""

    def __init__(self, model: nn.Module, *, sharding_strategy: str = "fsdp", hsdp_shard_size: int = 0,
                 mixed_precision: Optional[MixedPrecision] = None, device: Optional[torch.device] = None,
                 collective_impl: str = "auto", prefetch_depth: int = 2, param_init_fn=None,
                 mesh: Optional[DPMesh] = None, local_world: Optional[int] = None,
                 reshard_after_forward: bool = True, sync_module_states: bool = False, auto_wrap_policy=None,
                 grad_accum_steps: int = 1):
        """``grad_accum_steps``: micro-steps (``forward_backward`` / ``forward_backward_custom`` / ``model(x)`` then
        ``.backward()``) per optimizer step.  Their gradients are summed in fp32 and the optimizer sees the gradient of the
        MEAN micro-batch loss: ``clip_grad_norm_`` reports ``sqrt(sum ||g||^2) / k`` and AdamW scales by ``clip / k``.
        Sharded meshes reduce-scatter every micro-step into the fp32 shard (the HSDP replica all-reduce runs once, on the
        last one); unsharded meshes (1 GPU, ddp) accumulate locally in an fp32 gradient buffer and communicate once.

        ``sync_module_states``: broadcast global rank 0's initial parameters to every rank before sharding (torch
        FSDP's flag of the same name; the reference sets it for the speculator, ``train_speculator.py:205``).

        ``auto_wrap_policy``: predicate over the model's chain of blocks (``policies.get_wrapper(block_cls)``, the
        reference's ``wrapping.py:6-14`` contract): a block for which it is true becomes a shard unit of its own (gathered
        just in time, released after use); a block for which it is false stays in the ROOT unit next to embedding / head
        / final norm -- resident for the whole step, reduced with the root.  ``None`` = every block is a unit."""
        super().__init__()
        if int(grad_accum_steps) != grad_accum_steps or grad_accum_steps < 1:
            raise ValueError(f"grad_accum_steps must be an integer >= 1, got {grad_accum_steps!r}")
        self.grad_accum_steps = int(grad_accum_steps)
        self._micro = 0                 # micro-steps run since the last optimizer step
        self.module = model
        self._sync_module_states = bool(sync_module_states)
        self.device = torch.device(device) if device is not None else (
            torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu"))
        self.is_cuda = self.device.type == "cuda"
        self.mp = mixed_precision or fp32_policy
        self.mesh = mesh or build_mesh(sharding_strategy, hsdp_shard_size, local_world)
        self.sharding_strategy = sharding_strategy
        self.coll = make_collectives(collective_impl, self.mesh, self.device)
        self.prefetch_depth = max(1, int(prefetch_depth))
        self.reshard_after_forward = reshard_after_forward and self.mesh.shard_size > 1
        self._needs_reduce = self.mesh.world > 1
        import os as _os
        # fused all-gather: unit gathers ride inside GEMM kernels on the compute stream (fused collectives only)
        self._fuse_gather = (self.coll.name == "fused" and self.mesh.shard_size > 1
                             and _os.environ.get("FMS_B200_FUSED_GATHER", "1") == "1")
        self._placeholder = torch.empty(0, dtype=self.mp.param_dtype, device=self.device)

        if self.is_cuda:
            self.s_compute = torch.cuda.current_stream(self.device)
            self.s_gather = torch.cuda.Stream(self.device)
            self.s_reduce = torch.cuda.Stream(self.device)
            self.s_opt = torch.cuda.Stream(self.device)
        else:
            self.s_compute = self.s_gather = self.s_reduce = self.s_opt = None
        # asynchronous optimizer: the (bandwidth-bound) AdamW of step t runs on ``s_opt`` under the forward GEMMs of step
        # t+1; each unit's forward / gather waits only for that unit's own update.  Sharded runs additionally need every
        # PEER's shard of the unit to be updated before it is gathered: per-unit cross-rank flags on the signal pads
        # (fused collectives) replace the step barrier.
        self.async_optimizer = (self.is_cuda and os.environ.get("FMS_B200_ASYNC_OPT", "1") == "1"
                                and (self.mesh.shard_size == 1
                                     or (self.coll.name == "fused" and os.environ.get("FMS_B200_ASYNC_OPT_SHARDED", "1") == "1")))
        self._async_sharded = self.async_optimizer and self.mesh.shard_size > 1
        self._opt_epoch = 0            # number of optimizer steps whose per-unit flags have been posted
        self._nvtx_on = os.environ.get("FMS_B200_NVTX", "0") == "1"

        blocks, root_modules = model.engine_units()
        wrapped = [True if auto_wrap_policy is None else bool(auto_wrap_policy(b)) for b in blocks]
        self.blocks: List[ShardUnit] = []
        if self.mesh.world > 1:
            self._validate_same_everywhere("number of shard units", sum(wrapped) + 1)
        resident = [b for b, w in zip(blocks, wrapped) if not w]
        self.root = self._make_unit("root", list(root_modules) + resident, param_init_fn, prefix_of=model)
        # the forward chain: (block module, its own unit | None when its parameters live in the root unit)
        self._chain: List[Tuple[nn.Module, Optional[ShardUnit]]] = []
        for i, (blk, w) in enumerate(zip(blocks, wrapped)):
            u = None
            if w:
                u = self._make_unit(f"block{i}", [blk], param_init_fn, prefix_of=model)
                u.chain_pos = len(self._chain)
                self.blocks.append(u)
            self._chain.append((blk, u))
        for idx, u in enumerate(self.units):
            u.index = idx
        if self._async_sharded and len(self.units) > self.coll.max_units:
            self.async_optimizer = self._async_sharded = False   # more units than flag channels: keep the step barrier
        # anything not covered by a unit is a bug in the model's protocol
        covered = {id(p) for u in self.units for _, p in u.params}
        missing = [n for n, p in model.named_parameters() if id(p) not in covered]
        if missing:
            raise RuntimeError(f"parameters outside every shard unit: {missing[:5]}")
        for buf_name, b in list(model.named_buffers()):
            if b.is_meta:
                raise RuntimeError(f"buffer {buf_name} still on meta device")
        self._move_buffers()

        # pools
        self._full_pool: Dict[Tuple, List[_Buf]] = {}
        self._grad_pool: Dict[Tuple, List[_Buf]] = {}
        self._pool_made: Dict[Tuple, int] = {}
        self._bwd_gather_split = float(os.environ.get("FMS_B200_AG_SPLIT_BWD", "1.0"))
        # backward knobs: gradient-buffer pool depth (1 = the block's backward waits for
        # the previous unit's reduce, 2 = they overlap) and whether backward re-gathers ride inside the GEMMs
        self._grad_pool_depth = int(os.environ.get("FMS_B200_GRAD_POOL", "1"))
        self.poison_released_params = os.environ.get("FMS_B200_POISON", "0") == "1"
        # fused wgrad GEMM -> reduce-scatter (SURVEY.md N8): wgrad epilogues push their tiles straight into the owning
        # rank's staging slots over NVLink; after one flag round per unit the owner sums `world` local slots.  Staging
        # buffers rotate through a pool of ``_push_pool_depth`` (>= 2): buffer X of unit j may be pushed into again once
        # the flag round of unit j+1 has completed on the reduce stream (=> every rank has summed X).
        self._push_rs = (os.environ.get("FMS_B200_PUSH_RS", "1") == "1" and self.coll.name == "fused"
                         and self.mesh.shard_size > 1 and self.mp.reduce_dtype == torch.bfloat16)
        self._push_pool_depth = max(2, int(os.environ.get("FMS_B200_PUSH_POOL", "3")))
        self._push_pool: Dict[Tuple, List[_Buf]] = {}
        self._push_pending: Optional[_Buf] = None     # summed locally, waiting for the next flag round to become reusable
        self._fuse_gather_bwd = os.environ.get("FMS_B200_FUSED_GATHER_BWD", "1") != "0"
        if self._push_rs:
            self._warm_push_pool()
        self._gnorm_sq = torch.zeros((), dtype=torch.float32, device=self.device)
        self._clip_coef: Optional[torch.Tensor] = None
        # AdamW's gradient multiplier when the step was not clipped (k > 1); persistent for the asynchronous optimizer
        self._inv_accum = (torch.full((), 1.0 / self.grad_accum_steps, dtype=torch.float32, device=self.device)
                           if self.grad_accum_steps > 1 else None)
        self._saved = None
        self.step_count = 0
        self.last_grad_norm: Optional[torch.Tensor] = None

    # ------------------------------------------------------------------------------ construction
    @property
    def units(self) -> List[ShardUnit]:
        return [self.root] + self.blocks

    def _event(self):
        return torch.cuda.Event() if self.is_cuda else _NullEvent()

    def _move_buffers(self):
        for m in self.module.modules():
            for k, b in list(m._buffers.items()):
                if b is not None and b.device != self.device:
                    m._buffers[k] = b.to(self.device)

    def _validate_layout(self, name: str, layout: UnitLayout):
        """Every rank must shard the same unit the same way (cf. torch FSDP's exec-order validation, SURVEY.md N12):
        a model that differs across ranks would otherwise deadlock or silently mix shards.  One small object
        all-gather per unit at construction; on by default, ``FMS_B200_VALIDATE=0`` skips it."""
        if os.environ.get("FMS_B200_VALIDATE", "1") == "0":
            return
        mine = (name, layout.total, tuple((s.name, tuple(s.shape), s.offset) for s in layout.slots))
        self._validate_same_everywhere(f"shard unit '{name}' (parameter names / shapes / order)", mine)

    def _validate_same_everywhere(self, what: str, value):
        if os.environ.get("FMS_B200_VALIDATE", "1") == "0":
            return
        digest = int.from_bytes(hashlib.sha1(repr(value).encode()).digest()[:6], "big")   # same on every rank
        try:
            t = torch.tensor([digest], dtype=torch.int64, device=self.device)
            lo, hi = t.clone(), t.clone()
            dist.all_reduce(lo, op=dist.ReduceOp.MIN)
            dist.all_reduce(hi, op=dist.ReduceOp.MAX)
            lo, hi = int(lo), int(hi)
        except Exception as ex:   # a debugging aid must never take a healthy job down
            if self.mesh.rank == 0:
                print(f"[fms_fsdp_b200] cross-rank validation of {what} skipped: {ex!r}")
            return
        if lo != hi:
            raise RuntimeError(f"{what} differs across ranks (rank {self.mesh.rank}: {str(value)[:200]})")

    def _make_unit(self, name, modules, param_init_fn, prefix_of) -> ShardUnit:
        # materialise (meta -> device) one unit at a time: allocate the whole unit, then run the init
        # functions children-first so a parent's reset_parameters has the last word on its children
        for m in modules:
            if any(p.is_meta for p in m.parameters()) or any(b.is_meta for b in m.buffers()):
                m.to_empty(device=self.device)
                init = param_init_fn
                if init is None:
                    from fms_fsdp_b200.policies.param_init import param_init_function as init
                for sub in reversed(list(m.modules())):
                    try:
                        init(sub, self.device)
                    except TypeError:
                        init(sub)
        fqn = {id(p): n for n, p in prefix_of.named_parameters()}
        seen, params = set(), []
        for m in modules:
            for p in m.parameters():
                if id(p) not in seen:
                    seen.add(id(p))
                    params.append((fqn[id(p)], p))
        params.sort(key=lambda np_: np_[1].dim() > 1)  # stable: vectors (norm gains, biases) first, matrices after
        layout = build_layout(name, [(n, tuple(p.shape)) for n, p in params], self.mesh.shard_size)
        if self.mesh.world > 1:
            self._validate_layout(name, layout)
            if self._sync_module_states:
                for _, p in params:   # rank 0's initial values win everywhere (before the unit is cut into shards)
                    t = p.data.to(self.device).contiguous()
                    dist.broadcast(t, src=0)
                    p.data = t
        u = ShardUnit(name, modules, params, layout)
        n = layout.shard_numel
        lo, _ = layout.shard_range(self.mesh.shard_rank)
        u.master = torch.zeros(n, dtype=torch.float32, device=self.device)
        for (pn, p), s in zip(params, layout.slots):
            ps, ss, ln = layout.overlap(s, self.mesh.shard_rank)
            if ln:
                u.master[ss:ss + ln].copy_(p.data.reshape(-1)[ps:ps + ln].to(self.device, torch.float32))
        if self.mp.param_dtype == torch.float32:
            u.lowp = u.master
            if self.coll.name != "torch" and self.mesh.shard_size > 1:
                u.lowp = self.coll.alloc_shard(n, torch.float32)
                u.lowp.copy_(u.master)
                u.master = u.lowp
        else:
            u.lowp = self.coll.alloc_shard(n, self.mp.param_dtype)
            u.lowp.copy_(u.master)
        u.exp_avg = torch.zeros(n, dtype=torch.float32, device=self.device)
        u.exp_avg_sq = torch.zeros(n, dtype=torch.float32, device=self.device)
        u.ev_gathered = self._event()
        u.ev_updated = self._event()
        if self.mesh.shard_size == 1:
            # nothing to gather: parameters live in the shard itself
            for _, p in params:
                p.data = self._placeholder
            u.full = _Buf(u.lowp, self._event())
            u.bind_params(u.lowp)
            # accumulating micro-steps in bf16 would round every partial sum: k > 1 keeps this buffer in fp32
            gdt = self.mp.reduce_dtype if self.grad_accum_steps == 1 else torch.float32
            if self.mesh.replica_size == 1:
                u.grad_shard = torch.zeros(layout.total, dtype=gdt, device=self.device)
                u.full_grad = _Buf(u.grad_shard, self._event())
            else:
                u.grad_shard = self.coll.alloc_full(layout.total, gdt)
                u.full_grad = _Buf(u.grad_shard, self._event())
        else:
            u.grad_shard = self.coll.alloc_grad_shard(n)
            for _, p in params:
                p.data = self._placeholder
        for _, p in params:
            p._grad_buf = None
            p._grad_ready = False
        u.recompute = False
        return u

    # --------------------------------------------------------------------------------- buffers
    def _acquire(self, pool, unit: ShardUnit, dtype, symmetric: bool, min_depth: int = 1) -> _Buf:
        """Oldest pooled buffer of this shape once ``min_depth`` buffers exist.  Gradient buffers need depth 2: a unit's
        buffer goes back to the pool the moment its reduce-scatter is ENQUEUED, so the next block would otherwise pick the same
        buffer and stall the compute stream for the whole reduce (measured: 0.58 ms idle per block at 2 GPUs, ~1.1 ms at 8)."""
        key = (unit.layout.signature(), dtype)
        lst = pool.setdefault(key, [])
        made = self._pool_made.setdefault((id(pool), key), 0)
        # (the decision must not depend on timing: symmetric-heap allocations are collective across ranks)
        if lst and made >= min_depth:
            return lst.pop(0)
        # gradient buffers are read by peers (symmetric heap); gathered parameters are local
        t = self.coll.alloc_full(unit.layout.total, dtype, symmetric=symmetric)
        self._pool_made[(id(pool), key)] = made + 1
        return _Buf(t, self._event())

    def _give_back(self, pool, unit: ShardUnit, buf: _Buf, dtype):
        pool.setdefault((unit.layout.signature(), dtype), []).append(buf)

    # ---------------------------------------------------------------------------------- gather
    def _start_gather(self, u: ShardUnit, dependent: bool = False, fuse: Optional[bool] = None,
                      split: Optional[float] = None):
        if self.mesh.shard_size == 1 or u.full is not None:
            return
        buf = self._acquire(self._full_pool, u, self.mp.param_dtype, False)
        fuse = self._fuse_gather if fuse is None else fuse
        if fuse:
            # compute-stream gather: the small vector prefix now, the matrices inside the next GEMM kernel
            from fms_fsdp_b200.ops import cuda_kernels as CK
            self.s_compute.wait_event(buf.free_event)
            self._wait_unit_updated(u, self.s_compute)
            es = u.lowp.element_size()
            mb, total = u.layout.matrix_begin * es, u.layout.total * es
            if mb > 0:
                self.coll.gather_range(u.lowp, buf.t, 0, mb)
            u.ag_req = None
            if total > mb:
                u.ag_req = self.coll.ag_request(u.lowp, buf.t, mb, total, dependent)
                if split is not None:
                    u.ag_req["split"] = split
                CK.push_ag_request(u.ag_req)
            u.full = buf
            u.gather_pending = True
            u.gather_fused = True
            if dependent:
                u.bind_params(buf.t)   # the carrier GEMM must already see its weight inside the buffer
            return
        u.gather_fused = False
        if self.is_cuda:
            with torch.cuda.stream(self.s_gather):
                self.s_gather.wait_event(buf.free_event)
                self._wait_unit_updated(u, self.s_gather)
                self.coll.all_gather(u.lowp, buf.t)
                u.ev_gathered.record(self.s_gather)
        else:
            self.coll.all_gather(u.lowp, buf.t)
        u.full = buf
        u.gather_pending = True

    def _wait_unit_updated(self, u: ShardUnit, stream):
        """Asynchronous sharded optimizer: the gather of ``u`` enqueued on ``stream`` (the current stream) must see this
        rank's AND every peer's AdamW update of the unit (own: CUDA event; peers: cross-rank flags)."""
        if self._async_sharded and self._opt_epoch > 0 and getattr(u, "_seen_epoch", 0) != self._opt_epoch:
            stream.wait_event(u.ev_updated)
            self.coll.wait_unit_updated(u.index, self._opt_epoch)
            u._seen_epoch = self._opt_epoch   # the backward re-gather of the same step needs no second wait

    def _nvtx(self, name: str):
        if not self._nvtx_on:
            return contextlib.nullcontext()
        return torch.cuda.nvtx.range(name)

    def _wait_gather(self, u: ShardUnit, allow_pending_dependent: bool = False):
        if u.full is None:
            self._start_gather(u)
        if self.async_optimizer and not self._async_sharded:
            self.s_compute.wait_event(u.ev_updated)   # this unit's (asynchronous) AdamW update has landed
        if u.gather_pending:
            if getattr(u, "gather_fused", False):
                req = getattr(u, "ag_req", None)
                if req is not None and not req["consumed"] and not (allow_pending_dependent and req["dependent"]):
                    from fms_fsdp_b200.ops import cuda_kernels as CK
                    CK.flush_ag_request(req)       # no GEMM carried it: standalone gather on the compute stream
            elif self.is_cuda:
                self.s_compute.wait_event(u.ev_gathered)
            u.gather_pending = False
            u.bind_params(u.full.t)

    def _release(self, u: ShardUnit):
        if self.mesh.shard_size == 1 or u.full is None:
            return
        if self.poison_released_params:
            # debug trap (SURVEY.md 5.2): any kernel that still reads this unit's gathered parameters after release
            # now sees NaN instead of silently-stale weights
            u.full.t.fill_(float("nan"))
        if self.is_cuda:
            u.full.free_event.record(self.s_compute)
        u.unbind_params(self._placeholder)
        self._give_back(self._full_pool, u, u.full, self.mp.param_dtype)
        u.full = None

    # ------------------------------------------------------------------------------- gradients
    def _prepare_grads(self, u: ShardUnit, rebind: bool = True):
        """Bind the unit's parameters to their gradient destination for this step.  ``rebind=False``: keep an existing
        binding (the root unit is bound before the head stage of the forward, where the fused linear-cross-entropy
        already writes the head's dW; the backward must not reset that)."""
        if not rebind and getattr(u, "_grads_bound", False):
            return
        u._grads_bound = True
        if self._push_rs and self._push_eligible(u):
            from fms_fsdp_b200.ops.cuda_kernels import PushTarget
            if u.full_grad is None:
                # staging buffer, laid out [src rank][shard elements]; symmetric (peers write into it)
                u.full_grad = self._acquire(self._push_pool, u, self.mp.reduce_dtype, True, min_depth=self._push_pool_depth)
            self.s_compute.wait_event(u.full_grad.free_event)   # every rank has finished summing its previous contents
            staging = u.full_grad.t
            if getattr(u, "vec_grad", None) is None:
                u.vec_grad = torch.zeros(u.layout.matrix_begin, dtype=staging.dtype, device=self.device)
            table, n, r = self.coll.push_table(staging), u.layout.shard_numel, self.mesh.shard_rank
            W = self.mesh.shard_size
            u.bind_grads_push(u.vec_grad, lambda s: PushTarget(table, n, s.offset, r, s.shape, self.device, world=W))
            u.pushed = True
            return
        if u.full_grad is None:
            buf = self._acquire(self._grad_pool, u, self.mp.reduce_dtype, True, min_depth=self._grad_pool_depth)
            u.full_grad = buf
        if self.is_cuda:
            self.s_compute.wait_event(u.full_grad.free_event)
        u.pushed = False
        # unsharded gradient accumulation: micro-steps 2..k add into the persistent buffer
        u.bind_grads(u.full_grad.t, accumulate=self.mesh.shard_size == 1 and self._micro > 1)

    def _push_eligible(self, u: ShardUnit) -> bool:
        """Block units whose every parameter is a norm-style vector or a weight matrix large enough for the fused-epilogue
        wgrad GEMM (LLaMA blocks); the root unit (embedding / tied or chunk-accumulated head) and units with other
        parameter kinds (Mamba conv / SSM tensors) keep the pull path."""
        if u is self.root:
            return False
        ok = getattr(u, "_push_ok", None)
        if ok is None:
            from fms_fsdp_b200.ops.cuda_kernels import push_eligible_shape
            # (slot shapes, not p.shape: released parameters point at an empty placeholder)
            ok = (all(len(sl.shape) == 1 or push_eligible_shape(tuple(sl.shape)) for sl in u.layout.slots)
                  and u.layout.matrix_begin % 8 == 0 and u.layout.shard_numel % 8 == 0
                  and getattr(u.modules[0], "engine_push_wgrad", True))
            u._push_ok = ok
        return ok

    def _warm_push_pool(self):
        """Allocate (and zero) every staging buffer of the push path NOW, followed by a cross-rank barrier.  Peers
        write into these buffers, so a lazily allocated buffer's zero-fill on this rank's stream could land AFTER a
        faster peer's first pushed tiles (found by the 2-GPU gradient check: every freshly allocated buffer of the
        first backward lost part of the peer's contribution)."""
        made = False
        for u in self.blocks:
            if not self._push_eligible(u):
                continue
            key = (u.layout.signature(), self.mp.reduce_dtype)
            lst = self._push_pool.setdefault(key, [])
            while len(lst) < self._push_pool_depth:
                t = self.coll.alloc_full(u.layout.total, self.mp.reduce_dtype, symmetric=True)
                self._pool_made[(id(self._push_pool), key)] = self._pool_made.get((id(self._push_pool), key), 0) + 1
                lst.append(_Buf(t, self._event()))
                made = True
            if getattr(u, "vec_grad", None) is None:
                u.vec_grad = torch.zeros(u.layout.matrix_begin, dtype=self.mp.reduce_dtype, device=self.device)
        if made:
            torch.cuda.synchronize(self.device)
            self.coll.barrier()

    def _on_reduce_barrier(self):
        """Called right after a flag round has been enqueued on the reduce stream: once it completes, every rank has
        finished the slot sum that preceded it, so that staging buffer may be pushed into again."""
        if self._push_pending is not None:
            self._push_pending.free_event.record(self.s_reduce)
            self._push_pending = None

    def _reduce(self, u: ShardUnit):
        u.collect_grads()
        u.unbind_grads()
        u._grads_bound = False
        m, W = self.mesh, self.mesh.world
        # gradient accumulation: micro-step 1 overwrites the fp32 shard, later ones add; the HSDP replica all-reduce and
        # ||g||^2 belong to the last micro-step only.  Unsharded meshes communicate once, after the last micro-step.
        last = self._micro >= self.grad_accum_steps
        if m.shard_size == 1 and not last:
            return
        acc = {} if self.grad_accum_steps == 1 else dict(accumulate=self._micro > 1, replica=last)
        ctx = torch.cuda.stream(self.s_reduce) if self.is_cuda else contextlib.nullcontext()
        if self.is_cuda:
            self.s_reduce.wait_stream(self.s_compute)
        with ctx:
            if m.shard_size == 1:
                self.coll.all_reduce_full(u.full_grad.t, 1.0 / W, self._gnorm_sq)
            elif getattr(u, "pushed", False):
                if u.layout.matrix_begin:
                    self.coll.push_vectors(u.vec_grad, u.full_grad.t)
                self.coll.reduce_pushed(u.full_grad.t, u.grad_shard, 1.0 / W, self._gnorm_sq if last else None,
                                        on_barrier=self._on_reduce_barrier, **acc)
                self._push_pending = u.full_grad      # reusable after the NEXT flag round on this stream
            elif self._push_rs:
                self.coll.reduce_scatter(u.full_grad.t, u.grad_shard, 1.0 / W, self._gnorm_sq if last else None,
                                         on_barrier=self._on_reduce_barrier, **acc)
            else:
                self.coll.reduce_scatter(u.full_grad.t, u.grad_shard, 1.0 / W, self._gnorm_sq if last else None, **acc)
            if self.is_cuda and not getattr(u, "pushed", False):
                u.full_grad.free_event.record(self.s_reduce)
        if m.shard_size > 1:
            self._give_back(self._push_pool if getattr(u, "pushed", False) else self._grad_pool, u, u.full_grad,
                            self.mp.reduce_dtype)
            u.full_grad = None

    # ------------------------------------------------------------------------ forward / backward
    @staticmethod
    def _as_tuple(x):
        return x if isinstance(x, tuple) else (x,)

    def _detach_state(self, state, requires_grad=True):
        out = []
        for t in self._as_tuple(state):
            d = t.detach()
            if requires_grad and d.is_floating_point():
                d.requires_grad_(True)
            out.append(d)
        return tuple(out)

    def _run_block(self, blk: nn.Module, state):
        out = blk(*state)
        return self._as_tuple(out)

    def _begin_micro_step(self):
        """Count one training micro-step (a forward with autograd on).  Returns True for the first micro-step of an
        optimizer step, which resets the step-level state (||g||^2, clip coefficient)."""
        k = self.grad_accum_steps
        if k == 1:
            self._micro = 1
            return True
        if self._micro >= k:
            raise RuntimeError(f"grad_accum_steps={k}: {k} micro-steps have already run since the last optimizer step; "
                               "call optimizer.step() before the next forward")
        self._micro += 1
        return self._micro == 1

    def _check_accumulated(self, what: str):
        k = self.grad_accum_steps
        if k > 1 and self._micro != k:
            raise RuntimeError(f"{what} after {self._micro} micro-step(s); grad_accum_steps={k} needs exactly {k} "
                               "forward/backward micro-steps per optimizer step")

    def optimizer_grad_scale(self) -> Optional[torch.Tensor]:
        """Multiplier the fused AdamW applies to the gradient shard: the clip coefficient (None = not clipped) and, with
        ``grad_accum_steps = k > 1``, the 1/k that turns the accumulated sum into the mean micro-batch gradient."""
        self._check_accumulated("optimizer step")
        if self.grad_accum_steps > 1 and self._clip_coef is None:
            return self._inv_accum
        return self._clip_coef

    def _forward(self, tokens, labels=None, *, autograd_driven: bool = False, **head_kwargs):
        """``autograd_driven``: the backward will come from ``loss.backward()`` (``forward``), with an upstream gradient
        that may scale the loss, instead of from ``forward_backward``."""
        model, blocks = self.module, self.blocks
        first = self._begin_micro_step() if torch.is_grad_enabled() else True
        fuse = self._fuse_gather and torch.is_grad_enabled()
        depth = 1 if fuse else self.prefetch_depth
        if self.is_cuda:
            if self._async_sharded and self._opt_epoch > 0:
                pass    # per-unit optimizer flags order every gather (``_wait_unit_updated``); no step barrier
            elif fuse:
                self.coll.begin_step()                 # cross-GPU barrier on the compute stream
            self.s_gather.wait_stream(self.s_compute)  # shards were just written by the optimizer
            if not fuse and not (self._async_sharded and self._opt_epoch > 0):
                with torch.cuda.stream(self.s_gather):
                    self.coll.begin_step()             # ... on every rank (cross-GPU barrier, fused path)
        else:
            self.coll.begin_step()
        if first:
            self._gnorm_sq.zero_()
            self._clip_coef = None
        self._start_gather(self.root, fuse=False)
        if fuse and blocks:
            # block 0's own weights arrive INSIDE its first GEMM (QKV projection), consumed tile by tile
            self._start_gather(blocks[0], dependent=True)
        else:
            for u in blocks[: depth]:
                self._start_gather(u, fuse=False)
        self._wait_gather(self.root)
        grad_on = torch.is_grad_enabled()
        with torch.enable_grad() if grad_on else torch.no_grad():
            emb_out = self._as_tuple(model.engine_embed(tokens))
        saved = []
        state = emb_out
        i = -1                                  # index of the current unit among ``blocks``
        for blk, u in self._chain:
            if u is not None:
                i += 1
                self._wait_gather(u, allow_pending_dependent=True)
                nxt = i + depth
                if nxt < len(blocks):
                    self._start_gather(blocks[nxt], fuse=fuse)   # fused: rides in one of block i's GEMMs
            recompute = is_checkpointed(blk)
            if u is not None:
                u.recompute = recompute
            with self._nvtx(f"fwd {u.name if u is not None else 'root-resident block'}"):
                if not grad_on:
                    with torch.no_grad():
                        state = self._run_block(blk, self._detach_state(state, False))
                elif recompute:
                    x_in = self._detach_state(state)
                    with torch.no_grad():
                        state = self._run_block(blk, x_in)
                    saved.append((x_in, None))
                else:
                    x_in = self._detach_state(state)
                    state = self._run_block(blk, x_in)
                    saved.append((x_in, state))
            if u is not None:
                keep = (not self.reshard_after_forward) or (grad_on and i >= len(blocks) - 1)
                if not keep:
                    self._release(u)
        head_in = self._detach_state(state, grad_on)
        # the head's dW is produced by the fused linear-CE of the forward, straight into the bound gradient buffer.  Not so
        # for an autograd-driven micro-step >= 2 on an unsharded mesh: that buffer already holds the earlier micro-steps,
        # so the loss's upstream gradient could no longer scale this micro-step's dW alone.  The head then computes dW as
        # an ordinary gradient; the backward binds the buffer (accumulating) and ``collect_grads`` adds it.
        if grad_on and not (autograd_driven and self.mesh.shard_size == 1 and self._micro > 1):
            self._prepare_grads(self.root)
        with torch.enable_grad() if grad_on else torch.no_grad():
            out = model.engine_head(*head_in, labels=labels, **head_kwargs) if labels is not None \
                else model.engine_head(*head_in, **head_kwargs)
        if grad_on:
            self._saved = dict(emb_out=emb_out, blocks=saved, head_in=head_in, head_out=out)
        else:
            for u in blocks:
                self._release(u)
        return out

    def _backward(self, dout=None):
        sv, blocks = self._saved, self.blocks
        if sv is None:
            raise RuntimeError("backward without a recorded forward")
        self._saved = None
        fuse = self._fuse_gather and self._fuse_gather_bwd
        depth = 1 if fuse else self.prefetch_depth
        n = len(blocks)
        # re-gather ahead (the last block is still resident from forward)
        for j in range(n - 1, max(-1, n - 1 - depth), -1):
            self._start_gather(blocks[j], fuse=fuse)
        # ---- head stage (root unit weights are still gathered)
        self._prepare_grads(self.root, rebind=False)
        out = sv["head_out"]
        from fms_fsdp_b200.ops import functional as _F
        _F.set_unit_upstream(dout is None)      # our own schedule differentiates with an upstream gradient of 1
        try:
            torch.autograd.backward(out, dout if dout is not None else torch.ones_like(out))
        finally:
            _F.set_unit_upstream(False)
        dstate = tuple(t.grad for t in sv["head_in"])
        for t in sv["head_in"]:
            t.grad = None
        del out
        sv["head_out"] = None
        # ---- blocks in reverse, re-gathering ahead
        i = n                                   # index of the current unit among ``blocks``
        for pos in range(len(self._chain) - 1, -1, -1):
            blk, u = self._chain[pos]
            if u is not None:
                i -= 1
                self._wait_gather(u)
                nxt = i - depth
                if nxt >= 0:
                    # fused: rides inside block i's backward GEMMs (FMS_B200_AG_SPLIT_BWD < 1 spreads it over more of them)
                    self._start_gather(blocks[nxt], fuse=fuse, split=self._bwd_gather_split)
                self._prepare_grads(u)
            x_in, y = sv["blocks"][pos]
            with self._nvtx(f"bwd {u.name if u is not None else 'root-resident block'}"):
                if y is None:  # selective recompute with the weights that are resident for backward anyway
                    with torch.enable_grad():
                        y = self._run_block(blk, x_in)
                pairs = [(a, g) for a, g in zip(y, dstate) if g is not None and a.requires_grad]
                torch.autograd.backward([a for a, _ in pairs], [g for _, g in pairs])
            dstate = tuple(t.grad for t in x_in)
            for t in x_in:
                t.grad = None
            sv["blocks"][pos] = None
            del y, pairs
            if u is not None:
                with self._nvtx(f"reduce {u.name}"):
                    self._reduce(u)
                self._release(u)
        # ---- embedding stage
        pairs = [(a, g) for a, g in zip(sv["emb_out"], dstate) if g is not None and a.requires_grad]
        if pairs:
            torch.autograd.backward([a for a, _ in pairs], [g for _, g in pairs])
        self._reduce(self.root)
        self._release(self.root)
        if self.is_cuda:
            ev = getattr(self.coll, "last_reduce_done", None)
            if ev is not None:
                # the root's fp32 shard and ||g||^2 are complete; the trailing "peers are done reading my buffer" flag
                # round stays on the reduce stream (it only gates the buffer's reuse, ``_Buf.free_event``)
                self.s_compute.wait_event(ev)
                self.coll.last_reduce_done = None
            else:
                self.s_compute.wait_stream(self.s_reduce)

    def forward_backward(self, tokens, labels, **head_kwargs) -> torch.Tensor:
        """One training micro-step: returns the (detached) mean loss; gradients end up reduced,
        scaled by 1/world and sharded, with ||g||^2 accumulated for ``clip_grad_norm_`` (on the last of
        ``grad_accum_steps`` micro-steps; earlier ones add their gradient to the shard)."""
        loss = self._forward(tokens, labels, **head_kwargs)
        self._backward(None)
        return loss.detach()

    def forward_backward_custom(self, loss_closure) -> torch.Tensor:
        """Training micro-step for models that are a single (root) unit, e.g. the MLP speculator under NO_SHARD:
        ``loss_closure(module) -> scalar loss`` runs under autograd with the parameters gathered; gradients are
        reduced (all-reduce / reduce-scatter + replica reduce), scaled by 1/world and norm-accumulated."""
        if self.blocks:
            raise RuntimeError("forward_backward_custom is for root-only models")
        first = self._begin_micro_step()
        if self.is_cuda:
            self.s_gather.wait_stream(self.s_compute)
            with torch.cuda.stream(self.s_gather):
                self.coll.begin_step()
        else:
            self.coll.begin_step()
        if first:
            self._gnorm_sq.zero_()
            self._clip_coef = None
        self._start_gather(self.root, fuse=False)   # the step barrier above sits on the gather stream
        self._wait_gather(self.root)
        self._prepare_grads(self.root)
        with torch.enable_grad():
            loss = loss_closure(self.module)
        loss.backward()
        self._reduce(self.root)
        self._release(self.root)
        if self.is_cuda:
            self.s_compute.wait_stream(self.s_reduce)
        return loss.detach()

    # reference-style API: ``out = model(input)`` ... ``loss.backward()``
    def forward(self, tokens, labels=None, **head_kwargs):
        if not torch.is_grad_enabled():
            return self._forward(tokens, labels, **head_kwargs)
        out = self._forward(tokens, labels, autograd_driven=True, **head_kwargs)
        return _EngineOutput.apply(self, out.detach(), self._anchor())

    def _anchor(self):
        a = getattr(self, "_anchor_t", None)
        if a is None:
            a = torch.zeros((), device=self.device, requires_grad=True)
            self._anchor_t = a
        return a

    # --------------------------------------------------------------------------- grad clipping
    def clip_grad_norm_(self, max_norm: float, norm_type: float = 2.0) -> torch.Tensor:
        """Global L2 norm of the (already reduced) gradient; the clip factor is consumed by the fused
        optimizer step instead of a separate pass over the gradients (reference semantics:
        torch ``fully_sharded_data_parallel.py:1165-1215``, called at ``train_utils.py:96``)."""
        if norm_type != 2.0:
            raise NotImplementedError("only the L2 norm is supported")
        self._check_accumulated("clip_grad_norm_")
        k = self.grad_accum_steps
        total = self._gnorm_sq.clone()
        self.coll.all_reduce_scalar(total, over="shard")
        norm = total.sqrt()
        if k > 1:
            norm.div_(k)             # the shard holds the SUM of k micro-step gradients; the norm is that of their mean
        # engine-owned scalar: the asynchronous optimizer's kernels on ``s_opt`` read it after this call returns, so it
        # must not be a temporary the caching allocator could hand to the next step's compute-stream allocations
        if getattr(self, "_clip_coef_buf", None) is None:
            self._clip_coef_buf = torch.ones((), dtype=torch.float32, device=self.device)
        torch.clamp(max_norm / (norm + 1e-6), max=1.0, out=self._clip_coef_buf)
        if k > 1:
            self._clip_coef_buf.div_(k)   # AdamW's multiplier of the summed gradient: clip coefficient / k
        self._clip_coef = self._clip_coef_buf
        self.last_grad_norm = norm
        return norm

    # ------------------------------------------------------------------ full-parameter access
    def gather_unit_full(self, u: ShardUnit, which: str = "master") -> torch.Tensor:
        """All-gather one unit's fp32 shard (master / exp_avg / exp_avg_sq) into a flat fp32 tensor."""
        if self.async_optimizer:
            torch.cuda.current_stream(self.device).wait_stream(self.s_opt)
        shard = getattr(u, which)
        if self.mesh.shard_size == 1:
            return shard.float() if shard.dtype != torch.float32 else shard
        full = torch.empty(u.layout.total, dtype=shard.dtype, device=self.device)
        import torch.distributed as dist
        dist.all_gather_into_tensor(full, shard.contiguous(), group=self.mesh.shard_group)
        return full

    def named_unit_views(self, u: ShardUnit, flat: torch.Tensor):
        for s in u.layout.slots:
            yield s.name, flat[s.offset:s.offset + s.numel].view(s.shape)

    def load_unit_from_full(self, u: ShardUnit, which: str, tensors: Dict[str, torch.Tensor]):
        """Copy this rank's slice out of full (unsharded) per-parameter tensors."""
        shard = getattr(u, which)
        for s in u.layout.slots:
            if s.name not in tensors:
                continue
            ps, ss, ln = u.layout.overlap(s, self.mesh.shard_rank)
            if ln:
                shard[ss:ss + ln].copy_(tensors[s.name].reshape(-1)[ps:ps + ln])
        if which == "master" and u.lowp is not u.master:
            u.lowp.copy_(u.master)

    def full_state_dict(self, dtype=None, cpu=True) -> Dict[str, torch.Tensor]:
        """Unsharded parameters under their original (FMS) names; every rank gets the full dict."""
        out = {}
        for u in self.units:
            flat = self.gather_unit_full(u, "master")
            for name, v in self.named_unit_views(u, flat):
                t = v.to(dtype) if dtype is not None else v.clone()
                out[name] = t.cpu() if cpu else t
        return out

    def load_full_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        names = {s.name for u in self.units for s in u.layout.slots}
        missing = sorted(names - set(sd))
        unexpected = sorted(set(sd) - names)
        if strict and (missing or unexpected):
            raise RuntimeError(f"state dict mismatch: missing {missing[:5]} unexpected {unexpected[:5]}")
        for u in self.units:
            self.load_unit_from_full(u, "master", {k: v.to(self.device, torch.float32) for k, v in sd.items()
                                                  if k in {s.name for s in u.layout.slots}})
        return missing, unexpected

    @contextlib.contextmanager
    def summon_full_params(self):
        """Gather every unit (compute dtype) so the wrapped module can be used directly (eval, export)."""
        for u in self.units:
            self._wait_gather(u)
        try:
            yield self.module
        finally:
            if self.is_cuda:
                torch.cuda.current_stream().synchronize()
            for u in self.units:
                self._release(u)

    def param_count(self) -> int:
        return sum(u.layout.used for u in self.units)

    def extra_repr(self) -> str:
        m = self.mesh
        return (f"units={len(self.units)}, mesh=replica{m.replica_size}xshard{m.shard_size}, "
                f"param_dtype={self.mp.param_dtype}, collectives={self.coll.name}")


class _EngineOutput(torch.autograd.Function):
    """Bridges the engine's explicit backward schedule into ``loss.backward()`` for callers that use
    the reference-style loop (``out = model(x); loss = CE(out, y); loss.backward()``)."""

    @staticmethod
    def forward(ctx, engine, out, anchor):
        ctx.engine = engine
        return out.clone() if out.dim() == 0 else out

    @staticmethod
    def backward(ctx, dout):
        ctx.engine._backward(dout)
        return None, None, None
