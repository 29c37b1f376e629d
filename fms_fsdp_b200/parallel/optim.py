"""Sharded fused AdamW.

Reference: ``torch.optim.AdamW(lr, betas=(0.9, 0.95), weight_decay=0.1)`` over FSDP's sharded flat
parameters (``main_training_llama.py:113-115``), one parameter group so weight decay hits norm
gains and embeddings too (SURVEY.md Q14).  Here the update is one fused kernel per shard unit on
the fp32 master shard that also (a) applies the gradient-clip factor computed by
``ShardedModel.clip_grad_norm_`` and (b) writes the refreshed compute-dtype shard that the next
all-gather sends -- K11/K12/K13 of SURVEY.md §2.5 collapse into this step.
It is a real ``torch.optim.Optimizer`` so ``LambdaLR`` and friends work unchanged.
"""
from __future__ import annotations

from typing import Dict

import torch

from fms_fsdp_b200.ops.functional import kernels_for


class ShardedAdamW(torch.optim.Optimizer):
    def __init__(self, model, lr: float = 3e-4, betas=(0.9, 0.95), eps: float = 1e-8, weight_decay: float = 0.1):
        self.engine = model
        params = [u.master for u in model.units]
        for p in params:
            p.requires_grad_(False)
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay)
        super().__init__([{"params": params}], defaults)
        self._step = 0

    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        g = self.param_groups[0]
        eng = self.engine
        coef = eng.optimizer_grad_scale()     # clip coefficient, and 1/k under gradient accumulation
        self._step += 1
        lr, (b1, b2), eps, wd = float(g["lr"]), g["betas"], g["eps"], g["weight_decay"]

        sharded_async = eng.async_optimizer and getattr(eng, "_async_sharded", False)
        epoch = eng._opt_epoch + 1 if sharded_async else 0

        def update_all():
            nvtx = eng._nvtx("optimizer") if hasattr(eng, "_nvtx") else None
            if nvtx is not None:
                nvtx.__enter__()
            for u in eng.units:  # root first, then blocks in forward order: the order the next forward needs them
                K = kernels_for(u.master)
                K.adamw_step(u.master, u.grad_shard, u.exp_avg, u.exp_avg_sq,
                             None if u.lowp is u.master else u.lowp, lr, b1, b2, eps, wd, self._step, coef)
                if eng.async_optimizer:
                    u.ev_updated.record(eng.s_opt)
                    if sharded_async:   # tell every shard rank that my slice of this unit is updated
                        eng.coll.post_unit_updated(u.index, epoch)
            if nvtx is not None:
                nvtx.__exit__(None, None, None)

        if eng.async_optimizer:
            # Bandwidth-bound update on a side stream: it overlaps the next forward's (compute-bound) GEMMs; each
            # unit's forward waits only for that unit's own update (``ShardedModel._wait_gather``).  When peers read our
            # shards (shard group > 1) each unit's update is followed by a cross-rank flag that the peers' gathers of that
            # unit wait for (``ShardedModel._wait_unit_updated``) -- no step barrier.
            eng.s_opt.wait_stream(eng.s_compute)
            with torch.cuda.stream(eng.s_opt):
                update_all()
            if sharded_async:
                eng._opt_epoch = epoch
        else:
            update_all()
        eng._clip_coef = None
        eng._micro = 0
        eng.step_count = self._step
        return loss

    def zero_grad(self, set_to_none: bool = True):
        # gradient buffers are overwritten by the first micro-step after a step (and accumulated over the others when
        # the engine has ``grad_accum_steps > 1``): there is nothing to zero
        return None

    # flat, rank-local state (the Checkpointer uses the per-parameter sharded view instead)
    def state_dict(self) -> Dict:
        return {
            "step": self._step,
            "param_groups": [{k: v for k, v in g.items() if k != "params"} for g in self.param_groups],
            "units": {u.name: {"exp_avg": u.exp_avg, "exp_avg_sq": u.exp_avg_sq} for u in self.engine.units},
        }

    def load_state_dict(self, sd: Dict):
        self._step = int(sd.get("step", 0))
        for g, sg in zip(self.param_groups, sd.get("param_groups", [])):
            for k, v in sg.items():
                if k != "params":
                    g[k] = v
        for u in self.engine.units:
            st = sd.get("units", {}).get(u.name)
            if st is not None:
                u.exp_avg.copy_(st["exp_avg"])
                u.exp_avg_sq.copy_(st["exp_avg_sq"])
