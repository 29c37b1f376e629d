"""Training loop and runtime helpers.

Public names match reference ``fms_fsdp/utils/train_utils.py`` (``train, setup,
setup_environ_flags, get_mixed_precision_policy, get_policies, get_profiler``); the stdout
keys printed every ``report_interval`` are the reference's (``:135-149``) plus MFU and the
device-timed step (max over ranks), which the north-star metric requires.

Differences that are deliberate (SURVEY.md App. C): loss / grad-norm stay on the device between
reports (no two host syncs per step, Q10); step time is measured with CUDA events; inputs go
host->device from pinned memory asynchronously; ``tokens_seen`` is always defined when a
checkpoint fires (Q3).
"""
from __future__ import annotations

import math
import os
import sys
import time
from dataclasses import asdict
from datetime import timedelta
from functools import partial

import torch
import torch.distributed as dist

from fms_fsdp_b200 import ops
from fms_fsdp_b200.policies import (apply_fsdp_checkpointing, bfSixteen, fpSixteen, get_wrapper,
                                    param_init_function)


# ------------------------------------------------------------------------------------ process group
def pick_backend(cfg=None) -> str:
    want = getattr(cfg, "comm_backend", "auto") if cfg is not None else "auto"
    if want in ("nccl", "gloo"):
        return want
    return "nccl" if torch.cuda.is_available() else "gloo"


def setup(backend: str = None, cfg=None):
    """Rendezvous only (NCCL on GPU, gloo on CPU); hot-path collectives are the engine's own.
    Reference: ``fms_fsdp/utils/train_utils.py:183-184``."""
    backend = backend or pick_backend(cfg)
    if not dist.is_initialized():
        dist.init_process_group(backend, timeout=timedelta(seconds=60 * 60))
    return backend


def setup_environ_flags():
    """Reference: ``fms_fsdp/utils/train_utils.py:187-189``."""
    os.environ["TORCH_SHOW_CPP_STACKTRACES"] = str(1)
    os.environ["NCCL_ASYNC_ERROR_HANDLING"] = str(1)
    os.environ.setdefault("TORCH_NCCL_ASYNC_ERROR_HANDLING", str(1))


def torchrun_env():
    return (int(os.environ.get("LOCAL_RANK", 0)), int(os.environ.get("RANK", 0)),
            int(os.environ.get("WORLD_SIZE", 1)))


# ----------------------------------------------------------------------------------------- policies
def get_mixed_precision_policy(cfg, rank):
    """bf16 everywhere when the device supports it (always on H100), fp16 otherwise, None when off.
    Reference: ``fms_fsdp/utils/train_utils.py:192-214``."""
    if not cfg.mixed_precision:
        return None
    bf16_ready = (not torch.cuda.is_available()) or torch.cuda.is_bf16_supported()
    policy = bfSixteen if bf16_ready else fpSixteen
    if rank == 0:
        print("bFloat16 enabled for mixed precision - using bfSixteen policy" if bf16_ready else "FP16 enabled")
    if getattr(cfg, "grad_dtype", "bf16") == "fp32":
        # extension: keep the unsharded gradient buffer (what the wgrad GEMMs write and the reduce-scatter reads) in
        # fp32 instead of the reference's reduce_dtype = bf16
        import dataclasses
        policy = dataclasses.replace(policy, reduce_dtype=torch.float32)
    return policy


_STRATEGIES = {"fsdp": "fsdp", "hsdp": "hsdp", "ddp": "ddp"}


def get_policies(cfg, rank, block):
    """(mixed_precision_policy, wrapping_policy, sharding_strategy, apply_selective_ac, param_init_fn).
    Reference: ``fms_fsdp/utils/train_utils.py:217-253``."""
    precision = getattr(cfg, "precision", "bf16")
    if precision not in ("bf16", "fp8"):
        raise NotImplementedError(f"precision={precision!r}: bf16 (default) and fp8 (row-wise scaled e4m3 forward GEMMs, bf16 "
                                  "backward) exist; block-scaled mxfp8 operands are future work, see DESIGN.md section 6")
    from fms_fsdp_b200.ops.functional import set_gemm_precision
    set_gemm_precision(precision)
    if precision != "bf16" and rank == 0:
        print("--> forward GEMMs run on e4m3 operands (row-wise scales, fp32 accumulation); backward stays bf16")
    mixed_precision_policy = get_mixed_precision_policy(cfg, rank)
    wrapping_policy = get_wrapper(block)
    sharding_strategy = _STRATEGIES.get(cfg.sharding_strategy, "fsdp")  # unknown -> full shard, like the reference
    if rank == 0:
        print(f"Sharding strategy = {cfg.sharding_strategy}")
    apply_selective_ac = partial(apply_fsdp_checkpointing, block=block)
    param_init_fn = param_init_function if cfg.low_cpu_fsdp else None
    return (mixed_precision_policy, wrapping_policy, sharding_strategy, apply_selective_ac, param_init_fn)


def get_profiler(cfg, rank):
    """Reference: ``fms_fsdp/utils/train_utils.py:256-271``."""
    if not cfg.use_profiler:
        return None
    if cfg.profiler_rank0_only and rank != 0:
        return None
    acts = [torch.profiler.ProfilerActivity.CPU]
    if torch.cuda.is_available():
        acts.append(torch.profiler.ProfilerActivity.CUDA)
    return torch.profiler.profile(
        activities=acts,
        schedule=torch.profiler.schedule(wait=1, warmup=2, active=3, repeat=1),
        on_trace_ready=torch.profiler.tensorboard_trace_handler("profile_traces"),
        profile_memory=True, with_stack=False, record_shapes=True,
    )


# --------------------------------------------------------------------------------------- LR schedule
def lr_schedule_fn(cfg):
    """Reference ``main_training_llama.py:137-148``: quadratic warm-up over min(2000, steps/20) then
    cosine to 0.1x; 'annealing' = linear to zero."""
    if cfg.training_stage == "annealing":
        return lambda x: 1 - x / cfg.num_steps
    warmup = max(1, min(2000, cfg.num_steps // 20))
    return lambda x: min(
        1 - (1 - min(x, warmup) / warmup) ** 2,
        0.1 + 0.5 * (1 - 0.1) * (1 + math.cos(min(x, cfg.num_steps) / cfg.num_steps * math.pi)),
    )


def model_flops_per_token(n_params: int, n_layers: int, emb_dim: int, seq_len: int) -> float:
    """NanoGPT/PaLM accounting used by the reference README: 6N + 12 L D S."""
    return 6.0 * n_params + 12.0 * n_layers * emb_dim * seq_len


def peak_tflops() -> float:
    """Roofline denominator: measured cuBLAS bf16 (MEASURED_PEAKS.json) else the recipe's fallback."""
    import json
    for p in (os.path.join(os.path.dirname(__file__), "..", "..", "MEASURED_PEAKS.json"), "MEASURED_PEAKS.json"):
        try:
            with open(p) as f:
                return float(json.load(f)["bf16_tflops_sustained"])
        except Exception:
            continue
    return 989.0   # H100 SXM data-sheet dense bf16 (700 W); power-limited cards reach less


# ------------------------------------------------------------------------------------------ trackers
def _init_tracker(cfg, rank):
    if not cfg.tracker:
        return None
    if cfg.tracker not in ("wandb", "aim"):
        raise ValueError(f"tracker {cfg.tracker} not supported.")
    if cfg.tracker == "wandb":
        try:
            import wandb  # type: ignore
        except ImportError:
            raise ImportError("tracker is set to wandb but wandb is not installed.")
        if rank != 0:
            return None
        print("--> wandb is enabled!")
        try:
            wandb.init(project=cfg.tracker_project_name, dir=cfg.tracker_dir, resume="allow", id=cfg.tracker_run_id)
        except wandb.errors.UsageError:
            raise ValueError("wandb failed to init, did you pass your wandb api key via WANDB_API_KEY?")
        wandb.config = asdict(cfg)
        return wandb.log
    try:
        from aim import Run  # type: ignore
    except ImportError:
        raise ImportError("tracker is set to aim but aim is not installed.")
    if rank != 0:
        return None
    print("--> aim is enabled!")
    run = Run(experiment=cfg.tracker_project_name, repo=cfg.tracker_dir, run_hash=cfg.tracker_run_id)
    run["hparams"] = asdict(cfg)
    return run.track


# --------------------------------------------------------------------------------------------- train
# One page-locked arena per process for the loop's staging slots.  cudaHostAlloc maps the block into every visible device
# and takes the driver lock: with 8 GPUs visible each call cost tens of milliseconds (the first train() call of an 8-GPU
# job spent ~0.4 s in eight of them), so the slots are carved out of ONE allocation that later train() calls reuse.
_ARENA = {"buf": None, "used": 0}


def _pinned_slot(shape, dtype) -> torch.Tensor:
    n = 1
    for d in shape:
        n *= int(d)
    nbytes = (n * torch.empty((), dtype=dtype).element_size() + 255) // 256 * 256
    if _ARENA["buf"] is None or _ARENA["used"] + nbytes > _ARENA["buf"].numel():
        if _ARENA["buf"] is not None and nbytes <= _ARENA["buf"].numel():
            _ARENA["used"] = 0           # wrap: old slots belong to loops that have finished
        else:
            _ARENA["buf"] = torch.empty(max(4 << 20, 2 * nbytes), dtype=torch.uint8).pin_memory()
            _ARENA["used"] = 0
    off = _ARENA["used"]
    _ARENA["used"] += nbytes
    return _ARENA["buf"][off:off + n * torch.empty((), dtype=dtype).element_size()].view(dtype).view(shape)


class _H2DStager:
    """Host -> device path of the training loop: the loader's (pageable) batch is copied into a small ring of PINNED
    staging buffers and sent with an asynchronous copy, so the step's input transfer overlaps the previous step's
    compute instead of pinning fresh memory every step (cudaHostAlloc) or taking the synchronous pageable path."""

    def __init__(self, device, depth: int = 4):
        self.device, self.depth, self.slots, self.k = device, depth, {}, 0

    def __call__(self, t: torch.Tensor) -> torch.Tensor:
        if self.device.type != "cuda":
            return t.to(self.device)
        if t.is_cuda:
            return t
        key = (tuple(t.shape), t.dtype)
        ring = self.slots.get(key)
        if ring is None:
            ring = [(_pinned_slot(t.shape, t.dtype), torch.cuda.Event()) for _ in range(self.depth)]
            self.slots[key] = ring
        buf, ev = ring[self.k % self.depth]
        self.k += 1
        ev.synchronize()                 # the copy that last used this pinned slot has left the host
        buf.copy_(t)
        out = buf.to(self.device, non_blocking=True)
        ev.record(torch.cuda.current_stream(self.device))
        return out


class _LossReadback:
    """Every step: 4-byte asynchronous device -> host copy of the step's loss into pinned memory; the value is looked
    at ONE step later (non-finite guard without stalling the launch pipeline, SURVEY.md 5.3 / K15)."""

    def __init__(self, device, depth: int = 4):
        self.on = device.type == "cuda"
        if self.on:
            self.ring = [(_pinned_slot((1,), torch.float32), torch.cuda.Event(), [None]) for _ in range(depth)]
        self.k, self.depth, self.device, self.last = 0, depth, device, None

    def push(self, loss: torch.Tensor, step: int):
        """Returns (step, value) of the oldest completed read-back, or None."""
        if not self.on:
            return None
        buf, ev, tag = self.ring[self.k % self.depth]
        done = None
        if tag[0] is not None:
            ev.synchronize()
            done = (tag[0], float(buf[0]))
            self.last = done
        buf.copy_(loss.detach().reshape(1).float(), non_blocking=True)
        ev.record(torch.cuda.current_stream(self.device))
        tag[0] = step
        self.k += 1
        return done


def _step_groups(loader, k: int):
    """Consecutive groups of ``k`` loader batches: the micro-batches of one optimizer step."""
    group = []
    for batch in loader:
        group.append(batch)
        if len(group) == k:
            yield group
            group = []


def train(cfg, model, local_rank, rank, train_loader, optimizer, scheduler, profiler, checkpointer,
          start_step, tokens_seen):
    """Reference: ``fms_fsdp/utils/train_utils.py:21-180``.

    ``cfg.grad_accum_steps = k`` draws k loader batches per optimizer step (the engine averages their gradients).
    Steps, the LR schedule, report / checkpoint intervals and ``fault_inject_step`` count optimizer steps; the reported
    loss is the mean of the k micro-batch losses and token counts include all k micro-batches."""
    tracker_fn = _init_tracker(cfg, rank)
    is_cuda = torch.cuda.is_available() and getattr(model, "is_cuda", True)
    device = getattr(model, "device", torch.device("cuda", local_rank) if is_cuda else torch.device("cpu"))
    world_size = int(os.environ.get("WORLD_SIZE", 1))
    engine_mode = hasattr(model, "forward_backward")
    accum = int(getattr(cfg, "grad_accum_steps", 1))
    step_tokens = cfg.batch_size * cfg.seq_length * accum     # per GPU and optimizer step
    model.train()
    ddp_stats = torch.zeros(3, device=device)  # [sum loss, sum gnorm, steps]
    to_device = _H2DStager(device)
    readback = _LossReadback(device) if getattr(cfg, "loss_readback", True) else None

    n_params = model.param_count() if hasattr(model, "param_count") else sum(p.numel() for p in model.parameters())
    mcfg = getattr(getattr(model, "module", model), "config", None)
    flops_tok = None
    if mcfg is not None and hasattr(mcfg, "nlayers"):
        # a mixture-of-experts model: only the router and k of E experts per block run for a token
        n_active = n_params - (mcfg.inactive_params() if hasattr(mcfg, "inactive_params") else 0)
        flops_tok = model_flops_per_token(n_active, mcfg.nlayers, mcfg.emb_dim, cfg.seq_length)
    # MoE: the load-balancing loss of every micro-batch, summed on the device and read at report steps only
    inner = getattr(model, "module", model)
    moe_aux = torch.zeros((), device=device) if getattr(mcfg, "moe_num_experts", 0) > 0 else None
    # z-losses (coefficient-scaled), summed the same way; reported only when their coefficient is set
    z_coef = float(getattr(cfg, "z_loss_coef", 0.0) or 0.0)
    z_sum = torch.zeros((), device=device) if z_coef > 0 else None
    router_z_sum = torch.zeros((), device=device) if float(getattr(cfg, "moe_router_z_loss_coef", 0.0) or 0.0) > 0 \
        else None

    ev0 = ev1 = None
    if is_cuda:
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
    start = loop_start = time.time()
    train_loss = -1
    new_tokens_seen = 0
    for batch_idx, micro_batches in enumerate(_step_groups(train_loader, accum), start=start_step + 1):
        if batch_idx > cfg.num_steps:
            break
        if cfg.fault_inject_step and batch_idx == cfg.fault_inject_step and rank == min(1, world_size - 1):
            print(f"[fault-inject] rank {rank} exiting at step {batch_idx}", flush=True)
            os._exit(17)

        optimizer.zero_grad()
        loss = None
        for input, label in micro_batches:
            input = to_device(input)
            label = to_device(label)
            if engine_mode and cfg.fused_cross_entropy:
                micro_loss = model.forward_backward(input, label.long() if label.dtype != torch.long else label)
                if z_sum is not None:
                    z_sum += inner.z_loss().to(z_sum.device)
            else:
                output = model(input)
                output = output.logits if hasattr(output, "logits") else output
                if z_sum is not None:
                    # the output z-loss on the materialised logits: its gradient is folded into micro_loss's
                    micro_loss, micro_z = ops.cross_entropy_z(output.view(-1, output.size(-1)), label.view(-1).long(),
                                                              z_coef)
                    z_sum += micro_z.to(z_sum.device) * z_coef
                else:
                    micro_loss = torch.nn.functional.cross_entropy(output.view(-1, output.size(-1)).float(),
                                                                   label.view(-1).long())
                del output
                micro_loss.backward()
                micro_loss = micro_loss.detach()
            loss = micro_loss if loss is None else loss + micro_loss
            if moe_aux is not None:
                moe_aux += inner.moe_aux_loss().to(moe_aux.device)
            if router_z_sum is not None:
                router_z_sum += inner.moe_router_z_loss().to(router_z_sum.device)
        if accum > 1:
            loss = loss / accum
        gnorm = model.clip_grad_norm_(cfg.grad_clip_thresh)
        optimizer.step()
        scheduler.step()

        ddp_stats[0] += loss
        ddp_stats[1] += gnorm
        ddp_stats[2] += 1
        if readback is not None:
            seen = readback.push(loss, batch_idx)
            if seen is not None and not math.isfinite(seen[1]):
                msg = f"[non-finite] step {seen[0]}: loss {seen[1]}"
                if getattr(cfg, "nonfinite_action", "warn") == "halt":
                    raise FloatingPointError(msg + " -- halting (nonfinite_action=halt); restart resumes from the last checkpoint")
                if rank == 0:
                    print(msg, flush=True)

        if profiler:
            profiler.step()

        new_tokens_seen = (batch_idx - start_step) * world_size * step_tokens
        if batch_idx % cfg.report_interval == 0:
            dev_step_time = None
            if is_cuda:
                ev1.record()
                ev1.synchronize()
                t = torch.tensor([ev0.elapsed_time(ev1) / 1e3 / cfg.report_interval], device=device)
                if world_size > 1:
                    dist.all_reduce(t, op=dist.ReduceOp.MAX)
                dev_step_time = t.item()
            if world_size > 1:
                dist.all_reduce(ddp_stats, op=dist.ReduceOp.SUM)
                if moe_aux is not None:
                    dist.all_reduce(moe_aux, op=dist.ReduceOp.SUM)
                for t_ in (z_sum, router_z_sum):
                    if t_ is not None:
                        dist.all_reduce(t_, op=dist.ReduceOp.SUM)
            train_loss = ddp_stats[0] / ddp_stats[2]
            g_norm = ddp_stats[1] / ddp_stats[2]
            # failure detection the reference lacks (SURVEY.md 5.3): a non-finite loss / grad norm is surfaced at the
            # report step (already a sync point, so it costs nothing) and can stop the job so that restart + auto-resume
            # rolls back to the last checkpoint instead of training on garbage
            if not bool(torch.isfinite(train_loss)) or not bool(torch.isfinite(g_norm)):
                msg = f"[non-finite] step {batch_idx}: loss {train_loss.item()} gradient norm {g_norm.item()}"
                if getattr(cfg, "nonfinite_action", "warn") == "halt":
                    raise FloatingPointError(msg + " -- halting (nonfinite_action=halt); restart resumes from the last checkpoint")
                if rank == 0:
                    print(msg, flush=True)
            elapsed_time = time.time() - loop_start
            if rank == 0:
                total_tokens_seen = tokens_seen + new_tokens_seen
                current_loss = train_loss.item()
                current_lr = scheduler.get_last_lr()[0]
                current_gnorm = g_norm.item()
                current_step_time = (time.time() - start) / cfg.report_interval
                overall_step_time = elapsed_time / (batch_idx - start_step)
                current_throughput = int(step_tokens / current_step_time)
                overall_throughput = int(step_tokens / overall_step_time)
                reserved_mem = torch.cuda.max_memory_reserved(device) if is_cuda else 0
                allocated_mem = torch.cuda.max_memory_allocated(device) if is_cuda else 0
                print("step:", batch_idx)
                print("loss:", current_loss)
                print("LR:", current_lr)
                print("tokens seen:", total_tokens_seen)
                print("gradient norm:", current_gnorm)
                if moe_aux is not None:   # coef * mean over layers, micro-batches, steps and ranks
                    print("moe_aux_loss:", moe_aux.item() / (ddp_stats[2].item() * accum))
                # coef * mean over micro-batches, steps and ranks (and layers for the router's)
                z_report = {}
                if z_sum is not None:
                    z_report["z_loss"] = z_sum.item() / (ddp_stats[2].item() * accum)
                if router_z_sum is not None:
                    z_report["moe_router_z_loss"] = router_z_sum.item() / (ddp_stats[2].item() * accum)
                for k_, v_ in z_report.items():
                    print(f"{k_}:", v_)
                print("reserved memory:", reserved_mem)
                print("allocated memory:", allocated_mem)
                print("current step time:", current_step_time)
                print("overall step time:", overall_step_time)
                print("current token per gpu per sec:", current_throughput)
                print("overall token per gpu per sec:", overall_throughput)
                print("overall token per day:", int(new_tokens_seen / elapsed_time * 3600 * 24))
                if dev_step_time is not None:
                    print("device step time (max over ranks):", dev_step_time)
                    if flops_tok is not None:
                        tf = step_tokens / dev_step_time * flops_tok / 1e12
                        print("model TFLOP/s per gpu:", round(tf, 1), " MFU vs measured bf16 peak:",
                              round(tf / peak_tflops(), 4))
                sys.stdout.flush()
                if tracker_fn is not None:
                    tracker_fn({
                        "learning rate": current_lr,
                        "loss": current_loss,
                        "gradient norm": current_gnorm,
                        "token seen": total_tokens_seen,
                        "current throughput (token per gpu per sec)": current_throughput,
                        "overall throughput (token per gpu per sec)": overall_throughput,
                        "gpu reserved memory": reserved_mem,
                        "gpu allocated memory": allocated_mem,
                        **z_report,
                    }, step=batch_idx)
            start = time.time()
            if is_cuda:
                ev0.record()
            ddp_stats.zero_()
            for t_ in (moe_aux, z_sum, router_z_sum):
                if t_ is not None:
                    t_.zero_()
        if is_cuda:
            torch.cuda.reset_peak_memory_stats(device)

        if batch_idx % cfg.checkpoint_interval == 0 or batch_idx == cfg.num_steps:
            checkpointer.save(batch_idx, model, optimizer, None, tokens_seen=tokens_seen + new_tokens_seen)

    return train_loss
