"""Mamba2-hybrid pre-training entry point (CLI parity with reference ``main_training_mamba.py:28-175``).

Same skeleton as ``main_training_llama.py``; the model is ``MambaLMHeadModel(MambaConfig(**get_model_config(
variant)))`` (``mamba_9.8b`` from the reference zoo, ``mamba_2.8b`` for the BASELINE config), the shard unit is the
mamba ``Block``, and the output carries ``.logits`` on the reference-style path.
"""
import os

import torch
import torch.distributed as dist
from torch.optim.lr_scheduler import LambdaLR

from fms_fsdp_b200 import config
from fms_fsdp_b200.models.mamba import Block, MambaConfig, MambaLMHeadModel
from fms_fsdp_b200.ops import set_kernel_path
from fms_fsdp_b200.parallel import ShardedAdamW, ShardedModel
from fms_fsdp_b200.utils.checkpointing_utils import Checkpointer, resolve_load_path
from fms_fsdp_b200.utils.cli import run
from fms_fsdp_b200.utils.config_utils import get_model_config, update_config
from fms_fsdp_b200.utils.dataloader_utils import get_data_loader, get_dummy_loader
from fms_fsdp_b200.utils.train_utils import (get_policies, get_profiler, lr_schedule_fn, setup, setup_environ_flags,
                                             torchrun_env, train)


def main(**kwargs):
    cfg = config.train_config()
    update_config(cfg, **kwargs)
    if cfg.document_attention_mask:
        raise ValueError("--document_attention_mask is not supported for Mamba models: the SSD scan and the causal "
                         "conv1d carry state across document boundaries, so masking only the attention layers "
                         "would not isolate documents")
    if cfg.qk_norm:
        raise ValueError("--qk_norm is not supported for Mamba models: their attention layers have no q / k norm "
                         "weights, and the option would silently change nothing")
    if cfg.moe_router_z_loss_coef:
        raise ValueError("--moe_router_z_loss_coef is not supported for Mamba models: they have no mixture-of-experts "
                         "router")

    use_cuda = torch.cuda.is_available() and cfg.comm_backend != "gloo"
    if use_cuda:
        torch.cuda.manual_seed(cfg.seed)
    torch.manual_seed(cfg.seed)

    local_rank, rank, world_size = torchrun_env()
    if rank == 0:
        print(f"--> running with these configs {cfg}")

    if world_size > 1 or "RANK" in os.environ:
        setup(cfg=cfg)
    if use_cuda:
        torch.cuda.set_device(local_rank)
        torch.cuda.empty_cache()
    device = torch.device("cuda", local_rank) if use_cuda else torch.device("cpu")
    setup_environ_flags()
    if cfg.kernel_path != "auto":
        set_kernel_path(cfg.kernel_path)

    block = Block
    (mixed_precision_policy, wrapping_policy, sharding_strategy_policy, apply_selective_ac,
     param_init_fn) = get_policies(cfg, rank, block)

    config_data = get_model_config(cfg.model_variant)
    mamba_config = MambaConfig(**config_data)
    if use_cuda or cfg.low_cpu_fsdp:
        with torch.device("meta"):
            model = MambaLMHeadModel(mamba_config)
    else:
        model = MambaLMHeadModel(mamba_config)
        model.reset_parameters()
    model.z_loss_coef = float(cfg.z_loss_coef)

    if rank == 0:
        total_params = sum(p.numel() for p in model.parameters() if p.requires_grad)
        print(f"\n--> model has {total_params / 1e6} Million params\n")

    if rank == 0:
        print("Constructing datasets...")
    if not cfg.use_dummy_dataset:
        train_loader = get_data_loader(cfg, rank, world_size)
    else:
        train_loader = get_dummy_loader(cfg, rank, world_size)
    if rank == 0:
        print("Datasets constructed!")

    if cfg.fsdp_activation_checkpointing:
        if rank == 0:
            print("--> applying FSDP activation checkpointing...")
        apply_selective_ac(model, p=cfg.selective_checkpointing)

    model = ShardedModel(
        model,
        sharding_strategy=sharding_strategy_policy,
        hsdp_shard_size=cfg.hsdp_shard_size,
        mixed_precision=mixed_precision_policy,
        device=device,
        collective_impl=cfg.collective_impl,
        prefetch_depth=cfg.prefetch_depth,
        param_init_fn=param_init_fn,
        auto_wrap_policy=wrapping_policy,
        local_world=(torch.cuda.device_count() if use_cuda else None),
        grad_accum_steps=cfg.grad_accum_steps,
    )
    model.poison_released_params = bool(cfg.poison_released_params) or model.poison_released_params
    if rank == 0:
        print(f"--> sharded runtime: {model.extra_repr()}")

    optimizer = ShardedAdamW(model, lr=cfg.learning_rate, betas=(0.9, 0.95), weight_decay=0.1)

    checkpointer = Checkpointer(cfg.ckpt_save_path, 1000, sharding_strategy_policy, rank, local_rank)
    model, optimizer, _, start_step, tokens_seen, is_resuming = checkpointer.load(
        model, optimizer, None,
        path=resolve_load_path(cfg.ckpt_load_path),
        strict=False,
    )
    if not is_resuming:
        start_step = 0
        for g in optimizer.param_groups:
            g["initial_lr"] = cfg.learning_rate

    schedule = lr_schedule_fn(cfg)
    scheduler = LambdaLR(optimizer, lambda x: schedule(x + start_step))
    profiler = get_profiler(cfg, rank)

    if rank == 0:
        print(f"Training for {cfg.num_steps} steps")
    train(cfg, model, local_rank, rank, train_loader, optimizer, scheduler, profiler, checkpointer, start_step,
          tokens_seen)

    if dist.is_initialized():
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    run(main)
