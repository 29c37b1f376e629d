"""Llama pre-training entry point (CLI parity with reference ``main_training_llama.py:25-175``):

    torchrun --nproc_per_node=8 main_training_llama.py --model_variant=llama2_7b --use_dummy_dataset=True \
        --sharding_strategy=fsdp --num_steps=100 --report_interval=10

Every ``train_config`` field is a ``--field=value`` flag.  Same flow as the reference -- config, seeds,
process group, policies, model (optionally on the meta device), data loader, sharded wrap, RoPE table
precompute, selective recomputation, AdamW(0.9, 0.95, wd 0.1), checkpoint auto-resume, LR schedule,
profiler, train -- on the H100-native engine instead of torch FSDP + torch.compile.
"""
import os

import torch
import torch.distributed as dist
from torch.optim.lr_scheduler import LambdaLR

from fms_fsdp_b200 import config
from fms_fsdp_b200.models.llama import LLaMA, LLaMABlock
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

    block = LLaMABlock
    (mixed_precision_policy, wrapping_policy, sharding_strategy_policy, apply_selective_ac,
     param_init_fn) = get_policies(cfg, rank, block)

    llama_config = get_model_config(cfg.model_variant)
    if cfg.document_attention_mask:
        # packed lines hold several documents, each ended by the loader's eos_token: attend within a document only
        llama_config.doc_separator = cfg.eos_token
    if cfg.qk_norm:
        # per-head RMSNorm of q and k before RoPE (the qwen3_* variants have it already)
        llama_config.qk_norm = True
    if llama_config.moe_num_experts > 0:
        if cfg.precision == "fp8":
            raise ValueError("--precision fp8 is not supported with a mixture-of-experts variant: the grouped expert "
                             "GEMMs are bf16 only")
        if cfg.moe_aux_loss_coef is not None:
            llama_config.moe_aux_loss_coef = float(cfg.moe_aux_loss_coef)
    if cfg.low_cpu_fsdp or use_cuda:
        # one unit at a time is materialised directly on the device by the sharded runtime
        with torch.device("meta"):
            model = LLaMA(llama_config)
    else:
        model = LLaMA(llama_config)
        model.reset_parameters()

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

    # selective recomputation is a property of the blocks; flag them before the runtime takes over
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
    model.module.rot_emb.compute_freqs_cis(device, model.module.config.max_expected_seq_len)
    if rank == 0:
        print(f"--> sharded runtime: {model.extra_repr()}")
        if cfg.use_torch_compile:
            print("--> use_torch_compile is accepted for compatibility; this engine runs hand-written fused "
                  "sm_90a kernels and has no tracing compiler")

    optimizer = ShardedAdamW(model, lr=cfg.learning_rate, betas=(0.9, 0.95), weight_decay=0.1)

    checkpointer = Checkpointer(cfg.ckpt_save_path, 1000, sharding_strategy_policy, rank, local_rank)
    model, optimizer, _, start_step, tokens_seen, is_resuming = checkpointer.load(
        model, optimizer, None,
        path=resolve_load_path(cfg.ckpt_load_path),
        strict=False,
    )
    if not is_resuming:
        start_step = 0
        for g in optimizer.param_groups:  # loaded hyper-parameters yield to the current run's
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
