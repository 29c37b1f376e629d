"""Training configuration.

One flat dataclass; every field is a ``--field=value`` CLI flag of the entry
points (parity with the reference's ``fms_fsdp/config/training.py:5-74``).
Field names and defaults follow the reference so existing launch scripts keep
working; the block at the bottom holds the engine-specific extension knobs
(SURVEY.md App. B "new knobs"), whose defaults preserve reference behaviour.
"""
from dataclasses import dataclass, field
from typing import Optional, Union

_DEFAULT_CORPORA = ",".join(
    "lang=%s/dataset=%s" % pair
    for pair in (
        ("en", "commoncrawl"), ("en", "webhose"), ("en", "github_clean"),
        ("de", "wikipedia"), ("es", "wikipedia"), ("fr", "wikipedia"),
        ("ja", "wikipedia"), ("pt", "wikipedia"), ("en", "wikimedia"),
        ("en", "uspto"), ("en", "pubmedcentral"), ("en", "arxiv"),
        ("en", "stackexchange"),
    )
)


@dataclass
class train_config:
    # ---- which model, where checkpoints live
    """Reference: ``fms_fsdp/config/training.py:6-74``."""
    model_variant: str = "7b"                         # key of utils.config_utils.get_model_config (e.g. llama2_7b, mamba_9.8b)
    ckpt_load_path: str = "/fsx/output/ckpt"          # where to look for a checkpoint to start from (the save dir wins if it has one)
    ckpt_save_path: str = "/fsx/output/ckpt"          # step_<N>_ckp/ directories are written under <this>/checkpoints

    # ---- data
    use_dummy_dataset: bool = False                   # synthetic arange stream instead of the arrow/parquet loader (benchmarks)
    data_path: str = "/fsx/data"                      # root of the dataset tree: <data_path>/<dataset>/...shards
    file_type: str = "arrow"                          # arrow | hf_parquet | auto
    col_name: str = "tokens"                          # column holding the token ids (or text for hf_parquet)
    tokenizer_path: str = "/fsx/tokenizer"            # HF tokenizer, only needed when the loader tokenises (parquet text)
    datasets: str = _DEFAULT_CORPORA
    weights: str = "7725,500,550,28,17,22,25,8,100,500,175,250,100"  # sampling weights, one per entry of `datasets`
    seq_length: int = 4096                            # tokens per training sequence
    vocab_size: int = 32000                           # used by the dummy stream and sanity checks
    bos_token: Optional[int] = None                   # prepended to every document when set
    eos_token: int = 0                                # document delimiter appended by the loader
    bol_token: Optional[int] = None                   # optional begin-of-line marker inserted by the packer
    eol_token: Optional[int] = None                   # optional end-of-line marker inserted by the packer
    strip_tokens: str = ""                            # comma-separated token ids dropped from document ends
    logical_shards: int = 1024                        # fixed number of logical data shards (rescalable over world sizes dividing it)
    num_workers: int = 1                              # DataLoader worker processes per rank

    # ---- sharding policies
    sharding_strategy: str = "hsdp"          # fsdp | hsdp | ddp  (anything else -> fsdp)
    fsdp_activation_checkpointing: bool = False       # recompute block activations in backward
    selective_checkpointing: Union[float, str] = 1   # fraction of blocks to recompute, e.g. 0.5 or "1/3"
    mixed_precision: bool = True                      # bf16 compute / bf16 reduce, fp32 master weights
    low_cpu_fsdp: bool = False                        # build on the meta device and initialise shards in place

    # ---- optimisation
    batch_size: int = 2                               # sequences per GPU per step
    num_steps: int = 1000000                          # total optimizer steps of the schedule
    training_stage: str = "initial"          # initial | annealing
    learning_rate: float = 3e-4                       # peak LR (warmup 2000 steps, cosine to 10 %)
    grad_clip_thresh: float = 1.0                     # global gradient-norm clip
    seed: int = 2023                                  # torch / cuda / numpy seed

    # ---- continued training
    resuming_dataset: bool = False                    # load only the loader state from ckpt_load_path (new model, same data position)

    # ---- profiling
    use_profiler: bool = False                        # torch.profiler schedule around steps 1-3, traces under profile_traces/
    profiler_rank0_only: bool = True                  # profile rank 0 only

    # ---- reporting
    report_interval: int = 100                        # steps between stdout / tracker reports
    checkpoint_interval: int = 10000                  # steps between checkpoints
    tracker: Optional[str] = None            # None | "wandb" | "aim"
    tracker_dir: str = "/fsx/aim_logs/llama"          # aim repo / wandb dir
    tracker_project_name: str = "llama"
    tracker_run_id: Optional[str] = None

    # ---- graph capture.  The reference used torch.compile here; this engine has no tracing
    # compiler: the flag is accepted for CLI compatibility and selects the fused-kernel path.
    use_torch_compile: bool = True                    # accepted for CLI compatibility; this engine has no tracing compiler

    # ---- speculator training
    tp_size: int = 8                                  # speculator: tensor-parallel degree of the frozen base model
    model_arch: str = "embedllama"                    # speculator: embedllama | embedgpt_bigcode | embedmixtral
    model_path: str = "/path/to/model/"               # speculator: HF / FMS checkpoint of the frozen base model
    n_speculator_heads: int = 3                       # speculator: number of lookahead heads
    speculator_width: int = 4096                      # speculator: inner width of the MLP heads
    speculator_tie_weights: bool = True               # speculator: share embeddings / projections across heads
    speculator_scale_input: bool = True               # speculator: layer-norm the base hidden state first
    stage2_start_step: int = 15000                    # speculator: step at which training switches to generated continuations
    stage2_prompt_length: int = 64                    # speculator stage 2: prompt tokens taken from the data
    stage2_batch_size: int = 96                       # speculator stage 2: generation batch
    stage2_seq_length: int = 256                      # speculator stage 2: generated tokens per prompt

    # ---- engine extensions (not in the reference; defaults keep reference semantics)
    comm_backend: str = "auto"               # auto | nccl | gloo
    collective_impl: str = "auto"            # auto | fused (NVLink peer kernels) | torch (c10d collectives)
    hsdp_shard_size: int = 0                 # 0 = local device count (reference behaviour); 4 -> 2x4 on one box
    kernel_path: str = "auto"                # auto | fused (sm_90a kernels) | torch (ATen oracle)
    precision: str = "bf16"                  # bf16 | fp8 (opt-in: row-wise scaled e4m3 forward GEMMs, bf16 backward)
    prefetch_depth: int = 2                  # gathered-unit buffers in flight (reference limiter = 2)
    fused_cross_entropy: bool = True         # linear+CE without materialising logits
    fault_inject_step: int = 0               # >0: rank 1 exits at that step (resume drill)
    nonfinite_action: str = "warn"           # NaN/Inf loss or grad norm at a report step: warn | halt (restart + auto-resume)
    loss_readback: bool = True               # every step: async 4-byte D2H of the loss into pinned memory, checked one step later
    poison_released_params: bool = False     # debug: NaN-fill a unit's gathered parameters on release (use-after-free trap)
    grad_dtype: str = "bf16"                 # dtype of the unsharded gradient buffer (reference reduce_dtype=bf16)
    document_attention_mask: bool = False    # Llama: attention stops at eos_token in packed lines (RoPE positions are not reset)
    qk_norm: bool = False                    # Llama: per-head RMSNorm of q and k before RoPE (Qwen3 QK-norm), for any variant
    grad_accum_steps: int = 1                # micro-batches per optimizer step (global batch = world x batch_size x this)
