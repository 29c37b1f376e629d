"""LLaMA for the engine.

State-dict names, fused-weight layout, initialisation and numerics contract follow the
ibm-fms LLaMA that the reference trains (SURVEY.md §2.4 E2; names evidenced by reference
``fms_to_hf_llama.py:54-128``): ``shared.emb/head``, ``layers.N.{ln, attn.in_proj.qkv_fused,
attn.dense, ff_ln, ff_sub_layer.wg1_fused, ff_sub_layer.w2}``, ``dec_norm``; RoPE in the
interleaved-pair convention; RMSNorm in fp32; SwiGLU on ``[gate | up]``.

The architecture is *not* a module-per-op graph: each block is one straight-line sequence of
engine ops (``fms_fsdp_b200.ops``) that run as sm_90a kernels on GPU, and the model exposes
``engine_units()`` so the sharded runtime can schedule gather / compute / reduce per unit.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import List, Optional

import torch
import torch.nn as nn

from fms_fsdp_b200 import ops
from fms_fsdp_b200.ops import torch_kernels


@dataclass
class LLaMAConfig:
    src_vocab_size: int = 32000
    emb_dim: int = 4096
    norm_eps: float = 1e-5
    nheads: int = 32
    kvheads: int = 0
    nlayers: int = 32
    pad_id: int = -1
    hidden_grow_factor: float = 8 / 3
    multiple_of: int = 256
    activation_fn: str = "swish"
    p_dropout: float = 0.0
    max_expected_seq_len: int = 4096
    ntk_scaling: bool = False
    attn_bias: bool = False
    mlp_bias: bool = False
    tie_heads: bool = False
    rope_theta: float = 10000.0
    linear_config: Optional[dict] = None
    fused_weights: bool = True
    # extension (not an fms field): HF-style frequency rescaling of long-context checkpoints, e.g. Llama 3.1
    # {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0, "original_max_position_embeddings": 8192}
    rope_scaling: Optional[dict] = None
    # extension (not an fms field): token id that ends a document in packed rows (the loader's eos_token).  When set,
    # attention is masked at document boundaries.  RoPE positions stay absolute: rotary scores depend only on position
    # differences, so a document in the middle of a row attends exactly as it would from position 0.
    doc_separator: Optional[int] = None
    # extension (not an fms field): QK-norm (Qwen3) -- a per-head RMSNorm of q and k (weights ``attn.q_norm`` /
    # ``attn.k_norm`` [head_dim], eps ``norm_eps``) after the projection and before RoPE.
    qk_norm: bool = False
    # extension (not an fms field): head dimension when it is not emb_dim // nheads (Qwen3-0.6B / 4B: 128 with
    # emb_dim / nheads = 64 / 80).  None = emb_dim // nheads.
    attn_head_dim: Optional[int] = None
    # extension (not an fms field): q / k / v projection biases (Qwen2 / Qwen2.5) -- ``attn.in_proj.qkv_fused.bias``
    # [(nheads + 2 kv_heads) * head_dim], added before RoPE.  Unlike fms's ``attn_bias`` the output projection stays
    # bias-free.
    qkv_bias: bool = False
    # extension (not an fms field): sparse mixture-of-experts feed-forward (Qwen3-MoE, Mixtral).  moe_num_experts > 0
    # replaces every block's ``ff_sub_layer`` with ``moe``: router ``moe.gate.weight`` [E, D] and SwiGLU experts
    # ``moe.w1`` [E, 2F, D] ([gate | up] per expert) and ``moe.w2`` [E, D, F], F = moe_hidden_dim.  Each token goes to
    # its moe_top_k experts (dropless), weighted by their router probabilities, renormalised when moe_norm_topk.
    # moe_aux_loss_coef scales the Switch load-balancing loss coef * mean_layers(E * sum_e f_e * P_e), computed per layer
    # (HF instead concatenates all layers' router logits before taking the means).
    moe_num_experts: int = 0
    moe_top_k: int = 2
    moe_hidden_dim: int = 0
    moe_norm_topk: bool = True
    moe_aux_loss_coef: float = 0.0

    @property
    def hidden_dim(self) -> int:
        return self.multiple_of * ((int(self.hidden_grow_factor * self.emb_dim) + self.multiple_of - 1)
                                   // self.multiple_of)

    def inactive_params(self) -> int:
        """Expert parameters a token does not use: (E - k) experts per block (0 for a dense model).  Model FLOPs per
        token count the active parameters only."""
        if self.moe_num_experts <= 0:
            return 0
        return self.nlayers * (self.moe_num_experts - self.moe_top_k) * 3 * self.emb_dim * self.moe_hidden_dim

    @property
    def kv_heads(self) -> int:
        return self.nheads if self.kvheads == 0 else self.kvheads

    @property
    def head_dim(self) -> int:
        return self.attn_head_dim if self.attn_head_dim else self.emb_dim // self.nheads


class _Weight(nn.Module):
    """A bias-free linear weight holder: keeps FMS's ``<name>.weight`` state-dict key."""

    def __init__(self, out_features: int, in_features: int, device=None, dtype=None):
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        self.weight = nn.Parameter(torch.empty(out_features, in_features, device=device, dtype=dtype))

    def forward(self, x, residual=None):
        return ops.linear(x, self.weight, residual)


class RMSNorm(nn.Module):
    """FMS LayerNormParameterized(use_mean=False, elementwise_scale=True, no shift)."""

    def __init__(self, dim: int, eps: float, device=None, dtype=None):
        super().__init__()
        self.eps = eps
        self.weight = nn.Parameter(torch.empty(dim, device=device, dtype=dtype))

    def reset_parameters(self):
        nn.init.ones_(self.weight)

    def forward(self, x):
        return ops.rmsnorm(x, self.weight, self.eps)

    def fork(self, x):
        """(norm(x), x) with the residual-branch gradient folded into the norm's backward kernel."""
        return ops.rmsnorm_fork(x, self.weight, self.eps)


class RotaryEmbedding(nn.Module):
    """cos/sin table cache; attrs mirror what the reference exporter reads
    (``dim, ratio, max_seq_len, ntk_scaling, _alpha``: reference ``fms_to_hf_llama.py:43-51``)."""

    def __init__(self, dim: int, ratio: float = 10000.0, max_seq_len: int = 2048, ntk_scaling: bool = False, scaling=None):
        super().__init__()
        self.dim, self.ratio, self.max_seq_len, self.ntk_scaling = dim, ratio, max_seq_len, ntk_scaling
        self.scaling = dict(scaling) if scaling else None
        self._tables = {}

    def _alpha(self, seq_len) -> int:
        if not self.ntk_scaling:
            return 1
        return max(1, 2 ** math.ceil(math.log2(max(seq_len / self.max_seq_len, 1))))

    def compute_freqs_cis(self, device, max_seq_len: int = 2048):
        """Precompute (and cache per device) the [S, dim/2, 2] cos/sin table (reference
        ``main_training_llama.py:93-96`` calls this after wrapping)."""
        alpha = self._alpha(max_seq_len)
        key = (str(device), alpha)
        tab = self._tables.get(key)
        if tab is None or tab.shape[0] < max_seq_len:
            n = max(max_seq_len, self.max_seq_len * alpha)
            tab = torch_kernels.rope_table(n, self.dim, self.ratio, float(alpha), device=device, scaling=self.scaling)
            self._tables[key] = tab
        return tab

    def table(self, device, seq_len):
        return self.compute_freqs_cis(device, seq_len)


class _InProj(nn.Module):
    def __init__(self, cfg: LLaMAConfig, device=None, dtype=None):
        super().__init__()
        hd = cfg.head_dim
        self.splits = [cfg.nheads * hd, cfg.kv_heads * hd, cfg.kv_heads * hd]
        self.qkv_fused = _Weight(sum(self.splits), cfg.emb_dim, device, dtype)
        if cfg.qkv_bias:   # q / k sections in the interleaved RoPE pair order of the weight's rows
            self.qkv_fused.bias = nn.Parameter(torch.empty(sum(self.splits), device=device, dtype=dtype))


class MultiHeadAttention(nn.Module):
    def __init__(self, cfg: LLaMAConfig, device=None, dtype=None):
        super().__init__()
        self.nheads, self.kvheads, self.head_dim = cfg.nheads, cfg.kv_heads, cfg.head_dim
        self.emb_dim = cfg.emb_dim
        self.in_proj = _InProj(cfg, device, dtype)
        self.dense = _Weight(cfg.emb_dim, cfg.nheads * cfg.head_dim, device, dtype)
        self.qk_norm = bool(cfg.qk_norm)
        if self.qk_norm:   # per-head gains, indexed by position within a head (interleaved RoPE pair order)
            self.q_norm = RMSNorm(cfg.head_dim, cfg.norm_eps, device, dtype)
            self.k_norm = RMSNorm(cfg.head_dim, cfg.norm_eps, device, dtype)
        self.qkv_bias = bool(cfg.qkv_bias)

    def reset_parameters(self):
        for w in (self.in_proj.qkv_fused.weight, self.dense.weight):
            nn.init.trunc_normal_(w, mean=0.0, std=0.02)
        if self.qk_norm:
            self.q_norm.reset_parameters()
            self.k_norm.reset_parameters()
        if self.qkv_bias:
            nn.init.zeros_(self.in_proj.qkv_fused.bias)

    def qk_norm_args(self):
        """``ops.qkv_attention(qk_norm=...)``: None without QK-norm."""
        return (self.q_norm.weight, self.k_norm.weight, self.q_norm.eps) if self.qk_norm else None

    def qkv_bias_arg(self):
        """``ops.qkv_attention(qkv_bias=...)``: None without projection biases."""
        return self.in_proj.qkv_fused.bias if self.qkv_bias else None


class GatedLinearUnit(nn.Module):
    def __init__(self, cfg: LLaMAConfig, device=None, dtype=None):
        super().__init__()
        self.hidden_dim = cfg.hidden_dim
        self.wg1_fused = _Weight(2 * cfg.hidden_dim, cfg.emb_dim, device, dtype)
        self.w2 = _Weight(cfg.emb_dim, cfg.hidden_dim, device, dtype)

    def reset_parameters(self):
        for w in (self.wg1_fused.weight, self.w2.weight):
            nn.init.trunc_normal_(w, mean=0.0, std=0.02)


class MoEFeedForward(nn.Module):
    """Router + SwiGLU experts; the weights of all experts are single tensors (``ops.moe_mlp``)."""

    def __init__(self, cfg: LLaMAConfig, device=None, dtype=None):
        super().__init__()
        E, F, D = cfg.moe_num_experts, cfg.moe_hidden_dim, cfg.emb_dim
        self.config = cfg
        self.gate = _Weight(E, D, device, dtype)
        self.w1 = nn.Parameter(torch.empty(E, 2 * F, D, device=device, dtype=dtype))
        self.w2 = nn.Parameter(torch.empty(E, D, F, device=device, dtype=dtype))
        self.last_aux = None          # the load-balancing statistic of the last forward (device scalar)

    def reset_parameters(self):
        for w in (self.gate.weight, self.w1, self.w2):
            nn.init.trunc_normal_(w, mean=0.0, std=0.02)

    def forward(self, h, residual):
        cfg = self.config
        # the loss is the mean over layers: each block's share of the coefficient (read here, so that the gradient and
        # LLaMA.moe_aux_loss() always use the same value)
        y, self.last_aux = ops.moe_mlp(h, self.gate.weight, self.w1, self.w2, cfg.moe_top_k, cfg.moe_norm_topk,
                                       cfg.moe_aux_loss_coef / cfg.nlayers, residual=residual)
        return y


class WordEmbedding(nn.Module):
    """Embedding + reversible (untied unless tie_heads) output head: ``shared.emb`` / ``shared.head``."""

    def __init__(self, cfg: LLaMAConfig, device=None, dtype=None):
        super().__init__()
        self.vocab_size, self.emb_dim, self.tie_weights = cfg.src_vocab_size, cfg.emb_dim, cfg.tie_heads
        self.padding_idx = cfg.pad_id if cfg.pad_id >= 0 else None
        self.emb = nn.Embedding(cfg.src_vocab_size, cfg.emb_dim, device=device, dtype=dtype)
        self.head = _Weight(cfg.src_vocab_size, cfg.emb_dim, device, dtype)
        if self.tie_weights:
            self.head.weight = self.emb.weight

    def reset_parameters(self):
        nn.init.trunc_normal_(self.emb.weight, mean=0.0, std=self.emb_dim ** -0.5)
        if not self.tie_weights:
            nn.init.trunc_normal_(self.head.weight, mean=0.0, std=self.emb_dim ** -0.5)
        if self.padding_idx is not None:
            with torch.no_grad():
                self.emb.weight[self.padding_idx].zero_()

    def forward(self, x, reverse: bool = False):
        if reverse:
            return ops.linear(x, self.head.weight)
        return ops.embedding(x, self.emb.weight)


class LLaMABlock(nn.Module):
    """ln -> fused QKV -> RoPE -> causal flash attention -> dense(+res) -> ff_ln -> gate/up -> SwiGLU
    -> w2(+res).  Hot-op inventory K1-K8 of SURVEY.md §2.5(a)."""

    def __init__(self, cfg: LLaMAConfig, rot_emb: RotaryEmbedding, device=None, dtype=None):
        super().__init__()
        self.config = cfg
        self.ln = RMSNorm(cfg.emb_dim, cfg.norm_eps, device, dtype)
        self.ff_ln = RMSNorm(cfg.emb_dim, cfg.norm_eps, device, dtype)
        self.attn = MultiHeadAttention(cfg, device, dtype)
        if cfg.moe_num_experts > 0:
            self.moe = MoEFeedForward(cfg, device, dtype)
        else:
            self.ff_sub_layer = GatedLinearUnit(cfg, device, dtype)
        object.__setattr__(self, "_rot", rot_emb)  # shared, not a submodule (no params, not in state dict)

    def forward(self, x, doc=None):
        """``doc``: the ``ops.document_segments`` table of a packed batch; given one, the block returns ``(x, doc)``
        so the table travels with the hidden state from block to block."""
        a, cfg = self.attn, self.config
        B, S, _ = x.shape
        h, x = self.ln.fork(x)
        # projection + RoPE + attention: one node, RoPE fused into the GEMM / dq-dk epilogues
        ctx = ops.qkv_attention(h, a.in_proj.qkv_fused.weight, self._rot.table(x.device, S), a.nheads, a.kvheads,
                                a.head_dim, doc=doc, qk_norm=a.qk_norm_args(), qkv_bias=a.qkv_bias_arg())
        x = a.dense(ctx, residual=x)
        h, x = self.ff_ln.fork(x)
        if cfg.moe_num_experts > 0:
            x = self.moe(h, x)
            return x if doc is None else (x, doc)
        ff = self.ff_sub_layer
        # gate/up GEMM with the SwiGLU epilogue, down projection with the residual epilogue: one autograd node
        x = ops.gated_mlp(h, ff.wg1_fused.weight, ff.w2.weight, residual=x)
        return x if doc is None else (x, doc)


class LLaMA(nn.Module):
    def __init__(self, config: Optional[LLaMAConfig] = None, device=None, dtype=None, **kwargs):
        super().__init__()
        self.config = config if config is not None else LLaMAConfig()
        for k, v in kwargs.items():
            setattr(self.config, k, v)
        cfg = self.config
        self.width = cfg.emb_dim
        self.pad_id = cfg.pad_id
        self.max_expected_seq_len = cfg.max_expected_seq_len
        self.shared = WordEmbedding(cfg, device, dtype)
        self.rot_emb = RotaryEmbedding(cfg.head_dim, cfg.rope_theta, cfg.max_expected_seq_len, cfg.ntk_scaling,
                                       getattr(cfg, "rope_scaling", None))
        self.layers = nn.ModuleList([LLaMABlock(cfg, self.rot_emb, device, dtype) for _ in range(cfg.nlayers)])
        self.dec_norm = RMSNorm(cfg.emb_dim, cfg.norm_eps, device, dtype)

    def get_config(self) -> LLaMAConfig:
        return self.config

    def moe_aux_loss(self):
        """coef * mean over layers of the load-balancing statistic of the last forward, as a device scalar (its
        gradient is already part of the backward); None for a dense model or before the first forward."""
        if self.config.moe_num_experts <= 0 or self.layers[0].moe.last_aux is None:
            return None
        return torch.stack([blk.moe.last_aux for blk in self.layers]).mean() * self.config.moe_aux_loss_coef

    def reset_parameters(self):
        self.shared.reset_parameters()
        self.dec_norm.reset_parameters()
        for blk in self.layers:
            blk.ln.reset_parameters()
            blk.ff_ln.reset_parameters()
            blk.attn.reset_parameters()
            (blk.moe if self.config.moe_num_experts > 0 else blk.ff_sub_layer).reset_parameters()

    # ---- plain (unsharded) forward: logits, as the reference model returns
    def forward(self, x, labels=None, return_hidden: bool = False):
        h = self.shared(x)
        if self.config.doc_separator is None:
            for blk in self.layers:
                h = blk(h)
        else:
            state = (h, ops.document_segments(x, self.config.doc_separator))
            for blk in self.layers:
                state = blk(*state)
            h = state[0]
        h = self.dec_norm(h)
        if return_hidden:
            return h
        if labels is not None:
            return ops.linear_cross_entropy(h, self.shared.head.weight, labels)
        return self.shared(h, reverse=True)

    # ---- sharded-runtime protocol -------------------------------------------------------------
    def engine_units(self):
        """(blocks, root_modules): one shard unit per block; embedding+head+final norm form the root
        unit (reference wrapping policy, ``policies/wrapping.py:6-14``)."""
        return list(self.layers), [self.shared, self.dec_norm]

    def engine_embed(self, tokens):
        h = self.shared(tokens)
        if self.config.doc_separator is None:
            return h
        return h, ops.document_segments(tokens, self.config.doc_separator)

    def engine_head(self, h, *args, **kwargs):
        """``engine_head(h, labels=None, ignore_index=-100)``; with ``doc_separator`` set the engine's state is
        ``(h, seg)`` and the document table that follows ``h`` is ignored here."""
        if self.config.doc_separator is not None:
            args = args[1:]
        return self._head(h, *args, **kwargs)

    def _head(self, h, labels=None, ignore_index=-100):
        h = self.dec_norm(h)
        if labels is None:
            return self.shared(h, reverse=True)
        return ops.linear_cross_entropy(h, self.shared.head.weight, labels, ignore_index)


def param_count(model: nn.Module) -> int:
    return sum(p.numel() for p in model.parameters())
