"""Mamba2-hybrid language model for the engine.

Stands in for what the reference imports from ``mamba_ssm`` (``MambaConfig``, ``MambaLMHeadModel``,
``Block``, ``Mamba2``, ``MHA``, ``GatedMLP`` -- reference ``main_training_mamba.py:8-10,55,65-67``;
SURVEY.md §2.4 E3, §2.5(b)).  State-dict names follow mamba_ssm (``backbone.embedding``,
``backbone.layers.N.{norm,mixer,norm2,mlp}``, ``backbone.norm_f``, ``lm_head``) so
``fms_to_hf_mamba`` emits the familiar ``config.json`` + ``pytorch_model.bin``.

Every block is a straight line of engine ops (``fms_fsdp_b200.ops``): wgmma GEMMs for
in/out projections and the gated MLP, fused causal-conv1d+SiLU, the SSD chunked scan, gated
RMSNorm, the fp32 residual stream with fused add+norm, and -- for the attention layers of the
hybrid -- the same wgmma flash attention as Llama with partial (half-split) rotary.
"""
from __future__ import annotations

import math
from collections import namedtuple
from dataclasses import dataclass, field
from typing import List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from fms_fsdp_b200 import ops
from fms_fsdp_b200.ops import torch_kernels
from fms_fsdp_b200.ops.functional import _deliver_wgrad, _put_fp32

CausalLMOutput = namedtuple("CausalLMOutput", ["logits"])


@dataclass
class MambaConfig:
    d_model: int = 2560
    d_intermediate: int = 0
    n_layer: int = 64
    vocab_size: int = 50277
    ssm_cfg: dict = field(default_factory=dict)
    attn_layer_idx: list = field(default_factory=list)
    attn_cfg: dict = field(default_factory=dict)
    rms_norm: bool = True
    residual_in_fp32: bool = True
    fused_add_norm: bool = True
    pad_vocab_size_multiple: int = 8
    tie_embeddings: bool = True
    norm_epsilon: float = 1e-5

    @property
    def padded_vocab(self) -> int:
        m = self.pad_vocab_size_multiple
        return self.vocab_size if self.vocab_size % m == 0 else self.vocab_size + m - self.vocab_size % m

    # engine/bench helpers use Llama-style names
    @property
    def nlayers(self):
        return self.n_layer

    @property
    def emb_dim(self):
        return self.d_model


class _W(nn.Module):
    """bias-free linear weight holder (keeps ``<name>.weight`` keys)."""

    def __init__(self, out_features, in_features, device=None, dtype=None):
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        self.weight = nn.Parameter(torch.empty(out_features, in_features, device=device, dtype=dtype))

    def reset_parameters(self):
        nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))

    def forward(self, x, residual=None):
        return ops.linear(x, self.weight, residual)


class RMSNorm(nn.Module):
    def __init__(self, dim, eps=1e-5, device=None, dtype=None):
        super().__init__()
        self.eps = eps
        self.weight = nn.Parameter(torch.empty(dim, device=device, dtype=dtype))

    def reset_parameters(self):
        nn.init.ones_(self.weight)

    def forward(self, x):
        return ops.rmsnorm(x, self.weight, self.eps)


class RMSNormGated(RMSNorm):
    """y = rmsnorm_grouped(x * silu(z)) * w  (``norm_before_gate=False``)."""

    def __init__(self, dim, eps=1e-5, group_size=None, device=None, dtype=None):
        super().__init__(dim, eps, device, dtype)
        self.group_size = group_size or dim

    def forward(self, x, z):
        return ops.rmsnorm_gated(x, z, self.weight, self.eps, self.group_size)


class _Conv1dParams(nn.Module):
    """Depthwise conv parameters with nn.Conv1d's shapes/keys: weight [C, 1, K], bias [C]."""

    def __init__(self, channels, kernel, bias=True, device=None, dtype=None):
        super().__init__()
        self.channels, self.kernel = channels, kernel
        self.weight = nn.Parameter(torch.empty(channels, 1, kernel, device=device, dtype=dtype))
        self.bias = nn.Parameter(torch.empty(channels, device=device, dtype=dtype)) if bias else None

    def reset_parameters(self):
        nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))
        if self.bias is not None:
            bound = 1 / math.sqrt(self.kernel)
            nn.init.uniform_(self.bias, -bound, bound)


class Mamba2(nn.Module):
    def __init__(self, d_model, d_state=128, d_conv=4, expand=2, headdim=64, ngroups=1, A_init_range=(1, 16),
                 dt_min=0.001, dt_max=0.1, dt_init_floor=1e-4, chunk_size=256, conv_bias=True, layer_idx=None,
                 device=None, dtype=None, **_unused):
        super().__init__()
        self.d_model, self.d_state, self.d_conv, self.expand = d_model, d_state, d_conv, expand
        self.d_inner = expand * d_model
        self.headdim, self.ngroups, self.chunk_size = headdim, ngroups, chunk_size
        assert self.d_inner % headdim == 0
        self.nheads = self.d_inner // headdim
        self.A_init_range, self.dt_min, self.dt_max, self.dt_init_floor = A_init_range, dt_min, dt_max, dt_init_floor
        self.layer_idx = layer_idx
        d_in_proj = 2 * self.d_inner + 2 * ngroups * d_state + self.nheads
        self.conv_dim = self.d_inner + 2 * ngroups * d_state
        self.in_proj = _W(d_in_proj, d_model, device, dtype)
        self.conv1d = _Conv1dParams(self.conv_dim, d_conv, conv_bias, device, dtype)
        self.dt_bias = nn.Parameter(torch.empty(self.nheads, device=device, dtype=dtype))
        self.A_log = nn.Parameter(torch.empty(self.nheads, device=device, dtype=dtype))
        self.D = nn.Parameter(torch.empty(self.nheads, device=device, dtype=dtype))
        self.norm = RMSNormGated(self.d_inner, 1e-5, self.d_inner // ngroups, device, dtype)
        self.out_proj = _W(d_model, self.d_inner, device, dtype)

    def reset_parameters(self):
        self.in_proj.reset_parameters()
        self.out_proj.reset_parameters()
        self.conv1d.reset_parameters()
        self.norm.reset_parameters()
        with torch.no_grad():
            dt = torch.exp(torch.rand(self.nheads) * (math.log(self.dt_max) - math.log(self.dt_min))
                           + math.log(self.dt_min)).clamp(min=self.dt_init_floor)
            self.dt_bias.copy_(dt + torch.log(-torch.expm1(-dt)))  # inverse softplus
            self.A_log.copy_(torch.log(torch.empty(self.nheads).uniform_(*self.A_init_range)))
            self.D.fill_(1.0)

    def forward(self, u):
        B, S, _ = u.shape
        zxbcdt = self.in_proj(u).view(B * S, -1)
        z, xBC, dt = torch.split(zxbcdt, [self.d_inner, self.conv_dim, self.nheads], dim=-1)
        xBC = ops.causal_conv1d(xBC.contiguous(), self.conv1d.weight, self.conv1d.bias, S, True)
        x, Bm, Cm = torch.split(xBC, [self.d_inner, self.ngroups * self.d_state, self.ngroups * self.d_state], dim=-1)
        y = ops.ssd_scan(x.reshape(B * S, self.nheads, self.headdim), dt.contiguous(), _neg_exp(self.A_log),
                         Bm.reshape(B * S, self.ngroups, self.d_state), Cm.reshape(B * S, self.ngroups, self.d_state),
                         self.D, self.dt_bias, S, self.chunk_size)
        y = self.norm(y.reshape(B * S, self.d_inner), z.contiguous())
        return self.out_proj(y.view(B, S, self.d_inner))


def _neg_exp(A_log: nn.Parameter):
    return _NegExp.apply(A_log)


class _NegExp(torch.autograd.Function):
    @staticmethod
    def forward(ctx, A_log):
        data = A_log.data if isinstance(A_log, nn.Parameter) else A_log
        a = -torch.exp(data.float())
        ctx.save_for_backward(a)
        ctx.param = A_log
        return a

    @staticmethod
    def backward(ctx, dA):
        (a,) = ctx.saved_tensors
        g = dA * a  # d(-exp(x))/dx = -exp(x) = a
        return _deliver_wgrad(ctx.param, _put_fp32(g))


class _WB(nn.Module):
    """Linear parameter holder with a bias (``dt_proj`` of Mamba1: the bias goes into the scan as ``delta_bias``)."""

    def __init__(self, out_features, in_features, device=None, dtype=None):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(out_features, in_features, device=device, dtype=dtype))
        self.bias = nn.Parameter(torch.empty(out_features, device=device, dtype=dtype))


class Mamba1(nn.Module):
    """Mamba (v1) mixer, ``ssm_cfg = {"layer": "Mamba1"}`` -- mamba_ssm's default layer type: ``in_proj`` -> (x, z);
    causal depthwise conv + SiLU on x; ``x_proj`` -> (dt, B, C); ``dt_proj``; selective scan with per-channel state
    ``A = -exp(A_log)`` of width ``d_state``, skip ``D``, gate ``silu(z)``, ``delta = softplus(dt + dt_proj.bias)``; ``out_proj``.
    Parameter names are mamba_ssm's (and ``transformers.MambaForCausalLM``'s, against which the math is tested)."""

    def __init__(self, d_model, d_state=16, d_conv=4, expand=2, dt_rank="auto", dt_min=0.001, dt_max=0.1, dt_scale=1.0,
                 dt_init_floor=1e-4, conv_bias=True, layer_idx=None, device=None, dtype=None, **_unused):
        super().__init__()
        self.d_model, self.d_state, self.d_conv, self.expand = d_model, d_state, d_conv, expand
        self.d_inner = expand * d_model
        self.dt_rank = math.ceil(d_model / 16) if dt_rank == "auto" else int(dt_rank)
        self.dt_min, self.dt_max, self.dt_scale, self.dt_init_floor = dt_min, dt_max, dt_scale, dt_init_floor
        self.layer_idx = layer_idx
        self.in_proj = _W(2 * self.d_inner, d_model, device, dtype)
        self.conv1d = _Conv1dParams(self.d_inner, d_conv, conv_bias, device, dtype)
        self.x_proj = _W(self.dt_rank + 2 * d_state, self.d_inner, device, dtype)
        self.dt_proj = _WB(self.d_inner, self.dt_rank, device, dtype)
        self.A_log = nn.Parameter(torch.empty(self.d_inner, d_state, device=device, dtype=dtype))
        self.D = nn.Parameter(torch.empty(self.d_inner, device=device, dtype=dtype))
        self.out_proj = _W(d_model, self.d_inner, device, dtype)

    def reset_parameters(self):
        for m in (self.in_proj, self.x_proj, self.out_proj, self.conv1d):
            m.reset_parameters()
        with torch.no_grad():
            std = self.dt_rank ** -0.5 * self.dt_scale
            nn.init.uniform_(self.dt_proj.weight, -std, std)
            dt = torch.exp(torch.rand(self.d_inner) * (math.log(self.dt_max) - math.log(self.dt_min))
                           + math.log(self.dt_min)).clamp(min=self.dt_init_floor)
            self.dt_proj.bias.copy_(dt + torch.log(-torch.expm1(-dt)))            # inverse softplus
            self.A_log.copy_(torch.log(torch.arange(1, self.d_state + 1, dtype=torch.float32)).expand(self.d_inner, -1))
            self.D.fill_(1.0)

    def forward(self, u):
        B, S, _ = u.shape
        x, z = self.in_proj(u).view(B * S, -1).chunk(2, dim=-1)
        x = ops.causal_conv1d(x.contiguous(), self.conv1d.weight, self.conv1d.bias, S, True)
        dt, Bm, Cm = torch.split(ops.linear(x, self.x_proj.weight), [self.dt_rank, self.d_state, self.d_state], dim=-1)
        delta = ops.linear(dt.contiguous(), self.dt_proj.weight)
        y = ops.selective_scan(x, delta, _neg_exp(self.A_log), Bm.contiguous(), Cm.contiguous(), self.D, z.contiguous(),
                               self.dt_proj.bias, S)
        return self.out_proj(y.view(B, S, self.d_inner))


class MHA(nn.Module):
    """Attention layer of the hybrid: fused in_proj -> partial rotary (half-split) -> causal GQA flash
    attention -> out_proj (mamba_ssm ``MHA`` with ``d_conv=0``, no biases)."""

    def __init__(self, embed_dim, num_heads, num_heads_kv=None, head_dim=None, rotary_emb_dim=0,
                 rotary_emb_base=10000.0, causal=True, layer_idx=None, device=None, dtype=None, **_unused):
        super().__init__()
        self.embed_dim, self.num_heads = embed_dim, num_heads
        self.num_heads_kv = num_heads_kv or num_heads
        self.head_dim = head_dim or embed_dim // num_heads
        self.rotary_emb_dim, self.rotary_emb_base = rotary_emb_dim, rotary_emb_base
        self.layer_idx = layer_idx
        qkv_dim = self.head_dim * (self.num_heads + 2 * self.num_heads_kv)
        self.in_proj = _W(qkv_dim, embed_dim, device, dtype)
        self.out_proj = _W(embed_dim, self.head_dim * self.num_heads, device, dtype)
        self._tables = {}

    def reset_parameters(self):
        self.in_proj.reset_parameters()
        self.out_proj.reset_parameters()

    def _table(self, device, S):
        key = (str(device),)
        t = self._tables.get(key)
        if t is None or t.shape[0] < S:
            t = torch_kernels.rope_table(max(S, 4096), self.rotary_emb_dim, self.rotary_emb_base, device=device)
            self._tables[key] = t
        return t

    def forward(self, x):
        B, S, _ = x.shape
        qkv = self.in_proj(x)
        if self.rotary_emb_dim > 0:
            qkv = ops.rope_(qkv, self._table(x.device, S), S, self.num_heads, self.num_heads_kv, self.head_dim,
                            self.rotary_emb_dim, interleaved=False)
        ctx = ops.attention(qkv, self.num_heads, self.num_heads_kv, self.head_dim)
        return self.out_proj(ctx)


class GatedMLP(nn.Module):
    """fc1 -> (y, gate) halves -> y * silu(gate) -> fc2   (mamba_ssm ordering: value first, gate second)."""

    def __init__(self, in_features, hidden_features, device=None, dtype=None):
        super().__init__()
        self.fc1 = _W(2 * hidden_features, in_features, device, dtype)
        self.fc2 = _W(in_features, hidden_features, device, dtype)

    def reset_parameters(self):
        self.fc1.reset_parameters()
        self.fc2.reset_parameters()

    def forward(self, x):
        return ops.gated_mlp(x, self.fc1.weight, self.fc2.weight, gate_first=False)


class Block(nn.Module):
    """Pre-norm residual block with an fp32 residual stream: (hidden, residual) -> (hidden, residual)."""

    def __init__(self, dim, mixer: nn.Module, mlp: Optional[nn.Module], norm_eps=1e-5, residual_in_fp32=True,
                 device=None, dtype=None):
        super().__init__()
        self.residual_in_fp32 = residual_in_fp32
        self.norm = RMSNorm(dim, norm_eps, device, dtype)
        self.mixer = mixer
        self.mlp = mlp
        if mlp is not None:
            self.norm2 = RMSNorm(dim, norm_eps, device, dtype)

    def reset_parameters(self):
        self.norm.reset_parameters()
        if self.mlp is not None:
            self.norm2.reset_parameters()

    def forward(self, hidden, residual):
        hidden, residual = ops.add_rmsnorm(hidden, residual, self.norm.weight, self.norm.eps, self.residual_in_fp32)
        hidden = self.mixer(hidden)
        if self.mlp is not None:
            hidden, residual = ops.add_rmsnorm(hidden, residual, self.norm2.weight, self.norm2.eps,
                                               self.residual_in_fp32)
            hidden = self.mlp(hidden)
        return hidden, residual


class MixerModel(nn.Module):
    def __init__(self, cfg: MambaConfig, device=None, dtype=None):
        super().__init__()
        self.embedding = nn.Embedding(cfg.padded_vocab, cfg.d_model, device=device, dtype=dtype)
        layers = []
        for i in range(cfg.n_layer):
            if i in cfg.attn_layer_idx:
                a = dict(cfg.attn_cfg)
                mixer = MHA(cfg.d_model, a.get("num_heads"), a.get("num_heads_kv"), a.get("head_dim"),
                            a.get("rotary_emb_dim", 0), layer_idx=i, device=device, dtype=dtype)
            else:
                s = {k: v for k, v in cfg.ssm_cfg.items() if k != "layer"}
                kind = cfg.ssm_cfg.get("layer", "Mamba1")        # mamba_ssm's default (``create_block``)
                if kind not in ("Mamba1", "Mamba2"):
                    raise ValueError(f"Invalid ssm_layer: {kind}, only support Mamba1 and Mamba2")
                mixer = (Mamba2 if kind == "Mamba2" else Mamba1)(cfg.d_model, layer_idx=i, device=device, dtype=dtype, **s)
            mlp = GatedMLP(cfg.d_model, cfg.d_intermediate, device, dtype) if cfg.d_intermediate > 0 else None
            layers.append(Block(cfg.d_model, mixer, mlp, cfg.norm_epsilon, cfg.residual_in_fp32, device, dtype))
        self.layers = nn.ModuleList(layers)
        self.norm_f = RMSNorm(cfg.d_model, cfg.norm_epsilon, device, dtype)


class MambaLMHeadModel(nn.Module):
    def __init__(self, config: MambaConfig, device=None, dtype=None):
        super().__init__()
        self.config = config
        self.backbone = MixerModel(config, device, dtype)
        self.lm_head = _W(config.padded_vocab, config.d_model, device, dtype)
        if config.tie_embeddings:
            self.lm_head.weight = self.backbone.embedding.weight
        # output z-loss coefficient c (objective CE + c * mean_t lse_t^2, lse_t the logsumexp of token t's logits).  It
        # lives on the model, not in MambaConfig, whose fields are those of mamba_ssm's config.
        self.z_loss_coef = 0.0
        self.last_z = None

    def reset_parameters(self):
        cfg = self.config
        nn.init.normal_(self.backbone.embedding.weight, std=0.02)
        if not cfg.tie_embeddings:
            nn.init.normal_(self.lm_head.weight, std=0.02)
        self.backbone.norm_f.reset_parameters()
        n_resid = 2 if cfg.d_intermediate > 0 else 1
        for blk in self.backbone.layers:
            blk.reset_parameters()
            blk.mixer.reset_parameters()
            if blk.mlp is not None:
                blk.mlp.reset_parameters()
            # GPT-2 style rescale of the residual-branch output projections
            for w in [blk.mixer.out_proj.weight] + ([blk.mlp.fc2.weight] if blk.mlp is not None else []):
                with torch.no_grad():
                    w.div_(math.sqrt(n_resid * cfg.n_layer))

    # ---- plain forward (reference: output has ``.logits``, ``train_utils.py:89``)
    def forward(self, input_ids, labels=None, **_):
        hidden = self.engine_embed(input_ids)
        for blk in self.backbone.layers:
            hidden = blk(*hidden)
        out = self.engine_head(*hidden, labels=labels)
        return out if labels is not None else CausalLMOutput(logits=out)

    # ---- sharded-runtime protocol
    def engine_units(self):
        roots = [self.backbone.embedding, self.backbone.norm_f, self.lm_head]
        return list(self.backbone.layers), roots

    def engine_embed(self, tokens):
        h = ops.embedding(tokens, self.backbone.embedding.weight)
        # the residual stream starts at zero: block 0 computes residual = hidden + 0
        return h, torch.zeros_like(h, dtype=torch.float32 if self.config.residual_in_fp32 else h.dtype)

    def engine_head(self, hidden, residual, labels=None, ignore_index=-100):
        nf = self.backbone.norm_f
        hidden, _ = ops.add_rmsnorm(hidden, residual, nf.weight, nf.eps, self.config.residual_in_fp32)
        if labels is None:
            return ops.linear(hidden, self.lm_head.weight)
        if self.z_loss_coef > 0:
            ce, self.last_z = ops.linear_cross_entropy_z(hidden, self.lm_head.weight, labels, self.z_loss_coef,
                                                         ignore_index)
            return ce
        return ops.linear_cross_entropy(hidden, self.lm_head.weight, labels, ignore_index)

    def z_loss(self):
        """z_loss_coef * mean lse^2 of the output logits of the last loss forward (device scalar; its gradient is
        already part of the backward); None without a z-loss or before the first forward with labels."""
        if self.z_loss_coef <= 0 or self.last_z is None:
            return None
        return self.last_z * self.z_loss_coef

    # ---- mamba_ssm-style export (config.json + pytorch_model.bin)
    def save_pretrained(self, save_directory):
        import json
        import os
        os.makedirs(save_directory, exist_ok=True)
        torch.save(self.state_dict(), os.path.join(save_directory, "pytorch_model.bin"))
        cfg = {k: getattr(self.config, k) for k in self.config.__dataclass_fields__}
        with open(os.path.join(save_directory, "config.json"), "w") as f:
            json.dump(cfg, f, indent=4)
