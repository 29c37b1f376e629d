"""Load HuggingFace checkpoints (safetensors / .bin) into this repo's models (stand-in for
``fms.models.get_model(..., source="hf")``, SURVEY.md §2.4 E5; reference call ``speculator/train_speculator.py:150-160`` with
the adapters of ``train_speculator_utils.py:526-569``):

* Llama   -> ``LLaMA`` / ``EmbedLLaMA``: fuses q/k/v and gate/up, permutes q/k rows from HF's half-split RoPE layout back
  to the FMS interleaved-pair layout (the inverse of ``fms_to_hf_llama._interleaved_to_halfsplit``);
* Qwen3 (dense) -> ``LLaMA`` with ``qk_norm`` and an explicit head dim: as Llama, plus the per-head ``q_norm`` / ``k_norm``
  gains permuted the same way as the q / k rows (tied embeddings are read as an untied copy);
* Qwen2 / Qwen2.5 -> ``LLaMA`` with ``qkv_bias``: as Llama, plus the q / k / v biases fused like the weights, the q / k
  biases permuted head by head like their rows (tied embeddings are read as an untied copy);
* GPT-BigCode (multi-query attention, learned positions) -> ``EmbedGPTBigCode``;
* Mixtral (Llama attention + top-k sparse MoE) -> ``EmbedMixtral``; both the hub format (``block_sparse_moe.experts.N.w1/w2/w3``)
  and the fused in-memory format of recent transformers (``mlp.experts.gate_up_proj / down_proj``)."""
from __future__ import annotations

import glob
import json
import os
from typing import Dict, Optional

import torch

from fms_fsdp_b200.models.llama import LLaMA, LLaMAConfig


def _halfsplit_to_interleaved(w: torch.Tensor, nheads: int) -> torch.Tensor:
    return w.view(nheads, 2, -1, w.size(1)).transpose(1, 2).reshape(*w.size())


def _halfsplit_to_interleaved_vec(w: torch.Tensor) -> torch.Tensor:
    """A per-head-position vector [hd] (Qwen3 ``q_norm`` / ``k_norm``) in the order of the permuted q / k rows:
    out[2i] = w[i], out[2i + 1] = w[i + hd/2].  RMS is permutation-invariant, the elementwise gain is not."""
    return _halfsplit_to_interleaved(w.view(-1, 1), 1).view(-1)


def _halfsplit_to_interleaved_bias(b: torch.Tensor, nheads: int) -> torch.Tensor:
    """A q or k projection bias [nheads * hd] in the order of the permuted rows: each head's entries move like that
    head's rows (``_halfsplit_to_interleaved_vec`` would treat the whole bias as one head)."""
    return _halfsplit_to_interleaved(b.view(-1, 1), nheads).view(-1)


# model types whose differences from the Llama block are not implemented here (loading them would change the logits)
_REFUSED_MODEL_TYPES = {
    "olmo2": "q / k RMSNorm over the whole projection instead of per head",
    "olmo3": "q / k RMSNorm over the whole projection instead of per head",
    # Qwen2 is loaded when the checkpoint's tensors are at hand and show q / k / v biases without an output bias
    # (config_from_hf with ``tensors``); the config alone cannot show it
    "qwen2": "q / k / v projection biases; pass the checkpoint's tensors to detect them",
    # the engine trains these feed-forwards (LLaMAConfig.moe_num_experts) but does not import their checkpoints yet;
    # Mixtral is refused by convert_hf_state_dict instead (its attention config also serves the frozen speculator base)
    "qwen3_moe": "sparse mixture-of-experts feed-forward",
    "qwen2_moe": "shared experts and q / k / v projection biases",
}


def _has_qkv_bias_only(hf_cfg: dict, tensors: Optional[Dict[str, torch.Tensor]]) -> bool:
    """The checkpoint's tensors show Qwen2 attention: every layer biases q, k and v, and no layer biases o_proj."""
    if tensors is None:
        return False
    for i in range(hf_cfg["num_hidden_layers"]):
        s = f"model.layers.{i}.self_attn."
        if not all(s + f"{n}_proj.bias" in tensors for n in "qkv") or s + "o_proj.bias" in tensors:
            return False
    return True


def _refuse_unsupported(hf_cfg: dict, qkv_bias: bool = False):
    """Features this repo's models do not implement must stop the load instead of silently changing the logits.
    ``qkv_bias``: the tensors showed Qwen2's q / k / v biases, which are implemented (``LLaMAConfig.qkv_bias``)."""
    why = _REFUSED_MODEL_TYPES.get(hf_cfg.get("model_type"))
    if why and not (qkv_bias and hf_cfg.get("model_type") == "qwen2"):
        raise NotImplementedError(f"HF model type {hf_cfg['model_type']!r} is not supported ({why}); Llama, Qwen2 / Qwen2.5 "
                                  "and Qwen3 dense checkpoints are")
    scaling = hf_cfg.get("rope_scaling") or {}
    params = hf_cfg.get("rope_parameters") or {}
    kind = scaling.get("rope_type") or scaling.get("type") or params.get("rope_type") or "default"
    if kind not in ("default", None, "llama3", "linear"):
        raise NotImplementedError(f"HF checkpoint uses rope scaling {kind!r}; plain RoPE, 'linear' and 'llama3' (Llama 3.1 / 3.2) "
                                  "are implemented, loading it would change the logits")
    window = hf_cfg.get("sliding_window") if hf_cfg.get("use_sliding_window", True) else None
    if window and window < hf_cfg.get("max_position_embeddings", window):
        raise NotImplementedError(f"HF checkpoint uses sliding-window attention (window {window}); only full causal attention is "
                                  "implemented")
    if hf_cfg.get("attention_bias") or hf_cfg.get("mlp_bias"):
        raise NotImplementedError("HF checkpoint has attention / MLP biases; the LLaMA blocks here have q / k / v "
                                  "biases only (Qwen2), no output or MLP biases")


_Q_NORM_KEY = "model.layers.0.self_attn.q_norm.weight"


def config_from_hf(hf_cfg: dict, tensors: Optional[Dict[str, torch.Tensor]] = None) -> LLaMAConfig:
    """``tensors`` (optional): the checkpoint's tensors; a per-head ``self_attn.q_norm.weight`` there turns QK-norm on
    whatever ``model_type`` says, and q / k / v biases in every layer without an output bias (Qwen2) turn on
    ``qkv_bias``.  Without them a ``qwen2`` config is refused."""
    qkv_bias = hf_cfg.get("model_type") == "qwen2" and _has_qkv_bias_only(hf_cfg, tensors)
    _refuse_unsupported(hf_cfg, qkv_bias)
    D, F = hf_cfg["hidden_size"], hf_cfg["intermediate_size"]
    H = hf_cfg["num_attention_heads"]
    hd = hf_cfg.get("head_dim") or D // H
    qk_norm = hf_cfg.get("model_type") == "qwen3"
    if tensors is not None and _Q_NORM_KEY in tensors:
        if tensors[_Q_NORM_KEY].numel() != hd:
            raise NotImplementedError(f"HF checkpoint normalises q over {tensors[_Q_NORM_KEY].numel()} features; only a "
                                      f"per-head QK-norm (weight [head_dim = {hd}], Qwen3) is implemented")
        qk_norm = True
    rope = hf_cfg.get("rope_theta") or (hf_cfg.get("rope_parameters") or {}).get("rope_theta", 10000.0)
    scaling = hf_cfg.get("rope_scaling") or hf_cfg.get("rope_parameters") or {}
    kind = scaling.get("rope_type") or scaling.get("type")
    rope_scaling = {k: v for k, v in scaling.items() if k != "rope_theta"} if kind in ("llama3", "linear") else None
    return LLaMAConfig(
        src_vocab_size=hf_cfg["vocab_size"], emb_dim=D, norm_eps=hf_cfg.get("rms_norm_eps", 1e-5),
        nheads=H, kvheads=hf_cfg.get("num_key_value_heads", 0) or 0,
        nlayers=hf_cfg["num_hidden_layers"], hidden_grow_factor=F / D, multiple_of=1,
        max_expected_seq_len=hf_cfg.get("max_position_embeddings", 4096), rope_theta=float(rope),
        rope_scaling=rope_scaling, qk_norm=qk_norm, attn_head_dim=hd if hd != D // H else None, qkv_bias=qkv_bias)


def _read_hf_tensors(model_path: str) -> Dict[str, torch.Tensor]:
    out: Dict[str, torch.Tensor] = {}
    st = sorted(glob.glob(os.path.join(model_path, "*.safetensors")))
    if st:
        from safetensors.torch import load_file
        for f in st:
            out.update(load_file(f))
        return out
    for f in sorted(glob.glob(os.path.join(model_path, "pytorch_model*.bin"))):
        out.update(torch.load(f, map_location="cpu", weights_only=True))
    if not out:
        raise FileNotFoundError(f"no safetensors / pytorch_model*.bin under {model_path}")
    return out


def convert_hf_state_dict(hf: Dict[str, torch.Tensor], cfg: LLaMAConfig) -> Dict[str, torch.Tensor]:
    if any(".block_sparse_moe." in n or ".mlp.experts." in n or n.endswith(".mlp.gate.weight") for n in hf):
        raise NotImplementedError("mixture-of-experts checkpoints (Mixtral, Qwen3-MoE) are not imported for training yet; "
                                  "Llama and Qwen3 dense checkpoints are")
    sd = {"shared.emb.weight": hf["model.embed_tokens.weight"],
          "shared.head.weight": hf.get("lm_head.weight", hf["model.embed_tokens.weight"]),
          "dec_norm.weight": hf["model.norm.weight"]}
    for i in range(cfg.nlayers):
        s, d = f"model.layers.{i}.", f"layers.{i}."
        q = _halfsplit_to_interleaved(hf[s + "self_attn.q_proj.weight"], cfg.nheads)
        k = _halfsplit_to_interleaved(hf[s + "self_attn.k_proj.weight"], cfg.kv_heads)
        sd[d + "attn.in_proj.qkv_fused.weight"] = torch.cat([q, k, hf[s + "self_attn.v_proj.weight"]], dim=0)
        if (s + "self_attn.q_proj.bias" in hf) != bool(cfg.qkv_bias):
            raise ValueError(f"layer {i}: the checkpoint {'lacks' if cfg.qkv_bias else 'has'} q / k / v biases "
                             f"but the config says qkv_bias={cfg.qkv_bias}")
        if cfg.qkv_bias:   # the q / k biases follow their rows from half-split to interleaved order, head by head
            qb = _halfsplit_to_interleaved_bias(hf[s + "self_attn.q_proj.bias"], cfg.nheads)
            kb = _halfsplit_to_interleaved_bias(hf[s + "self_attn.k_proj.bias"], cfg.kv_heads)
            sd[d + "attn.in_proj.qkv_fused.bias"] = torch.cat([qb, kb, hf[s + "self_attn.v_proj.bias"]])
        sd[d + "attn.dense.weight"] = hf[s + "self_attn.o_proj.weight"]
        sd[d + "ff_sub_layer.wg1_fused.weight"] = torch.cat([hf[s + "mlp.gate_proj.weight"], hf[s + "mlp.up_proj.weight"]], dim=0)
        sd[d + "ff_sub_layer.w2.weight"] = hf[s + "mlp.down_proj.weight"]
        sd[d + "ln.weight"] = hf[s + "input_layernorm.weight"]
        sd[d + "ff_ln.weight"] = hf[s + "post_attention_layernorm.weight"]
        if (s + "self_attn.q_norm.weight" in hf) != bool(cfg.qk_norm):
            raise ValueError(f"layer {i}: the checkpoint {'lacks' if cfg.qk_norm else 'has'} q / k norm weights "
                             f"but the config says qk_norm={cfg.qk_norm}")
        if cfg.qk_norm:   # per-head gains follow the q / k rows from half-split to interleaved order
            for name in ("q_norm", "k_norm"):
                w = hf[s + f"self_attn.{name}.weight"]
                if w.numel() != cfg.head_dim:
                    raise NotImplementedError(f"{s}self_attn.{name}.weight has {w.numel()} elements; only a per-head "
                                              f"QK-norm over head_dim = {cfg.head_dim} is implemented")
                sd[d + f"attn.{name}.weight"] = _halfsplit_to_interleaved_vec(w)
    return sd


def load_hf_llama(model_path: str, device="cpu", dtype=torch.bfloat16, model_cls=LLaMA) -> LLaMA:
    tensors = _read_hf_tensors(model_path)
    with open(os.path.join(model_path, "config.json")) as f:
        cfg = config_from_hf(json.load(f), tensors)
    with torch.device("meta"):
        model = model_cls(cfg)
    model.to_empty(device=device)
    sd = convert_hf_state_dict(tensors, cfg)
    model.load_state_dict({k: v.to(dtype) for k, v in sd.items()})
    return model.to(dtype)


# ------------------------------------------------------------------------------------------ GPT-BigCode
def load_hf_gpt_bigcode(model_path: str, model_cls, device="cpu", dtype=torch.bfloat16):
    """``model_cls`` = ``speculator.train_speculator_utils.EmbedGPTBigCode`` (kept out of this module's imports)."""
    with open(os.path.join(model_path, "config.json")) as f:
        c = json.load(f)
    if not c.get("multi_query", True):
        raise ValueError("only multi-query GPT-BigCode checkpoints are supported")
    act = c.get("activation_function", "gelu_pytorch_tanh")
    if act not in ("gelu_pytorch_tanh", "gelu_new", "gelu_fast"):     # all three are the tanh approximation the block computes
        raise NotImplementedError(f"GPT-BigCode activation {act!r}: the block implements tanh-approximated GELU only")
    if not c.get("scale_attn_weights", True):
        raise NotImplementedError("GPT-BigCode checkpoints with scale_attn_weights=False are not supported")
    D = c["n_embd"]
    hidden = c.get("n_inner") or 4 * D
    if hidden % D:
        raise ValueError(f"n_inner {hidden} is not a multiple of n_embd {D}")
    with torch.device("meta"):
        model = model_cls(vocab=c["vocab_size"], emb_dim=D, nheads=c["n_head"], nlayers=c["n_layer"], max_pos=c["n_positions"],
                          hidden_mult=hidden // D, eps=c.get("layer_norm_epsilon", 1e-5))
    model.to_empty(device=device)
    hf = _read_hf_tensors(model_path)
    sd = {"emb.weight": hf["transformer.wte.weight"], "pos.weight": hf["transformer.wpe.weight"],
          "dec_norm.weight": hf["transformer.ln_f.weight"], "dec_norm.bias": hf["transformer.ln_f.bias"],
          "head.weight": hf.get("lm_head.weight", hf["transformer.wte.weight"])}
    names = {"ln": "ln_1", "ff_ln": "ln_2", "qkv": "attn.c_attn", "dense": "attn.c_proj", "w1": "mlp.c_fc", "w2": "mlp.c_proj"}
    for i in range(c["n_layer"]):
        for ours, theirs in names.items():
            for part in ("weight", "bias"):
                sd[f"layers.{i}.{ours}.{part}"] = hf[f"transformer.h.{i}.{theirs}.{part}"]
    model.load_state_dict({k: v.to(dtype) for k, v in sd.items()})
    return model.to(dtype)


# ---------------------------------------------------------------------------------------------- Mixtral
def load_hf_mixtral(model_path: str, model_cls, device="cpu", dtype=torch.bfloat16):
    """``model_cls`` = ``EmbedMixtral``.  Attention weights follow the Llama conversion; expert weights are stacked to
    ``moe.w1 [E, 2F, D]`` (gate | up) and ``moe.w2 [E, D, F]``."""
    with open(os.path.join(model_path, "config.json")) as f:
        c = json.load(f)
    cfg = config_from_hf(c)
    E, top_k = c["num_local_experts"], c.get("num_experts_per_tok", 2)
    with torch.device("meta"):
        model = model_cls(cfg, n_experts=E, top_k=top_k)
    model.to_empty(device=device)
    hf = _read_hf_tensors(model_path)
    sd = {"shared.emb.weight": hf["model.embed_tokens.weight"],
          "shared.head.weight": hf.get("lm_head.weight", hf["model.embed_tokens.weight"]),
          "dec_norm.weight": hf["model.norm.weight"]}
    for i in range(cfg.nlayers):
        s, d = f"model.layers.{i}.", f"layers.{i}."
        q = _halfsplit_to_interleaved(hf[s + "self_attn.q_proj.weight"], cfg.nheads)
        k = _halfsplit_to_interleaved(hf[s + "self_attn.k_proj.weight"], cfg.kv_heads)
        sd[d + "attn.in_proj.qkv_fused.weight"] = torch.cat([q, k, hf[s + "self_attn.v_proj.weight"]], dim=0)
        sd[d + "attn.dense.weight"] = hf[s + "self_attn.o_proj.weight"]
        sd[d + "ln.weight"] = hf[s + "input_layernorm.weight"]
        sd[d + "ff_ln.weight"] = hf[s + "post_attention_layernorm.weight"]
        if s + "mlp.experts.gate_up_proj" in hf:                       # fused in-memory layout of recent transformers
            sd[d + "moe.gate.weight"] = hf[s + "mlp.gate.weight"]
            sd[d + "moe.w1"] = hf[s + "mlp.experts.gate_up_proj"]
            sd[d + "moe.w2"] = hf[s + "mlp.experts.down_proj"]
        else:                                                          # hub layout: w1 = gate, w3 = up, w2 = down
            b = s + "block_sparse_moe."
            sd[d + "moe.gate.weight"] = hf[b + "gate.weight"]
            sd[d + "moe.w1"] = torch.stack([torch.cat([hf[f"{b}experts.{e}.w1.weight"], hf[f"{b}experts.{e}.w3.weight"]], 0)
                                            for e in range(E)])
            sd[d + "moe.w2"] = torch.stack([hf[f"{b}experts.{e}.w2.weight"] for e in range(E)])
    model.load_state_dict({k: v.to(dtype) for k, v in sd.items()})
    return model.to(dtype)
