"""Load HuggingFace checkpoints (safetensors / .bin) into this repo's models (stand-in for
``fms.models.get_model(..., source="hf")``, SURVEY.md §2.4 E5; reference call ``speculator/train_speculator.py:150-160`` with
the adapters of ``train_speculator_utils.py:526-569``):

* Llama   -> ``LLaMA`` / ``EmbedLLaMA``: fuses q/k/v and gate/up, permutes q/k rows from HF's half-split RoPE layout back
  to the FMS interleaved-pair layout (the inverse of ``fms_to_hf_llama._interleaved_to_halfsplit``);
* Qwen3 (dense) -> ``LLaMA`` with ``qk_norm`` and an explicit head dim: as Llama, plus the per-head ``q_norm`` / ``k_norm``
  gains permuted the same way as the q / k rows (tied embeddings are read as an untied copy);
* Qwen2 / Qwen2.5 -> ``LLaMA`` with ``qkv_bias``: as Llama, plus the q / k / v biases fused like the weights, the q / k
  biases permuted head by head like their rows (tied embeddings are read as an untied copy);
* Qwen3-MoE / Mixtral -> ``LLaMA`` with ``moe_num_experts``: attention as Qwen3 / Llama, every block's feed-forward the
  router ``moe.gate`` and the experts stacked into ``moe.w1 [E, 2F, D]`` (gate | up) and ``moe.w2 [E, D, F]``
  (``_stack_experts``, which reads the hub layouts of both families and the fused layout of transformers 5);
* GPT-BigCode (multi-query attention, learned positions) -> ``EmbedGPTBigCode``;
* Mixtral as a frozen speculator base -> ``EmbedMixtral`` (the same expert stacking, its own dense attention config).

``open_hf_tensors`` maps tensor names to lazily read safetensors entries, so a converter that goes layer by layer holds
its output and one layer, not the whole checkpoint twice."""
from __future__ import annotations

import dataclasses
import glob
import json
import os
from typing import Dict, Iterator, Mapping, Optional, Tuple

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
        raise NotImplementedError(f"HF model type {hf_cfg['model_type']!r} is not supported ({why}); Llama, Qwen2 / Qwen2.5, "
                                  "Qwen3, Qwen3-MoE and Mixtral checkpoints are")
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


def _moe_fields(hf_cfg: dict) -> dict:
    """The ``LLaMAConfig`` mixture-of-experts fields of a ``qwen3_moe`` or ``mixtral`` config ({} for other types).
    Every block here is a MoE block with a plain top-k router, so stacks that mix in dense blocks and Mixtral's router
    jitter (training-time noise on the router input) are refused."""
    kind = hf_cfg.get("model_type")
    if kind not in ("qwen3_moe", "mixtral"):
        return {}
    if kind == "qwen3_moe":
        # the hub's config.json says num_experts; transformers 5 writes the same field as num_local_experts
        E = hf_cfg.get("num_experts") or hf_cfg.get("num_local_experts")
        fields = dict(experts=E, num_experts_per_tok=hf_cfg.get("num_experts_per_tok"),
                      moe_intermediate_size=hf_cfg.get("moe_intermediate_size"))
        # transformers' default when the field is absent is False; the released checkpoints set it
        norm_topk = bool(hf_cfg.get("norm_topk_prob", False))
    else:
        fields = dict(experts=hf_cfg.get("num_local_experts"), num_experts_per_tok=hf_cfg.get("num_experts_per_tok", 2),
                      moe_intermediate_size=hf_cfg.get("intermediate_size"))
        norm_topk = True           # softmax, top-k, renormalise
    missing = [k for k, v in fields.items() if not v]
    if missing:
        raise NotImplementedError(f"HF model type {kind!r}: the config lacks the mixture-of-experts fields {missing}, so "
                                  "the expert count, top-k and expert width are unknown")
    if hf_cfg.get("decoder_sparse_step", 1) != 1 or hf_cfg.get("mlp_only_layers"):
        raise NotImplementedError(f"HF checkpoint mixes dense and mixture-of-experts blocks (decoder_sparse_step "
                                  f"{hf_cfg.get('decoder_sparse_step')}, mlp_only_layers {hf_cfg.get('mlp_only_layers')}); "
                                  "every block here is mixture-of-experts")
    if hf_cfg.get("router_jitter_noise"):
        raise NotImplementedError(f"HF checkpoint trains with router_jitter_noise {hf_cfg['router_jitter_noise']}; the "
                                  "router here has no input noise, training would differ")
    return dict(moe_num_experts=int(fields["experts"]), moe_top_k=int(fields["num_experts_per_tok"]),
                moe_hidden_dim=int(fields["moe_intermediate_size"]), moe_norm_topk=norm_topk,
                moe_aux_loss_coef=float(hf_cfg.get("router_aux_loss_coef") or 0.0))


def config_from_hf(hf_cfg: dict, tensors: Optional[Mapping[str, torch.Tensor]] = None) -> LLaMAConfig:
    """``tensors`` (optional): the checkpoint's tensors; a per-head ``self_attn.q_norm.weight`` there turns QK-norm on
    whatever ``model_type`` says, and q / k / v biases in every layer without an output bias (Qwen2) turn on
    ``qkv_bias``.  Without them a ``qwen2`` config is refused.  ``qwen3_moe`` and ``mixtral`` fill the
    ``moe_*`` fields (``_moe_fields``); the dense width (``hidden_dim``) stays ``intermediate_size``, unused by MoE
    blocks."""
    qkv_bias = hf_cfg.get("model_type") == "qwen2" and _has_qkv_bias_only(hf_cfg, tensors)
    _refuse_unsupported(hf_cfg, qkv_bias)
    moe = _moe_fields(hf_cfg)
    D, F = hf_cfg["hidden_size"], hf_cfg["intermediate_size"]
    H = hf_cfg["num_attention_heads"]
    hd = hf_cfg.get("head_dim") or D // H
    qk_norm = hf_cfg.get("model_type") in ("qwen3", "qwen3_moe")
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
        rope_scaling=rope_scaling, qk_norm=qk_norm, attn_head_dim=hd if hd != D // H else None, qkv_bias=qkv_bias,
        **moe)


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


class _LazyTensors(Mapping):
    """Tensor name -> tensor of a safetensors checkpoint, read from its file at each lookup and not kept.
    ``model.safetensors.index.json``, when present, says which shard holds each name.  Each lookup opens the shard
    anew: a handle kept open would keep every page read through its memory map resident, the whole checkpoint by the
    end of a conversion."""

    def __init__(self, model_path: str):
        from safetensors import safe_open
        self._path = model_path
        index = os.path.join(model_path, "model.safetensors.index.json")
        if os.path.exists(index):
            with open(index) as f:
                self._where = json.load(f)["weight_map"]
            return
        self._where = {}
        for f in sorted(glob.glob(os.path.join(model_path, "*.safetensors"))):
            with safe_open(f, framework="pt") as h:
                self._where.update({k: os.path.basename(f) for k in h.keys()})

    def __getitem__(self, name: str) -> torch.Tensor:
        from safetensors import safe_open
        with safe_open(os.path.join(self._path, self._where[name]), framework="pt") as h:
            return h.get_tensor(name)

    def __contains__(self, name) -> bool:
        return name in self._where

    def __iter__(self) -> Iterator[str]:
        return iter(self._where)

    def __len__(self) -> int:
        return len(self._where)


def open_hf_tensors(model_path: str) -> Mapping[str, torch.Tensor]:
    """The checkpoint's tensors by name: lazily read from safetensors files, or all of a ``pytorch_model*.bin`` loaded."""
    if glob.glob(os.path.join(model_path, "*.safetensors")):
        return _LazyTensors(model_path)
    return _read_hf_tensors(model_path)


def _stack_experts(hf: Mapping[str, torch.Tensor], layer: int, E: int, F: int, D: int,
                   dtype: Optional[torch.dtype] = None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """(router [E, D], w1 [E, 2F, D] = [gate | up] per expert, w2 [E, D, F]) of HF layer ``layer``, from whichever
    layout the checkpoint has:

    * the fused layout of transformers 5 state dicts: ``mlp.experts.gate_up_proj`` [E, 2F, D] (gate rows first) and
      ``mlp.experts.down_proj`` [E, D, F];
    * the Qwen3-MoE hub layout: ``mlp.experts.{e}.{gate,up,down}_proj.weight``;
    * the Mixtral hub layout: ``block_sparse_moe.experts.{e}.w1`` (gate), ``w3`` (up), ``w2`` (down).

    The router is ``mlp.gate.weight`` or ``block_sparse_moe.gate.weight``.  Per-expert tensors are copied one at a time
    into stacks built in ``dtype`` (default: the checkpoint's), so a lazily read checkpoint costs one expert on top of
    the result.  A missing expert, a wrong expert count or a wrong shape raises ``ValueError`` naming layer and expert."""
    s = f"model.layers.{layer}."

    def checked(name: str, t: torch.Tensor, shape: tuple, expert: Optional[int] = None) -> torch.Tensor:
        if tuple(t.shape) != shape:
            who = f"expert {expert}'s " if expert is not None else ""
            count = f" ({t.shape[0]} experts, the config says {E})" if len(shape) == 3 and t.shape[0] != E else ""
            raise ValueError(f"layer {layer}: {who}{name} has shape {tuple(t.shape)}, expected {shape}{count}")
        return t if dtype is None else t.to(dtype)

    b = s + ("block_sparse_moe." if s + "block_sparse_moe.gate.weight" in hf else "mlp.")
    if b + "gate.weight" not in hf:
        raise ValueError(f"layer {layer}: no router weight ({s}mlp.gate.weight or {s}block_sparse_moe.gate.weight)")
    router = hf[b + "gate.weight"]
    if router.shape[0] != E:
        raise ValueError(f"layer {layer}: the router scores {router.shape[0]} experts, the config says {E}")
    router = checked(b + "gate.weight", router, (E, D))
    if b + "experts.gate_up_proj" in hf:
        return (router, checked(b + "experts.gate_up_proj", hf[b + "experts.gate_up_proj"], (E, 2 * F, D)),
                checked(b + "experts.down_proj", hf[b + "experts.down_proj"], (E, D, F)))
    names = ("w1", "w3", "w2") if b.endswith("block_sparse_moe.") else ("gate_proj", "up_proj", "down_proj")
    if any(f"{b}experts.{E}.{n}.weight" in hf for n in names):
        raise ValueError(f"layer {layer}: the checkpoint has an expert {E}, the config says {E} experts")
    w1 = w2 = None
    for e in range(E):
        keys = [f"{b}experts.{e}.{n}.weight" for n in names]
        absent = [k for k in keys if k not in hf]
        if absent:
            raise ValueError(f"layer {layer}: expert {e} is missing {absent}")
        g, u, dn = (checked(k, hf[k], shape, e) for k, shape in zip(keys, ((F, D), (F, D), (D, F))))
        if w1 is None:
            w1, w2 = torch.empty(E, 2 * F, D, dtype=g.dtype), torch.empty(E, D, F, dtype=dn.dtype)
        w1[e, :F].copy_(g)
        w1[e, F:].copy_(u)
        w2[e].copy_(dn)
    return router, w1, w2


def convert_hf_state_dict(hf: Mapping[str, torch.Tensor], cfg: LLaMAConfig,
                          dtype: Optional[torch.dtype] = None) -> Dict[str, torch.Tensor]:
    """HF tensor names -> this repo's ``LLaMA`` state dict.  ``hf``: a dict or ``open_hf_tensors``'s lazy mapping, read
    layer by layer.  ``dtype`` casts each tensor as it is converted (None keeps the checkpoint's), so the peak memory is
    the result plus one layer.  With ``cfg.moe_num_experts > 0`` each block's feed-forward is the router and the
    stacked experts (``_stack_experts``)."""
    if cfg.moe_num_experts <= 0 and any(".block_sparse_moe." in n or ".mlp.experts." in n
                                        or n.endswith(".mlp.gate.weight") for n in hf):
        raise NotImplementedError("the checkpoint has mixture-of-experts tensors (Mixtral, Qwen3-MoE) but the config "
                                  "has no experts (moe_num_experts=0); config_from_hf of its config.json has them")
    cast = (lambda t: t) if dtype is None else (lambda t: t.to(dtype).contiguous())   # noqa: E731
    sd = {"shared.emb.weight": cast(hf["model.embed_tokens.weight"]),
          "shared.head.weight": cast(hf["lm_head.weight"] if "lm_head.weight" in hf else hf["model.embed_tokens.weight"]),
          "dec_norm.weight": cast(hf["model.norm.weight"])}
    for i in range(cfg.nlayers):
        s, d = f"model.layers.{i}.", f"layers.{i}."
        q = _halfsplit_to_interleaved(hf[s + "self_attn.q_proj.weight"], cfg.nheads)
        k = _halfsplit_to_interleaved(hf[s + "self_attn.k_proj.weight"], cfg.kv_heads)
        sd[d + "attn.in_proj.qkv_fused.weight"] = cast(torch.cat([q, k, hf[s + "self_attn.v_proj.weight"]], dim=0))
        if (s + "self_attn.q_proj.bias" in hf) != bool(cfg.qkv_bias):
            raise ValueError(f"layer {i}: the checkpoint {'lacks' if cfg.qkv_bias else 'has'} q / k / v biases "
                             f"but the config says qkv_bias={cfg.qkv_bias}")
        if cfg.qkv_bias:   # the q / k biases follow their rows from half-split to interleaved order, head by head
            qb = _halfsplit_to_interleaved_bias(hf[s + "self_attn.q_proj.bias"], cfg.nheads)
            kb = _halfsplit_to_interleaved_bias(hf[s + "self_attn.k_proj.bias"], cfg.kv_heads)
            sd[d + "attn.in_proj.qkv_fused.bias"] = cast(torch.cat([qb, kb, hf[s + "self_attn.v_proj.bias"]]))
        sd[d + "attn.dense.weight"] = cast(hf[s + "self_attn.o_proj.weight"])
        if cfg.moe_num_experts > 0:
            sd[d + "moe.gate.weight"], sd[d + "moe.w1"], sd[d + "moe.w2"] = _stack_experts(
                hf, i, cfg.moe_num_experts, cfg.moe_hidden_dim, cfg.emb_dim, dtype)
        else:
            sd[d + "ff_sub_layer.wg1_fused.weight"] = cast(torch.cat([hf[s + "mlp.gate_proj.weight"],
                                                                      hf[s + "mlp.up_proj.weight"]], dim=0))
            sd[d + "ff_sub_layer.w2.weight"] = cast(hf[s + "mlp.down_proj.weight"])
        sd[d + "ln.weight"] = cast(hf[s + "input_layernorm.weight"])
        sd[d + "ff_ln.weight"] = cast(hf[s + "post_attention_layernorm.weight"])
        if (s + "self_attn.q_norm.weight" in hf) != bool(cfg.qk_norm):
            raise ValueError(f"layer {i}: the checkpoint {'lacks' if cfg.qk_norm else 'has'} q / k norm weights "
                             f"but the config says qk_norm={cfg.qk_norm}")
        if cfg.qk_norm:   # per-head gains follow the q / k rows from half-split to interleaved order
            for name in ("q_norm", "k_norm"):
                w = hf[s + f"self_attn.{name}.weight"]
                if w.numel() != cfg.head_dim:
                    raise NotImplementedError(f"{s}self_attn.{name}.weight has {w.numel()} elements; only a per-head "
                                              f"QK-norm over head_dim = {cfg.head_dim} is implemented")
                sd[d + f"attn.{name}.weight"] = cast(_halfsplit_to_interleaved_vec(w))
    return sd


def load_hf_llama(model_path: str, device="cpu", dtype=torch.bfloat16, model_cls=LLaMA) -> LLaMA:
    tensors = open_hf_tensors(model_path)
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
    """``model_cls`` = ``EmbedMixtral``, which runs its own top-k feed-forward on a dense attention config (it refuses
    ``moe_num_experts > 0``).  Its state-dict names are the trainable ``LLaMA``'s, so the conversion is
    ``convert_hf_state_dict`` with the checkpoint's MoE config."""
    with open(os.path.join(model_path, "config.json")) as f:
        moe = config_from_hf(json.load(f))
    with torch.device("meta"):
        model = model_cls(dataclasses.replace(moe, moe_num_experts=0), n_experts=moe.moe_num_experts,
                          top_k=moe.moe_top_k)
    model.to_empty(device=device)
    sd = convert_hf_state_dict(open_hf_tensors(model_path), moe)
    model.load_state_dict({k: v.to(dtype) for k, v in sd.items()})
    return model.to(dtype)
