"""Import a HuggingFace ``LlamaForCausalLM``, ``Qwen2ForCausalLM``, ``Qwen3ForCausalLM``, ``Qwen3MoeForCausalLM`` or
``MixtralForCausalLM`` directory as a single-file model
checkpoint for this trainer -- the inverse of ``fms_to_hf_llama.py`` (the reference has only the export direction; continued pre-training /
fine-tuning from public weights needs the way back):

    python hf_to_fms_llama.py --hf_path <hf dir> --save_path llama.pth [--model_variant llama2_7b]
    torchrun ... main_training_llama.py --model_variant=llama2_7b --ckpt_load_path=llama.pth ...

The file holds ``{"model_state": {<fms parameter name>: tensor}}`` -- the single-file format ``Checkpointer.load`` accepts
(weights only; step count, optimizer and data-loader state start fresh, as in reference ``checkpointing_utils.py:216-233``).
q/k rows are permuted from HF's half-split RoPE layout to the FMS interleaved-pair layout and q/k/v, gate/up are fused
(``models/hf_loader.convert_hf_state_dict``).  Qwen3 checkpoints also carry per-head ``q_norm`` / ``k_norm`` gains, permuted
like the q / k rows; train them with a ``qwen3_*`` variant (it has ``qk_norm`` and head_dim 128).  Qwen2 / Qwen2.5
checkpoints carry q / k / v biases, fused like the weights; train them with a ``qwen2.5_*`` variant (``qkv_bias``).
Qwen3-MoE and Mixtral checkpoints become mixture-of-experts blocks: the router goes to ``layers.N.moe.gate.weight`` and
the experts are stacked into ``moe.w1`` / ``moe.w2``; train them with ``qwen3_moe_30b_a3b`` / ``mixtral_8x7b``.
Safetensors checkpoints are read lazily, layer by layer, so the peak host memory is about the output plus one layer.
``--model_variant`` is optional: when given, the HF config is checked against that entry of the model zoo so that a
mismatch is reported here and not as a shape error on 8 GPUs.  For MoE variants the expert count, top-k, expert width
and top-k renormalisation are checked in place of the dense width, which MoE blocks do not use (the aux-loss
coefficient is a training flag and is not checked).
"""
import json
import os

import torch

from fms_fsdp_b200.models.hf_loader import config_from_hf, convert_hf_state_dict, open_hf_tensors
from fms_fsdp_b200.utils.cli import run
from fms_fsdp_b200.utils.config_utils import get_model_config

_CHECKED = ("src_vocab_size", "emb_dim", "nheads", "kv_heads", "nlayers", "hidden_dim", "rope_theta", "rope_scaling",
            "qk_norm", "head_dim", "qkv_bias")
_CHECKED_MOE = ("moe_num_experts", "moe_top_k", "moe_hidden_dim", "moe_norm_topk")


def main(hf_path: str, save_path: str, model_variant: str = "", dtype: str = "bf16"):
    hf = open_hf_tensors(hf_path)
    with open(os.path.join(hf_path, "config.json")) as f:
        cfg = config_from_hf(json.load(f), hf)
    if model_variant:
        want = get_model_config(model_variant)
        checked = _CHECKED
        if cfg.moe_num_experts > 0 or want.moe_num_experts > 0:
            checked = tuple(k for k in _CHECKED if k != "hidden_dim") + _CHECKED_MOE
        bad = {k: (getattr(cfg, k), getattr(want, k)) for k in checked if getattr(cfg, k) != getattr(want, k)}
        if bad:
            raise ValueError(f"{hf_path} does not have the architecture of {model_variant}: (checkpoint, zoo) = {bad}")
    torch_dtype = {"bf16": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32}[dtype]
    sd = convert_hf_state_dict(hf, cfg, torch_dtype)
    os.makedirs(os.path.dirname(os.path.abspath(save_path)), exist_ok=True)
    torch.save({"model_state": sd}, save_path)
    n = sum(v.numel() for v in sd.values())
    print(f"--> wrote {save_path}: {len(sd)} tensors, {n / 1e6:.1f} M parameters, {dtype}")


if __name__ == "__main__":
    run(main)
