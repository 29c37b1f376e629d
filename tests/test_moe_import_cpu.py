"""Qwen3-MoE and Mixtral checkpoints on CPU: import against ``transformers`` logits (one file and sharded with an index;
the Qwen3-MoE, Mixtral and fused transformers-5 expert layouts), the export round trip through a sharded checkpoint, the
zoo check of ``hf_to_fms_llama.py``, every refusal, and the imported checkpoint's first training step on gloo (world 2)
against the ``transformers`` cross-entropy.  All models are tiny random ones built from a config, offline."""
import json
import os
import re
import subprocess
import sys

import pytest
import torch

from conftest import free_port
from fms_fsdp_b200.models.llama import LLaMA, LLaMAConfig
from fms_fsdp_b200.parallel import ShardedAdamW, ShardedModel
from fms_fsdp_b200.utils import config_utils
from fms_fsdp_b200.utils.checkpointing_utils import Checkpointer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _logits(model, x):
    with torch.no_grad():
        out = model(x)
    return getattr(out, "logits", out)


def _close(a, b):
    assert torch.allclose(a, b, atol=2e-4, rtol=1e-3), (a - b).abs().max()


def _qwen3_moe(norm_topk=True, seed=0, **over):
    from transformers import Qwen3MoeConfig, Qwen3MoeForCausalLM
    torch.manual_seed(seed)
    kw = dict(vocab_size=96, hidden_size=64, intermediate_size=128, moe_intermediate_size=32, num_hidden_layers=2,
              num_attention_heads=4, num_key_value_heads=2, head_dim=32,                  # head_dim != 64 / 4
              num_experts=8, num_experts_per_tok=2, norm_topk_prob=norm_topk, max_position_embeddings=64,
              rope_theta=50000.0, rms_norm_eps=1e-6, tie_word_embeddings=False)
    hf = Qwen3MoeForCausalLM(Qwen3MoeConfig(**{**kw, **over})).eval()
    with torch.no_grad():
        for layer in hf.model.layers:                                                     # non-unit q / k gains
            layer.self_attn.q_norm.weight.uniform_(0.3, 1.7)
            layer.self_attn.k_norm.weight.uniform_(0.3, 1.7)
            layer.mlp.gate.weight.mul_(20)                # routing that depends on the token (init scale is nearly flat)
    return hf


def _mixtral(seed=0, **over):
    from transformers import MixtralConfig, MixtralForCausalLM
    torch.manual_seed(seed)
    kw = dict(vocab_size=96, hidden_size=64, intermediate_size=48, num_hidden_layers=2, num_attention_heads=4,
              num_key_value_heads=2, num_local_experts=4, num_experts_per_tok=2, max_position_embeddings=64,
              rope_theta=50000.0, tie_word_embeddings=False)
    hf = MixtralForCausalLM(MixtralConfig(**{**kw, **over})).eval()
    with torch.no_grad():
        for layer in hf.model.layers:
            layer.mlp.gate.weight.mul_(20)
    return hf


X = torch.randint(0, 96, (2, 33), generator=torch.Generator().manual_seed(1))


# --------------------------------------------------------------------------------------------------- import
@pytest.mark.parametrize("sharded", [False, True])
@pytest.mark.parametrize("norm_topk", [True, False])
def test_qwen3_moe_import_matches_transformers(tmp_path, norm_topk, sharded):
    from fms_fsdp_b200.models.hf_loader import load_hf_llama
    hf = _qwen3_moe(norm_topk)
    d = str(tmp_path / "hf")
    hf.save_pretrained(d, **({"max_shard_size": "100KB"} if sharded else {}))
    shards = [f for f in os.listdir(d) if f.endswith(".safetensors")]
    assert (len(shards) > 1) == sharded and os.path.exists(os.path.join(d, "model.safetensors.index.json")) == sharded
    m = load_hf_llama(d, dtype=torch.float32).eval()
    c = m.config
    assert (c.moe_num_experts, c.moe_top_k, c.moe_hidden_dim, c.moe_norm_topk) == (8, 2, 32, norm_topk)
    assert c.qk_norm and c.head_dim == 32 and c.moe_aux_loss_coef == hf.config.router_aux_loss_coef
    _close(_logits(m, X), _logits(hf, X))


def test_qwen3_moe_norm_topk_defaults_to_false_like_transformers():
    from fms_fsdp_b200.models.hf_loader import config_from_hf
    c = _qwen3_moe().config.to_dict()
    c.pop("norm_topk_prob")
    assert not config_from_hf(c).moe_norm_topk
    c.pop("num_local_experts", None)
    assert config_from_hf(dict(c, num_experts=8)).moe_num_experts == 8       # the hub config's name for the count


@pytest.mark.parametrize("layout", ["hub", "fused"])
def test_mixtral_import_matches_transformers(tmp_path, layout):
    from safetensors import safe_open
    from safetensors.torch import save_file
    from fms_fsdp_b200.models.hf_loader import load_hf_llama
    hf = _mixtral()
    d = str(tmp_path / "hf")
    if layout == "hub":
        hf.save_pretrained(d)
    else:                                    # the in-memory state dict of transformers 5, written as it is
        sd = {k: v.detach().clone().contiguous() for k, v in hf.state_dict().items()}
        assert any(k.endswith("mlp.experts.gate_up_proj") for k in sd)
        os.makedirs(d)
        save_file(sd, os.path.join(d, "model.safetensors"))
        hf.config.save_pretrained(d)
    with safe_open(os.path.join(d, "model.safetensors"), "pt") as f:
        keys = set(f.keys())
    want = "model.layers.0.block_sparse_moe.experts.3.w3.weight" if layout == "hub" else "model.layers.0.mlp.experts.gate_up_proj"
    assert want in keys
    m = load_hf_llama(d, dtype=torch.float32).eval()
    c = m.config
    assert (c.moe_num_experts, c.moe_top_k, c.moe_hidden_dim, c.moe_norm_topk, c.qk_norm) == (4, 2, 48, True, False)
    _close(_logits(m, X), _logits(hf, X))


# --------------------------------------------------------------------------------------------------- export
def _random_moe(qk_norm):
    torch.manual_seed(2)
    cfg = LLaMAConfig(src_vocab_size=96, emb_dim=64, nheads=4, kvheads=2, nlayers=2, multiple_of=16,
                      max_expected_seq_len=64, rope_theta=50000.0, norm_eps=1e-6, qk_norm=qk_norm,
                      attn_head_dim=32 if qk_norm else None, moe_num_experts=8, moe_top_k=2, moe_hidden_dim=32,
                      moe_norm_topk=not qk_norm, moe_aux_loss_coef=0.01)
    m = LLaMA(cfg)
    m.reset_parameters()
    with torch.no_grad():
        for blk in m.layers:
            blk.moe.gate.weight.mul_(20)
            if qk_norm:
                blk.attn.q_norm.weight.uniform_(0.3, 1.7)
                blk.attn.k_norm.weight.uniform_(0.3, 1.7)
    return m.eval()


@pytest.mark.parametrize("family", ["qwen3_moe", "mixtral"])
def test_moe_export_roundtrip_from_a_sharded_checkpoint(tmp_path, monkeypatch, family):
    import fms_to_hf_llama as ex
    from safetensors import safe_open
    from transformers import AutoModelForCausalLM
    from fms_fsdp_b200.models.hf_loader import config_from_hf, convert_hf_state_dict, open_hf_tensors
    m = _random_moe(qk_norm=family == "qwen3_moe")
    ref_sd = {k: v.clone() for k, v in m.state_dict().items()}
    ours = _logits(m, X)
    eng = ShardedModel(m, device="cpu")
    opt = ShardedAdamW(eng)
    ck = str(tmp_path / "ck")
    Checkpointer(ck, 2, "fsdp", 0, 0).save(5, eng, opt, None, tokens_seen=1)
    monkeypatch.setattr(ex, "get_model_config", lambda v: LLaMAConfig(**m.config.__dict__))
    out = str(tmp_path / "export")
    ex.main("moe_test", load_path=os.path.join(ck, "checkpoints", "step_5_ckp"), save_path=out)

    with open(os.path.join(out, "config.json")) as f:
        exported = json.load(f)
    assert exported["model_type"] == family and not exported["tie_word_embeddings"]
    if family == "qwen3_moe":
        assert exported["decoder_sparse_step"] == 1 and exported["mlp_only_layers"] == []
        assert not exported["use_sliding_window"] and exported["head_dim"] == 32 and exported["moe_intermediate_size"] == 32
    else:
        assert exported["intermediate_size"] == 32 and exported["sliding_window"] is None
    back = AutoModelForCausalLM.from_pretrained(out).eval()
    assert type(back).__name__ == {"qwen3_moe": "Qwen3MoeForCausalLM", "mixtral": "MixtralForCausalLM"}[family]
    _close(_logits(back, X), ours)

    # what lands on disk is the per-expert hub layout, which other tools read
    keys = set()
    for f in os.listdir(out):
        if f.endswith(".safetensors"):
            with safe_open(os.path.join(out, f), "pt") as h:
                keys |= set(h.keys())
    assert not any("gate_up_proj" in k or k.endswith("experts.down_proj") for k in keys)
    per_expert = ([f"mlp.experts.{e}.{n}_proj.weight" for n in ("gate", "up", "down") for e in range(8)]
                  if family == "qwen3_moe" else [f"block_sparse_moe.experts.{e}.{n}.weight" for n in ("w1", "w2", "w3")
                                                 for e in range(8)])
    assert all(f"model.layers.{i}.{k}" in keys for i in range(2) for k in per_expert)

    # importing the export gives back the original state dict, bit for bit
    sd = convert_hf_state_dict(open_hf_tensors(out), config_from_hf(exported, open_hf_tensors(out)))
    assert set(sd) == set(ref_sd)
    for k, v in ref_sd.items():
        assert torch.equal(sd[k], v), k


def test_moe_export_refuses_what_no_hf_class_computes():
    import fms_to_hf_llama as ex
    m = _random_moe(qk_norm=False)
    m.config.moe_norm_topk = False                      # Mixtral-shaped without the renormalisation
    with pytest.raises(NotImplementedError, match="moe_norm_topk"):
        ex.convert_to_hf(m, "moe_x")
    m.config.moe_norm_topk, m.config.qkv_bias = True, True
    with pytest.raises(NotImplementedError, match="biases"):
        ex.convert_to_hf(m, "moe_x")


# ------------------------------------------------------------------------------------ hf_to_fms --model_variant
def test_hf_to_fms_checks_the_expert_fields_against_the_variant(tmp_path, monkeypatch):
    import hf_to_fms_llama as imp
    hf = _mixtral()
    d = str(tmp_path / "hf")
    hf.save_pretrained(d)
    # the dense width of the zoo entry (hidden_dim 176) differs from the checkpoint's intermediate_size 48: not checked
    entry = dict(src_vocab_size=96, emb_dim=64, nheads=4, kvheads=2, nlayers=2, multiple_of=16, rope_theta=50000.0,
                 moe_num_experts=4, moe_top_k=2, moe_hidden_dim=48, moe_norm_topk=True, moe_aux_loss_coef=0.5)
    monkeypatch.setitem(config_utils._LLAMA_ZOO, "mixtral_test", entry)
    pth = str(tmp_path / "w" / "mixtral.pth")
    imp.main(d, pth, model_variant="mixtral_test", dtype="fp32")
    m = LLaMA(config_utils.get_model_config("mixtral_test"))
    m.load_state_dict(torch.load(pth)["model_state"])                  # strict
    _close(_logits(m.eval(), X), _logits(hf, X))
    for field, wrong in (("moe_num_experts", 8), ("moe_top_k", 1), ("moe_hidden_dim", 64), ("moe_norm_topk", False)):
        monkeypatch.setitem(config_utils._LLAMA_ZOO, "mixtral_test", dict(entry, **{field: wrong}))
        with pytest.raises(ValueError, match=field):
            imp.main(d, pth, model_variant="mixtral_test")
    with pytest.raises(ValueError, match="moe_num_experts"):               # a MoE checkpoint against a dense variant
        imp.main(d, pth, model_variant="llama2_tiny")


# ------------------------------------------------------------------------------------------------- refusals
def test_config_refusals():
    from fms_fsdp_b200.models.hf_loader import config_from_hf
    q, x = _qwen3_moe().config.to_dict(), _mixtral().config.to_dict()
    for bad, msg in (((q, {"decoder_sparse_step": 2}), "dense and mixture-of-experts"),
                     ((q, {"mlp_only_layers": [1]}), "dense and mixture-of-experts"),
                     ((x, {"router_jitter_noise": 0.1}), "router_jitter_noise"),
                     ((x, {"sliding_window": 32}), "sliding-window"),
                     ((q, {"use_sliding_window": True, "sliding_window": 32}), "sliding-window"),
                     ((q, {"model_type": "qwen2_moe"}), "shared experts")):
        (base, over) = bad
        with pytest.raises(NotImplementedError, match=msg):
            config_from_hf({**base, **over})
    for field in ("moe_intermediate_size", "num_experts_per_tok"):       # fields that say how big the experts are
        with pytest.raises(NotImplementedError, match="qwen3_moe.*mixture-of-experts"):
            config_from_hf({k: v for k, v in q.items() if k != field})
    with pytest.raises(NotImplementedError, match="mixtral.*mixture-of-experts"):
        config_from_hf({k: v for k, v in x.items() if k != "num_local_experts"})
    # a window as long as the context is no window, and a switched-off one is ignored
    assert config_from_hf({**x, "sliding_window": 64}).moe_num_experts == 4
    assert config_from_hf({**q, "use_sliding_window": False, "sliding_window": 32}).moe_num_experts == 8


@pytest.mark.parametrize("family", ["qwen3_moe", "mixtral", "fused"])
def test_weight_refusals_name_the_layer_and_the_expert(family):
    from fms_fsdp_b200.models.hf_loader import config_from_hf, convert_hf_state_dict
    hf = _qwen3_moe() if family == "qwen3_moe" else _mixtral()
    if family == "fused":
        sd = {k: v.detach() for k, v in hf.state_dict().items()}
    else:                                  # the hub layout save_pretrained writes
        from safetensors.torch import load_file
        import tempfile
        d = tempfile.mkdtemp()
        hf.save_pretrained(d)
        sd = load_file(os.path.join(d, "model.safetensors"))
    cfg = config_from_hf(hf.config.to_dict(), sd)
    E = cfg.moe_num_experts
    assert convert_hf_state_dict(sd, cfg)["layers.1.moe.w1"].shape == (E, 2 * cfg.moe_hidden_dim, cfg.emb_dim)
    if family == "fused":
        key = "model.layers.1.mlp.experts.gate_up_proj"
        with pytest.raises(ValueError, match=r"layer 1: .*gate_up_proj .*\(3 experts, the config says 4\)"):
            convert_hf_state_dict({**sd, key: sd[key][:3]}, cfg)
        with pytest.raises(ValueError, match=r"layer 1: .*down_proj has shape"):
            convert_hf_state_dict({**sd, "model.layers.1.mlp.experts.down_proj": sd[key]}, cfg)
    else:
        b, (g, u, dn) = (("model.layers.1.mlp.experts.", ("gate_proj", "up_proj", "down_proj")) if family == "qwen3_moe"
                         else ("model.layers.1.block_sparse_moe.experts.", ("w1", "w3", "w2")))
        missing = {k: v for k, v in sd.items() if k != f"{b}3.{u}.weight"}
        with pytest.raises(ValueError, match="layer 1: expert 3 is missing"):
            convert_hf_state_dict(missing, cfg)
        extra = dict(sd, **{f"{b}{E}.{n}.weight": sd[f"{b}0.{n}.weight"] for n in (g, u, dn)})
        with pytest.raises(ValueError, match=f"layer 1: the checkpoint has an expert {E}"):
            convert_hf_state_dict(extra, cfg)
        with pytest.raises(ValueError, match=f"layer 1: expert 2's .*{dn}.weight has shape"):
            convert_hf_state_dict(dict(sd, **{f"{b}2.{dn}.weight": sd[f"{b}2.{g}.weight"]}), cfg)
    router = [k for k in sd if k.startswith("model.layers.1.") and k.endswith("gate.weight") and "experts" not in k][0]
    with pytest.raises(ValueError, match="layer 1: the router scores 3 experts"):
        convert_hf_state_dict(dict(sd, **{router: sd[router][:3]}), cfg)
    with pytest.raises(ValueError, match="layer 1: no router"):
        convert_hf_state_dict({k: v for k, v in sd.items() if k != router}, cfg)
    # a dense config never takes expert tensors
    dense = LLaMAConfig(**{**cfg.__dict__, "moe_num_experts": 0})
    with pytest.raises(NotImplementedError, match="mixture-of-experts"):
        convert_hf_state_dict(sd, dense)


# --------------------------------------------------------------------------------------------- training
def test_imported_mixtral_trains_with_the_transformers_loss_on_gloo_world2(tmp_path):
    """``hf_to_fms_llama.py`` -> ``main_training_llama.py`` on 2 gloo ranks with the file as ``--ckpt_load_path``: the
    first step's loss is the ``transformers`` cross-entropy of the same batch (the dummy stream's first two windows,
    labels = inputs), with the balancing loss off."""
    import hf_to_fms_llama as imp
    from transformers import MixtralConfig, MixtralForCausalLM
    torch.manual_seed(4)
    c = config_utils.get_model_config("llama_moe_tiny")
    hf = MixtralForCausalLM(MixtralConfig(
        vocab_size=c.src_vocab_size, hidden_size=c.emb_dim, intermediate_size=c.moe_hidden_dim,
        num_hidden_layers=c.nlayers, num_attention_heads=c.nheads, num_key_value_heads=c.kv_heads,
        num_local_experts=c.moe_num_experts, num_experts_per_tok=c.moe_top_k, max_position_embeddings=c.max_expected_seq_len,
        rope_theta=c.rope_theta, rms_norm_eps=c.norm_eps, tie_word_embeddings=False)).eval()
    with torch.no_grad():
        for layer in hf.model.layers:
            layer.mlp.gate.weight.mul_(20)
    d, pth = str(tmp_path / "hf"), str(tmp_path / "start.pth")
    hf.save_pretrained(d)
    imp.main(d, pth, model_variant="llama_moe_tiny", dtype="fp32")

    S, B = 32, 2
    x = (torch.arange(B * S) % c.src_vocab_size).view(B, S)
    with torch.no_grad():
        want = torch.nn.functional.cross_entropy(hf(x).logits.view(-1, c.src_vocab_size), x.view(-1)).item()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(free_port()), os.path.join(ROOT, "main_training_llama.py"), "--model_variant=llama_moe_tiny",
           "--use_dummy_dataset=True", "--sharding_strategy=fsdp", "--report_interval=1", f"--seq_length={S}",
           f"--vocab_size={c.src_vocab_size}", f"--batch_size={B}", "--num_steps=1", "--checkpoint_interval=100",
           f"--ckpt_load_path={pth}", f"--ckpt_save_path={tmp_path / 'run'}", "--comm_backend=gloo",
           "--mixed_precision=False", "--moe_aux_loss_coef=0", "--use_torch_compile=False"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT, env=dict(os.environ, OMP_NUM_THREADS="1"))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "single-file checkpoint" in r.stdout
    loss = [float(v) for v in re.findall(r"^loss: ([0-9.eE+-]+)$", r.stdout, flags=re.M)]
    assert len(loss) == 1 and loss[0] == pytest.approx(want, rel=1e-5), (loss, want)
