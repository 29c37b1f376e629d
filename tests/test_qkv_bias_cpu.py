"""q / k / v projection biases (Qwen2 / Qwen2.5) on CPU: the ATen oracle node against autograd of an independent fp64
formula, the Qwen2 import / export round trip against transformers, the refusals, the world-2 gloo engine against the
single-process oracle, the entry points, the qwen2.5_* zoo entries and the memory plan."""
import json
import os
import re
import subprocess
import sys
import tempfile

import pytest
import torch
import torch.multiprocessing as mp

import test_engine_cpu as TE
import test_grad_accum_cpu as GA
from conftest import free_port
from fms_fsdp_b200 import ops
from fms_fsdp_b200.models.llama import LLaMA, LLaMAConfig
from fms_fsdp_b200.ops import torch_kernels as TK
from fms_fsdp_b200.utils.config_utils import get_model_config, list_model_variants

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------- oracle ops
def _reference(h, w, b, cos, sin, H, KVH, hd, scale):
    """Independent formula: y = h w^T + b; each q / k head's pairs (y[2i], y[2i+1]) rotated as the complex number
    y[2i] + i y[2i+1] times e^{i theta}; causal softmax attention with every KV head shared by H / KVH query heads."""
    B, S, _ = h.shape
    y = (h @ w.t() + b).view(B, S, H + 2 * KVH, hd)
    qk = torch.view_as_complex(y[:, :, :H + KVH].reshape(B, S, H + KVH, hd // 2, 2).contiguous())
    qk = torch.view_as_real(qk * torch.complex(cos, sin).view(1, S, 1, hd // 2)).reshape(B, S, H + KVH, hd)
    q, k, v = qk[:, :, :H], qk[:, :, H:], y[:, :, H + KVH:]
    g = H // KVH
    k, v = k.repeat_interleave(g, dim=2), v.repeat_interleave(g, dim=2)
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) * scale
    s = s.masked_fill(~torch.ones(S, S, dtype=torch.bool).tril(), float("-inf"))
    return torch.einsum("bhqk,bkhd->bqhd", s.softmax(-1), v).reshape(B, S, H * hd)


@pytest.mark.parametrize("H,KVH,hd", [(4, 2, 16), (4, 4, 32), (12, 2, 16), (14, 2, 16), (7, 1, 32)])
def test_oracle_node_matches_autograd_of_an_independent_fp64_reference(H, KVH, hd):
    """``qkv_attention(qkv_bias=)`` on the ATen oracle (bias + RoPE projection, attention, ``bias_grad``) against fp64
    autograd, GQA groups 1, 2, 6 and 7 included."""
    g = torch.Generator().manual_seed(hd + H)
    B, S, D = 2, 13, 24
    h = torch.randn(B, S, D, dtype=torch.float64, generator=g)
    w = torch.randn((H + 2 * KVH) * hd, D, dtype=torch.float64, generator=g) * D ** -0.5
    b = torch.randn((H + 2 * KVH) * hd, dtype=torch.float64, generator=g)          # non-zero biases
    table = TK.rope_table(S, hd, 1e6).double()
    cos, sin = table[:, :, 0], table[:, :, 1]
    do = torch.randn(B, S, H * hd, dtype=torch.float64, generator=g)

    ref_in = [t.clone().requires_grad_() for t in (h, w, b)]
    ref = _reference(*ref_in, cos, sin, H, KVH, hd, hd ** -0.5)
    ref_grads = torch.autograd.grad(ref, ref_in, do)

    ins = [t.clone().requires_grad_() for t in (h, w, b)]
    o = ops.qkv_attention(ins[0], ins[1], table, H, KVH, hd, qkv_bias=ins[2])
    grads = torch.autograd.grad(o, ins, do)
    assert type(o.grad_fn).__name__.startswith("_QKVAttention")
    # the oracle attention runs in fp32
    assert torch.allclose(o.double(), ref, rtol=1e-4, atol=1e-5)
    for name, a, r in zip(("dh", "dw", "db"), grads, ref_grads):
        assert torch.allclose(a.double(), r, rtol=1e-4, atol=1e-4 * r.abs().max().item()), name
    # the bias gradient is the column sum of the pre-RoPE projection's gradient
    dqkv = torch.randn(B * S, (H + 2 * KVH) * hd, dtype=torch.float64, generator=g)
    assert torch.allclose(TK.bias_grad(dqkv), dqkv.sum(0), rtol=1e-12)


def test_oracle_gemm_adds_the_bias_before_the_rotation():
    g = torch.Generator().manual_seed(5)
    H, KVH, hd, S = 2, 1, 8, 6
    x = torch.randn(2 * S, 16, generator=g)
    w = torch.randn((H + 2 * KVH) * hd, 16, generator=g)
    b = torch.randn((H + 2 * KVH) * hd, generator=g)
    table = TK.rope_table(S, hd, 1e4)
    y = TK.gemm(x, w, "nt", rope=(table, S, hd, H, KVH), bias=b)
    expect = TK.rope_(x @ w.t() + b, table, S, H, KVH, hd)
    assert torch.allclose(y, expect, atol=1e-5)
    rotated_then_biased = TK.rope_(x @ w.t(), table, S, H, KVH, hd) + b
    assert (y - rotated_then_biased).abs().max() > 1e-2


def test_qkv_attention_bias_none_keeps_the_plain_node_and_refuses_combinations():
    from fms_fsdp_b200.ops import functional as Fn
    torch.manual_seed(0)
    h = torch.randn(1, 8, 32, requires_grad=True)
    w = torch.randn(64 + 2 * 32, 32, requires_grad=True)
    b = torch.randn(64 + 2 * 32, requires_grad=True)
    table = TK.rope_table(8, 16)
    o = ops.qkv_attention(h, w, table, 4, 2, 16)
    assert type(o.grad_fn).__name__.startswith("_QKVAttention")
    o_b = ops.qkv_attention(h, w, table, 4, 2, 16, qkv_bias=b)
    assert type(o_b.grad_fn).__name__.startswith("_QKVAttention")
    assert (o_b - o).abs().max() > 1e-2
    gb = torch.autograd.grad(o_b.sum(), b)[0]
    assert gb.isfinite().all() and gb.abs().max() > 0
    ones = torch.ones(16), torch.ones(16)
    with pytest.raises(ValueError, match="qk_norm"):
        ops.qkv_attention(h, w, table, 4, 2, 16, qk_norm=(*ones, 1e-6), qkv_bias=b)
    old = Fn.get_gemm_precision()
    Fn.set_gemm_precision("fp8")
    try:
        with pytest.raises(NotImplementedError, match="fp8"):
            ops.qkv_attention(h, w, table, 4, 2, 16, qkv_bias=b)
    finally:
        Fn.set_gemm_precision(old)


# ------------------------------------------------------------------------------------------- Qwen2 round trip
def _tiny_qwen2(tmp_path, tie=False):
    from transformers import Qwen2Config, Qwen2ForCausalLM
    torch.manual_seed(0)
    hf = Qwen2ForCausalLM(Qwen2Config(vocab_size=96, hidden_size=64, intermediate_size=96, num_hidden_layers=2,
                                      num_attention_heads=4, num_key_value_heads=2, max_position_embeddings=64,
                                      rope_theta=50000.0, rms_norm_eps=1e-6, tie_word_embeddings=tie,
                                      use_sliding_window=False)).eval()
    with torch.no_grad():   # HF initialises the biases to zero, which would let a wrong bias layout pass
        for layer in hf.model.layers:
            for proj in (layer.self_attn.q_proj, layer.self_attn.k_proj, layer.self_attn.v_proj):
                proj.bias.normal_(0.0, 0.5)
    d = str(tmp_path / "qwen2")
    hf.save_pretrained(d)
    return hf, d


def _logits(model, x):
    with torch.no_grad():
        out = model(x)
    return getattr(out, "logits", out)


@pytest.mark.parametrize("tie", [False, True])
def test_qwen2_import_export_roundtrip_matches_transformers(tmp_path, tie):
    import fms_to_hf_llama as ex
    import hf_to_fms_llama as imp
    from transformers import Qwen2ForCausalLM
    from fms_fsdp_b200.models.hf_loader import _read_hf_tensors, config_from_hf, load_hf_llama
    hf, d = _tiny_qwen2(tmp_path, tie)
    assert hf.model.layers[0].self_attn.o_proj.bias is None
    x = torch.randint(0, 96, (2, 33), generator=torch.Generator().manual_seed(1))
    theirs = _logits(hf, x)

    m = load_hf_llama(d, dtype=torch.float32).eval()
    assert m.config.qkv_bias and not m.config.qk_norm
    assert torch.allclose(_logits(m, x), theirs, atol=2e-4, rtol=1e-3), (_logits(m, x) - theirs).abs().max()

    pth = str(tmp_path / "w" / "qwen2.pth")
    imp.main(d, pth, dtype="fp32")
    with open(os.path.join(d, "config.json")) as f:
        cfg = config_from_hf(json.load(f), _read_hf_tensors(d))
    m2 = LLaMA(cfg)
    m2.load_state_dict(torch.load(pth)["model_state"])           # strict: every key, the biases included
    assert torch.allclose(_logits(m2.eval(), x), theirs, atol=2e-4, rtol=1e-3)

    out = str(tmp_path / "export")
    ex.convert_to_hf(m2, "qwen2_test").save_pretrained(out)
    with open(os.path.join(out, "config.json")) as f:
        exported = json.load(f)
    assert exported["model_type"] == "qwen2" and not exported["tie_word_embeddings"]
    assert not exported["use_sliding_window"]
    back = Qwen2ForCausalLM.from_pretrained(out).eval()
    assert back.model.layers[0].self_attn.o_proj.bias is None
    assert torch.allclose(_logits(back, x), theirs, atol=2e-4, rtol=1e-3)


@pytest.mark.parametrize("wrong", ["unpermuted", "single_head"])
def test_qwen2_import_without_the_per_head_bias_permutation_is_wrong(tmp_path, monkeypatch, wrong):
    """The q / k biases must move head by head like their rows: left in half-split order, or permuted as if the whole
    [H * hd] bias were one head, the logits are wrong."""
    from fms_fsdp_b200.models import hf_loader
    hf, d = _tiny_qwen2(tmp_path)
    x = torch.randint(0, 96, (1, 20), generator=torch.Generator().manual_seed(2))
    right = hf_loader.load_hf_llama(d, dtype=torch.float32).eval()
    err = (_logits(right, x) - _logits(hf, x)).abs().max().item()
    assert err < 2e-5
    bad = (lambda b, n: b) if wrong == "unpermuted" else (lambda b, n: hf_loader._halfsplit_to_interleaved_vec(b))
    monkeypatch.setattr(hf_loader, "_halfsplit_to_interleaved_bias", bad)
    model = hf_loader.load_hf_llama(d, dtype=torch.float32).eval()
    # the tiny model's logits are about 0.3 in size: a wrong bias layout moves them by 1e-3 and more
    assert (_logits(model, x) - _logits(hf, x)).abs().max() > 1e-3


def test_hf_import_detects_qwen2_from_the_tensors_and_refuses_the_rest(tmp_path):
    from fms_fsdp_b200.models.hf_loader import _read_hf_tensors, config_from_hf, convert_hf_state_dict
    base = dict(hidden_size=64, intermediate_size=96, num_attention_heads=4, num_key_value_heads=2, num_hidden_layers=2,
                vocab_size=96, max_position_embeddings=64)
    biases = {f"model.layers.{i}.self_attn.{n}_proj.bias": torch.zeros(1) for i in range(2) for n in "qkv"}
    assert config_from_hf(dict(base, model_type="qwen2"), biases).qkv_bias
    assert config_from_hf(dict(base, model_type="qwen2", sliding_window=4096, use_sliding_window=False), biases).qkv_bias
    # the config alone cannot show the biases: refused, naming the model type
    with pytest.raises(NotImplementedError, match="qwen2"):
        config_from_hf(dict(base, model_type="qwen2"))
    # a layer without a v bias, or with an output bias, is not Qwen2 attention
    for bad in ({k: v for k, v in biases.items() if k != "model.layers.1.self_attn.v_proj.bias"},
                dict(biases, **{"model.layers.0.self_attn.o_proj.bias": torch.zeros(1)})):
        with pytest.raises(NotImplementedError, match="qwen2"):
            config_from_hf(dict(base, model_type="qwen2"), bad)
    with pytest.raises(NotImplementedError, match="sliding-window"):
        config_from_hf(dict(base, model_type="qwen2", sliding_window=32, use_sliding_window=True), biases)
    with pytest.raises(NotImplementedError, match="shared experts"):
        config_from_hf(dict(base, model_type="qwen2_moe"), biases)
    with pytest.raises(NotImplementedError, match="biases"):
        config_from_hf(dict(base, model_type="llama", attention_bias=True), biases)
    # the biases stay off for other model types, and a Llama config never turns them on
    assert not config_from_hf(dict(base, model_type="llama"), biases).qkv_bias
    # a Qwen2 checkpoint read with a bias-free config stops instead of dropping the biases
    _, d = _tiny_qwen2(tmp_path)
    cfg = LLaMAConfig(src_vocab_size=96, emb_dim=64, nheads=4, kvheads=2, nlayers=2, hidden_grow_factor=1.5, multiple_of=1)
    with pytest.raises(ValueError, match="q / k / v biases"):
        convert_hf_state_dict(_read_hf_tensors(d), cfg)


def test_hf_to_fms_checks_qkv_bias_against_the_variant(tmp_path):
    import hf_to_fms_llama as imp
    _, d = _tiny_qwen2(tmp_path)
    with pytest.raises(ValueError, match="qkv_bias"):
        imp.main(d, str(tmp_path / "x.pth"), model_variant="llama2_tiny")
    assert "qkv_bias" in imp._CHECKED


def test_llama_export_is_unchanged_without_qkv_bias():
    import fms_to_hf_llama as ex
    torch.manual_seed(0)
    m = LLaMA(LLaMAConfig(src_vocab_size=97, emb_dim=64, nheads=4, kvheads=2, nlayers=1, multiple_of=16,
                          max_expected_seq_len=64))
    m.reset_parameters()
    hf = ex.convert_to_hf(m, "llama2_x")
    assert type(hf).__name__ == "LlamaForCausalLM" and hf.model.layers[0].self_attn.q_proj.bias is None


# ---------------------------------------------------------------------------------------------- model / config
def test_bias_is_a_vector_slot_before_the_matrices_initialised_to_zero():
    """The bias must sit in the unit's vector prefix: that prefix is gathered before the carrier GEMM, while block 0's
    QKV GEMM runs in dependent fused-gather mode and would read a bias inside the matrix range before it arrives."""
    from fms_fsdp_b200.parallel import ShardedModel
    cfg = get_model_config("qwen2_tiny")
    with torch.device("meta"):
        m = LLaMA(cfg)
    eng = ShardedModel(m, device="cpu")                        # meta-device path: param_init_function per unit
    sd = eng.full_state_dict()
    N = (cfg.nheads + 2 * cfg.kv_heads) * cfg.head_dim
    for i in range(cfg.nlayers):
        assert torch.equal(sd[f"layers.{i}.attn.in_proj.qkv_fused.bias"], torch.zeros(N))
    for u in (u for u in eng.units if u.name.startswith("block")):
        slot = next(s for s in u.layout.slots if s.name.endswith("attn.in_proj.qkv_fused.bias"))
        assert slot.shape == (N,) and slot.offset + slot.numel <= u.layout.matrix_begin
    eager = LLaMA(cfg)
    eager.reset_parameters()
    assert torch.equal(eager.layers[0].attn.in_proj.qkv_fused.bias, torch.zeros(N))
    plain = LLaMA(get_model_config("llama2_tiny"))
    assert not any(k.endswith(".bias") for k in plain.state_dict())


QWEN25 = {   # emb_dim, ffn, layers, heads, kv heads, vocab; published non-embedding parameter counts (billions)
    "qwen2.5_0.5b": (896, 4864, 24, 14, 2, 151936, 0.36),
    "qwen2.5_1.5b": (1536, 8960, 28, 12, 2, 151936, 1.31),
    "qwen2.5_3b": (2048, 11008, 36, 16, 2, 151936, 2.77),
    "qwen2.5_7b": (3584, 18944, 28, 28, 4, 152064, 6.53),
}


@pytest.mark.parametrize("name", sorted(QWEN25))
def test_qwen25_zoo_entries(name):
    from fms_fsdp_b200.ops.cuda_kernels import push_eligible_shape
    D, F, L, H, KV, V, nonemb = QWEN25[name]
    c = get_model_config(name)
    assert name in list_model_variants() and not name.startswith("llama")
    assert (c.emb_dim, c.hidden_dim, c.nlayers, c.nheads, c.kv_heads, c.src_vocab_size) == (D, F, L, H, KV, V)
    assert (c.rope_theta, c.norm_eps, c.multiple_of, c.qkv_bias, c.qk_norm) == (1e6, 1e-6, 1, True, False)
    hd = c.head_dim
    assert hd in (64, 128) and F % 128 == 0 and D % 8 == 0 and V % 8 == 0 and H % KV == 0
    for shape in (((H + 2 * KV) * hd, D), (D, H * hd), (2 * F, D), (D, F), (V, D)):
        assert push_eligible_shape(shape), shape
    with torch.device("meta"):
        m = LLaMA(c)
    n = sum(p.numel() for p in m.parameters())
    block = D * (H + 2 * KV) * hd + (H + 2 * KV) * hd + H * hd * D + 3 * D * F + 2 * D
    assert n == L * block + 2 * V * D + D                          # untied embedding and head
    assert abs((n - 2 * V * D) / 1e9 - nonemb) < 0.01 * nonemb + 0.005


def test_memory_plan_adds_the_bias_bytes_only_with_biases():
    from fms_fsdp_b200.utils import config_utils
    from fms_fsdp_b200.utils import memory_plan as MP
    for v in list_model_variants():
        if v.startswith("llama"):
            assert not get_model_config(v).qkv_bias
    c = get_model_config("qwen2.5_1.5b")
    N = (c.nheads + 2 * c.kv_heads) * c.head_dim
    try:
        config_utils._LLAMA_ZOO["qwen2.5_1.5b_nobias"] = dict(config_utils._LLAMA_ZOO["qwen2.5_1.5b"], qkv_bias=False)
        for gpus, per_param in ((1, 14.0 + 2.0), (8, None)):
            with_b = MP.plan_llama("qwen2.5_1.5b", gpus=gpus)
            without = MP.plan_llama("qwen2.5_1.5b_nobias", gpus=gpus)
            diff = (with_b.total_gib - without.total_gib) * 2 ** 30
            if per_param is not None:
                assert diff == pytest.approx(c.nlayers * N * per_param, rel=1e-6)
            else:   # sharded: state / 8, fp32 gradient shard, and the gathered / staged bf16 block buffers
                assert diff == pytest.approx(c.nlayers * N * 18.0 / 8 + 2.0 * (2 + 3) * N, rel=1e-6)
    finally:
        del config_utils._LLAMA_ZOO["qwen2.5_1.5b_nobias"]


# --------------------------------------------------------------------------------------------- sharded engine
def _bias_config(variant):
    cfg = get_model_config(variant)
    cfg.qkv_bias = True
    return cfg


def _bias_doc_config(variant):
    cfg = _bias_config(variant)
    cfg.doc_separator = 1
    return cfg


def _te_worker(rank, doc, *args):
    TE.get_model_config = _bias_doc_config if doc else _bias_config
    if doc:
        TE._batch = _doc_batch
    TE._worker(rank, *args)


def _doc_batch(rank, step, _plain=TE._batch):
    x = _plain(rank, step)
    x[0, [0, 9, 10, TE.S - 1]] = 1
    x[1, [3 + 5 * step + rank, 20]] = 1
    return x


@pytest.mark.parametrize("ac,doc", [(None, False), ("1/2", False), ("1/2", True)])
def test_world2_fsdp_with_qkv_bias_matches_oracle(ac, doc, monkeypatch):
    outdir = tempfile.mkdtemp()
    mp.spawn(_te_worker, args=(doc, 2, free_port(), "fsdp", 0, ac, outdir, None), nprocs=2, join=True)
    out = torch.load(os.path.join(outdir, "out.pt"), weights_only=False)
    assert any(k.endswith("attn.in_proj.qkv_fused.bias") for k in out["sd"])
    monkeypatch.setattr(TE, "get_model_config", _bias_doc_config if doc else _bias_config)
    if doc:
        monkeypatch.setattr(TE, "_batch", _doc_batch)
    TE._check(out, 2)          # loss, grad norm and every parameter (the biases included) after 3 steps
    b = out["sd"]["layers.0.attn.in_proj.qkv_fused.bias"]
    assert b.abs().max() > 0   # the zero-initialised biases were trained


def _ga_model(kind, _orig=GA._model):
    if kind != "llama":
        return _orig(kind)
    torch.manual_seed(0)
    m = LLaMA(_bias_config("llama2_tiny"))
    m.reset_parameters()
    return m


def _ga_worker(*args):
    GA._model = _ga_model
    GA._worker(*args)


@pytest.mark.parametrize("strategy,ac", [("fsdp", None), ("ddp", "1/2")])
def test_world2_qkv_bias_with_gradient_accumulation_matches_the_big_batch(strategy, ac, monkeypatch):
    outdir = tempfile.mkdtemp()
    mp.spawn(_ga_worker, args=(2, free_port(), "llama", strategy, 0, ac, 2, "fused", outdir), nprocs=2, join=True)
    out = torch.load(os.path.join(outdir, "out.pt"), weights_only=False)
    monkeypatch.setattr(GA, "_model", _ga_model)
    GA._check(out, "llama", 2, 2)


# ----------------------------------------------------------------------------------------------- entry points
def test_llama_entry_point_trains_qwen2_tiny_and_the_checkpoint_exports(tmp_path):
    ckpt = str(tmp_path / "ckpt")
    cmd = [sys.executable, os.path.join(ROOT, "main_training_llama.py"), "--model_variant=qwen2_tiny",
           "--use_dummy_dataset=True", "--seq_length=32", "--vocab_size=1024", "--batch_size=2", "--num_steps=3",
           "--report_interval=1", "--checkpoint_interval=3", f"--ckpt_save_path={ckpt}", "--sharding_strategy=fsdp",
           "--comm_backend=gloo", "--use_torch_compile=False"]
    env = dict(os.environ, OMP_NUM_THREADS="1")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT, env=env)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    losses = [float(x) for x in re.findall(r"^loss: ([0-9.eE+-]+)$", r.stdout, flags=re.M)]
    assert len(losses) == 3 and all(l == l for l in losses)
    step = [p for p in os.listdir(os.path.join(ckpt, "checkpoints")) if p.startswith("step_")][0]

    import fms_to_hf_llama as ex
    from transformers import Qwen2ForCausalLM
    out = str(tmp_path / "hf")
    ex.main("qwen2_tiny", load_path=os.path.join(ckpt, "checkpoints", step), save_path=out)
    back = Qwen2ForCausalLM.from_pretrained(out).eval()
    assert back.model.layers[0].self_attn.q_proj.bias.abs().max() > 0     # trained, exported biases

    bad = subprocess.run(cmd + ["--precision=fp8"], capture_output=True, text=True, timeout=600, cwd=ROOT, env=env)
    assert bad.returncode != 0 and "projection biases" in bad.stdout + bad.stderr


def test_speculator_refuses_a_biased_base():
    sys.path.insert(0, os.path.join(ROOT, "speculator"))
    from speculator.train_speculator_utils import EmbedLLaMA
    cfg = LLaMAConfig(src_vocab_size=64, emb_dim=64, nheads=4, kvheads=2, nlayers=1, multiple_of=16, qkv_bias=True)
    with pytest.raises(NotImplementedError, match="projection biases"):
        EmbedLLaMA(cfg)
