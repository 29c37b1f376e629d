"""QK-norm (per-head RMSNorm of q and k before RoPE, Qwen3) on CPU: the ATen oracle ops against autograd of an independent
fp64 formula, the Qwen3 import / export round trip against transformers, the world-2 gloo engine against the
single-process oracle, the entry points, the speculator refusal, the qwen3_* zoo entries and the memory plan."""
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
def _reference(x, wq, wk, cos, sin, H, KVH, hd, eps):
    """Independent formula: [M, H+2KVH, hd] -> RMSNorm over each q / k head, gains, then (x[2i], x[2i+1]) rotated as the
    complex number x[2i] + i x[2i+1] times e^{i theta}; V passes through."""
    M = x.shape[0]
    t = x.view(M, H + 2 * KVH, hd)
    qk, v = t[:, :H + KVH], t[:, H + KVH:]
    w = torch.cat([wq.expand(H, hd), wk.expand(KVH, hd)])
    n = qk / torch.sqrt((qk * qk).mean(-1, keepdim=True) + eps) * w
    z = torch.view_as_complex(n.reshape(M, H + KVH, hd // 2, 2).contiguous())
    rot = torch.view_as_real(z * torch.complex(cos, sin).unsqueeze(1)).reshape(M, H + KVH, hd)
    return torch.cat([rot, v], dim=1).reshape(M, -1)


@pytest.mark.parametrize("H,KVH,hd", [(4, 2, 64), (4, 4, 64), (2, 1, 128), (3, 3, 128)])
def test_oracle_ops_match_autograd_of_an_independent_fp64_reference(H, KVH, hd):
    g = torch.Generator().manual_seed(hd + H)
    B, S, eps = 2, 11, 1e-6
    M = B * S
    x = torch.randn(M, (H + 2 * KVH) * hd, dtype=torch.float64, generator=g) * 3
    wq = 0.5 + torch.rand(hd, dtype=torch.float64, generator=g)          # random, non-unit gains
    wk = 0.5 + torch.rand(hd, dtype=torch.float64, generator=g)
    table = TK.rope_table(S, hd, 1e6).double()
    pos = torch.arange(M) % S
    cos, sin = table[pos, :, 0], table[pos, :, 1]

    leaves = [t.clone().requires_grad_() for t in (x, wq, wk)]
    ref = _reference(*leaves, cos, sin, H, KVH, hd, eps)
    dy = torch.randn(ref.shape, dtype=torch.float64, generator=g)
    rdx, rdwq, rdwk = torch.autograd.grad(ref, leaves, dy)

    y = x.clone()
    xqk, rstd = TK.qk_norm_rope(y, wq, wk, table, S, H, KVH, hd, eps)
    assert torch.allclose(y, ref.detach(), rtol=1e-10, atol=1e-10)
    assert torch.equal(xqk, x[:, :(H + KVH) * hd]) and rstd.shape == (M, H + KVH)
    # what the attention backward hands over: the gradient of the normed heads before rotation (inverse RoPE, in fp64)
    d = dy.clone()
    qk = d.view(M, H + 2 * KVH, hd)[:, :H + KVH]
    z = torch.view_as_complex(qk.reshape(M, H + KVH, hd // 2, 2).contiguous())
    qk.copy_(torch.view_as_real(z * torch.complex(cos, -sin).unsqueeze(1)).reshape(M, H + KVH, hd))
    dwq, dwk = TK.qk_norm_bwd(d, xqk, rstd, wq, wk, H, KVH, hd)
    assert torch.allclose(d, rdx, rtol=1e-9, atol=1e-10)
    assert torch.allclose(dwq, rdwq, rtol=1e-9, atol=1e-10) and torch.allclose(dwk, rdwk, rtol=1e-9, atol=1e-10)


def test_qkv_attention_qk_norm_none_keeps_the_plain_node():
    torch.manual_seed(0)
    h = torch.randn(1, 8, 32, requires_grad=True)
    w = torch.randn(64 + 2 * 32, 32, requires_grad=True)
    table = TK.rope_table(8, 16)
    o = ops.qkv_attention(h, w, table, 4, 2, 16)
    assert type(o.grad_fn).__name__.startswith("_QKVAttention")
    ones = torch.ones(16, requires_grad=True), torch.ones(16, requires_grad=True)
    o2 = ops.qkv_attention(h, w, table, 4, 2, 16, qk_norm=(*ones, 1e-6))
    assert type(o2.grad_fn).__name__.startswith("_QKNormAttention")
    grads = torch.autograd.grad(o2.sum(), (h, w, *ones))
    assert all(g is not None and g.isfinite().all() for g in grads)


# ------------------------------------------------------------------------------------------- Qwen3 round trip
def _tiny_qwen3(tmp_path, tie=False):
    from transformers import Qwen3Config, Qwen3ForCausalLM
    torch.manual_seed(0)
    hf = Qwen3ForCausalLM(Qwen3Config(vocab_size=96, hidden_size=64, intermediate_size=96, num_hidden_layers=2,
                                      num_attention_heads=4, num_key_value_heads=2, head_dim=32,   # hd != 64 / 4
                                      max_position_embeddings=64, rope_theta=50000.0, rms_norm_eps=1e-6,
                                      tie_word_embeddings=tie)).eval()
    with torch.no_grad():
        for layer in hf.model.layers:
            layer.self_attn.q_norm.weight.uniform_(0.3, 1.7)
            layer.self_attn.k_norm.weight.uniform_(0.3, 1.7)
    d = str(tmp_path / "qwen3")
    hf.save_pretrained(d)
    return hf, d


def _logits(model, x):
    with torch.no_grad():
        out = model(x)
    return getattr(out, "logits", out)


@pytest.mark.parametrize("tie", [False, True])
def test_qwen3_import_export_roundtrip_matches_transformers(tmp_path, tie):
    import fms_to_hf_llama as ex
    import hf_to_fms_llama as imp
    from transformers import Qwen3ForCausalLM
    from fms_fsdp_b200.models.hf_loader import config_from_hf, load_hf_llama
    hf, d = _tiny_qwen3(tmp_path, tie)
    x = torch.randint(0, 96, (2, 33), generator=torch.Generator().manual_seed(1))
    theirs = _logits(hf, x)

    m = load_hf_llama(d, dtype=torch.float32).eval()
    assert m.config.qk_norm and m.config.head_dim == 32 and m.config.attn_head_dim == 32
    assert torch.allclose(_logits(m, x), theirs, atol=2e-4, rtol=1e-3), (_logits(m, x) - theirs).abs().max()

    pth = str(tmp_path / "w" / "qwen3.pth")
    imp.main(d, pth, dtype="fp32")
    with open(os.path.join(d, "config.json")) as f:
        cfg = config_from_hf(json.load(f))
    m2 = LLaMA(cfg)
    m2.load_state_dict(torch.load(pth)["model_state"])           # strict: every key, including q_norm / k_norm
    assert torch.allclose(_logits(m2.eval(), x), theirs, atol=2e-4, rtol=1e-3)

    out = str(tmp_path / "export")
    ex.convert_to_hf(m2, "qwen3_test").save_pretrained(out)
    with open(os.path.join(out, "config.json")) as f:
        exported = json.load(f)
    assert exported["model_type"] == "qwen3" and exported["head_dim"] == 32 and not exported["tie_word_embeddings"]
    back = Qwen3ForCausalLM.from_pretrained(out).eval()
    assert torch.allclose(_logits(back, x), theirs, atol=2e-4, rtol=1e-3)


def test_qwen3_import_without_the_norm_permutation_is_wrong(tmp_path, monkeypatch):
    """The q / k rows go from half-split to interleaved order; the per-head gains must follow them."""
    from fms_fsdp_b200.models import hf_loader
    hf, d = _tiny_qwen3(tmp_path)
    x = torch.randint(0, 96, (1, 20), generator=torch.Generator().manual_seed(2))
    monkeypatch.setattr(hf_loader, "_halfsplit_to_interleaved_vec", lambda w: w)
    wrong = hf_loader.load_hf_llama(d, dtype=torch.float32).eval()
    assert (_logits(wrong, x) - _logits(hf, x)).abs().max() > 1e-2


def test_hf_import_detects_and_refuses(tmp_path):
    from fms_fsdp_b200.models.hf_loader import config_from_hf, convert_hf_state_dict
    base = dict(hidden_size=64, intermediate_size=96, num_attention_heads=4, num_key_value_heads=2, num_hidden_layers=1,
                vocab_size=96, max_position_embeddings=64)
    # a q_norm tensor turns QK-norm on whatever model_type says; one over the whole projection (OLMo 2 style) is refused
    per_head = {"model.layers.0.self_attn.q_norm.weight": torch.ones(16)}
    assert config_from_hf(dict(base, model_type="llama"), per_head).qk_norm
    with pytest.raises(NotImplementedError, match="per-head"):
        config_from_hf(dict(base, model_type="llama"), {"model.layers.0.self_attn.q_norm.weight": torch.ones(64)})
    for kind in ("olmo2", "qwen2", "qwen3_moe"):
        with pytest.raises(NotImplementedError, match=kind):
            config_from_hf(dict(base, model_type=kind))
    with pytest.raises(NotImplementedError, match="sliding-window"):
        config_from_hf(dict(base, model_type="qwen3", sliding_window=32, use_sliding_window=True))
    assert config_from_hf(dict(base, model_type="qwen3", sliding_window=32, use_sliding_window=False)).qk_norm
    assert not config_from_hf(dict(base, model_type="llama")).qk_norm
    # a Qwen3 checkpoint read with a config that has no QK-norm stops instead of dropping the gains
    hf, d = _tiny_qwen3(tmp_path)
    from fms_fsdp_b200.models.hf_loader import _read_hf_tensors
    cfg = LLaMAConfig(src_vocab_size=96, emb_dim=64, nheads=4, kvheads=2, nlayers=2, hidden_grow_factor=1.5, multiple_of=1,
                      attn_head_dim=32)
    with pytest.raises(ValueError, match="q / k norm"):
        convert_hf_state_dict(_read_hf_tensors(d), cfg)


def test_hf_to_fms_checks_qk_norm_and_head_dim_against_the_variant(tmp_path):
    import hf_to_fms_llama as imp
    hf, d = _tiny_qwen3(tmp_path)
    with pytest.raises(ValueError, match="qk_norm|head_dim"):
        imp.main(d, str(tmp_path / "x.pth"), model_variant="llama2_tiny")
    assert "qk_norm" in imp._CHECKED and "head_dim" in imp._CHECKED


def test_llama_export_is_unchanged_without_qk_norm():
    import fms_to_hf_llama as ex
    torch.manual_seed(0)
    m = LLaMA(LLaMAConfig(src_vocab_size=97, emb_dim=64, nheads=4, kvheads=2, nlayers=1, multiple_of=16,
                          max_expected_seq_len=64))
    m.reset_parameters()
    hf = ex.convert_to_hf(m, "llama2_x")
    assert type(hf).__name__ == "LlamaForCausalLM" and hf.config.head_dim == 16


# ---------------------------------------------------------------------------------------------- model / config
def test_norm_weights_are_block_parameters_initialised_to_one():
    cfg = get_model_config("llama2_tiny")
    cfg.qk_norm = True
    with torch.device("meta"):
        m = LLaMA(cfg)
    from fms_fsdp_b200.parallel import ShardedModel
    eng = ShardedModel(m, device="cpu")                        # meta-device path: param_init_function per unit
    sd = eng.full_state_dict()
    for i in range(cfg.nlayers):
        for n in ("q_norm", "k_norm"):
            assert torch.equal(sd[f"layers.{i}.attn.{n}.weight"], torch.ones(cfg.head_dim))
    blocks = [u for u in eng.units if u.name.startswith("block")]
    assert all(any(n.endswith("attn.q_norm.weight") for n, _ in u.params) for u in blocks)
    plain = LLaMA(get_model_config("llama2_tiny"))
    assert not any("q_norm" in k for k in plain.state_dict())


QWEN3 = {   # emb_dim, ffn, layers, heads, kv heads; published non-embedding parameter counts (billions)
    "qwen3_0.6b": (1024, 3072, 28, 16, 8, 0.44),
    "qwen3_1.7b": (2048, 6144, 28, 16, 8, 1.4),
    "qwen3_4b": (2560, 9728, 36, 32, 8, 3.6),
    "qwen3_8b": (4096, 12288, 36, 32, 8, 6.95),
}


@pytest.mark.parametrize("name", sorted(QWEN3))
def test_qwen3_zoo_entries(name):
    from fms_fsdp_b200.ops.cuda_kernels import push_eligible_shape
    D, F, L, H, KV, nonemb = QWEN3[name]
    c = get_model_config(name)
    assert name in list_model_variants()
    assert (c.emb_dim, c.hidden_dim, c.nlayers, c.nheads, c.kv_heads) == (D, F, L, H, KV)
    assert (c.src_vocab_size, c.head_dim, c.rope_theta, c.norm_eps, c.max_expected_seq_len, c.qk_norm) == \
        (151936, 128, 1e6, 1e-6, 40960, True)
    # the native-kernel shape rules of tests/test_config.py
    hd = c.head_dim
    assert hd in (64, 128) and c.emb_dim % 8 == 0 and c.emb_dim <= 8192 and c.hidden_dim % 128 == 0
    assert c.src_vocab_size % 8 == 0 and c.nheads % c.kv_heads == 0
    for shape in ((c.nheads * hd + 2 * c.kv_heads * hd, c.emb_dim), (c.emb_dim, c.nheads * hd),
                  (2 * c.hidden_dim, c.emb_dim), (c.emb_dim, c.hidden_dim), (c.src_vocab_size, c.emb_dim)):
        assert push_eligible_shape(shape), shape
    with torch.device("meta"):
        m = LLaMA(c)
    n = sum(p.numel() for p in m.parameters())
    block = D * (H + 2 * KV) * hd + H * hd * D + 3 * D * F + 2 * D + 2 * hd
    assert n == L * block + 2 * 151936 * D + D                     # untied embedding and head
    assert abs((n - 2 * 151936 * D) / 1e9 - nonemb) < 0.01 * nonemb + 0.005


def test_memory_plan_adds_the_qk_norm_bytes_only_with_qk_norm():
    from fms_fsdp_b200.utils import memory_plan as MP
    llamas = [v for v in list_model_variants() if v.startswith("llama")]
    # the llama variants: unchanged (this is the plan before QK-norm, with 6D for the q section and attention output)
    for v in llamas:
        c = get_model_config(v)
        assert not c.qk_norm and c.nheads * c.head_dim == c.emb_dim
    assert abs(MP.plan_llama("llama2_1.4b").total_gib - 31.1807) < 1e-3

    from fms_fsdp_b200.utils import config_utils
    cfg = get_model_config("llama2_1.4b")
    base = MP.plan_llama("llama2_1.4b", batch_size=2, seq_length=4096)
    try:
        config_utils._LLAMA_ZOO["llama2_1.4b_qk"] = dict(config_utils._LLAMA_ZOO["llama2_1.4b"], qk_norm=True)
        qk = MP.plan_llama("llama2_1.4b_qk", batch_size=2, seq_length=4096)
    finally:
        del config_utils._LLAMA_ZOO["llama2_1.4b_qk"]
    T, nh, hd = 2 * 4096, cfg.nheads + cfg.kv_heads, cfg.head_dim
    act = 2.0 * T * nh * hd + 4.0 * T * nh                            # pre-norm q / k (bf16) + rstd (fp32)
    state = (14.0 + 2.0) * 2 * hd * cfg.nlayers                       # two norm vectors per block
    assert (qk.total_gib - base.total_gib) * 2 ** 30 == pytest.approx(cfg.nlayers * act + state, rel=1e-6)


# --------------------------------------------------------------------------------------------- sharded engine
def _qk_config(variant):
    cfg = get_model_config(variant)
    cfg.qk_norm = True
    return cfg


def _qk_doc_config(variant):
    cfg = _qk_config(variant)
    cfg.doc_separator = 1
    return cfg


def _te_worker(rank, doc, *args):
    TE.get_model_config = _qk_doc_config if doc else _qk_config
    if doc:
        TE._batch = _doc_batch
    TE._worker(rank, *args)


def _doc_batch(rank, step, _plain=TE._batch):
    x = _plain(rank, step)
    x[0, [0, 9, 10, TE.S - 1]] = 1
    x[1, [3 + 5 * step + rank, 20]] = 1
    return x


@pytest.mark.parametrize("ac,doc", [(None, False), ("1/2", False), ("1/2", True)])
def test_world2_fsdp_with_qk_norm_matches_oracle(ac, doc, monkeypatch):
    outdir = tempfile.mkdtemp()
    mp.spawn(_te_worker, args=(doc, 2, free_port(), "fsdp", 0, ac, outdir, None), nprocs=2, join=True)
    out = torch.load(os.path.join(outdir, "out.pt"), weights_only=False)
    assert any(k.endswith("attn.q_norm.weight") for k in out["sd"])
    monkeypatch.setattr(TE, "get_model_config", _qk_doc_config if doc else _qk_config)
    if doc:
        monkeypatch.setattr(TE, "_batch", _doc_batch)
    TE._check(out, 2)          # loss, grad norm and every parameter (q_norm / k_norm included) after 3 steps
    q = out["sd"]["layers.0.attn.q_norm.weight"]
    assert not torch.equal(q, torch.ones_like(q))


def _ga_model(kind, _orig=GA._model):
    if kind != "llama":
        return _orig(kind)
    torch.manual_seed(0)
    m = LLaMA(_qk_config("llama2_tiny"))
    m.reset_parameters()
    return m


def _ga_worker(*args):
    GA._model = _ga_model
    GA._worker(*args)


@pytest.mark.parametrize("strategy,ac", [("fsdp", None), ("ddp", "1/2")])
def test_world2_qk_norm_with_gradient_accumulation_matches_the_big_batch(strategy, ac, monkeypatch):
    outdir = tempfile.mkdtemp()
    mp.spawn(_ga_worker, args=(2, free_port(), "llama", strategy, 0, ac, 2, "fused", outdir), nprocs=2, join=True)
    out = torch.load(os.path.join(outdir, "out.pt"), weights_only=False)
    monkeypatch.setattr(GA, "_model", _ga_model)
    GA._check(out, "llama", 2, 2)


# ----------------------------------------------------------------------------------------------- entry points
def test_llama_entry_point_trains_with_qk_norm(tmp_path):
    ckpt = str(tmp_path / "ckpt")
    cmd = [sys.executable, os.path.join(ROOT, "main_training_llama.py"), "--model_variant=llama2_tiny",
           "--use_dummy_dataset=True", "--seq_length=32", "--vocab_size=1024", "--batch_size=2", "--num_steps=3",
           "--report_interval=1", "--checkpoint_interval=3", f"--ckpt_save_path={ckpt}", "--sharding_strategy=fsdp",
           "--comm_backend=gloo", "--use_torch_compile=False", "--qk_norm=True"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT, env=dict(os.environ, OMP_NUM_THREADS="1"))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    losses = [float(x) for x in re.findall(r"^loss: ([0-9.eE+-]+)$", r.stdout, flags=re.M)]
    assert len(losses) == 3 and all(l == l for l in losses)
    from torch.distributed.checkpoint import FileSystemReader
    step = [p for p in os.listdir(os.path.join(ckpt, "checkpoints")) if p.startswith("step_")][0]
    keys = FileSystemReader(os.path.join(ckpt, "checkpoints", step)).read_metadata().state_dict_metadata.keys()
    assert "model_state.layers.0.attn.q_norm.weight" in keys and "model_state.layers.1.attn.k_norm.weight" in keys


def test_mamba_entry_point_rejects_qk_norm():
    import main_training_mamba
    with pytest.raises(ValueError, match="qk_norm"):
        main_training_mamba.main(model_variant="mamba_tiny", qk_norm=True)


def test_speculator_refuses_a_qk_norm_base():
    sys.path.insert(0, os.path.join(ROOT, "speculator"))
    from speculator.train_speculator_utils import EmbedLLaMA
    cfg = LLaMAConfig(src_vocab_size=64, emb_dim=64, nheads=4, kvheads=2, nlayers=1, multiple_of=16, qk_norm=True)
    with pytest.raises(NotImplementedError, match="QK-norm"):
        EmbedLLaMA(cfg)
    cfg = LLaMAConfig(src_vocab_size=64, emb_dim=64, nheads=4, kvheads=2, nlayers=1, multiple_of=16, attn_head_dim=32)
    with pytest.raises(NotImplementedError, match="head_dim"):
        EmbedLLaMA(cfg)
    EmbedLLaMA(LLaMAConfig(src_vocab_size=64, emb_dim=64, nheads=4, kvheads=2, nlayers=1, multiple_of=16))
