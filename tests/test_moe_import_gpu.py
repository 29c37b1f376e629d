"""Qwen3-MoE and Mixtral checkpoints imported into the CUDA kernels against ``transformers``: the logits of two
truncated blocks at full width in bf16 against the same weights in float64, row by row, and one engine step
(``ShardedModel`` + ``ShardedAdamW``) of the Qwen3-MoE truncation against fp32 autograd in loss and in the router and
expert gradients, mapped through the converter.

Routing is discrete: a token whose k-th and (k+1)-th router logits are closer than the bf16 error can pick a different
expert in bf16 than in float64, and that one flip outweighs every rounding error of its row.  The checkpoints are
therefore built with a peaked router: token v's embedding points along the router rows of k experts of its own (the
rows orthonormal), so each token's top-k stands well clear of the rest.  The tests assert that margin in float64, per
token and layer, before they compare anything."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"

V, L = 32000, 2                                       # vocabulary cut to 32000, two blocks
QWEN3 = dict(family="qwen3_moe", D=2048, H=32, KV=4, hd=128, E=128, k=8, F=768)
MIXTRAL = dict(family="mixtral", D=4096, H=32, KV=8, hd=128, E=8, k=2, F=14336)
B, S = 2, 2048                                        # 4096 tokens

# about twice what one H100 80GB HBM3 measured (DESIGN.md §5): worst row 4.6e-3 (Qwen3-MoE) / 5.2e-3 (Mixtral), loss
# 1.0e-5, router 7.6e-3 and experts 6.8e-3 in relative Frobenius norm
TOL = {"logits_row": 1e-2, "loss": 1e-4, "grad_router": 1.5e-2, "grad_experts": 1.5e-2}


@pytest.fixture(scope="module")
def ck():
    from fms_fsdp_b200.ops import cuda_kernels
    assert cuda_kernels._C.__file__.endswith("_C.so")
    return cuda_kernels


def _hf(s, seed=0):
    """The ``transformers`` model of shape ``s`` on the GPU in fp32 holding bf16-representable weights: HF's
    initialisation (std 0.02), random q / k norm gains, and the peaked router described above (logit about 8 on the
    token's k experts, within about 1 of 0 elsewhere)."""
    from transformers import MixtralConfig, MixtralForCausalLM, Qwen3MoeConfig, Qwen3MoeForCausalLM
    D, E, k = s["D"], s["E"], s["k"]
    kw = dict(vocab_size=V, hidden_size=D, num_hidden_layers=L, num_attention_heads=s["H"], num_key_value_heads=s["KV"],
              head_dim=s["hd"], num_experts_per_tok=k, max_position_embeddings=S, rope_theta=1e6, rms_norm_eps=1e-6,
              tie_word_embeddings=False, attn_implementation="eager", experts_implementation="eager")
    if s["family"] == "qwen3_moe":
        cfg = Qwen3MoeConfig(**kw, intermediate_size=6144, moe_intermediate_size=s["F"], num_experts=E,
                             norm_topk_prob=True)
        cls = Qwen3MoeForCausalLM
    else:
        cfg = MixtralConfig(**kw, intermediate_size=s["F"], num_local_experts=E)
        cls = MixtralForCausalLM
    torch.manual_seed(seed)
    with torch.device(DEV):
        hf = cls(cfg).eval()
    g = torch.Generator(device=DEV).manual_seed(seed)
    U = torch.linalg.qr(torch.randn(D, E, device=DEV, generator=g)).Q.t()           # [E, D], orthonormal rows
    own = torch.rand(V, E, device=DEV, generator=g).topk(k, dim=1).indices           # token v's k experts
    with torch.no_grad():
        # residual stream rms about 4: attention and expert outputs (rms about 1) leave its direction mostly alone
        emb = 4 * math.sqrt(D / k) * U[own].sum(1) + 0.5 * torch.randn(V, D, device=DEV, generator=g)
        hf.model.embed_tokens.weight.copy_(emb)
        for layer in hf.model.layers:
            layer.mlp.gate.weight.copy_(8 / math.sqrt(D / k) * U)
            if s["family"] == "qwen3_moe":
                layer.self_attn.q_norm.weight.uniform_(0.5, 1.5, generator=g)
                layer.self_attn.k_norm.weight.uniform_(0.5, 1.5, generator=g)
        for p in hf.parameters():
            p.copy_(p.bfloat16())
    return hf


def _import(hf):
    from fms_fsdp_b200.models.hf_loader import config_from_hf, convert_hf_state_dict
    cfg = config_from_hf(hf.config.to_dict())
    sd = convert_hf_state_dict({k: v.detach().bfloat16() for k, v in hf.state_dict().items()}, cfg)
    return cfg, sd


def _router_margins(hf, x):
    """float64 forward of ``hf``; per layer, every token's k-th minus (k+1)-th router logit and a bound on its bf16
    error: eight roundings (2^-8 each) of the dot product's absolute terms, sum_d |h_d w_ed|, at the token's largest."""
    k = hf.config.num_experts_per_tok
    out = []

    def hook(mod, inp, _):
        h = inp[0].reshape(-1, inp[0].shape[-1])
        top = (h @ mod.weight.t()).topk(k + 1, dim=1).values
        bound = 8 * 2.0 ** -8 * (h.abs() @ mod.weight.abs().t()).max(1).values
        out.append((top[:, k - 1] - top[:, k], bound))

    hooks = [layer.mlp.gate.register_forward_hook(hook) for layer in hf.model.layers]
    try:
        with torch.no_grad():
            logits = hf(x).logits
    finally:
        for hk in hooks:
            hk.remove()
    return logits, out


@pytest.mark.parametrize("shape", [QWEN3, MIXTRAL], ids=["qwen3_30b_a3b", "mixtral_8x7b"])
def test_imported_logits_match_transformers_in_float64(ck, shape):
    from fms_fsdp_b200.models.llama import LLaMA
    hf = _hf(shape)
    cfg, sd = _import(hf)
    with torch.device("meta"):
        m = LLaMA(cfg)
    m.to_empty(device=DEV)
    m.load_state_dict(sd)
    m = m.to(torch.bfloat16).eval()
    del sd
    x = torch.randint(0, V, (B, S), generator=torch.Generator().manual_seed(1)).to(DEV)
    ck.reset_fallback_count()
    with torch.no_grad():
        ours = m(x).double().view(B * S, V)
    assert ck.fallback_count() == 0
    del m
    torch.cuda.empty_cache()

    ref, margins = _router_margins(hf.double(), x)
    for i, (margin, bound) in enumerate(margins):
        assert (margin > bound).all(), (i, (margin - bound).min().item())
    ref = ref.view(B * S, V)
    row = ((ours - ref).norm(dim=1) / ref.norm(dim=1)).max().item()
    print(f"[moe import {shape['family']}] min margin {min(m.min().item() for m, _ in margins):.3f}, max bound "
          f"{max(b.max().item() for _, b in margins):.3f}, worst row relative error {row:.3e}")
    assert row < TOL["logits_row"]


def test_engine_step_of_imported_qwen3_moe_matches_transformers_autograd(ck):
    from fms_fsdp_b200.models.hf_loader import convert_hf_state_dict
    from fms_fsdp_b200.models.llama import LLaMA
    from fms_fsdp_b200.parallel import ShardedAdamW, ShardedModel
    from fms_fsdp_b200.policies import bfSixteen
    hf = _hf(QWEN3, seed=2)
    cfg, sd = _import(hf)
    cfg.moe_aux_loss_coef = 0.0
    with torch.device("meta"):
        m = LLaMA(cfg)
    eng = ShardedModel(m, sharding_strategy="fsdp", mixed_precision=bfSixteen, device=torch.device(DEV, 0))
    eng.load_full_state_dict(sd)
    opt = ShardedAdamW(eng, lr=1e-4)
    del sd
    g = torch.Generator().manual_seed(3)
    x = torch.randint(0, V, (1, S), generator=g).to(DEV)
    labels = torch.randint(0, V, (1, S), generator=g).to(DEV)

    ck.reset_fallback_count()
    loss = float(eng.forward_backward(x, labels))
    assert ck.fallback_count() == 0
    torch.cuda.synchronize()
    ours = {}
    for u in eng.units:
        for name, v in eng.named_unit_views(u, u.grad_shard.float()):
            ours[name] = v.clone()
    before = eng.full_state_dict(cpu=False)
    opt.step()
    after = eng.full_state_dict(cpu=False)

    hf.train()
    logits = hf(x).logits
    want = torch.nn.functional.cross_entropy(logits.float().view(-1, V), labels.view(-1))
    want.backward()
    grads = convert_hf_state_dict({n: p.grad for n, p in hf.named_parameters()}, cfg)
    rel = lambda a, b: ((a.float() - b.float()).norm() / b.float().norm()).item()          # noqa: E731
    err = {"loss": abs(loss - want.item()) / want.item(),
           "grad_router": max(rel(ours[f"layers.{i}.moe.gate.weight"], grads[f"layers.{i}.moe.gate.weight"]) for i in range(L)),
           "grad_experts": max(rel(ours[f"layers.{i}.moe.{w}"], grads[f"layers.{i}.moe.{w}"])
                               for i in range(L) for w in ("w1", "w2"))}
    print(f"[moe import engine step] loss {loss:.6f} vs {want.item():.6f}, {err}")
    for key, e in err.items():
        assert e < TOL[key], (key, e)
    for i in range(L):                        # the optimizer moved the router and the experts
        for w in ("moe.gate.weight", "moe.w1", "moe.w2"):
            name = f"layers.{i}.{w}"
            assert after[name].isfinite().all() and not torch.equal(after[name], before[name]), name
