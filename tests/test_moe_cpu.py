"""Mixture of experts on CPU: the ATen oracle primitives against autograd of independent fp64 formulas built from dense
one-hot masks, ``ops.moe_mlp`` against a per-expert loop, the MoE Llama on the world-2 gloo engine against the
single-process oracle, and the zoo entries."""
import os
import tempfile

import pytest
import torch
import torch.multiprocessing as mp

import test_engine_cpu as TE
from conftest import free_port
from fms_fsdp_b200 import ops
from fms_fsdp_b200.models.llama import LLaMA
from fms_fsdp_b200.ops import torch_kernels as TK
from fms_fsdp_b200.utils.config_utils import get_model_config, list_model_variants


def _onehot_topk(logits, k):
    """[T, E] 0/1 mask of the k largest logits, ties to the lower index (selection by repeated argmax)."""
    T, E = logits.shape
    mask = torch.zeros(T, E, dtype=torch.float64)
    l = logits.detach().clone().double()
    order = torch.arange(E, dtype=torch.float64)
    for _ in range(k):
        best = l.max(1, keepdim=True).values
        first = torch.where(l == best, order, torch.full_like(order, E)).argmin(1)
        mask[torch.arange(T), first] = 1
        l[torch.arange(T), first] = -float("inf")
    return mask


@pytest.mark.parametrize("norm", [False, True])
def test_route_matches_dense_formula_and_breaks_ties_low(norm):
    torch.manual_seed(0)
    T, E, k = 50, 16, 4
    lg = torch.randn(T, E)
    lg[:10] = 0.0                                  # all tied: experts 0..k-1
    lg[10:20, 3] = lg[10:20, 7] = 5.0              # a tie for the top slot: 3 before 7
    ids, w, p = TK.moe_route(lg, k, norm)
    assert torch.equal(ids[:10], torch.arange(k, dtype=torch.int32).expand(10, k))
    assert torch.equal(ids[10:20, :2], torch.tensor([3, 7], dtype=torch.int32).expand(10, 2))
    mask = _onehot_topk(lg, k)
    pd = torch.softmax(lg.double(), -1)
    wd = pd * mask
    if norm:
        wd = wd / wd.sum(1, keepdim=True)
    dense = torch.zeros(T, E, dtype=torch.float64).scatter_(1, ids.long(), w.double())
    torch.testing.assert_close(dense, wd, rtol=1e-6, atol=1e-7)
    torch.testing.assert_close(p.double(), pd, rtol=1e-6, atol=1e-7)


def test_route_with_nan_and_inf_logits_keeps_ids_in_range_and_propagates_the_nan():
    T, E, k = 6, 16, 4
    lg = torch.randn(T, E)
    lg[0] = float("nan")                            # every logit NaN
    lg[1] = -float("inf")                           # every logit -inf
    lg[2, :E - 1] = float("nan")                    # one finite logit among NaNs
    lg[3, ::2] = float("nan")
    ids, w, p = TK.moe_route(lg, k, True)
    assert bool(((ids >= 0) & (ids < E)).all())
    for t in range(T):
        assert len(set(ids[t].tolist())) == k       # k distinct experts
    assert torch.equal(ids[0], torch.arange(k, dtype=torch.int32)) and torch.equal(ids[1], ids[0])
    assert int(ids[2, 0]) == E - 1
    assert bool(torch.isnan(w[0]).all()) and bool(torch.isnan(w[3]).all())
    assert bool(torch.isfinite(w[4:]).all())
    plan, _ = TK.moe_plan(ids, p)                   # a valid plan whatever the logits
    assert int(TK.moe_plan_views(plan, T, k, E)[2].sum()) == T * k
    h = torch.randn(T, 8)
    h[0, 3] = float("nan")
    y, _ = ops.moe_mlp(h, torch.randn(E, 8), torch.randn(E, 128, 8), torch.randn(E, 8, 64), k, True)
    assert bool(torch.isnan(y[0]).all()) and bool(torch.isfinite(y[1:]).all())


@pytest.mark.parametrize("T,E,k", [(37, 8, 2), (300, 16, 4), (5, 64, 8)])
def test_plan_layout(T, E, k):
    torch.manual_seed(T)
    lg = torch.randn(T, E)
    lg[:, E // 2:] -= 100.0                         # half the experts stay empty
    ids, _, probs = TK.moe_route(lg, k, False)
    plan, aux = TK.moe_plan(ids, probs)
    Mpad, NT = TK.moe_rows(T, k, E)
    assert Mpad % 128 == 0 and Mpad >= T * k + 127 * E
    tile, start, length, row, src = TK.moe_plan_views(plan, T, k, E)
    count = torch.bincount(ids.reshape(-1).long(), minlength=E)
    assert torch.equal(length.long(), count)
    padded = (count + 127) // 128 * 128
    assert torch.equal(start.long(), torch.cumsum(padded, 0) - padded) and bool((start % 128 == 0).all())
    for e in range(E):                              # rows of e: its segment, in (token, slot) order
        r = row.reshape(-1)[ids.reshape(-1) == e].long()
        assert torch.equal(r, start[e].long() + torch.arange(int(count[e])))
    used = int(padded.sum()) // 128
    assert bool((tile[used:] == -1).all())
    for i in range(used):
        e = int(tile[i])
        assert start[e] <= i * 128 < start[e] + padded[e]
    assert torch.equal(src[row.reshape(-1).long()].long(), torch.arange(T * k))
    pd = probs.double()
    ref = E * ((count.double() / T) * pd.mean(0)).sum()
    torch.testing.assert_close(aux.double(), ref, rtol=1e-5, atol=0)


def test_permute_combine_and_route_backward_match_autograd_of_the_dense_formula():
    """y = residual + sum_e (W_e ⊙ mask) · f(x W_e-ish) is written densely: every token times every expert, masked by
    the one-hot routing.  The oracle's permute -> per-row op -> combine chain and its backward (permute_bwd,
    combine_bwd, route_bwd with the auxiliary gradient) must give the same values and gradients."""
    torch.manual_seed(1)
    T, E, k, D = 29, 8, 3, 16
    for norm in (False, True):
        h = torch.randn(T, D, dtype=torch.float64, requires_grad=True)
        wr = torch.randn(E, D, dtype=torch.float64, requires_grad=True)
        scale = torch.randn(E, D, dtype=torch.float64)          # expert e: x -> tanh(x) * scale_e
        coef = 0.3
        # dense reference
        lg = h @ wr.t()
        mask = _onehot_topk(lg, k)
        p = torch.softmax(lg, -1)
        w = p * mask
        if norm:
            w = w / w.sum(1, keepdim=True)
        ye = torch.tanh(h)[:, None, :] * scale[None]             # [T, E, D]
        y_ref = (w[:, :, None] * ye).sum(1)
        aux_ref = E * ((mask.sum(0) / T) * p.mean(0)).sum()
        dy = torch.randn(T, D, dtype=torch.float64)
        (y_ref * dy).sum().backward(inputs=[h, wr], retain_graph=True)
        g_ref = [h.grad.clone(), wr.grad.clone()]
        h.grad = wr.grad = None
        (coef * aux_ref).backward(inputs=[h, wr])
        g_ref = [a + b for a, b in zip(g_ref, [h.grad, wr.grad])]
        # oracle primitives, backward by hand
        with torch.no_grad():
            logits = h @ wr.t()
            ids, wts, probs = TK.moe_route(logits, k, norm)
            plan, aux = TK.moe_plan(ids, probs)
            xp = TK.moe_permute(h, plan, k, E)
            tile = TK.moe_plan_views(plan, T, k, E)[0]
            e_row = torch.where(tile >= 0, tile, 0).long().repeat_interleave(128)
            yp = torch.tanh(xp) * scale[e_row]
            y = TK.moe_combine(yp, plan, wts, None, E)
            dyp, dw = TK.moe_combine_bwd(dy, yp, plan, wts, E)
            dxp = dyp * (1 - torch.tanh(xp) ** 2) * scale[e_row]
            dh = TK.moe_permute_bwd(dxp, plan, T, k, E)
            dl = TK.moe_route_bwd(probs, ids, wts, dw, plan, norm, coef * E / (T * T)).double()
            dh = dh + dl @ wr
            dwr = dl.t() @ h
        torch.testing.assert_close(y, y_ref.detach(), rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(aux.double(), aux_ref.detach(), rtol=1e-5, atol=0)
        torch.testing.assert_close(dh, g_ref[0], rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(dwr, g_ref[1], rtol=1e-5, atol=1e-6)


def _loop_moe(h2, wr, w1, w2, k, norm, F):
    """Straightforward per-expert loop (no permuted buffer)."""
    lg = h2 @ wr.t()
    p = torch.softmax(lg, -1)
    ids = torch.sort(lg.detach(), dim=-1, descending=True, stable=True).indices[:, :k]
    w = p.gather(1, ids)
    if norm:
        w = w / w.sum(1, keepdim=True)
    out = torch.zeros_like(h2)
    for e in range(wr.shape[0]):
        m = ids == e
        tok = m.any(1).nonzero().squeeze(1)
        if len(tok):
            g = h2[tok] @ w1[e].t()
            a = torch.nn.functional.silu(g[:, :F]) * g[:, F:]
            out = out.index_add(0, tok, (w * m)[tok].sum(1, keepdim=True) * (a @ w2[e].t()))
    return out


@pytest.mark.parametrize("norm", [False, True])
def test_moe_mlp_matches_a_per_expert_loop(norm):
    torch.manual_seed(2)
    B, S, D, E, F, k = 2, 37, 16, 8, 24, 2
    mk = lambda *s, sc=1.0: (torch.randn(*s, dtype=torch.float64) * sc).requires_grad_()
    h, x, wr, w1, w2 = mk(B, S, D), mk(B, S, D), mk(E, D), mk(E, 2 * F, D, sc=0.3), mk(E, D, F, sc=0.3)
    y, aux = ops.moe_mlp(h, wr, w1, w2, k, norm, 0.0, residual=x)
    y_ref = x + _loop_moe(h.reshape(-1, D), wr, w1, w2, k, norm, F).view(B, S, D)
    torch.testing.assert_close(y, y_ref, rtol=1e-5, atol=1e-5)
    g = torch.randn_like(y)
    got = torch.autograd.grad(y, [h, x, wr, w1, w2], g)
    ref = torch.autograd.grad(y_ref, [h, x, wr, w1, w2], g)
    for a, b in zip(got, ref):
        torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5)


def test_moe_llama_tiny_params_init_and_push_eligibility():
    from fms_fsdp_b200.ops.cuda_kernels import push_eligible_shape
    cfg = get_model_config("llama_moe_tiny")
    m = LLaMA(cfg)
    m.reset_parameters()
    sd = m.state_dict()
    E, F, D = cfg.moe_num_experts, cfg.moe_hidden_dim, cfg.emb_dim
    assert sd["layers.0.moe.gate.weight"].shape == (E, D)
    assert sd["layers.0.moe.w1"].shape == (E, 2 * F, D) and sd["layers.1.moe.w2"].shape == (E, D, F)
    assert not any("ff_sub_layer" in n for n in sd)
    assert abs(float(sd["layers.0.moe.w1"].std()) - 0.02) < 0.002
    # 3-D expert slots never take the push reduce-scatter: they use the pull path
    assert not push_eligible_shape(tuple(sd["layers.0.moe.w1"].shape))
    with torch.device("meta"):
        mm = LLaMA(cfg)
    from fms_fsdp_b200.parallel import ShardedModel
    eng = ShardedModel(mm, device="cpu")                        # meta-device path: param_init_function per unit
    w1 = eng.full_state_dict()["layers.0.moe.w1"]
    assert abs(float(w1.std()) - 0.02) < 0.002
    # forward reports the load-balancing loss
    tok = torch.randint(0, cfg.src_vocab_size, (2, 16))
    m(tok)
    aux = m.moe_aux_loss()
    assert aux is not None and float(aux) > 0


def test_moe_zoo_entries():
    for name in ("qwen3_moe_30b_a3b", "mixtral_8x7b", "llama_moe_tiny"):
        assert name in list_model_variants()
    q = get_model_config("qwen3_moe_30b_a3b")
    assert (q.emb_dim, q.nlayers, q.nheads, q.kv_heads, q.head_dim, q.qk_norm) == (2048, 48, 32, 4, 128, True)
    assert (q.moe_num_experts, q.moe_top_k, q.moe_hidden_dim, q.moe_norm_topk, q.moe_aux_loss_coef) == \
        (128, 8, 768, True, 0.001)
    assert (q.src_vocab_size, q.rope_theta, q.norm_eps) == (151936, 1e6, 1e-6)
    with torch.device("meta"):
        n = sum(p.numel() for p in LLaMA(q).parameters())
    assert abs(n / 1e9 - 30.5) < 0.2                                  # published: 30.5B total
    x = get_model_config("mixtral_8x7b")
    assert (x.emb_dim, x.nlayers, x.nheads, x.kv_heads, x.moe_num_experts, x.moe_top_k, x.moe_hidden_dim) == \
        (4096, 32, 32, 8, 8, 2, 14336)
    assert (x.src_vocab_size, x.rope_theta, x.moe_aux_loss_coef) == (32000, 1e6, 0.02)
    with torch.device("meta"):
        n = sum(p.numel() for p in LLaMA(x).parameters())
    assert abs(n / 1e9 - 46.7) < 0.2                                  # published: 46.7B total


@pytest.mark.parametrize("name", ["qwen3_moe_30b_a3b", "mixtral_8x7b", "llama_moe_tiny"])
def test_memory_plan_counts_moe_parameters_exactly(name):
    from fms_fsdp_b200.utils import memory_plan as MP
    c = get_model_config(name)
    for L in (None, 2):
        cc = get_model_config(name)
        cc.nlayers = L or c.nlayers
        with torch.device("meta"):
            n = sum(p.numel() for p in LLaMA(cc).parameters())
        plan = MP.plan_llama(name, gpus=8, nlayers=L)
        state = plan.parts_gib["master + bf16 shard + AdamW moments (14 B/param / shard)"]
        assert state * MP.GiB * 8 / 14.0 == pytest.approx(n, rel=1e-12)
    # active parameters: the router and k of E experts per block
    assert c.inactive_params() == c.nlayers * (c.moe_num_experts - c.moe_top_k) * 3 * c.emb_dim * c.moe_hidden_dim
    assert get_model_config("llama2_tiny").inactive_params() == 0
    # Qwen3-30B-A3B does not fit on 8 x 80 GB: optimizer state and gradient shards alone are about 64 GiB per GPU
    assert not MP.plan_llama("qwen3_moe_30b_a3b", gpus=8, batch_size=1, fsdp_activation_checkpointing=True).fits()


def test_llama_entry_point_trains_a_moe_variant_and_reports_the_aux_loss(tmp_path):
    import re
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, os.path.join(root, "main_training_llama.py"), "--model_variant=llama_moe_tiny",
           "--use_dummy_dataset=True", "--seq_length=32", "--vocab_size=1024", "--batch_size=2", "--num_steps=3",
           "--report_interval=1", "--checkpoint_interval=3", f"--ckpt_save_path={tmp_path}", "--sharding_strategy=fsdp",
           "--comm_backend=gloo", "--use_torch_compile=False", "--moe_aux_loss_coef=0.05"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=root, env=dict(os.environ, OMP_NUM_THREADS="1"))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    aux = [float(x) for x in re.findall(r"^moe_aux_loss: ([0-9.eE+-]+)$", r.stdout, flags=re.M)]
    losses = [float(x) for x in re.findall(r"^loss: ([0-9.eE+-]+)$", r.stdout, flags=re.M)]
    assert len(aux) == 3 and len(losses) == 3
    # coef * E * sum_e f_e P_e with sum_e f_e = k: about coef * k when balanced, at most coef * E * k
    assert all(0.05 * 2 * 0.5 < a < 0.05 * 8 * 2 for a in aux), aux
    bad = subprocess.run(cmd[:-1] + ["--precision=fp8"], capture_output=True, text=True, timeout=600, cwd=root)
    assert bad.returncode != 0 and "bf16 only" in bad.stdout + bad.stderr


def test_gradient_accumulation_scales_the_aux_gradient_like_the_loss():
    """k = 2 micro-batches on the unsharded engine against autograd of (L_a + L_b) / 2 on a copy whose coefficient is
    halved: the load-balancing gradient enters each micro-step at unit scale and the engine's 1/k applies to it."""
    import copy
    from fms_fsdp_b200.parallel import ShardedAdamW, ShardedModel
    from fms_fsdp_b200.policies import fp32_policy
    torch.manual_seed(0)
    cfg = get_model_config("llama_moe_tiny")
    cfg.moe_aux_loss_coef = 0.5                      # large enough that a wrong scale shows
    m = LLaMA(cfg)
    m.reset_parameters()
    ref = copy.deepcopy(m)
    ref.config.moe_aux_loss_coef = cfg.moe_aux_loss_coef / 2
    xa, xb = TE._batch(0, 0), TE._batch(1, 0)
    eng = ShardedModel(m, mixed_precision=fp32_policy, device="cpu", grad_accum_steps=2)
    opt = ShardedAdamW(eng, lr=1e-3)
    eng.forward_backward(xa, xa)
    eng.forward_backward(xb, xb)
    norm = eng.clip_grad_norm_(1e9).item()
    opt.step()
    ((ref(xa, labels=xa) + ref(xb, labels=xb)) / 2).backward()
    rnorm = torch.nn.utils.clip_grad_norm_(ref.parameters(), 1e9).item()
    torch.optim.AdamW(ref.parameters(), lr=1e-3, betas=(0.9, 0.95), weight_decay=0.1).step()
    assert norm == pytest.approx(rnorm, rel=1e-4)
    sd = eng.full_state_dict()
    for k_, v in ref.state_dict().items():
        assert torch.allclose(sd[k_], v, atol=2e-5, rtol=1e-4), k_


@pytest.mark.parametrize("kind", ["qwen3_moe", "qwen2_moe"])
def test_hf_import_refuses_moe_checkpoints(kind):
    from fms_fsdp_b200.models.hf_loader import config_from_hf
    hf = dict(model_type=kind, hidden_size=64, num_attention_heads=4, num_key_value_heads=2, num_hidden_layers=1,
              intermediate_size=128, vocab_size=64, rms_norm_eps=1e-6, max_position_embeddings=128)
    with pytest.raises(NotImplementedError, match="mixture-of-experts|shared experts"):
        config_from_hf(hf)


@pytest.mark.parametrize("key", ["model.layers.0.block_sparse_moe.gate.weight", "model.layers.0.mlp.gate.weight",
                                 "model.layers.0.mlp.experts.gate_up_proj"])
def test_llama_state_dict_conversion_refuses_expert_tensors(key):
    """Mixtral / Qwen3-MoE tensors into the trainable Llama (the frozen speculator base has its own Mixtral loader)."""
    from fms_fsdp_b200.models.hf_loader import convert_hf_state_dict
    with pytest.raises(NotImplementedError, match="mixture-of-experts"):
        convert_hf_state_dict({key: torch.zeros(8, 8)}, get_model_config("llama2_tiny"))


def test_moe_mlp_refuses_fp8():
    from fms_fsdp_b200.ops import functional as Fn
    old = Fn.get_gemm_precision()
    Fn.set_gemm_precision("fp8")
    try:
        with pytest.raises(NotImplementedError, match="bf16"):
            ops.moe_mlp(torch.randn(4, 8), torch.randn(8, 8), torch.randn(8, 16, 8), torch.randn(8, 8, 8), 2)
    finally:
        Fn.set_gemm_precision(old)


def test_speculator_refuses_a_moe_base():
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "speculator"))
    from speculator.train_speculator_utils import EmbedLLaMA
    with pytest.raises(NotImplementedError, match="mixture-of-experts"):
        EmbedLLaMA(get_model_config("llama_moe_tiny"))


# --------------------------------------------------------------------------------------------- sharded engine
def _moe_config(variant):
    return get_model_config("llama_moe_tiny")


def _moe_doc_config(variant):
    cfg = _moe_config(variant)
    cfg.doc_separator = 1
    return cfg


def _te_worker(rank, doc, *args):
    TE.get_model_config = _moe_doc_config if doc else _moe_config
    TE._worker(rank, *args)


def _oracle_config(doc, world):
    """The single-process oracle sums loss / world over the ranks' batches, but the load-balancing gradient enters each
    MoE backward at unit scale; the engine averages both over the ranks, so the oracle's coefficient is divided by world."""
    def get(variant):
        cfg = (_moe_doc_config if doc else _moe_config)(variant)
        cfg.moe_aux_loss_coef /= world
        return cfg
    return get


@pytest.mark.parametrize("world,strategy,shard,ac,doc", [(2, "fsdp", 0, None, False), (2, "fsdp", 0, "1/2", True),
                                                       (2, "ddp", 0, None, False), (4, "fsdp", 0, None, False),
                                                       (4, "hsdp", 2, None, False)])
def test_moe_engine_matches_oracle(world, strategy, shard, ac, doc, monkeypatch):
    """E = 8 experts; at world 4 each rank's shard of a block cuts through the middle of the expert tensors."""
    outdir = tempfile.mkdtemp()
    mp.spawn(_te_worker, args=(doc, world, free_port(), strategy, shard, ac, outdir, None), nprocs=world, join=True)
    out = torch.load(os.path.join(outdir, "out.pt"), weights_only=False)
    assert any(k.endswith("moe.w1") for k in out["sd"])
    monkeypatch.setattr(TE, "get_model_config", _oracle_config(doc, world))
    TE._check(out, world)          # loss, grad norm and every parameter (router and experts included) after 3 steps
