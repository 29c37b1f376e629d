"""Mixture of experts on the GPU: every kernel of ``csrc/moe.cu`` and every grouped GEMM mode against the ATen oracle,
run-to-run bit reproducibility, no host synchronisation, and the SASS of the new and the existing kernels."""
import json
import os
import re
import shutil
import subprocess

import pytest
import torch

from fms_fsdp_b200 import ops
from fms_fsdp_b200.ops import torch_kernels as tk

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ck():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from fms_fsdp_b200.ops import cuda_kernels
    return cuda_kernels


def _logits(kind, T, E, k, gen):
    lg = torch.randn(T, E, generator=gen)
    if kind == "same":                    # every token on experts E-k .. E-1
        lg[:, E - k:] += 50.0
    elif kind == "empty":                 # only the first 2k experts are ever chosen
        lg[:, 2 * k:] -= 50.0
    elif kind == "ties":                  # equal logits everywhere: the lowest k experts win
        lg = torch.zeros(T, E)
    return lg


CASES = [("uniform", 8192, 128, 8), ("uniform", 200, 8, 2), ("same", 1000, 128, 8), ("empty", 333, 64, 4),
         ("ties", 136, 16, 2), ("uniform", 1, 8, 2)]


@pytest.mark.parametrize("kind,T,E,k", CASES)
@pytest.mark.parametrize("norm", [False, True])
def test_route_and_plan_match_oracle(ck, kind, T, E, k, norm):
    gen = torch.Generator().manual_seed(T + E)
    lg = _logits(kind, T, E, k, gen)
    ids, wts, probs = ck.moe_route(lg.cuda(), k, norm)
    rid, rw, rp = tk.moe_route(lg, k, norm)
    assert torch.equal(ids.cpu(), rid)
    torch.testing.assert_close(probs.cpu(), rp, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(wts.cpu(), rw, rtol=1e-5, atol=1e-6)
    plan, aux = ck.moe_plan(ids, probs)
    rplan, raux = tk.moe_plan(rid, rp)
    g, r = tk.moe_plan_views(plan.cpu(), T, k, E), tk.moe_plan_views(rplan, T, k, E)
    for a, b in zip(g[:4], r[:4]):            # tile, start, len, row: exact
        assert torch.equal(a, b)
    routed = r[4] >= 0
    assert torch.equal(g[4][routed], r[4][routed])
    torch.testing.assert_close(aux.cpu(), raux, rtol=1e-4, atol=1e-6)


def test_route_with_nan_and_inf_logits_keeps_ids_in_range(ck):
    """A diverging run (NaN or -inf router logits) must route to valid experts so the plan stays in bounds; the NaN
    reaches the weights and the block's output, where the training loop's non-finite check sees it."""
    T, E, k = 300, 128, 8
    lg = torch.randn(T, E)
    lg[0] = float("nan")
    lg[1] = -float("inf")
    lg[2, :E - 1] = float("nan")
    lg[3, ::3] = float("nan")
    ids, wts, probs = ck.moe_route(lg.cuda(), k, True)
    rid, rw, _ = tk.moe_route(lg, k, True)
    assert torch.equal(ids.cpu(), rid)
    assert bool(((rid >= 0) & (rid < E)).all())
    assert bool(torch.isnan(wts[0].cpu()).all()) and bool(torch.isfinite(wts[4:].cpu()).all())
    plan, _ = ck.moe_plan(ids, probs)
    assert torch.equal(tk.moe_plan_views(plan.cpu(), T, k, E)[2], tk.moe_plan_views(tk.moe_plan(rid, probs.cpu())[0],
                                                                                     T, k, E)[2])
    h, res, wr, w1, w2, dy, kk = _moe_case(T=512)
    h = h.detach().clone()
    h[5, 0] = float("nan")
    y, _ = ops.moe_mlp(h, wr, w1, w2, kk, True, 0.01, residual=res)
    torch.cuda.synchronize()
    assert bool(torch.isnan(y[5]).all()) and bool(torch.isfinite(torch.cat([y[:5], y[6:]])).all())


def _routing(kind, T, E, k, norm=True):
    gen = torch.Generator().manual_seed(7 * T + E)
    lg = _logits(kind, T, E, k, gen)
    ids, wts, probs = tk.moe_route(lg, k, norm)
    plan, _ = tk.moe_plan(ids, probs)
    return ids, wts, probs, plan


@pytest.mark.parametrize("kind,T,E,k", CASES)
def test_permute_combine_and_route_bwd_match_oracle(ck, kind, T, E, k):
    D = 256
    ids, wts, probs, plan = _routing(kind, T, E, k)
    Mpad = tk.moe_rows(T, k, E)[0]
    valid = tk.moe_plan_views(plan, T, k, E)[0].repeat_interleave(128) >= 0     # rows of some segment
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(T, D, generator=gen).bfloat16()
    res = torch.randn(T, D, generator=gen).bfloat16()
    yp = torch.randn(Mpad, D, generator=gen).bfloat16()
    dy = torch.randn(T, D, generator=gen).bfloat16()
    c = lambda t: t.cuda()
    xp = ck.moe_permute(c(x), c(plan), k, E).cpu()
    assert torch.equal(xp[valid], tk.moe_permute(x, plan, k, E)[valid])      # padding rows included: zero
    assert torch.equal(ck.moe_permute_bwd(c(yp), c(plan), T, k, E).cpu(), tk.moe_permute_bwd(yp, plan, T, k, E))
    y = ck.moe_combine(c(yp), c(plan), c(wts), c(res), E).cpu()
    # the kernel fuses w * y + acc (one rounding), the oracle rounds twice: one bf16 ulp apart at most
    torch.testing.assert_close(y, tk.moe_combine(yp, plan, wts, res, E), rtol=1e-2, atol=1e-2)
    dyp, dw = ck.moe_combine_bwd(c(dy), c(yp), c(plan), c(wts), E)
    rdyp, rdw = tk.moe_combine_bwd(dy, yp, plan, wts, E)
    assert torch.equal(dyp.cpu()[valid], rdyp[valid])
    torch.testing.assert_close(dw.cpu(), rdw, rtol=1e-4, atol=1e-3)
    dwr = torch.randn(T, k, generator=gen)
    dl = ck.moe_route_bwd(c(probs), c(ids), c(wts), c(dwr), c(plan), True, 0.01 * E / (T * T)).cpu()
    rdl = tk.moe_route_bwd(probs, ids, wts, dwr, plan, True, 0.01 * E / (T * T))
    torch.testing.assert_close(dl.float(), rdl, rtol=2e-2, atol=1e-5)


@pytest.mark.parametrize("kind,T,E,k", [c for c in CASES if c[1] > 1] + [("uniform", 4096, 128, 8)])
def test_grouped_gemms_match_fp32_oracle(ck, kind, T, E, k):
    D, F = 256, 192
    ids, wts, probs, plan = _routing(kind, T, E, k)
    Mpad = tk.moe_rows(T, k, E)[0]
    valid = tk.moe_plan_views(plan, T, k, E)[0].repeat_interleave(128) >= 0
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(T, D, generator=gen).bfloat16()
    w1 = (torch.randn(E, 2 * F, D, generator=gen) * 0.1).bfloat16()
    w2 = (torch.randn(E, D, F, generator=gen) * 0.1).bfloat16()
    xp = tk.moe_permute(x, plan, k, E)
    dyp = tk.moe_combine_bwd(torch.randn(T, D, generator=gen).bfloat16(), torch.zeros(Mpad, D).bfloat16(), plan, wts,
                             E)[0]
    gp = c = lambda t: t.cuda()
    f = lambda t: t.float()
    close = lambda a, b: torch.testing.assert_close(a.cpu().float()[valid], b.float()[valid], rtol=2e-2, atol=2e-2)
    h, s = ck.moe_up_fwd(gp(xp), c(w1), c(plan), T, k)
    rh, rs = tk.moe_up_fwd(f(xp), f(w1), plan, T, k)
    close(h, rh)
    close(s, tk.swiglu_fwd(h.cpu().float()))
    yp = ck.moe_down_fwd(s, c(w2), c(plan), T, k)
    close(yp, tk.moe_down_fwd(f(s.cpu()), f(w2), plan, T, k))
    dh = ck.moe_down_bwd(c(dyp), c(w2), h, c(plan), T, k)
    close(dh, tk.moe_down_bwd(f(dyp), f(w2), f(h.cpu()), plan, T, k))
    dxp = ck.moe_up_dgrad(dh, c(w1), c(plan), T, k)
    close(dxp, tk.moe_up_dgrad(f(dh.cpu()), f(w1), plan, T, k))
    for dtype in (torch.float32, torch.bfloat16):
        ref = tk.moe_wgrad(f(dyp), f(s.cpu()), plan, T, k, torch.empty(E, D, F))
        out = torch.full((E, D, F), 7.0, dtype=dtype, device="cuda")
        ck.moe_wgrad(c(dyp), s, c(plan), T, k, out)                  # store: empty experts get zeros
        torch.testing.assert_close(out.cpu().float(), ref, rtol=2e-2, atol=2e-2)
        ck.moe_wgrad(c(dyp), s, c(plan), T, k, out, accumulate=True)
        torch.testing.assert_close(out.cpu().float(), 2 * ref, rtol=2e-2, atol=4e-2)


def _moe_case(T=8192 // 4, D=512, E=16, F=256, k=4, seed=0):
    gen = torch.Generator().manual_seed(seed)
    h = torch.randn(T, D, generator=gen).bfloat16().cuda().requires_grad_()
    res = torch.randn(T, D, generator=gen).bfloat16().cuda().requires_grad_()
    wr = (torch.randn(E, D, generator=gen) * 0.02).bfloat16().cuda().requires_grad_()
    w1 = (torch.randn(E, 2 * F, D, generator=gen) * 0.02).bfloat16().cuda().requires_grad_()
    w2 = (torch.randn(E, D, F, generator=gen) * 0.02).bfloat16().cuda().requires_grad_()
    dy = torch.randn(T, D, generator=gen).bfloat16().cuda()
    return h, res, wr, w1, w2, dy, k


def test_moe_mlp_bitwise_reproducible_and_matches_oracle(ck):
    h, res, wr, w1, w2, dy, k = _moe_case()
    runs = []
    for _ in range(2):
        y, aux = ops.moe_mlp(h, wr, w1, w2, k, True, 0.01, residual=res)
        grads = torch.autograd.grad(y, [h, wr, w1, w2], dy)
        runs.append([y, aux] + list(grads))
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    cpu = [t.detach().cpu().float().requires_grad_() for t in (h, res, wr, w1, w2)]
    y32, aux32 = ops.moe_mlp(cpu[0], cpu[2], cpu[3], cpu[4], k, True, 0.01, residual=cpu[1])
    g32 = torch.autograd.grad(y32, [cpu[0], cpu[2], cpu[3], cpu[4]], dy.cpu().float())
    torch.testing.assert_close(runs[0][0].cpu().float(), y32, rtol=2e-2, atol=3e-2)
    torch.testing.assert_close(runs[0][1].cpu(), aux32, rtol=1e-4, atol=1e-6)
    for g, r in zip(runs[0][2:], g32):
        err = (g.cpu().float() - r).norm() / r.norm()
        assert err < 2e-2, err


def test_moe_mlp_runs_without_host_sync(ck):
    h, res, wr, w1, w2, dy, k = _moe_case(T=1024)
    ops.moe_mlp(h, wr, w1, w2, k, True, 0.01, residual=res)    # warm up allocator and launch configuration
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        y, _ = ops.moe_mlp(h, wr, w1, w2, k, True, 0.01, residual=res)
        torch.autograd.grad(y, [h, wr, w1, w2], dy)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def _engine_step(cfg, x, steps=1):
    from fms_fsdp_b200.models.llama import LLaMA
    from fms_fsdp_b200.parallel import ShardedAdamW, ShardedModel
    from fms_fsdp_b200.policies import bfSixteen
    torch.manual_seed(0)
    with torch.device("meta"):
        m = LLaMA(cfg)
    eng = ShardedModel(m, sharding_strategy="fsdp", mixed_precision=bfSixteen, device=torch.device("cuda", 0))
    opt = ShardedAdamW(eng, lr=1e-4)
    out = []
    for _ in range(steps):
        loss = eng.forward_backward(x, x)
        out.append((float(loss), float(eng.clip_grad_norm_(1e9))))
        opt.step()
    return out


def test_engine_step_at_a_truncated_qwen3_moe_shape_matches_the_aten_path(ck):
    """Two Qwen3-30B-A3B blocks (D 2048, 128 experts, top 8, F 768, QK-norm; vocab cut to 32000) through the engine:
    the sm_90a kernels against the ATen oracle on the same device."""
    from fms_fsdp_b200.ops import functional as Fn
    from fms_fsdp_b200.utils.config_utils import get_model_config
    cfg = get_model_config("qwen3_moe_30b_a3b")
    cfg.nlayers, cfg.src_vocab_size = 2, 32000
    x = torch.randint(0, 32000, (1, 1024), generator=torch.Generator().manual_seed(0)).cuda()
    ck.reset_fallback_count()
    fused = _engine_step(cfg, x, steps=2)
    assert ck.fallback_count() == 0
    old = Fn.get_kernel_path()
    Fn.set_kernel_path("torch")
    try:
        ref = _engine_step(cfg, x, steps=2)
    finally:
        Fn.set_kernel_path(old)
    for (l, g), (rl, rg) in zip(fused, ref):
        assert l == pytest.approx(rl, rel=5e-3), (fused, ref)
        assert g == pytest.approx(rg, rel=3e-2), (fused, ref)


def test_allocator_peak_of_a_4_layer_qwen3_moe_matches_the_memory_plan(ck):
    from fms_fsdp_b200.utils.config_utils import get_model_config
    from fms_fsdp_b200.utils.memory_plan import plan_llama
    cfg = get_model_config("qwen3_moe_30b_a3b")
    cfg.nlayers = 4
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    x = torch.randint(0, cfg.src_vocab_size, (2, 4096), generator=torch.Generator().manual_seed(0)).cuda()
    _engine_step(cfg, x, steps=2)
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    plan = plan_llama("qwen3_moe_30b_a3b", gpus=1, batch_size=2, seq_length=4096, nlayers=4).total_gib
    print(f"allocator peak {peak:.3f} GiB, plan {plan:.3f} GiB")
    assert abs(peak - plan) / plan < 0.005, (peak, plan)


def _sass():
    so = os.path.join(ROOT, "fms_fsdp_b200", "_C.so")
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(so) or not os.path.exists(exe):
        pytest.skip("needs the built extension and cuobjdump")
    out = subprocess.run([exe, "-sass", so], capture_output=True, text=True, timeout=600).stdout
    import hashlib
    per, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            per[name] = []
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?;)", line)
        if name and m:
            per[name].append(m.group(1))
    return {k: hashlib.sha256("\n".join(v).encode()).hexdigest() for k, v in per.items()}, per


def test_sass_grouped_kernels_and_existing_kernels_unchanged():
    """``tests/golden/sass_before_moe.json``: per-kernel digests of every kernel of the extension before the MoE kernels
    were added (``scripts/sass_digest.py``, CUDA 12.9).  Grouped GEMM instantiations carry GRP_M (16) or GRP_K (32) in
    their EPI argument."""
    digests, per = _sass()
    grouped = [k for k in per if re.search(r"gemm_bf16_wgmmaILb[01]ELb[01]ELi(1[6-9]|2\d|3\d|4\d)E", k)]
    assert len(grouped) == 8, grouped
    for k in grouped:
        assert any("HGMMA" in i for i in per[k]) and any("UTMALDG" in i for i in per[k]), k
    new = grouped + [k for k in per if "moe_" in k]
    assert len(new) == 8 + 9, new
    for k in new:
        assert not any(re.match(r"(LDL|STL)\b", i) for i in per[k]), k
    with open(os.path.join(ROOT, "tests", "golden", "sass_before_moe.json")) as f:
        before = json.load(f)
    changed = [k for k, v in before.items() if digests.get(k) != v]
    assert not changed, changed
