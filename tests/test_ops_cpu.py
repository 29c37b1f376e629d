"""Hand-derived backward formulas of every op (ATen back-end) against autograd of the naive formula.
The same primitives are what the sm_90a kernels are checked against on the GPU box."""
import torch
import torch.nn.functional as F

from fms_fsdp_b200 import ops
from fms_fsdp_b200.ops import torch_kernels as TK

torch.manual_seed(0)


def _close(a, b, tol=1e-4):
    assert torch.allclose(a, b, atol=tol, rtol=tol), (a - b).abs().max()


def test_linear_and_residual():
    x = torch.randn(3, 5, 16, requires_grad=True); w = torch.nn.Parameter(torch.randn(24, 16)); r = torch.randn(3, 5, 24, requires_grad=True)
    y = ops.linear(x, w, r); y.sum().backward()
    x2 = x.detach().requires_grad_(); w2 = w.detach().requires_grad_(); r2 = r.detach().requires_grad_()
    y2 = F.linear(x2, w2) + r2; y2.sum().backward()
    _close(y, y2); _close(x.grad, x2.grad); _close(w.grad, w2.grad); _close(r.grad, r2.grad)


def test_rmsnorm():
    x = torch.randn(7, 32, requires_grad=True); w = torch.nn.Parameter(torch.rand(32) + 0.5)
    y = ops.rmsnorm(x, w, 1e-5); (y * torch.arange(32.)).sum().backward()
    x2 = x.detach().requires_grad_(); w2 = w.detach().requires_grad_()
    y2 = x2 * torch.rsqrt(x2.pow(2).mean(-1, keepdim=True) + 1e-5) * w2; (y2 * torch.arange(32.)).sum().backward()
    _close(y, y2); _close(x.grad, x2.grad); _close(w.grad, w2.grad)


def test_rmsnorm_fork_sums_residual_gradient():
    x = torch.randn(7, 32, requires_grad=True); w = torch.nn.Parameter(torch.rand(32) + 0.5)
    h, r = ops.rmsnorm_fork(x, w, 1e-5)
    (r + torch.tanh(h) * 3).pow(2).sum().backward()
    x2 = x.detach().requires_grad_(); w2 = w.detach().requires_grad_()
    h2 = x2 * torch.rsqrt(x2.pow(2).mean(-1, keepdim=True) + 1e-5) * w2
    (x2 + torch.tanh(h2) * 3).pow(2).sum().backward()
    _close(x.grad, x2.grad); _close(w.grad, w2.grad)
    # only the residual branch used
    x3 = x.detach().requires_grad_()
    _, r3 = ops.rmsnorm_fork(x3, w, 1e-5)
    r3.sum().backward()
    _close(x3.grad, torch.ones_like(x3))


def test_rmsnorm_gated():
    x = torch.randn(6, 32, requires_grad=True); z = torch.randn(6, 32, requires_grad=True); w = torch.nn.Parameter(torch.rand(32) + 0.5)
    y = ops.rmsnorm_gated(x, z, w, 1e-5, 16); (y * torch.arange(32.)).sum().backward()
    x2, z2, w2 = (t.detach().requires_grad_() for t in (x, z, w))
    u = (x2 * F.silu(z2)).view(6, 2, 16)
    y2 = (u * torch.rsqrt(u.pow(2).mean(-1, keepdim=True) + 1e-5)).view(6, 32) * w2
    (y2 * torch.arange(32.)).sum().backward()
    _close(y, y2); _close(x.grad, x2.grad); _close(z.grad, z2.grad); _close(w.grad, w2.grad)


def _naive_rope(q, S, hd, theta=10000.0):
    # q: [B,S,H,hd], interleaved pairs
    inv = 1.0 / (theta ** (torch.arange(0, hd, 2).float() / hd))
    ang = torch.outer(torch.arange(S).float(), inv)
    cos, sin = ang.cos()[None, :, None], ang.sin()[None, :, None]
    x0, x1 = q[..., 0::2], q[..., 1::2]
    return torch.stack([x0 * cos - x1 * sin, x0 * sin + x1 * cos], dim=-1).flatten(-2)


def test_rope_attention_block():
    B, S, H, KVH, hd = 2, 16, 4, 2, 8
    qkv = torch.randn(B, S, (H + 2 * KVH) * hd, requires_grad=True)
    tab = TK.rope_table(S, hd)
    out = ops.attention(ops.rope_(qkv * 1.0, tab, S, H, KVH, hd), H, KVH, hd)
    out.square().sum().backward()
    q2 = qkv.detach().requires_grad_()
    t = q2.view(B, S, H + 2 * KVH, hd)
    q = _naive_rope(t[:, :, :H], S, hd); k = _naive_rope(t[:, :, H:H + KVH], S, hd); v = t[:, :, H + KVH:]
    ref = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2).repeat_interleave(2, 1),
                                         v.transpose(1, 2).repeat_interleave(2, 1), is_causal=True)
    ref = ref.transpose(1, 2).reshape(B, S, H * hd)
    ref.square().sum().backward()
    _close(out, ref, 1e-4); _close(qkv.grad, q2.grad, 1e-3)


def test_swiglu_embedding_ce():
    gu = torch.randn(5, 24, requires_grad=True)
    y = ops.swiglu(gu); y.sum().backward()
    g2 = gu.detach().requires_grad_(); y2 = F.silu(g2[:, :12]) * g2[:, 12:]; y2.sum().backward()
    _close(y, y2); _close(gu.grad, g2.grad)

    w = torch.nn.Parameter(torch.randn(11, 6)); tok = torch.randint(0, 11, (3, 4))
    e = ops.embedding(tok, w); e.sum().backward()
    w2 = w.detach().requires_grad_(); F.embedding(tok, w2).sum().backward()
    _close(w.grad, w2.grad)

    h = torch.randn(10, 6, requires_grad=True); hw = torch.nn.Parameter(torch.randn(11, 6)); lab = torch.randint(0, 11, (10,)); lab[3] = -100
    loss = ops.linear_cross_entropy(h, hw, lab); loss.backward()
    h2 = h.detach().requires_grad_(); hw2 = hw.detach().requires_grad_()
    l2 = F.cross_entropy(h2 @ hw2.t(), lab, ignore_index=-100); l2.backward()
    _close(loss, l2); _close(h.grad, h2.grad); _close(hw.grad, hw2.grad)
    lg = torch.randn(10, 11, requires_grad=True)
    l3 = ops.cross_entropy(lg, lab); l3.backward()
    lg2 = lg.detach().requires_grad_(); F.cross_entropy(lg2, lab, ignore_index=-100).backward()
    _close(lg.grad, lg2.grad)


def test_adamw_matches_torch():
    p = torch.randn(64); g = torch.randn(64)
    ref = torch.nn.Parameter(p.clone()); opt = torch.optim.AdamW([ref], lr=1e-2, betas=(0.9, 0.95), weight_decay=0.1)
    m, v, mine = torch.zeros(64), torch.zeros(64), p.clone()
    for step in range(1, 4):
        ref.grad = g.clone(); opt.step()
        TK.adamw_step(mine, g, m, v, None, 1e-2, 0.9, 0.95, 1e-8, 0.1, step)
    _close(mine, ref.data, 1e-6)


def test_conv1d_bwd_formula():
    S, C, K = 12, 8, 4
    x = torch.randn(2 * S, C, requires_grad=True); w = torch.nn.Parameter(torch.randn(C, K)); b = torch.nn.Parameter(torch.randn(C))
    y = ops.causal_conv1d(x, w, b, S); (y * y).sum().backward()
    x2, w2, b2 = (t.detach().requires_grad_() for t in (x, w, b))
    xt = x2.view(2, S, C).transpose(1, 2)
    y2 = F.silu(F.conv1d(F.pad(xt, (K - 1, 0)), w2.unsqueeze(1), b2, groups=C)).transpose(1, 2).reshape(2 * S, C)
    (y2 * y2).sum().backward()
    _close(y, y2); _close(x.grad, x2.grad, 1e-3); _close(w.grad, w2.grad, 1e-3); _close(b.grad, b2.grad, 1e-3)


def test_ssd_scan_matches_chunked_reference():
    """Sequential oracle == the chunked (state-space dual) formulation the CUDA kernel implements."""
    S, H, P, G, N = 32, 4, 8, 1, 16
    x = torch.randn(S, H, P); dt = torch.rand(S, H); A = -torch.rand(H) - 0.1
    Bm = torch.randn(S, G, N); Cm = torch.randn(S, G, N); D = torch.randn(H)
    y = TK.ssd_scan_fwd(x, dt, A, Bm, Cm, D, None, S, 8, dt_softplus=False)
    # direct quadratic form: y_t = sum_{s<=t} C_t.B_s exp(sum_{s<r<=t} dt_r A) dt_s x_s + D x_t
    a = dt * A
    cs = torch.cumsum(a, 0)
    L = torch.exp(cs[:, None, :] - cs[None, :, :]) * (torch.arange(S)[:, None] >= torch.arange(S)[None, :])[..., None]
    CB = torch.einsum("tgn,sgn->ts", Cm, Bm)
    y2 = torch.einsum("ts,tsh,sh,shp->thp", CB, L, dt, x) + x * D[None, :, None]
    _close(y, y2, 1e-3)


def test_qkv_attention_fused_node_matches_separate_ops():
    """qkv_attention (projection + RoPE + attention as one node) == linear -> rope_ -> attention, values and grads."""
    torch.manual_seed(0)
    B, S, D, H, KVH, hd = 2, 16, 24, 4, 2, 8
    tab = TK.rope_table(S, hd)
    h = torch.randn(B, S, D, requires_grad=True)
    w = torch.nn.Parameter(torch.randn((H + 2 * KVH) * hd, D) * 0.2)
    y = ops.qkv_attention(h, w, tab, H, KVH, hd)
    (y * torch.arange(y.shape[-1]).float()).sum().backward()
    h2 = h.detach().requires_grad_(); w2 = torch.nn.Parameter(w.detach().clone())
    qkv = ops.rope_(ops.linear(h2, w2), tab, S, H, KVH, hd)
    y2 = ops.attention(qkv, H, KVH, hd)
    (y2 * torch.arange(y2.shape[-1]).float()).sum().backward()
    _close(y, y2); _close(h.grad, h2.grad); _close(w.grad, w2.grad)


def test_linear_ce_applies_the_upstream_gradient():
    """(loss / k).backward() through the fused linear-cross-entropy scales dh and dW (grad accumulation, weighted
    losses); only the engine's own schedule (upstream == 1, declared via set_unit_upstream) skips the multiply."""
    import torch
    from fms_fsdp_b200 import ops
    torch.manual_seed(0)
    h = torch.randn(6, 16, requires_grad=True)
    w = torch.nn.Parameter(torch.randn(32, 16) * 0.1)
    y = torch.randint(0, 32, (6,))
    (ops.linear_cross_entropy(h, w, y) * 0.25).backward()
    h2 = h.detach().clone().requires_grad_(); w2 = torch.nn.Parameter(w.detach().clone())
    (torch.nn.functional.cross_entropy(h2 @ w2.t(), y) * 0.25).backward()
    assert torch.allclose(h.grad, h2.grad, atol=1e-6) and torch.allclose(w.grad, w2.grad, atol=1e-6)


def test_gated_mlp_matches_autograd():
    import torch
    from fms_fsdp_b200 import ops
    torch.manual_seed(0)
    for gate_first in (True, False):
        x = torch.randn(3, 5, 16, requires_grad=True)
        w1 = torch.nn.Parameter(torch.randn(24, 16) * 0.2); w2 = torch.nn.Parameter(torch.randn(16, 12) * 0.2)
        y = ops.gated_mlp(x, w1, w2, residual=x, gate_first=gate_first)
        y.pow(2).sum().backward()
        x2 = x.detach().clone().requires_grad_(); a1 = torch.nn.Parameter(w1.detach().clone()); a2 = torch.nn.Parameter(w2.detach().clone())
        gu = x2 @ a1.t()
        g, u = (gu[..., :12], gu[..., 12:]) if gate_first else (gu[..., 12:], gu[..., :12])
        y2 = (torch.nn.functional.silu(g) * u) @ a2.t() + x2
        y2.pow(2).sum().backward()
        assert torch.allclose(y, y2, atol=1e-5)
        for a, b in ((x.grad, x2.grad), (w1.grad, a1.grad), (w2.grad, a2.grad)):
            assert torch.allclose(a, b, atol=1e-4)


def test_fp8_precision_switch_cpu_oracle():
    """precision=fp8: linear / qkv_attention / gated_mlp run their forward GEMMs on row-wise e4m3 operands (torch oracle on
    CPU), gradients come from the bf16 backward; default precision is untouched afterwards."""
    import torch
    from fms_fsdp_b200 import ops
    from fms_fsdp_b200.ops import functional as Fn
    from fms_fsdp_b200.ops import torch_kernels as TK
    torch.manual_seed(0)
    x = (torch.randn(4, 8, 32) * 0.5).bfloat16().requires_grad_()
    w1 = torch.nn.Parameter((torch.randn(64, 32) * 0.2).bfloat16()); w2 = torch.nn.Parameter((torch.randn(32, 32) * 0.2).bfloat16())
    ref = ops.gated_mlp(x, w1, w2, residual=x)
    Fn.set_gemm_precision("fp8")
    try:
        assert Fn.get_gemm_precision() == "fp8"
        y = ops.gated_mlp(x, w1, w2, residual=x)
        y.float().sum().backward()
    finally:
        Fn.set_gemm_precision("bf16")
    err = ((y.float() - ref.float()).abs().max() / ref.float().abs().max()).item()
    assert 0 < err < 0.1, err                       # really quantised, and close
    assert x.grad is not None and w1.grad is not None and w2.grad is not None
    q, s = TK.quant_rowwise_e4m3(x.detach().reshape(-1, 32))
    assert q.dtype == torch.uint8 and torch.all(s > 0)
    assert (q.view(torch.float8_e4m3fn).float().abs().amax(1) - 448).abs().max() < 1e-3   # every row uses the full range
