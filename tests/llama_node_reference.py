"""Float64 reference, per-row metric and CPU rounding emulation of the dense Llama autograd nodes of
``ops/functional.py`` (``linear``, ``rmsnorm`` / ``rmsnorm_fork``, ``gated_mlp`` and every form of ``qkv_attention``)
and of the QK-norm kernels (``qk_norm_rope_kernel`` / ``qk_norm_bwd_kernel``, ``csrc/elementwise.cu``), shared by
``tests/test_llama_nodes_cpu.py`` and ``tests/test_llama_nodes_gpu.py``.  Not a test module (no ``test_`` prefix).

Every function takes the node's bf16 inputs and returns float64 outputs, forward and backward.  With ``em=True`` it
rounds to bf16 exactly where the node stores bf16 and uses the GEMM (``gemm_reference``) and attention
(``attention_reference.emulate``) emulators inside each stage:

    qkv after the projection epilogue (bias and RoPE fused), and again after ``qk_norm_rope``
    o; dqkv after the attention backward (inverse RoPE applied), and again after ``qk_norm_bwd``
    gu and act of the gate/up GEMM; dgu of the down-projection dgrad; y; dh / dx of every node

rstd, dw_q / dw_k, db, the norm dw and the GEMM wgrads stay fp32 (sums in fp32, modelled as one running sum that
truncates at every add, the pessimistic order).  The fp8 branch quantises both operands of each forward GEMM row-wise to
e4m3 (``gemm_reference.quant_rowwise_e4m3``) and runs the bf16 backward; its RoPE, QK-norm and SwiGLU are separate
kernels, and its inverse RoPE is a separate pass over the attention's bf16 gradient.

The metric is ``moe_reference.ratio`` per row: rows are tokens for [M, .] outputs (o, y, dh, dx) and output rows for
the weight gradients [N, K]; a zero reference row must be exactly zero.  The QK-norm kernels are judged per (row,
head).  The [hd] and [N] vector gradients (dw_q, dw_k, db, the norm dw) are judged element by element against the sum
of the absolute values of the terms summed into the element (``vratio``).
"""
import math

import torch

import attention_reference as AR
import gemm_reference as GR
from moe_reference import BF16, F64, bf, f32, ratio, rz32

EPS_QK = 1e-6
RSQRT_ERR = 2.0 ** -22      # charged relative error of rsqrtf (its documented maximum is 2 ulp)

# Tolerances on the per-row ratio (``vratio`` for the vector gradients).  Each is 3x the worst ratio of the rounding
# emulation (``em=True``) over the regimes and shapes of tests/test_llama_nodes_cpu.py, rounded up.  Worst emulated ratios:
#   QK-norm kernels, given bf16 inputs (regimes init, tiny, outlier, gains; hd 64 and 128; M 111):
#     qk_y    3.8e-3   one bf16 rounding of the normed, rotated head (2^-8 of the head's max)
#     qk_rstd 4.1e-7   fp32 sum of squares and rsqrtf (outlier)
#     qk_dx   3.9e-3   one bf16 rounding of dx, against the head's scale r (|w g| + |xhat| mean|xhat w g|)
#     qk_dw   9.5e-6   the truncating fp32 running sum over 444 q heads, against the sum of |g xhat| (outlier, hd 128)
#   whole nodes, bf16 inputs (regimes init and outlier; causal, mid_tile and one_token documents; M 128 to 256, D 256):
#   the stored bf16 tensors' roundings propagate, so the fp32 outputs are bf16-sized too:
#     o 1.3e-2 (QK-norm, outlier)  dh 2.5e-2  dw 6.6e-2 (bias)  db 4.4e-3  dwqk 1.7e-3     attention, bf16 projection
#     o 1.4e-2  dh 2.9e-2  dw 5.2e-2 (plain, outlier)                                      attention, fp8 projection
#     y 6.8e-3  dx 5.7e-3  dwl 4.7e-2 (dwg1 / dw2, outlier)                                 linear, gated MLP
#     y 4.8e-2  dx 6.4e-3  dwl 2.3e-2 (outlier)                                             gated MLP, fp8
#     norm_y 3.7e-3  norm_dx 3.7e-3  norm_dw 1.8e-6 (outlier)                               rmsnorm, rmsnorm_fork
# The fp8 y carries the e4m3 accumulator model of gemm_reference (FP8_ACC_BITS) on an outlier-dominated row.
TOL = {
    "qk_y": 1.2e-2, "qk_rstd": 1.3e-6, "qk_dx": 1.2e-2, "qk_dw": 2.9e-5,
    "o": 3.9e-2, "dh": 7.6e-2, "dw": 0.2, "db": 1.4e-2, "dwqk": 5.3e-3,
    "o_fp8": 4.2e-2, "dh_fp8": 8.6e-2, "dw_fp8": 0.16,
    "y": 2.1e-2, "dx": 1.8e-2, "dwl": 0.15,
    "y_fp8": 0.15, "dx_fp8": 2e-2, "dwl_fp8": 7e-2,
    "norm_y": 1.2e-2, "norm_dx": 1.2e-2, "norm_dw": 5.4e-6,
}

# ``mut``: broken QK-norm kernels (these) and broken node code (norm_bwd_rotated_grad, inv_rope_after_norm_bwd,
# bias_grad_rotated, dres_dropped, residual_grad_dropped), each failing the check of tests/test_llama_nodes_cpu.py that
# targets it
QK_MUTATIONS = ("rstd_no_eps", "eps_after_sqrt", "norm_after_rope", "wq_wk_swapped", "bwd_mean_without_w",
                "dwq_sums_k_heads")


# --------------------------------------------------------------------------------------------------- metric
def vratio(out, ref, absum):
    """Worst |out - ref| / absum over the elements of a vector gradient; where absum is 0 the output must be 0."""
    return GR.ratio(out.reshape(-1), ref.reshape(-1).to(F64), absum.reshape(-1).to(F64))


def head_ratio(out, ref, hd, scale=None):
    """``ratio`` per (row, head) of [M, heads * hd] tensors."""
    return ratio(out.reshape(-1, hd), ref.reshape(-1, hd), None if scale is None else scale.reshape(-1, hd))


# ------------------------------------------------------------------------------------------------ arithmetic
def mm(a, b, em=False):
    """a [M, K] @ b [K, N] in float64, or (``em``) through the fp32 tensor-core accumulator."""
    a, b = a.to(F64), b.to(F64)
    return GR.acc_em(a, b) if em else a @ b


def st(x, em):
    """A bf16 storage point."""
    return bf(x) if em else x


def fsum_rows(t, em):
    """Sum over dim 0 of [R, n]: float64, or one fp32 running sum that truncates at every add."""
    if not em:
        return t.sum(0)
    acc = torch.zeros(t.shape[1:], dtype=F64, device=t.device)
    for r in range(t.shape[0]):
        acc = rz32(acc + t[r])
    return acc


def lane_sum(t, em):
    """Sum over the last dim of [..., n] (n = 8 G): each lane adds its 8 elements in order, then a butterfly over the G
    lanes, all in fp32 (the QK-norm kernels' per-head reduction); float64 without ``em``."""
    if not em:
        return t.sum(-1)
    v = t.reshape(*t.shape[:-1], -1, 8)
    s = v[..., 0]
    for i in range(1, 8):
        s = f32(s + v[..., i])
    G = s.shape[-1]
    o = G // 2
    while o:
        s = f32(s + s[..., torch.arange(G, device=s.device) ^ o])
        o //= 2
    return s[..., 0]


def rsqrt(v, em):
    r = 1.0 / torch.sqrt(v)
    if not em:
        return r
    sign = 1.0 - 2.0 * (torch.arange(r.numel(), device=r.device) % 2).view_as(r)
    return f32(f32(r) * (1.0 + RSQRT_ERR * sign))


def rope_cs(table, M, S, ncols, hd):
    """(cos, sin) [M, ncols / 2] of the interleaved pairs of ``ncols`` rotated columns at positions row % S."""
    return GR.rope_cs(table, torch.arange(M, device=table.device), ncols, hd, S, ncols)


def rot(x, c, s, em=False, inverse=False):
    """Interleaved rotation of x [M, 2 n] by (c, s) [M, n]; ``em``: fp32 products and sums, then bf16."""
    if inverse:
        s = -s
    if em:
        return GR.rope_em(x, c, s)
    x0, x1 = x[:, 0::2], x[:, 1::2]
    return torch.stack((x0 * c - x1 * s, x0 * s + x1 * c), -1).flatten(1)


def fp8_gemm(a, b, em):
    """a [M, K] @ b [N, K]^T on row-wise e4m3 operands (the fp8 branch's forward GEMM), scales applied; bf16 with ``em``."""
    qa, sa = GR.quant_rowwise_e4m3(a)
    qb, sb = GR.quant_rowwise_e4m3(b)
    if em:
        return GR.fp8_em(qa, qb.t(), sa, sb)
    return (qa @ qb.t()) * sa[:, None] * sb[None, :]


# ------------------------------------------------------------------------------------------------ QK-norm
def _gains(wq, wk, H, KVH, mut):
    a, b = (wk, wq) if mut == "wq_wk_swapped" else (wq, wk)
    return torch.cat([a.to(F64).expand(H, -1), b.to(F64).expand(KVH, -1)])        # [H + KVH, hd]


def qk_norm_fwd(qkv, wq, wk, table, S, H, KVH, hd, eps=EPS_QK, em=False, mut=None):
    """``qk_norm_rope`` on qkv [M, (H + 2 KVH) hd]: (qkv with its q / k heads normed and rotated [M, W], rstd
    [M, H + KVH]).  The V heads are returned unchanged."""
    M, nh = qkv.shape[0], H + KVH
    x = qkv.to(F64)[:, :nh * hd].reshape(M, nh, hd)
    c, s = rope_cs(table, M, S, nh * hd, hd)
    if mut == "norm_after_rope":
        x = rot(x.reshape(M, -1), c, s).view(M, nh, hd)      # the rotation keeps each head's sum of squares
    ms = lane_sum(f32(x * x) if em else x * x, em) / hd
    if mut == "rstd_no_eps":
        r = rsqrt(ms, em)
    elif mut == "eps_after_sqrt":
        r = 1.0 / (torch.sqrt(ms) + eps)
        r = f32(r) if em else r
    else:
        r = rsqrt(f32(ms + eps) if em else ms + eps, em)
    w = _gains(wq, wk, H, KVH, mut)
    y = f32(f32(x * r[..., None]) * w) if em else x * r[..., None] * w
    y = y.reshape(M, nh * hd)
    if mut != "norm_after_rope":
        y = rot(y, c, s, em)
    elif em:
        y = bf(y)
    return torch.cat([y, qkv.to(F64)[:, nh * hd:]], 1), r


def qk_norm_bwd(dqkv, xqk, rstd, wq, wk, H, KVH, hd, em=False, mut=None):
    """``qk_norm_bwd``: (dqkv with the q / k heads replaced by dx, dw_q, dw_k, |terms| sums of dw_q and dw_k, the dx row
    scale).  ``dqkv`` holds the gradient of the normed, un-rotated heads; ``xqk`` the pre-norm heads."""
    M, nh = dqkv.shape[0], H + KVH
    g = dqkv.to(F64)[:, :nh * hd].reshape(M, nh, hd)
    x = xqk.to(F64).reshape(M, nh, hd)
    r = rstd.to(F64).reshape(M, nh, 1)
    w = _gains(wq, wk, H, KVH, mut)
    xh = f32(x * r) if em else x * r
    gx = f32(g * xh) if em else g * xh
    wdot = gx if mut == "bwd_mean_without_w" else (f32(gx * w) if em else gx * w)
    dot = (lane_sum(wdot, em) / hd)[..., None]
    if em:
        dx = bf(f32(r * f32(f32(w * g) - f32(xh * dot))))
    else:
        dx = r * (w * g - xh * dot)
    scale = r * ((w * g).abs() + xh.abs() * (g * w * xh).abs().mean(-1, keepdim=True))
    gq, gk = gx[:, :H].reshape(-1, hd), gx[:, H:].reshape(-1, hd)
    dwq = fsum_rows(gk if mut == "dwq_sums_k_heads" else gq, em)
    dwk = fsum_rows(gk, em)
    out = torch.cat([dx.reshape(M, -1), dqkv.to(F64)[:, nh * hd:]], 1)
    return out, dwq, dwk, gq.abs().sum(0), gk.abs().sum(0), scale.reshape(M, -1)


# ------------------------------------------------------------------------------------------------ the nodes
def linear(x, w, dy, res=None, em=False, mut=None):
    """``linear``: {y, dx, dw, dres}.  x [M, K], w [N, K], dy [M, N]."""
    y = mm(x, w.t(), em)
    if res is not None:
        y = y + res.to(F64)
    dres = None
    if res is not None:
        dres = torch.zeros_like(dy, dtype=F64) if mut == "residual_grad_dropped" else dy.to(F64)
    return {"y": st(y, em), "dx": st(mm(dy, w, em), em), "dw": mm(dy.t(), x, em), "dres": dres}


def rmsnorm(x, w, dy, eps, dres=None, em=False, mut=None):
    """``rmsnorm`` (``dres`` None) or ``rmsnorm_fork`` with the residual branch's gradient ``dres``: {y, rstd, dx, dw,
    dw_abs}."""
    X, W, DY = x.to(F64), w.to(F64), dy.to(F64)
    D = X.shape[1]
    if em:
        from moe_reference import warp_sum
        r = rsqrt(f32(f32(warp_sum(f32(X * X)) / D) + eps), em)[:, None]
        y = bf(f32(f32(X * r) * W))
        xh = f32(X * r)
        dot = f32(warp_sum(f32(f32(DY * W) * xh)) / D)[:, None]
        dx = f32(r * f32(f32(DY * W) - f32(f32(X * r) * dot)))
    else:
        r = 1.0 / torch.sqrt((X * X).mean(1, keepdim=True) + eps)
        y = X * r * W
        xh = X * r
        dx = r * (DY * W - xh * (DY * W * xh).mean(1, keepdim=True))
    if dres is not None and mut != "dres_dropped":
        dx = dx + dres.to(F64)
        dx = f32(dx) if em else dx
    gx = f32(DY * xh) if em else DY * xh
    return {"y": y, "rstd": r.squeeze(1), "dx": st(dx, em), "dw": fsum_rows(gx, em), "dw_abs": gx.abs().sum(0)}


def gated_mlp(x, wg1, w2, dy, res=None, gate_first=True, fp8=False, em=False, mut=None):
    """``gated_mlp``: {y, dx, dwg1, dw2, dres, gu, act}.  x [M, D], wg1 [2F, D], w2 [D, F], dy [M, D]."""
    X, DY = x.to(F64), dy.to(F64)
    if fp8:
        gu = fp8_gemm(X, wg1, em)
        act = GR.swiglu_em(gu, gate_first)[1] if em else GR.swiglu_act(gu, gate_first)[0]
        y = fp8_gemm(act, w2, em)
        if res is not None:
            y = st(y + res.to(F64), em)
        dact = st(mm(DY, w2, em), em)
        dgu = GR.swiglu_bwd_em(dact, gu, gate_first) if em else GR.swiglu_bwd(dact, dact, gu, gate_first)[0]
    else:
        acc = mm(X, wg1.t(), em)
        gu, act = GR.swiglu_em(acc, gate_first) if em else (acc, GR.swiglu_act(acc, gate_first)[0])
        y = mm(act, w2.t(), em)
        if res is not None:
            y = y + res.to(F64)
        y = st(y, em)
        ds = mm(DY, w2, em)
        dgu = GR.swiglu_bwd_em(ds, gu, gate_first) if em else GR.swiglu_bwd(ds, ds, gu, gate_first)[0]
    dres = None
    if res is not None:
        dres = torch.zeros_like(DY) if mut == "residual_grad_dropped" else DY
    return {"y": y, "dx": st(mm(dgu, wg1, em), em), "dwg1": mm(dgu.t(), X, em), "dw2": mm(DY.t(), act, em),
            "dres": dres, "gu": gu, "act": act}


def qkv_attention(h, w, table, B, S, H, KVH, hd, do, seg=None, bias=None, qk=None, fp8=False, em=False, mut=None):
    """``qkv_attention`` in each form: plain, ``bias`` (the [N] projection bias) or ``qk`` = (w_q, w_k, eps); causal or
    with the document table ``seg``; the bf16 projection or (``fp8``) the row-wise e4m3 one.  h [B*S, D], w [N, D],
    do [B*S, H hd].  Returns {o, dh, dw, db, dwq, dwk} and the |terms| sums db_abs / dwq_abs / dwk_abs."""
    M = B * S
    nh = H + KVH
    H2 = h.to(F64).reshape(M, -1)
    c, s = rope_cs(table, M, S, nh * hd, hd)
    P = fp8_gemm(H2, w, em) if fp8 else mm(H2, w.t(), em)
    if bias is not None:
        P = P + bias.to(F64)[None]
        P = f32(P) if em else P
    out = {}
    if qk is not None:
        x0 = st(P, em)                                        # the plain projection, stored bf16
        qkv, rstd = qk_norm_fwd(x0, qk[0], qk[1], table, S, H, KVH, hd, qk[2], em)
    else:                                                     # RoPE in the projection epilogue (fp8: a separate pass)
        src = P if (em and not fp8) else st(P, em)
        qkv = torch.cat([rot(src[:, :nh * hd], c, s, em), st(src[:, nh * hd:], em)], 1)
    scale = hd ** -0.5
    # the attention backward's gradient of the rotated q / k (g_rot) and of the un-rotated ones (g)
    fused_inv = not fp8
    if em:
        o, _, g = AR.emulate(qkv.to(BF16).cpu(), do.cpu(), B, S, H, KVH, hd, scale, None if seg is None else seg.cpu(),
                             rope=table.cpu() if fused_inv and mut not in ("norm_bwd_rotated_grad",
                                                                           "inv_rope_after_norm_bwd",
                                                                           "bias_grad_rotated") else None)
        o, g = o.to(F64), g.to(F64)
        if not fused_inv or mut in ("norm_bwd_rotated_grad", "inv_rope_after_norm_bwd", "bias_grad_rotated"):
            g_rot = g
            g = torch.cat([rot(g_rot[:, :nh * hd], c, s, True, inverse=True), g_rot[:, nh * hd:]], 1)
        else:
            g_rot = None
    else:
        ref = AR.reference(qkv, do, B, S, H, KVH, hd, scale, seg=seg)
        o = ref["o"].reshape(M, H * hd)
        g_rot = torch.cat([ref["dq"].reshape(M, -1), ref["dk"].reshape(M, -1), ref["dv"].reshape(M, -1)], 1)
        del ref
        g = torch.cat([rot(g_rot[:, :nh * hd], c, s, inverse=True), g_rot[:, nh * hd:]], 1)
    out["o"] = o
    if qk is not None:
        src = g_rot if mut in ("norm_bwd_rotated_grad", "inv_rope_after_norm_bwd") else g
        xqk = x0[:, :nh * hd]
        g, dwq, dwk, aq, ak, _ = qk_norm_bwd(src, xqk, rstd, qk[0], qk[1], H, KVH, hd, em)
        if mut == "inv_rope_after_norm_bwd":
            g = torch.cat([rot(g[:, :nh * hd], c, s, em, inverse=True), g[:, nh * hd:]], 1)
        out.update(dwq=dwq, dwk=dwk, dwq_abs=aq, dwk_abs=ak)
    if bias is not None:
        gb = g_rot if mut == "bias_grad_rotated" else g
        out["db"] = fsum_rows(gb, em)
        out["db_abs"] = gb.abs().sum(0)
    out["dh"] = st(mm(g, w, em), em)
    out["dw"] = mm(g.t(), H2, em)
    return out


# ------------------------------------------------------------------------------ the independent autograd block
def _rope_ref(x, table, S):
    """Interleaved RoPE of x [B, S, n, hd] at positions 0..S-1, written out."""
    cs = table[:S].to(F64)
    c, s = cs[..., 0][None, :, None], cs[..., 1][None, :, None]
    x0, x1 = x[..., 0::2], x[..., 1::2]
    return torch.stack((x0 * c - x1 * s, x0 * s + x1 * c), -1).flatten(-2)


def _straight_through(exact, q):
    """q's value with exact's gradient (the fp8 branch: e4m3 forward, bf16 backward)."""
    return exact + (q - exact).detach()


def attention_autograd(h, w, table, B, S, H, KVH, hd, do, seg=None, bias=None, qk=None, fp8=False):
    """float64 autograd through a plain block: projection, optional bias, per-head RMSNorm, written-out RoPE, SDPA with
    an explicit causal or document mask.  Returns {o, dh, dw, db, dwq, dwk} as ``qkv_attention``."""
    leaves = {"h": h, "w": w}
    if bias is not None:
        leaves["b"] = bias
    if qk is not None:
        leaves["wq"], leaves["wk"] = qk[0], qk[1]
    L = {n: t.detach().to(F64).requires_grad_() for n, t in leaves.items()}
    x = L["h"].reshape(B * S, -1)
    qkv = x @ L["w"].t()
    if fp8:
        qkv = _straight_through(qkv, fp8_gemm(h.reshape(B * S, -1), w, False))
    if bias is not None:
        qkv = qkv + L["b"]
    t = qkv.view(B, S, H + 2 * KVH, hd)
    q, k, v = t[:, :, :H], t[:, :, H:H + KVH], t[:, :, H + KVH:]
    if qk is not None:
        eps = qk[2]
        q = q * torch.rsqrt(q.pow(2).mean(-1, keepdim=True) + eps) * L["wq"]
        k = k * torch.rsqrt(k.pow(2).mean(-1, keepdim=True) + eps) * L["wk"]
    q, k = _rope_ref(q, table, S), _rope_ref(k, table, S)
    G = H // KVH
    q, k, v = q.transpose(1, 2), k.repeat_interleave(G, 2).transpose(1, 2), v.repeat_interleave(G, 2).transpose(1, 2)
    pos = torch.arange(S, device=h.device)
    mask = pos[None, :] <= pos[:, None]
    if seg is not None:
        mask = mask[None] & (pos[None, None, :] >= seg[0].view(B, S).long()[:, :, None])
        mask = mask[:, None]
    o = torch.nn.functional.scaled_dot_product_attention(q, k, v, attn_mask=mask, scale=hd ** -0.5)
    o = o.transpose(1, 2).reshape(B * S, H * hd)
    grads = torch.autograd.grad((o * do.to(F64)).sum(), list(L.values()))
    gd = dict(zip(L.keys(), grads))
    out = {"o": o.detach(), "dh": gd["h"].reshape(B * S, -1), "dw": gd["w"]}
    if bias is not None:
        out["db"] = gd["b"]
    if qk is not None:
        out["dwq"], out["dwk"] = gd["wq"], gd["wk"]
    return out


def mlp_autograd(x, wg1, w2, dy, res=None, gate_first=True, fp8=False):
    L = [t.detach().to(F64).requires_grad_() for t in (x, wg1, w2)]
    X, WG1, W2 = L
    gu = X @ WG1.t()
    if fp8:
        gu = _straight_through(gu, fp8_gemm(x, wg1, False))
    F = gu.shape[1] // 2
    g, u = (gu[:, :F], gu[:, F:]) if gate_first else (gu[:, F:], gu[:, :F])
    act = torch.nn.functional.silu(g) * u
    y = act @ W2.t()
    if fp8:
        y = _straight_through(y, fp8_gemm(act.detach(), w2, False))
    R = None
    if res is not None:
        R = res.detach().to(F64).requires_grad_()
        y = y + R
    ins = L + ([R] if R is not None else [])
    gr = torch.autograd.grad((y * dy.to(F64)).sum(), ins)
    return {"y": y.detach(), "dx": gr[0], "dwg1": gr[1], "dw2": gr[2], "dres": gr[3] if R is not None else None}


def rmsnorm_autograd(x, w, dy, eps, dres=None):
    X, W = (t.detach().to(F64).requires_grad_() for t in (x, w))
    y = X * torch.rsqrt(X.pow(2).mean(1, keepdim=True) + eps) * W
    loss = (y * dy.to(F64)).sum() + (0 if dres is None else (X * dres.to(F64)).sum())   # the fork's second output is x
    dx, dw = torch.autograd.grad(loss, [X, W])
    return {"y": y.detach(), "dx": dx, "dw": dw}


# ------------------------------------------------------------------------------------------------ inputs
def qk_inputs(M, H, KVH, hd, regime, seed=0, device="cpu"):
    """bf16 (qkv [M, (H + 2 KVH) hd], w_q, w_k [hd], g [M, (H + 2 KVH) hd]) of one QK-norm regime:
      init     projections ~ N(0, 1), Qwen3-like gains around 1 (0.5 to 1.5, unequal within each pair)
      tiny     every q / k head at an rms of 10^u sqrt(eps), u uniform in [-1, 1] (mean square 0.01 to 100 eps), and
               every 7th head exactly zero
      outlier  one channel per head at 100x the others
      gains    gains log-uniform over 0.05 to 20 (a stress range, not read from a checkpoint)
    g ~ N(0, 1) is the gradient of the normed, un-rotated heads."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    nh, W = H + KVH, (H + 2 * KVH) * hd
    x = torch.randn(M, H + 2 * KVH, hd, generator=g)
    wq, wk = 0.5 + torch.rand(hd, generator=g), 0.5 + torch.rand(hd, generator=g)
    if regime == "tiny":
        u = torch.rand(M, nh, 1, generator=g) * 2 - 1
        x[:, :nh] *= (10.0 ** u) * math.sqrt(EPS_QK)
        x[:, :nh] *= (torch.arange(M * nh).view(M, nh, 1) % 7 != 0)
    elif regime == "outlier":
        ch = torch.randint(0, hd, (M, nh), generator=g)
        x[:, :nh].scatter_(2, ch[..., None], 100 * torch.sign(torch.randn(M, nh, 1, generator=g)))
    elif regime == "gains":
        lo, hi = math.log(0.05), math.log(20.0)
        wq, wk = (torch.exp(torch.rand(hd, generator=g) * (hi - lo) + lo) for _ in range(2))
    elif regime != "init":
        raise ValueError(regime)
    d = torch.randn(M, W, generator=g)
    return tuple(t.to(BF16).to(device) for t in (x.reshape(M, W), wq, wk, d))


def node_inputs(shapes, regime, seed=0, device="cpu"):
    """bf16 tensors of the given shapes ({name: shape}); names starting with ``w`` are weights at std 0.02 (``wq`` /
    ``wk``: gains 0.5 to 1.5; ``b``: a bias at std 0.5), the rest ~ N(0, 1).  ``outlier``: four channels of every
    activation at 30x (the last dim of ``h`` / ``x``)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    out = {}
    for n, shp in shapes.items():
        if n in ("wq", "wk"):
            t = 0.5 + torch.rand(*shp, generator=g)
        elif n.startswith("w"):
            t = torch.randn(*shp, generator=g) * 0.02
        elif n == "b":
            t = torch.randn(*shp, generator=g) * 0.5
        else:
            t = torch.randn(*shp, generator=g)
            if regime == "outlier" and n in ("h", "x"):
                t[..., torch.randint(0, shp[-1], (4,), generator=g)] *= 30
        out[n] = t.to(BF16).to(device)
    return out


# ------------------------------------------------------------------------------------- running the real nodes
UBF = 2.0 ** -8


def one_rounding(out, exact):
    """Worst |out - exact| / (2^-8 |exact|): at most 1 when ``out`` is ``exact`` rounded once to bf16 (to nearest);
    where ``exact`` is 0 the output must be 0."""
    return GR.ratio(out.reshape(-1), exact.reshape(-1).to(F64), UBF * exact.reshape(-1).to(F64).abs())


def run_node(call, acts, weights, dos, mode):
    """Run ``call()`` (the node on the leaves ``acts`` and the parameters ``weights``, both {name: tensor}) once per
    upstream gradient in ``dos``, delivering the weight gradients as ``mode`` says, the way ``ShardUnit.bind_grads``
    binds them:
      returned   no buffer: the node returns the gradient (one micro-batch only)
      fp32 / bf16  a zeroed slot of that dtype, stored by the first micro-batch and accumulated by the later ones
    Returns (the first micro-batch's output, {name: gradient of the activations, summed over the micro-batches},
    [{name: weight gradient or slot contents after each micro-batch}])."""
    for p in weights.values():
        p.grad, p._grad_ready = None, False
        p._grad_buf = None if mode == "returned" else torch.zeros(p.shape, dtype=getattr(torch, {
            "fp32": "float32", "bf16": "bfloat16"}[mode]), device=p.device)
    assert mode != "returned" or len(dos) == 1
    first, dacts, after = None, {}, []
    try:
        for do in dos:
            out = call()
            outs = out if isinstance(out, tuple) else (out,)
            first = outs if first is None else first
            # a whole backward, as the engine runs it: ``autograd.grad`` would skip the nodes that lead only to
            # parameters (``_NegExp`` of Mamba's A_log), whose gradients are delivered as a side effect
            for t in list(acts.values()) + list(weights.values()):
                t.grad = None
            torch.autograd.backward(outs, do if isinstance(do, tuple) else (do,))
            for n, a in acts.items():
                dacts[n] = a.grad if n not in dacts else dacts[n] + a.grad
            after.append({n: (p.grad if mode == "returned" else p._grad_buf.clone()) for n, p in weights.items()})
    finally:
        for t in list(acts.values()) + list(weights.values()):
            t.grad = None
        for p in weights.values():
            p._grad_buf, p._grad_ready = None, False
    return first, dacts, after
