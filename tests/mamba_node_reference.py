"""Float64 reference and CPU rounding emulation of the Mamba2-hybrid nodes of ``models/mamba.py`` (the ``Mamba2`` and
``Mamba1`` mixers, the hybrid's ``MHA`` layer, the value-first ``GatedMLP``, ``Block`` with its fp32 residual stream, and
the ends: ``engine_embed`` + ``engine_head``), shared by ``tests/test_mamba_nodes_cpu.py`` and
``tests/test_mamba_nodes_gpu.py``.  Not a test module (no ``test_`` prefix).

Each node is written out from its formulas in float64 (never through ``ops.torch_kernels``, the ATen path the suite
also compares against) and differentiated by autograd.  A vector parameter (A_log, dt_bias, D, the conv taps and bias,
the norm gains) enters as a per-token copy, a [M, ...] leaf broadcast from the parameter, so its gradient comes out as
the per-token contributions: their sum is the gradient and the sum of their absolute values is the scale it is judged
against (``LR.vratio``), so a wrong element of a small gradient cannot hide behind a large one.

The SSD scan has two forms: the sequential recurrence (``ssd_seq``) and the chunked state-space-dual form
(``ssd_chunked``) the kernels follow.  With ``em=True`` the nodes round to bf16 where the sm_90a kernels store bf16
(``st``: the value in forward and the gradient flowing back through that point in backward) and run every GEMM through
the fp32 tensor-core accumulator (``gemm_reference.acc_em``):

    GEMMs             bf16 outputs of the fp32 accumulator; fp32 weight gradients
    causal conv1d     bf16 output; bf16 dx
    SSD forward       bf16 CB, Mh, yd, xs, prev, yoff and y (chunk 128); fp32 dt, its cumulative sum and the states
    SSD backward      bf16 gradients at those points and at x, B, C and dt (dys, dMh, dxd, dCB, dstates, dxs, dx, ddt)
    selective scan    bf16 y, du, ddelta and dz; fp32 carried states
    gated RMSNorm     bf16 y, dx and dz; fp32 rstd
    add + RMSNorm     the fp32 residual sum, bf16 y and bf16 gradient of the hidden input
    attention         ``attention_reference.emulate``; the gated MLP ``LR.gated_mlp(em=True)``
"""
import math

import torch
import torch.nn.functional as Fn

import attention_reference as AR
import gemm_reference as GR
import llama_node_reference as LR
from moe_reference import BF16, F64, bf, f32, ratio

# Tolerances on the per-row ratio (``LR.vratio`` for the vector gradients).  Each is 3x the worst ratio of the rounding
# emulation (``em=True``) over the regimes (init, slow, trained) and the shapes of tests/test_mamba_nodes_cpu.py, rounded
# up.  Worst emulated ratios:
#     m2_y 1.8e-2   m2_dx 2.4e-2   m2_dw 1.7e-2   m2_dv 6.7e-3     Mamba2 mixer (trained; dv: A_log, dt_bias, D, conv, gain)
#     m1_y 8.9e-3   m1_dx 7.0e-3   m1_dw 3.5e-2   m1_dv 2.3e-2     Mamba1 mixer (dw: dt_proj's rows, slow)
#     mha_y 7.0e-3  mha_dx 6.1e-3  mha_dw 7.1e-3                   MHA
#     mlp_y 7.1e-3  mlp_dx 6.2e-3  mlp_dw 5.6e-3                   GatedMLP
#     blk_y 1.1e-2  blk_dx 2.0e-2  blk_dw 6.9e-2  blk_dv 2.5e-2    Block, both outputs and gradients (dw, dv: Mamba1)
#     end_loss 2.4e-5  end_dw 9.7e-3  end_tied_dw 0.16  end_dv 2.6e-3
#                   the ends (embedding, norm_f, fused head), logits at production scale: the head stores them bf16, and
#                   a tied head's logit of a token against its own row is about 51 at mamba_2.8b, where bf16 is 0.25
#                   coarse; the weight rows are judged against the sum of |terms|
TOL = {
    "m2_y": 5.4e-2, "m2_dx": 7.3e-2, "m2_dw": 5.1e-2, "m2_dv": 2.1e-2,
    "m1_y": 2.7e-2, "m1_dx": 2.1e-2, "m1_dw": 0.11, "m1_dv": 7e-2,
    "mha_y": 2.2e-2, "mha_dx": 1.9e-2, "mha_dw": 2.2e-2,
    "mlp_y": 2.2e-2, "mlp_dx": 1.9e-2, "mlp_dw": 1.7e-2,
    "blk_y": 3.3e-2, "blk_dx": 5.9e-2, "blk_dw": 0.21, "blk_dv": 7.6e-2,
    "end_loss": 7.2e-5, "end_dw": 2.9e-2, "end_tied_dw": 0.47, "end_dv": 7.9e-3,
}

# ``mut``: plausible bugs, each failing the check of tests/test_mamba_nodes_cpu.py that targets it
MIXER_MUTATIONS = ("conv_no_restart", "conv_taps_reversed", "dt_bias_after_softplus", "no_D", "state_across_rows",
                   "decay_off_by_one", "head_group_map", "norm_before_gate", "norm_all_groups", "split_zxbcdt",
                   "split_xBC", "negexp_sign")
MHA_MUTATIONS = ("rope_interleaved", "rope_all_dims", "rope_no_inverse_grad")

EPS = 1e-5


# ------------------------------------------------------------------------------------------------ roundings
class _Store(torch.autograd.Function):
    """A bf16 storage point: the value rounds in forward, the gradient flowing back through it rounds in backward."""

    @staticmethod
    def forward(ctx, x):
        return bf(x)

    @staticmethod
    def backward(ctx, g):
        return bf(g)


def st(x, em):
    return _Store.apply(x) if em else x


class _MM(torch.autograd.Function):
    """a [M, K] @ b [K, N] through the fp32 accumulator, forward and backward (``gemm_reference.acc_em``)."""

    @staticmethod
    def forward(ctx, a, b):
        ctx.save_for_backward(a, b)
        return GR.acc_em(a, b)

    @staticmethod
    def backward(ctx, g):
        a, b = ctx.saved_tensors
        return GR.acc_em(g, b.t()), GR.acc_em(a.t(), g)


def lin(x, w, em):
    """x @ w^T stored bf16 (``ops.linear``)."""
    return st(_MM.apply(x, w.t()) if em else x @ w.t(), em)


def silu(x):
    return x * torch.sigmoid(x)


def softplus(x):
    return torch.where(x > 20, x, torch.log1p(torch.exp(torch.clamp(x, max=20))))


def neg_exp(a_log, mut=None):
    """A = -exp(A_log); ``negexp_sign``: the right value with the gradient's sign flipped."""
    e = torch.exp(a_log)
    if mut == "negexp_sign":
        return -e.detach() + (e - e.detach())
    return -e


# ---------------------------------------------------------------------------------------------- the pieces
def conv(x, w, b, S, em=False, mut=None):
    """Depthwise causal conv (K taps, bias) + SiLU of x [M, C], restarting at each sequence of S tokens.  w [M, C, K] and
    b [M, C] are per-token copies; tap k multiplies x[t - (K - 1 - k)]."""
    M, C = x.shape
    K = w.shape[-1]
    rows = 1 if mut == "conv_no_restart" else M // S
    xv, wv = x.view(rows, -1, C), w.view(rows, -1, C, K)
    acc = b.view(rows, -1, C)
    for k in range(K):
        sh = K - 1 - k
        xs = Fn.pad(xv, (0, 0, sh, 0))[:, :xv.shape[1]]
        tap = wv[..., K - 1 - k] if mut == "conv_taps_reversed" else wv[..., k]
        acc = acc + tap * xs
    return st(silu(acc).reshape(M, C), em)


def _ssd_prep(x, dt, A, Bm, Cm, dt_bias, S, mut):
    M, H, P = x.shape
    G = Bm.shape[1]
    dtv = softplus(dt) + dt_bias if mut == "dt_bias_after_softplus" else softplus(dt + dt_bias)
    hg = torch.arange(H, device=x.device) % G if mut == "head_group_map" else torch.arange(H, device=x.device) // (H // G)
    a = dtv * A
    rows = 1 if mut == "state_across_rows" else M // S
    if mut == "decay_off_by_one":                  # step t decays by step t + 1's factor
        av = a.view(M // S, S, H)
        a = torch.cat([av[:, 1:], av[:, -1:]], 1).reshape(M, H)
    return dtv, a, Bm[:, hg], Cm[:, hg], rows


def ssd_seq(x, dt, A, Bm, Cm, D, dt_bias, S, mut=None):
    """SSD by its recurrence: h_t = exp(dt_t A) h_(t-1) + dt_t x_t B_t^T, y_t = h_t C_t + D x_t, restarting at each
    sequence.  x [M, H, P]; dt, A, D, dt_bias [M, H] (per token); Bm, Cm [M, G, N]; head h reads group h // (H / G)."""
    M, H, P = x.shape
    dtv, a, Bh, Ch, rows = _ssd_prep(x, dt, A, Bm, Cm, dt_bias, S, mut)
    L = M // rows
    xv, dv, av, Bv, Cv = (t.reshape(rows, L, *t.shape[1:]) for t in (x, dtv, a, Bh, Ch))
    h = torch.zeros(rows, H, P, Bm.shape[-1], dtype=x.dtype, device=x.device)
    ys = []
    for t in range(L):
        h = torch.exp(av[:, t])[..., None, None] * h + (dv[:, t, :, None] * xv[:, t])[..., None] * Bv[:, t, :, None, :]
        ys.append((h * Cv[:, t, :, None, :]).sum(-1))
    y = torch.stack(ys, 1).reshape(M, H, P)
    return y if mut == "no_D" else y + D[..., None] * x


def ssd_chunked(x, dt, A, Bm, Cm, D, dt_bias, S, chunk, em=False, mut=None):
    """SSD in the chunked form of ``csrc/ssd.cu``: per chunk, the intra-chunk term yd = Mh x with Mh = mask(C B^T
    exp(acs_i - acs_j) dt_j), the chunk-end states from xs = x dt exp(aL - acs), the states passed across chunks (prev),
    and yoff = C prev scaled by exp(acs).  A last chunk shorter than ``chunk`` is allowed."""
    M, H, P = x.shape
    dtv, a, Bh, Ch, rows = _ssd_prep(x, dt, A, Bm, Cm, dt_bias, S, mut)
    G = Bm.shape[1]
    L = M // rows
    xv, dv, av = (t.reshape(rows, L, *t.shape[1:]) for t in (x, dtv, a))
    Bg, Cg = Bm.reshape(rows, L, G, -1), Cm.reshape(rows, L, G, -1)
    Bv, Cv = Bh.reshape(rows, L, H, -1), Ch.reshape(rows, L, H, -1)
    hg = torch.arange(H, device=x.device) % G if mut == "head_group_map" else torch.arange(H, device=x.device) // (H // G)
    prev = torch.zeros(rows, H, P, Bm.shape[-1], dtype=x.dtype, device=x.device)
    ys = []
    for c0 in range(0, L, chunk):
        sl = slice(c0, min(c0 + chunk, L))
        n = sl.stop - c0
        xc, dc = xv[:, sl], dv[:, sl]
        acs = torch.cumsum(av[:, sl], 1)                                     # [r, n, H]
        acs = f32(acs) if em else acs
        CB = st(torch.einsum("bign,bjgn->bgij", Cg[:, sl], Bg[:, sl]), em)  # [r, G, n, n]
        mask = torch.ones(n, n, dtype=torch.bool, device=x.device).tril()
        seg = (acs.transpose(1, 2)[..., :, None] - acs.transpose(1, 2)[..., None, :]).masked_fill(~mask, -math.inf)
        Mh = st(CB[:, hg] * torch.exp(seg) * dc.transpose(1, 2)[:, :, None, :], em)      # [r, H, n, n]
        yd = st(torch.einsum("bhij,bjhp->bihp", Mh, xc), em)
        aL = acs[:, -1]                                                      # [r, H]
        xs = st(xc * (dc * torch.exp(aL[:, None] - acs))[..., None], em)
        states = torch.einsum("bjhn,bjhp->bhpn", Bv[:, sl], xs)
        yoff = st(torch.einsum("bihn,bhpn->bihp", Cv[:, sl], st(prev, em)), em)
        ys.append(yd + torch.exp(acs)[..., None] * yoff)
        prev = torch.exp(aL)[..., None, None] * prev + states
        prev = f32(prev) if em else prev
    y = torch.cat(ys, 1).reshape(M, H, P)
    return y if mut == "no_D" else y + D[..., None] * x


def gated_norm(x, z, w, group_size, em=False, mut=None):
    """RMSNormGated(norm_before_gate=False): rmsnorm over groups of ``group_size`` of x silu(z), times w [M, d]."""
    M, d = x.shape
    g = x if mut == "norm_before_gate" else x * silu(z)
    gs = d if mut == "norm_all_groups" else group_size
    u = g.view(M, d // gs, gs)
    r = 1.0 / torch.sqrt((u * u).mean(-1, keepdim=True) + EPS)
    r = f32(r) if em else r
    y = (u * r).view(M, d) * w
    if mut == "norm_before_gate":
        y = y * silu(z)
    return st(y, em)


def selective_scan(u, delta, A, Bm, Cm, D, z, delta_bias, S):
    """Mamba1: h_t = exp(d_t A) h_(t-1) + d_t u_t B_t, y = (h_t C_t + D u_t) silu(z_t), d = softplus(delta + bias).
    u, delta, z, D, delta_bias [M, C]; A [M, C, N]; Bm, Cm [M, N]."""
    M, C = u.shape
    rows = M // S
    d = softplus(delta + delta_bias)
    dv, uv, Av = d.view(rows, S, C), u.view(rows, S, C), A.view(rows, S, C, -1)
    Bv, Cv = Bm.view(rows, S, -1), Cm.view(rows, S, -1)
    h = torch.zeros(rows, C, A.shape[-1], dtype=u.dtype, device=u.device)
    ys = []
    for t in range(S):
        h = torch.exp(dv[:, t, :, None] * Av[:, t]) * h + (dv[:, t] * uv[:, t])[..., None] * Bv[:, t, None, :]
        ys.append((h * Cv[:, t, None, :]).sum(-1))
    y = torch.stack(ys, 1).reshape(M, C) + D * u
    return y * silu(z)


def rope_half(qkv, S, H, KVH, hd, rot, base=10000.0, mut=None):
    """mamba_ssm's partial rotary: columns (i, i + rot/2), i < rot/2, of each q and k head rotated by position * base^(-2i
    / rot); the other columns and V unchanged.  ``rope_interleaved``: pairs (2i, 2i + 1); ``rope_all_dims``: rot = hd;
    ``rope_no_inverse_grad``: the gradient passes back unrotated."""
    M = qkv.shape[0]
    rot = hd if mut == "rope_all_dims" else rot
    nh = H + KVH
    pos = (torch.arange(M, device=qkv.device) % S).to(F64)
    ang = pos[:, None] * base ** (-torch.arange(0, rot, 2, device=qkv.device, dtype=F64) / rot)
    c, s = torch.cos(ang)[:, None], torch.sin(ang)[:, None]
    src = qkv.detach() if mut == "rope_no_inverse_grad" else qkv
    h = src[:, :nh * hd].view(M, nh, hd)
    if mut == "rope_interleaved":
        x1, x2 = h[..., 0:rot:2], h[..., 1:rot:2]
        r = torch.stack((x1 * c - x2 * s, x1 * s + x2 * c), -1).flatten(-2)
    else:
        x1, x2 = h[..., :rot // 2], h[..., rot // 2:rot]
        r = torch.cat((x1 * c - x2 * s, x1 * s + x2 * c), -1)
    out = torch.cat((r, h[..., rot:]), -1).reshape(M, nh * hd)
    out = torch.cat((out, src[:, nh * hd:]), 1)
    if mut == "rope_no_inverse_grad":
        out = out + (qkv - qkv.detach())
    return out


class _Attention(torch.autograd.Function):
    """Causal GQA softmax attention on a roped projection [M, (H + 2 KVH) hd]: ``attention_reference.reference`` in
    float64, or its kernel emulation (``em``)."""

    @staticmethod
    def forward(ctx, qkv, B, S, H, KVH, hd, em):
        ctx.args = (B, S, H, KVH, hd, em)
        ctx.save_for_backward(qkv)
        return _Attention._run(qkv, torch.zeros(B * S, H * hd, dtype=F64, device=qkv.device), *ctx.args)[0]

    @staticmethod
    def backward(ctx, do):
        (qkv,) = ctx.saved_tensors
        return (_Attention._run(qkv, do, *ctx.args)[1],) + (None,) * 6

    @staticmethod
    def _run(qkv, do, B, S, H, KVH, hd, em):
        M = B * S
        if em:
            o, _, g = AR.emulate(qkv.to(BF16).cpu(), do.to(BF16).cpu(), B, S, H, KVH, hd, hd ** -0.5)
            return o.to(F64).to(qkv.device), g.to(F64).to(qkv.device)
        r = AR.reference(qkv, do, B, S, H, KVH, hd, hd ** -0.5)
        g = torch.cat([r["dq"].reshape(M, -1), r["dk"].reshape(M, -1), r["dv"].reshape(M, -1)], 1)
        return r["o"].reshape(M, H * hd), g


class _MLP(torch.autograd.Function):
    """``LR.gated_mlp`` as an autograd node."""

    @staticmethod
    def forward(ctx, x, wg1, w2, gate_first, em):
        ctx.args = (gate_first, em)
        ctx.save_for_backward(x, wg1, w2)
        return LR.gated_mlp(x, wg1, w2, torch.zeros(x.shape[0], w2.shape[0], dtype=F64, device=x.device),
                            gate_first=gate_first, em=em)["y"]

    @staticmethod
    def backward(ctx, dy):
        x, wg1, w2 = ctx.saved_tensors
        r = LR.gated_mlp(x, wg1, w2, dy, gate_first=ctx.args[0], em=ctx.args[1])
        return r["dx"], r["dwg1"], r["dw2"], None, None


# ------------------------------------------------------------------------------------------------ the nodes
def mamba2(p, u, S, cfg, em=False, mut=None, chunk=None):
    """``Mamba2.forward`` on u [M, D]; ``p``: {parameter name: float64 tensor}, vector parameters as per-token copies.
    ``chunk`` None: the sequential SSD; else the chunked form at that chunk length."""
    di, H, P, G, N = cfg["d_inner"], cfg["nheads"], cfg["headdim"], cfg["ngroups"], cfg["d_state"]
    C = di + 2 * G * N
    M = u.shape[0]
    zxbcdt = lin(u, p["in_proj.weight"], em)
    if mut == "split_zxbcdt":
        xBC, z, dt = torch.split(zxbcdt, [C, di, H], 1)
    else:
        z, xBC, dt = torch.split(zxbcdt, [di, C, H], 1)
    xc = conv(xBC, p["conv1d.weight"].view(M, C, -1), p["conv1d.bias"], S, em, mut)
    if mut == "split_xBC":
        x, Cm, Bm = torch.split(xc, [di, G * N, G * N], 1)
    else:
        x, Bm, Cm = torch.split(xc, [di, G * N, G * N], 1)
    x, Bm, Cm, z, dt = (st(t, em) for t in (x, Bm, Cm, z, dt))
    A = neg_exp(p["A_log"], mut)
    args = (x.reshape(M, H, P), dt, A, Bm.reshape(M, G, N), Cm.reshape(M, G, N), p["D"], p["dt_bias"], S)
    y = ssd_seq(*args, mut=mut) if chunk is None else ssd_chunked(*args, chunk, em, mut)
    y = gated_norm(st(y.reshape(M, di), em), z, p["norm.weight"], di // G, em, mut)
    return lin(y, p["out_proj.weight"], em)


def mamba1(p, u, S, cfg, em=False, mut=None):
    """``Mamba1.forward`` on u [M, D]."""
    di, N, R = cfg["d_inner"], cfg["d_state"], cfg["dt_rank"]
    M = u.shape[0]
    x, z = torch.split(lin(u, p["in_proj.weight"], em), [di, di], 1)
    x = conv(st(x, em), p["conv1d.weight"].view(M, di, -1), p["conv1d.bias"], S, em, mut)
    dt, Bm, Cm = torch.split(lin(x, p["x_proj.weight"], em), [R, N, N], 1)
    delta = lin(st(dt, em), p["dt_proj.weight"], em)
    y = selective_scan(st(x, em), st(delta, em), neg_exp(p["A_log"], mut), st(Bm, em), st(Cm, em), p["D"], st(z, em),
                       p["dt_proj.bias"], S)
    return lin(st(y, em), p["out_proj.weight"], em)


def mha(p, x, S, cfg, em=False, mut=None):
    """``MHA.forward`` on x [M, D]: projection, partial half-split rotary, causal GQA attention, out_proj."""
    H, KVH, hd, rot = cfg["num_heads"], cfg["num_heads_kv"], cfg["head_dim"], cfg["rotary_emb_dim"]
    M = x.shape[0]
    qkv = st(rope_half(lin(x, p["in_proj.weight"], em), S, H, KVH, hd, rot, mut=mut), em)
    o = _Attention.apply(qkv, M // S, S, H, KVH, hd, em)
    return lin(st(o, em), p["out_proj.weight"], em)


def gated_mlp(p, x, em=False, mut=None):
    """``GatedMLP.forward``: value first (``gate_first=False``); ``gate_value_swapped``: gate first."""
    return _MLP.apply(x, p["fc1.weight"], p["fc2.weight"], mut == "gate_value_swapped", em)


def add_rmsnorm(x, res, w, em=False, mut=None):
    """(rmsnorm(res + x) w stored bf16, res + x in fp32); ``residual_grad_dropped``: the residual output's gradient is
    lost."""
    ro = st(x, em) + res
    ro = f32(ro) if em else ro
    r = 1.0 / torch.sqrt((ro * ro).mean(-1, keepdim=True) + EPS)
    r = f32(r) if em else r
    y = st(ro * r * w, em)
    return y, (ro.detach() if mut == "residual_grad_dropped" else ro)


def block(p, hidden, residual, S, cfg, em=False, mut=None, chunk=None):
    """``Block.forward``: (hidden, residual) -> (hidden, residual)."""
    h, r = add_rmsnorm(hidden, residual, p["norm.weight"], em, mut)
    mp = {k[6:]: v for k, v in p.items() if k.startswith("mixer.")}
    kind = cfg["mixer"]
    if kind == "Mamba2":
        h = mamba2(mp, h, S, cfg, em, mut, chunk)
    elif kind == "MHA":
        h = mha(mp, h, S, cfg, em, mut)
    else:
        h = mamba1(mp, h, S, cfg, em, mut)
    if "norm2.weight" in p:
        h, r = add_rmsnorm(h, r, p["norm2.weight"], em, mut)
        h = gated_mlp({k[4:]: v for k, v in p.items() if k.startswith("mlp.")}, h, em, mut)
    return h, r


class _LinearCE(torch.autograd.Function):
    """Mean cross-entropy of y @ w^T over the labels that are not ``ignore``, computed in row blocks; ``em``: bf16
    logits and bf16 dlogits, as the fused head stores them.  Backward leaves |dlogits|^T |y|, the sum of the magnitudes
    of the terms of each element of dW, in ``stats["head_abs"]``."""

    @staticmethod
    def forward(ctx, y, w, labels, ignore, rows, em, stats):
        ctx.save_for_backward(y, w, labels)
        ctx.args, ctx.stats = (ignore, rows, em), stats
        loss, _, _, _ = _LinearCE._run(y, w, labels, ignore, rows, em, False)
        return loss

    @staticmethod
    def backward(ctx, g):
        y, w, labels = ctx.saved_tensors
        _, dy, dw, dw_abs = _LinearCE._run(y, w, labels, *ctx.args, True)
        if ctx.stats is not None:
            ctx.stats["head_abs"] = dw_abs * g.abs()
        return dy * g, dw * g, None, None, None, None, None

    @staticmethod
    def _run(y, w, labels, ignore, rows, em, grads):
        valid = labels != ignore
        n = valid.sum()
        loss = torch.zeros((), dtype=F64, device=y.device)
        dy = torch.zeros_like(y) if grads else None
        dw = torch.zeros_like(w) if grads else None
        dw_abs = torch.zeros_like(w) if grads else None
        for r0 in range(0, y.shape[0], rows):
            sl = slice(r0, r0 + rows)
            lg = st(y[sl] @ w.t(), em)
            lse = torch.logsumexp(lg, 1)
            v, lab = valid[sl], labels[sl].clamp(min=0)
            loss += ((lse - lg.gather(1, lab[:, None])[:, 0]) * v).sum() / n
            if grads:
                dl = torch.exp(lg - lse[:, None])
                dl[torch.arange(dl.shape[0], device=y.device), lab] -= 1
                dl *= (v / n)[:, None]
                dl = st(dl, em)
                dy[sl] = dl @ w
                dw += dl.t() @ y[sl]
                dw_abs += dl.abs().t() @ y[sl].abs()
        return loss, dy, dw, dw_abs


def ends(p, tokens, labels, tied, em=False, ignore=-100, rows=1024, stats=None):
    """``engine_embed`` then ``engine_head`` (norm_f on the fp32 residual, then the fused linear cross-entropy)."""
    emb = p["backbone.embedding.weight"]
    h = emb[tokens]
    y, _ = add_rmsnorm(h, torch.zeros_like(h), p["backbone.norm_f.weight"], em)
    return _LinearCE.apply(y, emb if tied else p["lm_head.weight"], labels, ignore, rows, em, stats)


def head_scales(res, stats, tied, emb="backbone.embedding.weight", head="lm_head.weight"):
    """Row scales of the head's weight gradient: each element's sum of |terms| (``stats`` of ``ends``), since a row of
    dW sums a token's dlogits times y over every token and those terms cancel.  ``tied``: the head was evaluated as a
    separate leaf holding the embedding's values; the embedding's gradient becomes the sum of the two, its scale the
    head's plus |embedding part|."""
    if tied:
        a, b = res[emb], res.pop(head)
        res[emb], res[emb + "_scale"] = a + b, a.abs() + stats["head_abs"]
    else:
        res[head + "_scale"] = stats["head_abs"]
    return res


# --------------------------------------------------------------------------------------- running the references
def is_vector(name, t):
    """Parameters judged element by element: every 1-D parameter, the conv taps and Mamba1's [C, N] A_log."""
    return t.dim() == 1 or name.endswith("conv1d.weight") or name.endswith("A_log")


def evaluate(fn, params, acts, douts, M, em=False, device=None):
    """Run ``fn(p, a)`` (returning a tuple of outputs) on float64 leaves made from the bf16 ``params`` and ``acts`` and
    differentiate it against ``douts``.  Returns {"out": [outputs], "d<act>": gradient, "<param>": gradient,
    "<param>_abs": sum over the tokens of |per-token contribution| (vector parameters only)}."""
    L = {}
    for n, t in params.items():
        t = t.detach().to(device=device, dtype=F64)
        L[n] = (t.expand(M, *t.shape).clone() if is_vector(n, t) else t).requires_grad_()
    A = {n: (t.detach().to(device=device, dtype=F64).requires_grad_() if t.is_floating_point() else t.to(device))
         for n, t in acts.items()}
    outs = fn(L, A)
    outs = outs if isinstance(outs, tuple) else (outs,)
    da = [n for n, t in A.items() if t.is_floating_point()]
    leaves = [A[n] for n in da] + list(L.values())
    pairs = [(o, d) for o, d in zip(outs, douts) if o.requires_grad]
    gr = torch.autograd.grad([o for o, _ in pairs], leaves, [d.to(device=device, dtype=F64) for _, d in pairs],
                             allow_unused=True)
    res = {"out": [o.detach() for o in outs]}
    for n, g in zip(da, gr[:len(da)]):
        res["d" + n] = torch.zeros_like(A[n]) if g is None else g
    for (n, t), g in zip(params.items(), gr[len(da):]):
        g = torch.zeros_like(L[n]) if g is None else g
        if is_vector(n, t):
            res[n] = (LR.fsum_rows(g.reshape(M, -1), True) if em else g.sum(0)).reshape(t.shape)
            res[n + "_abs"] = g.abs().sum(0).reshape(t.shape)
        else:
            res[n] = g
    return res


def ratios(prefix, out, ref, params, M):
    """{<prefix>_y, <prefix>_dx, <prefix>_dw, <prefix>_dv}: worst per-token ratio of the outputs and the activation
    gradients, per output row of the weight gradients, ``vratio`` of the vector gradients."""
    r = {prefix + "_y": max(ratio(o.reshape(M, -1), q.reshape(M, -1)) for o, q in zip(out["out"], ref["out"]))}
    acts = [k for k in ref if k != "out" and not k.endswith("_abs") and k not in params]
    r[prefix + "_dx"] = max(ratio(out[k].reshape(M, -1), ref[k].reshape(M, -1)) for k in acts)
    dw = [ratio(out[n], ref[n]) for n, t in params.items() if not is_vector(n, t)]
    dv = [LR.vratio(out[n], ref[n], ref[n + "_abs"]) for n, t in params.items() if is_vector(n, t)]
    if dw:
        r[prefix + "_dw"] = max(dw)
    if dv:
        r[prefix + "_dv"] = max(dv)
    return r


def mixer_cfg(m):
    """The config dict of a ``Mamba2`` / ``Mamba1`` / ``MHA`` module."""
    if hasattr(m, "nheads"):
        return dict(mixer="Mamba2", d_inner=m.d_inner, nheads=m.nheads, headdim=m.headdim, ngroups=m.ngroups,
                    d_state=m.d_state)
    if hasattr(m, "dt_rank"):
        return dict(mixer="Mamba1", d_inner=m.d_inner, d_state=m.d_state, dt_rank=m.dt_rank)
    return dict(mixer="MHA", num_heads=m.num_heads, num_heads_kv=m.num_heads_kv, head_dim=m.head_dim,
                rotary_emb_dim=m.rotary_emb_dim)


def set_regime(mixer, regime, seed=0):
    """Parameters of a Mamba2 / Mamba1 mixer for a regime (after ``reset_parameters``):
      init     as reset
      slow     A in [0.05, 0.5] and softplus(dt_bias) in [1e-3, 4e-3], so exp(dt A) summed over any 128-step chunk
               stays above 0.5
      trained  conv bias, D and dt_bias drawn from N(0, 0.3)"""
    g = torch.Generator().manual_seed(seed + 77)
    with torch.no_grad():
        if regime == "slow":
            n = mixer.A_log.shape[0]
            a = torch.empty(n).uniform_(0.05, 0.5, generator=g)
            mixer.A_log.copy_(torch.log(a).view(-1, *([1] * (mixer.A_log.dim() - 1))).expand_as(mixer.A_log))
            dt = torch.empty(n).uniform_(1e-3, 4e-3, generator=g)
            bias = mixer.dt_bias if hasattr(mixer, "dt_bias") else mixer.dt_proj.bias
            bias.copy_(dt + torch.log(-torch.expm1(-dt)))
        elif regime == "trained":
            mixer.conv1d.bias.copy_(torch.randn(mixer.conv1d.bias.shape, generator=g) * 0.3)
            mixer.D.copy_(torch.randn(mixer.D.shape, generator=g) * 0.3)
            bias = mixer.dt_bias if hasattr(mixer, "dt_bias") else mixer.dt_proj.bias
            bias.copy_(torch.randn(bias.shape, generator=g) * 0.3)
        elif regime != "init":
            raise ValueError(regime)
