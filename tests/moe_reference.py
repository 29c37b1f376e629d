"""Float64 reference, per-row metric and CPU rounding emulation of the mixture-of-experts kernels (``csrc/moe.cu`` and
the ``GRP_M`` / ``GRP_K`` grouped modes of ``csrc/gemm_sm90.cu``), shared by ``tests/test_moe_numerics_cpu.py`` and
``tests/test_moe_numerics_gpu.py``.  Not a test module (no ``test_`` prefix).

Every stage is a function of its inputs and a given plan (the int32 plan of ``moe_plan``), computed in float64 on the
inputs' device.  With ``em=True`` the same function instead rounds where the kernels round: the operands are bf16,
GEMM products are summed into an fp32 accumulator (modelled pessimistically below), and the results are rounded to
bf16 at exactly the points where a kernel writes bf16:

    h, and s = silu(gate) * up computed in fp32 from the rounded h          (gate/up GEMM, SwiGLU epilogue)
    yp; y after one fp32 combine over the slots (fused multiply-adds)       (down GEMM, combine)
    dY_perm = w dy; dH (SwiGLU backward of the fp32 dS and the bf16 h)      (combine backward, down dgrad)
    dX_perm; dh after the fp32 slot sum and the router dgrad's residual      (up dgrad, permute backward)
    dlogits (then once more after the router z-loss term is added)           (route backward)

The wgrads, logits, probabilities, weights and dw stay fp32.  fp32 accumulation: a tensor-core MMA sums 16 products
(k16) and adds them to the fp32 accumulator; the emulation adds each 16-product partial sum to the accumulator with
round-toward-zero (tensor cores are documented to truncate rather than round to nearest, so this is the pessimistic
model).  The softmax's exp and 1/x run as fast-math approximations; the emulation charges every exp a relative error of
2^-21 with alternating sign and rounds each step to fp32.

Routing is a discrete choice, so the node reference takes the top-k ids as an input (the kernels' own ids); near-ties
among 128 experts would otherwise dominate every comparison.

The metric (``ratio``): for every row, max|out - ref| over the row / max|ref| over the row; a row that is zero in the
reference must be exactly zero in the output (ratio 0, else inf); a non-finite output is inf.  Rows are tokens for y,
dh and every [Mpad, .] operand, and the output rows of each expert for the wgrads (dw1 [2F, D], dw2 [D, F]) and of the
router gradient [E, D].
"""
import math

import torch

F64, F32, BF16 = torch.float64, torch.float32, torch.bfloat16
KCHUNK = 16          # products the tensor core sums before they reach the fp32 accumulator (one k16 MMA)
EXP_ERR = 2.0 ** -21  # charged relative error of the fast-math exp / log

# Tolerances on the per-row ratio.  Each is 3x the worst ratio the rounding emulation (``em=True``) reaches over the
# regimes and shapes of tests/test_moe_numerics_cpu.py (init-scale, peaked and skewed routers at Qwen3-30B-A3B's D, E
# and k; the crafted segment counts with an 8448-row expert; norm_topk on and off), rounded up.  Worst emulated ratios:
#   bf16    3.9e-3  every bf16 output of one stage given its bf16 inputs (h, s, yp, y, dY_perm, dH, dX_perm, dx): one
#                   bf16 rounding, 2^-8 of the row max when the row max sits just under a power of two
#   dl      3.9e-3  dlogits of the route backward (bf16), per row against ``route_bwd_scale``
#   fp32    1.9e-5  fp32 outputs of a GEMM (the grouped wgrad stored or accumulated, the router logits): truncating
#                   fp32 accumulation, worst on the 8448-row segment
#   probs   8.5e-7  probabilities and weights: exp at 2^-21, the warp's fp32 sum and 1/x
#   dw      3.0e-6  dw of the combine backward, an fp32 dot over D
#   scalar  3.1e-6  aux and z
# Whole node (bf16 inputs, routing fixed to the kernels' ids): the bf16 roundings of h, s, dY_perm, dH and dlogits
# propagate, so these are bf16-sized even for the fp32 wgrads:
#   y 3.8e-3   dh 1.6e-2   dwr 1.7e-2 (peaked router, T 256)   dw1 4.2e-2 (peaked router)   dw2 2.3e-2
# The fp32 tolerance stays 65x below one bf16 rounding (3.9e-3): a kernel that passed an fp32 result through bf16
# fails it by that much.
TOL = {
    "bf16": 1.2e-2, "dl": 1.2e-2, "fp32": 6e-5, "probs": 2.6e-6, "dw": 1e-5, "scalar": 1e-5,
    "y": 1.2e-2, "dh": 4.8e-2, "dwr": 5e-2, "dw1": 0.13, "dw2": 7e-2,
}


# ------------------------------------------------------------------------------------------------ roundings
def bf(x):
    """Round to bf16 (through fp32, as a kernel's fp32 value is rounded), keep the dtype."""
    return x.to(F32).to(BF16).to(x.dtype)


def f32(x):
    return x.to(F32).to(x.dtype)


def rz32(x):
    """float64 -> the fp32 value next to it towards zero (truncation), as float64."""
    r = x.to(F32)
    over = r.to(F64).abs() > x.abs()
    return torch.where(over, torch.nextafter(r, torch.zeros_like(r)), r).to(F64)


def mm(a, b, em=False):
    """a [M, K] @ b [K, N] in float64; ``em``: the kernels' fp32 accumulation (k16 partial sums, truncating adds)."""
    a, b = a.to(F64), b.to(F64)
    if not em:
        return a @ b
    acc = torch.zeros(a.shape[0], b.shape[1], dtype=F64, device=a.device)
    for c in range(0, a.shape[1], KCHUNK):
        acc = rz32(acc + a[:, c:c + KCHUNK] @ b[c:c + KCHUNK])
    return acc


def warp_sum(x):
    """fp32 sum over the last dim the way a warp-per-row kernel sums it: element j of a row goes to lane j % 32 (8-wide
    vectors: lane (j / 8) % 32), each lane adds its elements in order, then a 5-level butterfly.  float64 in and out."""
    R, n = x.shape
    lanes = torch.zeros(R, 32, dtype=F64, device=x.device)
    for j in range(n):
        lanes[:, j % 32] = f32(lanes[:, j % 32] + x[:, j])
    for o in (16, 8, 4, 2, 1):
        lanes = f32(lanes + lanes[:, torch.arange(32, device=x.device) ^ o])
    return lanes[:, 0]


def _lane_order(x, vec):
    """Columns of x [R, D] reordered so that ``warp_sum``'s lane j % 32 gets what lane (d / vec) % 32 sums."""
    R, D = x.shape
    return x.view(R, D // (32 * vec), 32, vec).permute(0, 1, 3, 2).reshape(R, D) if D % (32 * vec) == 0 else x


def _exp(x, em):
    if not em:
        return torch.exp(x)
    sign = 1.0 - 2.0 * (torch.arange(x.numel(), device=x.device) % 2).view_as(x)
    return f32(torch.exp(x) * (1.0 + EXP_ERR * sign))


# --------------------------------------------------------------------------------------------------- metric
def ratio(out, ref, scale=None):
    """Worst per-row ratio max|out - ref| / max|ref| of two [R, N] tensors (a zero reference row must be exactly 0).
    ``scale``: judge each row against max|scale| over the row instead of max|ref| (``route_bwd_scale``)."""
    out, ref = out.to(F64).reshape(ref.shape[0], -1), ref.to(F64).reshape(ref.shape[0], -1)
    if out.numel() == 0:
        return 0.0
    err = torch.nan_to_num((out - ref).abs(), nan=math.inf).amax(1)
    mag = (ref if scale is None else scale.to(F64).reshape(ref.shape[0], -1)).abs().amax(1)
    r = torch.where(mag > 0, err / mag.clamp(min=1e-300), torch.where(err == 0, 0.0, math.inf))
    return float(r.max())


def scalar_ratio(out, ref):
    out, ref = float(out), float(ref)
    return abs(out - ref) / abs(ref) if ref else (0.0 if out == 0 else math.inf)


# ----------------------------------------------------------------------------------------------------- plan
def moe_rows(T, k, E):
    Mpad = (T * k + 127 * E + 127) // 128 * 128
    return Mpad, Mpad // 128


def views(plan, T, k, E):
    """(tile [NT], start [E], len [E], row [T, k], src [Mpad]) of a plan (``torch_kernels.moe_plan_views``)."""
    Mpad, NT = moe_rows(T, k, E)
    tile, start, length, row, src = torch.split(plan, [NT, E, E, T * k, Mpad])
    return tile.long(), start.long(), length.long(), row.view(T, k).long(), src.long()


def segments(plan, T, k, E):
    """[(start, len, padded len)] per expert, on the host."""
    _, start, length, _, _ = views(plan, T, k, E)
    return [(s, n, (n + 127) // 128 * 128) for s, n in zip(start.tolist(), length.tolist())]


def routed_rows(plan, T, k, E):
    """bool [Mpad]: rows that hold a (token, slot) entry."""
    Mpad = moe_rows(T, k, E)[0]
    m = torch.zeros(Mpad, dtype=torch.bool, device=plan.device)
    m[views(plan, T, k, E)[3].reshape(-1)] = True
    return m


def tile_experts(plan, T, k, E, mutation=None):
    """Expert of each 128-row tile (-1 past the last segment).  ``tile_first_shared_start``: a broken tile table that
    gives a tile to the first of several experts sharing its start (an empty one), not the last."""
    tile, start, _, _, _ = views(plan, T, k, E)
    if mutation == "tile_first_shared_start":
        first = torch.searchsorted(start, start, right=False)       # starts are non-decreasing
        tile = torch.where(tile >= 0, first[tile.clamp(min=0)], tile)
    return tile


# --------------------------------------------------------------------------------------------------- stages
def route(logits, ids, norm, em=False):
    """(probs [T, E], weights [T, k], lse [T]) of fp32 logits, for the given top-k ``ids``."""
    l = logits.to(F64)
    mx = l.amax(1, keepdim=True)
    x = l - mx
    if em:
        x = f32(x)
    e = _exp(x, em)
    s = warp_sum(e).unsqueeze(1) if em else e.sum(1, keepdim=True)
    if em:
        p = f32(e * f32(1.0 / s))
        lse = f32(f32(mx.squeeze(1) + torch.log(s.squeeze(1))) * (1.0 + EXP_ERR))
    else:
        p = e / s
        lse = mx.squeeze(1) + torch.log(s.squeeze(1))
    w = p.gather(1, ids.long())
    if norm:
        w = w / w.sum(1, keepdim=True)
        if em:
            w = f32(w)
    return p, w, lse


def aux_stat(probs, ids, E):
    """E / T^2 * sum_e count_e * sum_t p_te."""
    T = probs.shape[0]
    count = torch.bincount(ids.reshape(-1).long(), minlength=E).to(F64)
    return float((count * probs.to(F64).sum(0)).sum()) * E / (T * T)


def permute(x, plan, T, k, E):
    Mpad = moe_rows(T, k, E)[0]
    xp = torch.zeros(Mpad, x.shape[1], dtype=F64, device=x.device)
    xp[views(plan, T, k, E)[3].reshape(-1)] = x.to(F64).repeat_interleave(k, 0)
    return xp


def permute_bwd(dxp, plan, T, k, E, em=False):
    row = views(plan, T, k, E)[3]
    d = dxp.to(F64)
    acc = d[row[:, 0]]
    for s in range(1, k):
        acc = acc + d[row[:, s]]
        if em:
            acc = f32(acc)
    return bf(acc) if em else acc


def combine(yp, plan, wts, res, T, k, E, em=False):
    row = views(plan, T, k, E)[3]
    acc = res.to(F64) if res is not None else torch.zeros(T, yp.shape[1], dtype=F64, device=yp.device)
    for s in range(k):
        acc = acc + wts[:, s:s + 1].to(F64) * yp[row[:, s]].to(F64)
        if em:
            acc = f32(acc)                        # fused multiply-add: one fp32 rounding per slot
    return bf(acc) if em else acc


def combine_bwd(dy, yp, plan, wts, T, k, E, em=False):
    """(dY_perm [Mpad, D], zero in padding rows; dw [T, k] = <dy[t], Y_perm[row]>)."""
    row = views(plan, T, k, E)[3].reshape(-1)
    dyk = dy.to(F64).repeat_interleave(k, 0)
    dyp = torch.zeros(yp.shape, dtype=F64, device=yp.device)
    v = wts.reshape(-1, 1).to(F64) * dyk
    dyp[row] = bf(f32(v)) if em else v
    prod = dyk * yp[row].to(F64)
    if not em:
        return dyp, prod.sum(-1).view(T, k)
    # the kernel: each lane sums its 8-wide vectors two products at a time, then the butterfly
    pairs = f32(prod.view(prod.shape[0], -1, 2).sum(-1))
    return dyp, warp_sum(_lane_order(pairs, 4)).view(T, k)


def route_bwd(probs, ids, dw, norm, aux_scale, part="both", em=False, mutation=None):
    """dlogits [T, E] of the weights' gradient ``dw`` through the renormalisation and the softmax (part "dw"), of the
    load-balancing term aux_scale * count_e on every probability of expert e (part "aux"), or of both.  The weights
    are the probabilities' (renormalised) values, so only ``probs`` and ``ids`` are needed.  ``mutation``:
    ``aux_dropped`` / ``aux_negated``, a broken kernel's load-balancing term."""
    T, E = probs.shape
    il = ids.long()
    p = probs.to(F64)
    dp = torch.zeros_like(p)
    if part in ("dw", "both"):
        g = dw.to(F64)
        if norm:
            sel = p.gather(1, il)
            z = sel.sum(1, keepdim=True)
            g = (g - (g * sel / z).sum(1, keepdim=True)) / z
        dp.scatter_add_(1, il, g)
    if part in ("aux", "both"):
        a = aux_scale * {None: 1.0, "aux_dropped": 0.0, "aux_negated": -1.0}[mutation]
        dp = dp + a * torch.bincount(il.reshape(-1), minlength=E).to(F64)[None]
    if em:                          # the kernel: dp and the warp's dot in fp32, then p (dp - dot) rounded to bf16
        dp = f32(dp)
        return bf(f32(p * f32(dp - warp_sum(f32(p * dp)).unsqueeze(1))))
    return p * (dp - (p * dp).sum(1, keepdim=True))


def route_bwd_scale(probs, ids, dw, norm, aux_scale, part="both"):
    """What the route backward sums into each dlogit, in absolute values: p_e (|dp_e| + |sum_j p_j dp_j|).  A peaked
    softmax cancels dp_e against the dot in fp32 (the kernels' inputs are fp32), so dlogits are judged against this
    row scale rather than against max|dlogits|, which the cancellation can make arbitrarily small."""
    T, E = probs.shape
    il = ids.long()
    p = probs.to(F64)
    dp = torch.zeros_like(p)
    if part in ("dw", "both"):
        g = dw.to(F64)
        if norm:
            sel = p.gather(1, il)
            z = sel.sum(1, keepdim=True)
            g = (g - (g * sel / z).sum(1, keepdim=True)) / z
        dp.scatter_add_(1, il, g)
    if part in ("aux", "both"):
        dp = dp + aux_scale * torch.bincount(il.reshape(-1), minlength=E).to(F64)[None]
    return p * (dp.abs() + (p * dp).sum(1, keepdim=True).abs())


def _swiglu(h, em):
    F = h.shape[1] // 2
    g, u = h[:, :F], h[:, F:]
    s = g * torch.sigmoid(g) * u
    return bf(s) if em else s


def _swiglu_bwd(ds, h, em):
    F = h.shape[1] // 2
    g, u = h[:, :F], h[:, F:]
    sig = torch.sigmoid(g)
    d = torch.cat([ds * u * sig * (1 + g * (1 - sig)), ds * g * sig], 1)
    return bf(d) if em else d


def _grouped_m(a, w, plan, T, k, nt, em, mutation=None, epi=None, aux=None):
    """m-grouped product over each tile's expert: c[rows of e] = a @ w[e]^T (nt) or a @ w[e] (nn); rows of no expert
    are zero.  One expert's weights in float64 at a time."""
    E = w.shape[0]
    tile = tile_experts(plan, T, k, E, mutation).repeat_interleave(128)
    out = None
    for e in torch.unique(tile[tile >= 0]).tolist():
        idx = (tile == e).nonzero().squeeze(1)
        we = w[e].to(F64)
        c = mm(a[idx], we.t() if nt else we, em)
        if epi == "swiglu_bwd":
            c = _swiglu_bwd(c, aux[idx].to(F64), em)
        elif em:
            c = bf(c)
        if out is None:
            out = torch.zeros(a.shape[0], c.shape[1], dtype=F64, device=a.device)
        out[idx] = c
    return out


def up(xp, w1, plan, T, k, em=False, mutation=None):
    """(H = X_perm W1_e^T [Mpad, 2F], S = silu(gate) * up [Mpad, F]), S computed from H (rounded with ``em``)."""
    h = _grouped_m(xp, w1, plan, T, k, True, em, mutation)
    return h, _swiglu(h, em)


def down(sp, w2, plan, T, k, em=False):
    return _grouped_m(sp, w2, plan, T, k, True, em)


def down_bwd(dyp, w2, hp, plan, T, k, em=False):
    """dH = swiglu_bwd(dY_perm W2_e, H), the SwiGLU backward on the fp32 product."""
    return _grouped_m(dyp, w2, plan, T, k, False, em, epi="swiglu_bwd", aux=hp)


def up_dgrad(dhp, w1, plan, T, k, em=False):
    return _grouped_m(dhp, w1, plan, T, k, False, em)


def wgrad_expert(a, b, seg, em=False, base=None, mutation=None):
    """A_e^T B_e [M, N] of one expert (``seg`` = (start, len, padded len)) in float64; ``base``: the buffer it is
    accumulated onto.  ``em``: fp32 accumulation over the expert's 64-row k-blocks, stored (or added to ``base``) in
    fp32.  Mutations of the k-range (rows [64 kb0, 64 kb1) of the buffer, padding rows are zero):
      kend_floor_plus1   kb1 = floor((s + len) / 64) + 1: one k-block too many when len % 64 == 0
      kend_floor         kb1 = floor((s + len) / 64): the partial last k-block is dropped
      wgrad_bf16_store / wgrad_bf16_accum   the fp32 result (or the fp32 sum with ``base``) rounded through bf16"""
    s, n, _ = seg
    r1 = s + n
    if mutation == "kend_floor_plus1":
        r1 = (r1 // 64 + 1) * 64
    elif mutation == "kend_floor":
        r1 = r1 // 64 * 64
    r1 = min(r1, a.shape[0])
    if r1 <= s:
        c = torch.zeros(a.shape[1], b.shape[1], dtype=F64, device=a.device)
    else:
        c = mm(a[s:r1].t(), b[s:r1], em)
    if mutation == "wgrad_bf16_store" and base is None:
        c = bf(c)
    if base is not None:
        c = c + base.to(F64)
        if em:
            c = f32(c)
        if mutation == "wgrad_bf16_accum":
            c = bf(c)
    return c


# -------------------------------------------------------------------------------------------------- the node
def node(h, wr, w1, w2, res, dy, ids, norm, aux_coef, z_coef, em=False, on_expert=None, plan=None):
    """The whole ``moe_mlp`` node, forward and backward, with the routing fixed to ``ids``: a float64 reference, or
    with ``em`` the kernels' roundings.  Returns {y, dh, dwr, aux, z, logits, probs, wts}; the expert wgrads go to
    ``on_expert(e, dw1_e [2F, D], dw2_e [D, F])`` one expert at a time (a [T k, 2F] or [E, 2F, D] float64 buffer of a
    production shape would not fit next to the rest)."""
    T, D = h.shape
    E, k = wr.shape[0], ids.shape[1]
    if plan is None:
        from fms_fsdp_b200.ops import torch_kernels as TK
        plan = TK.moe_plan(ids.cpu(), torch.zeros(T, E))[0].to(h.device)
    H, WR = h.to(F64), wr.to(F64)
    logits = mm(H, WR.t(), em)
    probs, wts, lse = route(logits, ids, norm, em)
    aux = aux_stat(probs, ids, E)
    z = float((lse * lse).mean())
    xp = permute(H, plan, T, k, E)
    hp, sp = up(xp, w1, plan, T, k, em)
    yp = down(sp, w2, plan, T, k, em)
    y = combine(yp, plan, wts, res, T, k, E, em)
    dyp, dw = combine_bwd(dy, yp, plan, wts, T, k, E, em)
    dhp = down_bwd(dyp, w2, hp, plan, T, k, em)
    del yp
    for e, seg in enumerate(segments(plan, T, k, E)):
        if on_expert is not None:
            on_expert(e, wgrad_expert(dhp, xp, seg, em), wgrad_expert(dyp, sp, seg, em))
    del sp, hp, dyp
    dxp = up_dgrad(dhp, w1, plan, T, k, em)
    del dhp
    dhm = permute_bwd(dxp, plan, T, k, E, em)
    del dxp
    dl = route_bwd(probs, ids, dw, norm, aux_coef * E / (T * T), em=em)
    if z_coef > 0:
        zt = (2 * z_coef / T) * lse[:, None] * probs
        dl = bf(dl + f32(zt)) if em else dl + zt
    dh = mm(dl, WR, em) + dhm.to(F64)
    if em:
        dh = bf(f32(dh))
    dwr = mm(dl.t(), H, em)
    return {"y": y, "dh": dh, "dwr": dwr, "aux": aux, "z": z, "logits": logits, "probs": probs, "wts": wts}


def node_autograd(h, wr, w1, w2, res, dy, ids, norm, aux_coef, z_coef):
    """The same node by float64 autograd through a plain per-expert loop (no permuted buffer, no plan)."""
    T, D = h.shape
    E, k = wr.shape[0], ids.shape[1]
    F = w1.shape[1] // 2
    h, wr, w1, w2 = (t.detach().to(F64).requires_grad_() for t in (h, wr, w1, w2))
    lg = h @ wr.t()
    p = torch.softmax(lg, -1)
    lse = torch.logsumexp(lg, -1)
    il = ids.long()
    w = p.gather(1, il)
    if norm:
        w = w / w.sum(1, keepdim=True)
    out = torch.zeros_like(h)
    for e in range(E):
        m = il == e
        tok = m.any(1).nonzero().squeeze(1)
        if len(tok):
            g = h[tok] @ w1[e].t()
            a = torch.nn.functional.silu(g[:, :F]) * g[:, F:]
            out = out.index_add(0, tok, (w * m)[tok].sum(1, keepdim=True) * (a @ w2[e].t()))
    y = res.to(F64) + out
    count = torch.bincount(il.reshape(-1), minlength=E).to(F64)
    aux = (count * p.sum(0)).sum() * E / (T * T)
    z = (lse * lse).mean()
    loss = (y * dy.to(F64)).sum() + aux_coef * aux + z_coef * z
    dh, dwr, dw1, dw2 = torch.autograd.grad(loss, [h, wr, w1, w2])
    return {"y": y.detach(), "dh": dh, "dwr": dwr, "dw1": dw1, "dw2": dw2, "aux": float(aux), "z": float(z)}


# ---------------------------------------------------------------------------------------------------- inputs
def node_inputs(T, D, E, F, regime, seed=0, device="cpu"):
    """bf16 (h, router w, w1, w2, residual, dy).  Regimes: ``init`` (router std 0.02, logit std ~0.02 sqrt(D)),
    ``peaked`` (logit std ~4), ``skewed`` (every token leans towards a direction that four experts' router rows
    favour: their segments hold most of the rows).  Expert weights at std 0.02, like a fresh model."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, sc=1.0: torch.randn(*s, generator=g) * sc
    h = r(T, D)
    wr = r(E, D, sc=0.02 if regime != "peaked" else 4.0 / math.sqrt(D))
    if regime == "skewed":
        u = torch.nn.functional.normalize(r(D), dim=0)
        h = h + 2.0 * u
        wr[:4] += 1.5 / 2.0 * u          # logit ~ +1.5 on experts 0..3 for every token
    w1, w2 = r(E, 2 * F, D, sc=0.02), r(E, D, F, sc=0.02)
    res, dy = r(T, D), r(T, D)
    return tuple(t.to(BF16).to(device) for t in (h, wr, w1, w2, res, dy))


def crafted_ids(counts, T, k):
    """int32 ids [T, k] in which expert e is chosen by exactly ``counts[e]`` (token, slot) entries, each token's k
    experts distinct.  sum(counts) must be T k; entries are dealt round-robin over the experts' lists."""
    assert sum(counts) == T * k
    flat = torch.cat([torch.full((c,), e, dtype=torch.int32) for e, c in enumerate(counts)])
    # column-major deal: entry j goes to token j % T, slot j // T, so one expert's (contiguous) entries land on
    # distinct tokens as long as its count is <= T
    assert max(counts) <= T
    return flat.view(k, T).t().contiguous()
