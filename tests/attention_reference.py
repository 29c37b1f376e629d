"""Float64 reference, per-row error bound and CPU rounding emulation of the causal GQA attention kernels
(``csrc/attention_sm90.cu``), shared by ``tests/test_attention_numerics_cpu.py`` and
``tests/test_attention_numerics_gpu.py``.  Not a test module (no ``test_`` prefix).

Why per row.  For causal attention ``|o_q|`` shrinks roughly like ``1 / sqrt(q + 1)`` and dV of a late key sums few
queries, so a single ``max|a - b| / max|b|`` over a tensor is set by the first rows and lets the last rows of every head
be wrong by tens of percent.  Here every output row is judged against the size of what was summed into it: the same
expression with every factor replaced by its absolute value (the usual forward-error bound of a dot product),

    o   row q : P @ |V|
    dv  row k : P^T @ |dO|                                   (summed over the heads of the GQA group)
    dq  row q : scale * (P o (|dP| + |delta|_abs)) @ |K|     |delta|_abs = sum_d |dO| |O|
    dk  row k : scale * (P o (|dP| + |delta|_abs))^T @ |Q|   (summed over the heads of the GQA group)

and the row's error is its largest element error over the row's largest bound element.  ``|delta|_abs`` covers the
true cancellation in ``dP - delta`` on near-one-hot rows, where the kernel's delta (from the bf16 O) is off by up to
2^-8 |delta|_abs.  lse is checked per row in absolute terms, since it sits in an exponent.

Layouts follow the kernels: qkv [B*S, (H + 2 KVH) * hd] with the q heads, then the k heads, then the v heads; o and
dO [B*S, H * hd]; lse [B, H, S] in natural log; q head h reads kv head h // (H / KVH).
"""
import math

import torch

F64 = torch.float64
F32 = torch.float32
LOG2E = 1.4426950408889634
LN2 = 0.6931471805599453
TILE = 128          # kv tile of the forward kernels (the online-softmax step)

# Rows whose exact bound is below FLOOR are judged against FLOOR.  The kernels are built with --use_fast_math, so P
# below 2^-126 flushes to zero; what that drops from a row is at most S * 2^-126 * max|dO| < 2^-100 for S <= 2^16 and
# |dO| < 2^8, and a row that only holds such terms carries no information.
FLOOR = 2.0 ** -100

# Tolerances on the per-row ratio |error| / bound (lse: absolute error in natural-log units).  Each is the worst ratio
# of the CPU rounding emulation (``emulate`` below) over every regime, shape, document layout and the RoPE case of the
# test_emulated_kernel_* tests in tests/test_attention_numerics_cpu.py, times a safety factor of 3, rounded up.  Worst
# emulated ratios (and where):
#   o   6.1e-3  (documents, peaked16)  bf16 rounding of P (relative to the running max) and of O: each at most 2^-8
#   dv  6.7e-3  (documents, peaked16)  bf16 rounding of P and of dV: each at most 2^-8 (near-one-hot columns)
#   dq  2.2e-3  (sink, S 1000)         bf16 rounding of dS and of dQ, delta from the bf16 O
#   dk  5.2e-3  (documents, boosted)   as dq, summed over the GQA group
#   lse 1.9e-5  (peaked16)             fp32 running max and sum, the ln <-> log2 round trip, at logits up to ~75
# The tensor cores' fp32 accumulation order differs from the emulation's by fp32 roundings, ~2^-24 of the bound, and
# exp2 / log2 / 1/l run as fast-math approximations with relative errors near 2^-22: far below these.
TOL = {"o": 1.9e-2, "dv": 2.1e-2, "dq": 7e-3, "dk": 1.6e-2, "lse": 6e-5}

REGIMES = ("flat", "peaked6", "peaked16", "sink", "late_max", "ties")


# ------------------------------------------------------------------------------------------------------- inputs
def make_inputs(regime, B, S, H, KVH, hd, seed, boost=None):
    """bf16 (qkv [B*S, (H + 2 KVH) hd], dO [B*S, H hd]) on the CPU, independent data per batch row.

    flat      q, k, v, dO ~ N(0, 1): logits scale * q.k have std ~1
    peaked6   q and k scaled by sqrt(6): logit std ~6
    peaked16  q and k scaled by 4: logit std ~16, max ~75 over a 4096-long row (QK-norm models)
    sink      key 0 of every head lies along a direction u that every query leans towards: logit ~10 +- 2.5 against ~1
              for the others, so most queries put most of their probability on it (attention sinks)
    late_max  the keys of the last 160 positions (the last one or two kv tiles; the second half when S < 320) lean
              towards u by a logit of ~12: a row's running max jumps in its last kv tiles, after all the others were
              summed under the small max
    ties      q = 0 on a random half of the rows: exact ties, uniform softmax
    boosted   as late_max, on the key positions ``boost`` (bool [S]) instead
    """
    g = torch.Generator().manual_seed(seed)
    W = (H + 2 * KVH) * hd
    x = torch.randn(B, S, H + 2 * KVH, hd, generator=g, dtype=F64)
    do = torch.randn(B * S, H * hd, generator=g, dtype=F64)
    q, k = x[:, :, :H], x[:, :, H:H + KVH]
    G = H // KVH
    u = torch.nn.functional.normalize(torch.randn(B, 1, KVH, hd, generator=g, dtype=F64), dim=-1)
    uq = u.repeat_interleave(G, dim=2)
    if regime in ("peaked6", "peaked16"):
        c = math.sqrt(6.0) if regime == "peaked6" else 4.0
        q.mul_(c)
        k.mul_(c)
    elif regime == "sink":
        q.add_(4.0 * uq)                                       # q.u ~ 4 + N(0, 1)
        k[:, 0] = 2.5 * math.sqrt(hd) * u[:, 0]                 # scale * q.k0 = 2.5 q.u ~ 10 +- 2.5
    elif regime in ("late_max", "boosted"):
        if regime == "late_max":
            boost = torch.arange(S) >= max(S - 160, S // 2)
        q.add_(4.0 * uq)
        k[:, boost] += 3.0 * math.sqrt(hd) * u                  # scale * q.k ~ 12 + N(0, ~3) on the boosted keys
    elif regime == "ties":
        zero = torch.rand(B, S, H, generator=g) < 0.5
        q.masked_fill_(zero.unsqueeze(-1), 0.0)
    elif regime != "flat":
        raise ValueError(regime)
    return x.reshape(B * S, W).bfloat16(), do.bfloat16()


def segments(seps_per_row, S, device="cpu"):
    """``ops.document_segments`` table of a packed batch whose row r has separator tokens at ``seps_per_row[r]``."""
    from fms_fsdp_b200 import ops
    tok = torch.zeros(len(seps_per_row), S, dtype=torch.long)
    for r, seps in enumerate(seps_per_row):
        for p in seps:
            if p < S:
                tok[r, p] = 1
    return ops.document_segments(tok.to(device), 1)


def doc_layouts(S):
    """Separator positions per batch row: documents that start mid-tile, runs of 1-token documents (at a tile edge and
    at the end), and two documents the second of which has a far lower max (with the "boosted" regime on the first)."""
    return {
        "mid_tile": [[100, 300, 517, 700], [40, 250, 900]],
        "one_token": [[0, 1, 2, 127, 128, 129, 500, S - 2], [63, 64, 65, S - 1]],
        "low_after_high": [[S // 2 + 37], [S // 3]],
    }


def _split(qkv, B, S, H, KVH, hd):
    t = qkv.view(B, S, H + 2 * KVH, hd)
    return t[:, :, :H], t[:, :, H:H + KVH], t[:, :, H + KVH:]


def _visible(seg, b, S, device):
    """[S, S] bool: key k visible to query q (causal, and inside q's document when ``seg`` is given)."""
    kk = torch.arange(S, device=device)
    vis = kk.view(1, S) <= kk.view(S, 1)
    if seg is not None:
        vis &= kk.view(1, S) >= seg[0].view(-1, S)[b].long().view(S, 1)
    return vis


def _inv_rope(x, table, absolute=False):
    """Inverse interleaved RoPE of x [..., S, hd] at positions 0..S-1 (as the backward epilogue applies it); with
    ``absolute``, the same map with |cos| and |sin|, which carries a bound on x to a bound on the rotated x."""
    S, hd = x.shape[-2], x.shape[-1]
    cs = table[:S].to(x.dtype)
    c, s = cs[..., 0], cs[..., 1]
    if absolute:
        c, s = c.abs(), s.abs()
    x0, x1 = x[..., 0::2], x[..., 1::2]
    if absolute:
        return torch.stack([x0 * c + x1 * s, x0 * s + x1 * c], dim=-1).flatten(-2)
    return torch.stack([x0 * c + x1 * s, x1 * c - x0 * s], dim=-1).flatten(-2)


# ------------------------------------------------------------------------------------------ float64 reference
def reference(qkv, do, B, S, H, KVH, hd, scale, seg=None, rope=None):
    """Float64 attention forward and backward, with the per-row bounds, on the device of the inputs.

    Computed one (batch row, kv head) at a time, with the whole GQA group of that kv head at once, so S = 4096 at
    H = 32 fits.  ``rope``: the [S, hd/2, 2] table; dq and dk are returned with the inverse rotation applied, as the
    backward epilogue does.

    Returns a dict: o, dq [B, S, H, hd]; dk, dv [B, S, KVH, hd]; lse [B, H, S]; and the row bounds o_bound, dq_bound
    [B, S, H] and dk_bound, dv_bound [B, S, KVH].
    """
    G = H // KVH
    dev = qkv.device
    q, k, v = _split(qkv, B, S, H, KVH, hd)
    dO = do.view(B, S, H, hd)
    out = {n: torch.empty(B, S, H, hd, dtype=F64, device=dev) for n in ("o", "dq")}
    out.update({n: torch.empty(B, S, KVH, hd, dtype=F64, device=dev) for n in ("dk", "dv")})
    out.update({n: torch.empty(B, S, H, dtype=F64, device=dev) for n in ("o_bound", "dq_bound")})
    out.update({n: torch.empty(B, S, KVH, dtype=F64, device=dev) for n in ("dk_bound", "dv_bound")})
    out["lse"] = torch.empty(B, H, S, dtype=F64, device=dev)
    for b in range(B):
        vis = _visible(seg, b, S, dev)
        for kvh in range(KVH):
            hs = slice(kvh * G, kvh * G + G)
            qg = q[b, :, hs].transpose(0, 1).to(F64)                   # [G, S, hd]
            dog = dO[b, :, hs].transpose(0, 1).to(F64)
            kk, vv = k[b, :, kvh].to(F64), v[b, :, kvh].to(F64)         # [S, hd]
            s = (qg @ kk.T).mul_(scale).masked_fill_(~vis, -math.inf)   # [G, S, S]
            lse = torch.logsumexp(s, dim=-1)
            p = s.sub_(lse.unsqueeze(-1)).exp_()
            del s
            o = p @ vv
            dp = dog @ vv.T
            delta = (dog * o).sum(-1, keepdim=True)
            delta_abs = (dog.abs() * o.abs()).sum(-1, keepdim=True)
            ds = p * (dp - delta)
            x = p * dp.abs_().add_(delta_abs)                         # P o (|dP| + |delta|_abs)
            del dp
            dq, dq_b = scale * (ds @ kk), scale * (x @ kk.abs())
            dk, dk_b = scale * (ds.transpose(-1, -2) @ qg).sum(0), scale * (x.transpose(-1, -2) @ qg.abs()).sum(0)
            del ds, x
            if rope is not None:
                dq, dk = _inv_rope(dq, rope), _inv_rope(dk, rope)
                dq_b, dk_b = _inv_rope(dq_b, rope, absolute=True), _inv_rope(dk_b, rope, absolute=True)
            out["o"][b, :, hs] = o.transpose(0, 1)
            out["o_bound"][b, :, hs] = (p @ vv.abs()).amax(-1).T
            out["lse"][b, hs] = lse
            out["dv"][b, :, kvh] = (p.transpose(-1, -2) @ dog).sum(0)
            out["dv_bound"][b, :, kvh] = (p.transpose(-1, -2) @ dog.abs()).sum(0).amax(-1)
            del p
            out["dq"][b, :, hs] = dq.transpose(0, 1)
            out["dq_bound"][b, :, hs] = dq_b.amax(-1).T
            out["dk"][b, :, kvh] = dk
            out["dk_bound"][b, :, kvh] = dk_b.amax(-1)
    return out


def kernel_view(o, lse, dqkv, B, S, H, KVH, hd):
    """Kernel outputs (o [B*S, H hd], lse [B, H, S], dqkv) in the layout of ``reference``."""
    dq, dk, dv = _split(dqkv, B, S, H, KVH, hd)
    return {"o": o.view(B, S, H, hd), "lse": lse, "dq": dq, "dk": dk, "dv": dv}


def row_ratios(out, ref):
    """Per-row |error| / bound of o, dq, dk, dv ([B, S, heads]) and the absolute lse error ([B, heads, S])."""
    r = {}
    for n in ("o", "dq", "dk", "dv"):
        err = (out[n].to(F64) - ref[n]).abs().amax(-1)
        r[n] = err / ref[n + "_bound"].clamp(min=FLOOR)
    r["lse"] = (out["lse"].to(F64) - ref["lse"]).abs()
    return r


def worst(out, ref):
    """{output: worst per-row ratio (lse: worst absolute error)}."""
    return {n: v.max().item() for n, v in row_ratios(out, ref).items()}


def failures(out, ref):
    """Outputs whose worst per-row ratio exceeds its tolerance, or that hold a non-finite element."""
    bad = [n for n, v in worst(out, ref).items() if not v <= TOL[n]]
    return bad + [n + " not finite" for n, t in out.items() if not torch.isfinite(t).all()]


# ---------------------------------------------------------------------------------- the check this replaces
def old_check(o, lse, dqkv, ref, B, S, H, KVH, hd):
    """The global check of the first attention tests: max|a - b| / max|b| over o (< 1e-2), lse (< 1e-4) and the whole
    [dq | dk | dv] matrix (< 1.5e-2).  ``ref`` from ``reference``.  True = passes."""
    def rel(a, b):
        return ((a.to(F64) - b).abs().max() / b.abs().max()).item()
    dq = ref["dq"].reshape(B * S, H * hd)
    dk, dv = ref["dk"].reshape(B * S, KVH * hd), ref["dv"].reshape(B * S, KVH * hd)
    return (rel(o, ref["o"].reshape(B * S, H * hd)) < 1e-2 and rel(lse, ref["lse"]) < 1e-4
            and rel(dqkv, torch.cat([dq, dk, dv], dim=1)) < 1.5e-2)


# ---------------------------------------------------------------------------------- rounding emulation
MUTATIONS = ("no_o_rescale", "drop_last_kv_tile", "stale_lse_max", "lse_ln2_4_digits", "delta_next_row_tail",
             "dv_tail_x1.05", "gqa_last_group", "dkdv_floor_tiles", "dq_short_last_tile")


def _bf16(x):
    return x.to(torch.bfloat16).to(x.dtype)


def _fma_exp2(s, a, c):
    """exp2f(fmaf(s, a, c)) in fp32: the fma rounded once (through float64, exact for fp32 operands)."""
    return torch.exp2((s.to(F64) * a + c.to(F64)).to(F32))


def emulate(qkv, do, B, S, H, KVH, hd, scale, seg=None, rope=None, mutation=None):
    """The kernels' arithmetic in fp32 on the CPU, with their roundings: (o bf16, lse fp32, dqkv bf16) as the kernels
    return them.

    Forward, per kv tile of 128: S = Q K^T in fp32; running max m in log2 units (max of S times scale * log2 e, both
    fp32), m_sub = 0 while a row has seen no key; corr = exp2(m_old - m_sub); P = exp2(fma(S, scale log2e, -m_sub));
    l = l corr + sum P (fp32 P); O = O corr + bf16(P) V.  O = bf16(O * (1 / l)); lse = (m + log2 l) ln 2.
    Backward: delta = sum dO O over the bf16 O; P = exp2(fma(S, scale log2e, -lse log2e)); dS = P (dP - delta);
    dV = sum over the group of bf16(P)^T dO; dK = scale sum bf16(dS)^T Q; dQ = scale bf16(dS) K; inverse RoPE in fp32,
    then bf16.

    ``mutation`` (one of MUTATIONS) makes it a plausibly broken kernel:
      no_o_rescale       O not rescaled when the running max grows (corr applied to l only)
      drop_last_kv_tile  rows of the last q tile skip the last kv tile (their diagonal tile)
      stale_lse_max      lse written with the running max from before the row's last kv tile
      lse_ln2_4_digits   lse converted from log2 with ln 2 written as 0.6931 (a relative error of 7e-5)
      delta_next_row_tail  the backward reads delta of row q + 1 for the rows of the last 64-row tile
      dv_tail_x1.05      dV of the last 64 keys scaled by 1.05
      gqa_last_group     the forward maps the q heads of the last GQA group to kv head KVH - 2
      dkdv_floor_tiles   the dK/dV kernel counts its streamed 64-row q tiles as S // 64: the queries of a ragged
                         tail add nothing to dK / dV
      dq_short_last_tile the dQ kernel stops one streamed 64-row kv tile short for the rows of the last q tile
    """
    assert mutation is None or mutation in MUTATIONS, mutation
    G = H // KVH
    n_t = (S + TILE - 1) // TILE
    q, k, v = (t.float() for t in _split(qkv, B, S, H, KVH, hd))
    dO = do.view(B, S, H, hd).float()
    sl2 = torch.tensor(scale, dtype=F32) * torch.tensor(LOG2E, dtype=F32)   # scale * LOG2E, fp32 as on the device
    sc32 = torch.tensor(scale, dtype=F32)
    o_out = torch.empty(B, S, H, hd, dtype=F32)
    lse_out = torch.empty(B, H, S, dtype=F32)
    dqkv = torch.empty(B, S, H + 2 * KVH, hd, dtype=F32)
    rows = torch.arange(S)
    for b in range(B):
        vis = _visible(seg, b, S, "cpu")
        for kvh in range(KVH):
            hs = slice(kvh * G, kvh * G + G)
            qg = q[b, :, hs].transpose(0, 1)                     # [G, S, hd]
            fk = KVH - 2 if (mutation == "gqa_last_group" and kvh == KVH - 1 and KVH > 1) else kvh
            kk, vv = k[b, :, fk], v[b, :, fk]
            m = torch.full((G, S), -math.inf)
            m_stale = m.clone()
            l = torch.zeros(G, S)
            o = torch.zeros(G, S, hd)
            for j in range(n_t):
                ks = slice(j * TILE, min(j * TILE + TILE, S))
                s = (qg @ kk[ks].T).masked_fill(~vis[:, ks], -math.inf)
                if mutation == "drop_last_kv_tile" and j == n_t - 1 and n_t > 1:
                    s[:, (n_t - 1) * TILE:] = -math.inf
                m_new = torch.maximum(m, s.amax(-1) * sl2)
                m_sub = torch.where(m_new == -math.inf, torch.zeros(()), m_new)
                corr = torch.exp2(m - m_sub)
                p = _fma_exp2(s, sl2, -m_sub.unsqueeze(-1))
                l = l * corr + p.sum(-1)
                if mutation != "no_o_rescale":
                    o = o * corr.unsqueeze(-1)
                o = o + _bf16(p) @ vv[ks]
                m_stale = torch.where(rows // TILE == j, m, m_stale)   # the max before the row's diagonal tile
                m = m_new
            og = _bf16(o * (1.0 / l).unsqueeze(-1))
            m_lse = torch.where(m_stale == -math.inf, m, m_stale) if mutation == "stale_lse_max" else m
            lse = (m_lse + torch.log2(l)) * (0.6931 if mutation == "lse_ln2_4_digits" else LN2)
            o_out[b, :, hs] = og.transpose(0, 1)
            lse_out[b, hs] = lse
    for b in range(B):
        vis = _visible(seg, b, S, "cpu")
        for kvh in range(KVH):
            hs = slice(kvh * G, kvh * G + G)
            qg, dog, og = (t[b, :, hs].transpose(0, 1) for t in (q, dO, o_out))
            kk, vv = k[b, :, kvh], v[b, :, kvh]
            nd = -(dog * og).sum(-1)                                # -delta, from the bf16 O
            if mutation == "delta_next_row_tail":
                tail = rows >= (S - 1) // 64 * 64
                nd = torch.where(tail, nd[:, (rows + 1).clamp(max=S - 1)], nd)
            nl = -lse_out[b, hs] * torch.tensor(LOG2E, dtype=F32)
            p = _fma_exp2(qg @ kk.T, sl2, nl.unsqueeze(-1)).masked_fill(~vis, 0.0)
            ds = p * (dog @ vv.T + nd.unsqueeze(-1))
            if mutation == "dq_short_last_tile":
                short = (rows >= (S - 1) // TILE * TILE).view(S, 1) & (rows >= (S - 1) // 64 * 64).view(1, S)
                dq = (_bf16(ds.masked_fill(short, 0.0)) @ kk) * sc32
            else:
                dq = (_bf16(ds) @ kk) * sc32
            if mutation == "dkdv_floor_tiles":
                tail = (rows >= S // 64 * 64).view(S, 1)
                p, ds = p.masked_fill(tail, 0.0), ds.masked_fill(tail, 0.0)
            dv = (_bf16(p).transpose(-1, -2) @ dog).sum(0)
            if mutation == "dv_tail_x1.05":
                dv[-64:] *= 1.05
            dk = (_bf16(ds).transpose(-1, -2) @ qg).sum(0) * sc32
            if rope is not None:
                dq, dk = _inv_rope(dq, rope.float()), _inv_rope(dk, rope.float())
            dqkv[b, :, hs] = dq.transpose(0, 1)
            dqkv[b, :, H + kvh] = dk
            dqkv[b, :, H + KVH + kvh] = dv
    return (o_out.reshape(B * S, H * hd).bfloat16(), lse_out,
            dqkv.reshape(B * S, (H + 2 * KVH) * hd).bfloat16())
