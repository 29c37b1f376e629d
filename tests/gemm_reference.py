"""Float64 reference, element bound and CPU rounding emulation of the dense GEMM (``csrc/gemm_sm90.cu`` and the
128 x 256 tile of ``csrc/gemm_wide_sm90.cu``, which gives the same bits), shared by ``tests/test_gemm_numerics_cpu.py``
and ``tests/test_gemm_numerics_gpu.py``.  Not a test module (no ``test_`` prefix).

Reference.  Every epilogue is computed in float64 from the exact bf16 (or dequantised e4m3) operands: P = sum_k a b.
The RoPE table and the projection bias are taken as given (fp32 / bf16 values); the SwiGLU activation is computed from
the kernel's own bf16 projection ``gu``, as the kernel computes it, so the forward and the backward see the same values.

Element bound.  With A = sum_k |a| |b| (float64), the fp32 accumulator is within  delta = tau(K) 2^-24 A  of P.  delta
is carried through the epilogue's derivative (the pair's two accumulators for the rotation; |u s (1 + g (1 - s))| and
|g s| for the SwiGLU backward), the epilogue's own fp32 roundings are added (2^-24 per operation of the magnitudes
involved; the fast exp2f at 2^-21, as in tests/moe_reference.py), and one output rounding: 2^-8 of the magnitude for
bf16, 2^-24 for fp32.  ``ratio`` is max |out - ref| / bound over the elements; a non-finite output is inf, and where
the bound is 0 (an all-zero operand row) the output must be exactly 0.

The output rounding term is the exact worst case of a round-to-nearest bf16 store (half an ulp is 2^-8 of a value
just above a power of two), so a correct kernel can reach a ratio close to 1 on the bf16 outputs, and a truncating
store (up to a whole ulp) cannot hide below it.  Headroom is therefore measured on the other terms: ``bound(...,
slack=0.5)`` halves tau and the epilogue's fp32 terms and keeps the output rounding and the flushes of subnormal
results, which are exact worst cases too.

Emulation (``em`` functions).  The kernel's roundings: a k16 MMA sums 16 exact bf16 products and adds them to the fp32
accumulator with round-toward-zero (``moe_reference.mm``); the e4m3 MMA sums 32 products per instruction; the
epilogue's fp32 arithmetic rounds after every operation (the SwiGLU epilogues also flush subnormal results, as fast
math does); the bf16 pack rounds to nearest even.  ``MUTATIONS`` name
plausibly broken kernels the bound must reject.
"""
import math

import torch

from moe_reference import BF16, EXP_ERR, F32, F64, KCHUNK, bf, f32, rz32

U32 = 2.0 ** -24      # fp32 unit roundoff
UBF = 2.0 ** -8       # bf16 round to nearest: at most 2^-8 of the value
FTZ = 2.0 ** -126     # fast math flushes fp32 subnormal results; the sigmoid is 0 where sigmoid(g) < 2^-126
LOG2E = float(torch.tensor(1.4426950408889634, dtype=F32))   # the epilogue's fp32 constant
FP8_K = 32            # products one e4m3 MMA sums
FP8_BLOCK = 128       # e4m3 elements per k-block (one 128-byte swizzle row)

# tau(K): the accumulator's error in units of 2^-24 A.  Each add of a k16 partial sum loses at most one ulp of the
# running sum (truncation), at most 2^-23 A, so a hard bound would be 2 ceil(K / 16).  Over the emulated cases of
# tests/test_gemm_numerics_cpu.py (init and realistic regimes and an all-positive product, K from 8 to 16384) the worst
# emulated error stays under (0.8 ceil(K / 16) + 2) 2^-24 A: 1.9 at K = 8, 4.2 at 56, 44 at 896, 135 at 4104, 315 at
# 11008, 400 at 16384.  tau is 3x that.
TAU_PER_ADD = 2.4
TAU_MMA = 6.0
# e4m3 GEMM: the MMA is modelled as keeping FP8_ACC_BITS significant bits of the largest of (accumulator, products) at
# every k32 instruction (reported for Hopper: DeepSeek-V3 technical report, section 3.3.2), inside one 128-element
# k-block whose partial sum is then added into the fp32 register accumulator.  The emulated error, in units of 2^-24 A,
# is that of a few bad k-blocks and shrinks against A as K grows: worst 3757 at K = 512 (512 x 256 outputs, realistic),
# 1666 at 4096 and 1256 at 11008.  tau8(K) = 6144 max(1, sqrt(2048 / K)) is at least 3x that at each K.  Without the
# promotion the emulated error reaches 24281 at K = 4096 and 37891 at 11008 (256 x 256 outputs, realistic).
FP8_ACC_BITS = 14


def tau8(K):
    return 6144.0 * max(1.0, math.sqrt(2048.0 / K))


def tau(K):
    return TAU_PER_ADD * math.ceil(K / KCHUNK) + TAU_MMA


# -------------------------------------------------------------------------------------------------- operands
def operands(a, b, layout):
    """float64 (A [M, K], B [K, N]) of the kernel's operands in layout nt / nn / tn."""
    a, b = a.to(F64), b.to(F64)
    return (a.t() if layout == "tn" else a), (b.t() if layout == "nt" else b)


def product(A, B):
    """(P = A B, A_abs = |A| |B|) in float64."""
    return A @ B, A.abs() @ B.abs()


def out_bound(ref, d, odt):
    """d (the error before the store) plus one rounding to ``odt`` of the stored magnitude."""
    return d + (UBF if odt == BF16 else U32) * (ref.abs() + d)


def ratio(out, ref, bound):
    """max |out - ref| / bound; inf for a non-finite output or a non-zero error where the bound is 0."""
    err = torch.nan_to_num((out.to(F64) - ref).abs(), nan=math.inf, posinf=math.inf)
    r = torch.where(bound > 0, err / bound.clamp(min=1e-300), torch.where(err == 0, 0.0, math.inf))
    return float(r.max()) if r.numel() else 0.0


# -------------------------------------------------------------------------------------------------- reference
def linear(P, A_abs, K, extra=None, slack=1.0):
    """(pre-store value, its bound) of the store / +residual / accumulate epilogues; ``extra``: the residual or the old C
    (float64), added in fp32."""
    d = slack * tau(K) * U32 * A_abs
    if extra is None:
        return P, d
    ref = P + extra
    return ref, d + slack * U32 * ref.abs()


def rope_cs(table, rows, N, hd, S, rope_cols):
    """(cos, sin) [len(rows), N / 2] of each column pair at the rows' positions (row % S), zero sin / unit cos past
    rope_cols (float64)."""
    pos = (rows % S).long()
    pair = (torch.arange(0, N, 2, device=table.device) % hd) // 2
    cs = table.to(F64)[pos][:, pair]
    c, s = cs[..., 0], cs[..., 1]
    rot = torch.arange(0, N, 2, device=table.device) < rope_cols
    return torch.where(rot, c, 1.0), torch.where(rot, s, 0.0)


def rotate(x, dx, c, s, slack=1.0):
    """The interleaved rotation of the pairs (x_2i, x_2i+1) with its bound: the pair's two input errors through the
    rotation, and two fp32 roundings of |x0 c| + |x1 s| per output."""
    x0, x1, d0, d1 = x[:, 0::2], x[:, 1::2], dx[:, 0::2], dx[:, 1::2]
    r = torch.stack((x0 * c - x1 * s, x0 * s + x1 * c), -1).flatten(1)
    e = torch.stack((d0 * c.abs() + d1 * s.abs() + slack * 2 * U32 * ((x0 * c).abs() + (x1 * s).abs()),
                     d0 * s.abs() + d1 * c.abs() + slack * 2 * U32 * ((x0 * s).abs() + (x1 * c).abs())), -1).flatten(1)
    return r, e


def _sig_err(g, s, slack):
    """Relative error of the epilogue's sigmoid 1 / (1 + exp2f(-log2e g)): the exp (2^-21 for ex2.approx, plus the
    argument's and the constant's roundings, |g| 2^-24 each) enters as (1 - s) of its relative error; 1 + e and the
    reciprocal round once each."""
    return slack * ((1 - s) * (EXP_ERR + 2 * g.abs() * U32) + 2 * U32)


def split_gu(gu, gate_first):
    F = gu.shape[1] // 2
    a, b = gu[:, :F], gu[:, F:]
    return (a, b) if gate_first else (b, a)


def swiglu_act(gu, gate_first=True, slack=1.0):
    """(silu(g) u, its bound before the store) from the kernel's bf16 projection gu [M, 2F] (float64 values)."""
    g, u = split_gu(gu, gate_first)
    s = torch.sigmoid(g)
    act = g * s * u
    # flushes: of g s (then times u), of the result, and of s itself
    return act, act.abs() * (_sig_err(g, s, slack) + slack * 2 * U32) + FTZ * (1 + u.abs() + (g * u).abs())


def swiglu_bwd(ds, dds, gu, gate_first=True, slack=1.0):
    """(d gu [M, 2F], its bound before the store) of dS = ``ds`` (error ``dds``) and the bf16 projection gu."""
    g, u = split_gu(gu, gate_first)
    s = torch.sigmoid(g)
    t = 1 + g * (1 - s)
    es = _sig_err(g, s, slack) * s                          # absolute error of s
    dg = ds * u * s * t
    du = ds * g * s
    # ds's error through the derivative; then s's error through s t (t moves by |g| es) and five fp32 roundings
    e_dg = dds * (u * s * t).abs() + (ds * u).abs() * (es * t.abs() + s * g.abs() * es
                                                      + slack * 5 * U32 * (s * (1 + (g * (1 - s)).abs())))
    e_du = dds * (g * s).abs() + (ds * g).abs() * (es + slack * 2 * U32 * s)
    # flushes: of ds u s (then times t), of the result, and of s itself (dg, du)
    e_dg = e_dg + FTZ * (1 + t.abs() + (ds * u * t).abs())
    e_du = e_du + FTZ * (1 + (ds * g).abs())
    e = torch.cat((e_dg, e_du), 1) if gate_first else torch.cat((e_du, e_dg), 1)
    return (torch.cat((dg, du), 1) if gate_first else torch.cat((du, dg), 1)), e


def fp8_scaled(P, A_abs, K, sa, sb, slack=1.0):
    """(P sa sb, its bound before the store) of the e4m3 GEMM on the dequantised operands (P, A over the e4m3 values)."""
    sc = sa.to(F64)[:, None] * sb.to(F64)[None, :]
    ref = P * sc
    return ref, slack * (tau8(K) * U32 * A_abs * sc + 2 * U32 * ref.abs())


def binade(a):
    """floor(log2 a) of positive float64 values, exactly (frexp, not log2)."""
    return torch.frexp(a)[1].to(torch.int64) - 1


def pow2(e):
    """2^e as float64 for integer e in the normal range, built from its bits: a float64 ``2.0 ** e`` on the GPU is not
    always an exact power of two."""
    return ((e.to(torch.int64) + 1023) << 52).view(F64)


def e4m3_step(a):
    """Spacing of the e4m3 grid at |a| (2^-9 in the subnormal range below 2^-6)."""
    return pow2(binade(a.abs().clamp(min=2.0 ** -9)).clamp(min=-6) - 3)


def e4m3_rne(v):
    """float64 -> the nearest e4m3 (fn) value, ties to even, saturating at 448 (cvt.rn.satfinite)."""
    step = e4m3_step(v)
    return torch.sign(v) * (torch.round(v.abs() / step) * step).clamp(max=448.0)


def quant_rowwise_e4m3(x):
    """(q [R, K] float64 e4m3 values, scale [R] float64 = fp32(amax / 448), 1 for a zero row) of bf16 x: q is the
    round-to-nearest-even e4m3 of the fp32 quotient x / scale, saturating."""
    xf = x.to(F64)
    amax = xf.abs().amax(1)
    sc = torch.where(amax > 0, f32(amax / 448.0), torch.ones_like(amax))
    return e4m3_rne(f32(xf / sc[:, None])), sc


# -------------------------------------------------------------------------------------------------- emulation
MUTATIONS = ("store_truncates", "residual_after_round", "rope_cs_bf16", "bias_after_rotation", "sigmoid_1e-3",
             "swiglu_unrounded", "fp32_accum_through_bf16", "e4m3_acc_14bit")


def trunc_bf16(x):
    """float64 (an fp32 value) -> bf16 by dropping the low 16 bits."""
    i = x.to(F32).view(torch.int32) & ~0xFFFF
    return i.view(F32).to(F64)


def acc_em(A, B):
    """The fp32 accumulator: k16 partial sums added with truncation (``moe_reference.mm``)."""
    acc = torch.zeros(A.shape[0], B.shape[1], dtype=F64, device=A.device)
    for c in range(0, A.shape[1], KCHUNK):
        acc = rz32(acc + A[:, c:c + KCHUNK] @ B[c:c + KCHUNK])
    return acc


def _keep_bits(x, mag, bits):
    """x truncated toward zero to a grid of 2^(e - bits + 1), e the exponent of ``mag``."""
    q = pow2(binade(mag.clamp(min=1e-300)) - bits + 1)
    return torch.trunc(x / q) * q


def acc8_em(A, B, promote=True):
    """The e4m3 accumulator: each k32 MMA adds its 32 exact products and keeps FP8_ACC_BITS bits of the largest addend;
    ``promote``: a fresh partial sum per 128-element k-block, added into the fp32 accumulator with round-to-nearest."""
    M, K = A.shape
    acc = torch.zeros(M, B.shape[1], dtype=F64, device=A.device)
    part = torch.zeros_like(acc)
    for c in range(0, K, FP8_K):
        prods = A[:, c:c + FP8_K, None] * B[None, c:c + FP8_K]
        mag = torch.maximum(part.abs(), prods.abs().amax(1))
        part = _keep_bits(part + prods.sum(1), mag, FP8_ACC_BITS)
        if promote and ((c + FP8_K) % FP8_BLOCK == 0 or c + FP8_K >= K):
            acc, part = f32(acc + part), torch.zeros_like(part)
    return acc if promote else f32(part)


def fz(x):
    """fp32 rounding with fast math's flush of subnormal results."""
    x = f32(x)
    return torch.where(x.abs() < FTZ, torch.zeros_like(x), x)


def sigmoid_em(g, mutation=None):
    """1 / (1 + exp2f(-log2e g)) in fp32, exp2f charged 2^-21 with alternating sign."""
    sign = 1.0 - 2.0 * (torch.arange(g.numel(), device=g.device) % 2).view_as(g)
    e = fz(torch.exp2(fz(-LOG2E * g)) * (1.0 + EXP_ERR * sign))
    s = fz(1.0 / fz(1.0 + e))
    return s * (1 + 1e-3) if mutation == "sigmoid_1e-3" else s


def store_em(v, odt, mutation=None):
    if odt != BF16:
        return f32(v)
    return trunc_bf16(v) if mutation == "store_truncates" else bf(v)


def linear_em(acc, odt, extra=None, mutation=None):
    """store / +residual / accumulate: ``extra`` (the residual or the old C, float64 values of its dtype) added in fp32."""
    if extra is None:
        return store_em(acc, odt, mutation)
    if mutation == "residual_after_round" or (mutation == "fp32_accum_through_bf16" and odt != BF16):
        return store_em(f32(bf(acc) + extra), odt)
    return store_em(f32(acc + extra), odt, mutation)


def rope_em(acc, c, s, bias=None, mutation=None):
    x = acc if bias is None or mutation == "bias_after_rotation" else f32(acc + bias)
    if mutation == "rope_cs_bf16":
        c, s = bf(c), bf(s)
    x0, x1 = x[:, 0::2], x[:, 1::2]
    r = torch.stack((f32(f32(x0 * c) - f32(x1 * s)), f32(f32(x0 * s) + f32(x1 * c))), -1).flatten(1)
    if mutation == "bias_after_rotation" and bias is not None:
        r = f32(r + bias)
    return bf(r)


def swiglu_em(acc, gate_first=True, mutation=None):
    """(gu, act) of the SwiGLU forward epilogue: act from the ROUNDED projection (unless ``swiglu_unrounded``)."""
    gu = bf(acc)
    g, u = split_gu(acc if mutation == "swiglu_unrounded" else gu, gate_first)
    return gu, bf(fz(fz(g * sigmoid_em(g, mutation)) * u))


def swiglu_bwd_em(ds, gu, gate_first=True, mutation=None):
    g, u = split_gu(gu, gate_first)
    s = sigmoid_em(g, mutation)
    dg = fz(fz(fz(ds * u) * s) * fz(1 + fz(g * fz(1 - s))))
    du = fz(fz(ds * g) * s)
    return bf(torch.cat((dg, du), 1) if gate_first else torch.cat((du, dg), 1))


def fp8_em(A, B, sa, sb, mutation=None):
    acc = acc8_em(A, B, promote=mutation != "e4m3_acc_14bit")
    return bf(f32(acc * f32(sa.to(F64)[:, None] * sb.to(F64)[None, :])))


def tile_rel(out, ref, bm=128, bn=256):
    """The former check: max |out - ref| / max |ref| over each bm x bn tile."""
    out, ref = out.to(F64), ref.to(F64)
    M, N = ref.shape
    pm, pn = (-M) % bm, (-N) % bn
    e = torch.nn.functional.pad((out - ref).abs(), (0, pn, 0, pm))
    r = torch.nn.functional.pad(ref.abs(), (0, pn, 0, pm))
    blk = lambda x: x.view((M + pm) // bm, bm, (N + pn) // bn, bn).amax(dim=(1, 3))
    return float((blk(e) / blk(r).clamp(min=1e-6)).max())


# ------------------------------------------------------------------------------------------ one GEMM, by rows
def gemm_ratios(outs, a, b, layout, epi="store", extra=None, rope=None, bias=None, aux=None, gate_first=True,
                unfused=False):
    """Worst ``ratio`` of each output of one GEMM against its float64 reference, computed on the operands' device in
    row chunks.  ``outs``: the kernel's outputs ([c]; [gu, act] for ``swiglu``; [dgu] for ``swiglu_bwd``).
    ``extra``: the residual (any row stride, 0 included) or the C accumulated onto; ``rope`` = (table, S, hd,
    rope_cols); ``bias`` [N] (added before the rotation); ``aux``: gu of the SwiGLU backward.  ``unfused``: the RoPE
    fallback, a bf16 GEMM (the bias as a broadcast residual) and then the stand-alone rotation, two bf16 roundings."""
    A, B = operands(a, b, layout)
    K = A.shape[1]
    M, N = A.shape[0], B.shape[1]
    step = max(8, (1 << 25) // max(N, 1))
    worst = [0.0] * len(outs)
    odt = outs[0].dtype
    for r0 in range(0, M, step):
        r1 = min(M, r0 + step)
        P, Aa = product(A[r0:r1], B)
        if epi == "swiglu":
            ref, d = linear(P, Aa, K)
            gu = outs[0][r0:r1].to(F64)
            act, ad = swiglu_act(gu, gate_first)
            res = [(ref, out_bound(ref, d, BF16)), (act, out_bound(act, ad, BF16))]
        elif epi == "swiglu_bwd":
            ds, dds = linear(P, Aa, K)
            ref, d = swiglu_bwd(ds, dds, aux[r0:r1].to(F64), gate_first)
            res = [(ref, out_bound(ref, d, BF16))]
        elif rope is not None:
            table, S, hd, cols = rope
            x, dx = linear(P, Aa, K, None if bias is None else bias.to(F64)[None])
            if unfused:
                dx = out_bound(x, dx, BF16)
            c, s = rope_cs(table, torch.arange(r0, r1, device=table.device), N, hd, S, cols)
            ref, d = rotate(x, dx, c, s)
            res = [(ref, out_bound(ref, d, BF16))]
        else:
            ref, d = linear(P, Aa, K, None if extra is None else extra[r0:r1].to(F64))
            res = [(ref, out_bound(ref, d, odt))]
        for i, (o, (ref, bnd)) in enumerate(zip(outs, res)):
            worst[i] = max(worst[i], ratio(o[r0:r1], ref, bnd))
        del P, Aa, res
    return worst


def fp8_ratio(y, qa, qb, sa, sb):
    """Worst ``ratio`` of the e4m3 GEMM's output y = (qa qb^T) sa sb against the dequantised float64 reference, by rows
    (qa, qb: the e4m3 bytes as uint8)."""
    A = qa.view(torch.float8_e4m3fn).to(F64)
    B = qb.view(torch.float8_e4m3fn).to(F64).t()
    step = max(8, (1 << 25) // B.shape[1])
    worst = 0.0
    for r0 in range(0, A.shape[0], step):
        r1 = min(A.shape[0], r0 + step)
        P, Aa = product(A[r0:r1], B)
        ref, d = fp8_scaled(P, Aa, A.shape[1], sa[r0:r1], sb)
        worst = max(worst, ratio(y[r0:r1], ref, out_bound(ref, d, BF16)))
    return worst


# ----------------------------------------------------------------------------------------------------- inputs
def operand(rows, cols, role, regime, g, device="cpu"):
    """A bf16 operand [rows, cols] of one role: ``w`` a weight at init std 0.02; ``x`` activations (tokens x features);
    ``dy`` a gradient (tokens x features).  ``realistic``: per-token scales log-uniform over 1e-3 to 1e2, four channels
    of x at 100x, dy at 1/T magnitude with every 16th token's row exactly zero (masked)."""
    if role == "w":
        return (torch.randn(rows, cols, generator=g, device=device) * 0.02).to(BF16)
    x = torch.randn(rows, cols, generator=g, device=device)
    if regime == "realistic":
        lo, hi = math.log(1e-3), math.log(1e2)
        x *= torch.exp(torch.rand(rows, 1, generator=g, device=device) * (hi - lo) + lo)
        if role == "x":
            x[:, torch.randint(0, cols, (4,), generator=g, device=device)] *= 100
        else:
            x /= rows
            x[3::16] = 0
    return x.to(BF16)


def gate_up(rows, F, regime, g, device="cpu"):
    """A bf16 projection [rows, 2F] for the SwiGLU backward: gate and up at unit scale (per-token scales in the
    realistic regime), and every 8th column of both halves near +-30, where the sigmoid saturates."""
    gu = torch.randn(rows, 2 * F, generator=g, device=device) * 2
    if regime == "realistic":
        gu *= torch.exp(torch.rand(rows, 1, generator=g, device=device) * math.log(1e3) - math.log(1e1))
    gu[:, 0::8] = 30 * torch.sign(gu[:, 0::8]) + torch.rand(rows, len(range(0, 2 * F, 8)), generator=g, device=device)
    return gu.to(BF16)
