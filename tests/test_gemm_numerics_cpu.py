"""CPU tier of the dense GEMM's element check (tests/gemm_reference.py): the float64 reference equals torch's float64
(autograd for the SwiGLU backward, ``torch_kernels.rope_`` for the rotation, torch's e4m3 conversion for the
quantisation); the CPU emulation of the kernel's roundings passes the element bound with its tau and fp32 terms
halved, at each GPU case's real K (M and N reduced); and plausibly broken kernels fail it.  Each broken kernel is also
run through the former check (max error / max |ref| < 1e-2 over each 128 x 256 tile), and the test prints which of them
that check lets through."""

import pytest
import torch

import gemm_reference as GR
from fms_fsdp_b200.ops import torch_kernels as TK

F64, BF16, F32 = torch.float64, torch.bfloat16, torch.float32
ROPE = (64, 2, 1, 96)      # hd, H, KVH, S of the reduced RoPE cases: rope_cols 192 ends mid-way, positions wrap

# (name, epilogue, layout, M, N, K, output dtype): the GPU cases' epilogues at their real K, M and N reduced
CASES = [
    ("store_k2048", "store", "nt", 128, 256, 2048, BF16),
    ("store_k11008", "store", "nt", 128, 256, 11008, BF16),
    ("store_k8", "store", "nn", 128, 256, 8, BF16),
    ("store_k56", "store", "tn", 128, 256, 56, BF16),
    ("store_k4104", "store", "tn", 128, 256, 4104, BF16),
    ("fp32_store_k8192", "store", "tn", 128, 256, 8192, F32),
    ("residual_k2048", "residual", "nt", 128, 256, 2048, BF16),
    ("residual_broadcast_k896", "broadcast", "nt", 128, 256, 896, BF16),
    ("accum_bf16_k4096", "accumulate", "tn", 128, 256, 4096, BF16),
    ("accum_fp32_k8192", "accumulate", "tn", 128, 256, 8192, F32),
    ("rope_k2048", "rope", "nt", 128, 256, 2048, BF16),
    ("rope_bias_k896", "rope_bias", "nt", 128, 256, 896, BF16),
    ("swiglu_k2048", "swiglu", "nt", 128, 512, 2048, BF16),
    ("swiglu_up_first_k1024", "swiglu_up", "nt", 128, 512, 1024, BF16),
    ("swiglu_bwd_k2048", "swiglu_bwd", "nn", 128, 256, 2048, BF16),
    ("swiglu_bwd_k11008", "swiglu_bwd", "nn", 128, 256, 11008, BF16),
    ("fp8_k512", "fp8", "nt", 128, 128, 512, BF16),
    ("fp8_k4096", "fp8", "nt", 256, 256, 4096, BF16),
    ("fp8_k11008", "fp8", "nt", 256, 256, 11008, BF16),
]
BY_NAME = {c[0]: c for c in CASES}
# each broken kernel and the cases it is run on
BROKEN = {
    "store_truncates": ["store_k2048", "store_k11008"],
    "residual_after_round": ["residual_k2048"],
    "rope_cs_bf16": ["rope_k2048"],
    "bias_after_rotation": ["rope_bias_k896"],
    "sigmoid_1e-3": ["swiglu_k2048", "swiglu_bwd_k2048"],
    "swiglu_unrounded": ["swiglu_k2048"],
    "fp32_accum_through_bf16": ["accum_fp32_k8192"],
    "e4m3_acc_14bit": ["fp8_k4096", "fp8_k11008"],
}


def run(case, regime, mutation=None, slack=1.0, seed=0):
    """[(output name, emulated output, float64 reference, bound)] of one case."""
    name, epi, layout, M, N, K, odt = case
    g = torch.Generator().manual_seed(seed)
    op = lambda r, c, role: GR.operand(r, c, role, regime, g)
    if epi == "fp8":
        qa, sa = GR.quant_rowwise_e4m3(op(M, K, "x"))
        qb, sb = GR.quant_rowwise_e4m3(op(N, K, "w"))
        P, Aa = GR.product(qa, qb.t())
        ref, d = GR.fp8_scaled(P, Aa, K, sa, sb, slack)
        return [("y", GR.fp8_em(qa, qb.t(), sa, sb, mutation), ref, GR.out_bound(ref, d, odt))]
    if layout == "nt":
        a, b = op(M, K, "x"), op(N, K, "w")
    elif layout == "nn":
        a, b = op(M, K, "dy"), op(K, N, "w")
    else:
        a, b = op(K, M, "dy"), op(K, N, "x")
    A, B = GR.operands(a, b, layout)
    P, Aa = GR.product(A, B)
    acc = GR.acc_em(A, B)
    if epi.startswith("swiglu") and epi != "swiglu_bwd":
        gf = epi == "swiglu"
        gu, act = GR.swiglu_em(acc, gf, mutation)
        ref, d = GR.linear(P, Aa, K, slack=slack)
        aref, ad = GR.swiglu_act(gu, gf, slack)
        return [("gu", gu, ref, GR.out_bound(ref, d, odt)), ("act", act, aref, GR.out_bound(aref, ad, odt))]
    if epi == "swiglu_bwd":
        gu = GR.gate_up(M, N, regime, g).to(F64)
        ds, dds = GR.linear(P, Aa, K, slack=slack)
        ref, d = GR.swiglu_bwd(ds, dds, gu, True, slack)
        return [("dgu", GR.swiglu_bwd_em(acc, gu, True, mutation), ref, GR.out_bound(ref, d, odt))]
    if epi in ("rope", "rope_bias"):
        hd, H, KVH, S = ROPE
        table = TK.rope_table(S, hd)
        bias = (torch.randn(N, generator=g) * 0.02).to(BF16).to(F64)[None] if epi == "rope_bias" else None
        c, s = GR.rope_cs(table, torch.arange(M), N, hd, S, (H + KVH) * hd)
        x, dx = GR.linear(P, Aa, K, bias, slack)
        ref, d = GR.rotate(x, dx, c, s, slack)
        return [("qkv", GR.rope_em(acc, c, s, bias, mutation), ref, GR.out_bound(ref, d, odt))]
    extra = None
    if epi == "residual":
        extra = op(M, N, "x").to(F64)
    elif epi == "broadcast":
        extra = (torch.randn(1, N, generator=g) * 0.02).to(BF16).to(F64).expand(M, N)
    elif epi == "accumulate":
        extra = (torch.randn(M, N, generator=g) * P.abs().amax()).to(odt).to(F64)
    ref, d = GR.linear(P, Aa, K, extra, slack)
    return [("c", GR.linear_em(acc, odt, extra, mutation), ref, GR.out_bound(ref, d, odt))]


def test_reference_equals_torch_float64():
    g = torch.Generator().manual_seed(1)
    # SwiGLU backward against float64 autograd of silu(g) u, both orders of the halves
    gu = GR.gate_up(64, 96, "init", g).to(F64)
    ds = torch.randn(64, 96, generator=g, dtype=F64)
    for gf in (True, False):
        x = gu.clone().requires_grad_()
        gg, uu = GR.split_gu(x, gf)
        (torch.nn.functional.silu(gg) * uu * ds).sum().backward()
        ref, _ = GR.swiglu_bwd(ds, torch.zeros_like(ds), gu, gf)
        torch.testing.assert_close(ref, x.grad, rtol=1e-13, atol=1e-300)
        act, _ = GR.swiglu_act(gu, gf)
        torch.testing.assert_close(act, torch.nn.functional.silu(gg.detach()) * uu.detach(), rtol=1e-13, atol=1e-300)
    # the rotation against torch_kernels.rope_ in float64 (positions wrap, the rotated heads end mid-way)
    hd, H, KVH, S = ROPE
    table = TK.rope_table(S, hd)
    M, N = 200, (H + 2 * KVH) * hd
    x = torch.randn(M, N, generator=g, dtype=F64)
    c, s = GR.rope_cs(table, torch.arange(M), N, hd, S, (H + KVH) * hd)
    r, _ = GR.rotate(x, torch.zeros_like(x), c, s)
    torch.testing.assert_close(r, TK.rope_(x.clone(), table.to(F64), S, H, KVH, hd), rtol=1e-13, atol=1e-15)
    # e4m3: round to nearest even and saturation against torch's conversion, over every fp32 exponent in range
    v = torch.cat([torch.randn(100000, generator=g) * 10.0 ** torch.randint(-4, 4, (100000,), generator=g),
                   torch.tensor([0.0, 448.0, 455.9, 464.0, 470.0, 1e6, -1e6, 2.0 ** -9, 2.0 ** -10, 3 * 2.0 ** -11])])
    q = GR.e4m3_rne(v.to(F64))
    assert torch.equal(q, v.clamp(-448, 448).to(torch.float8_e4m3fn).to(F64))
    # row-wise quantisation: the scale is the fp32 quotient amax / 448, a zero row has scale 1 and q = 0
    x = (torch.randn(64, 256, generator=g) * 3).to(BF16)
    x[5] = 0
    q, sc = GR.quant_rowwise_e4m3(x)
    q0, sc0 = TK.quant_rowwise_e4m3(x)
    assert torch.equal(sc, sc0.to(F64)) and torch.equal(q, q0.view(torch.float8_e4m3fn).to(F64))
    assert sc[5] == 1 and not q[5].any()


@pytest.mark.parametrize("regime", ["init", "realistic"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_emulated_kernel_passes_with_headroom(case, regime):
    for out, slack in ((False, 0.5), (True, 1.0)):
        worst = {n: GR.ratio(o, r, b) for n, o, r, b in run(case, regime, slack=slack)}
        if out:
            print(f"MEASURE gemm emulated {case[0]} {regime}: " + " ".join(f"{n} {v:.3f}" for n, v in worst.items())
                  + " x bound")
        assert all(v <= 1.0 for v in worst.values()), (case[0], regime, slack, worst)


def test_broken_kernels_fail():
    rows, slipped = [], []
    for mutation, names in BROKEN.items():
        for name in names:
            for regime in ("init", "realistic"):
                for n, o, r, b in run(BY_NAME[name], regime, mutation):
                    new, old = GR.ratio(o, r, b), GR.tile_rel(o, r)
                    rows.append((mutation, name, regime, n, new, old))
    caught = {}
    for mutation, name, regime, n, new, old in rows:
        caught[mutation] = caught.get(mutation, False) or new > 1.0
        if old < 1e-2:
            slipped.append(f"{mutation} ({name} {regime} {n}: tile_rel {old:.2e}, element check {new:.2f} x bound)")
        print(f"MEASURE gemm broken {mutation} {name} {regime} {n}: element check {new:.2f} x bound, tile_rel {old:.2e}")
    print("passes the former tile_rel < 1e-2 check: " + ("; ".join(slipped) or "none"))
    assert all(caught.values()), {m: c for m, c in caught.items() if not c}
    # every broken kernel fails on every case it is run on, in at least one regime
    for mutation, names in BROKEN.items():
        for name in names:
            assert max(new for m, nm, _, _, new, _ in rows if m == mutation and nm == name) > 1.0, (mutation, name)
