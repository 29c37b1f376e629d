"""GPU tier of the dense GEMM's element check: every output element of the sm_90a GEMM against the float64 reference
and element bound of tests/gemm_reference.py, under the 128 x 128 tile (tile mode 1) and the 128 x 256 tile (mode 2),
and for the cases that go through the Python entry also as the launcher chooses (mode 0); one launch of our kernel per
GEMM.  The 15 GEMMs of the Llama2-1.4B step at T = 8192, shapes of other supported models where they reach edges the
headline does not, per-layout edges of M, N and K, strided and offset outputs, RoPE and SwiGLU edges, gradient
accumulation over four micro-batches, and the e4m3 path (the row-wise quantisation bit for bit, the GEMM up to K =
11008).  Two input regimes: init scale, and realistic (per-token scales over 1e-3 to 1e2, 100x outlier channels,
exact-zero rows of dy, dy at 1/T).  Each case prints its worst ratio as a fraction of the bound ("MEASURE ...").  The
bounds come from the CPU rounding emulation (tests/test_gemm_numerics_cpu.py), not from a GPU run; the float64
references run on the GPU in row chunks.
"""
import time

import pytest
import torch

import gemm_reference as GR

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64, F32, BF16 = torch.float64, torch.float32, torch.bfloat16
LAYOUT = {"nt": 0, "nn": 1, "tn": 2}
EPI = {"store": 0, "residual": 1, "accumulate": 2, "rope": 3, "swiglu": 5, "swiglu_bwd": 6, "rope_bias": 8}
T, D, F, H, KVH, HD, V, S = 8192, 2048, 6144, 16, 4, 128, 32000, 4096
QKV = (H + 2 * KVH) * HD

# (name, layout, M, N, K, epilogue, output dtype, options).  The SwiGLU forward's N is 2F; the backward's N is F.
# options: rope (hd, H, KVH, S); ldc / ldr pads; offset (of the output inside a flat buffer); gate_first;
# broadcast (residual row stride 0); entry (run through the Python entry: also tile mode 0)
HEADLINE = [
    ("qkv_fwd", "nt", T, QKV, D, "rope", BF16, {"rope": (HD, H, KVH, S), "entry": True}),
    ("o_fwd", "nt", T, D, H * HD, "residual", BF16, {"entry": True}),
    ("gateup_fwd", "nt", T, 2 * F, D, "swiglu", BF16, {"entry": True}),
    ("down_fwd", "nt", T, D, F, "residual", BF16, {"entry": True}),
    ("down_dgrad", "nn", T, F, D, "swiglu_bwd", BF16, {"entry": True}),
    ("down_wgrad", "tn", D, F, T, "store", F32, {"entry": True}),
    ("gateup_dgrad", "nn", T, D, 2 * F, "store", BF16, {"entry": True}),
    ("gateup_wgrad", "tn", 2 * F, D, T, "store", F32, {"entry": True}),
    ("o_dgrad", "nn", T, H * HD, D, "store", BF16, {"entry": True}),
    ("o_wgrad", "tn", D, H * HD, T, "store", F32, {"entry": True}),
    ("qkv_dgrad", "nn", T, D, QKV, "store", BF16, {"entry": True}),
    ("qkv_wgrad", "tn", QKV, D, T, "store", F32, {"entry": True}),
    ("head_logits", "nt", 4096, V, D, "store", BF16, {"entry": True}),
    ("head_dh", "nn", 4096, D, V, "store", BF16, {"entry": True}),
    ("head_dw", "tn", V, D, 4096, "accumulate", F32, {"entry": True}),
]
OTHER = [
    # Llama2-7B MLP (D 4096, F 11008): K = 11008 in the down projection, its dgrad with the SwiGLU backward, up wgrad
    ("llama7b_down_fwd", "nt", 2048, 4096, 11008, "residual", BF16, {"entry": True}),
    ("llama7b_down_dgrad", "nn", 2048, 11008, 4096, "swiglu_bwd", BF16, {"entry": True}),
    ("llama7b_up_wgrad", "tn", 2 * 11008, 4096, 2048, "store", F32, {"entry": True}),
    # Qwen2.5-0.5B: D 896, hd 64, H 14 / KVH 2 with q / k / v biases, F 4864, the 151936-word head (last wide tile half empty)
    ("qwen25_qkv_bias", "nt", 4096, (14 + 2 * 2) * 64, 896, "rope_bias", BF16, {"rope": (64, 14, 2, 4096), "entry": True}),
    ("qwen25_gateup", "nt", 4096, 2 * 4864, 896, "swiglu", BF16, {"entry": True}),
    ("qwen25_down_dgrad", "nn", 4096, 4864, 896, "swiglu_bwd", BF16, {"entry": True}),
    ("qwen25_head", "nt", 1024, 151936, 896, "store", BF16, {"entry": True}),
    # Qwen3-0.6B: a plain nt QKV (QK-norm follows) whose q width 2048 differs from D = 1024
    ("qwen3_qkv", "nt", 4096, (16 + 2 * 8) * 128, 1024, "store", BF16, {"entry": True}),
    # Mixtral router: fp32 logits with N = 8; the dgrad with the residual and K = 8; the wgrad with M = 8
    ("mixtral_router_logits", "nt", 4096, 8, 4096, "store", F32, {"entry": True}),
    ("mixtral_router_dgrad", "nn", 4096, 4096, 8, "residual", BF16, {"entry": True}),
    ("mixtral_router_wgrad", "tn", 8, 4096, 4096, "store", F32, {"entry": True}),
]
EDGES = [
    # M in {8, 120, 136, 1000}, N in {8, 136, 264, 520}, K in {8, 56, 72, 4104}: each value on each layout
    ("nt_m8_n520_k4104", "nt", 8, 520, 4104, "store", BF16, {"entry": True}),
    ("nt_m120_n8_k72", "nt", 120, 8, 72, "store", F32, {"entry": True}),
    ("nt_m136_n264_k8", "nt", 136, 264, 8, "residual", BF16, {"entry": True}),
    ("nt_m1000_n136_k56", "nt", 1000, 136, 56, "store", BF16, {"entry": True}),
    ("nn_m8_n264_k56", "nn", 8, 264, 56, "store", BF16, {"entry": True}),
    ("nn_m120_n520_k8", "nn", 120, 520, 8, "store", F32, {"entry": True}),
    ("nn_m136_n136_k4104", "nn", 136, 136, 4104, "residual", BF16, {"entry": True}),
    ("nn_m1000_n8_k72", "nn", 1000, 8, 72, "store", BF16, {"entry": True}),
    ("tn_m8_n136_k72", "tn", 8, 136, 72, "accumulate", F32, {"entry": True}),
    ("tn_m120_n264_k4104", "tn", 120, 264, 4104, "store", BF16, {"entry": True}),
    ("tn_m136_n8_k56", "tn", 136, 8, 56, "accumulate", BF16, {"entry": True}),
    ("tn_m1000_n520_k8", "tn", 1000, 520, 8, "store", F32, {"entry": True}),
    # strided outputs and residuals, and an output bound at a 64-element offset of a flat buffer (a gradient slot)
    ("residual_ldc_ldr", "nt", 1000, 776, 264, "residual", BF16, {"ldc": 8, "ldr": 24}),
    ("store_ldc_fp32", "nn", 640, 1288, 256, "store", F32, {"ldc": 8}),
    ("accum_offset64_fp32", "tn", 1000, 520, 200, "accumulate", F32, {"offset": 64}),
    ("accum_offset64_bf16", "tn", 776, 264, 1000, "accumulate", BF16, {"offset": 64}),
    ("broadcast_residual", "nt", 1000, 776, 264, "residual", BF16, {"broadcast": True}),
    # RoPE: positions wrap (M % S != 0) and rope_cols = 360 ends 8 columns into a 32-column subtile
    ("rope_wrap_mid_subtile", "nt", 1000, (4 + 2 * 1) * 72, 256, "rope", BF16, {"rope": (72, 4, 1, 300)}),
    ("rope_bias_wrap", "nt", 1000, (14 + 2 * 2) * 64, 896, "rope_bias", BF16, {"rope": (64, 14, 2, 384)}),
    # the unfused RoPE path of M < 256: GEMM (bias as a broadcast residual), then the rotation kernel
    ("rope_bias_unfused_m120", "nt", 120, (4 + 2 * 2) * 64, 256, "rope_bias", BF16, {"rope": (64, 4, 2, 100), "entry": True}),
    # SwiGLU both ways at F = 320 (the wide tile takes F % 128 == 0 only) and 384, saturated gates in the backward
    ("swiglu_f320_gate_first", "nt", 1000, 2 * 320, 256, "swiglu", BF16, {"ldc": 8, "ld_aux": 16}),
    ("swiglu_f384_up_first", "nt", 512, 2 * 384, 256, "swiglu", BF16, {"gate_first": False}),
    ("swiglu_bwd_f320_up_first", "nn", 1000, 320, 256, "swiglu_bwd", BF16, {"gate_first": False}),
    ("swiglu_bwd_f384_gate_first", "nn", 512, 384, 4104, "swiglu_bwd", BF16, {"ldc": 8, "ld_aux": 24}),
]
FP8_SHAPES = [(1024, 768, 512), (8192, 12288, 4096), (8192, 22016, 4096), (8192, 4096, 11008)]


@pytest.fixture(scope="module")
def CK():
    from fms_fsdp_b200.ops import cuda_kernels as CK
    assert CK._C.__file__.endswith("_C.so")
    return CK


def strided(rows, cols, pad, dtype, offset=0):
    """A [rows, cols] view with row stride cols + pad, ``offset`` elements into a flat buffer."""
    buf = torch.full((offset + rows * (cols + pad),), 7.0, dtype=dtype, device=DEV)
    return buf[offset:].view(rows, cols + pad)[:, :cols]


def make(CK, case, regime):
    """(run(): the kernel's outputs, keyword arguments of GR.gemm_ratios)."""
    name, layout, M, N, Kd, epi, odt, opt = case
    g = torch.Generator(device=DEV).manual_seed(sum(map(ord, name)))
    op = lambda r, c, role: GR.operand(r, c, role, regime, g, DEV)
    gf = opt.get("gate_first", True)
    entry = opt.get("entry", False)
    if layout == "nt":
        a, b = op(M, Kd, "x"), op(N, Kd, "w")
    elif layout == "nn":
        a, b = op(M, Kd, "dy"), op(Kd, N, "w")
    else:
        a, b = op(Kd, M, "dy"), op(Kd, N, "x")
    ref = dict(a=a, b=b, layout=layout, epi=epi, gate_first=gf)
    if epi == "swiglu":
        Fh = N // 2
        if entry:
            return (lambda: list(CK.gated_up_fwd(a, b, gf))), ref

        def run():
            gu, act = strided(M, N, opt.get("ldc", 0), BF16), strided(M, Fh, opt.get("ld_aux", 0), BF16)
            CK._C.gemm(a, b, gu, 0, EPI[epi], None, aux=act, swiglu_F=Fh, gate_first=gf)
            return [gu, act]
        return run, ref
    if epi == "swiglu_bwd":
        gu = strided(M, 2 * N, opt.get("ld_aux", 0), BF16)
        gu.copy_(GR.gate_up(M, N, regime, g, DEV))
        ref["aux"] = gu
        if entry:
            return (lambda: [CK.gated_down_bwd(a, b, gu, gf)]), ref

        def run():
            dgu = strided(M, 2 * N, opt.get("ldc", 0), BF16)
            CK._C.gemm(a, b, dgu, 1, EPI[epi], None, aux=gu, swiglu_F=N, gate_first=gf)
            return [dgu]
        return run, ref
    if epi in ("rope", "rope_bias"):
        from fms_fsdp_b200.ops import torch_kernels as TK
        hd, h, kvh, Sr = opt["rope"]
        table = TK.rope_table(Sr, hd, theta=1e6 if epi == "rope_bias" else 1e4, device=DEV)
        bias = (torch.randn(N, generator=g, device=DEV) * 0.02).to(BF16) if epi == "rope_bias" else None
        ref.update(rope=(table, Sr, hd, (h + kvh) * hd), bias=bias, unfused=M < 256)
        if entry:
            return (lambda: [CK.gemm(a, b, "nt", rope=(table, Sr, hd, h, kvh), bias=bias)]), ref
        kw = dict(rope_table=table, rope_S=Sr, rope_hd=hd, rope_cols=(h + kvh) * hd, bias=bias)

        def run():
            c = strided(M, N, opt.get("ldc", 0), BF16)
            CK._C.gemm(a, b, c, 0, EPI[epi], None, **kw)
            return [c]
        return run, ref
    r = c0 = None
    if epi == "residual":
        if opt.get("broadcast"):
            r = (torch.randn(1, N, generator=g, device=DEV) * 0.02).to(BF16).expand(M, N)
        else:
            r = strided(M, N, opt.get("ldr", 0), BF16)
            r.copy_(op(M, N, "x"))
        ref["extra"] = r
    if epi == "accumulate":
        c0 = (torch.randn(M, N, generator=g, device=DEV) * (0.01 if regime == "init" else 1e-4)).to(odt)
        ref["extra"] = c0

    def run():
        c = strided(M, N, opt.get("ldc", 0), odt, opt.get("offset", 0))
        if c0 is not None:
            c.copy_(c0)
        if entry:
            CK.gemm(a, b, layout, out=c, accumulate=c0 is not None, residual=r)
        else:
            CK._C.gemm(a, b, c, LAYOUT[layout], EPI[epi], r)
        return [c]
    return run, ref


def check(CK, case, regime):
    name, opt = case[0], case[7]
    t0 = time.time()
    run, ref = make(CK, case, regime)
    launches = 2 if ref.get("unfused") else 1         # the unfused RoPE: GEMM, then the rotation kernel
    worst = {}
    for mode in ((0, 1, 2) if opt.get("entry") else (1, 2)):
        CK._C._set_gemm_tile(mode)
        try:
            n0 = CK.launch_count()
            outs = run()
            torch.cuda.synchronize()
            assert CK.launch_count() == n0 + launches, (name, mode, "launches of our kernels")
        finally:
            CK._C._set_gemm_tile(0)
        worst[mode] = GR.gemm_ratios(outs, **ref)
        del outs
    print(f"MEASURE gemm {name} {regime}: " + " ".join(
        f"tile{m} " + "/".join(f"{v:.3f}" for v in w) for m, w in worst.items()) + f" x bound; {time.time() - t0:.1f} s")
    bad = {m: w for m, w in worst.items() if not all(v <= 1.0 for v in w)}
    assert not bad, (name, regime, bad)


@pytest.mark.parametrize("regime", ["init", "realistic"])
@pytest.mark.parametrize("case", HEADLINE, ids=[c[0] for c in HEADLINE])
def test_headline_step(CK, case, regime):
    check(CK, case, regime)


@pytest.mark.parametrize("regime", ["init", "realistic"])
@pytest.mark.parametrize("case", OTHER, ids=[c[0] for c in OTHER])
def test_other_model_shapes(CK, case, regime):
    check(CK, case, regime)


@pytest.mark.parametrize("regime", ["init", "realistic"])
@pytest.mark.parametrize("case", EDGES, ids=[c[0] for c in EDGES])
def test_edges(CK, case, regime):
    check(CK, case, regime)


@pytest.mark.parametrize("odt", [F32, BF16], ids=["fp32_slot", "bf16_slot"])
@pytest.mark.parametrize("tile", [0, 1, 2], ids=["auto", "narrow", "wide"])
def test_gradient_accumulation(CK, odt, tile):
    """A wgrad (dW = dy^T x, the o projection's shape at 2048 tokens per micro-batch) accumulated over four
    micro-batches into one slot, against the float64 sum: each step adds one accumulator error and one rounding to the
    slot's type of the running sum."""
    M, N, Tm = D, H * HD, 2048
    g = torch.Generator(device=DEV).manual_seed(5)
    slot = torch.zeros(M, N, dtype=odt, device=DEV)
    ref = torch.zeros(M, N, dtype=F64, device=DEV)
    bound = torch.zeros_like(ref)
    CK._C._set_gemm_tile(tile)
    try:
        for _ in range(4):
            dy, x = GR.operand(Tm, M, "dy", "realistic", g, DEV), GR.operand(Tm, N, "x", "realistic", g, DEV)
            n0 = CK.launch_count()
            CK.gemm(dy, x, "tn", out=slot, accumulate=True)
            torch.cuda.synchronize()
            assert CK.launch_count() == n0 + 1
            P, Aa = GR.product(*GR.operands(dy, x, "tn"))
            ref, d = GR.linear(P, Aa, Tm, ref)
            bound = GR.out_bound(ref, d + bound, odt)
    finally:
        CK._C._set_gemm_tile(0)
    r = GR.ratio(slot, ref, bound)
    print(f"MEASURE gemm grad_accum {odt} tile {tile}: {r:.3f} x bound")
    assert r <= 1.0


def test_quant_rowwise_e4m3_exact(CK):
    """scale = fp32(amax / 448) bit for bit; q = the round-to-nearest-even e4m3 of the fp32 quotient x / scale,
    saturating, bit for bit; a zero row gives scale 1 and q = 0."""
    g = torch.Generator(device=DEV).manual_seed(6)
    for rows, K, regime in ((1024, 4096, "init"), (4096, 11008, "realistic"), (333, 528, "realistic")):
        x = GR.operand(rows, K, "x", regime, g, DEV)
        x[7] = 0
        q, sc = CK.quant_rowwise_e4m3(x)
        q0, sc0 = GR.quant_rowwise_e4m3(x)
        assert torch.equal(sc.to(F64), sc0), ("scale", (sc.to(F64) - sc0).abs().max().item())
        bad = (q.view(torch.float8_e4m3fn).to(F64) != q0).sum().item()
        assert bad == 0, ("q", rows, K, regime, bad)
        assert sc[7] == 1 and not q[7].any()


@pytest.mark.parametrize("shape", FP8_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_gemm_fp8(CK, shape):
    M, N, Kd = shape
    for regime in ("init", "realistic"):
        g = torch.Generator(device=DEV).manual_seed(Kd)
        x, w = GR.operand(M, Kd, "x", regime, g, DEV), GR.operand(N, Kd, "w", regime, g, DEV)
        xq, sx = CK.quant_rowwise_e4m3(x)
        wq, sw = CK.quant_rowwise_e4m3(w)
        n0 = CK.launch_count()
        y = CK.gemm_fp8(xq, wq, sx, sw)
        torch.cuda.synchronize()
        assert CK.launch_count() == n0 + 1
        r = GR.fp8_ratio(y, xq, wq, sx, sw)
        print(f"MEASURE gemm fp8 {M}x{N}x{Kd} {regime}: {r:.3f} x bound")
        assert r <= 1.0, (shape, regime, r)


# ------------------------------------------------------------------------------------ dense fp32 outputs
# (name, layout, M, N, K, accumulate): fp32-output GEMMs at the wide-tile test shapes and the router-logit GEMM of
# Qwen3-30B-A3B, against the float64 product
DENSE_FP32 = [
    ("fp32_store", "nn", 640, 1288, 256, False),
    ("fp32_accum", "tn", 1000, 520, 200, True),
    ("head_dw_fp32", "tn", 32000, 2048, 4096, True),
    ("router_logits", "nt", 8192, 128, 2048, False),
]


@pytest.mark.parametrize("case", DENSE_FP32, ids=lambda c: c[0])
@pytest.mark.parametrize("tile", [0, 1, 2], ids=["auto", "narrow", "wide"])
def test_dense_fp32_outputs(CK, case, tile):
    name, layout, M, N, Kd, acc = case
    g = torch.Generator(device=DEV).manual_seed(9)
    a = torch.randn(*((M, Kd) if layout != "tn" else (Kd, M)), generator=g, device=DEV).to(BF16)
    b = torch.randn(*((N, Kd) if layout == "nt" else (Kd, N)), generator=g, device=DEV).to(BF16)
    base = torch.randn(M, N, generator=g, device=DEV)
    out = base.clone() if acc else torch.empty(M, N, device=DEV)
    CK._C._set_gemm_tile(tile)
    try:
        CK.gemm(a, b, layout, out=out, accumulate=acc)
    finally:
        CK._C._set_gemm_tile(0)
    r = GR.gemm_ratios([out], a, b, layout, "accumulate" if acc else "store", extra=base if acc else None)[0]
    print(f"MEASURE gemm dense fp32 {name} tile {tile}: {r:.3f} x bound")
    assert r <= 1.0
