"""The shared-memory epilogue of the 128 x 256 GEMM tile (``gemm_wide_staged_bf16`` in csrc/gemm_wide_sm90.cu): results
leave through TMA stores and the epilogue operands arrive by TMA loads.  Every GEMM of the headline step at its real epilogue and
output dtype, and the edges of the TMA boxes, must give the same bits as the 128 x 128 tile on the same operands, keep
every element within the float64 bound of tests/gemm_reference.py, and leave every element around C and aux untouched (the stores clip at M and N)."""

import pytest
import torch

import gemm_reference as GR

DEV = "cuda"
T, D, F, H, KVH, HD, V, S = 8192, 2048, 6144, 16, 4, 128, 32000, 4096
QKV = (H + 2 * KVH) * HD
LAYOUT = {"nt": 0, "nn": 1, "tn": 2}
EPI = {"store": 0, "residual": 1, "accumulate": 2, "rope": 3, "swiglu": 5, "swiglu_bwd": 6, "rope_bias": 8}
GUARD = 1234.0   # exact in bf16 and fp32

# (name, layout, M, N, K, epilogue, output dtype, options); the SwiGLU forward's N is 2F, the rows of the fused weight.
# options: ldc / ldr / ld_aux pads (elements past the row), gate_first, rope (hd, H, KVH, S), broadcast (residual)
HEADLINE = [
    ("qkv_fwd", "nt", T, QKV, D, "rope", torch.bfloat16, {}),
    ("o_fwd", "nt", T, D, H * HD, "residual", torch.bfloat16, {}),
    ("gateup_fwd", "nt", T, 2 * F, D, "swiglu", torch.bfloat16, {}),
    ("down_fwd", "nt", T, D, F, "residual", torch.bfloat16, {}),
    ("down_dgrad", "nn", T, F, D, "swiglu_bwd", torch.bfloat16, {}),
    ("down_wgrad", "tn", D, F, T, "store", torch.bfloat16, {}),
    ("gateup_dgrad", "nn", T, D, 2 * F, "store", torch.bfloat16, {}),
    ("gateup_wgrad", "tn", 2 * F, D, T, "store", torch.bfloat16, {}),
    ("o_dgrad", "nn", T, H * HD, D, "store", torch.bfloat16, {}),
    ("o_wgrad", "tn", D, H * HD, T, "store", torch.bfloat16, {}),
    ("qkv_dgrad", "nn", T, D, QKV, "store", torch.bfloat16, {}),
    ("qkv_wgrad", "tn", QKV, D, T, "store", torch.bfloat16, {}),
    ("head_logits", "nt", 4096, V, D, "store", torch.bfloat16, {}),
    ("head_dh", "nn", 4096, D, V, "store", torch.bfloat16, {}),
    ("head_dw", "tn", V, D, 4096, "accumulate", torch.bfloat16, {}),
]
EDGES = [
    ("store_m1000", "nt", 1000, 512, 256, "store", torch.bfloat16, {}),
    ("store_n520", "nn", 512, 520, 256, "store", torch.bfloat16, {}),
    ("store_n776_ldc", "tn", 1000, 776, 192, "store", torch.bfloat16, {"ldc": 40}),
    ("residual_ldr_ne_ldc", "nt", 1000, 776, 264, "residual", torch.bfloat16, {"ldc": 8, "ldr": 24}),
    ("accum_ragged_ldc", "tn", 1000, 520, 200, "accumulate", torch.bfloat16, {"ldc": 16}),
    ("fp32_store", "nn", 640, 1288, 256, "store", torch.float32, {"ldc": 8}),
    ("fp32_accum", "tn", 1000, 520, 200, "accumulate", torch.float32, {"ldc": 4 * 8}),
    # rope_cols = (H + KVH) * hd = 360 ends 8 columns into a 32-column subtile; positions wrap at S = 300
    ("rope_cols_mid_subtile", "nt", 1000, (4 + 2 * 1) * 72, 256, "rope", torch.bfloat16, {"rope": (72, 4, 1, 300)}),
    ("rope_bias_qwen_n1152", "nt", 1000, 1152, 896, "rope_bias", torch.bfloat16, {"rope": (64, 14, 2, 512)}),
    ("rope_bias_qwen_n4608", "nt", 2048, 4608, 512, "rope_bias", torch.bfloat16, {"rope": (128, 28, 4, 1024)}),
    ("swiglu_gate_first", "nt", 1000, 2 * 384, 256, "swiglu", torch.bfloat16, {"ldc": 8, "ld_aux": 16}),
    ("swiglu_up_first", "nt", 512, 2 * 256, 256, "swiglu", torch.bfloat16, {"gate_first": False}),
    ("swiglu_bwd_gate_first", "nn", 1000, 328, 256, "swiglu_bwd", torch.bfloat16, {"ldc": 8, "ld_aux": 24}),
    ("swiglu_bwd_up_first", "nn", 512, 320, 256, "swiglu_bwd", torch.bfloat16, {"gate_first": False}),
]
# operands a TMA map cannot describe: they run on the 128 x 128 tile whatever the tile mode
FALLBACK = [
    ("fp32_residual", "nt", 1000, 776, 264, "residual", torch.float32, {}),
    # row stride 0: the bias of the unfused QKV path rides in the residual epilogue as a broadcast row
    ("broadcast_residual", "nt", 1000, 776, 264, "residual", torch.bfloat16, {"broadcast": True}),
]


@pytest.fixture(scope="module")
def K():
    from fms_fsdp_b200.ops import cuda_kernels as CK
    from fms_fsdp_b200.ops import torch_kernels as TK
    assert CK._C.__file__.endswith("_C.so")
    return CK, TK


def guarded(rows, cols, pad, dtype):
    """A [rows, cols] view with row stride cols + pad into a buffer of GUARD values with 16 guard rows on each side."""
    buf = torch.full((rows + 32, cols + pad), GUARD, dtype=dtype, device=DEV)
    return buf, buf[16:16 + rows, :cols]


def untouched(buf, rows, cols):
    mask = torch.ones_like(buf, dtype=torch.bool)
    mask[16:16 + rows, :cols] = False
    return bool((buf[mask] == GUARD).all())


def make_case(CK, TK, case):
    """(run: () -> [(buffer, view)] of the outputs, keyword arguments of GR.gemm_ratios)."""
    name, layout, M, N, Kd, epi, odt, opt = case
    g = torch.Generator(device=DEV).manual_seed(sum(map(ord, name)))
    rnd = lambda *s, scale=1.0: (torch.randn(*s, generator=g, device=DEV) * scale).bfloat16()
    gate_first = opt.get("gate_first", True)
    if epi == "swiglu":
        Fh = N // 2
        x, w = rnd(M, Kd, scale=0.5), rnd(N, Kd, scale=Kd ** -0.5)

        def run():
            gu = guarded(M, N, opt.get("ldc", 0), torch.bfloat16)
            act = guarded(M, Fh, opt.get("ld_aux", 0), torch.bfloat16)
            CK._C.gemm(x, w, gu[1], 0, EPI[epi], None, aux=act[1], swiglu_F=Fh, gate_first=gate_first)
            return [gu, act]
        return run, dict(a=x, b=w, layout="nt", epi=epi, gate_first=gate_first)
    if epi == "swiglu_bwd":
        dy, w2 = rnd(M, Kd, scale=0.5), rnd(Kd, N, scale=Kd ** -0.5)
        gu_buf, gu = guarded(M, 2 * N, opt.get("ld_aux", 0), torch.bfloat16)
        gu.copy_(rnd(M, 2 * N))

        def run():
            dgu = guarded(M, 2 * N, opt.get("ldc", 0), torch.bfloat16)
            CK._C.gemm(dy, w2, dgu[1], 1, EPI[epi], None, aux=gu, swiglu_F=N, gate_first=gate_first)
            return [dgu]
        return run, dict(a=dy, b=w2, layout="nn", epi=epi, aux=gu, gate_first=gate_first)
    a = rnd(*((M, Kd) if layout != "tn" else (Kd, M)), scale=0.5)
    b = rnd(*((N, Kd) if layout == "nt" else (Kd, N)), scale=Kd ** -0.5)
    kw, r, ref = {}, None, dict(a=a, b=b, layout=layout, epi=epi)
    if epi in ("rope", "rope_bias"):
        hd, h, kvh, Sr = opt.get("rope", (HD, H, KVH, S))
        ang = torch.arange(Sr, device=DEV, dtype=torch.float32)[:, None] * (1e4 ** (-torch.arange(0, hd, 2, device=DEV) / hd))
        table = torch.stack((ang.cos(), ang.sin()), -1).contiguous()
        bias = rnd(N) if epi == "rope_bias" else None
        kw = dict(rope_table=table, rope_S=Sr, rope_hd=hd, rope_cols=(h + kvh) * hd)
        if bias is not None:
            kw["bias"] = bias
        ref.update(rope=(table, Sr, hd, (h + kvh) * hd), bias=bias)
    if epi == "residual":
        if opt.get("broadcast"):
            r = rnd(1, N).expand(M, N)
        else:
            r = guarded(M, N, opt.get("ldr", 0), torch.bfloat16)[1]
            r.copy_(rnd(M, N))
        ref["extra"] = r
    c0 = rnd(M, N).to(odt) if epi == "accumulate" else None
    if c0 is not None:
        ref["extra"] = c0

    def run():
        c = guarded(M, N, opt.get("ldc", 0), odt)
        if c0 is not None:
            c[1].copy_(c0)
        CK._C.gemm(a, b, c[1], LAYOUT[layout], EPI[epi], r, **kw)
        return [c]
    return run, ref


def run_tiles(K, case, modes):
    """{tile mode: the outputs of one run of the case under it} (one launch of our kernel each), and the keyword
    arguments of GR.gemm_ratios."""
    CK, TK = K
    run, ref = make_case(CK, TK, case)
    outs = {}
    for mode in modes:
        CK._C._set_gemm_tile(mode)
        try:
            n0 = CK.launch_count()
            outs[mode] = run()
            torch.cuda.synchronize()
            assert CK.launch_count() == n0 + 1, "one launch of our kernel per GEMM"
        finally:
            CK._C._set_gemm_tile(0)
    return outs, ref


def within_bound(outs, ref, what):
    r = GR.gemm_ratios([v for _, v in outs], **ref)
    assert all(v <= 1.0 for v in r), (what, r)


def check(K, case):
    """Staged epilogue (tile mode 2) and the 128 x 128 tile (1): the same bits, every element outside the outputs
    untouched, and every element within the float64 bound."""
    outs, ref = run_tiles(K, case, (2, 1))
    for (sb, sv), (nb, nv) in zip(outs[2], outs[1]):
        assert untouched(sb, *sv.shape), (case[0], "the staged epilogue wrote outside its output")
        assert torch.equal(sb, nb), (case[0], "staged and 128 x 128 differ", (sv.float() - nv.float()).abs().max().item())
    within_bound(outs[2], ref, case[0])


@pytest.mark.gpu
@pytest.mark.parametrize("case", HEADLINE, ids=[c[0] for c in HEADLINE])
def test_wide_epilogue_headline_shapes(K, case):
    check(K, case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", EDGES, ids=[c[0] for c in EDGES])
def test_wide_epilogue_edges(K, case):
    check(K, case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", FALLBACK, ids=[c[0] for c in FALLBACK])
def test_operands_tma_cannot_describe_run_the_128x128_tile(K, case):
    """Chosen per launch (tile mode 0) or forced to 128 x 256 (2), these GEMMs give the bits of the 128 x 128 tile (1),
    write nothing outside their output and keep every element within the float64 bound."""
    outs, ref = run_tiles(K, case, (0, 2, 1))
    for mode in (0, 2):
        for (b, v), (nb, _) in zip(outs[mode], outs[1]):
            assert untouched(b, *v.shape), (case[0], mode, "wrote outside the output")
            assert torch.equal(b, nb), (case[0], mode, "differs from the 128 x 128 tile")
    within_bound(outs[1], ref, case[0])
