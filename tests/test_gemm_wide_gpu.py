"""The 128 x 256 GEMM tile (``gemm_wide_bf16`` in csrc/gemm_sm90.cu): every GEMM of the Llama2-1.4B headline step at its
real shape, layout, epilogue and output dtype, and the edge cases of the tile, against the fp32 oracle and against the
128 x 128 tile on the same operands.  Both tiles sum each output element over k in the same order (64-wide k-blocks,
k16 MMAs in sequence), so they agree to the last bit."""
import contextlib
import os
import re
import shutil
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"
T, D, F, H, KVH, HD, V, S = 8192, 2048, 6144, 16, 4, 128, 32000, 4096
QKV = (H + 2 * KVH) * HD

# (name, layout, M, N, K, epilogue, output dtype); the SwiGLU forward's N is 2F, the rows of the fused weight
HEADLINE = [
    ("qkv_fwd", "nt", T, QKV, D, "rope", torch.bfloat16),
    ("o_fwd", "nt", T, D, H * HD, "residual", torch.bfloat16),
    ("gateup_fwd", "nt", T, 2 * F, D, "swiglu", torch.bfloat16),
    ("down_fwd", "nt", T, D, F, "residual", torch.bfloat16),
    ("down_dgrad", "nn", T, F, D, "swiglu_bwd", torch.bfloat16),
    ("down_wgrad", "tn", D, F, T, "store", torch.bfloat16),
    ("gateup_dgrad", "nn", T, D, 2 * F, "store", torch.bfloat16),
    ("gateup_wgrad", "tn", 2 * F, D, T, "store", torch.bfloat16),
    ("o_dgrad", "nn", T, H * HD, D, "store", torch.bfloat16),
    ("o_wgrad", "tn", D, H * HD, T, "store", torch.bfloat16),
    ("qkv_dgrad", "nn", T, D, QKV, "store", torch.bfloat16),
    ("qkv_wgrad", "tn", QKV, D, T, "store", torch.bfloat16),
    ("head_logits", "nt", 4096, V, D, "store", torch.bfloat16),
    ("head_dh", "nn", 4096, D, V, "store", torch.bfloat16),
    ("head_dw", "tn", V, D, 4096, "accumulate", torch.bfloat16),
    ("head_dw_fp32", "tn", V, D, 4096, "accumulate", torch.float32),   # gradient accumulation into an fp32 buffer
]
EDGES = [
    ("m384_odd_mtiles", "nt", 384, 1024, 256, "store", torch.bfloat16),
    ("m1000_ragged", "nn", 1000, 768, 512, "store", torch.bfloat16),
    ("n520_ragged", "tn", 512, 520, 384, "store", torch.bfloat16),
    ("k72_tail", "nt", 768, 512, 72, "store", torch.bfloat16),
    ("ragged_all", "tn", 1000, 520, 200, "accumulate", torch.float32),
    ("fp32_store", "nn", 640, 1280, 256, "store", torch.float32),
    ("residual_ragged", "nt", 1000, 776, 264, "residual", torch.bfloat16),
    ("rope_small", "nt", 512, (4 + 2 * 2) * 64, 256, "rope", torch.bfloat16),
    ("swiglu_f384", "nt", 512, 2 * 384, 256, "swiglu", torch.bfloat16),
    ("swiglu_f320_falls_back", "nt", 512, 2 * 320, 256, "swiglu", torch.bfloat16),   # F % 128 != 0: 128 x 128 tile
    ("swiglu_bwd_f320", "nn", 512, 320, 256, "swiglu_bwd", torch.bfloat16),
]


@pytest.fixture(scope="module")
def K():
    from fms_fsdp_b200.ops import cuda_kernels as CK
    from fms_fsdp_b200.ops import torch_kernels as TK
    assert CK._C.__file__.endswith("_C.so")
    return CK, TK


@contextlib.contextmanager
def tile(CK, mode):
    CK._C._set_gemm_tile({"narrow": 1, "wide": 2}[mode])
    try:
        yield
    finally:
        CK._C._set_gemm_tile(0)


def tile_rel(out, ref, bm=128, bn=256):
    """Largest per-tile relative error: max |out - ref| / max |ref| over each bm x bn block."""
    out, ref = out.float(), ref.float()
    M, N = ref.shape
    pm, pn = (-M) % bm, (-N) % bn
    e = torch.nn.functional.pad((out - ref).abs(), (0, pn, 0, pm))
    r = torch.nn.functional.pad(ref.abs(), (0, pn, 0, pm))
    blk = lambda x: x.view((M + pm) // bm, bm, (N + pn) // bn, bn).amax(dim=(1, 3))
    return (blk(e) / blk(r).clamp(min=1e-6)).max().item()


def make_case(CK, TK, layout, M, N, Kd, epi, odt, seed):
    """(run: () -> outputs, oracle outputs in fp32).  run() returns a tuple of the tensors the GEMM wrote."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    rnd = lambda *s, scale=1.0: (torch.randn(*s, generator=g, device=DEV) * scale).bfloat16()
    if epi == "swiglu":
        Fh = N // 2
        x, w = rnd(M, Kd, scale=0.5), rnd(N, Kd, scale=Kd ** -0.5)
        gu0 = x.float() @ w.float().t()

        def run():   # the launcher itself, so that an F the wide tile cannot take reaches it
            gu = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
            act = torch.empty(M, Fh, dtype=torch.bfloat16, device=DEV)
            CK._C.set_gemm_swiglu(act, Fh, True)
            CK._C.gemm(x, w, gu, 0, 5, None)
            return gu, act
        return run, (gu0, None)
    if epi == "swiglu_bwd":
        dy, w2, gu = rnd(M, Kd, scale=0.5), rnd(Kd, N, scale=Kd ** -0.5), rnd(M, 2 * N)
        ref = TK.swiglu_bwd(dy.float() @ w2.float(), gu.float())
        return (lambda: (CK.gated_down_bwd(dy, w2, gu),)), (ref,)
    a = rnd(*((M, Kd) if layout != "tn" else (Kd, M)), scale=0.5)
    b = rnd(*((N, Kd) if layout == "nt" else (Kd, N)), scale=Kd ** -0.5)
    ref = TK.gemm(a.float(), b.float(), layout)
    if epi == "rope":
        hd, kvh = (HD, KVH) if N == QKV else (64, 2)
        h = N // hd - 2 * kvh
        ang = torch.arange(M, device=DEV, dtype=torch.float32)[:, None] * (1e4 ** (-torch.arange(0, hd, 2, device=DEV) / hd))
        table = torch.stack((ang.cos(), ang.sin()), -1).contiguous()
        Sr = min(M, S)
        ref = TK.gemm(a.float(), b.float(), layout, rope=(table, Sr, hd, h, kvh))
        return (lambda: (CK.gemm(a, b, layout, rope=(table, Sr, hd, h, kvh)),)), (ref,)
    if epi == "residual":
        r = rnd(M, N)
        return (lambda: (CK.gemm(a, b, layout, residual=r),)), (ref + r.float(),)
    if epi == "accumulate":
        c0 = rnd(M, N).to(odt)

        def run():
            c = c0.clone()
            CK.gemm(a, b, layout, out=c, accumulate=True)
            return (c,)
        return run, (ref + c0.float(),)
    return (lambda: (CK.gemm(a, b, layout, out_dtype=odt),)), (ref,)


def check(K, case):
    CK, TK = K
    name, layout, M, N, Kd, epi, odt = case
    run, refs = make_case(CK, TK, layout, M, N, Kd, epi, odt, seed=sum(map(ord, name)))
    outs = {}
    for mode in ("wide", "narrow"):
        with tile(CK, mode):
            n0 = CK.launch_count()
            outs[mode] = run()
            torch.cuda.synchronize()
            assert CK.launch_count() == n0 + 1, "one launch of our kernel per GEMM"
    if epi == "swiglu":   # the activation of the bf16-rounded projection, as both kernels compute it
        refs = (refs[0], TK.swiglu_fwd(outs["narrow"][0].float()))
    worst = 0.0
    for w, n, ref in zip(outs["wide"], outs["narrow"], refs):
        assert tile_rel(w, ref) < 1e-2, name
        d = (w.float() - n.float()).abs()
        worst = max(worst, d.max().item())
        # the same per-element k order: equal up to the last bit of the output type
        ulp = 2.0 ** -7 if w.dtype == torch.bfloat16 else 2.0 ** -20
        assert bool((d <= n.float().abs() * ulp + 1e-30).all()), (name, d.max().item())
    print(f"{name}: max |wide - narrow| = {worst:.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("case", HEADLINE, ids=[c[0] for c in HEADLINE])
def test_wide_tile_headline_shapes(K, case):
    check(K, case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", EDGES, ids=[c[0] for c in EDGES])
def test_wide_tile_edges(K, case):
    check(K, case)


def test_wide_kernel_sass():
    """The wide instantiations issue m64n256k16 warpgroup MMAs, load operands by TMA and never touch local memory."""
    so = os.path.join(ROOT, "fms_fsdp_b200", "_C.so")
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(so) or not os.path.exists(exe):
        pytest.skip("needs the built extension and cuobjdump")
    out = subprocess.run([exe, "-sass", so], capture_output=True, text=True, timeout=600).stdout
    per, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1) if "gemm_wide_bf16" in m.group(1) else None
            if name:
                per[name] = []
        elif name and "/*" in line:
            per[name].append(line)
    assert len(per) >= 9, sorted(per)
    for k, lines in per.items():
        body = "\n".join(lines)
        assert re.search(r"HGMMA\.64x256x16\.F32\.BF16", body), k
        assert not re.search(r"HGMMA\.64x128x16", body), k
        assert re.search(r"UTMALDG\.2D", body), k
        assert not re.search(r"\b(LDL|STL)\b", body), k
