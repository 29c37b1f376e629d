"""GPU tier: document-masked flash attention (``seg`` table) on the sm_90a kernels against the fp32 oracle, against the
unmasked kernel on single documents and on documents run one at a time, and the engine on the fused kernels against the
ATen kernel path."""
import pytest
import torch

from fms_fsdp_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"
SEP = 1


@pytest.fixture(scope="module")
def K():
    from fms_fsdp_b200.ops import cuda_kernels as CK
    from fms_fsdp_b200.ops import torch_kernels as TK
    assert CK._C.__file__.endswith("_C.so")
    return CK, TK


def rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).abs().max() / b.abs().max().clamp(min=1e-6)).item()


def _seg(seps_per_row, S):
    """segment table of rows whose separators sit at the given positions"""
    tok = torch.zeros(len(seps_per_row), S, dtype=torch.long)
    for r, seps in enumerate(seps_per_row):
        for p in seps:
            if p < S:
                tok[r, p] = SEP
    return ops.document_segments(tok.to(DEV), SEP)


# row 0: documents ending on 64- and 128-row tile edges and a one-token document (127, 128);
# row 1: boundaries in the middle of tiles, a one-token document (40, 41) and one at the row end
LAYOUTS = {
    "edges": [[63, 127, 128, 191, 255, 383], [40, 41, 200, 300, 511]],
    "single": [[], []],
    "first_token": [[0], [0, 1, 2]],
}


def _inputs(B, S, H, KVH, hd, seed=1):
    g = torch.Generator(device=DEV).manual_seed(seed)
    qkv = torch.randn(B * S, (H + 2 * KVH) * hd, device=DEV, generator=g).bfloat16()
    do = torch.randn(B * S, H * hd, device=DEV, generator=g).bfloat16()
    return qkv, do


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("cfg", [(128, 4, 4, 128), (384, 4, 2, 128), (512, 2, 2, 64), (384, 4, 1, 64), (512, 4, 2, 128)])
def test_doc_attention_matches_oracle(K, cfg, layout):
    CK, TK = K
    S, H, KVH, hd = cfg
    B = 2
    seg = _seg(LAYOUTS[layout], S)
    qkv, do = _inputs(B, S, H, KVH, hd)
    sc = hd ** -0.5
    n0, f0 = CK.launch_count(), CK.fallback_count()
    o1, l1 = CK.attn_fwd(qkv, B, S, H, KVH, hd, sc, seg=seg)
    g1 = CK.attn_bwd(do, qkv, o1, l1, B, S, H, KVH, hd, sc, seg=seg)
    assert CK.launch_count() == n0 + 4 and CK.fallback_count() == f0    # our forward + delta/dKdV/dQ ran
    o0, l0 = TK.attn_fwd(qkv.float(), B, S, H, KVH, hd, sc, seg=seg)
    g0 = TK.attn_bwd(do.float(), qkv.float(), o0, l0, B, S, H, KVH, hd, sc, seg=seg)
    assert l1.isfinite().all() and o1.isfinite().all() and g1.isfinite().all()
    assert rel(o1, o0) < 1e-2 and rel(l1, l0) < 1e-4
    assert rel(g1, g0) < 1.5e-2


@pytest.mark.parametrize("cfg", [(2, 512, 4, 2, 128), (1, 384, 2, 2, 64), (2, 200, 4, 1, 128)])
def test_single_document_table_is_bitwise_the_causal_kernel(K, cfg):
    CK, _ = K
    B, S, H, KVH, hd = cfg
    seg = _seg([[]] * B, S)
    qkv, do = _inputs(B, S, H, KVH, hd, seed=2)
    sc = hd ** -0.5
    o1, l1 = CK.attn_fwd(qkv, B, S, H, KVH, hd, sc, seg=seg)
    o0, l0 = CK.attn_fwd(qkv, B, S, H, KVH, hd, sc)
    assert torch.equal(o1, o0) and torch.equal(l1, l0)
    tab = torch.randn(S, hd // 2, 2, device=DEV)          # inverse-RoPE epilogue path as well
    for rope in (None, tab):
        g1 = CK.attn_bwd(do, qkv, o0, l0, B, S, H, KVH, hd, sc, rope_table=rope, seg=seg)
        g0 = CK.attn_bwd(do, qkv, o0, l0, B, S, H, KVH, hd, sc, rope_table=rope)
        assert torch.equal(g1, g0)


@pytest.mark.parametrize("H,KVH,hd", [(4, 2, 128), (2, 2, 64)])
def test_packed_row_equals_documents_run_separately(K, H, KVH, hd):
    CK, _ = K
    lens = [100, 1, 27, 128, 64, 192]                     # sums to 512
    S = sum(lens)
    seps = list(torch.tensor(lens).cumsum(0)[:-1] - 1)
    seg = _seg([[int(p) for p in seps]], S)
    qkv, do = _inputs(1, S, H, KVH, hd, seed=3)
    sc = hd ** -0.5
    o, l = CK.attn_fwd(qkv, 1, S, H, KVH, hd, sc, seg=seg)
    g = CK.attn_bwd(do, qkv, o, l, 1, S, H, KVH, hd, sc, seg=seg)
    p0 = 0
    for n in lens:
        q_d, do_d = qkv[p0:p0 + n].contiguous(), do[p0:p0 + n].contiguous()
        od, ld = CK.attn_fwd(q_d, 1, n, H, KVH, hd, sc)
        gd = CK.attn_bwd(do_d, q_d, od, ld, 1, n, H, KVH, hd, sc)
        assert rel(o[p0:p0 + n], od) < 1e-2, (p0, n)
        assert rel(l[:, :, p0:p0 + n], ld) < 1e-4, (p0, n)
        assert rel(g[p0:p0 + n], gd) < 1.5e-2, (p0, n)
        p0 += n


def test_headline_length_random_documents(K):
    CK, TK = K
    B, S, H, KVH, hd = 1, 4096, 8, 2, 128
    g = torch.Generator().manual_seed(7)
    lens = []
    while sum(lens) < S:
        lens.append(int(torch.randint(1, 1200, (1,), generator=g)))
    seps = torch.tensor(lens).cumsum(0) - 1
    seg = _seg([[int(p) for p in seps if p < S - 1]], S)
    qkv, do = _inputs(B, S, H, KVH, hd, seed=4)
    sc = hd ** -0.5
    o1, l1 = CK.attn_fwd(qkv, B, S, H, KVH, hd, sc, seg=seg)
    g1 = CK.attn_bwd(do, qkv, o1, l1, B, S, H, KVH, hd, sc, seg=seg)
    o0, l0 = TK.attn_fwd(qkv.float(), B, S, H, KVH, hd, sc, seg=seg)
    g0 = TK.attn_bwd(do.float(), qkv.float(), o0, l0, B, S, H, KVH, hd, sc, seg=seg)
    assert rel(o1, o0) < 1e-2 and rel(l1, l0) < 1e-4 and rel(g1, g0) < 1.5e-2


def test_bad_segment_tables_are_rejected(K):
    CK, _ = K
    B, S, H, KVH, hd = 1, 128, 2, 2, 64
    qkv, _ = _inputs(B, S, H, KVH, hd)
    seg = _seg([[10]], S)
    for bad in (seg.long(), seg[:, :64].contiguous(), seg.cpu(), seg.t().contiguous().t()):
        with pytest.raises(RuntimeError, match="seg"):
            CK._C.attn_fwd(qkv, B, S, H, KVH, hd, hd ** -0.5, bad)


def test_engine_with_document_mask_fused_matches_aten_path():
    """Same model + packed data with separators: sm_90a kernel path vs ATen path (bf16), with selective recompute."""
    from fms_fsdp_b200.models.llama import LLaMA, LLaMABlock, LLaMAConfig
    from fms_fsdp_b200.ops import cuda_kernels as CK
    from fms_fsdp_b200.ops import set_kernel_path
    from fms_fsdp_b200.parallel import ShardedAdamW, ShardedModel
    from fms_fsdp_b200.policies import apply_fsdp_checkpointing, bfSixteen

    def run(path, doc=True):
        set_kernel_path(path)
        torch.manual_seed(0); torch.cuda.manual_seed(0)
        cfg = LLaMAConfig(src_vocab_size=2048, emb_dim=512, nheads=4, kvheads=2, nlayers=3, multiple_of=256,
                          max_expected_seq_len=256, doc_separator=SEP if doc else None)
        with torch.device("meta"):
            m = LLaMA(cfg)
        apply_fsdp_checkpointing(m, LLaMABlock, "1/2")
        eng = ShardedModel(m, mixed_precision=bfSixteen, device=torch.device("cuda", 0))
        opt = ShardedAdamW(eng, lr=1e-3)
        x = torch.randint(2, 2048, (2, 256), generator=torch.Generator().manual_seed(3))
        x[0, [37, 38, 127, 200]] = SEP
        x[1, [0, 64, 191]] = SEP
        x = x.cuda()
        out = []
        for _ in range(4):
            l = eng.forward_backward(x, x); g = eng.clip_grad_norm_(1.0); opt.step(); out.append((l.item(), g.item()))
        return out
    try:
        n0, f0 = CK.launch_count(), CK.fallback_count()
        fused = run("fused")
        assert CK.launch_count() - n0 > 100 and CK.fallback_count() == f0
        aten = run("torch")
        plain = run("fused", doc=False)
    finally:
        set_kernel_path("auto")
    for (lf, gf), (la, ga) in zip(fused, aten):
        assert abs(lf - la) < 3e-2 * abs(la) and abs(gf - ga) < 6e-2 * abs(ga)
    assert fused[-1][0] < fused[0][0]
    assert [l for l, _ in fused] != [l for l, _ in plain]
