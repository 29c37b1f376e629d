"""GPU tier: the warp-specialised attention kernels (``attn_fwd_pipe_kernel`` / ``attn_bwd_pipe_kernel``) against the
fp32 oracle and bit for bit against the lock-step kernels they replace, where the producer ring wraps or runs short
(1-5 streamed tiles against a ring of 2 / 3 stages), on ragged sequences, every GQA group size and document layouts with
1-, 64- and 513-token documents; and run-to-run determinism at the headline shape.  ``tests/test_sass.py`` checks their
SASS."""

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


def _inputs(B, S, H, KVH, hd, seed=3):
    g = torch.Generator(device=DEV).manual_seed(seed)
    qkv = torch.randn(B * S, (H + 2 * KVH) * hd, device=DEV, generator=g).bfloat16()
    do = torch.randn(B * S, H * hd, device=DEV, generator=g).bfloat16()
    return qkv, do


def _seg(seps_per_row, S):
    tok = torch.zeros(len(seps_per_row), S, dtype=torch.long)
    for r, seps in enumerate(seps_per_row):
        for p in seps:
            if p < S:
                tok[r, p] = SEP
    return ops.document_segments(tok.to(DEV), SEP)


def _both(CK, qkv, do, B, S, H, KVH, hd, seg=None, rope=None):
    """(pipelined, lock-step) outputs: o, lse, dqkv"""
    C = CK._C
    sc = hd ** -0.5
    o, l = C.attn_fwd(qkv, B, S, H, KVH, hd, sc, seg)
    g = C.attn_bwd(do, qkv, o, l, B, S, H, KVH, hd, sc, rope, seg)
    o_r, l_r = C.attn_fwd_lockstep(qkv, B, S, H, KVH, hd, sc, seg)
    g_r = C.attn_bwd_lockstep(do, qkv, o_r, l_r, B, S, H, KVH, hd, sc, rope, seg)
    return (o, l, g), (o_r, l_r, g_r)


def _assert_bitwise(new, ref):
    for name, a, b in zip(("o", "lse", "dqkv"), new, ref):
        assert torch.equal(a, b), (name, (a.float() - b.float()).abs().max().item())


# S: 64 -> one streamed tile per head; 200 / 320 / 384 ragged and 2-6 tiles; 640 -> 5 kv tiles in the forward
@pytest.mark.parametrize("S", [64, 128, 200, 320, 384, 640])
@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("G", [1, 2, 4, 8])
def test_pipeline_matches_oracle_and_lockstep(K, S, hd, G):
    CK, TK = K
    B, KVH = 2, 2
    H = G * KVH
    qkv, do = _inputs(B, S, H, KVH, hd)
    new, ref = _both(CK, qkv, do, B, S, H, KVH, hd)
    _assert_bitwise(new, ref)
    sc = hd ** -0.5
    o0, l0 = TK.attn_fwd(qkv, B, S, H, KVH, hd, sc)
    g0 = TK.attn_bwd(do, qkv, o0, l0, B, S, H, KVH, hd, sc)
    assert rel(new[0], o0) < 1e-2 and rel(new[1], l0) < 1e-4
    assert rel(new[2], g0) < 1.5e-2


# documents of 1 token, of 64 tokens (tile-aligned) and of 513 tokens (one past a tile edge)
DOC_LAYOUTS = {
    "one_token": [[0, 1, 2, 130, 131, 700], [5, 6, 7, 8, 600]],
    "sixty_four": [list(range(63, 1024, 64)), list(range(63, 1024, 64))],
    "five_thirteen": [[512, 1025], [512]],
}


@pytest.mark.parametrize("layout", sorted(DOC_LAYOUTS))
@pytest.mark.parametrize("cfg", [(1024, 4, 1, 128), (800, 8, 2, 64), (1024, 16, 4, 128)])
def test_pipeline_doc_matches_oracle_and_lockstep(K, layout, cfg):
    CK, TK = K
    S, H, KVH, hd = cfg
    B = 2
    seg = _seg(DOC_LAYOUTS[layout], S)
    qkv, do = _inputs(B, S, H, KVH, hd)
    new, ref = _both(CK, qkv, do, B, S, H, KVH, hd, seg=seg)
    _assert_bitwise(new, ref)
    sc = hd ** -0.5
    o0, l0 = TK.attn_fwd(qkv.float(), B, S, H, KVH, hd, sc, seg=seg)
    g0 = TK.attn_bwd(do.float(), qkv.float(), o0, l0, B, S, H, KVH, hd, sc, seg=seg)
    assert rel(new[0], o0) < 1e-2 and rel(new[1], l0) < 1e-4
    assert rel(new[2], g0) < 1.5e-2


def test_pipeline_with_rope_epilogue_matches_lockstep(K):
    CK, _ = K
    B, S, H, KVH, hd = 2, 1024, 16, 4, 128
    qkv, do = _inputs(B, S, H, KVH, hd)
    rope = ops.torch_kernels.rope_table(S, hd, 1e4, device=DEV)
    new, ref = _both(CK, qkv, do, B, S, H, KVH, hd, rope=rope)
    _assert_bitwise(new, ref)


@pytest.mark.parametrize("H,KVH", [(16, 4), (32, 32)])
def test_headline_shape_bitwise_lockstep_and_deterministic(K, H, KVH):
    CK, _ = K
    B, S, hd = 2, 4096, 128
    qkv, do = _inputs(B, S, H, KVH, hd, seed=11)
    new, ref = _both(CK, qkv, do, B, S, H, KVH, hd)
    _assert_bitwise(new, ref)
    again, _ = _both(CK, qkv, do, B, S, H, KVH, hd)
    _assert_bitwise(again, new)
