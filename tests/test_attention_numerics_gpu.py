"""GPU tier of the per-row attention check: the sm_90a kernels (``_C.attn_fwd`` / ``_C.attn_bwd``, the pipelined ones
the model runs) against the float64 reference of ``tests/attention_reference.py``, row by row, in flat, peaked,
sink-dominated, late-max and tied softmax regimes; at sequence lengths around the 64- and 128-row tile edges (S = 1 to
4096), head dims 64 and 128, GQA groups 1, 2, 4, 7 and 8, two batch rows of different data; at the headline shapes;
with the inverse-RoPE backward epilogue at S = 4096; and with document masks.  Every element of every output must be
finite.  Each case prints its worst per-row ratio over the tolerance ("MEASURE ... x tol"), so the headroom is in the
log.  The tolerances come from the CPU rounding emulation (tests/test_attention_numerics_cpu.py), not from a GPU run.
The float64 reference runs on the GPU, one (batch row, kv head) at a time.
"""
import pytest
import torch

import attention_reference as AR

pytestmark = pytest.mark.gpu
DEV = "cuda"
GROUPS = (1, 2, 4, 7, 8)


@pytest.fixture(scope="module")
def C():
    from fms_fsdp_b200.ops import cuda_kernels as CK
    assert CK._C.__file__.endswith("_C.so")
    return CK._C


def measure(C, tag, regime, B, S, H, KVH, hd, seed=7, seg=None, rope=None, boost=None):
    """Run the kernels once, print the worst per-row ratios; returns the failures (empty when the case passes)."""
    qkv, do = (t.to(DEV) for t in AR.make_inputs(regime, B, S, H, KVH, hd, seed, boost=boost))
    sc = hd ** -0.5
    o, lse = C.attn_fwd(qkv, B, S, H, KVH, hd, sc, seg)
    dqkv = C.attn_bwd(do, qkv, o, lse, B, S, H, KVH, hd, sc, rope, seg)
    bad = [n + " not finite" for n, t in (("o", o), ("lse", lse), ("dqkv", dqkv)) if not torch.isfinite(t).all()]
    ref = AR.reference(qkv, do, B, S, H, KVH, hd, sc, seg=seg, rope=rope)
    out = AR.kernel_view(o, lse, dqkv, B, S, H, KVH, hd)
    w = AR.worst(out, ref)
    print(f"MEASURE attn {tag}: " + " ".join(f"{n} {v / AR.TOL[n]:.2f}" for n, v in w.items()) + " x tol")
    bad += [f"{n} {v:.2e} > {AR.TOL[n]:.0e}" for n, v in w.items() if not v <= AR.TOL[n]]
    return [f"{tag}: {b}" for b in bad]


# S around the tile edges: below one 64-row tile, at and one past the 64 / 128 edges, 5 kv tiles, ragged 1000.  Every
# regime runs once per (S, hd), with the GQA group rotating so each group meets every regime and both head dims.
@pytest.mark.parametrize("S", [1, 63, 64, 65, 127, 128, 129, 640, 1000])
@pytest.mark.parametrize("hd", [64, 128])
def test_regimes_at_tile_edges(C, S, hd):
    KVH = 2
    fails = []
    for i, regime in enumerate(AR.REGIMES):
        G = GROUPS[(i + S + hd // 64) % len(GROUPS)]
        fails += measure(C, f"{regime} B2 S{S} H{G * KVH} KVH{KVH} hd{hd}", regime, 2, S, G * KVH, KVH, hd)
    assert not fails, fails


# the running max and the sink at full length, Qwen2.5's 14 / 2 grouping
@pytest.mark.parametrize("regime", ["sink", "late_max"])
def test_regimes_at_4096(C, regime):
    fails = measure(C, f"{regime} B2 S4096 H14 KVH2 hd64", regime, 2, 4096, 14, 2, 64)
    assert not fails, fails


@pytest.mark.parametrize("shape", [(2, 4096, 16, 4, 128), (1, 4096, 32, 32, 128)],
                         ids=lambda s: "B{}_S{}_H{}_KVH{}_hd{}".format(*s))
@pytest.mark.parametrize("regime", ["flat", "peaked16"])
def test_headline_shapes(C, shape, regime):
    B, S, H, KVH, hd = shape
    fails = measure(C, f"{regime} headline B{B} S{S} H{H} KVH{KVH}", regime, B, S, H, KVH, hd)
    assert not fails, fails


def test_inverse_rope_epilogue_at_4096(C):
    from fms_fsdp_b200.ops import torch_kernels as TK
    B, S, H, KVH, hd = 2, 4096, 16, 4, 128
    rope = TK.rope_table(S, hd, 1e4, device=DEV)
    fails = measure(C, "flat rope B2 S4096 H16 KVH4", "flat", B, S, H, KVH, hd, rope=rope)
    assert not fails, fails


@pytest.mark.parametrize("layout", ["mid_tile", "one_token", "low_after_high"])
@pytest.mark.parametrize("cfg", [(8, 2, 128), (14, 2, 64)], ids=lambda c: "H{}_KVH{}_hd{}".format(*c))
def test_document_masks(C, layout, cfg):
    H, KVH, hd = cfg
    B, S = 2, 1000
    seps = AR.doc_layouts(S)[layout]
    seg = AR.segments(seps, S, DEV)
    fails = []
    if layout == "low_after_high":   # the first document of each row leans towards u by a logit of ~12
        boost = torch.arange(S) < min(p for r in seps for p in r)
        fails += measure(C, f"doc {layout} boosted H{H} hd{hd}", "boosted", B, S, H, KVH, hd, seg=seg, boost=boost)
    for regime in ("flat", "peaked16"):
        fails += measure(C, f"doc {layout} {regime} H{H} hd{hd}", regime, B, S, H, KVH, hd, seg=seg)
    assert not fails, fails
