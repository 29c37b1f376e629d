"""GPU tier: the warp-specialised attention kernels (``attn_fwd_pipe_kernel`` / ``attn_bwd_pipe_kernel``) against the
fp32 oracle and bit for bit against the outputs recorded in ``tests/golden/attention_bits.json``, where the producer
ring wraps or runs short (1-5 streamed tiles against a ring of 2 / 3 stages), on ragged sequences, every GQA group size
and document layouts with 1-, 64- and 513-token documents; and run-to-run determinism at the headline shape.
``tests/test_attention_numerics_gpu.py`` checks the same kernels row by row against float64; ``tests/test_sass.py``
checks their SASS.

The golden holds the SHA-256 of every case's input bytes (qkv, dO, and the document or RoPE table where the case has
one) and output bytes (o, lse, dqkv).  The inputs come from a CPU generator, so they do not depend on the CUDA RNG.  A
change that means to change attention numerics regenerates the golden in the same commit, from the repository root:

    PYTHONPATH=. python tests/test_attention_pipeline_gpu.py
"""

import hashlib
import json
import os

import pytest
import torch

from fms_fsdp_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"
SEP = 1
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "attention_bits.json")


@pytest.fixture(scope="module")
def K():
    from fms_fsdp_b200.ops import cuda_kernels as CK
    from fms_fsdp_b200.ops import torch_kernels as TK
    assert CK._C.__file__.endswith("_C.so")
    return CK, TK


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as f:
        return json.load(f)


def rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).abs().max() / b.abs().max().clamp(min=1e-6)).item()


def sha256(t):
    return hashlib.sha256(t.detach().contiguous().cpu().view(torch.uint8).numpy().tobytes()).hexdigest()


def _inputs(B, S, H, KVH, hd, seed=3):
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(B * S, (H + 2 * KVH) * hd, generator=g).bfloat16()
    do = torch.randn(B * S, H * hd, generator=g).bfloat16()
    return qkv.to(DEV), do.to(DEV)


def _seg(seps_per_row, S):
    tok = torch.zeros(len(seps_per_row), S, dtype=torch.long)
    for r, seps in enumerate(seps_per_row):
        for p in seps:
            if p < S:
                tok[r, p] = SEP
    return ops.document_segments(tok.to(DEV), SEP)


# S: 64 -> one streamed tile per head; 200 / 320 / 384 ragged and 2-6 tiles; 640 -> 5 kv tiles in the forward
CAUSAL_S = [64, 128, 200, 320, 384, 640]
CAUSAL_HD = [64, 128]
CAUSAL_G = [1, 2, 4, 8]
# documents of 1 token, of 64 tokens (tile-aligned) and of 513 tokens (one past a tile edge)
DOC_LAYOUTS = {
    "one_token": [[0, 1, 2, 130, 131, 700], [5, 6, 7, 8, 600]],
    "sixty_four": [list(range(63, 1024, 64)), list(range(63, 1024, 64))],
    "five_thirteen": [[512, 1025], [512]],
}
DOC_CFGS = [(1024, 4, 1, 128), (800, 8, 2, 64), (1024, 16, 4, 128)]
HEADLINE = [(16, 4), (32, 32)]


def causal_case(S, hd, G):
    KVH = 2
    return f"causal_S{S}_hd{hd}_G{G}", dict(B=2, S=S, H=G * KVH, KVH=KVH, hd=hd)


def doc_case(layout, cfg):
    S, H, KVH, hd = cfg
    return f"doc_{layout}_S{S}_H{H}_KVH{KVH}_hd{hd}", dict(B=2, S=S, H=H, KVH=KVH, hd=hd, layout=layout)


def rope_case():
    return "rope_S1024_H16_KVH4_hd128", dict(B=2, S=1024, H=16, KVH=4, hd=128, rope=True)


def headline_case(H, KVH):
    return f"headline_S4096_H{H}_KVH{KVH}_hd128", dict(B=2, S=4096, H=H, KVH=KVH, hd=128, seed=11)


def all_cases():
    return ([causal_case(S, hd, G) for S in CAUSAL_S for hd in CAUSAL_HD for G in CAUSAL_G]
            + [doc_case(layout, cfg) for layout in sorted(DOC_LAYOUTS) for cfg in DOC_CFGS]
            + [rope_case()] + [headline_case(H, KVH) for H, KVH in HEADLINE])


def case_inputs(c):
    """{name: tensor} of a case's inputs on the GPU: qkv, do and, where the case has one, seg or rope"""
    x = dict(zip(("qkv", "do"), _inputs(c["B"], c["S"], c["H"], c["KVH"], c["hd"], c.get("seed", 3))))
    if "layout" in c:
        x["seg"] = _seg(DOC_LAYOUTS[c["layout"]], c["S"])
    if c.get("rope"):
        x["rope"] = ops.torch_kernels.rope_table(c["S"], c["hd"], 1e4, device=DEV)
    return x


def run(C, c, x):
    """(o, lse, dqkv) of the kernels the model runs"""
    B, S, H, KVH, hd = c["B"], c["S"], c["H"], c["KVH"], c["hd"]
    sc = hd ** -0.5
    seg = x.get("seg")
    o, l = C.attn_fwd(x["qkv"], B, S, H, KVH, hd, sc, seg)
    g = C.attn_bwd(x["do"], x["qkv"], o, l, B, S, H, KVH, hd, sc, x.get("rope"), seg)
    return o, l, g


def digests(x, outs):
    return {**{k: sha256(v) for k, v in x.items()}, **{k: sha256(v) for k, v in zip(("o", "lse", "dqkv"), outs)}}


def _assert_golden(golden, name, x, outs):
    want, have = golden[name], digests(x, outs)
    for k in x:
        assert have[k] == want[k], f"{name}: input {k} changed (not the kernels): its bytes no longer match the golden"
    for k in ("o", "lse", "dqkv"):
        assert have[k] == want[k], f"{name}: {k} differs from the golden bits"


@pytest.mark.parametrize("S", CAUSAL_S)
@pytest.mark.parametrize("hd", CAUSAL_HD)
@pytest.mark.parametrize("G", CAUSAL_G)
def test_pipeline_matches_oracle_and_golden(K, golden, S, hd, G):
    CK, TK = K
    name, c = causal_case(S, hd, G)
    B, H, KVH = c["B"], c["H"], c["KVH"]
    x = case_inputs(c)
    new = run(CK._C, c, x)
    _assert_golden(golden, name, x, new)
    qkv, do = x["qkv"], x["do"]
    sc = hd ** -0.5
    o0, l0 = TK.attn_fwd(qkv, B, S, H, KVH, hd, sc)
    g0 = TK.attn_bwd(do, qkv, o0, l0, B, S, H, KVH, hd, sc)
    assert rel(new[0], o0) < 1e-2 and rel(new[1], l0) < 1e-4
    assert rel(new[2], g0) < 1.5e-2


@pytest.mark.parametrize("layout", sorted(DOC_LAYOUTS))
@pytest.mark.parametrize("cfg", DOC_CFGS)
def test_pipeline_doc_matches_oracle_and_golden(K, golden, layout, cfg):
    CK, TK = K
    name, c = doc_case(layout, cfg)
    B, S, H, KVH, hd = c["B"], c["S"], c["H"], c["KVH"], c["hd"]
    x = case_inputs(c)
    new = run(CK._C, c, x)
    _assert_golden(golden, name, x, new)
    qkv, do, seg = x["qkv"], x["do"], x["seg"]
    sc = hd ** -0.5
    o0, l0 = TK.attn_fwd(qkv.float(), B, S, H, KVH, hd, sc, seg=seg)
    g0 = TK.attn_bwd(do.float(), qkv.float(), o0, l0, B, S, H, KVH, hd, sc, seg=seg)
    assert rel(new[0], o0) < 1e-2 and rel(new[1], l0) < 1e-4
    assert rel(new[2], g0) < 1.5e-2


def test_pipeline_with_rope_epilogue_matches_golden(K, golden):
    CK, _ = K
    name, c = rope_case()
    x = case_inputs(c)
    _assert_golden(golden, name, x, run(CK._C, c, x))


@pytest.mark.parametrize("H,KVH", HEADLINE)
def test_headline_shape_matches_golden_and_deterministic(K, golden, H, KVH):
    CK, _ = K
    name, c = headline_case(H, KVH)
    x = case_inputs(c)
    new = run(CK._C, c, x)
    _assert_golden(golden, name, x, new)
    again = run(CK._C, c, x)
    for what, a, b in zip(("o", "lse", "dqkv"), again, new):
        assert torch.equal(a, b), (what, (a.float() - b.float()).abs().max().item())


def record(C):
    """{case: {input and output: SHA-256}} of every case, from the kernels of ``C``"""
    out = {}
    for name, c in all_cases():
        x = case_inputs(c)
        out[name] = digests(x, run(C, c, x))
    return out


if __name__ == "__main__":
    from fms_fsdp_b200.ops import cuda_kernels as CK
    bits = record(CK._C)
    with open(GOLDEN, "w") as f:
        json.dump(bits, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"wrote {len(bits)} cases to {GOLDEN}")
