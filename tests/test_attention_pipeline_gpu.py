"""GPU tier: the warp-specialised attention kernels (``attn_fwd_pipe_kernel`` / ``attn_bwd_pipe_kernel``) against the
fp32 oracle and bit for bit against the lock-step kernels they replace, where the producer ring wraps or runs short
(1-5 streamed tiles against a ring of 2 / 3 stages), on ragged sequences, every GQA group size and document layouts with
1-, 64- and 513-token documents; run-to-run determinism at the headline shape; and the SASS of the new kernels."""
import json
import os
import re
import shutil
import subprocess

import pytest
import torch

from fms_fsdp_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
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


# --------------------------------------------------------------------------------------------------------- SASS
def _sass():
    so = os.path.join(ROOT, "fms_fsdp_b200", "_C.so")
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(so) or not os.path.exists(exe):
        pytest.skip("needs the built extension and cuobjdump")
    out = subprocess.run([exe, "-sass", so], capture_output=True, text=True, timeout=600).stdout
    import hashlib
    per, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            per[name] = []
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?;)", line)      # instruction lines only, without addresses
        if name and m:
            per[name].append(m.group(1))
    return {k: hashlib.sha256("\n".join(v).encode()).hexdigest() for k, v in per.items()}, per


def test_sass_pipelined_kernels_and_existing_kernels_unchanged():
    """``tests/golden/sass_before_attn_pipeline.json``: per-kernel digests of every kernel of the extension before the
    pipelined attention kernels were added (``scripts/sass_digest.py``, CUDA 12.9), the lock-step attention kernels
    included.  setmaxnreg is ``USETMAXREG`` in SASS; the dK/dV instantiations bring -lse / -delta in by ``UBLKCP``."""
    digests, per = _sass()
    new = [k for k in per if "attn_fwd_pipe_kernel" in k or "attn_bwd_pipe_kernel" in k]
    assert len(new) == 4 + 8, new
    for k in new:
        body = per[k]
        assert any(i.startswith("HGMMA") for i in body) and any(i.startswith("UTMALDG") for i in body), k
        assert sum(i.startswith("USETMAXREG") for i in body) == 2, k          # producer dec + consumer inc
        assert not any(re.match(r"(LDL|STL)\b", i) for i in body), k
        # the overlap survives register allocation: a kernel whose wgmmas ptxas serialised (C7512) waits after every
        # HGMMA; the schedule waits at most 4 times (forward: S, PV in the loop and around it; backward: S, dP, end)
        depbar = sum(i.startswith("WARPGROUP.DEPBAR") for i in body)
        hgmma = sum(i.startswith("HGMMA") for i in body)
        assert depbar <= 4 and 3 * depbar <= hgmma, (k, depbar, hgmma)
        if "attn_bwd_pipe_kernelILi128ELi0E" in k or "attn_bwd_pipe_kernelILi64ELi0E" in k:
            assert any(i.startswith("UBLKCP") for i in body), k
    with open(os.path.join(ROOT, "tests", "golden", "sass_before_attn_pipeline.json")) as f:
        before = json.load(f)
    changed = [k for k, v in before.items() if digests.get(k) != v]
    assert not changed, changed
