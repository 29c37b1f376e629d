"""GPU tier: the QK-norm kernels (``qk_norm_rope`` / ``qk_norm_bwd``) against the fp32 oracle, their determinism,
``qkv_attention(qk_norm=...)`` on the fused kernels against the ATen path (plain, document-masked and fp8), one engine step
of a Qwen3-1.7B-shaped model, and the SASS of the new kernels."""
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


@pytest.fixture(scope="module")
def K():
    from fms_fsdp_b200.ops import cuda_kernels as CK
    from fms_fsdp_b200.ops import torch_kernels as TK
    assert CK._C.__file__.endswith("_C.so")
    return CK, TK


def rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).abs().max() / b.abs().max().clamp(min=1e-6)).item()


def _inputs(B, S, H, KVH, hd, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    qkv = (torch.randn(B * S, (H + 2 * KVH) * hd, device=DEV, generator=g) * 2).to(torch.bfloat16)
    wq = (0.5 + torch.rand(hd, device=DEV, generator=g)).to(torch.bfloat16)     # random, non-unit gains
    wk = (0.5 + torch.rand(hd, device=DEV, generator=g)).to(torch.bfloat16)
    table = ops.torch_kernels.rope_table(S, hd, 1e6, device=DEV)
    return qkv, wq, wk, table


# (B, S, H, KVH, hd): B*S = 3*37 = 111 rows (not a multiple of any row block), GQA and MHA, both head dims, and S = 4096
CASES = [(3, 37, 4, 2, 64), (3, 37, 4, 4, 128), (2, 256, 16, 8, 128), (1, 4096, 16, 4, 128), (2, 4096, 8, 2, 64)]


@pytest.mark.parametrize("B,S,H,KVH,hd", CASES)
def test_kernels_match_the_fp32_oracle(K, B, S, H, KVH, hd):
    CK, TK = K
    qkv, wq, wk, table = _inputs(B, S, H, KVH, hd)
    f0 = CK.fallback_count()
    y = qkv.clone()
    xqk, rstd = CK.qk_norm_rope(y, wq, wk, table, S, H, KVH, hd, 1e-6)
    y32 = qkv.float()
    xqk32, rstd32 = TK.qk_norm_rope(y32, wq, wk, table, S, H, KVH, hd, 1e-6)
    assert torch.equal(xqk, qkv[:, :(H + KVH) * hd])                    # the pre-norm q / k, bit for bit
    assert torch.allclose(rstd, rstd32, rtol=1e-5, atol=0)
    assert rel(y, y32) < 8e-3
    assert torch.equal(y[:, (H + KVH) * hd:], qkv[:, (H + KVH) * hd:])  # V untouched

    g = torch.Generator(device=DEV).manual_seed(1)
    d = torch.randn(B * S, (H + 2 * KVH) * hd, device=DEV, generator=g).to(torch.bfloat16)
    dx = d.clone()
    dwq, dwk = CK.qk_norm_bwd(dx, xqk, rstd, wq, wk, H, KVH, hd)
    dx32 = d.float()
    dwq32, dwk32 = TK.qk_norm_bwd(dx32, xqk.float(), rstd, wq, wk, H, KVH, hd)
    assert CK.fallback_count() == f0
    assert dwq.dtype == torch.float32 and dwq.shape == (hd,)
    assert rel(dx, dx32) < 8e-3
    assert torch.equal(dx[:, (H + KVH) * hd:], d[:, (H + KVH) * hd:])
    assert rel(dwq, dwq32) < 1e-4 and rel(dwk, dwk32) < 1e-4


def test_backward_is_bitwise_deterministic(K):
    CK, _ = K
    B, S, H, KVH, hd = 2, 4096, 16, 8, 128
    qkv, wq, wk, table = _inputs(B, S, H, KVH, hd, seed=4)
    xqk, rstd = CK.qk_norm_rope(qkv, wq, wk, table, S, H, KVH, hd, 1e-6)
    d = torch.randn(B * S, (H + 2 * KVH) * hd, device=DEV).to(torch.bfloat16)
    outs = []
    for _ in range(2):
        dx = d.clone()
        outs.append((dx, *CK.qk_norm_bwd(dx, xqk, rstd, wq, wk, H, KVH, hd)))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def _node(path, H, KVH, hd, doc, precision="bf16"):
    from fms_fsdp_b200.ops import set_kernel_path
    from fms_fsdp_b200.ops.functional import set_gemm_precision
    B, S, D = 2, 512, H * 64
    g = torch.Generator(device=DEV).manual_seed(7)
    h = (torch.randn(B, S, D, device=DEV, generator=g)).to(torch.bfloat16).requires_grad_()
    w = (torch.randn((H + 2 * KVH) * hd, D, device=DEV, generator=g) * D ** -0.5).to(torch.bfloat16).requires_grad_()
    wq = (0.5 + torch.rand(hd, device=DEV, generator=g)).to(torch.bfloat16).requires_grad_()
    wk = (0.5 + torch.rand(hd, device=DEV, generator=g)).to(torch.bfloat16).requires_grad_()
    table = ops.torch_kernels.rope_table(S, hd, 1e6, device=DEV)
    do = torch.randn(B, S, H * hd, device=DEV, generator=g).to(torch.bfloat16)
    seg = None
    if doc:
        tok = torch.full((B, S), 5, device=DEV)
        tok[0, [63, 200, 201]] = 1
        tok[1, [128, 400]] = 1
        seg = ops.document_segments(tok, 1)
    set_kernel_path(path)
    set_gemm_precision(precision)
    try:
        o = ops.qkv_attention(h, w, table, H, KVH, hd, doc=seg, qk_norm=(wq, wk, 1e-6))
        grads = torch.autograd.grad(o, (h, w, wq, wk), do)
    finally:
        set_kernel_path("auto")
        set_gemm_precision("bf16")
    return o, grads


@pytest.mark.parametrize("doc", [False, True])
@pytest.mark.parametrize("H,KVH,hd", [(8, 2, 128), (4, 4, 64)])
def test_qkv_attention_with_qk_norm_matches_the_aten_path(K, H, KVH, hd, doc):
    CK, _ = K
    f0, n0 = CK.fallback_count(), CK.launch_count()
    o, grads = _node("fused", H, KVH, hd, doc)
    assert CK.fallback_count() == f0 and CK.launch_count() - n0 >= 8
    o_ref, grads_ref = _node("torch", H, KVH, hd, doc)
    assert rel(o, o_ref) < 2e-2
    for name, a, b in zip(("dh", "dw", "dw_q", "dw_k"), grads, grads_ref):
        assert rel(a, b) < 3e-2, name
    if doc:   # the mask reached the node
        o_plain, _ = _node("fused", H, KVH, hd, False)
        assert rel(o, o_plain) > 5e-2


def test_qkv_attention_with_qk_norm_fp8_branch(K):
    CK, _ = K
    f0 = CK.fallback_count()
    o, grads = _node("fused", 8, 2, 128, True, precision="fp8")
    assert CK.fallback_count() == f0
    o_ref, grads_ref = _node("torch", 8, 2, 128, True, precision="fp8")
    o_bf16, _ = _node("fused", 8, 2, 128, True)
    assert rel(o, o_ref) < 3e-2 and rel(o, o_bf16) < 1e-1
    for name, a, b in zip(("dh", "dw", "dw_q", "dw_k"), grads, grads_ref):
        assert rel(a, b) < 5e-2, name


def test_engine_step_qwen3_shape_fused_matches_aten_path():
    """A 2-layer model with the Qwen3-1.7B block (D 2048, 16 / 8 heads of 128, F 6144, QK-norm): one optimizer step on the
    sm_90a kernels against the ATen path, with no fallback on the kernel path."""
    from fms_fsdp_b200.models.llama import LLaMA
    from fms_fsdp_b200.ops import cuda_kernels as CK
    from fms_fsdp_b200.ops import set_kernel_path
    from fms_fsdp_b200.parallel import ShardedAdamW, ShardedModel
    from fms_fsdp_b200.policies import bfSixteen
    from fms_fsdp_b200.utils.config_utils import get_model_config

    def run(path):
        set_kernel_path(path)
        torch.manual_seed(0); torch.cuda.manual_seed(0)
        cfg = get_model_config("qwen3_1.7b")
        cfg.nlayers, cfg.src_vocab_size = 2, 32768
        with torch.device("meta"):
            m = LLaMA(cfg)
        eng = ShardedModel(m, mixed_precision=bfSixteen, device=torch.device("cuda", 0))
        opt = ShardedAdamW(eng, lr=1e-3)
        x = torch.randint(0, cfg.src_vocab_size, (2, 1024), generator=torch.Generator().manual_seed(3)).cuda()
        out = []
        for _ in range(2):
            l = eng.forward_backward(x, x); gn = eng.clip_grad_norm_(1.0); opt.step(); out.append((l.item(), gn.item()))
        qn = eng.full_state_dict()["layers.0.attn.q_norm.weight"].float().cpu()
        return out, qn
    try:
        f0 = CK.fallback_count()
        fused, qf = run("fused")
        assert CK.fallback_count() == f0
        aten, qa = run("torch")
    finally:
        set_kernel_path("auto")
    for (lf, gf), (la, ga) in zip(fused, aten):
        assert abs(lf - la) < 2e-2 * abs(la) and abs(gf - ga) < 5e-2 * abs(ga)
    assert not torch.equal(qf, torch.ones_like(qf))          # the norm gains were trained
    assert (qf - qa).abs().max() < 2e-3


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


def test_sass_new_kernels_no_local_memory_and_existing_kernels_unchanged():
    """``tests/golden/sass_before_qk_norm.json``: per-kernel digests of the instructions of every kernel of the extension as
    it was before the QK-norm kernels were added (``scripts/sass_digest.py``, CUDA 12.9).  Adding QK-norm changes none."""
    digests, per = _sass()
    new = [k for k in per if "qk_norm" in k]
    assert len(new) == 4, new
    for k in new:
        assert not any(re.match(r"(LDL|STL)\b", i) for i in per[k]), k
    with open(os.path.join(ROOT, "tests", "golden", "sass_before_qk_norm.json")) as f:
        before = json.load(f)
    changed = [k for k, v in before.items() if digests.get(k) != v]
    assert not changed, changed
