"""GPU tier: the QK-norm kernels (``qk_norm_rope`` / ``qk_norm_bwd``) against float64 per (row, head), their determinism,
``qkv_attention(qk_norm=...)`` on the fused kernels against the ATen path (plain, document-masked and fp8), one engine step
of a Qwen3-1.7B-shaped model.  ``tests/test_sass.py`` checks their SASS."""

import pytest
import torch

import llama_node_reference as LR
from fms_fsdp_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"


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
    """The kernels' exact invariants, and their accuracy per (row, head) against the float64 reference of
    tests/llama_node_reference.py (which tests/test_llama_nodes_gpu.py runs at the Qwen3 shapes and regimes)."""
    CK, _ = K
    qkv, wq, wk, table = _inputs(B, S, H, KVH, hd)
    nh = H + KVH
    f0 = CK.fallback_count()
    y = qkv.clone()
    xqk, rstd = CK.qk_norm_rope(y, wq, wk, table, S, H, KVH, hd, 1e-6)
    assert torch.equal(xqk, qkv[:, :nh * hd])                    # the pre-norm q / k, bit for bit
    assert torch.equal(y[:, nh * hd:], qkv[:, nh * hd:])          # V untouched
    yr, rr = LR.qk_norm_fwd(qkv, wq, wk, table, S, H, KVH, hd, 1e-6)
    assert LR.head_ratio(y[:, :nh * hd], yr[:, :nh * hd], hd) <= LR.TOL["qk_y"]
    assert LR.ratio(rstd.reshape(-1, 1), rr.reshape(-1, 1)) <= LR.TOL["qk_rstd"]

    g = torch.Generator(device=DEV).manual_seed(1)
    d = torch.randn(B * S, (H + 2 * KVH) * hd, device=DEV, generator=g).to(torch.bfloat16)
    dx = d.clone()
    dwq, dwk = CK.qk_norm_bwd(dx, xqk, rstd, wq, wk, H, KVH, hd)
    assert CK.fallback_count() == f0
    assert dwq.dtype == torch.float32 and dwq.shape == (hd,)
    assert torch.equal(dx[:, nh * hd:], d[:, nh * hd:])
    ref, rq, rk, aq, ak, sc = LR.qk_norm_bwd(d, xqk, rstd, wq, wk, H, KVH, hd)
    assert LR.head_ratio(dx[:, :nh * hd], ref[:, :nh * hd], hd, sc) <= LR.TOL["qk_dx"]
    assert LR.vratio(dwq, rq, aq) <= LR.TOL["qk_dw"] and LR.vratio(dwk, rk, ak) <= LR.TOL["qk_dw"]


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
