"""GPU tier: the q / k / v bias + RoPE epilogue of the QKV GEMM (``EPI_ROPE_BIAS``) on the 128 x 128 tile, the 128 x 256
tile and the fused all-gather build, ``bias_grad`` against an fp64 column sum and its determinism,
``qkv_attention(qkv_bias=...)`` on the fused kernels against the ATen path (plain and document-masked), one engine step of
a Qwen2.5-1.5B-shaped model.  ``tests/test_sass.py`` checks their SASS."""
import contextlib

import pytest
import torch

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


@contextlib.contextmanager
def tile(CK, mode):
    CK._C._set_gemm_tile({"narrow": 1, "wide": 2}[mode])
    try:
        yield
    finally:
        CK._C._set_gemm_tile(0)


# the QKV projections of Qwen2.5-0.5B (D 896, H 14 / KVH 2 of 64), 1.5B (D 1536, 12 / 2 of 128) and 7B (D 3584, 28 / 4 of
# 128): N = 1152, 2048, 4608
SHAPES = {"0.5b": (896, 14, 2, 64), "1.5b": (1536, 12, 2, 128), "7b": (3584, 28, 4, 128)}


def _proj_inputs(D, H, KVH, hd, B, S, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    N = (H + 2 * KVH) * hd
    x = torch.randn(B * S, D, device=DEV, generator=g).to(torch.bfloat16)
    w = (torch.randn(N, D, device=DEV, generator=g) * D ** -0.5).to(torch.bfloat16)
    b = (torch.randn(N, device=DEV, generator=g) * 2).to(torch.bfloat16)           # non-zero, larger than x w^T
    table = ops.torch_kernels.rope_table(S, hd, 1e6, device=DEV)
    return x, w, b, table


@pytest.mark.parametrize("BS", [(2, 1024), (5, 200)])          # M = 2048 (16 row tiles) and 1000 (ragged last tile)
@pytest.mark.parametrize("name", sorted(SHAPES))
def test_bias_rope_epilogue_matches_the_oracle_on_both_tiles(K, name, BS):
    CK, TK = K
    D, H, KVH, hd = SHAPES[name]
    B, S = BS
    x, w, b, table = _proj_inputs(D, H, KVH, hd, B, S)
    rope = (table, S, hd, H, KVH)
    f0 = CK.fallback_count()
    with tile(CK, "narrow"):
        narrow = CK.gemm(x, w, "nt", rope=rope, bias=b)
    with tile(CK, "wide"):
        wide = CK.gemm(x, w, "nt", rope=rope, bias=b)
    auto = CK.gemm(x, w, "nt", rope=rope, bias=b)
    assert CK.fallback_count() == f0
    ref = TK.gemm(x.float(), w.float(), "nt", rope=rope, bias=b.float())
    assert rel(narrow, ref) < 8e-3
    assert torch.equal(narrow, wide) and torch.equal(narrow, auto)
    # the bias went in before the rotation: against the bias-free epilogue, the difference is the rotated bias
    plain = CK.gemm(x, w, "nt", rope=rope)
    shift = TK.rope_(b.float().expand(B * S, -1).clone(), table, S, H, KVH, hd)
    assert rel(narrow.float() - plain.float(), shift) < 2e-2


def test_unfused_small_m_path_adds_the_bias_before_rope(K):
    """Fewer than 256 rows: the GEMM (bias in the residual epilogue) and the stand-alone RoPE kernel."""
    CK, TK = K
    D, H, KVH, hd = SHAPES["0.5b"]
    x, w, b, table = _proj_inputs(D, H, KVH, hd, 1, 64, seed=3)
    n0, f0 = CK.launch_count(), CK.fallback_count()
    y = CK.gemm(x, w, "nt", rope=(table, 64, hd, H, KVH), bias=b)
    assert CK.launch_count() - n0 == 2 and CK.fallback_count() == f0
    ref = TK.gemm(x.float(), w.float(), "nt", rope=(table, 64, hd, H, KVH), bias=b.float())
    assert rel(y, ref) < 8e-3


def _table(tensors):
    return torch.tensor([t.data_ptr() for t in tensors], dtype=torch.int64, device=DEV)


@pytest.mark.parametrize("dependent", [True, False])
def test_fused_all_gather_build_gives_the_same_bits(K, dependent):
    """The all-gather build of the epilogue (the multi-GPU QKV projection), driven from a table of two local 'peer'
    shards: the gathered buffer is exact and the output equals the single-GPU launch bit for bit."""
    CK, _ = K
    D, H, KVH, hd = SHAPES["1.5b"]
    N, B, S, W = (H + 2 * KVH) * hd, 2, 512, 2
    x, w_ref, b, table = _proj_inputs(D, H, KVH, hd, B, S, seed=5)
    total = (N * D + 65536) // (W * 64) * (W * 64)
    n = total // W
    flat = torch.zeros(total, dtype=torch.bfloat16, device=DEV)
    flat[:N * D] = w_ref.reshape(-1)
    shards = [flat[i * n:(i + 1) * n].clone() for i in range(W)]
    with tile(CK, "narrow"):
        want = CK.gemm(x, w_ref, "nt", rope=(table, S, hd, H, KVH), bias=b)
    for r in (0, W - 1):
        full = torch.zeros(total, dtype=torch.bfloat16, device=DEV)
        flags = torch.zeros((total * 2 + 65535) // 65536, dtype=torch.int32, device=DEV)
        wm = (full if dependent else flat)[:N * D].view(N, D)
        y = torch.empty(B * S, N, dtype=torch.bfloat16, device=DEV)
        CK._C.gemm_ag(x, wm, y, 0, 8, None, _table(shards), full, n * 2, 0, total * 2, W, r, flags, 1, dependent,
                      rope_table=table, rope_S=S, rope_hd=hd, rope_cols=(H + KVH) * hd, bias=b)
        torch.cuda.synchronize()
        assert torch.equal(full, flat)
        assert torch.equal(y, want)


# ------------------------------------------------------------------------------------------------- bias_grad
@pytest.mark.parametrize("T,N", [(8192, 1152), (8191, 1152), (4097, 4608), (33, 4608), (1, 1152), (777, 8)])
def test_bias_grad_matches_an_fp64_column_sum_and_is_deterministic(K, T, N):
    CK, _ = K
    g = torch.Generator(device=DEV).manual_seed(T + N)
    dy = torch.randn(T, N, device=DEV, generator=g).to(torch.bfloat16)
    f0, n0 = CK.fallback_count(), CK.launch_count()
    db = CK.bias_grad(dy)
    again = CK.bias_grad(dy)
    assert CK.fallback_count() == f0 and CK.launch_count() - n0 == 4
    assert db.dtype == torch.float32 and db.shape == (N,)
    ref = dy.double().sum(0)
    assert (db.double() - ref).abs().max().item() < 1e-5 * T ** 0.5 + 1e-6 * ref.abs().max().item()
    assert torch.equal(db, again)


# ------------------------------------------------------------------------------------------------- the op
def _node(path, H, KVH, hd, doc):
    from fms_fsdp_b200.ops import set_kernel_path
    B, S, D = 2, 512, H * 64
    g = torch.Generator(device=DEV).manual_seed(7)
    N = (H + 2 * KVH) * hd
    h = (torch.randn(B, S, D, device=DEV, generator=g)).to(torch.bfloat16).requires_grad_()
    w = (torch.randn(N, D, device=DEV, generator=g) * D ** -0.5).to(torch.bfloat16).requires_grad_()
    b = torch.randn(N, device=DEV, generator=g).to(torch.bfloat16).requires_grad_()
    table = ops.torch_kernels.rope_table(S, hd, 1e6, device=DEV)
    do = torch.randn(B, S, H * hd, device=DEV, generator=g).to(torch.bfloat16)
    seg = None
    if doc:
        tok = torch.full((B, S), 5, device=DEV)
        tok[0, [63, 200, 201]] = 1
        tok[1, [128, 400]] = 1
        seg = ops.document_segments(tok, 1)
    set_kernel_path(path)
    try:
        o = ops.qkv_attention(h, w, table, H, KVH, hd, doc=seg, qkv_bias=b)
        grads = torch.autograd.grad(o, (h, w, b), do)
    finally:
        set_kernel_path("auto")
    return o, grads


@pytest.mark.parametrize("doc", [False, True])
@pytest.mark.parametrize("H,KVH,hd", [(14, 2, 64), (28, 4, 128)])     # GQA groups of 7
def test_qkv_attention_with_bias_matches_the_aten_path(K, H, KVH, hd, doc):
    CK, _ = K
    f0, n0 = CK.fallback_count(), CK.launch_count()
    o, grads = _node("fused", H, KVH, hd, doc)
    # forward: GEMM + attention; backward: attention, bias_grad (2), dgrad, wgrad
    assert CK.fallback_count() == f0 and CK.launch_count() - n0 >= 7
    o_ref, grads_ref = _node("torch", H, KVH, hd, doc)
    assert rel(o, o_ref) < 2e-2
    for name, a, r in zip(("dh", "dw", "db"), grads, grads_ref):
        assert rel(a, r) < 3e-2, name
    if doc:   # the mask reached the node
        o_plain, _ = _node("fused", H, KVH, hd, False)
        assert rel(o, o_plain) > 5e-2


def test_engine_step_qwen25_shape_fused_matches_aten_path():
    """A 2-layer model with the Qwen2.5-1.5B block (D 1536, 12 / 2 heads of 128, F 8960, q / k / v biases): two optimizer
    steps on the sm_90a kernels against the ATen path, with no fallback on the kernel path."""
    from fms_fsdp_b200.models.llama import LLaMA
    from fms_fsdp_b200.ops import cuda_kernels as CK
    from fms_fsdp_b200.ops import set_kernel_path
    from fms_fsdp_b200.parallel import ShardedAdamW, ShardedModel
    from fms_fsdp_b200.policies import bfSixteen
    from fms_fsdp_b200.utils.config_utils import get_model_config

    def run(path):
        set_kernel_path(path)
        torch.manual_seed(0); torch.cuda.manual_seed(0)
        cfg = get_model_config("qwen2.5_1.5b")
        cfg.nlayers, cfg.src_vocab_size = 2, 32768
        with torch.device("meta"):
            m = LLaMA(cfg)
        eng = ShardedModel(m, mixed_precision=bfSixteen, device=torch.device("cuda", 0))
        opt = ShardedAdamW(eng, lr=1e-3)
        x = torch.randint(0, cfg.src_vocab_size, (2, 1024), generator=torch.Generator().manual_seed(3)).cuda()
        out = []
        for _ in range(2):
            l = eng.forward_backward(x, x); gn = eng.clip_grad_norm_(1.0); opt.step(); out.append((l.item(), gn.item()))
        bias = eng.full_state_dict()["layers.0.attn.in_proj.qkv_fused.bias"].float().cpu()
        return out, bias
    try:
        f0 = CK.fallback_count()
        fused, bf = run("fused")
        assert CK.fallback_count() == f0
        aten, ba = run("torch")
    finally:
        set_kernel_path("auto")
    for (lf, gf), (la, ga) in zip(fused, aten):
        assert abs(lf - la) < 2e-2 * abs(la) and abs(gf - ga) < 5e-2 * abs(ga)
    assert bf.abs().max() > 0                                  # the zero-initialised biases were trained
    # AdamW moves every element by about lr per step whatever the size of its gradient, so an element whose gradient is
    # near zero may step the other way on the two paths; nearly all elements must agree to a small part of the step
    d = (bf - ba).abs()
    assert d.median() < 1e-4 and (d < 2e-4).float().mean() > 0.95
