"""z-losses on the GPU: the kernels of ``csrc/losses_sm90.cu`` against float64 on the same bf16-rounded logits at
production vocabularies, run-to-run bit reproducibility, the c = 0 head against the plain fused cross-entropy, and an
engine step with both losses against the ATen path.  ``tests/test_sass.py`` checks their SASS."""

import pytest
import torch

from fms_fsdp_b200 import ops
from fms_fsdp_b200.ops import torch_kernels as tk
from test_z_loss_cpu import GPU_TOL, rel

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ck():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from fms_fsdp_b200.ops import cuda_kernels
    assert cuda_kernels._C.__file__.endswith("_C.so")
    return cuda_kernels


def _head(M, D, V, amp, seed=0):
    """bf16 h, w whose logits have a standard deviation of about ``amp`` (amp 10: values out to +-40), 10 % ignored."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    h = torch.randn(M, D, generator=g, device="cuda").bfloat16()
    w = (torch.randn(V, D, generator=g, device="cuda") * (amp / D ** 0.5)).bfloat16()
    labels = torch.randint(0, V, (M,), generator=g, device="cuda")
    labels[torch.rand(M, generator=g, device="cuda") < 0.1] = -100
    return h, w, labels


def _fp64_reference(ck, h, w, labels, c, rows=1024):
    """(ce, z, dh, dw) in float64 from the bf16 logits the kernel sees (our GEMM, bf16 out), row block by row block."""
    M, V = h.shape[0], w.shape[0]
    ok = labels != -100
    n = ok.sum().clamp(min=1).double()
    ce = z = 0.0
    dh = torch.empty(M, h.shape[1], dtype=torch.float64, device="cuda")
    dw = torch.zeros(V, h.shape[1], dtype=torch.float64, device="cuda")
    w64 = w.double()
    for s in range(0, M, rows):
        e = min(M, s + rows)
        lg = ck.gemm(h[s:e], w, "nt").double()
        c_s, z_s, G = tk._ce_z_grad(lg, labels[s:e], ok[s:e], n, c)
        ce, z = ce + c_s, z + z_s
        dh[s:e] = G @ w64
        dw += G.t() @ h[s:e].double()
        del lg, G
    return ce / n, z / n, dh, dw


def _run(h, w, labels, c):
    hl, wl = h.clone().requires_grad_(), w.clone().requires_grad_()
    ce, z = ops.linear_cross_entropy_z(hl, wl, labels, c)
    ce.backward()
    return ce.detach(), z, hl.grad, wl.grad


HEAD = [(8192, 4096, 32000, 1.0), (4096, 4096, 128256, 1.0), (8192, 896, 151936, 1.0), (8, 896, 151936, 1.0),
        (1000, 896, 32000, 1.0), (2048, 896, 32000, 10.0), (2048, 4096, 128256, 10.0)]


@pytest.mark.parametrize("M,D,V,amp", HEAD)
@pytest.mark.parametrize("c", [1e-4, 1e-2])
def test_head_matches_fp64_and_reruns_bit_identically(ck, M, D, V, amp, c):
    h, w, labels = _head(M, D, V, amp)
    ce, z, dh, dw = _run(h, w, labels, c)
    rce, rz, rdh, rdw = _fp64_reference(ck, h, w, labels, c)
    err = dict(ce=abs(float(ce) / float(rce) - 1), z=abs(float(z) / float(rz) - 1), dh=rel(dh, rdh), dw=rel(dw, rdw))
    print(f"[z-loss head] M {M} D {D} V {V} amp {amp} c {c}: " + " ".join(f"{k} {v:.2e}" for k, v in err.items()))
    assert err["ce"] < GPU_TOL["stat"] and err["z"] < GPU_TOL["stat"], err
    assert err["dh"] < GPU_TOL["grad"] and err["dw"] < GPU_TOL["grad"], err
    again = _run(h, w, labels, c)
    for a, b in zip((ce, z, dh, dw), again):
        assert torch.equal(a, b)


@pytest.mark.parametrize("V,amp", [(32000, 10.0), (151936, 10.0)])
def test_logit_gradient_and_its_z_part_match_fp64(ck, V, amp):
    """The materialised-logits entry at logits out to +-40: the whole gradient, and G(c) - G(0) alone at c = 1e-2."""
    M, D, c = 2048, 896, 1e-2
    h, w, labels = _head(M, D, V, amp, seed=1)
    lg = ck.gemm(h, w, "nt")
    ce, z, G = ck.cross_entropy_z_fwd_bwd(lg, labels, c)
    rce, rz, RG = tk.cross_entropy_z_fwd_bwd(lg.double(), labels, c)
    RG0 = tk.cross_entropy_z_fwd_bwd(lg.double(), labels, 0.0)[2]
    err = dict(ce=abs(float(ce) / float(rce) - 1), z=abs(float(z) / float(rz) - 1), grad=rel(G, RG),
               zpart=rel(G.double() - RG0, RG - RG0))
    print(f"[z-loss logits] V {V} amp {amp}: " + " ".join(f"{k} {v:.2e}" for k, v in err.items()))
    assert err["ce"] < GPU_TOL["stat"] and err["z"] < GPU_TOL["stat"], err
    assert err["grad"] < GPU_TOL["grad"] and err["zpart"] < GPU_TOL["zpart"], err
    assert float(lg.float().abs().max()) > 30


def test_zero_coefficient_gradient_is_bitwise_the_plain_head(ck):
    h, w, labels = _head(4096, 4096, 32000, 1.0)
    ce, z, dh, dw = _run(h, w, labels, 0.0)
    hl, wl = h.clone().requires_grad_(), w.clone().requires_grad_()
    ce0 = ops.linear_cross_entropy(hl, wl, labels)
    ce0.backward()
    assert torch.equal(dh, hl.grad) and torch.equal(dw, wl.grad)
    # the plain head sums its loss with float atomics (order varies run to run), the z entry in a fixed order
    assert float(ce) == pytest.approx(float(ce0), rel=1e-5) and float(z) > 0


@pytest.mark.parametrize("T,E,k", [(8192, 128, 8), (8192, 8, 2), (1000, 8, 2)])
def test_router_kernels_match_fp64_and_rerun_bit_identically(ck, T, E, k):
    g = torch.Generator(device="cuda").manual_seed(T + E)
    logits = torch.randn(T, E, generator=g, device="cuda") * 2
    ids, wts, probs = ck.moe_route(logits, k, True)
    plan, _ = ck.moe_plan(ids, probs)
    dwr = torch.randn(T, k, generator=g, device="cuda")
    scale = 2 * 1e-2 / T
    lse, z = ck.router_z_fwd(logits)
    rlse, rz = tk.router_z_fwd(logits.double())
    assert rel(lse, rlse) < 1e-6 and abs(float(z) / float(rz) - 1) < GPU_TOL["stat"]
    rpart = tk.router_z_bwd(torch.zeros(T, E, dtype=torch.float64, device="cuda"), torch.softmax(logits.double(), -1),
                            rlse, scale)
    # the z part alone (added to a zero gradient: one bf16 rounding), then on top of the routing gradient
    zpart = ck.router_z_bwd(torch.zeros(T, E, dtype=torch.bfloat16, device="cuda"), probs, lse, scale)
    err = rel(zpart, rpart)
    d0 = ck.moe_route_bwd(probs, ids, wts, dwr / T, plan, True, 0.0)
    dl = ck.router_z_bwd(d0.clone(), probs, lse, scale)
    whole = rel(dl, d0.double() + rpart)
    print(f"[router z] T {T} E {E} k {k}: lse {rel(lse, rlse):.2e} z {abs(float(z) / float(rz) - 1):.2e} "
          f"zpart {err:.2e} whole {whole:.2e}")
    assert err < GPU_TOL["router_zpart"] and whole < GPU_TOL["grad"], (err, whole)
    lse2, z2 = ck.router_z_fwd(logits)
    assert torch.equal(lse, lse2) and torch.equal(z, z2)
    assert torch.equal(dl, ck.router_z_bwd(d0.clone(), probs, lse2, scale))


def _engine_step(cfg, x, steps=2):
    from fms_fsdp_b200.models.llama import LLaMA
    from fms_fsdp_b200.parallel import ShardedAdamW, ShardedModel
    from fms_fsdp_b200.policies import bfSixteen
    torch.manual_seed(0)
    with torch.device("meta"):
        m = LLaMA(cfg)
    eng = ShardedModel(m, sharding_strategy="fsdp", mixed_precision=bfSixteen, device=torch.device("cuda", 0))
    opt = ShardedAdamW(eng, lr=1e-4)
    out = []
    for _ in range(steps):
        loss = eng.forward_backward(x, x)
        out.append((float(loss), float(m.z_loss()), float(m.moe_router_z_loss()), float(eng.clip_grad_norm_(1e9))))
        opt.step()
    return out


def test_engine_step_with_both_losses_at_a_truncated_qwen3_moe_shape_matches_the_aten_path(ck):
    from fms_fsdp_b200.ops import functional as Fn
    from fms_fsdp_b200.utils.config_utils import get_model_config
    cfg = get_model_config("qwen3_moe_30b_a3b")
    cfg.nlayers, cfg.src_vocab_size = 2, 32000
    cfg.z_loss_coef, cfg.moe_router_z_loss_coef = 1e-2, 1e-1        # large enough that a wrong gradient shows
    x = torch.randint(0, 32000, (1, 1024), generator=torch.Generator().manual_seed(0)).cuda()
    ck.reset_fallback_count()
    fused = _engine_step(cfg, x)
    assert ck.fallback_count() == 0
    old = Fn.get_kernel_path()
    Fn.set_kernel_path("torch")
    try:
        ref = _engine_step(cfg, x)
    finally:
        Fn.set_kernel_path(old)
    print(f"[z-loss engine] fused {fused} aten {ref}")
    for a, b in zip(fused, ref):
        assert a[:3] == pytest.approx(b[:3], rel=5e-3), (fused, ref)
        assert a[3] == pytest.approx(b[3], rel=3e-2), (fused, ref)
