"""CPU tier of the Llama step's elementwise, loss and optimizer kernels (csrc/elementwise.cu): the ATen oracles in
``ops/torch_kernels.py`` are pinned in float64 to autograd or to first principles, and every probe of
``tests/test_llama_kernels_gpu.py`` is shown to fail on a plausible kernel bug by at least 10x its tolerance.

Errors are max-abs over the reference's max-abs (row by row for [M, D] outputs), as on the GPU.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from fms_fsdp_b200.ops import torch_kernels as TK

F64 = torch.float64
# tolerances of tests/test_llama_kernels_gpu.py
TOL_RMS_DW = 1.2e-6
TOL_ROPE = 1.2e-2
TOL_CE_DH = 3.5e-2
TOL_ADAMW = 2.2e-3
EMB_ULPS = 1.0


def rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).abs().max() / b.abs().max().clamp(min=1e-300)).item()


def gen(seed):
    return torch.Generator().manual_seed(seed)


def zipf_tokens(V, M, seed):
    """M tokens drawn with probability 1 / rank over V ids, as in natural text; shared with the GPU tests."""
    p = 1.0 / torch.arange(1, V + 1, dtype=F64)
    return torch.multinomial(p, M, replacement=True, generator=gen(seed))


def bf16_ulps(a, ref):
    """max over elements of |a - round_bf16(ref)| in units of the bf16 ulp of round_bf16(ref)."""
    r = ref.double().to(torch.bfloat16).double()
    e = torch.floor(torch.log2(r.abs().clamp(min=2.0 ** -126)))
    return ((a.double() - r).abs() / torch.exp2(e - 7)).max().item()


# ------------------------------------------------------------------------------------------ RMSNorm
def test_rmsnorm_oracle_is_autograd_in_fp64():
    g = gen(0)
    x = torch.randn(37, 96, dtype=F64, generator=g)
    x[3] *= 1e3
    x[5] *= 1e-4
    w = 1 + 0.1 * torch.randn(96, dtype=F64, generator=g)
    dy, dres = torch.randn(37, 96, dtype=F64, generator=g), torch.randn(37, 96, dtype=F64, generator=g)
    y, rstd = TK.rmsnorm_fwd(x, w, 1e-5)
    assert y.dtype == F64 and rstd.dtype == F64
    xl, wl = x.clone().requires_grad_(), w.clone().requires_grad_()
    ref = xl * torch.rsqrt(xl.pow(2).mean(-1, keepdim=True) + 1e-5) * wl
    torch.testing.assert_close(y, ref.detach(), rtol=1e-13, atol=0)
    gx, gw = torch.autograd.grad(ref, (xl, wl), dy)
    dx, dw = TK.rmsnorm_bwd(dy, x, w, rstd)
    torch.testing.assert_close(dx, gx, rtol=1e-11, atol=1e-13)
    torch.testing.assert_close(dw, gw, rtol=1e-11, atol=1e-13)
    dx2, _ = TK.rmsnorm_bwd(dy, x, w, rstd, dres)
    torch.testing.assert_close(dx2, gx + dres, rtol=1e-11, atol=1e-13)


def test_guard_rmsnorm_dw_with_one_row_per_cta_fails_the_gpu_probe():
    """The GPU probe runs M = 8192 on 528 CTAs: a dw that kept only each CTA's first row is far off."""
    M, D, grid = 8192, 64, 528
    g = gen(1)
    x, dy = torch.randn(M, D, dtype=F64, generator=g), torch.randn(M, D, dtype=F64, generator=g)
    w = torch.ones(D, dtype=F64)
    _, rstd = TK.rmsnorm_fwd(x, w, 1e-5)
    _, dw = TK.rmsnorm_bwd(dy, x, w, rstd)
    _, dw_first = TK.rmsnorm_bwd(dy[:grid], x[:grid], w, rstd[:grid])
    assert rel(dw_first, dw) >= 10 * TOL_RMS_DW


# ------------------------------------------------------------------------------------------- SwiGLU
@pytest.mark.parametrize("gate_first", [True, False])
def test_swiglu_oracle_is_autograd_in_fp64_with_saturated_gates(gate_first):
    g = gen(2)
    F_ = 24
    gu = 3 * torch.randn(16, 2 * F_, dtype=F64, generator=g)
    gu[0], gu[1], gu[2] = 0.0, 80.0, -80.0         # silu(0) = 0; exp(-g) overflows fp32 / the sigmoid saturates
    ds = torch.randn(16, F_, dtype=F64, generator=g)
    leaf = gu.clone().requires_grad_()
    a, b = leaf[:, :F_], leaf[:, F_:]
    gate, up = (a, b) if gate_first else (b, a)
    ref = F.silu(gate) * up
    torch.testing.assert_close(TK.swiglu_fwd(gu, gate_first), ref.detach(), rtol=1e-13, atol=0)
    (grad,) = torch.autograd.grad(ref, leaf, ds)
    torch.testing.assert_close(TK.swiglu_bwd(ds, gu, gate_first), grad, rtol=1e-12, atol=1e-300)


# ------------------------------------------------------------------------------------ cross-entropy
def _labels(M, V, g, ignored=0.2):
    lab = torch.randint(0, V, (M,), generator=g)
    lab[torch.rand(M, generator=g) < ignored] = -100
    lab[1], lab[2] = 0, V - 1
    return lab


def test_ce_gradient_is_autograd_of_the_loss_and_valid_rows_sum_to_zero():
    g = gen(3)
    M, V = 40, 50
    logits = 30 * torch.randn(M, V, dtype=F64, generator=g)
    lab = _labels(M, V, g)
    loss, d = TK.cross_entropy_fwd_bwd(logits, lab)
    leaf = logits.clone().requires_grad_()
    ref = F.cross_entropy(leaf, lab, ignore_index=-100)
    (grad,) = torch.autograd.grad(ref, leaf)
    assert loss.dtype == F64 and d.dtype == F64
    torch.testing.assert_close(loss, ref.detach(), rtol=1e-13, atol=0)
    torch.testing.assert_close(d, grad, rtol=1e-11, atol=1e-15)
    valid = lab != -100
    assert d[valid].sum(-1).abs().max() < 1e-15 and not d[~valid].any()


@pytest.mark.parametrize("chunk_rows", [1, 7, 16, 50, 64])
def test_linear_ce_is_the_same_for_every_chunk_size_and_accumulates(chunk_rows):
    g = gen(4)
    M, D, V = 50, 12, 40
    h, w = torch.randn(M, D, dtype=F64, generator=g), torch.randn(V, D, dtype=F64, generator=g)
    lab = _labels(M, V, g)
    lab[16:32] = -100                                               # one whole 16-row chunk ignored
    dw = torch.empty(V, D, dtype=F64)
    loss, dh = TK.linear_ce_fwd_bwd(h, w, lab, dw, chunk_rows=chunk_rows)
    hl, wl = h.clone().requires_grad_(), w.clone().requires_grad_()
    ref = F.cross_entropy(hl @ wl.t(), lab, ignore_index=-100)
    gh, gw = torch.autograd.grad(ref, (hl, wl))
    torch.testing.assert_close(loss, ref.detach(), rtol=1e-13, atol=0)
    torch.testing.assert_close(dh, gh, rtol=1e-11, atol=1e-15)
    torch.testing.assert_close(dw, gw, rtol=1e-11, atol=1e-15)
    base = torch.randn(V, D, dtype=F64, generator=g)
    acc = base.clone()
    TK.linear_ce_fwd_bwd(h, w, lab, acc, chunk_rows=chunk_rows, accumulate=True)
    torch.testing.assert_close(acc, base + gw, rtol=1e-11, atol=1e-15)


def test_all_ignored_batch_gives_zero_loss_and_zero_gradients():
    g = gen(5)
    h, w = torch.randn(24, 8, dtype=F64, generator=g), torch.randn(16, 8, dtype=F64, generator=g)
    lab = torch.full((24,), -100)
    dw = torch.full((16, 8), float("nan"), dtype=F64)
    loss, dh = TK.linear_ce_fwd_bwd(h, w, lab, dw, chunk_rows=10)
    assert loss.item() == 0 and not dh.any() and not dw.any()
    loss, d = TK.cross_entropy_fwd_bwd(h @ w.t(), lab)
    assert loss.item() == 0 and not d.any() and not d.isnan().any()


def test_guard_ce_with_n_valid_counted_per_chunk_fails_the_gpu_probe():
    """The GPU probe's 20 % ignored, 3000-row chunks of M = 8192: the mean taken per chunk scales dh by the wrong count."""
    g = gen(6)
    M, D, V, C = 8192, 16, 64, 3000
    h, w = torch.randn(M, D, dtype=F64, generator=g), torch.randn(V, D, dtype=F64, generator=g)
    lab = _labels(M, V, g)
    _, dh = TK.linear_ce_fwd_bwd(h, w, lab, torch.empty(V, D, dtype=F64), chunk_rows=C)
    per_chunk = torch.cat([TK.cross_entropy_fwd_bwd(h[s:s + C] @ w.t(), lab[s:s + C])[1] @ w for s in range(0, M, C)])
    assert rel(per_chunk, dh) >= 10 * TOL_CE_DH


# -------------------------------------------------------------------------------------------- AdamW
@pytest.mark.parametrize("wd", [0.0, 0.1])
def test_adamw_oracle_matches_torch_optim_over_ten_steps(wd):
    g = gen(7)
    n = 64
    p0 = torch.randn(n, dtype=F64, generator=g)
    master, m, v = p0.clone(), torch.zeros(n, dtype=F64), torch.zeros(n, dtype=F64)
    ref = torch.nn.Parameter(p0.clone())
    opt = torch.optim.AdamW([ref], lr=1.0, betas=(0.9, 0.95), eps=1e-8, weight_decay=wd)
    scale = torch.tensor(0.37, dtype=F64)                         # the clip coefficient
    for step in range(1, 11):
        lr = 1e-3 * (1 + step) / 2                                  # warm-up-like schedule
        grad = torch.randn(n, dtype=F64, generator=g)
        grad[:8] = 0                                                # never a gradient
        if step == 4:
            grad.zero_()                                            # a step without gradient
        TK.adamw_step(master, grad, m, v, None, lr, 0.9, 0.95, 1e-8, wd, step, grad_scale=scale)
        opt.param_groups[0]["lr"] = lr
        ref.grad = grad * scale
        opt.step()
        torch.testing.assert_close(master, ref.detach(), rtol=1e-12, atol=1e-15)
    state = opt.state[ref]
    torch.testing.assert_close(m, state["exp_avg"], rtol=1e-12, atol=1e-18)
    torch.testing.assert_close(v, state["exp_avg_sq"], rtol=1e-12, atol=1e-18)


def test_guard_adamw_with_bias_correction_one_step_off_fails_the_gpu_probe():
    g = gen(8)
    n = 4096
    p0 = torch.randn(n, dtype=F64, generator=g)
    grads = [torch.randn(n, dtype=F64, generator=g) for _ in range(10)]

    def run(off):
        p, m, v = p0.clone(), torch.zeros(n, dtype=F64), torch.zeros(n, dtype=F64)
        for k, gr in enumerate(grads, 1):
            TK.adamw_step(p, gr, m, v, None, 1e-3, 0.9, 0.95, 1e-8, 0.1, k + off)
        return p - p0

    assert rel(run(1), run(0)) >= 10 * TOL_ADAMW


# --------------------------------------------------------------------------------------------- RoPE
def _table64(S, rot, theta=10000.0):
    """[S, rot/2, 2] (cos, sin) computed in float64, so a rotation and its inverse cancel to float64 rounding."""
    inv = theta ** (-torch.arange(0, rot, 2, dtype=F64) / rot)
    ang = torch.outer(torch.arange(S, dtype=F64), inv)
    return torch.stack([ang.cos(), ang.sin()], -1)


def _qkv(M, H, KVH, hd, seed):
    return torch.randn(M, (H + 2 * KVH) * hd, dtype=F64, generator=gen(seed))


@pytest.mark.parametrize("interleaved", [True, False])
@pytest.mark.parametrize("rot", [64, 32, 48])
def test_rope_then_its_inverse_is_the_identity(interleaved, rot):
    S, H, KVH, hd = 20, 4, 2, 64
    table = _table64(S + 7, rot)
    x = _qkv(2 * S, H, KVH, hd, 9)
    y = TK.rope_(x.clone(), table, S, H, KVH, hd, rot, pos_offset=7, interleaved=interleaved)
    assert rel(y, x) > 0.1
    back = TK.rope_(y.clone(), table, S, H, KVH, hd, rot, inverse=True, pos_offset=7, interleaved=interleaved)
    torch.testing.assert_close(back, x, rtol=1e-13, atol=1e-13)


def test_rope_half_split_pairs_are_the_interleaved_rotation_of_the_permuted_head():
    S, H, KVH, hd, rot = 16, 2, 1, 64, 48
    table = _table64(S, rot)
    x = _qkv(S, H, KVH, hd, 10)
    perm = torch.arange(hd)
    perm[:rot] = torch.stack([torch.arange(rot // 2), torch.arange(rot // 2) + rot // 2], -1).reshape(-1)
    cols = (torch.arange(H + 2 * KVH)[:, None] * hd + perm[None]).reshape(-1)   # (i, i + rot/2) -> (2i, 2i + 1)
    half = TK.rope_(x.clone(), table, S, H, KVH, hd, rot, interleaved=False)
    inter = TK.rope_(x[:, cols].clone(), table, S, H, KVH, hd, rot, interleaved=True)
    torch.testing.assert_close(half[:, cols], inter, rtol=0, atol=0)


@pytest.mark.parametrize("bug", ["no_pos_offset", "restart_per_chunk"])
def test_guard_rope_position_bugs_fail_the_gpu_probe(bug):
    """The GPU probe: B = 2 sequences of S = 4096 at pos_offset 1000 (the table is fp32, the math float64)."""
    S, H, KVH, hd, off = 4096, 2, 1, 64, 1000
    table = TK.rope_table(S + off, hd, 500000.0)
    x = _qkv(2 * S, H, KVH, hd, 11)
    ref = TK.rope_(x.clone(), table, S, H, KVH, hd, pos_offset=off)
    if bug == "no_pos_offset":
        bad = TK.rope_(x.clone(), table, S, H, KVH, hd)
    else:                                                       # positions restart every 1024 rows
        bad = TK.rope_(x.clone(), table, 1024, H, KVH, hd, pos_offset=off)
    assert rel(bad, ref) >= 10 * TOL_ROPE


# ---------------------------------------------------------------------------------------- embedding
def test_embedding_oracle_sums_in_fp64_for_fp64_and_rounds_bf16_once():
    V, D, M = 300, 16, 2000
    tok = zipf_tokens(V, M, 12)
    dx = torch.randn(M, D, dtype=F64, generator=gen(13))
    exact = torch.zeros(V, D, dtype=F64).index_add_(0, tok, dx)
    out = torch.full((V, D), float("nan"), dtype=F64)
    torch.testing.assert_close(TK.embedding_bwd(dx, tok, out), exact, rtol=1e-13, atol=1e-13)
    base = torch.randn(V, D, generator=gen(14)).to(torch.bfloat16)
    dxb = dx.to(torch.bfloat16)
    ref = base.double().index_add_(0, tok, dxb.double())
    acc = TK.embedding_bwd(dxb, tok.int(), base.clone(), accumulate=True)
    assert bf16_ulps(acc, ref) <= 1.0
    fresh = TK.embedding_bwd(dxb, tok, torch.empty(V, D, dtype=torch.bfloat16))
    assert bf16_ulps(fresh, torch.zeros(V, D, dtype=F64).index_add_(0, tok, dxb.double())) <= 1.0


def emulate_bf16_atomics(dx, tok, V):
    """Every add rounded to bf16, as ``atomicAdd(__nv_bfloat162*)`` does: the k-th occurrences of all tokens are added in
    round k (one order the atomics can take)."""
    M, D = dx.shape
    srt, order = torch.sort(tok, stable=True)
    start = torch.searchsorted(srt, srt)
    rank = torch.empty(M, dtype=torch.long)
    rank[order] = torch.arange(M) - start
    acc = torch.zeros(V, D, dtype=torch.bfloat16)
    for k in range(int(rank.max()) + 1):
        sel = rank == k
        t = tok[sel]
        acc[t] = (acc[t].float() + dx[sel].float()).to(torch.bfloat16)
    return acc


def test_guard_per_add_bf16_rounding_fails_the_embedding_probe():
    """The Zipf stream of the GPU probe (V 32000, M 8192): rounding every add to bf16 is many ulps off, where the kernel
    must stay within one."""
    V, D, M = 32000, 256, 8192
    tok = zipf_tokens(V, M, 15)
    dx = (1e-3 * torch.randn(M, D, generator=gen(16))).to(torch.bfloat16)
    ref = torch.zeros(V, D, dtype=F64).index_add_(0, tok, dx.double())
    bad = emulate_bf16_atomics(dx, tok, V)
    ulps = bf16_ulps(bad, ref)
    print(f"MEASURE per-add bf16 emulation: {ulps:.0f} ulps, max-abs/max-abs {rel(bad, ref):.2e}")
    assert ulps >= 10 * EMB_ULPS
    assert bf16_ulps(TK.embedding_bwd(dx, tok, torch.empty(V, D, dtype=torch.bfloat16)), ref) <= EMB_ULPS
    assert math.isfinite(ulps)
