"""The Llama step's elementwise, loss and optimizer kernels (csrc/elementwise.cu) on the H100 against float64 references,
at the shapes production runs: RMSNorm with several rows per CTA, RoPE with offsets, partial rotation and GQA, SwiGLU
with saturated gates, the embedding gather and its fixed-order fp32 backward, the fused linear-cross-entropy at real
vocabularies, AdamW and the sum of squares.

Inputs are bf16 (or fp32) as the kernels take them; the references get them in float64 and never round their outputs.
Errors are max-abs over the reference's max-abs, row by row for [M, D] outputs (a row's scale is its own).  Every native
call must launch our kernels and take no ATen fallback, except where a test asserts the counted fallback.
``tests/test_llama_kernels_cpu.py`` pins the references and shows each probe fails on a plausible bug.
"""

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64 = torch.float64

# about 3x the largest error measured on an H100 80GB HBM3 at 700 W (DESIGN.md); tests/test_llama_kernels_cpu.py keeps a
# copy.  bf16 outputs sit near half a bf16 ulp (2^-9 = 2e-3) of their row's largest element.  The CE loss, dh and dw are
# held against the oracle that rounds the logits to bf16 as the kernel stores them; the AdamW update is over the fp32
# master, whose rounding (2^-24 of |p|) is about 1e-3 of a 3e-4 step.
TOL_RMS_Y, TOL_RMS_DX, TOL_RMS_DW, TOL_RSTD = 1.2e-2, 1.2e-2, 1.2e-6, 3e-7
TOL_ROPE = 1.2e-2
TOL_SWIGLU = 1.2e-2
TOL_CE_LOSS, TOL_CE_DH, TOL_CE_DW = 2.5e-5, 3.5e-2, 2.5e-2
TOL_ADAMW, TOL_ADAMW_STATE, TOL_SUMSQ = 2.2e-3, 1e-6, 3e-6
TOL_EMB_F32 = 4e-7
EMB_ULPS = 1.0


@pytest.fixture(scope="module")
def K():
    from fms_fsdp_b200.ops import cuda_kernels as CK
    from fms_fsdp_b200.ops import torch_kernels as TK
    assert CK._C.__file__.endswith("_C.so")
    return CK, TK


class Native:
    """Asserts the block launched our kernels (``launches`` of them when given) and took no ATen fallback."""

    def __init__(self, CK, launches=None):
        self.CK, self.launches = CK, launches

    def __enter__(self):
        self.n0, self.f0 = self.CK.launch_count(), self.CK.fallback_count()
        return self

    def __exit__(self, et, *_):
        if et is None:
            n = self.CK.launch_count() - self.n0
            assert n > 0 if self.launches is None else n == self.launches, n
            assert self.CK.fallback_count() == self.f0, dict(self.CK.FALLBACKS)


def err(a, b):
    a, b = a.double(), b.double()
    return ((a - b).abs().max() / b.abs().max().clamp(min=1e-300)).item()


def err_rows(a, b):
    a, b = a.double(), b.double()
    return ((a - b).abs().amax(-1) / b.abs().amax(-1).clamp(min=1e-300)).max().item()


def check(tag, e, tol):
    print(f"MEASURE {tag}: {e:.2e} tol {tol:.0e}")
    assert e <= tol, (tag, e, tol)


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def randn(*shape, seed, scale=1.0):
    return scale * torch.randn(*shape, device=DEV, generator=gen(seed))


# ------------------------------------------------------------------------------------------ RMSNorm
@pytest.mark.parametrize("M", [1, 7, 528, 529, 792, 793, 8192])
@pytest.mark.parametrize("D", [8, 896, 1536, 2048, 3584, 4096, 5120, 8192])
def test_rmsnorm_fwd_bwd_several_rows_per_cta(K, D, M):
    CK, TK = K
    x = randn(M, D, seed=D + M)
    if M > 2:
        x[1] *= 1e3                                             # |x| ~ 1e3
        x[2] *= 1e-4                                            # mean square below eps
    x = x.bfloat16()
    w = (1 + randn(D, seed=1, scale=0.1)).bfloat16()
    dy, dres = randn(M, D, seed=2).bfloat16(), randn(M, D, seed=3).bfloat16()
    with Native(CK, 1):
        y, rstd = CK.rmsnorm_fwd(x, w, 1e-5)
    with Native(CK, 4):
        dx, dw = CK.rmsnorm_bwd(dy, x, w, rstd)
        dx2, dw2 = CK.rmsnorm_bwd(dy, x, w, rstd, dres)
    yr, rr = TK.rmsnorm_fwd(x.double(), w.double(), 1e-5)
    dxr, dwr = TK.rmsnorm_bwd(dy.double(), x.double(), w.double(), rr)
    check(f"rmsnorm D{D} M{M} y", err_rows(y, yr), TOL_RMS_Y)
    check(f"rmsnorm D{D} M{M} rstd", err(rstd, rr), TOL_RSTD)
    check(f"rmsnorm D{D} M{M} dx", err_rows(dx, dxr), TOL_RMS_DX)
    check(f"rmsnorm D{D} M{M} dx+dres", err_rows(dx2, dxr + dres.double()), TOL_RMS_DX)
    check(f"rmsnorm D{D} M{M} dw", err(dw, dwr), TOL_RMS_DW)
    assert torch.equal(dw, dw2)


def test_rmsnorm_wider_than_8192_takes_the_counted_fallback(K):
    from fms_fsdp_b200 import ops
    CK, TK = K
    M, D = 64, 8200
    x = randn(M, D, seed=4).bfloat16().requires_grad_()
    w = (1 + randn(D, seed=5, scale=0.1)).bfloat16().requires_grad_()
    dy = randn(M, D, seed=6).bfloat16()
    f0 = CK.fallback_count()
    y = ops.rmsnorm(x, w)
    dx, dw = torch.autograd.grad(y, (x, w), dy)
    assert CK.fallback_count() - f0 == 2
    yr, rr = TK.rmsnorm_fwd(x.detach().double(), w.detach().double(), 1e-5)
    dxr, dwr = TK.rmsnorm_bwd(dy.double(), x.detach().double(), w.detach().double(), rr)
    check("rmsnorm D8200 fallback y", err_rows(y, yr), TOL_RMS_Y)
    check("rmsnorm D8200 fallback dx", err_rows(dx, dxr), TOL_RMS_DX)
    check("rmsnorm D8200 fallback dw", err(dw, dwr), TOL_RMS_Y)


# --------------------------------------------------------------------------------------------- RoPE
ROPE = [(32, 8, 128, 128), (32, 8, 128, 64), (32, 8, 128, 96), (28, 4, 128, 128), (28, 4, 128, 96), (12, 2, 64, 64),
        (12, 2, 64, 32)]


@pytest.mark.parametrize("interleaved", [True, False])
@pytest.mark.parametrize("H,KVH,hd,rot", ROPE)
def test_rope_gqa_partial_rotation_and_offset(K, H, KVH, hd, rot, interleaved):
    CK, TK = K
    B, S, off = 2, 4096, 777
    table = TK.rope_table(S + off, rot, 500000.0, device=DEV)
    _rope_case(CK, TK, f"rope H{H}/{KVH} hd{hd} rot{rot} {'inter' if interleaved else 'half'}", table, B, S, H, KVH,
               hd, rot, off, interleaved)


@pytest.mark.parametrize("interleaved", [True, False])
def test_rope_llama3_scaled_table_at_8192(K, interleaved):
    CK, TK = K
    scaling = {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
               "original_max_position_embeddings": 8192}
    table = TK.rope_table(8192, 128, 500000.0, device=DEV, scaling=scaling)
    _rope_case(CK, TK, f"rope llama3 S8192 {'inter' if interleaved else 'half'}", table, 2, 8192, 32, 8, 128, 128, 0,
               interleaved)


def _rope_case(CK, TK, tag, table, B, S, H, KVH, hd, rot, off, interleaved):
    qkv = randn(B * S, (H + 2 * KVH) * hd, seed=hd + rot).bfloat16()
    out = qkv.clone()
    with Native(CK, 1):
        CK.rope_(out, table, S, H, KVH, hd, rot, pos_offset=off, interleaved=interleaved)
    ref = TK.rope_(qkv.double(), table, S, H, KVH, hd, rot, pos_offset=off, interleaved=interleaved)
    nrot = (H + KVH) * hd
    assert torch.equal(out[:, nrot:], qkv[:, nrot:])                         # V heads
    heads = out[:, :nrot].view(-1, H + KVH, hd)
    assert torch.equal(heads[..., rot:], qkv[:, :nrot].view(-1, H + KVH, hd)[..., rot:])   # unrotated tail
    check(tag, err_rows(out[:, :nrot], ref[:, :nrot]), TOL_ROPE)


# ------------------------------------------------------------------------------------------- SwiGLU
@pytest.mark.parametrize("gate_first", [True, False])
@pytest.mark.parametrize("F_", [8, 1408, 4864, 11008, 14336, 18944])
def test_swiglu_fwd_bwd_with_saturated_gates(K, F_, gate_first):
    CK, TK = K
    M = 1001 if F_ == 8 else 8192
    gu = randn(M, 2 * F_, seed=F_, scale=3.0)
    gate = slice(0, F_) if gate_first else slice(F_, 2 * F_)
    g = gu[:, gate]
    g[0], g[1], g[2], g[3] = 0.0, 80.0, -80.0, -30.0           # silu(0); exp(-g) large / the sigmoid saturates
    g[4:, :8] = torch.linspace(-80, 80, 8, device=DEV)
    gu = gu.bfloat16()
    ds = randn(M, F_, seed=F_ + 1).bfloat16()
    with Native(CK, 2):
        s = CK.swiglu_fwd(gu, gate_first)
        dgu = CK.swiglu_bwd(ds, gu, gate_first)
    check(f"swiglu F{F_} gf{int(gate_first)} fwd", err_rows(s, TK.swiglu_fwd(gu.double(), gate_first)), TOL_SWIGLU)
    check(f"swiglu F{F_} gf{int(gate_first)} bwd", err_rows(dgu, TK.swiglu_bwd(ds.double(), gu.double(), gate_first)),
          TOL_SWIGLU)


# ---------------------------------------------------------------------------------------- embedding
@pytest.mark.parametrize("idx", [torch.int32, torch.int64])
@pytest.mark.parametrize("V", [128256, 151936])
def test_embedding_fwd_is_an_exact_gather(K, V, idx):
    CK, _ = K
    D, M = 4096, 8192
    w = randn(V, D, seed=V).bfloat16()
    tok = torch.randint(0, V, (M,), device=DEV, generator=gen(7)).to(idx)
    tok[0], tok[1], tok[-1] = 0, V - 1, V - 1
    with Native(CK, 1):
        y = CK.embedding_fwd(tok, w)
    assert torch.equal(y, w[tok.long()])


def zipf_tokens(V, M, seed):
    """M tokens drawn with probability 1 / rank over V ids, as in natural text (tests/test_llama_kernels_cpu.py)."""
    p = 1.0 / torch.arange(1, V + 1, dtype=F64)
    return torch.multinomial(p, M, replacement=True, generator=torch.Generator().manual_seed(seed)).to(DEV)


def bf16_ulps(a, ref):
    """max over elements of |a - round_bf16(ref)| in bf16 ulps of round_bf16(ref).  Elements whose exact sum cancels to
    below 2^-20 of the largest are held to the ulp at that scale: an fp32 sum cannot resolve them more finely."""
    r = ref.double().to(torch.bfloat16).double()
    floor = 2.0 ** -20 * r.abs().max().item()
    e = torch.floor(torch.log2(r.abs().clamp(min=max(floor, 2.0 ** -126))))
    return ((a.double() - r).abs() / torch.exp2(e - 7)).max().item()


def _stream(kind, V, M):
    if kind == "zipf":
        return zipf_tokens(V, M, 15)
    if kind == "one_token":
        return torch.full((M,), 4321, device=DEV)
    return torch.randint(0, V, (M,), device=DEV, generator=gen(8))


def _emb_launches(M):
    merges = 0
    L = 4096
    while L < M:
        L, merges = 2 * L, merges + 1
    return 3 + merges


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("kind", ["zipf", "one_token", "uniform"])
def test_embedding_bwd_sums_each_row_in_fp32_once_and_deterministically(K, kind, dtype, accumulate):
    CK, _ = K
    V, D, M = 32000, 4096, 8192
    tok = _stream(kind, V, M)
    dx = randn(M, D, seed=9, scale=1e-3).bfloat16()
    base = randn(V, D, seed=10, scale=1e-2).to(dtype) if accumulate else torch.zeros(V, D, device=DEV, dtype=dtype)
    ref = base.double().index_add_(0, tok, dx.double())
    outs = []
    for idx in (torch.int64, torch.int32):
        out = base.clone() if accumulate else torch.full((V, D), float("nan"), device=DEV, dtype=dtype)
        with Native(CK, _emb_launches(M)):
            CK.embedding_bwd(dx, tok.to(idx), out, accumulate=accumulate)
        outs.append(out)
    assert torch.equal(outs[0], outs[1])                                     # the same bits, run to run
    tag = f"embedding_bwd {kind} {str(dtype)[6:]} acc{int(accumulate)}"
    if dtype == torch.bfloat16:
        u = bf16_ulps(outs[0], ref)
        print(f"MEASURE {tag}: {u:.2f} ulps, max-abs/max-abs {err(outs[0], ref):.2e}")
        assert u <= EMB_ULPS, u
    else:
        check(tag, err(outs[0], ref), TOL_EMB_F32)


@pytest.mark.parametrize("M", [1, 4095, 4097, 8191, 20000])
def test_embedding_bwd_sort_and_chunk_edges(K, M):
    """M around the 4096-key sort tile and the 64-key chunks; a narrow D with an unused tail of the column block."""
    CK, _ = K
    V, D = 1000, 1032
    tok = zipf_tokens(V, M, M)
    dx = randn(M, D, seed=11).bfloat16()
    out = torch.zeros(V, D, device=DEV)
    with Native(CK, _emb_launches(M)):
        CK.embedding_bwd(dx, tok, out)
    check(f"embedding_bwd M{M} f32", err(out, torch.zeros(V, D, device=DEV, dtype=F64).index_add_(0, tok, dx.double())),
          TOL_EMB_F32)


def test_embedding_op_writes_into_a_bound_bf16_grad_buffer(K):
    """``ops.embedding`` with the bf16 ``_grad_buf`` the engine binds: the first contribution overwrites it, a second
    (a tied head that wrote the buffer first) adds onto it."""
    from fms_fsdp_b200 import ops
    CK, _ = K
    V, D, M = 32000, 1024, 8192
    tok = zipf_tokens(V, M, 16).view(2, M // 2)
    w = torch.nn.Parameter(randn(V, D, seed=12).bfloat16())
    w._grad_buf = torch.full((V, D), float("nan"), device=DEV, dtype=torch.bfloat16)
    dy = randn(2, M // 2, D, seed=13, scale=1e-3).bfloat16()
    with Native(CK, 1 + _emb_launches(M)):                           # the gather and the backward
        ops.embedding(tok, w).backward(dy)
    assert w.grad is None and w._grad_ready
    ref = torch.zeros(V, D, device=DEV, dtype=F64).index_add_(0, tok.reshape(-1), dy.reshape(M, D).double())
    assert bf16_ulps(w._grad_buf, ref) <= EMB_ULPS
    first = w._grad_buf.clone()
    with Native(CK, 1 + _emb_launches(M)):
        ops.embedding(tok, w).backward(dy)
    assert bf16_ulps(w._grad_buf, first.double().index_add_(0, tok.reshape(-1), dy.reshape(M, D).double())) <= EMB_ULPS


# ------------------------------------------------------------------------------------ cross-entropy
def _ce_ref(h, w, lab, round_logits, ref_rows=1024):
    """float64 (loss, dh, dw) of mean CE(h w^T); ``round_logits`` first rounds the logits to bf16, as the kernel stores
    them."""
    M = h.shape[0]
    hd, wd = h.double(), w.double()
    valid = lab != -100
    n = valid.sum().clamp(min=1).double()
    loss = torch.zeros((), device=DEV, dtype=F64)
    dh = torch.zeros(M, w.shape[1], device=DEV, dtype=F64)
    dw = torch.zeros_like(wd)
    for s in range(0, M, ref_rows):
        e = min(M, s + ref_rows)
        lg = hd[s:e] @ wd.t()
        if round_logits:
            lg = lg.to(torch.bfloat16).double()
        lse = torch.logsumexp(lg, -1)
        ok = valid[s:e]
        safe = lab[s:e].clamp(min=0)
        loss += ((lse - lg.gather(1, safe[:, None])[:, 0]) * ok).sum()
        p = torch.exp(lg - lse[:, None])
        p[torch.arange(e - s, device=DEV), safe] -= 1
        p *= ok[:, None] / n
        dh[s:e] = p @ wd
        dw += p.t() @ hd[s:e]
    return loss / n, dh, dw


# (V, D, M, chunk_rows, ignored fraction, logit std, accumulate)
CE = [(32000, 4096, 8192, 4096, 0.2, 1.0, False), (128256, 4096, 1000, 256, 0.0, 8.0, False),
      (151936, 896, 8192, 3000, 0.2, 1.0, False), (151936, 896, 8, 4096, 0.0, 8.0, False),
      (32000, 896, 1000, 3000, 1.0, 1.0, False), (128256, 896, 8192, 4096, 0.2, 8.0, True),
      (32000, 896, 8192, 3000, "chunk", 8.0, True)]


@pytest.mark.parametrize("V,D,M,chunk,ignored,std,accumulate", CE)
def test_linear_ce_at_production_vocabularies(K, V, D, M, chunk, ignored, std, accumulate):
    CK, _ = K
    h = randn(M, D, seed=V + M).bfloat16()
    w = randn(V, D, seed=D, scale=std / D ** 0.5).bfloat16()                 # logits ~ N(0, std^2), up to ~ +-5 std
    lab = torch.randint(0, V, (M,), device=DEV, generator=gen(17))
    lab[0], lab[-1] = 0, V - 1
    if ignored == "chunk":
        lab[chunk:2 * chunk] = -100                                          # one whole chunk ignored
    elif ignored:
        lab[torch.rand(M, device=DEV, generator=gen(18)) < ignored] = -100
    base = randn(V, D, seed=19, scale=1e-3).bfloat16() if accumulate else None
    dw = base.clone() if accumulate else torch.full((V, D), float("nan"), device=DEV, dtype=torch.bfloat16)
    with Native(CK):
        loss, dh = CK.linear_ce_fwd_bwd(h, w, lab, dw, chunk_rows=chunk, accumulate=accumulate)
    tag = f"linear_ce V{V} D{D} M{M} c{chunk} ign{ignored}"
    if ignored == 1.0:
        assert loss.item() == 0 and not dh.any() and not dw.any()
        return
    for name, rnd in (("fp64 logits", False), ("bf16 logits", True)):
        lr, dhr, dwr = _ce_ref(h, w, lab, rnd)
        if accumulate:
            dwr = dwr + base.double()
        print(f"MEASURE {tag} vs {name}: loss {abs(loss.item() - lr.item()) / lr.item():.2e} dh {err(dh, dhr):.2e} "
              f"dw {err(dw, dwr):.2e}")
        if rnd:
            check(tag + " loss", abs(loss.item() - lr.item()) / lr.item(), TOL_CE_LOSS)
            check(tag + " dh", err(dh, dhr), TOL_CE_DH)
            check(tag + " dw", err(dw, dwr), TOL_CE_DW)


def test_cross_entropy_op_on_explicit_logits(K):
    from fms_fsdp_b200 import ops
    CK, _ = K
    M, V = 1000, 32000
    logits = randn(M, V, seed=20, scale=8.0).bfloat16().requires_grad_()
    lab = torch.randint(0, V, (M,), device=DEV, generator=gen(21))
    lab[::5] = -100
    lab[1], lab[2] = 0, V - 1
    with Native(CK, 2):
        loss = ops.cross_entropy(logits, lab)
    (g,) = torch.autograd.grad(loss, logits)
    leaf = logits.detach().double().requires_grad_()
    ref = torch.nn.functional.cross_entropy(leaf, lab, ignore_index=-100)
    (gr,) = torch.autograd.grad(ref, leaf)
    check("cross_entropy loss", abs(loss.item() - ref.item()) / ref.item(), TOL_CE_LOSS)
    check("cross_entropy dlogits", err_rows(g[lab != -100], gr[lab != -100]), TOL_CE_DH)
    assert not g[lab == -100].any()


# -------------------------------------------------------------------------------------------- AdamW
@pytest.mark.parametrize("wd", [0.0, 0.1])
@pytest.mark.parametrize("scale", [None, 0.37, "1/k"])
@pytest.mark.parametrize("lowp", [False, True])
@pytest.mark.parametrize("gdt", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("n", [4, 12, 1000, 2 ** 20 + 4])
def test_adamw_ten_steps_against_torch_optim_in_fp64(K, n, gdt, lowp, scale, wd):
    CK, TK = K
    p0 = randn(n, seed=n)
    master, m, v = p0.clone(), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    lp = torch.empty(n, device=DEV, dtype=torch.bfloat16) if lowp else None
    ref = torch.nn.Parameter(p0.double())
    opt = torch.optim.AdamW([ref], lr=1.0, betas=(0.9, 0.95), eps=1e-8, weight_decay=wd)
    for k in range(1, 11):
        lr = 3e-4 * k / 10
        g = randn(n, seed=100 + k).to(gdt)
        if k == 4:
            g.zero_()
        sc = None if scale is None else torch.tensor(scale if scale != "1/k" else 1.0 / k, device=DEV)
        with Native(CK, 1):
            CK.adamw_step(master, g, m, v, lp, lr, 0.9, 0.95, 1e-8, wd, k, sc)
        opt.param_groups[0]["lr"] = lr
        ref.grad = g.double() * (1.0 if sc is None else sc.double())
        opt.step()
    tag = f"adamw n{n} {str(gdt)[6:]} lowp{int(lowp)} s{scale} wd{wd}"
    check(tag + " update", err(master - p0, ref.detach() - p0.double()), TOL_ADAMW)
    st = opt.state[ref]
    check(tag + " m", err(m, st["exp_avg"]), TOL_ADAMW_STATE)
    check(tag + " v", err(v, st["exp_avg_sq"]), TOL_ADAMW_STATE)
    if lowp:
        assert torch.equal(lp, master.bfloat16())
    # a late step: the bias corrections are 1 to fp32
    prev, m64, v64 = master.double(), m.double(), v.double()
    want = prev.clone()
    g = randn(n, seed=999).to(gdt)
    with Native(CK, 1):
        CK.adamw_step(master, g, m, v, lp, 1e-3, 0.9, 0.95, 1e-8, wd, 10000)
    TK.adamw_step(want, g, m64, v64, None, 1e-3, 0.9, 0.95, 1e-8, wd, 10000)
    check(tag + " step 10000 update", err(master.double() - prev, want - prev), TOL_ADAMW)
    check(tag + " step 10000 v", err(v, v64), TOL_ADAMW_STATE)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("n", [1, 7, 15, 16, 17, 4095, 2 ** 24 + 3])
def test_sumsq_accumulates_into_out(K, n, dtype):
    CK, _ = K
    x = randn(n, seed=n).to(dtype)
    out = torch.full((), 1.5, device=DEV)
    with Native(CK, 2):
        CK.sumsq(x, out)
        CK.sumsq(x, out)
    ref = 1.5 + 2 * x.double().pow(2).sum()
    check(f"sumsq n{n} {str(dtype)[6:]}", abs(out.item() - ref.item()) / ref.item(), TOL_SUMSQ)


def test_sumsq_misaligned_view_takes_the_counted_fallback(K):
    CK, _ = K
    x = randn(4097, seed=22).bfloat16()[1:]
    assert x.data_ptr() % 16
    f0 = CK.fallback_count()
    s = CK.sumsq(x)
    assert CK.fallback_count() == f0 + 1
    ref = x.double().pow(2).sum()
    check("sumsq misaligned", abs(s.item() - ref.item()) / ref.item(), TOL_SUMSQ)
