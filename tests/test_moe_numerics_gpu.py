"""GPU tier of the per-row mixture-of-experts check: the sm_90a routing, plan, permute / combine and grouped GEMM
kernels (and the whole ``ops.moe_mlp`` node) against the float64 reference of ``tests/moe_reference.py``, row by row, at
the Qwen3-30B-A3B and Mixtral 8x7B shapes and on a crafted plan with every segment edge; every grouped GEMM mode
against the 128 x 128 dense GEMM on each expert's rows, bit for bit; the exact invariants of the permuted buffers.
Each case prints its worst per-row ratio as a fraction of its tolerance ("MEASURE ... x tol") and the allocator peak.
The tolerances come from the CPU rounding emulation (tests/test_moe_numerics_cpu.py), not from a GPU run.  The float64
references run on the GPU one expert at a time.
"""
import contextlib
import time

import pytest
import torch

import moe_reference as MR

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64, BF16 = torch.float64, torch.bfloat16
QWEN3 = dict(T=8192, D=2048, E=128, k=8, F=768, aux=0.001)
MIXTRAL = dict(T=4096, D=4096, E=8, k=2, F=14336, aux=0.02)
CRAFTED = [0, 1, 63, 64, 65, 127, 128, 129, 0, 0, 256, 8448, 2560, 2560, 2495, 0]     # E 16, T 8448, k 2
ROUTER_Z = 0.001


@pytest.fixture(scope="module")
def CK():
    from fms_fsdp_b200.ops import cuda_kernels as CK
    assert CK._C.__file__.endswith("_C.so")
    return CK


@contextlib.contextmanager
def narrow(CK):
    CK._C._set_gemm_tile(1)
    try:
        yield
    finally:
        CK._C._set_gemm_tile(0)


class Judge:
    """Collects worst ratios per (quantity, tolerance key) and prints them as fractions of the tolerance."""

    def __init__(self, tag):
        self.tag, self.w, self.t0 = tag, {}, time.time()
        torch.cuda.reset_peak_memory_stats()

    def __call__(self, name, key, v):
        n = f"{name}[{key}]"
        self.w[n] = (max(self.w.get(n, (0.0, key))[0], v), key)

    def done(self, enforce=True):
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() / 2 ** 30
        print(f"MEASURE moe {self.tag}: " + " ".join(f"{n} {v / MR.TOL[k]:.3f}" for n, (v, k) in self.w.items())
              + f" x tol; {time.time() - self.t0:.1f} s, peak {peak:.1f} GiB")
        bad = {n: v for n, (v, k) in self.w.items() if not v <= MR.TOL[k]}
        assert not (enforce and bad), (self.tag, bad)


def rnd(g, *s, sc=1.0):
    return (torch.randn(*s, generator=g, device=DEV) * sc).to(BF16)


def routing(CK, T, D, E, k, regime, norm, seed=0):
    """(x, router w, logits, ids, weights, probs) of the kernels for one router regime."""
    x, wr = MR.node_inputs(T, D, E, 8, regime, seed=seed, device=DEV)[:2]
    logits = CK.gemm(x, wr, "nt", out_dtype=torch.float32)
    ids, wts, probs = CK.moe_route(logits, k, norm)
    return x, wr, logits, ids, wts, probs


# --------------------------------------------------------------------------------------------------- routing
@pytest.mark.parametrize("shape", [QWEN3, MIXTRAL], ids=["qwen3_30b_a3b", "mixtral_8x7b"])
@pytest.mark.parametrize("regime", ["init", "peaked"])
def test_routing_combine_and_route_bwd(CK, shape, regime):
    T, D, E, k = shape["T"], shape["D"], shape["E"], shape["k"]
    J = Judge(f"routing {regime} T{T} D{D} E{E} k{k}")
    x, wr, logits, ids, wts, probs = routing(CK, T, D, E, k, regime, True)
    rl = MR.mm(x, wr.to(F64).t())
    J("logits", "fp32", MR.ratio(logits, rl))
    # ids: the float64 top-k wherever the k-th and (k+1)-th logits are further apart than twice the logit error bound
    top = torch.sort(rl, -1, descending=True)
    gap = top.values[:, k - 1] - top.values[:, k]
    clear = gap > 2 * MR.TOL["fp32"] * rl.abs().amax(1)
    assert torch.equal(torch.sort(ids[clear].long(), -1).values, torch.sort(top.indices[clear, :k], -1).values)
    print(f"ids checked on {int(clear.sum())} / {T} tokens")
    rp, rw, _ = MR.route(logits, ids, True)
    J("probs", "probs", MR.ratio(probs, rp))
    J("weights", "probs", MR.ratio(wts, rw))
    plan, aux = CK.moe_plan(ids, probs)
    J("aux", "scalar", MR.scalar_ratio(aux, MR.aux_stat(probs, ids, E)))
    g = torch.Generator(device=DEV).manual_seed(1)
    Mpad = MR.moe_rows(T, k, E)[0]
    routed = MR.routed_rows(plan, T, k, E)
    yp = rnd(g, Mpad, D) * routed[:, None].to(BF16)
    res, dy = rnd(g, T, D), rnd(g, T, D)
    y = CK.moe_combine(yp, plan, wts, res, E)
    J("combine", "bf16", MR.ratio(y, MR.combine(yp, plan, wts, res, T, k, E)))
    dyp, dw = CK.moe_combine_bwd(dy, yp, plan, wts, E)
    rdyp, rdw = MR.combine_bwd(dy, yp, plan, wts, T, k, E)
    J("combine_bwd dY_perm", "bf16", MR.ratio(dyp[routed], rdyp[routed]))
    J("combine_bwd dw", "dw", MR.ratio(dw, rdw))
    J("permute_bwd", "bf16", MR.ratio(CK.moe_permute_bwd(yp, plan, T, k, E), MR.permute_bwd(yp, plan, T, k, E)))
    scale = shape["aux"] * E / (T * T)
    for part, s, d in (("dw", 0.0, dw), ("aux", scale, torch.zeros_like(dw)), ("both", scale, dw)):
        dl = CK.moe_route_bwd(probs, ids, wts, d, plan, True, s)
        J(f"route_bwd {part}", "dl", MR.ratio(dl, MR.route_bwd(probs, ids, d, True, scale, part),
                                              MR.route_bwd_scale(probs, ids, d, True, scale, part)))
    J.done()


# ----------------------------------------------------------------------------------------- grouped GEMMs
def grouped_case(CK, T, D, E, F, k, ids, tag, bitwise=False):
    """Every grouped GEMM mode on the plan of ``ids`` against float64 per row, the exact invariants of the permuted
    buffers, and (``bitwise``) against the 128 x 128 dense GEMM on each expert's rows."""
    J = Judge(tag)
    g = torch.Generator(device=DEV).manual_seed(3)
    probs = torch.full((T, E), 1.0 / E, device=DEV)
    plan, _ = CK.moe_plan(ids, probs)
    Mpad = MR.moe_rows(T, k, E)[0]
    segs = MR.segments(plan, T, k, E)
    end = max(s + n for s, _, n in segs)                      # rows past the last segment belong to no expert
    routed = MR.routed_rows(plan, T, k, E)
    pad = ~routed
    pad[end:] = False
    x, dy = rnd(g, T, D), rnd(g, T, D)
    w1, w2 = rnd(g, E, 2 * F, D, sc=0.02), rnd(g, E, D, F, sc=0.02)
    wts = torch.rand(T, k, generator=g, device=DEV)
    guard = lambda n: torch.full((Mpad, n), 7.0, dtype=BF16, device=DEV)
    xp = CK.moe_permute(x, plan, k, E)
    hp, sp = guard(2 * F), guard(F)
    CK._C.gemm_grouped(xp, w1, hp, plan, T, k, 0, 5, aux=sp, swiglu_F=F, gate_first=True)
    yp = guard(D)
    CK._C.gemm_grouped(sp, w2, yp, plan, T, k, 0, 0)
    dyp, _ = CK.moe_combine_bwd(dy, yp, plan, wts, E)
    dhp = guard(2 * F)
    CK._C.gemm_grouped(dyp, w2, dhp, plan, T, k, 1, 6, aux=hp, swiglu_F=F, gate_first=True)
    dxp = guard(D)
    CK._C.gemm_grouped(dhp, w1, dxp, plan, T, k, 1, 0)
    for n, t in (("xp", xp), ("hp", hp), ("sp", sp), ("yp", yp), ("dY_perm", dyp), ("dH", dhp), ("dX_perm", dxp)):
        assert not t[pad].any(), f"{tag}: a padding row of {n} is not zero"
        if n not in ("xp", "dY_perm"):
            assert bool((t[end:] == 7.0).all()), f"{tag}: {n} wrote past the last segment"
    rows = slice(0, end)
    rh, _ = MR.up(xp, w1, plan, T, k)
    J("up h", "bf16", MR.ratio(hp[rows], rh[rows]))
    del rh
    J("up s", "bf16", MR.ratio(sp[rows], MR._swiglu(hp[rows].to(F64), False)))
    J("down", "bf16", MR.ratio(yp[rows], MR.down(sp, w2, plan, T, k)[rows]))
    J("down_bwd", "bf16", MR.ratio(dhp[rows], MR.down_bwd(dyp, w2, hp, plan, T, k)[rows]))
    J("up_dgrad", "bf16", MR.ratio(dxp[rows], MR.up_dgrad(dhp, w1, plan, T, k)[rows]))
    for name, a, b, M, N in (("wgrad dw1", dhp, xp, 2 * F, D), ("wgrad dw2", dyp, sp, D, F)):
        for dt in (torch.float32, BF16):
            out = torch.full((E, M, N), 7.0, dtype=dt, device=DEV)
            CK._C.gemm_grouped(a, b, out, plan, T, k, 2, 0)
            base = torch.randn(E, M, N, generator=g, device=DEV).to(dt) if dt == torch.float32 else None
            acc = base.clone() if base is not None else None
            if acc is not None:
                CK._C.gemm_grouped(a, b, acc, plan, T, k, 2, 2)
            key = "fp32" if dt == torch.float32 else "bf16"
            for e, seg in enumerate(segs):
                ref = MR.wgrad_expert(a, b, seg)
                if seg[1] == 0:
                    assert not out[e].any(), f"{tag}: empty expert {e}'s {name} store is not zero"
                    if acc is not None:
                        assert torch.equal(acc[e], base[e]), f"{tag}: empty expert {e}'s {name} accumulate moved"
                J(f"{name} {'store' if acc is None else 'store+accumulate'}", key, MR.ratio(out[e], ref))
                if acc is not None:
                    J(f"{name} store+accumulate", key, MR.ratio(acc[e], ref + base[e].to(F64)))
                del ref
            if bitwise:
                _bitwise_wgrad(CK, a, b, out, acc, base, segs, f"{name} {dt}")
            del out, acc, base
    if bitwise:
        _bitwise_m(CK, xp, hp, sp, yp, dyp, dhp, dxp, w1, w2, segs, Mpad, F)
    J.done()


def _window(s, n, Mpad):
    """Rows [lo, lo + W) of at least 256 rows (the fused epilogues' minimum) that hold the segment [s, s + n)."""
    W = max(n, 256)
    lo = min(s, Mpad - W)
    return lo, W


def _bitwise_m(CK, xp, hp, sp, yp, dyp, dhp, dxp, w1, w2, segs, Mpad, F):
    """The m-grouped modes give the dense 128 x 128 GEMM's bits on each expert's (padded) rows: segments start on a
    128-row tile, so every row sees the same k-blocks in the same order."""
    C = CK._C
    with narrow(CK):
        for e, (s, n, npad) in enumerate(segs):
            if not n:
                continue
            lo, W = _window(s, npad, Mpad)
            r = slice(s - lo, s - lo + npad)
            seg = slice(s, s + npad)
            gu = torch.empty(W, 2 * F, dtype=BF16, device=DEV)
            act = torch.empty(W, F, dtype=BF16, device=DEV)
            C.gemm(xp[lo:lo + W], w1[e], gu, 0, 5, None, aux=act, swiglu_F=F, gate_first=True)
            assert torch.equal(gu[r], hp[seg]) and torch.equal(act[r], sp[seg]), f"up, expert {e}"
            o = torch.empty(W, w2.shape[1], dtype=BF16, device=DEV)
            C.gemm(sp[lo:lo + W].contiguous(), w2[e], o, 0, 0, None)
            assert torch.equal(o[r], yp[seg]), f"down, expert {e}"
            dgu = torch.empty(W, 2 * F, dtype=BF16, device=DEV)
            C.gemm(dyp[lo:lo + W].contiguous(), w2[e], dgu, 1, 6, None, aux=hp[lo:lo + W].contiguous(), swiglu_F=F,
                   gate_first=True)
            assert torch.equal(dgu[r], dhp[seg]), f"down_bwd, expert {e}"
            o = torch.empty(W, w1.shape[2], dtype=BF16, device=DEV)
            C.gemm(dhp[lo:lo + W].contiguous(), w1[e], o, 1, 0, None)
            assert torch.equal(o[r], dxp[seg]), f"up_dgrad, expert {e}"


def _bitwise_wgrad(CK, a, b, out, acc, base, segs, what):
    """The k-grouped wgrad gives the dense tn GEMM's bits over the expert's padded rows (the padding rows are zero,
    so the dense kernel's extra k-block, if any, adds exact zeros)."""
    with narrow(CK):
        for e, (s, n, npad) in enumerate(segs):
            if not n:
                continue
            d = torch.empty_like(out[e])
            CK._C.gemm(a[s:s + npad], b[s:s + npad], d, 2, 0, None)
            assert torch.equal(d, out[e]), f"{what} store, expert {e}"
            if acc is not None:
                d = base[e].clone()
                CK._C.gemm(a[s:s + npad], b[s:s + npad], d, 2, 2, None)
                assert torch.equal(d, acc[e]), f"{what} accumulate, expert {e}"


def test_grouped_gemms_on_crafted_segments(CK):
    """E 16, D 2048, F 768: empty first / last experts, counts 1, 63 / 64 / 65, 127 / 128 / 129, two empty experts in
    a row, and an expert of 8448 rows; every mode also bit for bit against the dense GEMM."""
    T, k = 8448, 2
    ids = MR.crafted_ids(CRAFTED, T, k).to(DEV)
    grouped_case(CK, T, 2048, len(CRAFTED), 768, k, ids, "grouped crafted E16 D2048 F768", bitwise=True)


@pytest.mark.parametrize("shape", [QWEN3, MIXTRAL], ids=["qwen3_30b_a3b", "mixtral_8x7b"])
def test_grouped_gemms_at_production_shapes(CK, shape):
    T, D, E, k, F = shape["T"], shape["D"], shape["E"], shape["k"], shape["F"]
    ids = routing(CK, T, D, E, k, "init", True)[3]
    grouped_case(CK, T, D, E, F, k, ids, f"grouped T{T} D{D} E{E} k{k} F{F}", bitwise=E <= 16)


# ---------------------------------------------------------------------------------------------- the node
def _run_node(h, wr, w1, w2, res, dy, k, norm, aux_coef):
    """ops.moe_mlp forward and backward with fp32 gradient buffers on the weights, as the sharded engine runs it."""
    from fms_fsdp_b200 import ops
    ws = [t.detach().clone() for t in (wr, w1, w2)]
    for w in ws:
        w._grad_buf = torch.empty(w.shape, dtype=torch.float32, device=DEV)
        w._grad_ready = False
        w.requires_grad_()
    hh = h.detach().clone().requires_grad_()
    y, aux, z = ops.moe_mlp(hh, ws[0], ws[1], ws[2], k, norm, aux_coef, residual=res, router_z_coef=ROUTER_Z,
                            return_router_z=True)
    y.backward(dy)
    return y.detach(), hh.grad, ws[0]._grad_buf, ws[1]._grad_buf, ws[2]._grad_buf, aux, z


@pytest.mark.parametrize("shape", [QWEN3, MIXTRAL], ids=["qwen3_30b_a3b", "mixtral_8x7b"])
@pytest.mark.parametrize("regime", ["init", "peaked"])
def test_moe_mlp_node(CK, shape, regime):
    from fms_fsdp_b200.ops import functional as Fn
    from fms_fsdp_b200.ops import torch_kernels as TK
    T, D, E, k, F = shape["T"], shape["D"], shape["E"], shape["k"], shape["F"]
    h, wr, w1, w2, res, dy = MR.node_inputs(T, D, E, F, regime, seed=4, device=DEV)
    # The ATen path runs through the same check for comparison, but is not held to it: its bf16 x bf16 products come
    # out of ``a @ b`` in bf16, so its router logits and its wgrads pass through bf16 where the kernels keep fp32
    # (with a peaked router that alone moves y and z past their tolerances at the Mixtral shape).
    for path in ("cuda", "torch"):
        old = Fn.get_kernel_path()
        Fn.set_kernel_path("torch" if path == "torch" else old)
        try:
            y, dh, dwr, dw1, dw2, aux, z = _run_node(h, wr, w1, w2, res, dy, k, True, shape["aux"])
        finally:
            Fn.set_kernel_path(old)
        K = TK if path == "torch" else CK
        ids = K.moe_route(K.gemm(h, wr, "nt", out_dtype=torch.float32), k, True)[0]    # the node's own ids
        J = Judge(f"node {path} {regime} T{T} D{D} E{E} k{k} F{F}")

        def expert(e, r1, r2):
            J("dw1", "dw1", MR.ratio(dw1[e], r1))
            J("dw2", "dw2", MR.ratio(dw2[e], r2))
        ref = MR.node(h, wr, w1, w2, res, dy, ids, True, shape["aux"], ROUTER_Z, on_expert=expert)
        for n, t in (("y", y), ("dh", dh), ("dwr", dwr)):
            J(n, n, MR.ratio(t, ref[n]))
        J("aux", "scalar", MR.scalar_ratio(aux, ref["aux"]))
        J("z", "scalar", MR.scalar_ratio(z, ref["z"]))
        del ref, y, dh, dwr, dw1, dw2
        J.done(enforce=path == "cuda")
