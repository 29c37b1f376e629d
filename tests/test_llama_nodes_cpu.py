"""CPU tier of the dense Llama node check (``tests/llama_node_reference.py``): the float64 node references are pinned to
float64 autograd through an independent plain block, the rounding emulation of the sm_90a kernels passes every
tolerance with at least 2x headroom, plausibly broken kernels and broken node code fail the check that targets them,
and the node code itself (``ops.*`` on float64 CPU tensors) delivers its weight gradients into all three destinations
(returned, an fp32 slot, a bf16 slot) as the reference says.
"""
import pytest
import torch

import attention_reference as AR
import llama_node_reference as LR
from fms_fsdp_b200 import ops
from fms_fsdp_b200.ops import functional as FN

F64, BF16 = torch.float64, torch.bfloat16
B, S, D = 2, 128, 256
QK_M, QK_S = 111, 37                   # 3 batch rows of 37: not a multiple of any row block


def table_of(hd, theta=1e6, S=S):
    return ops.torch_kernels.rope_table(S, hd, theta)


def seg_of(layout):
    return None if layout is None else AR.segments(AR.doc_layouts(S)[layout], S)


# form: (H, KVH, hd, bias, qk, fp8)
ATTN_FORMS = {
    "plain": (4, 2, 64, False, False, False),
    "bias": (4, 1, 64, True, False, False),
    "qk_norm": (4, 2, 128, False, True, False),
    "plain_fp8": (4, 2, 64, False, False, True),
    "qk_norm_fp8": (4, 4, 128, False, True, True),
}


def attn_case(form, regime, layout, seed=0):
    H, KVH, hd, bias, qk, fp8 = ATTN_FORMS[form]
    N = (H + 2 * KVH) * hd
    shp = {"h": (B * S, D), "w": (N, D), "do": (B * S, H * hd)}
    if bias:
        shp["b"] = (N,)
    if qk:
        shp["wq"], shp["wk"] = (hd,), (hd,)
    t = LR.node_inputs(shp, regime, seed)
    kw = dict(seg=seg_of(layout), bias=t.get("b"), qk=(t["wq"], t["wk"], 1e-6) if qk else None, fp8=fp8)
    return (t["h"], t["w"], table_of(hd), B, S, H, KVH, hd, t["do"]), kw


def attn_ratios(form, out, ref):
    fp8 = ATTN_FORMS[form][5]
    sfx = "_fp8" if fp8 else ""
    r = {"o" + sfx: LR.ratio(out["o"], ref["o"]), "dh" + sfx: LR.ratio(out["dh"], ref["dh"]),
         "dw" + sfx: LR.ratio(out["dw"], ref["dw"])}
    if "db" in ref:
        r["db"] = LR.vratio(out["db"], ref["db"], ref["db_abs"])
    if "dwq" in ref:
        r["dwqk"] = max(LR.vratio(out["dwq"], ref["dwq"], ref["dwq_abs"]),
                        LR.vratio(out["dwk"], ref["dwk"], ref["dwk_abs"]))
    return r


def mlp_case(regime, res, seed=0, F=384):
    shp = {"x": (B * S // 2, D), "wg1": (2 * F, D), "w2": (D, F), "dy": (B * S // 2, D), "res": (B * S // 2, D)}
    t = LR.node_inputs(shp, regime, seed)
    return t["x"], t["wg1"], t["w2"], t["dy"], (t["res"] if res else None)


def mlp_ratios(out, ref, fp8):
    sfx = "_fp8" if fp8 else ""
    r = {"y" + sfx: LR.ratio(out["y"], ref["y"]), "dx" + sfx: LR.ratio(out["dx"], ref["dx"]),
         "dwl" + sfx: max(LR.ratio(out["dwg1"], ref["dwg1"]), LR.ratio(out["dw2"], ref["dw2"]))}
    if ref["dres"] is not None:
        r["dx" + sfx] = max(r["dx" + sfx], LR.ratio(out["dres"], ref["dres"]))
    return r


def norm_case(regime, seed=0):
    t = LR.node_inputs({"x": (B * S // 2, D), "w": (D,), "dy": (B * S // 2, D), "dres": (B * S // 2, D)}, regime, seed)
    t["w"] = (1 + torch.randn(D, generator=torch.Generator().manual_seed(seed)) * 0.3).to(BF16)
    return t["x"], t["w"], t["dy"], t["dres"]


def norm_ratios(out, ref):
    return {"norm_y": LR.ratio(out["y"], ref["y"]), "norm_dx": LR.ratio(out["dx"], ref["dx"]),
            "norm_dw": LR.vratio(out["dw"], ref["dw"], ref["dw_abs"])}


def linear_ratios(out, ref):
    r = {"y": LR.ratio(out["y"], ref["y"]), "dx": LR.ratio(out["dx"], ref["dx"]), "dwl": LR.ratio(out["dw"], ref["dw"])}
    if ref["dres"] is not None:
        r["dx"] = max(r["dx"], LR.ratio(out["dres"], ref["dres"]))
    return r


def qk_ratios(M, S_, H, KVH, hd, regime, mut=None, seed=0):
    """Emulated QK-norm kernels (with ``mut``) against the float64 reference, per (row, head)."""
    qkv, wq, wk, d = LR.qk_inputs(M, H, KVH, hd, regime, seed)
    table = table_of(hd, S=S_)
    nh = H + KVH
    y, r = LR.qk_norm_fwd(qkv, wq, wk, table, S_, H, KVH, hd, em=True, mut=mut)
    yr, rr = LR.qk_norm_fwd(qkv, wq, wk, table, S_, H, KVH, hd)
    out = {"qk_y": LR.head_ratio(y[:, :nh * hd], yr[:, :nh * hd], hd),
           "qk_rstd": LR.ratio(r.reshape(-1, 1), rr.reshape(-1, 1))}
    xqk = qkv[:, :nh * hd]
    dx, dwq, dwk, *_ = LR.qk_norm_bwd(d, xqk, r, wq, wk, H, KVH, hd, em=True, mut=mut)
    for rs in (r, rr):                     # the kernel's own rstd, and the reference's
        ref, rq, rk, aq, ak, sc = LR.qk_norm_bwd(d, xqk, rs, wq, wk, H, KVH, hd)
        out["qk_dx"] = max(out.get("qk_dx", 0.0), LR.head_ratio(dx[:, :nh * hd], ref[:, :nh * hd], hd, sc))
        out["qk_dw"] = max(out.get("qk_dw", 0.0), LR.vratio(dwq, rq, aq), LR.vratio(dwk, rk, ak))
    return out


# ------------------------------------------------------------------------------ the reference is float64 autograd
@pytest.mark.parametrize("layout", [None, "mid_tile"])
@pytest.mark.parametrize("form", list(ATTN_FORMS))
def test_attention_reference_is_autograd_in_float64(form, layout):
    args, kw = attn_case(form, "init", layout)
    ref = LR.qkv_attention(*args, **kw)
    ag = LR.attention_autograd(*args, **kw)
    for n in ag:
        if n + "_abs" in ref:           # a vector gradient: against the sum of |terms| (its elements may cancel)
            assert LR.vratio(ref[n], ag[n], ref[n + "_abs"]) < 1e-12, n
        else:
            assert LR.ratio(ref[n], ag[n]) < 1e-10, n


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("gate_first", [True, False])
@pytest.mark.parametrize("res", [False, True])
def test_mlp_reference_is_autograd_in_float64(res, gate_first, fp8):
    x, wg1, w2, dy, r = mlp_case("init", res)
    ref = LR.gated_mlp(x, wg1, w2, dy, r, gate_first, fp8)
    ag = LR.mlp_autograd(x, wg1, w2, dy, r, gate_first, fp8)
    for n in ("y", "dx", "dwg1", "dw2") + (("dres",) if res else ()):
        assert LR.ratio(ref[n], ag[n]) < 1e-10, n


@pytest.mark.parametrize("fork", [False, True])
def test_norm_and_linear_references_are_autograd_in_float64(fork):
    x, w, dy, dres = norm_case("init")
    ref = LR.rmsnorm(x, w, dy, 1e-5, dres if fork else None)
    ag = LR.rmsnorm_autograd(x, w, dy, 1e-5, dres if fork else None)
    for n in ("y", "dx"):
        assert LR.ratio(ref[n], ag[n]) < 1e-10, n
    assert LR.ratio(ref["dw"].view(1, -1), ag["dw"].view(1, -1)) < 1e-10
    # linear, with the residual when ``fork``
    wl, dl = torch.randn(96, D).to(BF16), torch.randn(x.shape[0], 96).to(BF16)
    X, W = (t.to(F64).requires_grad_() for t in (x, wl))
    res = dres[:, :96].to(F64).requires_grad_() if fork else None
    y = X @ W.t() + (res if fork else 0)
    gr = torch.autograd.grad((y * dl.to(F64)).sum(), [X, W] + ([res] if fork else []))
    lin = LR.linear(x, wl, dl, dres[:, :96] if fork else None)
    assert LR.ratio(lin["dx"], gr[0]) < 1e-10 and LR.ratio(lin["dw"], gr[1]) < 1e-10
    assert LR.ratio(lin["y"], y.detach()) < 1e-10
    if fork:
        assert LR.ratio(lin["dres"], gr[2]) < 1e-10


def test_qk_norm_reference_is_autograd_in_float64():
    H, KVH, hd = 4, 2, 64
    qkv, wq, wk, d = LR.qk_inputs(QK_M, H, KVH, hd, "gains")
    table = table_of(hd, S=QK_S)
    nh = H + KVH
    y, r = LR.qk_norm_fwd(qkv, wq, wk, table, QK_S, H, KVH, hd)
    dx, dwq, dwk, *_ = LR.qk_norm_bwd(d, qkv[:, :nh * hd], r, wq, wk, H, KVH, hd)
    X, WQ, WK = (t.to(F64).requires_grad_() for t in (qkv, wq, wk))
    x = X.view(QK_M, H + 2 * KVH, hd)
    w = torch.cat([WQ.expand(H, -1), WK.expand(KVH, -1)])
    n = x[:, :nh] * torch.rsqrt(x[:, :nh].pow(2).mean(-1, keepdim=True) + LR.EPS_QK) * w
    c, s = LR.rope_cs(table, QK_M, QK_S, nh * hd, hd)
    rot = LR.rot(n.reshape(QK_M, -1), c, s)
    # the backward's input is the gradient of the normed, un-rotated heads: differentiate n against d
    gx, gq, gk = torch.autograd.grad((n.reshape(QK_M, -1) * d[:, :nh * hd].to(F64)).sum(), [X, WQ, WK])
    assert LR.ratio(y[:, :nh * hd], rot.detach()) < 1e-12
    assert LR.ratio(dx[:, :nh * hd], gx[:, :nh * hd]) < 1e-10
    assert LR.ratio(dwq.view(1, -1), gq.view(1, -1)) < 1e-10 and LR.ratio(dwk.view(1, -1), gk.view(1, -1)) < 1e-10


# ---------------------------------------------------------------------------------- the emulation has headroom
def _headroom(r):
    bad = {k: (v, LR.TOL[k]) for k, v in r.items() if not v <= LR.TOL[k] / 2}
    assert not bad, bad


@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("regime", ["init", "tiny", "outlier", "gains"])
def test_emulated_qk_norm_kernels_pass_with_headroom(regime, hd):
    _headroom(qk_ratios(QK_M, QK_S, 4, 2, hd, regime))


@pytest.mark.parametrize("layout", [None, "mid_tile", "one_token"])
@pytest.mark.parametrize("regime", ["init", "outlier"])
@pytest.mark.parametrize("form", list(ATTN_FORMS))
def test_emulated_attention_node_passes_with_headroom(form, regime, layout):
    args, kw = attn_case(form, regime, layout)
    _headroom(attn_ratios(form, LR.qkv_attention(*args, **kw, em=True), LR.qkv_attention(*args, **kw)))


@pytest.mark.parametrize("regime", ["init", "outlier"])
def test_emulated_mlp_norm_and_linear_pass_with_headroom(regime):
    r = {}
    for res in (False, True):
        x, wg1, w2, dy, rr = mlp_case(regime, res)
        for gf in (True, False):
            for fp8 in (False, True):
                for k, v in mlp_ratios(LR.gated_mlp(x, wg1, w2, dy, rr, gf, fp8, em=True),
                                       LR.gated_mlp(x, wg1, w2, dy, rr, gf, fp8), fp8).items():
                    r[k] = max(r.get(k, 0.0), v)
        dl =torch.randn(x.shape[0], w2.shape[0], generator=torch.Generator().manual_seed(5)).to(BF16)
        xl = torch.randn(x.shape[0], w2.shape[1], generator=torch.Generator().manual_seed(6)).to(BF16)
        for k, v in linear_ratios(LR.linear(xl, w2, dl, rr, em=True), LR.linear(xl, w2, dl, rr)).items():
            r[k] = max(r.get(k, 0.0), v)
    x, w, dy, dres = norm_case(regime)
    for dr in (None, dres):
        for k, v in norm_ratios(LR.rmsnorm(x, w, dy, 1e-5, dr, em=True), LR.rmsnorm(x, w, dy, 1e-5, dr)).items():
            r[k] = max(r.get(k, 0.0), v)
    _headroom(r)


# ---------------------------------------------------------------------------------- broken variants fail
QK_TARGET = {"rstd_no_eps": "tiny", "eps_after_sqrt": "tiny", "norm_after_rope": "gains", "wq_wk_swapped": "init",
             "bwd_mean_without_w": "gains", "dwq_sums_k_heads": "init"}


@pytest.mark.parametrize("mut", LR.QK_MUTATIONS)
def test_broken_qk_norm_kernel_fails(mut):
    r = qk_ratios(QK_M, QK_S, 4, 2, 64, QK_TARGET[mut], mut=mut)
    assert any(not v <= LR.TOL[k] for k, v in r.items()), r


@pytest.mark.parametrize("mut", ["norm_bwd_rotated_grad", "inv_rope_after_norm_bwd"])
def test_norm_backward_fed_the_rotated_gradient_fails(mut):
    args, kw = attn_case("qk_norm", "init", None)
    r = attn_ratios("qk_norm", LR.qkv_attention(*args, **kw, em=True, mut=mut), LR.qkv_attention(*args, **kw))
    assert r["dh"] > LR.TOL["dh"] and r["dwqk"] > LR.TOL["dwqk"], r


def test_bias_grad_from_the_rotated_gradient_fails():
    args, kw = attn_case("bias", "init", None)
    r = attn_ratios("bias", LR.qkv_attention(*args, **kw, em=True, mut="bias_grad_rotated"),
                    LR.qkv_attention(*args, **kw))
    assert r["db"] > LR.TOL["db"], r


def test_dropped_dres_and_residual_gradients_fail():
    x, w, dy, dres = norm_case("init")
    r = norm_ratios(LR.rmsnorm(x, w, dy, 1e-5, dres, em=True, mut="dres_dropped"), LR.rmsnorm(x, w, dy, 1e-5, dres))
    assert r["norm_dx"] > LR.TOL["norm_dx"], r
    x, wg1, w2, dy, res = mlp_case("init", True)
    r = mlp_ratios(LR.gated_mlp(x, wg1, w2, dy, res, em=True, mut="residual_grad_dropped"),
                   LR.gated_mlp(x, wg1, w2, dy, res), False)
    assert r["dx"] > LR.TOL["dx"], r
    wl = wg1[:D]
    r = linear_ratios(LR.linear(x, wl, dy, res, em=True, mut="residual_grad_dropped"), LR.linear(x, wl, dy, res))
    assert r["dx"] > LR.TOL["dx"], r


# --------------------------------------------------------------------- the node code delivers its gradients
def _qk_norm_node(seed=0):
    """The QK-norm attention node on float64 CPU tensors (bf16 values) through ``ops``: (call, acts, weights, dos,
    reference of dos[0], reference of dos[0] + dos[1])."""
    args, kw = attn_case("qk_norm", "init", "mid_tile", seed)
    h, w, table, B_, S_, H, KVH, hd, do = args
    h = h.to(F64).view(B_, S_, -1).requires_grad_()
    W = {"w": torch.nn.Parameter(w.to(F64)), "wq": torch.nn.Parameter(kw["qk"][0].to(F64)),
         "wk": torch.nn.Parameter(kw["qk"][1].to(F64))}
    do2 = torch.randn(do.shape, generator=torch.Generator().manual_seed(seed + 9)).to(BF16)
    refs = [LR.qkv_attention(*args, **kw), LR.qkv_attention(*args[:-1], do.to(F64) + do2.to(F64), **kw)]

    def call():
        return ops.qkv_attention(h, W["w"], table, H, KVH, hd, doc=kw["seg"], qk_norm=(W["wq"], W["wk"], 1e-6))
    return call, {"h": h}, W, [t.to(F64).view(B_, S_, -1) for t in (do, do2)], refs


def test_node_code_delivers_every_gradient_to_every_destination():
    call, acts, W, dos, refs = _qk_norm_node()
    _, _, ret = LR.run_node(call, acts, W, dos[:1], "returned")
    _, _, f32 = LR.run_node(call, acts, W, dos, "fp32")
    names = {"w": "dw", "wq": "dwq", "wk": "dwk"}
    for got, ref in ((ret[0], refs[0]), (f32[0], refs[0]), (f32[1], refs[1])):
        for n, k in names.items():
            r = LR.vratio(got[n], ref[k], ref[k + "_abs"]) if n != "w" else LR.ratio(got[n], ref[k])
            assert r < 1e-5, (n, r)          # the ATen attention computes in fp32
    # a bf16 slot: the stored value, then the old slot plus the fp32 contribution, each rounded once
    _, _, only2 = LR.run_node(call, acts, W, dos[1:], "fp32")
    _, _, b16 = LR.run_node(call, acts, W, dos, "bf16")
    for n in ("wq", "wk"):
        assert LR.one_rounding(b16[0][n], f32[0][n]) <= 1.0
        assert LR.one_rounding(b16[1][n], b16[0][n].to(F64) + only2[0][n].to(F64)) <= 1.0


def test_accumulated_gain_gradient_written_with_copy_fails(monkeypatch):
    def copy_put(val):
        return lambda out, acc: out.copy_(val)
    monkeypatch.setattr(FN, "_put_fp32", copy_put)
    call, acts, W, dos, refs = _qk_norm_node()
    _, _, f32 = LR.run_node(call, acts, W, dos, "fp32")
    assert LR.vratio(f32[1]["wq"], refs[1]["dwq"], refs[1]["dwq_abs"]) > LR.TOL["dwqk"]
