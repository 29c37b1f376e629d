"""GPU tier of the dense Llama node check (``tests/llama_node_reference.py``).

The QK-norm kernels are judged per (row, head) against float64 at the Qwen3 head layouts, M 1 / 111 / 8191 / 8192 and
four regimes; the backward both on the kernel's own pre-norm heads and rstd and against the reference's rstd.  The
dense nodes (``ops.qkv_attention`` in every form, ``gated_mlp``, ``rmsnorm`` / ``rmsnorm_fork``, ``linear``) run on
the fused kernels at Llama 2 / Llama 3 / Qwen2.5 / Qwen3 shapes and are judged tensor by tensor, with every weight
gradient delivered three ways (returned, an fp32 slot stored then accumulated, a bf16 slot accumulated).  Each case
prints its worst ratios as fractions of the tolerance ("MEASURE ... x tol"); the tolerances come from the CPU rounding
emulation (tests/test_llama_nodes_cpu.py), not from a GPU run.  The ATen path's ratios are printed, not asserted.
"""
import subprocess
import time

import pytest
import torch

import attention_reference as AR
import llama_node_reference as LR
from fms_fsdp_b200 import ops
from fms_fsdp_b200.ops import functional as FN

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64, F32, BF16 = torch.float64, torch.float32, torch.bfloat16


@pytest.fixture(scope="module")
def CK():
    from fms_fsdp_b200.ops import cuda_kernels as CK
    assert CK._C.__file__.endswith("_C.so")
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        card = torch.cuda.get_device_name()
    print(f"\nMEASURE card: {card}")
    return CK


class Judge:
    """Worst fraction of tolerance per quantity; ``done`` prints them with the run time and the allocator peak."""

    def __init__(self, tag):
        self.tag, self.w, self.t0 = tag, {}, time.time()
        torch.cuda.reset_peak_memory_stats()

    def __call__(self, name, frac):
        self.w[name] = max(self.w.get(name, 0.0), frac)

    def done(self, enforce=True):
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() / 2 ** 30
        print(f"MEASURE {self.tag}: " + " ".join(f"{n} {v:.3f}" for n, v in self.w.items())
              + f" x tol; {time.time() - self.t0:.1f} s, peak {peak:.1f} GiB")
        bad = {n: v for n, v in self.w.items() if not v <= 1.0}
        assert not (enforce and bad), (self.tag, bad)


def frac_rows(out, ref, key, rounded=False, scale=None):
    """Per-row ratio as a fraction of TOL[key] (plus one bf16 rounding of the row's max when ``rounded``)."""
    return LR.ratio(out, ref, scale) / (LR.TOL[key] + (LR.UBF if rounded else 0.0))


def frac_vec(out, ref, absum, key, rounded=()):
    """Vector gradient: |err| / (TOL[key] absum + one bf16 rounding of each of the values ``rounded``), worst
    element."""
    bound = LR.TOL[key] * absum + sum(LR.UBF * r.to(F64).abs() for r in rounded)
    return LR.GR.ratio(out.reshape(-1), ref.to(F64).reshape(-1), bound.reshape(-1))


def charged(refs, key, mode, mb):
    """The bf16 roundings a vector gradient's delivery adds: none into an fp32 slot; the stored (and then the
    accumulated) value into a bf16 slot or a bf16 returned gradient."""
    return () if mode == "fp32" else tuple(refs[i][key] for i in range(1, mb + 1))


def rnd(g, *s, sc=1.0):
    return (torch.randn(*s, generator=g, device=DEV) * sc).to(BF16)


# ============================================================================================== QK-norm kernels
QK_HEADS = {"qwen3_0.6b_1.7b": (16, 8, 128), "qwen3_4b_8b": (32, 8, 128), "qwen3_30b_a3b": (32, 4, 128),
            "hd64_gqa": (8, 2, 64)}
QK_ROWS = {"M1": (1, 1), "M111": (3, 37), "M8191": (1, 8191), "M8192": (2, 4096)}     # (B, S)


@pytest.mark.parametrize("rows", list(QK_ROWS))
@pytest.mark.parametrize("heads", list(QK_HEADS))
def test_qk_norm_kernels_per_head_against_float64(CK, heads, rows):
    H, KVH, hd = QK_HEADS[heads]
    B, S = QK_ROWS[rows]
    M, nh = B * S, H + KVH
    table = ops.torch_kernels.rope_table(S, hd, 1e6, device=DEV)
    J = Judge(f"qk_norm {heads} {rows}")
    f0 = CK.fallback_count()
    for i, regime in enumerate(("init", "tiny", "outlier", "gains")):
        qkv, wq, wk, d = LR.qk_inputs(M, H, KVH, hd, regime, seed=i, device=DEV)
        y = qkv.clone()
        xqk, rstd = CK.qk_norm_rope(y, wq, wk, table, S, H, KVH, hd, LR.EPS_QK)
        assert torch.equal(xqk, qkv[:, :nh * hd])                         # the pre-norm q / k, bit for bit
        assert torch.equal(y[:, nh * hd:], qkv[:, nh * hd:])              # V untouched
        yr, rr = LR.qk_norm_fwd(qkv, wq, wk, table, S, H, KVH, hd)
        J(f"y[{regime}]", LR.head_ratio(y[:, :nh * hd], yr[:, :nh * hd], hd) / LR.TOL["qk_y"])
        J(f"rstd[{regime}]", LR.ratio(rstd.reshape(-1, 1), rr.reshape(-1, 1)) / LR.TOL["qk_rstd"])
        del yr
        dx = d.clone()
        dwq, dwk = CK.qk_norm_bwd(dx, xqk, rstd, wq, wk, H, KVH, hd)
        assert dwq.dtype == F32 and dwq.shape == (hd,)
        assert torch.equal(dx[:, nh * hd:], d[:, nh * hd:])
        for which, rs in (("kernel_rstd", rstd), ("ref_rstd", rr)):
            ref, rq, rk, aq, ak, sc = LR.qk_norm_bwd(d, xqk, rs, wq, wk, H, KVH, hd)
            J(f"dx[{regime},{which}]", LR.head_ratio(dx[:, :nh * hd], ref[:, :nh * hd], hd, sc) / LR.TOL["qk_dx"])
            J(f"dw[{regime},{which}]", max(LR.vratio(dwq, rq, aq), LR.vratio(dwk, rk, ak)) / LR.TOL["qk_dw"])
            del ref, sc
    assert CK.fallback_count() == f0
    J.done()


# ================================================================================================= the nodes
MODELS = {
    "llama2_7b": dict(D=4096, H=32, KVH=32, hd=128, F=11008, theta=1e4),
    "llama3_8b": dict(D=4096, H=32, KVH=8, hd=128, F=14336, theta=5e5),
    "qwen2.5_7b": dict(D=3584, H=28, KVH=4, hd=128, F=18944, theta=1e6, bias=True),
    "qwen2.5_0.5b": dict(D=896, H=14, KVH=2, hd=64, F=4864, theta=1e6, bias=True),
    "qwen3_0.6b": dict(D=1024, H=16, KVH=8, hd=128, F=3072, theta=1e6, qk=True),
    "qwen3_8b": dict(D=4096, H=32, KVH=8, hd=128, F=12288, theta=1e6, qk=True),
}


def set_paths(path, precision):
    ops.set_kernel_path(path)
    FN.set_gemm_precision(precision)


def reset_paths():
    ops.set_kernel_path("auto")
    FN.set_gemm_precision("bf16")


def deliveries(J, CK, tag, call, acts, weights, dos, check, fp8=False):
    """Run the node on the fused kernels with every delivery and on the ATen path; ``check(J, label, out, dacts,
    grads, mode, mb)`` judges one result (mb 1: against the reference of dos[0], mb 2: of dos[0] + dos[1]).  Vector
    gradients are also checked for one bf16 rounding of the accumulated sum (``one_rounding``)."""
    prec = "fp8" if fp8 else "bf16"
    f0 = CK.fallback_count()
    set_paths("fused", prec)
    try:
        out, dacts, after = LR.run_node(call, acts, weights, dos[:1], "returned")
        check(J, "returned", out, dacts, after[0], "returned", 1)
        _, dacts, after32 = LR.run_node(call, acts, weights, dos, "fp32")
        check(J, "fp32_store", None, None, after32[0], "fp32", 1)
        check(J, "fp32_accum", None, dacts, after32[1], "fp32", 2)
        _, _, only2 = LR.run_node(call, acts, weights, dos[1:], "fp32")
        _, _, after16 = LR.run_node(call, acts, weights, dos, "bf16")
        check(J, "bf16_store", None, None, after16[0], "bf16", 1)
        check(J, "bf16_accum", None, None, after16[1], "bf16", 2)
        for n, p in weights.items():
            if p.dim() == 1:                 # host-side adds: the slot is the old slot plus the fp32 value, rounded once
                J(f"{n}.bf16_store_one_rounding", LR.one_rounding(after16[0][n], after32[0][n]))
                J(f"{n}.bf16_accum_one_rounding", LR.one_rounding(
                    after16[1][n], after16[0][n].to(F64) + only2[0][n].to(F64)) / (1 + 2.0 ** -15))
        assert CK.fallback_count() == f0, f"{tag}: a fused call fell back to ATen"
        set_paths("torch", prec)
        out, dacts, after = LR.run_node(call, acts, weights, dos[:1], "returned")
        A = Judge(f"{tag} ATen path (not asserted)")
        check(A, "aten", out, dacts, after[0], "returned", 1)
        A.done(enforce=False)
    finally:
        reset_paths()


def attention_case(CK, model, B, S, layout=None, fp8=False, seed=0):
    m = MODELS[model]
    D, H, KVH, hd = m["D"], m["H"], m["KVH"], m["hd"]
    N, M = (H + 2 * KVH) * hd, B * S
    form = "qk_norm" if m.get("qk") else ("bias" if m.get("bias") else "plain")
    tag = f"attention {model} {form}{' fp8' if fp8 else ''} B{B} S{S} {layout or 'causal'}"
    J = Judge(tag)
    g = torch.Generator(device=DEV).manual_seed(seed)
    h = rnd(g, B, S, D).requires_grad_()
    w = torch.nn.Parameter(rnd(g, N, D, sc=D ** -0.5))
    weights = {"w": w}
    b = qk = None
    if m.get("bias"):
        b = weights["b"] = torch.nn.Parameter(rnd(g, N, sc=0.5))
    if m.get("qk"):
        weights["wq"] = torch.nn.Parameter((0.5 + torch.rand(hd, generator=g, device=DEV)).to(BF16))
        weights["wk"] = torch.nn.Parameter((0.5 + torch.rand(hd, generator=g, device=DEV)).to(BF16))
        qk = (weights["wq"], weights["wk"], LR.EPS_QK)
    table = ops.torch_kernels.rope_table(S, hd, m["theta"], device=DEV)
    seps = None if layout is None else AR.doc_layouts(S)[layout]
    seg = None if layout is None else AR.segments([seps[i % len(seps)] for i in range(B)], S, device=DEV)
    dos = (rnd(g, B, S, H * hd), rnd(g, B, S, H * hd))
    refs = {}
    for mb, do in ((1, dos[0].reshape(M, -1)), (2, dos[0].reshape(M, -1).to(F64) + dos[1].reshape(M, -1).to(F64))):
        refs[mb] = LR.qkv_attention(h.detach().reshape(M, D), w.detach(), table, B, S, H, KVH, hd, do, seg=seg,
                                    bias=None if b is None else b.detach(),
                                    qk=None if qk is None else (qk[0].detach(), qk[1].detach(), qk[2]), fp8=fp8)
    sfx = "_fp8" if fp8 else ""

    def call():
        return ops.qkv_attention(h, w, table, H, KVH, hd, doc=seg, qk_norm=qk, qkv_bias=b)

    def check(J, label, out, dacts, grads, mode, mb):
        ref = refs[mb]
        rounded = mode != "fp32"
        if out is not None:
            J("o", frac_rows(out[0].reshape(M, -1), ref["o"], "o" + sfx))
        if dacts is not None:
            J("dh", frac_rows(dacts["h"].reshape(M, -1), ref["dh"], "dh" + sfx))
        J(f"dw.{label}", frac_rows(grads["w"], ref["dw"], "dw" + sfx, rounded))
        if b is not None:
            J(f"db.{label}", frac_vec(grads["b"], ref["db"], ref["db_abs"], "db", charged(refs, "db", mode, mb)))
        if qk is not None:
            J(f"dw_q.{label}", frac_vec(grads["wq"], ref["dwq"], ref["dwq_abs"], "dwqk", charged(refs, "dwq", mode, mb)))
            J(f"dw_k.{label}", frac_vec(grads["wk"], ref["dwk"], ref["dwk_abs"], "dwqk", charged(refs, "dwk", mode, mb)))

    deliveries(J, CK, tag, call, {"h": h}, weights, dos, check, fp8)
    J.done()


def mlp_case(CK, model, B, S, fp8=False, gate_first=True, seed=1):
    m = MODELS[model]
    D, F, M = m["D"], m["F"], B * S
    tag = f"gated_mlp {model}{' fp8' if fp8 else ''} gate_first={gate_first} B{B} S{S}"
    J = Judge(tag)
    g = torch.Generator(device=DEV).manual_seed(seed)
    x, res = rnd(g, B, S, D).requires_grad_(), rnd(g, B, S, D).requires_grad_()
    wg1 = torch.nn.Parameter(rnd(g, 2 * F, D, sc=D ** -0.5))
    w2 = torch.nn.Parameter(rnd(g, D, F, sc=F ** -0.5))
    dos = (rnd(g, B, S, D), rnd(g, B, S, D))
    refs = {mb: LR.gated_mlp(x.detach().reshape(M, D), wg1.detach(), w2.detach(), do, res.detach().reshape(M, D),
                             gate_first, fp8)
            for mb, do in ((1, dos[0].reshape(M, D)), (2, dos[0].reshape(M, D).to(F64) + dos[1].reshape(M, D).to(F64)))}
    for r in refs.values():
        del r["gu"], r["act"]
    sfx = "_fp8" if fp8 else ""

    def call():
        return ops.gated_mlp(x, wg1, w2, residual=res, gate_first=gate_first)

    def check(J, label, out, dacts, grads, mode, mb):
        ref = refs[mb]
        if out is not None:
            J("y", frac_rows(out[0].reshape(M, -1), ref["y"], "y" + sfx))
        if dacts is not None:
            J("dx", frac_rows(dacts["x"].reshape(M, -1), ref["dx"], "dx" + sfx))
            J("dres", frac_rows(dacts["res"].reshape(M, -1), ref["dres"], "dx" + sfx))
        J(f"dwg1.{label}", frac_rows(grads["wg1"], ref["dwg1"], "dwl" + sfx, mode != "fp32"))
        J(f"dw2.{label}", frac_rows(grads["w2"], ref["dw2"], "dwl" + sfx, mode != "fp32"))

    deliveries(J, CK, tag, call, {"x": x, "res": res}, {"wg1": wg1, "w2": w2}, dos, check, fp8)
    J.done()


def norm_linear_case(CK, model, B, S, seed=2):
    """rmsnorm_fork (with the residual branch's gradient), rmsnorm, and the output projection with its residual."""
    m = MODELS[model]
    D, Hd, M = m["D"], m["H"] * m["hd"], B * S
    J = Judge(f"norms and linear {model} B{B} S{S}")
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = rnd(g, B, S, D).requires_grad_()
    wn = torch.nn.Parameter((1 + 0.3 * torch.randn(D, generator=g, device=DEV)).to(BF16))
    dys = [(rnd(g, B, S, D), rnd(g, B, S, D)) for _ in range(2)]
    for fork in (True, False):
        refs = {}
        for mb in (1, 2):
            dy = sum(d[0].reshape(M, D).to(F64) for d in dys[:mb])
            dr = sum(d[1].reshape(M, D).to(F64) for d in dys[:mb]) if fork else None
            refs[mb] = LR.rmsnorm(x.detach().reshape(M, D), wn.detach(), dy, 1e-5, dr)

        def call():
            return ops.rmsnorm_fork(x, wn, 1e-5) if fork else ops.rmsnorm(x, wn, 1e-5)

        def check(J, label, out, dacts, grads, mode, mb, fork=fork, refs=refs):
            ref = refs[mb]
            p = "fork" if fork else "rmsnorm"
            if out is not None:
                J(f"{p}.y", frac_rows(out[0].reshape(M, -1), ref["y"], "norm_y"))
            if dacts is not None:
                J(f"{p}.dx", frac_rows(dacts["x"].reshape(M, -1), ref["dx"], "norm_dx"))
            J(f"{p}.dw.{label}", frac_vec(grads["w"], ref["dw"], ref["dw_abs"], "norm_dw",
                                          charged(refs, "dw", mode, mb)))

        dos = dys if fork else [d[0] for d in dys]
        deliveries(J, CK, f"norm {model}", call, {"x": x}, {"w": wn}, dos, check)
    # the attention output projection: H hd -> D, with the residual (H hd != D for Qwen3-0.6B)
    o, res = rnd(g, B, S, Hd).requires_grad_(), rnd(g, B, S, D).requires_grad_()
    wo = torch.nn.Parameter(rnd(g, D, Hd, sc=Hd ** -0.5))
    dos = (rnd(g, B, S, D), rnd(g, B, S, D))
    refs = {mb: LR.linear(o.detach().reshape(M, Hd), wo.detach(), do, res.detach().reshape(M, D))
            for mb, do in ((1, dos[0].reshape(M, D)), (2, dos[0].reshape(M, D).to(F64) + dos[1].reshape(M, D).to(F64)))}

    def check(J, label, out, dacts, grads, mode, mb):
        ref = refs[mb]
        if out is not None:
            J("linear.y", frac_rows(out[0].reshape(M, -1), ref["y"], "y"))
        if dacts is not None:
            J("linear.dx", frac_rows(dacts["o"].reshape(M, -1), ref["dx"], "dx"))
            J("linear.dres", frac_rows(dacts["res"].reshape(M, -1), ref["dres"], "dx"))
        J(f"linear.dw.{label}", frac_rows(grads["w"], ref["dw"], "dwl", mode != "fp32"))

    deliveries(J, CK, f"linear {model}", lambda: ops.linear(o, wo, res), {"o": o, "res": res}, {"w": wo}, dos, check)
    J.done()


ATTN_CASES = [("llama2_7b", 2, 4096, None), ("llama3_8b", 2, 4096, None), ("qwen2.5_7b", 2, 4096, None),
              ("qwen2.5_7b", 2, 4096, "low_after_high"), ("qwen2.5_0.5b", 2, 4096, "mid_tile"),
              ("qwen3_0.6b", 2, 4096, None), ("qwen3_0.6b", 2, 4096, "one_token"), ("qwen3_8b", 2, 4096, None),
              # edges: a ragged 65-long row, S 1000 with three rows (B S a multiple of 8: the GEMMs need it, and a
              # smaller one would run the counted ATen fallback).  Not S 1: a query with one key has a q / k gradient of
              # exactly 0 in float64, which the kernels' dP - delta reproduces only to rounding, so the exact-zero rule
              # of the metric cannot hold there (the MLP and norm cases run S 1)
              ("qwen3_0.6b", 8, 65, None), ("qwen3_0.6b", 3, 1000, "mid_tile"),
              ("qwen2.5_0.5b", 8, 65, None), ("qwen2.5_0.5b", 3, 1000, "one_token")]


@pytest.mark.parametrize("model,B,S,layout", ATTN_CASES, ids=[f"{m}-B{b}-S{s}-{l or 'causal'}" for m, b, s, l in ATTN_CASES])
def test_attention_node_against_float64(CK, model, B, S, layout):
    attention_case(CK, model, B, S, layout)


@pytest.mark.parametrize("model,layout", [("llama3_8b", None), ("qwen3_8b", None), ("qwen3_0.6b", "mid_tile")])
def test_attention_node_fp8_against_float64(CK, model, layout):
    attention_case(CK, model, 2, 4096, layout, fp8=True)


MLP_CASES = [("llama2_7b", 2, 4096, False, True), ("llama3_8b", 2, 4096, False, True),
             ("qwen2.5_7b", 2, 4096, False, True), ("qwen2.5_0.5b", 2, 4096, False, False),
             ("qwen3_0.6b", 8, 1, False, True), ("qwen3_0.6b", 8, 65, False, False), ("qwen3_0.6b", 3, 1000, False, True),
             ("llama3_8b", 2, 4096, True, True), ("qwen3_0.6b", 8, 65, True, False)]


@pytest.mark.parametrize("model,B,S,fp8,gate_first", MLP_CASES,
                         ids=[f"{m}-B{b}-S{s}{'-fp8' if f else ''}-{'gate_up' if gf else 'up_gate'}"
                              for m, b, s, f, gf in MLP_CASES])
def test_gated_mlp_node_against_float64(CK, model, B, S, fp8, gate_first):
    mlp_case(CK, model, B, S, fp8, gate_first)


NORM_CASES = [("llama2_7b", 2, 4096), ("qwen2.5_7b", 2, 4096), ("qwen2.5_0.5b", 2, 4096), ("qwen3_0.6b", 2, 4096),
              ("qwen3_0.6b", 8, 1), ("qwen3_0.6b", 3, 1000)]


@pytest.mark.parametrize("model,B,S", NORM_CASES, ids=[f"{m}-B{b}-S{s}" for m, b, s in NORM_CASES])
def test_norm_and_linear_nodes_against_float64(CK, model, B, S):
    norm_linear_case(CK, model, B, S)
