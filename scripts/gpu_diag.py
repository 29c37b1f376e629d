"""GPU diagnostic: numerics + timing of every sm_90a kernel against the ATen oracle.
Writes $DIAG_OUT/diag.json (default diag_out/ in the repository root; one record per check), so one run answers many
questions.   usage: python scripts/gpu_diag.py [gemm] [gemm2] [elem] [attn] [ssd] [selscan] ...
Each check is isolated in try/except; a CUDA error aborts the remaining checks of that group only
when the context is poisoned.
"""
import json
import os
import sys
import time
import traceback

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

OUT = os.environ.get("DIAG_OUT") or os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "diag_out")
os.makedirs(OUT, exist_ok=True)
records = []


def rec(name, **kw):
    kw["name"] = name
    records.append(kw)
    print(json.dumps(kw), flush=True)
    with open(os.path.join(OUT, "diag.json"), "w") as f:
        json.dump(records, f, indent=1)


SMALL = os.environ.get("DIAG_SMALL") == "1"   # under compute-sanitizer: numerics on small shapes only, no timing loops


def time_ms(fn, iters=10, warmup=3):
    if SMALL:
        fn()
        torch.cuda.synchronize()
        return 0.0
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def relerr(a, b):
    a, b = a.float(), b.float()
    return ((a - b).abs().max() / b.abs().max().clamp(min=1e-6)).item()


def main(groups):
    from fms_fsdp_b200.ops import torch_kernels as TK
    from fms_fsdp_b200.ops import cuda_kernels as CK
    dev = torch.device("cuda")
    torch.manual_seed(0)
    rec("env", device=torch.cuda.get_device_name(0), torch=torch.__version__)

    if "gemm2" in groups:
        # the fused-epilogue GEMM entry vs cuBLAS on training shapes
        for layout, (M, N, K) in [("nt", (8192, 12288, 4096)), ("nt", (8192, 22016, 4096)), ("nt", (8192, 4096, 11008)),
                                  ("nn", (8192, 4096, 12288)), ("nn", (8192, 4096, 22016)), ("tn", (12288, 4096, 8192)),
                                  ("tn", (22016, 4096, 8192)), ("nt", (256, 512, 128)), ("nn", (512, 768, 192)), ("tn", (1000, 520, 72))]:
            try:
                if layout == "nt":
                    a = torch.randn(M, K, device=dev).bfloat16(); b = torch.randn(N, K, device=dev).bfloat16()
                elif layout == "nn":
                    a = torch.randn(M, K, device=dev).bfloat16(); b = torch.randn(K, N, device=dev).bfloat16()
                else:
                    a = torch.randn(K, M, device=dev).bfloat16(); b = torch.randn(K, N, device=dev).bfloat16()
                ref = TK.gemm(a, b, layout).float()
                r = dict(layout=layout, M=M, N=N, K=K)
                out = CK.gemm(a, b, layout)
                torch.cuda.synchronize()
                r["relerr"] = relerr(out, ref)
                if M >= 4096:
                    ms = time_ms(lambda: CK.gemm(a, b, layout))
                    r["tflops"] = 2 * M * N * K / ms / 1e9
                    ms = time_ms(lambda: TK.gemm(a, b, layout))
                    r["tflops_cublas"] = 2 * M * N * K / ms / 1e9
                rec("gemm2", **r)
            except Exception as ex:
                rec("gemm2", layout=layout, M=M, N=N, K=K, ok=False, error=repr(ex)[:400])
        try:
            M, N, K = 512, 768, 256
            a = torch.randn(M, K, device=dev).bfloat16(); b = torch.randn(N, K, device=dev).bfloat16()
            r_ = torch.randn(M, N, device=dev).bfloat16(); ref = a.float() @ b.float().t()
            rec("gemm2_residual", relerr=relerr(CK.gemm(a, b, "nt", residual=r_), ref + r_.float()))
            c = torch.randn(M, N, device=dev); c0 = c.clone(); CK.gemm(a, b, "nt", out=c, accumulate=True)
            rec("gemm2_accum_f32", relerr=relerr(c, ref + c0))
        except Exception as ex:
            rec("gemm2_epilogues", ok=False, error=repr(ex)[:400])

    if "gemm" in groups:
        shapes = [(128, 256, 64), (256, 512, 256), (384, 768, 192), (8, 8, 8), (1000, 520, 72),
                  (2048, 4096, 4096), (8192, 12288, 4096)][:(2 if SMALL else None)]
        for layout in ("nt", "nn", "tn"):
            for (M, N, K) in shapes:
                try:
                    if layout == "nt":
                        a = torch.randn(M, K, device=dev).bfloat16(); b = torch.randn(N, K, device=dev).bfloat16()
                    elif layout == "nn":
                        a = torch.randn(M, K, device=dev).bfloat16(); b = torch.randn(K, N, device=dev).bfloat16()
                    else:
                        a = torch.randn(K, M, device=dev).bfloat16(); b = torch.randn(K, N, device=dev).bfloat16()
                    ref = TK.gemm(a.float(), b.float(), layout)
                    out = CK.gemm(a, b, layout)
                    torch.cuda.synchronize()
                    e = relerr(out, ref)
                    r = dict(layout=layout, M=M, N=N, K=K, relerr=e, ok=bool(e < 2e-2))
                    if M >= 2048:
                        ms = time_ms(lambda: CK.gemm(a, b, layout))
                        ms_ref = time_ms(lambda: TK.gemm(a, b, layout))
                        r.update(ms=ms, tflops=2 * M * N * K / ms / 1e9, cublas_ms=ms_ref,
                                 cublas_tflops=2 * M * N * K / ms_ref / 1e9)
                    rec("gemm", **r)
                except Exception as ex:
                    rec("gemm", layout=layout, M=M, N=N, K=K, ok=False, error=repr(ex)[:400])
        # epilogues
        try:
            M, N, K = 512, 768, 256
            a = torch.randn(M, K, device=dev).bfloat16(); b = torch.randn(N, K, device=dev).bfloat16()
            r_ = torch.randn(M, N, device=dev).bfloat16()
            ref = a.float() @ b.float().t()
            out = CK.gemm(a, b, "nt", residual=r_)
            rec("gemm_residual", relerr=relerr(out, ref + r_.float()))
            c = torch.randn(M, N, device=dev).bfloat16(); c0 = c.clone()
            CK.gemm(a, b, "nt", out=c, accumulate=True)
            rec("gemm_accum_bf16", relerr=relerr(c, ref + c0.float()))
            c = torch.randn(M, N, device=dev); c0 = c.clone()
            CK.gemm(a, b, "nt", out=c, accumulate=True)
            rec("gemm_accum_f32", relerr=relerr(c, ref + c0))
            c = torch.empty(M, N, device=dev)
            CK.gemm(a, b, "nt", out=c)
            rec("gemm_out_f32", relerr=relerr(c, ref))
        except Exception as ex:
            rec("gemm_epilogues", ok=False, error=repr(ex)[:400])

    if "elem" in groups:
        def chk(name, fn):
            try:
                fn()
            except Exception as ex:
                rec(name, ok=False, error=repr(ex)[:400], tb=traceback.format_exc()[-600:])
        M, D = 1024, 4096

        def t_rms():
            x = torch.randn(M, D, device=dev).bfloat16(); w = (1 + 0.1 * torch.randn(D, device=dev)).bfloat16()
            dy = torch.randn(M, D, device=dev).bfloat16()
            y0, r0 = TK.rmsnorm_fwd(x, w, 1e-5); y1, r1 = CK.rmsnorm_fwd(x, w, 1e-5)
            dx0, dw0 = TK.rmsnorm_bwd(dy, x, w, r0); dx1, dw1 = CK.rmsnorm_bwd(dy, x, w, r1)
            xb = torch.randn(256 if SMALL else 8192, 4096, device=dev).bfloat16()
            ms = time_ms(lambda: CK.rmsnorm_fwd(xb, w, 1e-5))
            dres = torch.randn(M, D, device=dev).bfloat16()
            dxr = relerr(CK.rmsnorm_bwd(dy, x, w, r1, dres)[0], TK.rmsnorm_bwd(dy, x, w, r0, dres)[0])
            dyb = torch.randn(xb.shape[0], 4096, device=dev).bfloat16(); _, rb = CK.rmsnorm_fwd(xb, w, 1e-5)
            msb = time_ms(lambda: CK.rmsnorm_bwd(dyb, xb, w, rb, dyb))
            q = torch.randn(256 if SMALL else 8192, 12288, device=dev).bfloat16(); tab = TK.rope_table(4096, 128, device=dev)
            msr = time_ms(lambda: CK.rope_(q, tab, 4096, 32, 32, 128))
            g = torch.randn(1 << 20 if SMALL else 202383360, device=dev).bfloat16()
            mss = time_ms(lambda: CK.sumsq(g))
            rec("rmsnorm", y=relerr(y1, y0), rstd=relerr(r1, r0), dx=relerr(dx1, dx0), dw=relerr(dw1, dw0), dx_dres=dxr,
                fwd_ms_8192x4096=ms, fwd_gbs=2 * xb.numel() * 2 / ms / 1e6, bwd_dres_ms=msb,
                bwd_gbs=4 * xb.numel() * 2 / msb / 1e6, rope_ms=msr, rope_gbs=2 * 8192 * 8192 * 2 / msr / 1e6,
                sumsq_ms=mss, sumsq_gbs=g.numel() * 2 / mss / 1e6)
        chk("rmsnorm", t_rms)

        def t_addnorm():
            x = torch.randn(M, D, device=dev).bfloat16(); res = torch.randn(M, D, device=dev); w = (1 + 0.1 * torch.randn(D, device=dev)).bfloat16()
            dy = torch.randn(M, D, device=dev).bfloat16()
            y0, ro0, r0 = TK.add_rmsnorm_fwd(x, res, w, 1e-5); y1, ro1, r1 = CK.add_rmsnorm_fwd(x, res, w, 1e-5)
            dx0, dw0 = TK.rmsnorm_bwd(dy, ro0, w, r0); dx1, dw1 = CK.rmsnorm_bwd(dy, ro1, w, r1)
            rec("add_rmsnorm", y=relerr(y1, y0), res=relerr(ro1, ro0), rstd=relerr(r1, r0), dx=relerr(dx1, dx0), dw=relerr(dw1, dw0))
        chk("add_rmsnorm", t_addnorm)

        def t_gated():
            x = torch.randn(M, D, device=dev).bfloat16(); z = torch.randn(M, D, device=dev).bfloat16(); w = (1 + 0.1 * torch.randn(D, device=dev)).bfloat16()
            dy = torch.randn(M, D, device=dev).bfloat16()
            y0, r0 = TK.rmsnorm_gated_fwd(x, z, w, 1e-5, D); y1, r1 = CK.rmsnorm_gated_fwd(x, z, w, 1e-5, D)
            g0 = TK.rmsnorm_gated_bwd(dy, x, z, w, r0, D); g1 = CK.rmsnorm_gated_bwd(dy, x, z, w, r1, D)
            rec("rmsnorm_gated", y=relerr(y1, y0), dx=relerr(g1[0], g0[0]), dz=relerr(g1[1], g0[1]), dw=relerr(g1[2], g0[2]))
        chk("rmsnorm_gated", t_gated)

        def t_rope():
            S, H, KVH, hd = 256, 8, 4, 128
            tab = TK.rope_table(S, hd, device=dev)
            q = torch.randn(2 * S, (H + 2 * KVH) * hd, device=dev).bfloat16()
            a = TK.rope_(q.clone(), tab, S, H, KVH, hd); b = CK.rope_(q.clone(), tab, S, H, KVH, hd)
            ai = TK.rope_(a.clone(), tab, S, H, KVH, hd, inverse=True); bi = CK.rope_(b.clone(), tab, S, H, KVH, hd, inverse=True)
            rec("rope", fwd=relerr(b, a), inv=relerr(bi, ai), roundtrip=relerr(bi, q))
            tab2 = TK.rope_table(S, 64, device=dev)
            a = TK.rope_(q.clone(), tab2, S, H, KVH, hd, 64); b = CK.rope_(q.clone(), tab2, S, H, KVH, hd, 64)
            rec("rope_partial", fwd=relerr(b, a))
        chk("rope", t_rope)

        def t_swiglu():
            gu = torch.randn(M, 2 * 11008, device=dev).bfloat16(); ds = torch.randn(M, 11008, device=dev).bfloat16()
            rec("swiglu", fwd=relerr(CK.swiglu_fwd(gu), TK.swiglu_fwd(gu)), bwd=relerr(CK.swiglu_bwd(ds, gu), TK.swiglu_bwd(ds, gu)))
        chk("swiglu", t_swiglu)

        def t_emb():
            V = 32000
            w = torch.randn(V, D, device=dev).bfloat16(); tok = torch.randint(0, V, (M,), device=dev, dtype=torch.int32)
            dx = torch.randn(M, D, device=dev).bfloat16()
            o0 = TK.embedding_fwd(tok, w); o1 = CK.embedding_fwd(tok, w)
            g0 = TK.embedding_bwd(dx, tok, torch.empty(V, D, device=dev)); g1 = CK.embedding_bwd(dx, tok, torch.empty(V, D, device=dev))
            g2 = CK.embedding_bwd(dx, tok.long(), torch.empty(V, D, device=dev, dtype=torch.bfloat16))
            rec("embedding", fwd=relerr(o1, o0), bwd_f32=relerr(g1, g0), bwd_bf16=relerr(g2, g0))
        chk("embedding", t_emb)

        def t_ce():
            V, Dm, Mm = 32000, 1024, 2048
            h = (0.5 * torch.randn(Mm, Dm, device=dev)).bfloat16(); w = (0.05 * torch.randn(V, Dm, device=dev)).bfloat16()
            lab = torch.randint(0, V, (Mm,), device=dev); lab[::7] = -100
            dw0 = torch.zeros(V, Dm, device=dev); dw1 = torch.zeros(V, Dm, device=dev, dtype=torch.bfloat16)
            l0, dh0 = TK.linear_ce_fwd_bwd(h.float(), w.float(), lab, dw0)
            l1, dh1 = CK.linear_ce_fwd_bwd(h, w, lab, dw1, chunk_rows=512)
            rec("linear_ce", loss_ref=l0.item(), loss=l1.item(), dh=relerr(dh1, dh0), dw=relerr(dw1, dw0))
        chk("linear_ce", t_ce)

        def t_adam():
            n = 1 << 20
            p = torch.randn(n, device=dev); g = torch.randn(n, device=dev).bfloat16()
            m = torch.zeros(n, device=dev); v = torch.zeros(n, device=dev)
            p2, m2, v2 = p.clone(), m.clone(), v.clone(); lp = torch.empty(n, device=dev, dtype=torch.bfloat16); lp2 = lp.clone()
            sc = torch.tensor(0.5, device=dev)
            for step in (1, 2, 3):
                TK.adamw_step(p, g, m, v, lp, 1e-3, 0.9, 0.95, 1e-8, 0.1, step, sc)
                CK.adamw_step(p2, g, m2, v2, lp2, 1e-3, 0.9, 0.95, 1e-8, 0.1, step, sc)
            s0 = TK.sumsq(g); s1 = CK.sumsq(g)
            rec("adamw", p=relerr(p2, p), m=relerr(m2, m), v=relerr(v2, v), lowp=relerr(lp2, lp), sumsq=abs(s1.item() - s0.item()) / s0.item())
        chk("adamw", t_adam)

        def t_conv():
            S, C = 256, 1024
            x = torch.randn(2 * S, C, device=dev).bfloat16(); w = (0.5 * torch.randn(C, 4, device=dev)).bfloat16()
            b = (0.1 * torch.randn(C, device=dev)).bfloat16(); dy = torch.randn(2 * S, C, device=dev).bfloat16()
            y0 = TK.causal_conv1d_fwd(x, w, b, S); y1 = CK.causal_conv1d_fwd(x, w, b, S)
            g0 = TK.causal_conv1d_bwd(dy, x, w, b, S); g1 = CK.causal_conv1d_bwd(dy, x, w, b, S)
            rec("conv1d", fwd=relerr(y1, y0), dx=relerr(g1[0], g0[0]), dw=relerr(g1[1], g0[1]), db=relerr(g1[2], g0[2]))
        chk("conv1d", t_conv)

    if "ssd" in groups:
        def t_ssd():
            for (Bs, S, H, P, G, N) in [(2, 256, 8, 64, 1, 128), (1, 384, 8, 64, 2, 64), (2, 4096, 128, 64, 1, 128)]:
                M = Bs * S
                x = torch.randn(M, H, P, device=dev).bfloat16().requires_grad_()
                dt = (torch.randn(M, H, device=dev) * 0.5 - 1.0).bfloat16().requires_grad_()
                A = -(torch.rand(H, device=dev) * 4 + 0.5)
                Bm = (torch.randn(M, G, N, device=dev) * 0.3).bfloat16().requires_grad_()
                Cm = (torch.randn(M, G, N, device=dev) * 0.3).bfloat16().requires_grad_()
                D = torch.randn(H, device=dev); bias = torch.randn(H, device=dev) * 0.2
                dy = torch.randn(M, H, P, device=dev).bfloat16()
                r = dict(B=Bs, S=S, H=H, P=P, G=G, N=N)
                y1 = CK.ssd_scan_fwd(x.detach(), dt.detach(), A, Bm.detach(), Cm.detach(), D, bias, S, 256)
                g1 = CK.ssd_scan_bwd(dy, x.detach(), dt.detach(), A, Bm.detach(), Cm.detach(), D, bias, S, 256)
                torch.cuda.synchronize()
                if M <= 4096:
                    Al, Dl, bl = A.clone().requires_grad_(), D.clone().requires_grad_(), bias.clone().requires_grad_()
                    y0 = TK.ssd_scan_chunked(x, dt, Al, Bm, Cm, Dl, bl, S, 128)
                    g0 = torch.autograd.grad(y0, [x, dt, Al, Bm, Cm, Dl, bl], dy.float())
                    r.update(y=relerr(y1, y0))
                    for nm, a, b in zip(["dx", "ddt", "dA", "dB", "dC", "dD", "dbias"], g1, g0):
                        r[nm] = relerr(a, b)
                else:
                    r["fwd_ms"] = time_ms(lambda: CK.ssd_scan_fwd(x.detach(), dt.detach(), A, Bm.detach(), Cm.detach(), D, bias, S, 256))
                    r["bwd_ms"] = time_ms(lambda: CK.ssd_scan_bwd(dy, x.detach(), dt.detach(), A, Bm.detach(), Cm.detach(), D, bias, S, 256))
                    r["aten_fwd_ms"] = time_ms(lambda: TK.ssd_scan_chunked(x.detach(), dt.detach(), A, Bm.detach(), Cm.detach(), D, bias, S, 256), iters=3)
                    r["finite"] = bool(torch.isfinite(y1).all()) and all(bool(torch.isfinite(t).all()) for t in g1)
                rec("ssd", **r)
        try:
            t_ssd()
        except Exception as ex:
            rec("ssd", ok=False, error=repr(ex)[:500], tb=traceback.format_exc()[-900:])

    if "selscan" in groups:
        def t_sel():
            for (Bs, S, Dm, N, use_z) in [(2, 64, 64, 16, True), (1, 96, 32, 16, False), (2, 4096, 5120, 16, True)]:
                M = Bs * S
                u = torch.randn(M, Dm, device=dev).bfloat16().requires_grad_()
                dl = (torch.randn(M, Dm, device=dev) * 0.5 - 1.0).bfloat16().requires_grad_()
                A = (-(torch.rand(Dm, N, device=dev) * 4 + 0.5)).requires_grad_()
                Bm = (torch.randn(M, N, device=dev) * 0.5).bfloat16().requires_grad_()
                Cm = (torch.randn(M, N, device=dev) * 0.5).bfloat16().requires_grad_()
                D = torch.randn(Dm, device=dev).requires_grad_(); bias = (torch.randn(Dm, device=dev) * 0.2).requires_grad_()
                z = torch.randn(M, Dm, device=dev).bfloat16().requires_grad_() if use_z else None
                dy = torch.randn(M, Dm, device=dev).bfloat16()
                dd = lambda t: None if t is None else t.detach()
                r = dict(B=Bs, S=S, Dm=Dm, N=N, z=use_z)
                y1 = CK.selective_scan_fwd(dd(u), dd(dl), dd(A), dd(Bm), dd(Cm), dd(D), dd(z), dd(bias), S)
                g1 = CK.selective_scan_bwd(dy, dd(u), dd(dl), dd(A), dd(Bm), dd(Cm), dd(D), dd(z), dd(bias), S)
                torch.cuda.synchronize()
                if M <= 512:
                    y0 = TK.selective_scan_fwd(u, dl, A, Bm, Cm, D, z, bias, S)
                    ins = [u, dl, A, Bm, Cm, D] + ([z] if use_z else []) + [bias]
                    g0 = list(torch.autograd.grad(y0, ins, dy.float()))
                    names = ["du", "ddelta", "dA", "dB", "dC", "dD"] + (["dz"] if use_z else []) + ["dbias"]
                    mine = list(g1[:6]) + ([g1[6]] if use_z else []) + [g1[7]]
                    r.update(y=relerr(y1, y0))
                    for nm, a, b in zip(names, mine, g0):
                        r[nm] = relerr(a, b)
                else:
                    r["fwd_ms"] = time_ms(lambda: CK.selective_scan_fwd(dd(u), dd(dl), dd(A), dd(Bm), dd(Cm), dd(D), dd(z), dd(bias), S))
                    r["bwd_ms"] = time_ms(lambda: CK.selective_scan_bwd(dy, dd(u), dd(dl), dd(A), dd(Bm), dd(Cm), dd(D), dd(z), dd(bias), S))
                    r["finite"] = bool(torch.isfinite(y1).all()) and all(bool(torch.isfinite(t).all()) for t in g1 if t is not None)
                rec("selscan", **r)
        try:
            t_sel()
        except Exception as ex:
            rec("selscan", ok=False, error=repr(ex)[:500], tb=traceback.format_exc()[-900:])

    if "attn" in groups:
        for (B, S, H, KVH, hd) in [(1, 128, 1, 1, 128), (2, 256, 4, 2, 128), (1, 384, 2, 1, 128), (1, 512, 2, 2, 64), (2, 4096, 32, 32, 128)][:(4 if SMALL else None)]:
          try:
              qkv = torch.randn(B * S, (H + 2 * KVH) * hd, device=dev).bfloat16()
              do = torch.randn(B * S, H * hd, device=dev).bfloat16()
              sc = hd ** -0.5
              r = dict(B=B, S=S, H=H, KVH=KVH, hd=hd)
              o1, l1 = CK.attn_fwd(qkv, B, S, H, KVH, hd, sc)
              torch.cuda.synchronize()
              if S <= 1024:
                  o0, l0 = TK.attn_fwd(qkv, B, S, H, KVH, hd, sc)
                  r.update(o=relerr(o1, o0), lse=relerr(l1, l0))
                  g1 = CK.attn_bwd(do, qkv, o1, l1, B, S, H, KVH, hd, sc)
                  g0 = TK.attn_bwd(do, qkv, o0, l0, B, S, H, KVH, hd, sc)
                  r.update(dqkv=relerr(g1, g0))
              else:
                  o0 = CK._sdpa_fwd(qkv, B, S, H, KVH, hd, sc)
                  r.update(o_vs_sdpa=relerr(o1, o0))
                  fl = 4 * B * H * S * S * hd / 2
                  ms = time_ms(lambda: CK.attn_fwd(qkv, B, S, H, KVH, hd, sc))
                  ms0 = time_ms(lambda: CK._sdpa_fwd(qkv, B, S, H, KVH, hd, sc))
                  r.update(fwd_ms=ms, fwd_tflops=fl / ms / 1e9, sdpa_fwd_ms=ms0, sdpa_fwd_tflops=fl / ms0 / 1e9)
                  ms = time_ms(lambda: CK.attn_bwd(do, qkv, o1, l1, B, S, H, KVH, hd, sc))
                  r.update(bwd_ms=ms, bwd_tflops=2.5 * fl / ms / 1e9)
              rec("attn", **r)
          except Exception as ex:
              rec("attn", B=B, S=S, H=H, KVH=KVH, hd=hd, ok=False, error=repr(ex)[:500])

    rec("done", launches=CK.launch_count())


if __name__ == "__main__":
    g = sys.argv[1:] or ["gemm", "elem"]
    try:
        main(g)
    except Exception as ex:
        rec("fatal", error=repr(ex)[:500], tb=traceback.format_exc()[-1500:])
        raise
