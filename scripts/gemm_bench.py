"""Every GEMM of the headline step (Llama2-1.4B, batch 2 x seq 4096 = 8192 tokens, one GPU) at its real shape, layout,
epilogue and output dtype: the 128x128 tile (forced), the launcher's own choice (auto), the 128x256 tile (forced) and
torch.matmul (cuBLAS, plain store) on the same operands.  The implementations alternate within each shape, three rounds;
each figure is the median round.  Prints the card, its power limit and SM clocks read in the same run, then one line
per shape; writes $DIAG_OUT/gemm_bench.json (default diag_out/ in the repository root).

    python scripts/gemm_bench.py [--iters-ms 60]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from fms_fsdp_b200.ops import cuda_kernels as CK

T, D, F, H, KVH, HD, V, S = 8192, 2048, 6144, 16, 4, 128, 32000, 4096
QKV = (H + 2 * KVH) * HD
HEAD_ROWS = 4096          # the fused linear-CE head runs in chunks of 4096 rows
bf16, f32 = torch.bfloat16, torch.float32

# (name, layout, M, N, K, epilogue, output dtype, launches per step); N of the SwiGLU forward is 2F (the fused weight)
SHAPES = [
    ("qkv fwd", "nt", T, QKV, D, "rope", bf16, 24),
    ("o fwd", "nt", T, D, H * HD, "residual", bf16, 24),
    ("gate/up fwd", "nt", T, 2 * F, D, "swiglu", bf16, 24),
    ("down fwd", "nt", T, D, F, "residual", bf16, 24),
    ("down dgrad", "nn", T, F, D, "swiglu_bwd", bf16, 24),
    ("down wgrad", "tn", D, F, T, "store", bf16, 24),
    ("gate/up dgrad", "nn", T, D, 2 * F, "store", bf16, 24),
    ("gate/up wgrad", "tn", 2 * F, D, T, "store", bf16, 24),
    ("o dgrad", "nn", T, H * HD, D, "store", bf16, 24),
    ("o wgrad", "tn", D, H * HD, T, "store", bf16, 24),
    ("qkv dgrad", "nn", T, D, QKV, "store", bf16, 24),
    ("qkv wgrad", "tn", QKV, D, T, "store", bf16, 24),
    ("head logits", "nt", HEAD_ROWS, V, D, "store", bf16, 2),
    ("head dh", "nn", HEAD_ROWS, D, V, "store", bf16, 2),
    ("head dW", "tn", V, D, HEAD_ROWS, "accumulate", bf16, 2),
]
TILE = {"narrow": 1, "auto": 0, "wide": 2}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return dict(zip(q.split(","), (x.strip() for x in r.stdout.strip().split(","))))
    except Exception as ex:          # the numbers stay usable; say why the card could not be read
        return {"error": repr(ex)}


def operands(layout, M, N, K, g):
    r = lambda *s: (torch.randn(*s, generator=g, device="cuda") * 0.5).to(bf16)
    if layout == "nt":
        return r(M, K), r(N, K)
    if layout == "nn":
        return r(M, K), r(K, N)
    return r(K, M), r(K, N)


def runner(row, a, b, g):
    """(ours, cublas): closures that launch the GEMM of this row once."""
    name, layout, M, N, K, epi, odt, _ = row
    mm = {"nt": lambda: a @ b.t(), "nn": lambda: a @ b, "tn": lambda: a.t() @ b}[layout]
    if epi == "swiglu":
        return (lambda: CK.gated_up_fwd(a, b)), mm
    if epi == "swiglu_bwd":
        gu = (torch.randn(M, 2 * N, generator=g, device="cuda")).to(bf16)
        return (lambda: CK.gated_down_bwd(a, b, gu)), mm
    out = torch.zeros(M, N, dtype=odt, device="cuda")
    if epi == "rope":
        ang = torch.arange(S, device="cuda", dtype=f32)[:, None] * (1e4 ** (-torch.arange(0, HD, 2, device="cuda") / HD))
        table = torch.stack((ang.cos(), ang.sin()), -1).contiguous()
        return (lambda: CK.gemm(a, b, layout, out=out, rope=(table, S, HD, H, KVH))), mm
    if epi == "residual":
        res = torch.randn(M, N, generator=g, device="cuda").to(bf16)
        return (lambda: CK.gemm(a, b, layout, out=out, residual=res)), mm
    return (lambda: CK.gemm(a, b, layout, out=out, accumulate=(epi == "accumulate"))), mm


def time_ms(fn, target_ms):
    """Mean device time of one launch over a window of about target_ms."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); fn(); e1.record(); torch.cuda.synchronize()
    n = max(5, int(target_ms / max(e0.elapsed_time(e1), 1e-3)))
    e0.record()
    for _ in range(n):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters-ms", type=float, default=60.0, help="timed window per implementation and round")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    can_force = hasattr(CK._C, "_set_gemm_tile")
    impls = ["narrow", "auto", "wide", "cublas"] if can_force else ["auto", "cublas"]
    info = card()
    print(json.dumps({"card": info}), flush=True)
    g = torch.Generator(device="cuda").manual_seed(0)
    rows, step_ms = [], {k: 0.0 for k in impls}
    for row in SHAPES:
        name, layout, M, N, K, epi, odt, count = row
        a, b = operands(layout, M, N, K, g)
        ours, mm = runner(row, a, b, g)
        fns = {k: ours for k in impls if k != "cublas"}
        fns["cublas"] = mm

        def run(k):
            if can_force and k != "cublas":
                CK._C._set_gemm_tile(TILE[k])
            try:
                return time_ms(fns[k], args.iters_ms)
            finally:
                if can_force:
                    CK._C._set_gemm_tile(0)

        for k in impls:                      # warm-up: module loads, cuBLAS heuristics, clocks
            run(k); run(k)
        ts = {k: [] for k in impls}
        for _ in range(args.rounds):
            for k in impls:
                ts[k].append(run(k))
        flop = 2.0 * M * N * K
        rec = {"name": name, "layout": layout, "M": M, "N": N, "K": K, "epi": epi, "out": str(odt).split(".")[-1],
               "per_step": count}
        for k in impls:
            s = sorted(ts[k])
            rec[k] = {"ms": s[len(s) // 2], "min_ms": s[0], "max_ms": s[-1], "tflops": flop / s[len(s) // 2] / 1e9}
            step_ms[k] += count * s[len(s) // 2]
        rows.append(rec)
        print(f"{name:14s} {layout} M{M:6d} N{N:6d} K{K:6d} {epi:10s} "
              + " ".join(f"{k}={rec[k]['tflops']:6.1f}TF({rec[k]['ms']:.3f}ms)" for k in impls), flush=True)
        del a, b, ours, mm, fns
        torch.cuda.empty_cache()
    total_flop = sum(2.0 * r["M"] * r["N"] * r["K"] * r["per_step"] for r in rows)
    summary = {k: {"ms_per_step": step_ms[k], "tflops": total_flop / step_ms[k] / 1e9} for k in impls}
    info_after = card()
    print(json.dumps({"step_gemm": summary, "card_after": info_after}), flush=True)
    out_dir = os.environ.get("DIAG_OUT") or os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                                         "diag_out")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "gemm_bench.json"), "w") as fh:
        json.dump({"card": info, "card_after": info_after, "rows": rows, "step_gemm": summary}, fh, indent=1)


if __name__ == "__main__":
    main()
