"""Mixture-of-experts block at the Qwen3-30B-A3B shape (T = 8192 tokens = B2 x S4096, D 2048, 128 experts, top 8,
F 768), timed in one process, alternating:

* ``ops.moe_mlp`` forward + backward (the grouped wgmma GEMMs and the routing kernels of ``csrc/moe.cu``);
* ``ops.gated_mlp`` at D 2048, F 6144 forward + backward: the dense SwiGLU block with exactly the same GEMM FLOPs
  (k F = 6144);
* a per-expert loop of cuBLAS GEMMs in torch over the same routing (the usual eager implementation).

It then times every grouped GEMM and every routing kernel alone with CUDA events and prints grouped-GEMM TFLOP/s on
routed rows (T k) and on padded rows (each expert rounded up to 128), the bandwidth of route / permute / combine from
the bytes they must move, and the card, its power limit and clocks.

    python scripts/moe_bench.py [--iters 20] [--rounds 5]
"""
import argparse
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from fms_fsdp_b200 import ops  # noqa: E402
from fms_fsdp_b200.ops import cuda_kernels as CK  # noqa: E402


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters * 1e-3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("moe_bench needs a GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    T, D, E, k, F = 8192, 2048, 128, 8, 768
    g = torch.Generator(device="cuda").manual_seed(0)
    mk = lambda *s, sc=1.0: (torch.randn(*s, device="cuda", generator=g) * sc).bfloat16().requires_grad_()
    h, res = mk(T, D), mk(T, D)
    wr, w1, w2 = mk(E, D, sc=0.02), mk(E, 2 * F, D, sc=0.02), mk(E, D, F, sc=0.02)
    wg1, wd2 = mk(2 * k * F, D, sc=0.02), mk(D, k * F, sc=0.02)
    dy = torch.randn(T, D, device="cuda", generator=g).bfloat16()

    def moe():
        y, _ = ops.moe_mlp(h, wr, w1, w2, k, True, 0.001, residual=res)
        torch.autograd.grad(y, [h, wr, w1, w2], dy)

    def dense():
        y = ops.gated_mlp(h, wg1, wd2, residual=res)
        torch.autograd.grad(y, [h, wg1, wd2], dy)

    def loop():   # eager reference: routing in torch, one cuBLAS GEMM chain per expert
        hh = h.detach().requires_grad_()
        lg = (hh @ wr.t()).float()
        p = torch.softmax(lg, -1)
        wts, ids = p.topk(k, dim=-1)
        wts = wts / wts.sum(-1, keepdim=True)
        out = res.detach().clone().float()
        flat = ids.reshape(-1)
        order = torch.argsort(flat, stable=True)
        counts = torch.bincount(flat, minlength=E).tolist()
        tok = order // k
        s = 0
        for e in range(E):
            n = counts[e]
            if n:
                t = tok[s:s + n]
                gu = hh[t] @ w1[e].t()
                act = torch.nn.functional.silu(gu[:, :F]) * gu[:, F:]
                ye = act @ w2[e].t()
                out = out.index_add(0, t, ye.float() * wts.reshape(-1)[order[s:s + n], None])
            s += n
        torch.autograd.grad(out, [hh, wr, w1, w2], dy.float())

    arms = {"moe_mlp": moe, "gated_mlp (same FLOPs)": dense, "per-expert cuBLAS loop": loop}
    times = {n: [] for n in arms}
    for _ in range(a.rounds):
        for n, fn in arms.items():
            times[n].append(timed(fn, a.iters))
    print(f"card: {card}")
    print(f"shape: T {T} D {D} E {E} top-{k} F {F}; forward + backward, median of {a.rounds} rounds x {a.iters} iters")
    for n, ts in times.items():
        print(f"  {n:<26} {statistics.median(ts) * 1e3:8.3f} ms  (min {min(ts) * 1e3:.3f}, max {max(ts) * 1e3:.3f})")

    # ---- the pieces, each timed alone
    with torch.no_grad():
        logits = CK.gemm(h.detach(), wr.detach(), "nt", out_dtype=torch.float32)
        ids, wts, probs = CK.moe_route(logits, k, True)
        plan, _ = CK.moe_plan(ids, probs)
        xp = CK.moe_permute(h.detach(), plan, k, E)
        hp, sp = CK.moe_up_fwd(xp, w1.detach(), plan, T, k)
        yp = CK.moe_down_fwd(sp, w2.detach(), plan, T, k)
        dyp, dw = CK.moe_combine_bwd(dy, yp, plan, wts, E)
        dhp = CK.moe_down_bwd(dyp, w2.detach(), hp, plan, T, k)
        lens = CK.moe_plan_views(plan, T, k, E)[2].long()
        padded = int(((lens + 127) // 128 * 128).sum())
        routed = T * k
        gw1 = torch.empty(E, 2 * F, D, device="cuda", dtype=torch.float32)
        gw2 = torch.empty(E, D, F, device="cuda", dtype=torch.float32)
        gemms = {
            "up nt + SwiGLU": (lambda: CK.moe_up_fwd(xp, w1.detach(), plan, T, k), 2 * D * 2 * F),
            "down nt": (lambda: CK.moe_down_fwd(sp, w2.detach(), plan, T, k), 2 * F * D),
            "down dgrad nn + SwiGLU bwd": (lambda: CK.moe_down_bwd(dyp, w2.detach(), hp, plan, T, k), 2 * D * F),
            "up dgrad nn": (lambda: CK.moe_up_dgrad(dhp, w1.detach(), plan, T, k), 2 * 2 * F * D),
            "w2 wgrad tn (fp32)": (lambda: CK.moe_wgrad(dyp, sp, plan, T, k, gw2), 2 * D * F),
            "w1 wgrad tn (fp32)": (lambda: CK.moe_wgrad(dhp, xp, plan, T, k, gw1), 2 * 2 * F * D),
        }
        print(f"grouped GEMMs: {routed} routed rows, {padded} padded rows")
        tot_t = tot_f = 0.0
        for n, (fn, fpr) in gemms.items():
            t = timed(fn, a.iters)
            tot_t += t
            tot_f += fpr
            print(f"  {n:<28} {t * 1e6:8.1f} us  {fpr * routed / t / 1e12:6.1f} TFLOP/s routed  "
                  f"{fpr * padded / t / 1e12:6.1f} padded")
        print(f"  {'all six':<28} {tot_t * 1e6:8.1f} us  {tot_f * routed / tot_t / 1e12:6.1f} TFLOP/s routed  "
              f"{tot_f * padded / tot_t / 1e12:6.1f} padded")
        mem = {
            "route": (lambda: CK.moe_route(logits, k, True), 4 * T * E * 2 + 8 * T * k),
            "plan (3 kernels)": (lambda: CK.moe_plan(ids, probs), 4 * T * E + 4 * T * k * 3),
            "permute": (lambda: CK.moe_permute(h.detach(), plan, k, E), 2 * D * (routed + padded)),
            "combine": (lambda: CK.moe_combine(yp, plan, wts, res.detach(), E), 2 * D * (routed + 2 * T) + 8 * T * k),
            "combine backward": (lambda: CK.moe_combine_bwd(dy, yp, plan, wts, E), 2 * D * (routed + 2 * padded)),
            "permute backward": (lambda: CK.moe_permute_bwd(xp, plan, T, k, E), 2 * D * (routed + T) + 4 * T * k),
        }
        print("memory-bound kernels (bytes they must move / time):")
        for n, (fn, nbytes) in mem.items():
            t = timed(fn, a.iters)
            print(f"  {n:<28} {t * 1e6:8.1f} us  {nbytes / t / 1e12:5.2f} TB/s")


if __name__ == "__main__":
    main()
