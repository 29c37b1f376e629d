"""Cost of the z-losses on the GPU (CUDA events, alternated rounds, medians):

    python scripts/z_loss_bench.py [--rounds 7] [--iters 20] [--out z_loss_bench.json]

* head: fused linear + cross-entropy forward + backward (``ops.linear_cross_entropy``, c = 0) against the z-loss entry
  (``ops.linear_cross_entropy_z``, c = 1e-4) at B 2 x S 4096 tokens, D 4096, V 32000 and 128256; and the gradient
  kernels alone on one 4096-row logits chunk (``ce_grad_inplace`` against ``ce_zloss_grad_inplace``);
* router: the router z-loss forward (``router_z_fwd``: lse + mean of squares) and backward (``router_z_bwd``) at the
  Qwen3-MoE block (T 8192, E 128), next to the routing kernels they accompany (``moe_route``, ``moe_route_bwd``).

The card's name, power limit and SM clock are printed with the numbers.  Nothing is written unless --out is given."""
import argparse
import json
import statistics
import subprocess
import sys
import os

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from fms_fsdp_b200 import ops  # noqa: E402
from fms_fsdp_b200.ops import cuda_kernels as CK  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unavailable ({e})"


def time_ms(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def alternate(cases, rounds, iters):
    """cases: {name: fn}.  Every round times every case once, in an order rotated by the round; medians per case."""
    for fn in cases.values():          # warm-up of every shape in the timed window
        fn()
        fn()
    torch.cuda.synchronize()
    names = list(cases)
    got = {n: [] for n in names}
    for r in range(rounds):
        for n in names[r % len(names):] + names[:r % len(names)]:
            got[n].append(time_ms(cases[n], iters))
    return {n: dict(median_ms=statistics.median(v), min_ms=min(v), max_ms=max(v)) for n, v in got.items()}


def head(V, rounds, iters, M=8192, D=4096):
    g = torch.Generator(device="cuda").manual_seed(0)
    h = torch.randn(M, D, generator=g, device="cuda").bfloat16().requires_grad_()
    w = (torch.randn(V, D, generator=g, device="cuda") / D ** 0.5).bfloat16().requires_grad_()
    labels = torch.randint(0, V, (M,), generator=g, device="cuda")

    def plain():
        ops.linear_cross_entropy(h, w, labels).backward()

    def zloss():
        ops.linear_cross_entropy_z(h, w, labels, 1e-4)[0].backward()

    res = alternate({"ce": plain, "ce_z": zloss}, rounds, iters)
    # the gradient kernels alone on one 4096-row chunk (the head's chunk size); each call rewrites the same buffer
    rows = 4096
    lg0 = CK.gemm(h.detach()[:rows], w.detach(), "nt")
    lg = lg0.clone()
    lab = labels[:rows]
    n_valid = torch.full((), float(rows), device="cuda")
    loss_sum = torch.zeros((), device="cuda")
    part = torch.empty(rows, 2, device="cuda")
    kern = alternate({"ce_grad_inplace": lambda: CK._C.ce_grad_inplace(lg, lab, n_valid, loss_sum, -100),
                      "ce_zloss_grad_inplace": lambda: CK._C.ce_zloss_grad_inplace(lg, lab, n_valid, part, -100, 1e-4),
                      "copy_back": lambda: lg.copy_(lg0)}, rounds, iters)
    res.update(kern)
    res["chunk_bytes_per_pass"] = rows * V * 2
    return res


def router(rounds, iters, T=8192, E=128, k=8):
    g = torch.Generator(device="cuda").manual_seed(0)
    logits = torch.randn(T, E, generator=g, device="cuda")
    ids, wts, probs = CK.moe_route(logits, k, True)
    plan, _ = CK.moe_plan(ids, probs)
    dw = torch.randn(T, k, generator=g, device="cuda")
    lse, _ = CK.router_z_fwd(logits)
    dl = CK.moe_route_bwd(probs, ids, wts, dw, plan, True, 0.0)
    return alternate({"moe_route": lambda: CK.moe_route(logits, k, True),
                      "router_z_fwd": lambda: CK.router_z_fwd(logits),
                      "moe_route_bwd": lambda: CK.moe_route_bwd(probs, ids, wts, dw, plan, True, 0.0),
                      "router_z_bwd": lambda: CK.router_z_bwd(dl, probs, lse, 1e-9)}, rounds, iters)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("z_loss_bench needs a GPU")
    out = dict(gpu_before=gpu_info(), rounds=a.rounds, iters=a.iters)
    out["head_V32000"] = head(32000, a.rounds, a.iters)
    out["head_V128256"] = head(128256, a.rounds, a.iters)
    out["router_qwen3_moe"] = router(a.rounds, a.iters * 10)
    out["gpu_after"] = gpu_info()
    out["fallbacks"] = CK.fallback_count()
    print(json.dumps(out, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
