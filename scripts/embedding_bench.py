"""Embedding backward on one H100 at the headline batch: B2 S4096 (M = 8192 tokens), D 4096, V 32000, for three token
streams -- uniform ids, a Zipf stream (probability 1 / rank, as in natural text) and every position the same token --
into a bf16 and an fp32 gradient.

    python scripts/embedding_bench.py [--out results/embedding_bench.json] [--rounds 15]

Times ``cuda_kernels.embedding_bwd(dx, tokens, out)`` as the engine calls it (zeroing ``out``, then the kernels) and,
separately, the kernels alone (``accumulate=True``), from CUDA events around 50 calls; the median over rounds with the
min and max.  Prints the card, its power limit and max SM clock, read in the same run, and the kernel launches per call.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from fms_fsdp_b200.ops import cuda_kernels as CK                    # noqa: E402

B, S, D, V = 2, 4096, 4096, 32000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def timed(fn, iters=50):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1e3      # us


def spread(xs):
    return {"median": round(statistics.median(xs), 1), "min": round(min(xs), 1), "max": round(max(xs), 1)}


def stream(kind, g):
    M = B * S
    if kind == "uniform":
        return torch.randint(0, V, (M,), device="cuda", generator=g)
    if kind == "one_token":
        return torch.full((M,), 4321, device="cuda")
    p = 1.0 / torch.arange(1, V + 1, dtype=torch.float64, device="cuda")
    return torch.multinomial(p, M, replacement=True, generator=g)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--out", default="")
    p.add_argument("--rounds", type=int, default=15)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("embedding_bench.py measures on the GPU; no CUDA device found")
    g = torch.Generator(device="cuda").manual_seed(0)
    dx = (1e-3 * torch.randn(B * S, D, device="cuda", generator=g)).bfloat16()
    res = {"card": card(), "shape": f"B{B} S{S} D{D} V{V}", "cases": []}
    for kind in ("uniform", "zipf", "one_token"):
        tok = stream(kind, g)
        for dtype in (torch.bfloat16, torch.float32):
            out = torch.zeros(V, D, device="cuda", dtype=dtype)
            n0 = CK.launch_count()
            CK.embedding_bwd(dx, tok, out, accumulate=True)
            launches = CK.launch_count() - n0
            call, kern = [], []
            for _ in range(a.rounds):
                call.append(timed(lambda: CK.embedding_bwd(dx, tok, out)))
                kern.append(timed(lambda: CK.embedding_bwd(dx, tok, out, accumulate=True)))
            res["cases"].append({"stream": kind, "grad": str(dtype)[6:], "distinct_tokens": int(tok.unique().numel()),
                                 "launches": launches, "call_us": spread(call), "kernels_us": spread(kern)})
    res["aten_fallbacks"] = CK.fallback_count()
    print(json.dumps(res, indent=1), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
