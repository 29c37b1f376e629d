"""q / k / v projection biases on one H100: the QKV GEMM with the bias + RoPE epilogue against the RoPE epilogue alone,
``bias_grad`` at real block shapes, and the attention node's forward + backward with and without the bias, alternated
round by round in one process.

    python scripts/qkv_bias_bench.py [--out results/qkv_bias_bench.json] [--rounds 15]

Prints (and writes) the card, its power limit and max SM clock, read in the same run; times come from CUDA events around
many launches, reported as the median over rounds with the min and max.  ``bias_grad`` bytes count what it must move: the
bf16 gradient read once (2 B per element); its fp32 row-slice partials stay mostly in L2 and are not counted.  HBM3
data-sheet bandwidth of the H100 SXM: 3.35 TB/s.  The allocator peak of a whole training step comes from ``bench.py
--model qwen2.5_1.5b`` (its ``mem_gb``); ``plan_gib`` here is the memory plan of that run for comparison.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from fms_fsdp_b200 import ops                                      # noqa: E402
from fms_fsdp_b200.ops import cuda_kernels as CK                    # noqa: E402
from fms_fsdp_b200.utils.config_utils import get_model_config      # noqa: E402
from fms_fsdp_b200.utils.memory_plan import plan_llama             # noqa: E402

HBM_TBS = 3.35
B, S = 2, 4096


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def timed(fn, iters):
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


def _shape(variant):
    c = get_model_config(variant)
    return c, c.nheads, c.kv_heads, c.head_dim, c.emb_dim, (c.nheads + 2 * c.kv_heads) * c.head_dim


def gemm(variant, rounds, iters=50):
    c, H, KVH, hd, D, N = _shape(variant)
    x = torch.randn(B * S, D, device="cuda").to(torch.bfloat16)
    w = (torch.randn(N, D, device="cuda") * D ** -0.5).to(torch.bfloat16)
    bias = torch.randn(N, device="cuda").to(torch.bfloat16)
    rope = (ops.torch_kernels.rope_table(S, hd, c.rope_theta, device="cuda"), S, hd, H, KVH)
    with_b, without = [], []
    for _ in range(rounds):
        without.append(timed(lambda: CK.gemm(x, w, "nt", rope=rope), iters))
        with_b.append(timed(lambda: CK.gemm(x, w, "nt", rope=rope, bias=bias), iters))
    over = [b / a - 1 for a, b in zip(without, with_b)]
    return {"shape": f"{variant} M{B * S} N{N} K{D}", "rounds": rounds, "rope_us": spread(without),
            "rope_bias_us": spread(with_b), "overhead": {k: round(v, 4) for k, v in
                                                          (("median", statistics.median(over)), ("min", min(over)),
                                                           ("max", max(over)))},
            "rope_bias_tflops_median": round(2.0 * B * S * N * D / statistics.median(with_b) / 1e6, 1)}


def bias_grad(variant, rounds, iters=200):
    _, _, _, _, _, N = _shape(variant)
    dy = torch.randn(B * S, N, device="cuda").to(torch.bfloat16)
    ts = [timed(lambda: CK.bias_grad(dy), iters) for _ in range(rounds)]
    nbytes = 2 * B * S * N
    return {"shape": f"{variant} T{B * S} N{N}", "us": spread(ts),
            "TBps_median": round(nbytes / statistics.median(ts) / 1e6, 3), "bytes_per_call": nbytes,
            "hbm_datasheet_TBps": HBM_TBS}


def node(variant, rounds, iters=10):
    """qkv_attention forward + backward, with and without the bias, alternated round by round."""
    c, H, KVH, hd, D, N = _shape(variant)
    h = torch.randn(B, S, D, device="cuda").to(torch.bfloat16).requires_grad_()
    w = (torch.randn(N, D, device="cuda") * D ** -0.5).to(torch.bfloat16).requires_grad_()
    bias = torch.randn(N, device="cuda").to(torch.bfloat16).requires_grad_()
    table = ops.torch_kernels.rope_table(S, hd, c.rope_theta, device="cuda")
    do = torch.randn(B, S, H * hd, device="cuda").to(torch.bfloat16)

    def step(biased):
        o = ops.qkv_attention(h, w, table, H, KVH, hd, qkv_bias=bias if biased else None)
        torch.autograd.grad(o, (h, w, bias) if biased else (h, w), do)

    plain, biased = [], []
    for _ in range(rounds):
        plain.append(timed(lambda: step(False), iters))
        biased.append(timed(lambda: step(True), iters))
    over = [b / a - 1 for a, b in zip(plain, biased)]
    return {"shape": f"{variant} B{B} S{S}", "rounds": rounds, "plain_us": spread(plain), "bias_us": spread(biased),
            "overhead": {k: round(v, 4) for k, v in (("median", statistics.median(over)), ("min", min(over)),
                                                      ("max", max(over)))}}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--out", default="")
    p.add_argument("--rounds", type=int, default=15)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("qkv_bias_bench.py measures on the GPU; no CUDA device found")
    res = {"card": card(),
           "qkv_gemm": [gemm(v, a.rounds) for v in ("qwen2.5_1.5b", "qwen2.5_7b")],
           "bias_grad": [bias_grad(v, a.rounds) for v in ("qwen2.5_0.5b", "qwen2.5_1.5b", "qwen2.5_7b")],
           "attention_node": [node(v, a.rounds) for v in ("qwen2.5_1.5b", "qwen2.5_7b")],
           "plan_gib_qwen2.5_1.5b_B2_S4096_1gpu": round(plan_llama("qwen2.5_1.5b", gpus=1).total_gib, 2),
           "aten_fallbacks": CK.fallback_count()}
    print(json.dumps(res, indent=1), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
