"""QK-norm on one H100: the stand-alone ``qk_norm_rope`` / ``qk_norm_bwd`` kernels at real block shapes, and the
attention node's forward + backward with and without QK-norm, alternated in one process.

    python scripts/qk_norm_bench.py [--out results/qk_norm_bench.json] [--rounds 15]

Prints (and writes) the card, its power limit and max SM clock, read in the same run; kernel times come from CUDA events
around many launches.  Achieved bytes/s count what each kernel must move: forward reads the q / k heads and writes them
back plus the pre-norm copy (3 x 2 B per element) and rstd (4 B per head-row); backward reads the gradient and the
pre-norm copy, writes dx (3 x 2 B per element) and reads rstd.  The RoPE table and the per-CTA dw partials stay in L2 and
are not counted.  HBM3 data-sheet bandwidth of the H100 SXM: 3.35 TB/s.
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

HBM_TBS = 3.35
SHAPES = ("llama2_1.4b", "qwen3_8b")


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


def kernels(variant, B=2, S=4096, iters=200):
    c = get_model_config(variant)
    H, KVH, hd = c.nheads, c.kv_heads, c.head_dim
    T, nh = B * S, H + KVH
    qkv = torch.randn(T, (H + 2 * KVH) * hd, device="cuda").to(torch.bfloat16)
    wq = torch.ones(hd, device="cuda", dtype=torch.bfloat16)    # unit gains keep the in-place backward's values bounded
    wk = torch.ones(hd, device="cuda", dtype=torch.bfloat16)
    table = ops.torch_kernels.rope_table(S, hd, c.rope_theta, device="cuda")
    xqk, rstd = CK.qk_norm_rope(qkv, wq, wk, table, S, H, KVH, hd, 1e-6)
    d = torch.randn_like(qkv)
    fwd = timed(lambda: CK.qk_norm_rope(qkv, wq, wk, table, S, H, KVH, hd, 1e-6), iters)
    bwd = timed(lambda: CK.qk_norm_bwd(d, xqk, rstd, wq, wk, H, KVH, hd), iters)   # in place on d: values drift, bytes do not
    nbytes = 3 * 2 * T * nh * hd + 4 * T * nh
    return {"shape": f"{variant} B{B} S{S} H{H} KVH{KVH} hd{hd}",
            "qk_norm_rope_us": round(fwd, 1), "qk_norm_rope_TBps": round(nbytes / fwd / 1e6, 3),
            "qk_norm_bwd_us": round(bwd, 1), "qk_norm_bwd_TBps": round(nbytes / bwd / 1e6, 3),
            "bytes_per_call": nbytes, "hbm_datasheet_TBps": HBM_TBS}


def node(variant, rounds, B=2, S=4096, iters=10):
    """qkv_attention forward + backward, with and without QK-norm, alternated round by round."""
    c = get_model_config(variant)
    H, KVH, hd, D = c.nheads, c.kv_heads, c.head_dim, c.emb_dim
    h = torch.randn(B, S, D, device="cuda").to(torch.bfloat16).requires_grad_()
    w = (torch.randn((H + 2 * KVH) * hd, D, device="cuda") * D ** -0.5).to(torch.bfloat16).requires_grad_()
    wq = torch.ones(hd, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    wk = torch.ones(hd, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    table = ops.torch_kernels.rope_table(S, hd, c.rope_theta, device="cuda")
    do = torch.randn(B, S, H * hd, device="cuda").to(torch.bfloat16)

    def step(qk):
        o = ops.qkv_attention(h, w, table, H, KVH, hd, qk_norm=(wq, wk, 1e-6) if qk else None)
        torch.autograd.grad(o, (h, w, wq, wk) if qk else (h, w), do)

    # the projection alone: the plain node's GEMM carries the RoPE epilogue, the QK-norm node's is a plain store
    h2, wd = h.detach().reshape(B * S, D), w.detach()
    plain, normed, g_rope, g_store = [], [], [], []
    for _ in range(rounds):
        plain.append(timed(lambda: step(False), iters))
        normed.append(timed(lambda: step(True), iters))
        g_rope.append(timed(lambda: CK.gemm(h2, wd, "nt", rope=(table, S, hd, H, KVH)), iters))
        g_store.append(timed(lambda: CK.gemm(h2, wd, "nt"), iters))
    over = [n / p - 1 for p, n in zip(plain, normed)]
    return {"shape": f"{variant} B{B} S{S}", "rounds": rounds,
            "plain_us_median": round(statistics.median(plain), 1), "qk_norm_us_median": round(statistics.median(normed), 1),
            "overhead_median": round(statistics.median(over), 4), "overhead_min": round(min(over), 4),
            "overhead_max": round(max(over), 4),
            "qkv_gemm_rope_epilogue_us_median": round(statistics.median(g_rope), 1),
            "qkv_gemm_store_us_median": round(statistics.median(g_store), 1)}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--out", default="")
    p.add_argument("--rounds", type=int, default=15)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("qk_norm_bench.py measures on the GPU; no CUDA device found")
    res = {"card": card(), "kernels": [kernels(v) for v in SHAPES],
           "attention_node": [node(v, a.rounds) for v in SHAPES], "aten_fallbacks": CK.fallback_count()}
    print(json.dumps(res, indent=1), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
