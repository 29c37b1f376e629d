"""Attention kernels at the headline shape (B2 H32 S4096 hd128, causal): ours vs the library (cuDNN / flash SDPA through
torch), forward and backward, plus numerics vs the fp32 oracle at a small shape.
Writes $DIAG_OUT/attn_bench.json (default diag_out/ in the repository root).   usage: python scripts/attn_bench.py"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from fms_fsdp_b200.ops import cuda_kernels as CK
from fms_fsdp_b200.ops import torch_kernels as TK

dev = "cuda"
out = []


def time_ms(fn, iters=20, warm=5):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()                       # > L2: every timed launch starts cold
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).abs().max() / b.abs().max().clamp(min=1e-6)).item()


torch.manual_seed(0)
# numerics (small, multi-tile, GQA)
B, S, H, KVH, hd = 2, 512, 4, 2, 128
qkv_s = (torch.randn(B * S, (H + 2 * KVH) * hd, device=dev) * 0.8).bfloat16()
do_s = torch.randn(B * S, H * hd, device=dev).bfloat16()
o0, l0 = TK.attn_fwd(qkv_s.float(), B, S, H, KVH, hd, hd ** -0.5)
g0 = TK.attn_bwd(do_s.float(), qkv_s.float(), o0, l0, B, S, H, KVH, hd, hd ** -0.5)
o1, l1 = CK.attn_fwd(qkv_s, B, S, H, KVH, hd, hd ** -0.5)
g1 = CK.attn_bwd(do_s, qkv_s, o1, l1, B, S, H, KVH, hd, hd ** -0.5)
out.append(dict(kind="numerics", o=rel(o1, o0), lse=rel(l1, l0), dqkv=rel(g1, g0)))

# timing at the headline shape
B, S, H, KVH, hd = 2, 4096, 32, 32, 128
qkv = (torch.randn(B * S, (H + 2 * KVH) * hd, device=dev) * 0.8).bfloat16()
do = torch.randn(B * S, H * hd, device=dev).bfloat16()
fl = 4 * B * H * S * S * hd / 2
ms = time_ms(lambda: CK.attn_fwd(qkv, B, S, H, KVH, hd, hd ** -0.5))
out.append(dict(kind="fwd", ms=ms, tflops=fl / ms / 1e9))
o1, l1 = CK.attn_fwd(qkv, B, S, H, KVH, hd, hd ** -0.5)
ms = time_ms(lambda: CK.attn_bwd(do, qkv, o1, l1, B, S, H, KVH, hd, hd ** -0.5))
out.append(dict(kind="bwd", ms=ms, tflops=2.5 * fl / ms / 1e9))

# the library bar: torch SDPA per backend, forward and backward
from torch.nn.attention import SDPBackend, sdpa_kernel
q, k, v = (t.reshape(B, S, H, hd).transpose(1, 2).contiguous().requires_grad_() for t in qkv.view(B * S, 3, H * hd).unbind(1))
dO = do.view(B, S, H, hd).transpose(1, 2).contiguous()
for name, be in (("cudnn", SDPBackend.CUDNN_ATTENTION), ("flash", SDPBackend.FLASH_ATTENTION)):
    try:
        with sdpa_kernel([be]):
            f = lambda: torch.nn.functional.scaled_dot_product_attention(q, k, v, is_causal=True)
            ms_f = time_ms(f)
            y = f()
            ms_b = time_ms(lambda: torch.autograd.grad(y, (q, k, v), dO, retain_graph=True))
        out.append(dict(kind="library", backend=name, fwd_ms=ms_f, fwd_tflops=fl / ms_f / 1e9, bwd_ms=ms_b,
                        bwd_tflops=2.5 * fl / ms_b / 1e9))
    except Exception as ex:
        out.append(dict(kind="library", backend=name, error=repr(ex)[:300]))
out_dir = os.environ.get("DIAG_OUT") or os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "diag_out")
os.makedirs(out_dir, exist_ok=True)
with open(os.path.join(out_dir, "attn_bench.json"), "w") as fh:
    json.dump(out, fh, indent=1)
for r in out:
    print(json.dumps(r))
