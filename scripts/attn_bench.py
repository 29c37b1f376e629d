"""Attention kernels, causal, hd 128: the pipelined kernels (what the model runs) against the library (cuDNN / flash
SDPA through torch), forward and backward, in alternated rounds; plus numerics vs the fp32 oracle at a small shape.
Shapes: the Llama2-1.4B headline block (B2 H16 KVH4 S4096), B2 H32 S4096, and both with 512-token documents.  Prints
the card, its power limit and the SM clock from the same run.

    python scripts/attn_bench.py [--rounds 5] [--dump DIR]

--dump DIR writes o / lse / dqkv of the headline and H32 shapes for fixed seeds (DIR/<shape>.pt), so two builds can be
compared bitwise.  Writes $DIAG_OUT/attn_bench.json (default diag_out/ in the repository root)."""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from fms_fsdp_b200 import ops
from fms_fsdp_b200.ops import cuda_kernels as CK
from fms_fsdp_b200.ops import torch_kernels as TK

dev = "cuda"
out = []


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except Exception as ex:  # noqa: BLE001
        r = repr(ex)[:200]
    return dict(kind="card", query=q, value=r, torch_name=torch.cuda.get_device_name(0))


def time_ms(fn, iters=10, warm=3):
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


def doc_seg(B, S, L):
    tok = torch.zeros(B, S, dtype=torch.long, device=dev)
    tok[:, L - 1::L] = 1
    return ops.document_segments(tok, 1)


def visible_pairs(B, S, seg):
    if seg is None:
        return B * S * (S + 1) / 2
    return float((torch.arange(S, device=dev).view(1, S) - seg[0].view(B, S) + 1).sum())   # keys seg0[q] .. q


p = argparse.ArgumentParser()
p.add_argument("--rounds", type=int, default=5)
p.add_argument("--dump", default="")
a = p.parse_args()
C = CK._C
out.append(card())

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

SHAPES = [("h16_kvh4", 16, 4, None), ("h32", 32, 32, None), ("h16_kvh4_doc512", 16, 4, 512), ("h32_doc512", 32, 32, 512)]
B, S, hd = 2, 4096, 128
sc = hd ** -0.5
from torch.nn.attention import SDPBackend, sdpa_kernel  # noqa: E402

for name, H, KVH, L in SHAPES:
    g = torch.Generator(device=dev).manual_seed(1234)
    qkv = (torch.randn(B * S, (H + 2 * KVH) * hd, device=dev, generator=g) * 0.8).bfloat16()
    do = torch.randn(B * S, H * hd, device=dev, generator=g).bfloat16()
    seg = doc_seg(B, S, L) if L else None
    pairs = visible_pairs(B, S, seg)
    fl = 4 * H * pairs * hd                 # useful forward FLOPs: 2 GEMMs over the visible pairs
    o, l = C.attn_fwd(qkv, B, S, H, KVH, hd, sc, seg)
    dq = C.attn_bwd(do, qkv, o, l, B, S, H, KVH, hd, sc, None, seg)
    if a.dump and L is None:
        os.makedirs(a.dump, exist_ok=True)
        torch.save(dict(o=o.cpu(), lse=l.cpu(), dqkv=dq.cpu()), os.path.join(a.dump, f"{name}.pt"))
    arms = {
        "pipelined": (lambda: C.attn_fwd(qkv, B, S, H, KVH, hd, sc, seg),
                      lambda: C.attn_bwd(do, qkv, o, l, B, S, H, KVH, hd, sc, None, seg)),
    }
    if L is None:                           # the library bar (causal only)
        q = qkv[:, :H * hd].reshape(B, S, H, hd).transpose(1, 2).contiguous().requires_grad_()
        k = qkv[:, H * hd:(H + KVH) * hd].reshape(B, S, KVH, hd).transpose(1, 2)
        v = qkv[:, (H + KVH) * hd:].reshape(B, S, KVH, hd).transpose(1, 2)
        if KVH != H:                        # expand the kv heads: cuDNN SDPA takes equal head counts
            k, v = (t.repeat_interleave(H // KVH, dim=1) for t in (k, v))
        k, v = (t.contiguous().requires_grad_() for t in (k, v))
        dO = do.view(B, S, H, hd).transpose(1, 2).contiguous()
        f = lambda: torch.nn.functional.scaled_dot_product_attention(q, k, v, is_causal=True)  # noqa: E731
        try:
            with sdpa_kernel([SDPBackend.CUDNN_ATTENTION]):
                y = f()
                torch.autograd.grad(y, (q, k, v), dO, retain_graph=True)

            def lib_fwd():
                with sdpa_kernel([SDPBackend.CUDNN_ATTENTION]):
                    f()

            def lib_bwd():
                torch.autograd.grad(y, (q, k, v), dO, retain_graph=True)
            arms["cudnn"] = (lib_fwd, lib_bwd)
        except Exception as ex:  # noqa: BLE001
            out.append(dict(kind="library", shape=name, error=repr(ex)[:300]))
    ts = {k: ([], []) for k in arms}
    for _ in range(a.rounds):               # alternated: every arm once per round
        for arm, (ff, fb) in list(arms.items()):
            try:
                ts[arm][0].append(time_ms(ff))
                ts[arm][1].append(time_ms(fb))
            except Exception as ex:  # noqa: BLE001  (the library arm only; our kernels raise through _C.check)
                if arm != "cudnn":
                    raise
                out.append(dict(kind="library", shape=name, error=repr(ex)[:300]))
                del arms[arm], ts[arm]
    for arm, (tf, tb) in ts.items():
        out.append(dict(kind="time", shape=name, arm=arm, fwd_ms=statistics.median(tf), fwd_min=min(tf), fwd_max=max(tf),
                        bwd_ms=statistics.median(tb), bwd_min=min(tb), bwd_max=max(tb),
                        fwd_tflops=fl / statistics.median(tf) / 1e9, bwd_tflops=2.5 * fl / statistics.median(tb) / 1e9))
    del arms
    torch.cuda.empty_cache()

out.append(card())
out_dir = os.environ.get("DIAG_OUT") or os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "diag_out")
os.makedirs(out_dir, exist_ok=True)
with open(os.path.join(out_dir, "attn_bench.json"), "w") as fh:
    json.dump(out, fh, indent=1)
for r in out:
    print(json.dumps(r))
