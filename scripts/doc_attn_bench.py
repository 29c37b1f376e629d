"""Document-masked attention at the headline shape (B2 H32 S4096 hd128, plus a GQA row at KVH8): the masked kernels
(``seg`` table) against the unmasked causal kernels in the same process, timed alternately, for several packings of
the rows; "useful" TFLOP/s counts only the sum(L_i (L_i + 1) / 2) visible query-key pairs.  Also: numerics against
the fp32 oracle at a small shape, and torch FlexAttention with a document block mask as the library bar.
Writes $DIAG_OUT/doc_attn_bench.json (default diag_out/ in the repository root).
usage: python scripts/doc_attn_bench.py"""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from fms_fsdp_b200 import ops
from fms_fsdp_b200.ops import cuda_kernels as CK
from fms_fsdp_b200.ops import torch_kernels as TK

dev = "cuda"
out = []
SEP = 1


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                           capture_output=True, text=True, timeout=60)
        return r.stdout.strip()
    except Exception as ex:
        return f"nvidia-smi unavailable: {ex!r}"


def time_pair(fa, fb, iters=20, warm=5):
    """median ms of cold launches of fa and of fb, alternating the two"""
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    for _ in range(warm):
        fa(); fb()
    ts = ([], [])
    for _ in range(iters):
        for k, f in enumerate((fa, fb)):
            flush.zero_()                       # > L2: every timed launch starts cold
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); f(); e1.record(); torch.cuda.synchronize()
            ts[k].append(e0.elapsed_time(e1))
    med = []
    for t in ts:
        t.sort()
        med.append(dict(ms=t[len(t) // 2], p10=t[len(t) // 10], p90=t[(9 * len(t)) // 10]))
    return med


def rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).abs().max() / b.abs().max().clamp(min=1e-6)).item()


def layout_tokens(B, S, lens_per_row):
    tok = torch.full((B, S), 2, dtype=torch.long)
    for r, lens in enumerate(lens_per_row):
        p = 0
        for n in lens:
            p += n
            if p - 1 < S - 1:
                tok[r, p - 1] = SEP
    return tok.to(dev)


def doc_lengths(tok):
    lens = []
    for row in tok.tolist():
        n = 0
        for t in row:
            n += 1
            if t == SEP:
                lens.append(n); n = 0
        if n:
            lens.append(n)
    return lens


def random_mix(S, seed, mean=600):
    g = torch.Generator().manual_seed(seed)
    lens = []
    while sum(lens) < S:
        lens.append(int(torch.randint(16, 2 * mean - 16, (1,), generator=g)))
    return lens


print(gpu_info())
out.append(dict(kind="gpu", nvidia_smi=gpu_info()))
torch.manual_seed(0)

# numerics (small, multi-tile, GQA, boundaries on and off tile edges)
B, S, H, KVH, hd = 2, 512, 4, 2, 128
tok = layout_tokens(B, S, [[64, 64, 1, 200, 183], random_mix(S, 1, 120)])
seg = ops.document_segments(tok, SEP)
qkv_s = (torch.randn(B * S, (H + 2 * KVH) * hd, device=dev) * 0.8).bfloat16()
do_s = torch.randn(B * S, H * hd, device=dev).bfloat16()
o0, l0 = TK.attn_fwd(qkv_s.float(), B, S, H, KVH, hd, hd ** -0.5, seg=seg)
g0 = TK.attn_bwd(do_s.float(), qkv_s.float(), o0, l0, B, S, H, KVH, hd, hd ** -0.5, seg=seg)
o1, l1 = CK.attn_fwd(qkv_s, B, S, H, KVH, hd, hd ** -0.5, seg=seg)
g1 = CK.attn_bwd(do_s, qkv_s, o1, l1, B, S, H, KVH, hd, hd ** -0.5, seg=seg)
out.append(dict(kind="numerics", shape=[B, S, H, KVH, hd], o=rel(o1, o0), lse=rel(l1, l0), dqkv=rel(g1, g0)))

# timing at the headline shape
B, S, hd = 2, 4096, 128
layouts = {"one_doc": [[S]] * B}
for L in (2048, 1024, 512, 256):
    layouts[f"fixed_{L}"] = [[L] * (S // L)] * B
layouts["random_mean600"] = [random_mix(S, 10 + r) for r in range(B)]

for H, KVH in ((32, 32), (32, 8)):
    qkv = (torch.randn(B * S, (H + 2 * KVH) * hd, device=dev) * 0.8).bfloat16()
    do = torch.randn(B * S, H * hd, device=dev).bfloat16()
    sc = hd ** -0.5
    o_c, l_c = CK.attn_fwd(qkv, B, S, H, KVH, hd, sc)
    causal_pairs = B * S * (S + 1) / 2
    for name, lens in layouts.items():
        tok = layout_tokens(B, S, lens)
        seg = ops.document_segments(tok, SEP)
        pairs = sum(n * (n + 1) / 2 for n in doc_lengths(tok))
        fl = 4 * H * hd * pairs                              # QK^T and PV over the visible pairs
        o_m, l_m = CK.attn_fwd(qkv, B, S, H, KVH, hd, sc, seg=seg)
        f_m, f_c = time_pair(lambda: CK.attn_fwd(qkv, B, S, H, KVH, hd, sc, seg=seg),
                             lambda: CK.attn_fwd(qkv, B, S, H, KVH, hd, sc))
        b_m, b_c = time_pair(lambda: CK.attn_bwd(do, qkv, o_m, l_m, B, S, H, KVH, hd, sc, seg=seg),
                             lambda: CK.attn_bwd(do, qkv, o_c, l_c, B, S, H, KVH, hd, sc))
        out.append(dict(kind="doc", H=H, KVH=KVH, layout=name, n_docs=len(doc_lengths(tok)),
                        visible_pair_fraction=pairs / causal_pairs,
                        fwd_ms=f_m["ms"], fwd_causal_ms=f_c["ms"], fwd_ratio=f_m["ms"] / f_c["ms"],
                        fwd_spread_ms=[f_m["p10"], f_m["p90"], f_c["p10"], f_c["p90"]],
                        bwd_ms=b_m["ms"], bwd_causal_ms=b_c["ms"], bwd_ratio=b_m["ms"] / b_c["ms"],
                        bwd_spread_ms=[b_m["p10"], b_m["p90"], b_c["p10"], b_c["p90"]],
                        fwd_useful_tflops=fl / f_m["ms"] / 1e9, bwd_useful_tflops=2.5 * fl / b_m["ms"] / 1e9))
        print(json.dumps(out[-1]), flush=True)

# the library bar: FlexAttention with a document block mask (MHA headline shape, 512-token documents and random mix)
try:
    from torch.nn.attention.flex_attention import create_block_mask, flex_attention
    flex = torch.compile(flex_attention)
    H = KVH = 32
    qkv = (torch.randn(B * S, 3 * H * hd, device=dev) * 0.8).bfloat16()
    q, k, v = (t.reshape(B, S, H, hd).transpose(1, 2).contiguous().requires_grad_()
               for t in qkv.view(B * S, 3, H * hd).unbind(1))
    dO = torch.randn(B, H, S, hd, device=dev).bfloat16()
    for name in ("fixed_512", "random_mean600"):
        tok = layout_tokens(B, S, layouts[name])
        seg0 = ops.document_segments(tok, SEP)[0].view(B, S).long()

        def doc_causal(b, h, qi, ki):
            return (ki <= qi) & (ki >= seg0[b, qi])
        bm = create_block_mask(doc_causal, B, None, S, S, device=dev)
        f = lambda: flex(q, k, v, block_mask=bm)
        y = f()
        fb, _ = time_pair(f, f)
        bb, _ = time_pair(lambda: torch.autograd.grad(y, (q, k, v), dO, retain_graph=True),
                          lambda: None)
        pairs = sum(n * (n + 1) / 2 for n in doc_lengths(tok))
        fl = 4 * H * hd * pairs
        out.append(dict(kind="library", backend="flex_attention", layout=name, fwd_ms=fb["ms"],
                        fwd_useful_tflops=fl / fb["ms"] / 1e9, bwd_ms=bb["ms"], bwd_useful_tflops=2.5 * fl / bb["ms"] / 1e9))
except Exception as ex:
    out.append(dict(kind="library", backend="flex_attention", error=repr(ex)[:300]))

out_dir = os.environ.get("DIAG_OUT") or os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "diag_out")
os.makedirs(out_dir, exist_ok=True)
with open(os.path.join(out_dir, "doc_attn_bench.json"), "w") as fh:
    json.dump(out, fh, indent=1)
for r in out:
    print(json.dumps(r))
