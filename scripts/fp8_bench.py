"""Opt-in fp8 forward path: e4m3 wgmma GEMM and the row-wise quantisation kernel at the Llama2-7B
forward shapes, against the bf16 GEMM of the same shape.  Writes gpurun_out/fp8_bench.json."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from fms_fsdp_b200.ops import cuda_kernels as CK
dev = "cuda"
def time_ms(fn, iters=20, warm=5):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    for _ in range(warm): fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize(); ts.append(e0.elapsed_time(e1))
    ts.sort(); return ts[len(ts) // 2]
out = []
torch.manual_seed(0)
for (M, N, K) in [(8192, 12288, 4096), (8192, 22016, 4096), (8192, 4096, 11008)]:
    x = (torch.randn(M, K, device=dev) * 0.5).bfloat16(); w = (torch.randn(N, K, device=dev) * 0.03).bfloat16()
    xq, sx = CK.quant_rowwise_e4m3(x); wq, sw = CK.quant_rowwise_e4m3(w)
    y = CK.gemm_fp8(xq, wq, sx, sw); ref = CK.gemm(x, w, "nt")
    err = ((y.float() - ref.float()).abs().max() / ref.float().abs().max()).item()
    fl = 2.0 * M * N * K
    t8 = time_ms(lambda: CK.gemm_fp8(xq, wq, sx, sw)); t16 = time_ms(lambda: CK.gemm(x, w, "nt"))
    tq = time_ms(lambda: CK.quant_rowwise_e4m3(x)); tw = time_ms(lambda: CK.quant_rowwise_e4m3(w))
    out.append(dict(M=M, N=N, K=K, fp8_ms=t8, fp8_tflops=fl / t8 / 1e9, bf16_ms=t16, bf16_tflops=fl / t16 / 1e9,
                    quant_x_ms=tq, quant_w_ms=tw, rel_err_vs_bf16=err))
    print(json.dumps(out[-1]), flush=True)
os.makedirs("gpurun_out", exist_ok=True)
json.dump(out, open("gpurun_out/fp8_bench.json", "w"), indent=1)
