"""The multi-GPU kernels on ONE GPU: every collective kernel of ``csrc/comm.cu`` and the two fused GEMM paths
(all-gather inside the GEMM, wgrad push -> slot sum) take a *table of pointers*, so W "ranks" can be W local buffers.
That checks all the index math, the flag protocols and the numerics against fp32 torch sums on the 1-GPU test box;
NVLink itself only changes where the addresses point (``scripts/gpu_multi_check.py`` covers that on 2/4/8 GPUs).
"""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def C():
    from fms_fsdp_b200.ops import cuda_kernels as CK
    assert CK._C.__file__.endswith("_C.so")
    return CK._C


def table(tensors):
    return torch.tensor([t.data_ptr() for t in tensors], dtype=torch.int64, device=DEV)


def tile_rel(a, b, tile=256):
    """max over 256x256 tiles of (max |a-b| in the tile) / (max |b| in the tile): a wrong low-magnitude tile fails."""
    a, b = a.float(), b.float()
    M, N = b.shape
    worst = 0.0
    for i in range(0, M, tile):
        d = (a[i:i + tile] - b[i:i + tile]).abs()
        r = b[i:i + tile].abs()
        for j in range(0, N, tile):
            worst = max(worst, (d[:, j:j + tile].max() / r[:, j:j + tile].max().clamp(min=1e-6)).item())
    return worst


@pytest.mark.parametrize("W", [2, 3, 4, 8])
@pytest.mark.parametrize("bf16", [True, False])
def test_reduce_scatter_kernel_vs_fp32_sum(C, W, bf16):
    torch.manual_seed(W)
    n = 8 * 1024 * 3            # shard elements
    dt = torch.bfloat16 if bf16 else torch.float32
    fulls = [(torch.randn(W * n, device=DEV) * 0.1).to(dt) for _ in range(W)]
    tab = table(fulls)
    for r in range(W):
        out = torch.zeros(n, device=DEV)
        ss = torch.zeros((), device=DEV)
        C.reduce_scatter(tab, out, r * n, W, r, bf16, 1.0 / W, ss)
        ref = sum(f[r * n:(r + 1) * n].float() for f in fulls) / W
        assert (out - ref).abs().max().item() < 1e-5 * max(1.0, ref.abs().max().item())
        assert abs(ss.item() - ref.pow(2).sum().item()) < 1e-3 * ref.pow(2).sum().item()


@pytest.mark.parametrize("W", [2, 3, 8])
@pytest.mark.parametrize("bf16", [True, False])
def test_two_phase_allreduce_kernels(C, W, bf16):
    """HSDP replica / DDP all-reduce: reduce_slice_inplace for every 'rank', then the slice all-gather."""
    torch.manual_seed(10 + W)
    vec = 8 if bf16 else 4
    n = W * vec * 1000
    dt = torch.bfloat16 if bf16 else torch.float32
    bufs = [(torch.randn(n, device=DEV) * 0.1).to(dt) for _ in range(W)]
    ref = sum(b.float() for b in bufs) * 0.5
    tab = table(bufs)
    anchor = torch.zeros(1, device=DEV)
    for r in range(W):
        C.allreduce_inplace(tab, n, W, r, bf16, 0.5, None, anchor)
    ns = n // W
    es = 2 if bf16 else 4
    for r in range(W):
        slice_tab = torch.tensor([b.data_ptr() + i * ns * es for i, b in enumerate(bufs)], dtype=torch.int64, device=DEV)
        C.p2p_allgather(slice_tab, bufs[r], ns * es, W, r)
    tol = 1e-2 if bf16 else 1e-5
    for r in range(W):
        assert (bufs[r].float() - ref).abs().max().item() < tol * ref.abs().max().item()
    assert all(torch.equal(bufs[0], b) for b in bufs[1:])       # every rank ends with identical bits


@pytest.mark.parametrize("W", [2, 4, 8])
def test_allgather_and_gather_range(C, W):
    torch.manual_seed(3)
    n = 4096 * 5
    shards = [torch.randn(n, device=DEV).bfloat16() for _ in range(W)]
    ref = torch.cat(shards)
    tab = table(shards)
    for r in range(W):
        full = torch.zeros(W * n, dtype=torch.bfloat16, device=DEV)
        C.p2p_allgather(tab, full, n * 2, W, r)
        assert torch.equal(full, ref)
    full = torch.zeros(W * n, dtype=torch.bfloat16, device=DEV)
    lo, hi = 4096 * 2, n * 2 + 1024               # byte range crossing a shard boundary
    C.p2p_gather_range(tab, full, n * 2, lo, hi)
    assert torch.equal(full[lo // 2:hi // 2], ref[lo // 2:hi // 2]) and full[:lo // 2].abs().sum() == 0


def test_signal_post_wait_and_scalar_allreduce(C):
    """Flag rounds with 2 emulated ranks on 2 streams (the kernels must be co-resident, as on 2 GPUs)."""
    W = 2
    pads = [torch.zeros(32 * 16, dtype=torch.int32, device=DEV) for _ in range(W)]
    ptab = table(pads)
    anchor = torch.zeros(1, device=DEV)
    streams = [torch.cuda.Stream() for _ in range(W)]
    torch.cuda.synchronize()
    # one-sided: both post epoch 5 on channel 3, then both wait
    for r in range(W):
        C.signal_barrier(ptab, W, r, 5, anchor, 32 * 3, 1)
    for r in range(W):
        C.signal_barrier(ptab, W, r, 5, anchor, 32 * 3, 2)
    torch.cuda.synchronize()
    assert all(int(p[32 * 3 + r]) == 5 for p in pads for r in range(W))
    assert int(pads[0][:32 * 3].abs().sum()) == 0              # other channels untouched
    # full barrier, concurrently on two streams
    for r in range(W):
        with torch.cuda.stream(streams[r]):
            C.signal_barrier(ptab, W, r, 1, anchor, 0, 0)
    torch.cuda.synchronize()
    # scalar all-reduce: rank r contributes r + 1.5 (and a second value), three rounds
    bufs = [torch.zeros(1024, dtype=torch.int32, device=DEV) for _ in range(W)]
    btab = table(bufs)
    for epoch in range(1, 4):
        vals = [torch.tensor([r + 1.5 * epoch, 10.0 * r], device=DEV) for r in range(W)]
        for r in range(W):
            with torch.cuda.stream(streams[r]):
                C.scalar_allreduce(btab, W, r, epoch, vals[r])
        torch.cuda.synchronize()
        for r in range(W):
            assert vals[r].tolist() == [sum(q + 1.5 * epoch for q in range(W)), 10.0 * sum(range(W))]


@pytest.mark.parametrize("W", [2, 8])
@pytest.mark.parametrize("dependent", [True, False])
def test_ag_gemm_gathers_from_pointer_table(C, W, dependent):
    """All-gather fused into the GEMM: the comm warps pull W 'peer' shards into the gathered buffer; in
    dependent mode the GEMM's own B operand is that buffer, consumed tile by tile behind the ready flags."""
    from fms_fsdp_b200.ops import cuda_kernels as CK
    torch.manual_seed(5)
    N, Kd, M = 1536, 1024, 1024
    total = N * Kd + 65536
    total = total // (W * 64) * (W * 64)
    n = total // W
    shards = [(torch.randn(n, device=DEV) * 0.05).bfloat16() for _ in range(W)]
    ref_full = torch.cat(shards)
    x = torch.randn(M, Kd, device=DEV).bfloat16()
    yref = x.float() @ ref_full[:N * Kd].view(N, Kd).float().t()
    for r in (0, W - 1):
        full = torch.zeros(total, dtype=torch.bfloat16, device=DEV)
        flags = torch.zeros((total * 2 + 65535) // 65536, dtype=torch.int32, device=DEV)
        Wm = (full if dependent else ref_full)[:N * Kd].view(N, Kd)
        y = torch.empty(M, N, dtype=torch.bfloat16, device=DEV)
        C.gemm_ag(x, Wm, y, 0, 0, None, table(shards), full, n * 2, 0, total * 2, W, r, flags, 1, dependent)
        torch.cuda.synchronize()
        assert torch.equal(full, ref_full)
        assert tile_rel(y, yref) < 1e-2


@pytest.mark.parametrize("bulk", [True, False])
@pytest.mark.parametrize("shape", [(2048, 1024, 512, 8), (1000, 520, 256, 4), (512, 4096, 512, 2), (768, 768, 256, 3)])
def test_wgrad_push_epilogue_then_slot_sum_is_reduce_scatter(C, shape, bulk):
    """P_EPI_PUSH: every 'rank' pushes its wgrad tiles into the owners' staging slots [src rank][shard]; the owner's
    local slot sum must equal the reduce-scatter of the per-rank wgrads (fp32 torch reference)."""
    from fms_fsdp_b200.ops import cuda_kernels as CK
    Nw, Kd, T, W = shape                      # dW [Nw, Kd] = dy^T x ;  T tokens
    torch.manual_seed(7)
    off = 64 * 3                              # the weight does not start at the beginning of the flat unit
    total = (off + Nw * Kd + W * 64 - 1) // (W * 64) * (W * 64)
    n = total // W
    staging = [torch.zeros(W * n, dtype=torch.bfloat16, device=DEV) for _ in range(W)]   # one per owner
    tab = table(staging)
    ref = torch.zeros(total, device=DEV)
    for r in range(W):
        dy = (torch.randn(T, Nw, device=DEV) * 0.1).bfloat16()
        x = (torch.randn(T, Kd, device=DEV) * 0.1).bfloat16()
        C.gemm_push(dy, x, push_bases=tab, push_n=n, push_off=off, push_rank=r, push_bulk=bulk,
                    push_world=W if Nw != 512 else 1)   # rank-rotated tile raster (and one case without)
        ref[off:off + Nw * Kd] += (dy.float().t() @ x.float()).bfloat16().float().reshape(-1)
    torch.cuda.synchronize()
    for o in range(W):
        slots = torch.tensor([staging[o].data_ptr() + s * n * 2 for s in range(W)], dtype=torch.int64, device=DEV)
        out = torch.zeros(n, device=DEV)
        ss = torch.zeros((), device=DEV)
        C.reduce_scatter(slots, out, 0, W, 0, True, 1.0, ss)
        r_ = ref[o * n:(o + 1) * n]
        assert (out - r_).abs().max().item() <= 2e-2 * r_.abs().max().clamp(min=1e-6).item(), (o, shape, bulk)
        assert abs(ss.item() - out.pow(2).sum().item()) <= 1e-3 * max(1e-6, out.pow(2).sum().item())
    # nothing outside [off, off + Nw*Kd) was touched (gaps of the flat unit stay zero for the slot sum)
    flat = torch.stack([s.view(W, n) for s in staging])            # [owner][src][n]
    per_src = flat.permute(1, 0, 2).reshape(W, W * n)               # [src][flat element]
    assert per_src[:, :off].abs().sum() == 0 and per_src[:, off + Nw * Kd:].abs().sum() == 0


def test_push_range_vectors(C):
    W, n = 4, 64 * 10
    torch.manual_seed(9)
    staging = [torch.zeros(W * n, dtype=torch.bfloat16, device=DEV) for _ in range(W)]
    tab = table(staging)
    vecs = [torch.randn(n + 64 * 5, device=DEV).bfloat16() for _ in range(W)]      # spans the first two owners
    for r in range(W):
        C.push_range(vecs[r], tab, n, 0, r)
    torch.cuda.synchronize()
    for r in range(W):
        assert torch.equal(staging[0].view(W, n)[r], vecs[r][:n])
        assert torch.equal(staging[1].view(W, n)[r][:64 * 5], vecs[r][n:])


@pytest.mark.parametrize("layout", ["nt", "nn", "tn"])
def test_gemm_headline_shape_per_tile_error(layout):
    """The gate/up projection of Llama2-7B at the benchmark shape (8192 tokens): every 256x256 output tile within
    bf16 rounding of the fp32 reference."""
    from fms_fsdp_b200.ops import cuda_kernels as CK
    torch.manual_seed(11)
    M, N, Kd = 8192, 22016, 4096
    if layout == "tn":
        M, N, Kd = 22016, 4096, 8192
    a = (torch.randn((M, Kd) if layout != "tn" else (Kd, M), device=DEV) * 0.5).bfloat16()
    b = (torch.randn((N, Kd) if layout == "nt" else (Kd, N), device=DEV) * 0.5).bfloat16()
    out = CK.gemm(a, b, layout)
    af = a.float() if layout != "tn" else a.float().t()
    bf = b.float().t() if layout == "nt" else b.float()
    ref = af @ bf
    assert tile_rel(out, ref) < 1e-2


@pytest.mark.parametrize("H,KVH", [(8, 8), (8, 2)])
def test_attention_headline_seq_4096(H, KVH):
    """Causal attention at S = 4096 (32 k/v tiles per row block, causal tile skipping, GQA) vs the fp32 oracle."""
    from fms_fsdp_b200.ops import cuda_kernels as CK
    from fms_fsdp_b200.ops import torch_kernels as TK
    torch.manual_seed(13)
    B, S, hd = 1, 4096, 128
    qkv = (torch.randn(B * S, (H + 2 * KVH) * hd, device=DEV) * 0.7).bfloat16()
    do = torch.randn(B * S, H * hd, device=DEV).bfloat16()
    scale = hd ** -0.5
    o, lse = CK.attn_fwd(qkv, B, S, H, KVH, hd, scale)
    o_ref, lse_ref = TK.attn_fwd(qkv.float(), B, S, H, KVH, hd, scale)
    assert tile_rel(o, o_ref, tile=128) < 2e-2
    g = CK.attn_bwd(do, qkv, o, lse, B, S, H, KVH, hd, scale)
    g_ref = TK.attn_bwd(do.float(), qkv.float(), o_ref, lse_ref, B, S, H, KVH, hd, scale)
    # per 128-row block and per q / k / v section
    for name, lo, hi in (("dq", 0, H * hd), ("dk", H * hd, (H + KVH) * hd), ("dv", (H + KVH) * hd, (H + 2 * KVH) * hd)):
        assert tile_rel(g[:, lo:hi], g_ref[:, lo:hi], tile=128) < 4e-2, name
