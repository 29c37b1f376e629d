"""Gradient accumulation on the H100: the accumulate mode of the reduce-scatter kernels (through local pointer tables, as
in test_gpu_collectives_1gpu.py) and the engine at ``grad_accum_steps = 2`` on the fused sm_90a kernels."""
import os
import tempfile

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def C():
    from fms_fsdp_b200.ops import cuda_kernels as CK
    assert CK._C.__file__.endswith("_C.so")
    return CK._C


def table(tensors):
    return torch.tensor([t.data_ptr() for t in tensors], dtype=torch.int64, device=DEV)


@pytest.mark.parametrize("W", [2, 3, 4, 8])
@pytest.mark.parametrize("bf16", [True, False])
def test_reduce_scatter_accumulates(C, W, bf16):
    """Two 'micro-steps': the first overwrites, the second adds; sumsq is that of the accumulated result.  The output is
    a view into a larger buffer whose guard elements on both sides must stay untouched (W = 3 runs the dynamic kernel)."""
    torch.manual_seed(20 + W)
    n = 8 * 1024 * 3
    guard = 64
    dt = torch.bfloat16 if bf16 else torch.float32
    steps = [[(torch.randn(W * n, device=DEV) * 0.1).to(dt) for _ in range(W)] for _ in range(2)]
    for r in (0, W - 1):
        buf = torch.full((n + 2 * guard,), 7.0, device=DEV)
        out = buf[guard:guard + n]
        out.fill_(float("nan"))                                   # micro-step 1 must not read the old contents
        ss = torch.full((), 7.0, device=DEV)
        C.reduce_scatter(table(steps[0]), out, r * n, W, r, bf16, 1.0 / W, None)
        C.reduce_scatter(table(steps[1]), out, r * n, W, r, bf16, 1.0 / W, ss, accumulate=True)
        assert torch.all(buf[:guard] == 7.0) and torch.all(buf[guard + n:] == 7.0)
        ref = sum(f[r * n:(r + 1) * n].float() for s in steps for f in s) / W
        assert (out - ref).abs().max().item() < 1e-5 * max(1.0, ref.abs().max().item())
        assert abs(ss.item() - 7.0 - out.pow(2).sum().item()) < 1e-3 * out.pow(2).sum().item()
        before = out.clone()
        C.reduce_scatter(table(steps[1]), out, r * n, W, r, bf16, 1.0 / W, None, accumulate=True)
        step2 = sum(f[r * n:(r + 1) * n].float() for f in steps[1]) / W
        assert (out - before - step2).abs().max().item() < 1e-5 * max(1.0, ref.abs().max().item())
        assert torch.all(buf[:guard] == 7.0) and torch.all(buf[guard + n:] == 7.0)


def test_push_epilogue_slot_sum_accumulates_over_micro_steps(C):
    """wgrad push epilogue -> owner's slot sum, twice: the second slot sum with accumulate=True equals the sum of both
    micro-steps' reduce-scatters."""
    Nw, Kd, T, W = 1024, 512, 256, 4
    off = 64 * 3
    total = (off + Nw * Kd + W * 64 - 1) // (W * 64) * (W * 64)
    n = total // W
    staging = [torch.zeros(W * n, dtype=torch.bfloat16, device=DEV) for _ in range(W)]
    tab = table(staging)
    torch.manual_seed(31)
    ref = torch.zeros(total, device=DEV)
    outs = [torch.zeros(n, device=DEV) for _ in range(W)]
    ss = torch.zeros((), device=DEV)
    for micro in range(2):
        for r in range(W):
            dy = (torch.randn(T, Nw, device=DEV) * 0.1).bfloat16()
            x = (torch.randn(T, Kd, device=DEV) * 0.1).bfloat16()
            C.set_gemm_push(tab, n, off, r, True, W)
            C.gemm_push(dy, x)
            ref[off:off + Nw * Kd] += (dy.float().t() @ x.float()).bfloat16().float().reshape(-1)
        torch.cuda.synchronize()
        for o in range(W):
            slots = torch.tensor([staging[o].data_ptr() + s * n * 2 for s in range(W)], dtype=torch.int64, device=DEV)
            C.reduce_scatter(slots, outs[o], 0, W, 0, True, 1.0, ss if micro == 1 else None, accumulate=micro == 1)
    torch.cuda.synchronize()
    for o in range(W):
        r_ = ref[o * n:(o + 1) * n]
        assert (outs[o] - r_).abs().max().item() <= 2e-2 * r_.abs().max().clamp(min=1e-6).item(), o
    tot = sum(o_.pow(2).sum().item() for o_ in outs)
    assert abs(ss.item() - tot) <= 1e-3 * tot


def _tiny_llama(nlayers=3):
    from fms_fsdp_b200.models.llama import LLaMA, LLaMAConfig
    cfg = LLaMAConfig(src_vocab_size=2048, emb_dim=512, nheads=4, kvheads=2, nlayers=nlayers, multiple_of=256,
                      max_expected_seq_len=256)
    with torch.device("meta"):
        return LLaMA(cfg)


def _tiny_mamba():
    from fms_fsdp_b200.models.mamba import MambaConfig, MambaLMHeadModel
    from fms_fsdp_b200.utils.config_utils import get_model_config
    with torch.device("meta"):
        return MambaLMHeadModel(MambaConfig(**get_model_config("mamba_tiny")))


def _train(kind, path, k, batch, steps=4, autograd=False):
    """Losses (mean over the k micro-batches) and grad norms.  Step s draws k*batch sequences and splits them into k
    micro-batches, so k = 2 at b and k = 1 at 2b see the same sequences.  ``autograd``: micro-steps as
    ``loss = engine(x, labels); loss.backward()`` instead of ``forward_backward``."""
    from fms_fsdp_b200.ops import set_kernel_path
    from fms_fsdp_b200.parallel import ShardedAdamW, ShardedModel
    from fms_fsdp_b200.policies import bfSixteen
    set_kernel_path(path)
    torch.manual_seed(0); torch.cuda.manual_seed(0)
    m = _tiny_llama() if kind == "llama" else _tiny_mamba()
    V = 2048 if kind == "llama" else 512
    eng = ShardedModel(m, mixed_precision=bfSixteen, device=torch.device("cuda", 0), grad_accum_steps=k)
    if kind == "llama":
        m.rot_emb.compute_freqs_cis(torch.device("cuda", 0), 256)
    opt = ShardedAdamW(eng, lr=1e-3)
    out = []
    for st in range(steps):
        xs = torch.randint(0, V, (batch * k, 256), generator=torch.Generator().manual_seed(3 + st)).cuda()
        ls = []
        for x in xs.split(batch):
            if autograd:
                l = eng(x, x)
                l.backward()
                ls.append(l.detach())
            else:
                ls.append(eng.forward_backward(x, x))
        g = eng.clip_grad_norm_(1.0)
        opt.step()
        out.append((sum(l.item() for l in ls) / k, g.item()))
    return out


@pytest.mark.parametrize("kind", ["llama", "mamba"])
def test_engine_accumulation_fused_matches_aten_path(kind):
    from fms_fsdp_b200.ops import cuda_kernels as CK
    from fms_fsdp_b200.ops import set_kernel_path

    def touched(before):
        return {name for name, c in CK.FALLBACKS.items() if c != before.get(name, 0)}
    try:
        f0 = dict(CK.FALLBACKS)
        n0 = CK.launch_count()
        fused = _train(kind, "fused", 2, 2)
        assert CK.launch_count() - n0 > 100
        k2_fallbacks = touched(f0)
        f1 = dict(CK.FALLBACKS)
        fused_k1 = _train(kind, "fused", 1, 2)
        # accumulation adds no ATen fallback: none at all for Llama, none beyond the k = 1 run's for the Mamba hybrid
        assert k2_fallbacks <= touched(f1) and (kind != "llama" or not k2_fallbacks), k2_fallbacks
        aten = _train(kind, "torch", 2, 2)
    finally:
        set_kernel_path("auto")
    for (lf, gf), (la, ga) in zip(fused, aten):
        assert abs(lf - la) < 3e-2 * abs(la) and abs(gf - ga) < 6e-2 * abs(ga)
    assert fused[-1][0] < fused[0][0] and fused_k1[-1][0] < fused_k1[0][0]


def test_engine_k2_at_b_matches_k1_at_2b():
    from fms_fsdp_b200.ops import cuda_kernels as CK
    from fms_fsdp_b200.ops import set_kernel_path
    try:
        f0 = CK.fallback_count()
        acc = _train("llama", "fused", 2, 1)
        big = _train("llama", "fused", 1, 2)
        assert CK.fallback_count() == f0
    finally:
        set_kernel_path("auto")
    for (la, ga), (lb, gb) in zip(acc, big):
        assert abs(la - lb) < 2e-2 * abs(lb) and abs(ga - gb) < 5e-2 * abs(gb)


def test_fused_loss_autograd_form_accumulates_like_forward_backward():
    """One GPU (unsharded): micro-step 2 of ``engine(x, labels).backward()`` computes the head's dW as an ordinary
    gradient that is added to the fp32 buffer; the step equals the ``forward_backward`` form within bf16 rounding."""
    from fms_fsdp_b200.ops import cuda_kernels as CK
    from fms_fsdp_b200.ops import set_kernel_path
    try:
        f0 = CK.fallback_count()
        a = _train("llama", "fused", 2, 2, autograd=True)
        b = _train("llama", "fused", 2, 2)
        assert CK.fallback_count() == f0
    finally:
        set_kernel_path("auto")
    for (la, ga), (lb, gb) in zip(a, b):
        assert abs(la - lb) < 1e-2 * abs(lb) and abs(ga - gb) < 2e-2 * abs(gb)


def _two_gpu_worker(rank, port, impl, outdir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE="2",
                      LOCAL_RANK=str(rank), LOCAL_WORLD_SIZE="2")
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=2, device_id=torch.device("cuda", rank))
    try:
        from fms_fsdp_b200.parallel import ShardedAdamW, ShardedModel
        from fms_fsdp_b200.policies import bfSixteen
        torch.manual_seed(0)
        m = _tiny_llama()
        dev = torch.device("cuda", rank)
        eng = ShardedModel(m, sharding_strategy="fsdp", mixed_precision=bfSixteen, device=dev, collective_impl=impl,
                           grad_accum_steps=2)
        m.rot_emb.compute_freqs_cis(dev, 256)
        opt = ShardedAdamW(eng, lr=1e-3)
        out = []
        for st in range(3):
            xs = torch.randint(0, 2048, (4, 256), generator=torch.Generator().manual_seed(10 * st + rank)).to(dev)
            ls = [eng.forward_backward(x, x) for x in xs.split(2)]
            g = eng.clip_grad_norm_(1.0)
            opt.step()
            out.append((sum(l.item() for l in ls) / 2, g.item()))
        if rank == 0:
            torch.save(dict(out=out, push=eng._push_rs, coll=eng.coll.name), os.path.join(outdir, f"{impl}.pt"))
        torch.cuda.synchronize()
    finally:
        dist.barrier()
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs with peer access")
def test_two_gpu_fsdp_push_path_accumulates_like_nccl():
    from conftest import free_port
    outdir = tempfile.mkdtemp()
    for impl in ("fused", "torch"):
        mp.spawn(_two_gpu_worker, args=(free_port(), impl, outdir), nprocs=2, join=True)
    f = torch.load(os.path.join(outdir, "fused.pt"), weights_only=False)
    t = torch.load(os.path.join(outdir, "torch.pt"), weights_only=False)
    assert f["coll"] == "fused" and f["push"] and t["coll"] == "torch"
    for (lf, gf), (lt, gt) in zip(f["out"], t["out"]):
        assert abs(lf - lt) < 2e-2 * abs(lt) and abs(gf - gt) < 2e-2 * gt
