"""z-losses on CPU: the ATen oracles of the output z-loss (fused linear + CE) and of the ST-MoE router z-loss against
float64 autograd of the textbook formulas, probes showing that plausible bugs miss by far more than the GPU tolerances,
the world-2 gloo engine with both losses against the single-process oracle, the entry points, and a short training
run in which the z-loss does what it is for."""
import os
import re
import subprocess
import sys
import tempfile

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

from conftest import free_port
from fms_fsdp_b200 import ops
from fms_fsdp_b200.models.llama import LLaMA
from fms_fsdp_b200.ops import torch_kernels as TK
from fms_fsdp_b200.utils.config_utils import get_model_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# Tolerances of tests/test_z_loss_gpu.py (relative errors against float64, about 3x the errors measured on an H100):
# the statistics, the head's dh / dW, the z part of the logit gradient (G(c) - G(0)) at c = 1e-2, and the router's.
GPU_TOL = dict(stat=3e-7, grad=1e-2, zpart=1.5e-2, router_zpart=5e-3)


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp(min=1e-300))


def _head_case(M, D, V, frac_ignored, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    h = torch.randn(M, D, generator=g, dtype=torch.float64) * scale
    w = torch.randn(V, D, generator=g, dtype=torch.float64) / D ** 0.5
    labels = torch.randint(0, V, (M,), generator=g)
    labels[torch.rand(M, generator=g) < frac_ignored] = -100
    return h, w, labels


def _autograd_ce_z(h, w, labels, c):
    """(ce, z, dh, dw) by float64 autograd of CE + c z, z = mean over non-ignored rows of logsumexp^2."""
    h, w = h.clone().requires_grad_(), w.clone().requires_grad_()
    logits = h @ w.t()
    ok = labels != -100
    n = ok.sum().clamp(min=1)
    ce = F.cross_entropy(logits, labels, ignore_index=-100, reduction="sum") / n
    z = (torch.logsumexp(logits, -1) ** 2 * ok).sum() / n
    (ce + c * z).backward()
    return ce.detach(), z.detach(), h.grad, w.grad


@pytest.mark.parametrize("chunk", [256, 3000, 4096])
@pytest.mark.parametrize("c", [1e-5, 1e-4, 1e-2])
def test_linear_ce_z_oracle_matches_fp64_autograd(chunk, c):
    h, w, labels = _head_case(5000, 16, 64, 0.2, scale=3.0)
    ce0, z0, dh0, dw0 = _autograd_ce_z(h, w, labels, c)
    dw = torch.empty_like(w)
    ce, z, dh = TK.linear_ce_z_fwd_bwd(h, w, labels, dw, c, chunk_rows=chunk)
    assert float(ce) == pytest.approx(float(ce0), rel=1e-12)
    assert float(z) == pytest.approx(float(z0), rel=1e-12)
    assert rel(dh, dh0) < 1e-12 and rel(dw, dw0) < 1e-12
    ce2, z2, dl = TK.cross_entropy_z_fwd_bwd(h @ w.t(), labels, c)
    assert float(ce2) == pytest.approx(float(ce0), rel=1e-12) and float(z2) == pytest.approx(float(z0), rel=1e-12)
    assert rel(dl @ w, dh0) < 1e-12


def test_wholly_ignored_batch_gives_zero_loss_and_gradient():
    h, w, labels = _head_case(64, 16, 64, 1.0)
    assert bool((labels == -100).all())
    dw = torch.full_like(w, 7.0)
    ce, z, dh = TK.linear_ce_z_fwd_bwd(h, w, labels, dw, 1e-2)
    assert float(ce) == 0 and float(z) == 0 and not dh.any() and not dw.any()


def test_ops_entries_fold_the_z_gradient_into_ce_and_keep_their_signatures():
    h, w, labels = _head_case(96, 16, 64, 0.25, scale=3.0)
    c = 1e-2
    ce0, z0, dh0, dw0 = _autograd_ce_z(h, w, labels, c)
    hl, wl = h.clone().requires_grad_(), w.clone().requires_grad_()
    ce, z = ops.linear_cross_entropy_z(hl, wl, labels, c)
    assert not z.requires_grad
    (2.0 * ce).backward()                                   # a scaled upstream gradient applies to the z part too
    ce = ce.detach()
    assert float(ce) == pytest.approx(float(ce0), rel=1e-12) and float(z) == pytest.approx(float(z0), rel=1e-12)
    assert rel(hl.grad, 2 * dh0) < 1e-12 and rel(wl.grad, 2 * dw0) < 1e-12
    lg = (h @ w.t()).requires_grad_()
    ce, z = ops.cross_entropy_z(lg, labels, c)
    ce.backward()
    assert rel(lg.grad @ w, dh0) < 1e-12 and float(z) == pytest.approx(float(z0), rel=1e-12)


# ------------------------------------------------------------------------------------------------ router
def _router_case(T, E, k, norm, seed=0):
    g = torch.Generator().manual_seed(seed + E + k)
    logits = torch.randn(T, E, generator=g, dtype=torch.float64) * 2
    G = torch.randn(T, k, generator=g, dtype=torch.float64)
    return logits, G


def _autograd_router(logits, G, k, norm, aux_coef, cz):
    """float64 autograd of sum_ts G_ts w_ts + aux_coef E / T^2 sum_e count_e sum_t p_te + cz mean_t lse_t^2 (ST-MoE)."""
    T, E = logits.shape
    ids = TK.moe_route(logits, k, norm)[0].long()
    count = torch.bincount(ids.reshape(-1), minlength=E).double()
    l = logits.clone().requires_grad_()
    p = torch.softmax(l, -1)
    wts = p.gather(1, ids)
    if norm:
        wts = wts / wts.sum(1, keepdim=True)
    obj = (G * wts).sum() + aux_coef * E / T ** 2 * (count * p.sum(0)).sum() \
        + cz * (torch.logsumexp(l, -1) ** 2).mean()
    obj.backward()
    return l.grad


def _oracle_router(logits, G, k, norm, aux_coef, cz, topk_bug=False):
    T, E = logits.shape
    ids, wts, probs = TK.moe_route(logits, k, norm)
    plan, _ = TK.moe_plan(ids, probs)
    dl = TK.moe_route_bwd(probs, ids, wts, G, plan, norm, aux_coef * E / (T * T))
    lse, z = TK.router_z_fwd(logits)
    if topk_bug:     # the z term on the top-k probabilities only
        probs = torch.zeros_like(probs).scatter_(1, ids.long(), probs.gather(1, ids.long()))
    return TK.router_z_bwd(dl, probs, lse, 2 * cz / T), z


@pytest.mark.parametrize("E,k", [(8, 2), (128, 8), (8, 8), (128, 2)])
@pytest.mark.parametrize("norm", [False, True])
def test_router_z_oracle_matches_fp64_autograd_with_the_aux_loss(E, k, norm):
    T = 64
    logits, G = _router_case(T, E, k, norm)
    ref = _autograd_router(logits, G, k, norm, 0.01, 1e-3)
    dl, z = _oracle_router(logits, G, k, norm, 0.01, 1e-3)
    assert rel(dl, ref) < 1e-6                        # the routing oracle computes in fp32
    # the z part alone stays in float64
    l = logits.clone().requires_grad_()
    (1e-3 * (torch.logsumexp(l, -1) ** 2).mean()).backward()
    lse, z = TK.router_z_fwd(logits)
    dz = TK.router_z_bwd(torch.zeros_like(logits), torch.softmax(logits, -1), lse, 2 * 1e-3 / T)
    assert rel(dz, l.grad) < 1e-12
    assert float(z) == pytest.approx(float((torch.logsumexp(logits, -1) ** 2).mean()), rel=1e-14)


# ------------------------------------------------------------------------------------------------ probes
def _zpart_error(h, w, labels, c, grad_of):
    """Relative error of the z part of the logit gradient, G(c) - G(0), that ``grad_of`` implies."""
    G0 = TK.cross_entropy_z_fwd_bwd(h @ w.t(), labels, 0.0)[2]
    Gc = TK.cross_entropy_z_fwd_bwd(h @ w.t(), labels, c)[2]
    return rel(grad_of() - G0, Gc - G0)


def test_probes_plausible_head_bugs_miss_by_ten_times_the_gpu_tolerance():
    h, w, labels = _head_case(512, 16, 64, 0.5, scale=3.0)
    c = 1e-2
    logits = h @ w.t()
    ok = labels != -100
    n, M = int(ok.sum()), labels.numel()
    lse = torch.logsumexp(logits, -1)
    z_ref = (lse ** 2 * ok).sum() / n
    assert abs(float((lse ** 2 * ok).sum() / M / z_ref) - 1) > 10 * GPU_TOL["stat"]      # divided by M, not n
    assert abs(float((lse ** 2).sum() / n / z_ref) - 1) > 10 * GPU_TOL["stat"]           # ignored rows counted
    assert abs(float((lse ** 2).mean() / z_ref) - 1) > 10 * GPU_TOL["stat"]              # both
    # the z gradient without its factor 2, or divided by M, or given to the ignored rows
    p = torch.softmax(logits, -1)
    onehot = F.one_hot(labels.clamp(min=0), 64).double()
    no2 = lambda: ((1 + c * lse)[:, None] * p - onehot) * ok[:, None] / n
    by_m = lambda: (p - onehot) * ok[:, None] / n + 2 * c * lse[:, None] * p * ok[:, None] / M
    all_rows = lambda: (p - onehot) * ok[:, None] / n + 2 * c * lse[:, None] * p / n
    for bug in (no2, by_m, all_rows):
        assert _zpart_error(h, w, labels, c, bug) > 10 * GPU_TOL["zpart"]
    # the true gradient passes the same measure
    assert _zpart_error(h, w, labels, c, lambda: TK.cross_entropy_z_fwd_bwd(logits, labels, c)[2]) < 1e-12


@pytest.mark.parametrize("E,k", [(8, 2), (128, 8)])
def test_probes_plausible_router_bugs_miss_by_ten_times_the_gpu_tolerance(E, k):
    """On router logits of the size they have at initialisation (std 0.1), in float64."""
    T, cz = 256, 1e-3
    logits = torch.randn(T, E, generator=torch.Generator().manual_seed(E), dtype=torch.float64) * 0.1
    ids = TK.moe_route(logits, k, True)[0].long()
    p = torch.softmax(logits, -1)
    lse, _ = TK.router_z_fwd(logits)
    zpart = lambda probs, scale: TK.router_z_bwd(torch.zeros_like(logits), probs, lse, scale)
    good = zpart(p, 2 * cz / T)
    topk = zpart(torch.zeros_like(p).scatter_(1, ids, p.gather(1, ids)), 2 * cz / T)   # top-k probabilities only
    half = zpart(p, cz / T)                                                            # the factor 2 missing
    for bad in (topk, half):
        assert rel(bad, good) > 10 * GPU_TOL["router_zpart"]


# ------------------------------------------------------------------------------------------------ models
def test_zero_coefficients_take_todays_path(monkeypatch):
    """c = 0 never touches the z entries, and moe_mlp keeps its (y, aux) return."""
    def boom(*a, **k):
        raise AssertionError("z entry called with a zero coefficient")
    monkeypatch.setattr(ops, "linear_cross_entropy_z", boom)
    for v in ("llama2_tiny", "llama_moe_tiny"):
        torch.manual_seed(0)
        m = LLaMA(get_model_config(v))
        m.reset_parameters()
        x = torch.randint(0, 1024, (2, 16))
        m(x, labels=x).backward()
        assert m.z_loss() is None and m.moe_router_z_loss() is None
        if v == "llama_moe_tiny":
            assert m.layers[0].moe.last_router_z is None


def test_moe_model_reports_coefficient_scaled_terms():
    cfg = get_model_config("llama_moe_tiny")
    cfg.z_loss_coef, cfg.moe_router_z_loss_coef = 1e-3, 1e-2
    torch.manual_seed(0)
    m = LLaMA(cfg)
    m.reset_parameters()
    x = torch.randint(0, 1024, (2, 16))
    ce = m(x, labels=x)
    h = m(x, return_hidden=True)
    lse = torch.logsumexp(h.reshape(-1, h.shape[-1]) @ m.shared.head.weight.t(), -1)
    assert float(m.z_loss().detach()) == pytest.approx(1e-3 * float((lse ** 2).mean()), rel=1e-5)
    zr = torch.stack([b.moe.last_router_z for b in m.layers]).mean()
    assert float(m.moe_router_z_loss()) == pytest.approx(1e-2 * float(zr), rel=1e-6)
    assert ce.requires_grad and float(ce) > 0


# ------------------------------------------------------------------------------------------------ engine
STEPS, ACCUM, B, S, V = 2, 2, 2, 32, 1024
ZC, RZC = 1e-2, 5e-2


def _cfg():
    cfg = get_model_config("llama_moe_tiny")
    cfg.z_loss_coef, cfg.moe_router_z_loss_coef = ZC, RZC
    return cfg


def _batch(rank, step, micro):
    g = torch.Generator().manual_seed(1000 * step + 10 * micro + rank)
    return torch.randint(0, V, (B, S), generator=g)


def _worker(rank, world, port, outdir):
    from fms_fsdp_b200.parallel import ShardedAdamW, ShardedModel
    from fms_fsdp_b200.policies import fp32_policy
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        torch.manual_seed(0)
        m = LLaMA(_cfg())
        m.reset_parameters()
        eng = ShardedModel(m, sharding_strategy="fsdp", mixed_precision=fp32_policy, device="cpu",
                           collective_impl="torch", grad_accum_steps=ACCUM)
        opt = ShardedAdamW(eng, lr=1e-3)
        losses, norms = [], []
        for st in range(STEPS):
            tot = 0.0
            for mb in range(ACCUM):
                x = _batch(rank, st, mb)
                t = eng.forward_backward(x, x).clone()
                dist.all_reduce(t)
                tot += t.item() / (world * ACCUM)
            norms.append(eng.clip_grad_norm_(1.0).item())
            opt.step()
            losses.append(tot)
        sd = eng.full_state_dict()
        if rank == 0:
            torch.save(dict(losses=losses, norms=norms, sd=sd), os.path.join(outdir, "out.pt"))
    finally:
        dist.barrier()
        dist.destroy_process_group()


def test_world2_fsdp_with_accumulation_and_both_z_losses_matches_the_oracle():
    """The output z-loss's gradient rides in the head's, so the loss scaling of the oracle applies to it; the router's
    enters each MoE backward at unit scale (like the load-balancing gradient), so the oracle's router coefficient is
    divided by world x micro-batches."""
    world = 2
    outdir = tempfile.mkdtemp()
    mp.spawn(_worker, args=(world, free_port(), outdir), nprocs=world, join=True)
    out = torch.load(os.path.join(outdir, "out.pt"), weights_only=False)
    torch.manual_seed(0)
    cfg = _cfg()
    cfg.moe_router_z_loss_coef = RZC / (world * ACCUM)
    cfg.moe_aux_loss_coef /= world * ACCUM
    m = LLaMA(cfg)
    m.reset_parameters()
    opt = torch.optim.AdamW(m.parameters(), lr=1e-3, betas=(0.9, 0.95), weight_decay=0.1)
    for st in range(STEPS):
        opt.zero_grad()
        tot = 0.0
        for r in range(world):
            for mb in range(ACCUM):
                x = _batch(r, st, mb)
                l = m(x, labels=x) / (world * ACCUM)
                l.backward()
                tot += l.item()
        norm = torch.nn.utils.clip_grad_norm_(m.parameters(), 1.0).item()
        opt.step()
        assert out["losses"][st] == pytest.approx(tot, rel=2e-4, abs=2e-4)
        assert out["norms"][st] == pytest.approx(norm, rel=2e-3)
    for k_, v in m.state_dict().items():
        assert torch.allclose(out["sd"][k_], v, atol=2e-5, rtol=1e-4), k_


# ------------------------------------------------------------------------------------------------ entry points
def _train(variant, *flags):
    cmd = [sys.executable, os.path.join(ROOT, "main_training_llama.py"), f"--model_variant={variant}",
           "--use_dummy_dataset=True", "--seq_length=32", "--vocab_size=1024", "--batch_size=2", "--num_steps=2",
           "--report_interval=1", "--checkpoint_interval=1000", f"--ckpt_save_path={tempfile.mkdtemp()}",
           "--sharding_strategy=fsdp", "--comm_backend=gloo", "--use_torch_compile=False", *flags]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT,
                       env=dict(os.environ, OMP_NUM_THREADS="1"))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    keys = lambda name: [float(x) for x in re.findall(rf"^{name}: ([0-9.eE+-]+)$", r.stdout, flags=re.M)]
    return keys("loss"), keys("z_loss"), keys("moe_router_z_loss")


def test_entry_point_prints_the_z_keys_only_when_enabled():
    loss, z, rz = _train("llama2_tiny")
    assert len(loss) == 2 and not z and not rz
    loss, z, rz = _train("llama2_tiny", "--z_loss_coef=1e-3")
    # coef * mean lse^2, lse about log(1024) at init
    assert len(z) == 2 and not rz and all(1e-3 * 20 < v < 1e-3 * 200 for v in z), z
    assert all(5 < l < 9 for l in loss), loss                # loss stays the cross-entropy
    loss, z, rz = _train("llama_moe_tiny", "--z_loss_coef=1e-3", "--moe_router_z_loss_coef=1e-2")
    # router logits start near 0: lse about log(E) = log 8
    assert len(z) == 2 and len(rz) == 2 and all(1e-2 * 2 < v < 1e-2 * 10 for v in rz), rz


def test_router_coefficient_on_a_model_without_router_is_refused():
    import main_training_llama
    import main_training_mamba
    with pytest.raises(ValueError, match="mixture-of-experts"):
        main_training_llama.main(model_variant="llama2_tiny", moe_router_z_loss_coef=1e-3, use_dummy_dataset=True,
                                 comm_backend="gloo")
    with pytest.raises(ValueError, match="router"):
        main_training_mamba.main(model_variant="mamba_tiny", moe_router_z_loss_coef=1e-3, use_dummy_dataset=True,
                                 comm_backend="gloo")


def test_mamba_head_folds_the_z_gradient():
    from fms_fsdp_b200.models.mamba import MambaConfig, MambaLMHeadModel
    from fms_fsdp_b200.utils.config_utils import get_model_config as gmc
    torch.manual_seed(0)
    m = MambaLMHeadModel(MambaConfig(**gmc("mamba_tiny")))
    m.reset_parameters()
    x = torch.randint(0, 256, (2, 32))
    ref = m(x, labels=x)
    assert m.z_loss() is None
    m.z_loss_coef = 1e-2
    ce = m(x, labels=x)
    assert float(ce) == pytest.approx(float(ref), rel=1e-6) and float(m.z_loss()) > 0
    g = torch.autograd.grad(ce, m.lm_head.weight)[0]
    g0 = torch.autograd.grad(ref, m.lm_head.weight)[0]
    assert not torch.allclose(g, g0)


# ------------------------------------------------------------------------------------------------ effect
def _mean_lse2_after_training(c, steps=20):
    torch.manual_seed(0)
    cfg = get_model_config("llama2_tiny")
    cfg.z_loss_coef, cfg.src_vocab_size = c, 1024
    m = LLaMA(cfg)
    m.reset_parameters()
    opt = torch.optim.AdamW(m.parameters(), lr=3e-3)
    g = torch.Generator().manual_seed(0)
    for _ in range(steps):
        x = torch.randint(0, cfg.src_vocab_size, (2, 32), generator=g)
        opt.zero_grad()
        m(x, labels=x).backward()
        opt.step()
    x = torch.randint(0, cfg.src_vocab_size, (4, 32), generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        return float((torch.logsumexp(m(x).float(), -1) ** 2).mean())


def test_a_large_z_loss_keeps_the_normaliser_small():
    assert _mean_lse2_after_training(1e-1) < 0.9 * _mean_lse2_after_training(0.0)
