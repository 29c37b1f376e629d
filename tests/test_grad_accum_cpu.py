"""Gradient accumulation (``grad_accum_steps = k``) on CPU / gloo.

k micro-batches of b sequences per optimizer step must give the update of ONE step over k*b sequences: the engine
sums the micro-step gradients in fp32 and applies 1/k where a scale is applied anyway (the clip coefficient handed to
the fused AdamW).  The oracle is the plain single-process model trained with torch.optim.AdamW on the big batch."""
import os
import re
import subprocess
import sys
import tempfile

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import free_port
from fms_fsdp_b200.models.llama import LLaMA, LLaMABlock
from fms_fsdp_b200.models.mamba import Block as MambaBlock, MambaConfig, MambaLMHeadModel
from fms_fsdp_b200.parallel import ShardedAdamW, ShardedModel
from fms_fsdp_b200.policies import apply_fsdp_checkpointing, bfSixteen, fp32_policy
from fms_fsdp_b200.utils.config_utils import get_model_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STEPS, B, S = 3, 2, 32
# AdamW's eps: its first steps move every weight by about lr * g / (|g| + eps), so gradient elements that cancel to ~1e-9
# would turn last-bit summation differences into visible weight differences; 1e-6 keeps the comparison well conditioned
# (weights then agree to within 0.5 % of one lr step: atol 5e-6 at lr 1e-3)
EPS = 1e-6
VOCAB = {"llama": 1024, "mamba": 512}


def _model(kind):
    torch.manual_seed(0)
    if kind == "llama":
        m = LLaMA(get_model_config("llama2_tiny"))
    else:
        m = MambaLMHeadModel(MambaConfig(**get_model_config("mamba_tiny")))
    m.reset_parameters()
    return m


def _micro_batch(kind, rank, step, micro):
    g = torch.Generator().manual_seed(100000 * step + 1000 * micro + rank)
    return torch.randint(0, VOCAB[kind], (B, S), generator=g)


def _oracle(kind, world, k):
    """One step = per rank ONE batch of k*b sequences (the k micro-batches concatenated), loss averaged over ranks."""
    m = _model(kind)
    opt = torch.optim.AdamW(m.parameters(), lr=1e-3, betas=(0.9, 0.95), eps=EPS, weight_decay=0.1)
    losses, norms = [], []
    for st in range(STEPS):
        opt.zero_grad()
        tot = 0.0
        for r in range(world):
            x = torch.cat([_micro_batch(kind, r, st, j) for j in range(k)])
            l = m(x, labels=x) / world
            l.backward()
            tot += l.item()
        norms.append(torch.nn.utils.clip_grad_norm_(m.parameters(), 1.0).item())
        opt.step()
        losses.append(tot)
    return losses, norms, {n: p.detach().clone() for n, p in m.named_parameters()}


def _train(eng, opt, kind, rank, k, form):
    losses, norms = [], []
    for st in range(STEPS):
        tot = 0.0
        for j in range(k):
            x = _micro_batch(kind, rank, st, j)
            if form == "fused":
                l = eng.forward_backward(x, x)
            elif form == "fused_autograd":  # reference-style with the fused loss: loss = model(x, labels); loss.backward()
                l = eng(x, x)
                l.backward()
            else:                         # reference-style: logits, external cross-entropy, loss.backward()
                out = eng(x)
                l = torch.nn.functional.cross_entropy(out.view(-1, out.size(-1)), x.view(-1))
                l.backward()
            tot = tot + l.detach()
        norms.append(eng.clip_grad_norm_(1.0).item())
        opt.step()
        losses.append(tot / k)
    return losses, norms


def _worker(rank, world, port, kind, strategy, shard, ac, k, form, outdir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        m = _model(kind)
        if ac:
            apply_fsdp_checkpointing(m, LLaMABlock if kind == "llama" else MambaBlock, ac)
        eng = ShardedModel(m, sharding_strategy=strategy, hsdp_shard_size=shard, mixed_precision=fp32_policy,
                           device="cpu", collective_impl="torch", grad_accum_steps=k)
        opt = ShardedAdamW(eng, lr=1e-3, eps=EPS)
        # count the HSDP replica all-reduces of gradient shards: one per unit and OPTIMIZER step, not per micro-step
        replica_calls = [0]
        real_all_reduce = dist.all_reduce

        def counting_all_reduce(t, *a, **kw):
            if eng.mesh.replica_size > 1 and kw.get("group") is eng.mesh.replica_group:
                replica_calls[0] += 1
            return real_all_reduce(t, *a, **kw)
        dist.all_reduce = counting_all_reduce
        try:
            losses, norms = _train(eng, opt, kind, rank, k, form)
        finally:
            dist.all_reduce = real_all_reduce
        mean_losses = []
        for l in losses:
            t = l.clone(); dist.all_reduce(t); mean_losses.append(t.item() / world)
        sd = eng.full_state_dict()
        if rank == 0:
            torch.save(dict(losses=mean_losses, norms=norms, sd=sd, replica_calls=replica_calls[0],
                            units=len(eng.units)), os.path.join(outdir, "out.pt"))
    finally:
        dist.barrier()
        dist.destroy_process_group()


def _run(world, kind="llama", strategy="fsdp", shard=0, ac=None, k=2, form="fused"):
    outdir = tempfile.mkdtemp()
    mp.spawn(_worker, args=(world, free_port(), kind, strategy, shard, ac, k, form, outdir), nprocs=world, join=True)
    return torch.load(os.path.join(outdir, "out.pt"), weights_only=False)


def _check(out, kind, world, k):
    losses, norms, sd = _oracle(kind, world, k)
    assert out["losses"] == pytest.approx(losses, rel=1e-5)
    assert out["norms"] == pytest.approx(norms, rel=1e-5)
    for n, v in sd.items():
        assert torch.allclose(out["sd"][n], v, rtol=1e-5, atol=5e-6), (n, (out["sd"][n] - v).abs().max())


@pytest.mark.parametrize("world,strategy,shard,k,ac,form", [
    (2, "fsdp", 0, 2, None, "fused"),
    (4, "fsdp", 0, 4, None, "fused"),
    (2, "ddp", 0, 2, None, "fused"),
    (2, "fsdp", 0, 2, "1/2", "fused"),
    (2, "fsdp", 0, 2, None, "logits"),
    (2, "ddp", 0, 4, "1/2", "logits"),
    (2, "ddp", 0, 2, None, "fused_autograd"),
    (2, "fsdp", 0, 2, None, "fused_autograd"),
])
def test_accumulation_equals_the_big_batch(world, strategy, shard, k, ac, form):
    _check(_run(world, "llama", strategy, shard, ac, k, form), "llama", world, k)


def test_hsdp_2x2_replica_all_reduce_once_per_step():
    out = _run(4, "llama", "hsdp", 2, None, 2, "fused")
    _check(out, "llama", 4, 2)
    assert out["replica_calls"] == STEPS * out["units"]


def test_mamba_hybrid_accumulation_equals_the_big_batch():
    _check(_run(2, "mamba", "fsdp", 0, None, 2, "fused"), "mamba", 2, 2)


@pytest.mark.parametrize("form", ["fused", "logits", "fused_autograd"])
def test_single_process_accumulates_locally(form):
    """One process = unsharded: micro-gradients add up in the persistent (fp32) gradient buffer, nothing is reduced."""
    eng = ShardedModel(_model("llama"), mixed_precision=fp32_policy, device="cpu", grad_accum_steps=3)
    assert all(u.grad_shard.dtype == torch.float32 for u in eng.units)
    losses, norms = _train(eng, ShardedAdamW(eng, lr=1e-3, eps=EPS), "llama", 0, 3, form)
    ref_losses, ref_norms, sd = _oracle("llama", 1, 3)
    assert [l.item() for l in losses] == pytest.approx(ref_losses, rel=1e-5)
    assert norms == pytest.approx(ref_norms, rel=1e-5)
    mine = eng.full_state_dict()
    for n, v in sd.items():
        assert torch.allclose(mine[n], v, rtol=1e-5, atol=5e-6), (n, (mine[n] - v).abs().max())


def test_scaled_fused_loss_scales_every_micro_step():
    """``(model(x, labels) * c).backward()`` on every micro-step scales the accumulated gradient by c, also from micro-step
    2 on, where the unsharded (one-process) mesh already holds micro-step 1 in its gradient buffer."""
    norms = []
    for c in (1.0, 0.25):
        eng = ShardedModel(_model("llama"), mixed_precision=fp32_policy, device="cpu", grad_accum_steps=2)
        for j in range(2):
            x = _micro_batch("llama", 0, 0, j)
            (eng(x, x) * c).backward()
        norms.append(eng.clip_grad_norm_(1e9).item())
    assert norms[1] == pytest.approx(0.25 * norms[0], rel=1e-5)


def test_unsharded_gradient_buffer_is_fp32_under_accumulation():
    """bf16 policy: the gradient buffer follows reduce_dtype at k = 1 and is fp32 at k > 1."""
    e1 = ShardedModel(_model("llama"), mixed_precision=bfSixteen, device="cpu")
    e2 = ShardedModel(_model("llama"), mixed_precision=bfSixteen, device="cpu", grad_accum_steps=2)
    assert {u.grad_shard.dtype for u in e1.units} == {torch.bfloat16}
    assert {u.grad_shard.dtype for u in e2.units} == {torch.float32}
    opt = ShardedAdamW(e2, lr=3e-3)
    x0, x1 = _micro_batch("llama", 0, 0, 0), _micro_batch("llama", 0, 0, 1)
    first = None
    for _ in range(6):
        l = (e2.forward_backward(x0, x0) + e2.forward_backward(x1, x1)) / 2
        e2.clip_grad_norm_(1.0); opt.step()
        first = l.item() if first is None else first
    assert l.item() < first


@pytest.mark.parametrize("policy", ["fp32", "bf16"])
def test_k1_is_bitwise_unchanged(policy):
    mp_ = fp32_policy if policy == "fp32" else bfSixteen

    def run(**kw):
        eng = ShardedModel(_model("llama"), mixed_precision=mp_, device="cpu", **kw)
        return eng, _train(eng, ShardedAdamW(eng, lr=1e-3), "llama", 0, 1, "fused")

    ea, (la, na) = run()
    eb, (lb, nb) = run(grad_accum_steps=1)
    assert [x.item() for x in la] == [x.item() for x in lb] and na == nb
    sa, sb = ea.full_state_dict(), eb.full_state_dict()
    assert all(torch.equal(sa[n], sb[n]) for n in sa)
    assert all(u.grad_shard.dtype == v.grad_shard.dtype for u, v in zip(ea.units, eb.units))


def test_errors():
    with pytest.raises(ValueError, match="grad_accum_steps"):
        ShardedModel(_model("llama"), device="cpu", grad_accum_steps=0)
    eng = ShardedModel(_model("llama"), mixed_precision=fp32_policy, device="cpu", grad_accum_steps=3)
    opt = ShardedAdamW(eng, lr=1e-3)
    x = _micro_batch("llama", 0, 0, 0)
    eng.forward_backward(x, x)
    eng.forward_backward(x, x)
    with pytest.raises(RuntimeError, match="after 2 micro-step"):
        eng.clip_grad_norm_(1.0)
    with pytest.raises(RuntimeError, match="after 2 micro-step"):
        opt.step()
    assert opt._step == 0
    eng.forward_backward(x, x)
    with pytest.raises(RuntimeError, match="already run"):
        eng.forward_backward(x, x)
    eng.clip_grad_norm_(1.0)
    opt.step()                                          # exactly k micro-steps: fine
    assert opt._step == 1
    with pytest.raises(RuntimeError, match="after 0 micro-step"):
        opt.step()


def test_unclipped_step_uses_the_mean_gradient():
    """Without clip_grad_norm_ AdamW still sees the mean micro-batch gradient (scale 1/k): summing two identical
    micro-batches at k = 2 gives exactly the update of one of them at k = 1."""
    x = _micro_batch("llama", 0, 0, 0)
    e1 = ShardedModel(_model("llama"), mixed_precision=fp32_policy, device="cpu")
    e2 = ShardedModel(_model("llama"), mixed_precision=fp32_policy, device="cpu", grad_accum_steps=2)
    o1, o2 = ShardedAdamW(e1, lr=1e-3, eps=1e-30), ShardedAdamW(e2, lr=1e-3, eps=1e-30)
    e1.forward_backward(x, x); o1.step()
    e2.forward_backward(x, x); e2.forward_backward(x, x); o2.step()
    s1, s2 = e1.full_state_dict(), e2.full_state_dict()
    for n in s1:
        assert torch.allclose(s1[n], s2[n], rtol=1e-6, atol=1e-8), n


def test_memory_plan_unsharded_gradient_is_fp32():
    from fms_fsdp_b200.utils.memory_plan import plan_llama
    p1 = plan_llama("llama2_1.4b", gpus=1)
    p2 = plan_llama("llama2_1.4b", gpus=1, grad_accum_steps=2)
    eng_params = (p1.parts_gib["master + bf16 shard + AdamW moments (14 B/param / shard)"]) / 14.0
    assert p2.total_gib - p1.total_gib == pytest.approx(2.0 * eng_params, rel=1e-9)
    for kw in (dict(gpus=8), dict(gpus=8, sharding_strategy="hsdp", hsdp_shard_size=4)):
        assert plan_llama("llama2_1.4b", grad_accum_steps=4, **kw).total_gib == \
            pytest.approx(plan_llama("llama2_1.4b", **kw).total_gib, rel=1e-12)


# ------------------------------------------------------------------------------------------------ entry point
def _write_arrow(path, docs):
    import pyarrow as pa
    os.makedirs(os.path.dirname(path), exist_ok=True)
    schema = pa.schema([pa.field("tokens", pa.uint32())])
    with pa.ipc.new_file(path, schema) as w:
        for d in docs:
            w.write(pa.record_batch([pa.array(d, type=pa.uint32())], schema=schema))


def _corpus(tmp):
    _write_arrow(f"{tmp}/dataset_1/a.arrow", [[(7 * i + j) % 500 + 1 for j in range(90)] for i in range(60)])
    _write_arrow(f"{tmp}/dataset_2/b.arrow", [[(11 * i + 3 * j) % 500 + 1 for j in range(40)] for i in range(80)])
    os.makedirs(f"{tmp}/meta")
    with open(f"{tmp}/meta/combined_counts.csv", "w") as f:
        f.write("dataset/filename,documents,tokens\n/dataset_1/a.arrow,60,5400\n/dataset_2/b.arrow,80,3200\n")


def _main(ckpt, steps, k, data=None, interval=100):
    cmd = [sys.executable, os.path.join(ROOT, "main_training_llama.py"), "--model_variant=llama2_tiny",
           "--seq_length=32", "--vocab_size=512", "--batch_size=2", f"--num_steps={steps}", "--report_interval=1",
           f"--checkpoint_interval={interval}", f"--ckpt_save_path={ckpt}", f"--ckpt_load_path={ckpt}",
           "--sharding_strategy=fsdp", "--comm_backend=gloo", "--use_torch_compile=False", f"--grad_accum_steps={k}"]
    if data is None:
        cmd.append("--use_dummy_dataset=True")
    else:
        cmd += ["--use_dummy_dataset=False", f"--data_path={data}", "--datasets=dataset_1,dataset_2", "--weights=2,1",
                "--file_type=arrow", "--col_name=tokens", "--logical_shards=8", "--num_workers=1", "--eos_token=0"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT,
                       env=dict(os.environ, OMP_NUM_THREADS="1"))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout


def _report(out, key):
    return [float(v) for v in re.findall(rf"^{key}: ([0-9.eE+-]+)$", out, flags=re.M)]


def _model_tensors(step_dir):
    import torch.distributed.checkpoint as dcp
    ref = LLaMA(get_model_config("llama2_tiny"))
    full = {"model_state": {k: torch.empty_like(v) for k, v in ref.state_dict().items()}}
    dcp.load(full, checkpoint_id=step_dir, no_dist=True)
    return full["model_state"]


@pytest.mark.parametrize("loader", ["dummy", "arrow"])
def test_entrypoint_counts_optimizer_steps_and_tokens(tmp_path, loader):
    data = None
    if loader == "arrow":
        data = str(tmp_path / "data")
        _corpus(data)
    o1 = _main(str(tmp_path / "k1"), 4, 1, data, interval=2)
    o2 = _main(str(tmp_path / "k2"), 4, 2, data, interval=2)
    assert _report(o2, "step") == [1, 2, 3, 4]
    t1, t2 = _report(o1, "tokens seen"), _report(o2, "tokens seen")
    assert t2 == [2 * t for t in t1] and t1[-1] == 4 * 2 * 32
    for step in (2, 4):
        d = tmp_path / "k2" / "checkpoints" / f"step_{step}_ckp"
        files = os.listdir(d)
        assert "metadata.pth" in files, files
        if loader == "arrow":                     # loader state written at the same optimizer steps as the model
            assert any(f.startswith("loader_state") for f in files), files
    if loader == "arrow":
        # the loader counts optimizer steps: at step 2 of k = 2 it has emitted the 8 sequences k = 1 emits by step 4 (a
        # loader counting its own batches would save the k = 1 step-2 state there instead)
        def state(run, step):
            return torch.load(tmp_path / run / "checkpoints" / f"step_{step}_ckp" / "loader_state_0.pth", weights_only=False)
        assert _same(state("k2", 2), state("k1", 4))
        assert not _same(state("k2", 2), state("k1", 2))


def _same(a, b):
    if torch.is_tensor(a):
        return torch.is_tensor(b) and torch.equal(a, b)
    if isinstance(a, dict):
        return isinstance(b, dict) and a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return isinstance(b, (list, tuple)) and len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return a == b


def test_checkpoint_resume_mid_run_matches_uninterrupted(tmp_path):
    """k = 2: stop after optimizer step 2, save, load into a fresh engine and continue -- steps 3 and 4 give the losses
    and weights of the uninterrupted run (same micro-batches; the micro-step counter starts over after a step)."""
    from fms_fsdp_b200.utils.checkpointing_utils import Checkpointer

    def engine(seed):
        torch.manual_seed(seed)
        m = LLaMA(get_model_config("llama2_tiny")); m.reset_parameters()
        eng = ShardedModel(m, mixed_precision=fp32_policy, device="cpu", grad_accum_steps=2)
        return eng, ShardedAdamW(eng, lr=1e-3, eps=EPS)

    def steps(eng, opt, first, last):
        out = []
        for st in range(first, last):
            ls = [eng.forward_backward(x, x) for x in (_micro_batch("llama", 0, st, j) for j in range(2))]
            out.append(((ls[0] + ls[1]) / 2).item())
            eng.clip_grad_norm_(1.0); opt.step()
        return out

    eng, opt = engine(0)
    full = steps(eng, opt, 0, 4)
    ref = eng.full_state_dict()
    eng, opt = engine(0)
    steps(eng, opt, 0, 2)
    Checkpointer(str(tmp_path), 5, "fsdp", 0, 0).save(2, eng, opt, None, tokens_seen=2 * 2 * B * S)
    eng, opt = engine(7)                      # different init: everything must come from the checkpoint
    _, _, _, step, ntok, resuming = Checkpointer(str(tmp_path), 5, "fsdp", 0, 0).load(eng, opt, None, path="")
    assert (step, ntok, resuming, opt._step) == (2, 2 * 2 * B * S, True, 2)
    assert steps(eng, opt, 2, 4) == pytest.approx(full[2:], rel=1e-6)
    mine = eng.full_state_dict()
    for n, v in ref.items():
        assert torch.allclose(mine[n], v, rtol=1e-6, atol=1e-7), n
