"""Gradient accumulation on one H100: Llama2-1.4B, seq 4096, batch 2, grad_accum_steps k in {1, 2, 4}.

Device-timed tokens/s per optimizer step (CUDA events around whole optimizer steps: k forward_backward micro-steps, clip,
AdamW), the k values timed alternately in rounds within one process; the allocator peak of each engine next to its
memory plan; the card's name, power limit and max SM clock read in the same run.  Two engines live in the process (three
do not fit in 80 GB): one at k = 1 (bf16 unsharded gradient buffer) and one accumulating engine (fp32 buffer) whose k is
switched between 2 and 4 between optimizer steps.  The allocator peak of each k is measured over a step at that k, net of
the memory the other engine holds.
Writes $DIAG_OUT/accum_bench.json (default diag_out/ in the repository root).
usage: python scripts/accum_bench.py [--rounds 5] [--steps 3]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from fms_fsdp_b200.models.llama import LLaMA
from fms_fsdp_b200.ops import cuda_kernels as CK
from fms_fsdp_b200.parallel import ShardedAdamW, ShardedModel
from fms_fsdp_b200.policies import bfSixteen
from fms_fsdp_b200.utils.config_utils import get_model_config
from fms_fsdp_b200.utils.memory_plan import plan_llama

MODEL, SEQ, BATCH = "llama2_1.4b", 4096, 2
GiB = float(2 ** 30)


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        return r.stdout.strip()
    except Exception as ex:
        return f"nvidia-smi unavailable: {ex!r}"


def build(k, dev):
    mcfg = get_model_config(MODEL)
    with torch.device("meta"):
        model = LLaMA(mcfg)
    eng = ShardedModel(model, sharding_strategy="fsdp", mixed_precision=bfSixteen, device=dev, grad_accum_steps=k)
    model.rot_emb.compute_freqs_cis(dev, mcfg.max_expected_seq_len)
    return eng, ShardedAdamW(eng, lr=3e-4, betas=(0.9, 0.95), weight_decay=0.1), mcfg.src_vocab_size


def set_accum(eng, k):
    """Switch the accumulating engine between k values between optimizer steps (its fp32 buffer serves any k > 1)."""
    eng.grad_accum_steps = k
    eng._inv_accum.fill_(1.0 / k)


def step(eng, opt, batches):
    for x in batches:
        eng.forward_backward(x, x)
    eng.clip_grad_norm_(1.0)
    opt.step()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3, help="optimizer steps per timed window")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("accum_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = gpu_info()
    g = torch.Generator().manual_seed(0)
    pool = [torch.randint(0, 32000, (BATCH, SEQ), generator=g).to(dev) for _ in range(4)]

    res = {"gpu": info, "model": MODEL, "seq": SEQ, "batch": BATCH, "rounds": a.rounds, "steps_per_window": a.steps}
    engines, own, peaks = {}, {}, {}
    for key, k in (("k1", 1), ("acc", 2)):
        before = torch.cuda.memory_allocated(dev)
        engines[key] = build(k, dev)[:2]
        step(*engines[key], pool[:k])                     # first step: every lazily allocated buffer exists afterwards
        torch.cuda.synchronize()
        own[key] = torch.cuda.memory_allocated(dev) - before     # what this engine holds between steps
    for k in (1, 2, 4):
        key = "k1" if k == 1 else "acc"
        eng, opt = engines[key]
        if k > 1:
            set_accum(eng, k)
        step(eng, opt, pool[:k])                          # warm-up: every shape of the timed window
        torch.cuda.synchronize()
        rest = torch.cuda.memory_allocated(dev)           # both engines between steps
        torch.cuda.reset_peak_memory_stats(dev)
        step(eng, opt, pool[:k])
        torch.cuda.synchronize()
        # this engine's resident memory + what one step at this k adds on top of everything resident
        peaks[k] = (own[key] + torch.cuda.max_memory_allocated(dev) - rest) / GiB

    f0 = CK.fallback_count()
    times = {1: [], 2: [], 4: []}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(a.rounds):
        for k in (1, 2, 4):
            eng, opt = engines["k1" if k == 1 else "acc"]
            if k > 1:
                set_accum(eng, k)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(a.steps):
                step(eng, opt, pool[:k])
            e1.record()
            e1.synchronize()
            times[k].append(e0.elapsed_time(e1) / 1e3 / a.steps)
    res["aten_fallbacks_in_timed_window"] = CK.fallback_count() - f0
    for k in (1, 2, 4):
        ts = times[k]
        tok = [k * BATCH * SEQ / t for t in ts]
        plan = plan_llama(MODEL, gpus=1, batch_size=BATCH, seq_length=SEQ, grad_accum_steps=k)
        res[f"k{k}"] = {
            "step_s_median": statistics.median(ts),
            "tokens_per_s_median": statistics.median(tok),
            "tokens_per_s_min": min(tok), "tokens_per_s_max": max(tok),
            "alloc_peak_gib": peaks[k],
            "plan_gib": plan.total_gib,
        }
    res["gpu_after"] = gpu_info()
    out_dir = os.environ.get("DIAG_OUT", os.path.join(ROOT, "diag_out"))
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "accum_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
