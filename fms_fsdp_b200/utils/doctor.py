"""Environment check before a run:  ``python -m fms_fsdp_b200.utils.doctor``

Reports, without starting a job: Python / torch / CUDA versions, whether the in-tree sm_90a extension is built and loads, the
visible GPUs (name, compute capability, memory, SM count), peer access between every pair of GPUs (the NVLink collectives need
it), NCCL and symmetric-memory availability, the measured roofline file the MFU line uses, and the reference install the bench's
reference arm needs.  Exit status 1 if something that a GPU training run requires is missing; on a machine without a GPU it
only describes the CPU (ATen) path.
"""
from __future__ import annotations

import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def collect() -> dict:
    import torch
    import torch.distributed as dist

    info: dict = {"python": sys.version.split()[0], "torch": torch.__version__, "cuda_runtime": torch.version.cuda,
                  "problems": [], "notes": []}
    so = os.path.join(ROOT, "fms_fsdp_b200", "_C.so")
    info["extension_built"] = os.path.exists(so)
    try:
        from fms_fsdp_b200.ops import _ext
        info["extension_loads"] = bool(_ext.available())
    except Exception as e:   # a broken build must not take the report down
        info["extension_loads"] = False
        info["notes"].append(f"extension import failed: {e!r}"[:200])
    info["nccl_available"] = bool(dist.is_available() and dist.is_nccl_available())
    try:
        import torch.distributed._symmetric_memory  # noqa: F401
        info["symmetric_memory_module"] = True
    except Exception:
        info["symmetric_memory_module"] = False
    peaks = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(peaks):
        with open(peaks) as f:
            p = json.load(f)
        info["measured_peaks"] = {k: p.get(k) for k in ("hbm_gbs", "bf16_tflops", "bf16_tflops_sustained", "gpu_name")}
    else:
        info["notes"].append("MEASURED_PEAKS.json absent: the MFU line uses the recipe's fallback of 1400 TFLOP/s")
    info["reference_install"] = os.path.isdir(os.path.join(ROOT, "baseline", "_ref", "fms_fsdp"))

    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    info["gpus"] = []
    for i in range(n):
        pr = torch.cuda.get_device_properties(i)
        info["gpus"].append({"index": i, "name": pr.name, "capability": f"{pr.major}.{pr.minor}",
                             "memory_gib": round(pr.total_memory / 2 ** 30, 1), "sms": pr.multi_processor_count})
    if n == 0:
        info["notes"].append("no CUDA device: ops run on the ATen path (kernel_path=torch), collectives on gloo")
        return info
    if not info["extension_built"] or not info["extension_loads"]:
        info["problems"].append("fms_fsdp_b200/_C.so missing or not loadable: run python -c 'import __graft_entry__ as g; g.build()'")
    for g in info["gpus"]:
        if g["capability"] != "9.0":
            info["problems"].append(f"GPU {g['index']} ({g['name']}) is sm_{g['capability'].replace('.', '')}; the kernels are "
                                    "compiled for sm_90a only")
    no_peer = [(a, b) for a in range(n) for b in range(n) if a != b and not torch.cuda.can_device_access_peer(a, b)]
    info["peer_access_all_pairs"] = not no_peer
    if no_peer:
        info["problems"].append(f"no peer access between GPU pairs {no_peer[:6]}: collective_impl=fused cannot be used "
                                "(collective_impl=torch runs over NCCL)")
    if n > 1 and not info["nccl_available"]:
        info["problems"].append("NCCL is not available: multi-GPU bootstrap needs it")
    if n > 1 and not info["symmetric_memory_module"]:
        info["problems"].append("torch symmetric memory is missing: the NVLink peer collectives cannot allocate their buffers")
    return info


def main() -> int:
    info = collect()
    for k, v in info.items():
        if k in ("problems", "notes", "gpus"):
            continue
        print(f"{k:26s} {v}")
    for g in info["gpus"]:
        print(f"gpu {g['index']}: {g['name']}, sm_{g['capability'].replace('.', '')}, {g['memory_gib']} GiB, {g['sms']} SMs")
    for n in info["notes"]:
        print("note:", n)
    for p in info["problems"]:
        print("PROBLEM:", p)
    print("ok" if not info["problems"] else f"{len(info['problems'])} problem(s)")
    return 1 if info["problems"] else 0


if __name__ == "__main__":
    sys.exit(main())
