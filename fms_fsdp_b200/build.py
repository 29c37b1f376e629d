"""In-tree build of the sm_90a extension ``fms_fsdp_b200/_C.so``.

    python -m fms_fsdp_b200.build            # incremental
    python -m fms_fsdp_b200.build --force

* every ``csrc/*.cu`` is torch-free and compiled by nvcc for ``compute_90a/sm_90a`` with ``-lineinfo``
  (ncu source pages) -- nvcc cross-compiles without a GPU;
* ``csrc/bindings.cpp`` (torch/pybind) is compiled by g++ only;
* the .so stays in the tree (git-ignored), next to the package, so the package imports from the source tree.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "..", "build", "sm90_ext")
OUT = os.path.join(HERE, "_C.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CXX = os.environ.get("CXX", "g++")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O3", "-lineinfo",
              "--use_fast_math", "-Xcompiler", "-fPIC", "-Xptxas", "-v"]


def _digest(paths, extra=""):
    h = hashlib.sha1(extra.encode())
    for p in sorted(paths):
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def _run(cmd, log):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    with open(log, "w") as f:
        f.write(" ".join(cmd) + "\n" + r.stdout)
    if r.returncode != 0:
        raise RuntimeError(f"build step failed: {' '.join(cmd)}\n{r.stdout[-4000:]}")
    return r.stdout


def build(force: bool = False, verbose: bool = True) -> str:
    import torch
    from torch.utils import cpp_extension as ce

    os.makedirs(BUILD, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    cus = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))
    cpp = os.path.join(CSRC, "bindings.cpp")
    hdr_digest = _digest(headers, " ".join(NVCC_FLAGS) + torch.__version__)

    jobs = []
    objs = []
    for src in cus + [cpp]:
        base = os.path.basename(src)
        obj = os.path.join(BUILD, base + ".o")
        stamp = obj + ".sha"
        want = _digest([src], hdr_digest)
        objs.append(obj)
        have = open(stamp).read() if os.path.exists(stamp) else ""
        if force or have != want or not os.path.exists(obj):
            if src.endswith(".cu"):
                cmd = [NVCC] + NVCC_FLAGS + ["-I", CSRC, "-c", src, "-o", obj]
            else:
                incs = []
                for p in ce.include_paths(device_type="cuda") if "device_type" in ce.include_paths.__code__.co_varnames \
                        else ce.include_paths(cuda=True):
                    incs += ["-isystem", p]
                incs += ["-isystem", sysconfig.get_paths()["include"]]
                cmd = [CXX, "-std=c++17", "-O2", "-fPIC", "-DTORCH_EXTENSION_NAME=_C",
                       "-DTORCH_API_INCLUDE_EXTENSION_H", f"-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}",
                       "-I", CSRC] + incs + ["-c", src, "-o", obj]
            jobs.append((cmd, obj + ".log", stamp, want, base))

    def do(job):
        cmd, log, stamp, want, base = job
        _run(cmd, log)
        with open(stamp, "w") as f:
            f.write(want)
        return base

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for base in ex.map(do, jobs):
                if verbose:
                    print(f"[build] compiled {base}", flush=True)
    if jobs or force or not os.path.exists(OUT):
        tlib = os.path.join(os.path.dirname(torch.__file__), "lib")
        cuda_lib = "/usr/local/cuda/lib64"
        cmd = [CXX, "-shared", "-o", OUT] + objs + [
            f"-L{tlib}", f"-L{cuda_lib}", "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch",
            "-ltorch_python", "-lcudart", f"-Wl,-rpath,{tlib}", f"-Wl,-rpath,{cuda_lib}"]
        _run(cmd, os.path.join(BUILD, "link.log"))
        if verbose:
            print(f"[build] linked {OUT}", flush=True)
    return OUT


def ptxas_report() -> str:
    """Registers / spills per kernel from the last compile logs (``-Xptxas -v``)."""
    out = []
    if os.path.isdir(BUILD):
        for f in sorted(os.listdir(BUILD)):
            if f.endswith(".cu.o.log"):
                with open(os.path.join(BUILD, f)) as fh:
                    out.append(f"== {f}\n" + "".join(l for l in fh if "registers" in l or "spill" in l or "Compiling" in l))
    return "\n".join(out)


if __name__ == "__main__":
    build(force="--force" in sys.argv)
