"""The shipped extension is Hopper-native: every tensor-core instruction in it is a warpgroup MMA (SASS ``HGMMA`` /
``QGMMA``, from ``wgmma.mma_async``), operands arrive by TMA (``UTMALDG``) -- and there is not a single legacy warp-level
``HMMA`` (``mma.sync`` / ``wmma``) in the binary.  Runs wherever ``cuobjdump`` and the built ``_C.so`` exist (no GPU needed)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "fms_fsdp_b200", "_C.so")


@pytest.fixture(scope="module")
def kernels():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(SO) or not os.path.exists(exe):
        pytest.skip("needs the built extension and cuobjdump")
    out = subprocess.run([exe, "-sass", SO], capture_output=True, text=True, timeout=600).stdout
    assert "arch = sm_90a" in out
    assert not re.search(r"arch = sm_(?!90a)", out)
    per = {}
    name = None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            per[name] = []
        elif name and "/*" in line:
            per[name].append(line)
    return {k: "\n".join(v) for k, v in per.items()}


def _has(kernels, name_part, *mnemonics):
    hits = [k for k in kernels if name_part in k]
    assert hits, name_part
    for k in hits:
        for mn in mnemonics:
            assert re.search(mn, kernels[k]), (k, mn)
    return hits


def test_no_legacy_warp_level_mma_anywhere(kernels):
    legacy = [k for k, body in kernels.items() if re.search(r"(?<![A-Z])HMMA\.|(?<![A-Z])IMMA\.|(?<![A-Z])QMMA\.", body)]
    assert not legacy, legacy[:5]
    assert sum("HGMMA" in b or "QGMMA" in b for b in kernels.values()) >= 40     # GEMM + attention instantiations


def test_hot_kernels_use_wgmma_and_tma(kernels):
    gemm = _has(kernels, "gemm_bf16_wgmma", r"HGMMA\.64x128x16|QGMMA\.64x128x32", r"UTMALDG\.[24]D", r"WARPGROUP\.ARRIVE")
    assert len(gemm) >= 20
    _has(kernels, "attn_fwd_kernel", r"HGMMA\.64x128x16", r"UTMALDG", r"MUFU\.EX2")
    _has(kernels, "attn_bwd_kernel", r"HGMMA\.64x64x16", r"UTMALDG", r"MUFU\.EX2")
    # fp8 instantiation: e4m3 warpgroup MMA
    assert any("QGMMA.64x128x32.F32.E4M3.E4M3" in b for k, b in kernels.items() if "gemm_bf16_wgmma" in k)


def test_push_epilogue_and_peer_collectives(kernels):
    # EPI_PUSH = 4: wgrad push, with and without the fused all-gather
    push = [k for k in kernels if "gemm_bf16_wgmma" in k and "ELi4E" in k]
    assert len(push) >= 2
    assert all("UBLKCP.G.S" in kernels[k] for k in push)     # staged rows leave as cp.async.bulk stores
    # comm warps of the all-gather GEMMs read peers with system-scope 16-byte loads
    assert any("LDG.E.128.STRONG.SYS" in b for k, b in kernels.items() if "gemm_bf16_wgmma" in k)
    _has(kernels, "signal_barrier_kernel", r"ST\S*\.STRONG\.SYS|STG\S*\.SYS", r"LD\S*\.STRONG\.SYS")
    _has(kernels, "reduce_scatter", r"LDG\.E\.128")
