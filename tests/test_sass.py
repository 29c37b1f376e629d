"""The SASS of the built extension ``_C.so``, read once with ``cuobjdump`` (no GPU needed).

``tests/golden/sass_kernels.json`` pins the instructions of every kernel (``scripts/sass_digest.py``, CUDA 12.9): a
change that means to change, add or remove kernels regenerates it with that script in the same commit, and its diff
names every kernel that changed.  The other tests hold each kernel family to the instructions it was written for: the
extension is Hopper-native (warpgroup MMAs, ``HGMMA`` / ``QGMMA``, fed by TMA, ``UTMALDG``, and not a single legacy
warp-level ``HMMA``), and the hot kernels keep out of local memory."""
import importlib.util
import json
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "fms_fsdp_b200", "_C.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "sass_kernels.json")

_spec = importlib.util.spec_from_file_location("sass_digest", os.path.join(ROOT, "scripts", "sass_digest.py"))
sass_digest = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(sass_digest)


@pytest.fixture(scope="module")
def per():
    """{kernel: [instruction text]} of every kernel of ``_C.so``."""
    exe = shutil.which("cuobjdump") or sass_digest.CUOBJDUMP
    if not os.path.exists(SO) or not os.path.exists(exe):
        pytest.skip("needs the built extension and cuobjdump")
    out = subprocess.run([exe, "-sass", SO], capture_output=True, text=True, timeout=600, check=True).stdout
    assert "arch = sm_90a" in out
    assert not re.search(r"arch = sm_(?!90a)", out)
    return sass_digest.parse(out)


@pytest.fixture(scope="module")
def kernels(per):
    """{kernel: its instructions as one text}"""
    return {k: "\n".join(v) for k, v in per.items()}


def _has(kernels, name_part, *mnemonics):
    hits = [k for k in kernels if name_part in k]
    assert hits, name_part
    for k in hits:
        for mn in mnemonics:
            assert re.search(mn, kernels[k]), (k, mn)
    return hits


def _no_local_memory(per, names):
    for k in names:
        assert not any(re.search(r"\b(LDL|STL)\b", i) for i in per[k]), k


def test_every_kernel_matches_the_golden(per):
    have = sass_digest.digests(per)
    with open(GOLDEN) as f:
        want = json.load(f)
    missing = sorted(set(want) - set(have))
    extra = sorted(set(have) - set(want))
    changed = sorted(k for k in set(want) & set(have) if want[k] != have[k])
    assert not (missing or extra or changed), dict(missing=missing, extra=extra, changed=changed)


def test_no_legacy_warp_level_mma_anywhere(kernels):
    legacy = [k for k, body in kernels.items() if re.search(r"(?<![A-Z])HMMA\.|(?<![A-Z])IMMA\.|(?<![A-Z])QMMA\.", body)]
    assert not legacy, legacy[:5]
    assert sum("HGMMA" in b or "QGMMA" in b for b in kernels.values()) >= 40     # GEMM + attention instantiations


def test_hot_kernels_use_wgmma_and_tma(kernels):
    gemm = _has(kernels, "gemm_bf16_wgmma", r"HGMMA\.64x128x16|QGMMA\.64x128x32", r"UTMALDG\.[24]D", r"WARPGROUP\.ARRIVE")
    assert len(gemm) >= 20
    _has(kernels, "attn_fwd_pipe_kernel", r"HGMMA\.64x128x16", r"UTMALDG", r"MUFU\.EX2")
    _has(kernels, "attn_bwd_pipe_kernel", r"HGMMA\.64x64x16", r"UTMALDG", r"MUFU\.EX2")
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


def test_wide_gemm_is_the_staged_kernel_with_tma_stores(kernels):
    """Every output of the 128 x 256 tile leaves through TMA stores: m64n256k16 MMAs, TMA loads and stores, no STG at
    all, no local memory; the tile has no other kernel."""
    staged = [k for k in kernels if "gemm_wide_staged_bf16" in k]
    # 4 layouts x (store, accumulate) x (bf16, fp32), +residual x 4, RoPE x 2, SwiGLU x 2
    assert len(staged) == 24, sorted(staged)
    for k in staged:
        body = kernels[k]
        assert re.search(r"HGMMA\.64x256x16\.F32\.BF16", body), k
        assert not re.search(r"HGMMA\.64x128x16", body), k
        assert re.search(r"UTMALDG\.2D", body), k
        assert re.search(r"UTMASTG", body), k
        assert not re.search(r"\bSTG\b", body), k
        assert not re.search(r"\b(LDL|STL)\b", body), k
    assert not [k for k in kernels if re.search(r"gemm_wide_(?!staged_bf16)", k)]


def test_grouped_gemm_and_moe_kernels(per):
    """Grouped GEMM instantiations carry GRP_M (16) or GRP_K (32) in their EPI argument."""
    grouped = [k for k in per if re.search(r"gemm_bf16_wgmmaILb[01]ELb[01]ELi(1[6-9]|2\d|3\d|4\d)E", k)]
    assert len(grouped) == 8, grouped
    for k in grouped:
        assert any("HGMMA" in i for i in per[k]) and any("UTMALDG" in i for i in per[k]), k
    moe = [k for k in per if "moe_" in k]
    assert len(moe) == 9, moe
    _no_local_memory(per, grouped + moe)


def test_qk_norm_kernels(per):
    qk = [k for k in per if "qk_norm" in k]
    assert len(qk) == 4, qk
    _no_local_memory(per, qk)


def test_pipelined_attention_kernels(per):
    """setmaxnreg is ``USETMAXREG`` in SASS; the dK/dV instantiations bring -lse / -delta in by ``UBLKCP``."""
    pipe = [k for k in per if "attn_fwd_pipe_kernel" in k or "attn_bwd_pipe_kernel" in k]
    assert len(pipe) == 4 + 8, pipe
    for k in pipe:
        body = per[k]
        assert any(i.startswith("HGMMA") for i in body) and any(i.startswith("UTMALDG") for i in body), k
        assert sum(i.startswith("USETMAXREG") for i in body) == 2, k          # producer dec + consumer inc
        assert not any(re.search(r"\b(LDL|STL)\b", i) for i in body), k
        # the overlap survives register allocation: a kernel whose wgmmas ptxas serialised (C7512) waits after every
        # HGMMA; the schedule waits at most 4 times (forward: S, PV in the loop and around it; backward: S, dP, end)
        depbar = sum(i.startswith("WARPGROUP.DEPBAR") for i in body)
        hgmma = sum(i.startswith("HGMMA") for i in body)
        assert depbar <= 4 and 3 * depbar <= hgmma, (k, depbar, hgmma)
        if "attn_bwd_pipe_kernelILi128ELi0E" in k or "attn_bwd_pipe_kernelILi64ELi0E" in k:
            assert any(i.startswith("UBLKCP") for i in body), k


def test_qkv_bias_kernels(per):
    """EPI_ROPE_BIAS = 8 in the 128 x 128 kernel (plain and all-gather builds) and the 128 x 256 kernel, and
    ``bias_grad``."""
    rope_bias = [k for k in per if re.search(r"(gemm_bf16_wgmma|gemm_wide_staged_bf16)ILb[01]ELb[01]ELi8E", k)]
    assert len(rope_bias) == 3, rope_bias
    assert sum("gemm_bf16_wgmma" in k for k in rope_bias) == 2, rope_bias
    bias_grad = [k for k in per if "bias_grad" in k]
    assert bias_grad
    _no_local_memory(per, rope_bias + bias_grad)


def test_embedding_backward_is_the_fixed_order_sum(per):
    """The sort tile and merge, segmented sum and combine for bf16 and fp32 gradients replace the atomic kernels."""
    atomic = {
        "_ZN4b20020embedding_bwd_kernelIiEEvPKT_PK13__nv_bfloat16PS4_mi",
        "_ZN4b20020embedding_bwd_kernelIxEEvPKT_PK13__nv_bfloat16PS4_mi",
        "_ZN4b20024embedding_bwd_f32_kernelIiEEvPKT_PK13__nv_bfloat16Pfmi",
        "_ZN4b20024embedding_bwd_f32_kernelIxEEvPKT_PK13__nv_bfloat16Pfmi",
    }
    assert not atomic & set(per)
    fixed = [k for k in per if re.search(r"embedding_(sort_tile|merge|seg_sum|seg_combine)_kernel", k)]
    assert len(fixed) == 7, fixed
    _no_local_memory(per, fixed)


def test_z_loss_kernels_use_no_float_atomics(per):
    want = ["ce_zloss_grad_inplace_kernel", "loss_partials_reduce_kernel", "router_z_fwd_kernel", "router_z_bwd_kernel"]
    z = [k for k in per if any(w in k for w in want)]
    assert len(z) == 4 and all(sum(w in k for k in z) == 1 for w in want), z
    _no_local_memory(per, z)
    for k in z:
        assert not any(re.search(r"\bRED\.E\.ADD\.F32|\bATOMG?\.E\.ADD\.F32", i) for i in per[k]), k      # no float atomics
