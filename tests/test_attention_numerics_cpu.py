"""CPU tier of the per-row attention check (``tests/attention_reference.py``): the float64 reference is pinned to
autograd, the rounding emulation of the sm_90a kernels passes the per-row bound with headroom in every logit regime
(that emulation is where the tolerances come from), and plausibly broken kernels fail it -- including ones the global
``max|a - b| / max|b|`` check of the first attention tests lets through.
"""
import math

import pytest
import torch

import attention_reference as AR

F64 = torch.float64
# (B, S, H, KVH, hd): a ragged and a tile-aligned S, GQA groups 1, 2 and 7, both head dims, 65 = one past a 64-row tile
SHAPES = [(2, 640, 4, 2, 64), (2, 200, 14, 2, 128), (1, 1000, 8, 1, 64), (2, 65, 4, 1, 128)]


def run(regime, B, S, H, KVH, hd, seed=1, seg=None, rope=None, boost=None, mutation=None):
    qkv, do = AR.make_inputs(regime, B, S, H, KVH, hd, seed, boost=boost)
    sc = hd ** -0.5
    ref = AR.reference(qkv, do, B, S, H, KVH, hd, sc, seg=seg, rope=rope)
    o, lse, dqkv = AR.emulate(qkv, do, B, S, H, KVH, hd, sc, seg=seg, rope=rope, mutation=mutation)
    return AR.kernel_view(o, lse, dqkv, B, S, H, KVH, hd), ref, (o, lse, dqkv)


def assert_headroom(tag, out, ref):
    """The tolerances are 3x the emulation's worst ratio: every emulated ratio stays under half of them."""
    w = AR.worst(out, ref)
    print(f"EMULATED {tag}: " + " ".join(f"{n} {v:.2e} ({v / AR.TOL[n]:.2f} tol)" for n, v in w.items()))
    assert all(torch.isfinite(t).all() for t in out.values()), tag
    bad = {n: v for n, v in w.items() if not v <= AR.TOL[n] / 2}
    assert not bad, (tag, bad)


# ------------------------------------------------------------------------------------------ the reference
@pytest.mark.parametrize("doc", [False, True])
def test_reference_is_autograd_in_float64(doc):
    """o, lse and the gradients of the reference equal autograd through a plain masked softmax, GQA and documents."""
    B, S, H, KVH, hd = 2, 70, 6, 2, 16
    qkv, do = AR.make_inputs("peaked6", B, S, H, KVH, hd, seed=5)
    seg = AR.segments([[9, 10, 40], [0, 33]], S) if doc else None
    sc = hd ** -0.5
    ref = AR.reference(qkv, do, B, S, H, KVH, hd, sc, seg=seg)
    x = qkv.to(F64).view(B, S, H + 2 * KVH, hd).requires_grad_()
    q, k, v = x[:, :, :H], x[:, :, H:H + KVH], x[:, :, H + KVH:]
    k, v = (t.repeat_interleave(H // KVH, dim=2) for t in (k, v))
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) * sc
    pos = torch.arange(S)
    vis = (pos.view(1, S) <= pos.view(S, 1)).expand(B, S, S)
    if doc:
        vis = vis & (pos.view(1, 1, S) >= seg[0].view(B, S, 1).long())
    s = s.masked_fill(~vis.unsqueeze(1), -math.inf)
    lse = torch.logsumexp(s, -1)
    o = torch.einsum("bhqk,bkhd->bqhd", s.softmax(-1), v)
    (g,) = torch.autograd.grad(o, x, do.to(F64).view(B, S, H, hd))
    torch.testing.assert_close(ref["o"], o.detach(), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(ref["lse"], lse.detach(), rtol=1e-12, atol=1e-12)
    for name, got in (("dq", g[:, :, :H]), ("dk", g[:, :, H:H + KVH]), ("dv", g[:, :, H + KVH:])):
        torch.testing.assert_close(ref[name], got, rtol=1e-10, atol=1e-11, msg=name)


def test_reference_inverse_rope():
    """``rope`` applies the inverse rotation of ``torch_kernels.rope_`` to dq / dk."""
    from fms_fsdp_b200.ops import torch_kernels as TK
    B, S, H, KVH, hd = 1, 50, 4, 2, 16
    qkv, do = AR.make_inputs("flat", B, S, H, KVH, hd, seed=2)
    sc = hd ** -0.5
    table = TK.rope_table(S, hd, 1e4)
    plain = AR.reference(qkv, do, B, S, H, KVH, hd, sc)
    roped = AR.reference(qkv, do, B, S, H, KVH, hd, sc, rope=table)
    g = torch.cat([plain["dq"], plain["dk"], plain["dv"]], dim=2).reshape(B * S, -1)
    TK.rope_(g, table.double(), S, H, KVH, hd, inverse=True)
    g = g.view(B, S, H + 2 * KVH, hd)
    torch.testing.assert_close(roped["dq"], g[:, :, :H], rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(roped["dk"], g[:, :, H:H + KVH], rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(roped["dv"], plain["dv"], rtol=0, atol=0)


# -------------------------------------------------------------------------------- the emulated correct kernel
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "B{}_S{}_H{}_KVH{}_hd{}".format(*s))
def test_emulated_kernel_passes_with_headroom(shape):
    for regime in AR.REGIMES:
        out, ref, _ = run(regime, *shape)
        assert_headroom(f"{regime} {shape}", out, ref)


@pytest.mark.parametrize("layout", ["mid_tile", "one_token", "low_after_high"])
def test_emulated_kernel_passes_with_documents(layout):
    B, S, H, KVH, hd = 2, 1000, 4, 2, 64
    seps = AR.doc_layouts(S)[layout]
    seg = AR.segments(seps, S)
    if layout == "low_after_high":   # the first document of each row leans towards u by a logit of ~12
        boost = torch.arange(S) < min(p for r in seps for p in r)
        out, ref, _ = run("boosted", B, S, H, KVH, hd, seg=seg, boost=boost)
        assert_headroom(f"{layout} boosted", out, ref)
    for regime in ("flat", "peaked16"):
        out, ref, _ = run(regime, B, S, H, KVH, hd, seg=seg)
        assert_headroom(f"{layout} {regime}", out, ref)


def test_emulated_kernel_passes_with_inverse_rope():
    from fms_fsdp_b200.ops import torch_kernels as TK
    B, S, H, KVH, hd = 2, 300, 4, 1, 128
    table = TK.rope_table(S, hd, 1e4)
    for regime in ("flat", "peaked16"):
        out, ref, _ = run(regime, B, S, H, KVH, hd, rope=table)
        assert_headroom(f"rope {regime}", out, ref)


# ------------------------------------------------------------------------------------- broken kernels
# (B, S, H, KVH, hd) of the mutation probes: S = 1000 is ragged (a 104-row last tile, 40 rows in the last 64-row tile)
MUT_SHAPE = (2, 1000, 4, 2, 64)


@pytest.fixture(scope="module")
def mutation_verdicts():
    """{mutation: (per-row check fails, global check fails, worst per-row ratios / tolerance)} in the flat regime."""
    B, S, H, KVH, hd = MUT_SHAPE
    out = {}
    for m in AR.MUTATIONS:
        view, ref, raw = run("flat", *MUT_SHAPE, mutation=m)
        w = AR.worst(view, ref)
        out[m] = (bool(AR.failures(view, ref)), not AR.old_check(*raw, ref, B, S, H, KVH, hd),
                  {n: v / AR.TOL[n] for n, v in w.items()})
    print("mutation               per-row  global   worst ratio / tol")
    for m, (new, old, r) in out.items():
        print(f"{m:22s} {'FAILS' if new else 'passes':7s}  {'FAILS' if old else 'passes':7s}  "
              + " ".join(f"{n} {v:.1f}" for n, v in r.items()))
    return out


@pytest.mark.parametrize("mutation", AR.MUTATIONS)
def test_mutation_fails_the_per_row_check(mutation_verdicts, mutation):
    new_fails, _, ratios = mutation_verdicts[mutation]
    assert new_fails, (mutation, ratios)


def test_per_row_check_catches_what_the_global_check_misses(mutation_verdicts):
    """The point of the per-row bound: these broken kernels pass max|a - b| / max|b| < 1e-2 / 1e-4 / 1.5e-2."""
    missed = sorted(m for m, (new, old, _) in mutation_verdicts.items() if new and not old)
    assert set(missed) >= {"lse_ln2_4_digits", "delta_next_row_tail", "dv_tail_x1.05", "dq_short_last_tile"}, missed


def test_unmutated_emulation_passes_both_checks():
    B, S, H, KVH, hd = MUT_SHAPE
    view, ref, raw = run("flat", *MUT_SHAPE)
    assert not AR.failures(view, ref)
    assert AR.old_check(*raw, ref, B, S, H, KVH, hd)
