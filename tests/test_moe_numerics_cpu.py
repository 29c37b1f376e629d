"""CPU tier of the per-row mixture-of-experts check (``tests/moe_reference.py``): the float64 node reference is pinned
to autograd, the rounding emulation of the sm_90a kernels passes every tolerance with at least 2x headroom (init-scale
and peaked routers, skewed routing, crafted segment counts), and plausibly broken kernels fail it -- most of which the
older checks of ``tests/test_moe_gpu.py`` let through.
"""
import pytest
import torch

import moe_reference as MR
from fms_fsdp_b200.ops import torch_kernels as TK

F64 = torch.float64
# the crafted plan: an empty first and last expert, counts 1, 63 / 64 / 65 and 127 / 128 / 129 around the 64-row
# k-block and the 128-row tile, a run of two empty experts, and one expert owning 8448 = 66 x 128 rows (a k-range of
# 132 k-blocks ending exactly where the next expert's segment starts)
CRAFTED = [0, 1, 63, 64, 65, 127, 128, 129, 0, 0, 256, 8448, 2560, 2560, 2495, 0]
CRAFTED_T, CRAFTED_K = 8448, 2


def plan_of(ids, E):
    return TK.moe_plan(ids, torch.zeros(ids.shape[0], E))[0]


def stage_ratios(h, wr, w1, w2, res, dy, ids, norm, mutation=None, aux_coef=0.01):
    """Run the emulated kernels stage by stage and judge each output against the float64 reference of the same stage
    on the same (emulated) inputs, as the GPU tier judges the kernels.  Returns {tolerance key: worst ratio}."""
    T, D = h.shape
    E, k = wr.shape[0], ids.shape[1]
    plan = plan_of(ids, E)
    w = {}
    put = lambda key, v: w.__setitem__(key, max(w.get(key, 0.0), v))
    H, WR = h.to(F64), wr.to(F64)
    logits = MR.mm(H, WR.t(), em=True)
    put("fp32", MR.ratio(logits, MR.mm(H, WR.t())))
    probs, wts, _ = MR.route(logits, ids, norm, em=True)
    rp, rw, _ = MR.route(logits, ids, norm)
    put("probs", max(MR.ratio(probs, rp), MR.ratio(wts, rw)))
    put("scalar", MR.scalar_ratio(f32s(MR.aux_stat(probs, ids, E)), MR.aux_stat(rp, ids, E)))
    xp = MR.permute(H, plan, T, k, E)
    hp, sp = MR.up(xp, w1, plan, T, k, em=True, mutation=mutation)
    rh, _ = MR.up(xp, w1, plan, T, k)
    put("bf16", max(MR.ratio(hp, rh), MR.ratio(sp, MR._swiglu(hp, False))))
    yp = MR.down(sp, w2, plan, T, k, em=True)
    put("bf16", MR.ratio(yp, MR.down(sp, w2, plan, T, k)))
    put("bf16", MR.ratio(MR.combine(yp, plan, wts, res, T, k, E, em=True), MR.combine(yp, plan, wts, res, T, k, E)))
    dyp, dw = MR.combine_bwd(dy, yp, plan, wts, T, k, E, em=True)
    rdyp, rdw = MR.combine_bwd(dy, yp, plan, wts, T, k, E)
    put("bf16", MR.ratio(dyp, rdyp))
    put("dw", MR.ratio(dw, rdw))
    dhp = MR.down_bwd(dyp, w2, hp, plan, T, k, em=True)
    put("bf16", MR.ratio(dhp, MR.down_bwd(dyp, w2, hp, plan, T, k)))
    dxp = MR.up_dgrad(dhp, w1, plan, T, k, em=True)
    put("bf16", MR.ratio(dxp, MR.up_dgrad(dhp, w1, plan, T, k)))
    put("bf16", MR.ratio(MR.permute_bwd(dxp, plan, T, k, E, em=True), MR.permute_bwd(dxp, plan, T, k, E)))
    wm = mutation if mutation in ("wgrad_bf16_store", "kend_floor_plus1", "kend_floor") else None
    am = mutation if mutation == "wgrad_bf16_accum" else None
    for e, seg in enumerate(MR.segments(plan, T, k, E)):
        for a, b in ((dhp, xp), (dyp, sp)):
            ref = MR.wgrad_expert(a, b, seg)
            put("fp32", MR.ratio(MR.wgrad_expert(a, b, seg, em=True, mutation=wm), ref))
            base = torch.randn(ref.shape, generator=torch.Generator().manual_seed(e)).to(torch.float32)
            acc = MR.wgrad_expert(a, b, seg, em=True, base=base, mutation=am)
            put("fp32", MR.ratio(acc, ref + base.to(F64)))
    scale = aux_coef * E / (T * T)
    rm = mutation if mutation in ("aux_dropped", "aux_negated") else None
    for part, dwp in (("dw", dw), ("aux", torch.zeros_like(dw)), ("both", dw)):
        put("dl", MR.ratio(MR.route_bwd(probs, ids, dwp, norm, scale, part, em=True, mutation=rm),
                           MR.route_bwd(probs, ids, dwp, norm, scale, part),
                           MR.route_bwd_scale(probs, ids, dwp, norm, scale, part)))
    return w


def f32s(x):
    return float(torch.tensor(x, dtype=torch.float32))


def route_ids(h, wr, k):
    """The top-k of the emulated fp32 logits (what the kernels would pick)."""
    lg = MR.mm(h.to(F64), wr.to(F64).t(), em=True)
    return torch.sort(lg, dim=-1, descending=True, stable=True).indices[:, :k].to(torch.int32)


def assert_headroom(tag, w):
    """Every tolerance is 3x the emulation's worst ratio: every emulated ratio stays under half of it."""
    print(f"EMULATED {tag}: " + " ".join(f"{n} {v:.2e} ({v / MR.TOL[n]:.2f} tol)" for n, v in w.items()))
    bad = {n: v for n, v in w.items() if not v <= MR.TOL[n] / 2}
    assert not bad, (tag, bad)


# ------------------------------------------------------------------------------------------ the reference
@pytest.mark.parametrize("norm", [False, True])
def test_node_reference_is_autograd_in_float64(norm):
    """y, dh, d(router), dw1, dw2, aux and z of the float64 node (permuted buffer, plan, hand-written backward) equal
    float64 autograd through a plain per-expert loop, with the load-balancing and z-loss terms on."""
    T, D, E, F, k = 300, 64, 8, 32, 2
    h, wr, w1, w2, res, dy = MR.node_inputs(T, D, E, F, "peaked", seed=3)
    ids = route_ids(h, wr, k)
    ids[:5] = torch.tensor([E - 1, 0], dtype=torch.int32)      # expert order inside a token does not matter
    dws = {}
    ref = MR.node(h, wr, w1, w2, res, dy, ids, norm, 0.05, 0.01, on_expert=lambda e, a, b: dws.__setitem__(e, (a, b)))
    ag = MR.node_autograd(h, wr, w1, w2, res, dy, ids, norm, 0.05, 0.01)
    for n in ("y", "dh", "dwr"):
        torch.testing.assert_close(ref[n], ag[n], rtol=1e-10, atol=1e-12, msg=n)
    torch.testing.assert_close(torch.stack([dws[e][0] for e in range(E)]), ag["dw1"], rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(torch.stack([dws[e][1] for e in range(E)]), ag["dw2"], rtol=1e-10, atol=1e-12)
    assert ref["aux"] == pytest.approx(ag["aux"], rel=1e-12) and ref["z"] == pytest.approx(ag["z"], rel=1e-12)


def test_route_bwd_parts_add_up_and_aux_part_is_the_balancing_gradient():
    """The aux part alone is the gradient of aux_scale * sum_e count_e sum_t p_te through the softmax."""
    T, E, k = 50, 16, 4
    lg = torch.randn(T, E, dtype=F64, requires_grad=True)
    ids = torch.sort(lg.detach(), -1, descending=True).indices[:, :k]
    dw = torch.randn(T, k, dtype=F64)
    p = torch.softmax(lg, -1)
    count = torch.bincount(ids.reshape(-1), minlength=E).to(F64)
    (g,) = torch.autograd.grad((count * p.sum(0)).sum() * 0.3, lg)
    pd = p.detach()
    torch.testing.assert_close(MR.route_bwd(pd, ids, dw, True, 0.3, "aux"), g, rtol=1e-12, atol=1e-14)
    both = MR.route_bwd(pd, ids, dw, True, 0.3)
    torch.testing.assert_close(both, MR.route_bwd(pd, ids, dw, True, 0.3, "dw") + g, rtol=1e-12, atol=1e-14)


def test_crafted_ids_have_the_asked_counts():
    ids = MR.crafted_ids(CRAFTED, CRAFTED_T, CRAFTED_K)
    assert torch.bincount(ids.reshape(-1).long(), minlength=len(CRAFTED)).tolist() == CRAFTED
    assert all(len(set(r)) == CRAFTED_K for r in ids.tolist())


# -------------------------------------------------------------------------------- the emulated correct kernels
NODE_SHAPE = (256, 2048, 128, 128, 8)         # T, D, E, F, k: the routing and K of Qwen3-30B-A3B, few tokens


@pytest.mark.parametrize("regime,norm", [("init", False), ("peaked", True), ("skewed", True), ("peaked", False)])
def test_emulated_node_passes_with_headroom(regime, norm):
    T, D, E, F, k = NODE_SHAPE
    h, wr, w1, w2, res, dy = MR.node_inputs(T, D, E, F, regime, seed=1)
    ids = route_ids(h, wr, k)
    dws = {}
    got = MR.node(h, wr, w1, w2, res, dy, ids, norm, 0.02, 0.001, em=True,
                  on_expert=lambda e, a, b: dws.__setitem__(e, (a, b)))
    ref = MR.node(h, wr, w1, w2, res, dy, ids, norm, 0.02, 0.001,
                  on_expert=lambda e, a, b: dws.__setitem__(e, dws[e] + (a, b)))
    w = {n: MR.ratio(got[n], ref[n]) for n in ("y", "dh", "dwr")}
    w["dw1"] = max(MR.ratio(d[0], d[2]) for d in dws.values())
    w["dw2"] = max(MR.ratio(d[1], d[3]) for d in dws.values())
    w["scalar"] = max(MR.scalar_ratio(f32s(got[n]), ref[n]) for n in ("aux", "z"))
    assert_headroom(f"node {regime} norm={norm}", w)
    assert_headroom(f"stages {regime} norm={norm}", stage_ratios(h, wr, w1, w2, res, dy, ids, norm))


def test_emulated_stages_pass_with_headroom_on_crafted_segments():
    T, k, E, D, F = CRAFTED_T, CRAFTED_K, len(CRAFTED), 64, 64
    h, wr, w1, w2, res, dy = MR.node_inputs(T, D, E, F, "init", seed=2)
    ids = MR.crafted_ids(CRAFTED, T, k)
    assert_headroom("stages crafted", stage_ratios(h, wr, w1, w2, res, dy, ids, True))


# ------------------------------------------------------------------------------------- broken kernels
MUTATIONS = ("wgrad_bf16_store", "wgrad_bf16_accum", "aux_dropped", "aux_negated", "kend_floor_plus1", "kend_floor",
             "tile_first_shared_start")


def old_checks_pass(mutation):
    """Would the broken kernel pass the matching check of tests/test_moe_gpu.py?  Emulated at that test's own shapes
    and tolerances (D 256, F 192, the seeds of its routing cases)."""
    if mutation in ("aux_dropped", "aux_negated"):
        # test_permute_combine_and_route_bwd_match_oracle: assert_close(rtol=2e-2, atol=1e-5) on every CASES entry
        cases = [("uniform", 8192, 128, 8), ("uniform", 200, 8, 2), ("same", 1000, 128, 8), ("empty", 333, 64, 4),
                 ("ties", 136, 16, 2), ("uniform", 1, 8, 2)]
        for kind, T, E, k in cases:
            ids, wts, probs, dwr = _old_routing(kind, T, E, k)
            scale = 0.01 * E / (T * T)
            good = MR.route_bwd(probs, ids, dwr, True, scale)
            bad = MR.route_bwd(probs, ids, dwr, True, scale, mutation=mutation)
            if not torch.allclose(bad, good, rtol=2e-2, atol=1e-5):
                return False
        return True
    # test_grouped_gemms_match_fp32_oracle: rtol = atol = 2e-2 on stored and 2e-2 / 4e-2 on accumulated wgrads and
    # on the m-grouped outputs, D 256, F 192
    for kind, T, E, k in [("uniform", 8192, 128, 8), ("uniform", 200, 8, 2), ("same", 1000, 128, 8),
                          ("empty", 333, 64, 4), ("ties", 136, 16, 2), ("uniform", 4096, 128, 8)]:
        ids, wts, probs, _ = _old_routing(kind, T, E, k)
        plan = plan_of(ids, E)
        g = torch.Generator().manual_seed(5)
        D, F = 256, 192
        x = torch.randn(T, D, generator=g).bfloat16()
        w1 = (torch.randn(E, 2 * F, D, generator=g) * 0.1).bfloat16()
        xp = MR.permute(x, plan, T, k, E)
        if mutation == "tile_first_shared_start":
            bad = MR.up(xp, w1, plan, T, k, mutation=mutation)[0]
            if not torch.allclose(bad, MR.up(xp, w1, plan, T, k)[0], rtol=2e-2, atol=2e-2):
                return False
            continue
        a = torch.randn(xp.shape[0], D, generator=g).bfloat16().to(F64) * MR.routed_rows(plan, T, k, E)[:, None]
        for e, seg in enumerate(MR.segments(plan, T, k, E)):
            ref = MR.wgrad_expert(a, xp, seg)
            if mutation == "wgrad_bf16_accum":
                bad = MR.wgrad_expert(a, xp, seg, base=ref.float(), mutation=mutation)
                ok = torch.allclose(bad, 2 * ref, rtol=2e-2, atol=4e-2)
            else:
                ok = torch.allclose(MR.wgrad_expert(a, xp, seg, mutation=mutation), ref, rtol=2e-2, atol=2e-2)
            if not ok:
                return False
    return True


def _old_routing(kind, T, E, k):
    """The routing of tests/test_moe_gpu.py's cases (its _logits and seeds)."""
    gen = torch.Generator().manual_seed(T + E)
    lg = torch.randn(T, E, generator=gen)
    if kind == "same":
        lg[:, E - k:] += 50.0
    elif kind == "empty":
        lg[:, 2 * k:] -= 50.0
    elif kind == "ties":
        lg = torch.zeros(T, E)
    ids, wts, probs = TK.moe_route(lg, k, True)
    return ids, wts, probs, torch.randn(T, k, generator=gen)


@pytest.fixture(scope="module")
def verdicts():
    """{mutation: (fails the new per-row check, worst ratio / tolerance per key, passes the old check)}, on the
    crafted segments (every edge the mutations touch) with an init-scale router."""
    T, k, E, D, F = CRAFTED_T, CRAFTED_K, len(CRAFTED), 64, 64
    h, wr, w1, w2, res, dy = MR.node_inputs(T, D, E, F, "init", seed=2)
    ids = MR.crafted_ids(CRAFTED, T, k)
    out = {}
    for m in MUTATIONS:
        w = stage_ratios(h, wr, w1, w2, res, dy, ids, True, mutation=m)
        r = {n: v / MR.TOL[n] for n, v in w.items()}
        out[m] = (any(v > 1 for v in r.values()), r, old_checks_pass(m))
    print("mutation                  per-row  old check  worst ratio / tol")
    for m, (new, r, old) in out.items():
        worst = max(r, key=r.get)
        print(f"{m:25s} {'FAILS' if new else 'passes':7s}  {'passes' if old else 'FAILS':9s}  {worst} {r[worst]:.3g}")
    return out


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_mutation_fails_the_per_row_check(verdicts, mutation):
    new_fails, ratios, _ = verdicts[mutation]
    assert new_fails, (mutation, ratios)


def test_per_row_check_catches_what_the_old_checks_miss(verdicts):
    """A wgrad rounded through bf16 passes test_moe_gpu.py's wgrad checks.  (A dropped or negated load-balancing term
    fails that file's route-backward check only on its degenerate "empty" and "ties" routings at T <= 333.)"""
    missed = sorted(m for m, (new, _, old) in verdicts.items() if new and old)
    print("pass the old checks:", missed)
    assert set(missed) >= {"wgrad_bf16_store", "wgrad_bf16_accum"}, missed
