"""CPU tier of the Mamba2-hybrid node check (``tests/mamba_node_reference.py``): the float64 references are pinned to the
project's modules run in float64 on the ATen path, the chunked SSD form to the recurrence, the rounding emulation of
the sm_90a kernels passes every tolerance with at least 2x headroom, plausibly broken code fails the check that
targets it, and the node code (``models/mamba.py`` on bf16 CPU parameters) delivers every weight gradient into all
three destinations (returned, an fp32 slot, a bf16 slot) with at most one rounding.
"""
import pytest
import torch

import llama_node_reference as LR
import mamba_node_reference as MR
from fms_fsdp_b200.models.mamba import MHA, Block, GatedMLP, Mamba1, Mamba2, MambaConfig, MambaLMHeadModel

F64, F32, BF16 = torch.float64, torch.float32, torch.bfloat16
B, S = 2, 256
M = B * S


def build(kind, dtype=BF16, regime="init", seed=0, mlp=True):
    """A Block (``kind`` Mamba2 / Mamba1 / MHA, with a GatedMLP when ``mlp``) at CPU size, parameters reset."""
    torch.manual_seed(seed)
    D = 128 if kind != "MHA" else 256
    if kind == "Mamba2":
        mixer = Mamba2(D, d_state=32, headdim=32, ngroups=2, dtype=dtype)
    elif kind == "Mamba1":
        mixer = Mamba1(D, d_state=16, dtype=dtype)
    else:
        mixer = MHA(D, 4, 2, 64, 32, dtype=dtype)
    blk = Block(D, mixer, GatedMLP(D, 192, dtype=dtype) if mlp else None, dtype=dtype)
    for m in blk.modules():
        if m is not blk and hasattr(m, "reset_parameters") and not isinstance(m, (Mamba2, Mamba1, MHA, GatedMLP)):
            m.reset_parameters()
    mixer.reset_parameters()
    if mlp:
        blk.mlp.reset_parameters()
    with torch.no_grad():                        # gains away from 1, so a dropped or swapped gain shows
        for n, p in blk.named_parameters():
            if n.endswith("norm.weight") or n.endswith("norm2.weight"):
                p.copy_(1 + 0.3 * torch.randn(p.shape, generator=torch.Generator().manual_seed(seed + 3)))
    if kind != "MHA":
        MR.set_regime(mixer, regime, seed)
    return blk


def inputs(D, seed=0):
    g = torch.Generator().manual_seed(seed + 11)
    return {n: torch.randn(M, D, generator=g).to(BF16) for n in ("hidden", "res", "dh", "dr")}


def params_of(mod, prefix=""):
    return {prefix + n: p.detach() for n, p in mod.named_parameters()}


def mixer_run(blk, em, mut=None, chunk=None, seed=0):
    mix = blk.mixer
    cfg = MR.mixer_cfg(mix)
    t = inputs(blk.norm.weight.shape[0], seed)
    fn = {"Mamba2": lambda p, a: MR.mamba2(p, a["u"], S, cfg, em, mut, chunk),
          "Mamba1": lambda p, a: MR.mamba1(p, a["u"], S, cfg, em, mut),
          "MHA": lambda p, a: MR.mha(p, a["u"], S, cfg, em, mut)}[cfg["mixer"]]
    return MR.evaluate(fn, params_of(mix), {"u": t["hidden"]}, (t["dh"],), M, em), params_of(mix)


def block_run(blk, em, mut=None, chunk=None, seed=0):
    cfg = MR.mixer_cfg(blk.mixer)
    t = inputs(blk.norm.weight.shape[0], seed)
    return MR.evaluate(lambda p, a: MR.block(p, a["hidden"], a["res"], S, cfg, em, mut, chunk), params_of(blk),
                       {"hidden": t["hidden"], "res": t["res"].float()}, (t["dh"], t["dr"].float()), M, em), params_of(blk)


def mlp_run(blk, em, mut=None, seed=0):
    t = inputs(blk.norm.weight.shape[0], seed)
    return MR.evaluate(lambda p, a: MR.gated_mlp(p, a["x"], em, mut), params_of(blk.mlp), {"x": t["hidden"]},
                       (t["dh"],), M, em), params_of(blk.mlp)


def ends_model(tied, seed=0):
    torch.manual_seed(seed)
    cfg = MambaConfig(d_model=128, n_layer=1, vocab_size=1000, ssm_cfg={"layer": "Mamba2"}, tie_embeddings=tied)
    model = MambaLMHeadModel(cfg, dtype=BF16)
    model.reset_parameters()
    with torch.no_grad():
        model.backbone.norm_f.weight.copy_(1 + 0.3 * torch.randn(128))
        # the logits at production scale, where their bf16 rounding is what it is there.  A tied head scores each
        # token against its own embedding row: that logit is about D std, 51 for mamba_2.8b's 2560 x 0.02 (a bf16
        # logit is 0.25 coarse there); std 0.4 gives it at D 128.  An untied head's logits have a std of about
        # sqrt(D) std, 1.3 for mamba_9.8b's 4096 x 0.02; std 0.11 gives it at D 128
        if tied:
            model.backbone.embedding.weight.normal_(std=0.4)
        else:
            model.lm_head.weight.normal_(std=0.11)
    g = torch.Generator().manual_seed(seed + 5)
    tokens = torch.randint(0, 1000, (B, S), generator=g)
    labels = torch.randint(0, 1000, (B, S), generator=g)
    labels[torch.rand(B, S, generator=g) < 0.1] = -100
    return model, tokens, labels


def ends_run(tied, em, seed=0):
    model, tokens, labels = ends_model(tied, seed)
    names = ["backbone.embedding.weight", "backbone.norm_f.weight"] + ([] if tied else ["lm_head.weight"])
    prm = {n: p.detach() for n, p in model.named_parameters() if n in names}
    if tied:
        prm["lm_head.weight"] = prm["backbone.embedding.weight"]
    stats = {}
    out = MR.evaluate(lambda p, a: MR.ends(p, a["tokens"].reshape(-1), a["labels"].reshape(-1), False, em, stats=stats),
                      prm, {"tokens": tokens, "labels": labels}, (torch.ones((), dtype=F64),), M, em)
    if tied:
        del prm["lm_head.weight"]
    return MR.head_scales(out, stats, tied), prm


def end_ratios(out, ref, prm, tied):
    r = {"end_loss": abs(float(out["out"][0]) - float(ref["out"][0])) / abs(float(ref["out"][0]))}
    r["end_tied_dw" if tied else "end_dw"] = max(MR.ratio(out[n], ref[n], ref.get(n + "_scale")) for n in prm
                      if n.endswith("embedding.weight") or n.startswith("lm_head"))
    r["end_dv"] = LR.vratio(out["backbone.norm_f.weight"], ref["backbone.norm_f.weight"],
                            ref["backbone.norm_f.weight_abs"])
    return r


PREFIX = {"Mamba2": "m2", "Mamba1": "m1", "MHA": "mha"}


# ------------------------------------------------------------------------------ the reference is the model in float64
@pytest.mark.parametrize("kind", ["Mamba2", "Mamba1", "MHA"])
def test_block_reference_matches_the_modules_in_float64(kind):
    """The formulas against the project's Block run on float64 CPU tensors (the ATen path, which keeps some fp32
    arithmetic: hence 1e-5, far below any bf16 effect)."""
    blk = build(kind, F64)
    ref, prm = block_run(blk, False, chunk=None)
    t = inputs(blk.norm.weight.shape[0])
    hidden = t["hidden"].to(F64).view(B, S, -1).requires_grad_()
    res = t["res"].to(F64).view(B, S, -1).requires_grad_()
    h, r = blk(hidden, res)
    leaves = [hidden, res] + list(blk.parameters())
    gr = torch.autograd.grad((h, r), leaves, (t["dh"].to(F64).view(B, S, -1), t["dr"].to(F64).view(B, S, -1)))
    assert MR.ratio(h.detach().reshape(M, -1), ref["out"][0]) < 1e-5
    assert MR.ratio(r.detach().reshape(M, -1), ref["out"][1]) < 1e-5
    assert MR.ratio(gr[0].reshape(M, -1), ref["dhidden"]) < 1e-5
    assert MR.ratio(gr[1].reshape(M, -1), ref["dres"]) < 1e-5
    for (n, p), g in zip(blk.named_parameters(), gr[2:]):
        if MR.is_vector(n, p):
            assert LR.vratio(g, ref[n], ref[n + "_abs"]) < 1e-5, n
        else:
            assert MR.ratio(g, ref[n]) < 1e-5, n


@pytest.mark.parametrize("tied", [True, False])
def test_ends_reference_matches_the_model_in_float64(tied):
    model, tokens, labels = ends_model(tied)
    model = model.to(F64)
    ref, prm = ends_run(tied, False)
    loss = model.engine_head(*model.engine_embed(tokens), labels=labels.reshape(-1))
    ps = [p for n, p in model.named_parameters() if n in prm]
    gr = torch.autograd.grad(loss, ps)
    assert abs(float(loss) - float(ref["out"][0])) < 1e-7 * abs(float(loss))
    for n, g in zip([n for n, _ in model.named_parameters() if n in prm], gr):
        if g.dim() == 1:
            assert LR.vratio(g, ref[n], ref[n + "_abs"]) < 1e-5, n
        else:
            assert MR.ratio(g, ref[n], ref.get(n + "_scale")) < 1e-5, n


@pytest.mark.parametrize("S_, chunk", [(256, 128), (256, 96), (200, 64)])
def test_chunked_ssd_is_the_recurrence(S_, chunk):
    """The chunked form (the GPU tier's reference) equals the recurrence in value and in every gradient, for chunks
    that do and do not divide S."""
    g = torch.Generator().manual_seed(3)
    Mr, H, P, G, N = 2 * S_, 8, 16, 2, 16
    x, dt, Bm, Cm = (torch.randn(*s, generator=g, dtype=F64) for s in ((Mr, H, P), (Mr, H), (Mr, G, N), (Mr, G, N)))
    A_log, D, bias = (torch.rand(Mr, H, generator=g, dtype=F64) for _ in range(3))
    leaves = [t.requires_grad_() for t in (x, dt, Bm, Cm, A_log, D, bias)]
    dy = torch.randn(Mr, H, P, generator=g, dtype=F64)
    outs = []
    for fn in (lambda: MR.ssd_seq(x, dt, -torch.exp(A_log), Bm, Cm, D, bias, S_),
               lambda: MR.ssd_chunked(x, dt, -torch.exp(A_log), Bm, Cm, D, bias, S_, chunk)):
        y = fn()
        outs.append((y.detach(),) + torch.autograd.grad(y, leaves, dy))
    for a, b in zip(*outs):
        # per token, against the token's max plus 1e-6 of the tensor's: some tokens' exact gradients are 0 (A_log's at
        # a sequence start, where the state is 0), which one form reaches only to rounding
        a, b = a.reshape(a.shape[0], -1), b.reshape(b.shape[0], -1)
        assert MR.ratio(a, b, b.abs() + 1e-6 * b.abs().max()) < 1e-8


# ---------------------------------------------------------------------------------- the emulation has headroom
def emulated(kind, regime):
    """Worst emulated ratio per tolerance key for one mixer kind and regime: the mixer, the block with an MLP (the
    Mamba2 block also without), and (Mamba2) the MLP and the ends."""
    blk = build(kind, regime=regime)
    chunk = 128 if kind == "Mamba2" else None
    p = PREFIX[kind]
    r = MR.ratios(p, mixer_run(blk, True, chunk=chunk)[0], *mixer_run(blk, False), M)
    r.update(MR.ratios("blk", block_run(blk, True, chunk=chunk)[0], *block_run(blk, False), M))
    if kind == "Mamba2":
        r.update(MR.ratios("mlp", mlp_run(blk, True)[0], *mlp_run(blk, False), M))
        for tied in (True, False):
            e, prm = ends_run(tied, True)
            for k, v in end_ratios(e, ends_run(tied, False)[0], prm, tied).items():
                r[k] = max(r.get(k, 0.0), v)
    return r


def _headroom(r):
    bad = {k: (v, MR.TOL[k]) for k, v in r.items() if not v <= MR.TOL[k] / 2}
    assert not bad, bad


@pytest.mark.parametrize("regime", ["init", "slow", "trained"])
@pytest.mark.parametrize("kind", ["Mamba2", "Mamba1", "MHA"])
def test_emulated_nodes_pass_with_headroom(kind, regime):
    if kind == "MHA" and regime != "init":
        pytest.skip("the regimes set SSM parameters")
    _headroom(emulated(kind, regime))


# ---------------------------------------------------------------------------------- broken variants fail
MIXER_TARGET = {"norm_all_groups": "Mamba2", "head_group_map": "Mamba2"}


@pytest.mark.parametrize("mut", MR.MIXER_MUTATIONS)
def test_broken_mamba2_mixer_fails(mut):
    blk = build("Mamba2", regime="trained" if mut in ("conv_no_restart", "decay_off_by_one") else "slow")
    ref, prm = mixer_run(blk, False)
    r = MR.ratios("m2", mixer_run(blk, True, mut=mut, chunk=128)[0], ref, prm, M)
    assert any(not v <= MR.TOL[k] for k, v in r.items()), r


@pytest.mark.parametrize("mut", ["conv_no_restart", "conv_taps_reversed", "negexp_sign"])
def test_broken_mamba1_mixer_fails(mut):
    blk = build("Mamba1", regime="trained" if mut == "conv_no_restart" else "slow")
    ref, prm = mixer_run(blk, False)
    r = MR.ratios("m1", mixer_run(blk, True, mut=mut)[0], ref, prm, M)
    assert any(not v <= MR.TOL[k] for k, v in r.items()), r


@pytest.mark.parametrize("mut", MR.MHA_MUTATIONS)
def test_broken_rotary_fails(mut):
    blk = build("MHA")
    ref, prm = mixer_run(blk, False)
    r = MR.ratios("mha", mixer_run(blk, True, mut=mut)[0], ref, prm, M)
    key = "mha_dx" if mut == "rope_no_inverse_grad" else "mha_y"
    assert r[key] > MR.TOL[key], r


def test_gate_and_value_swapped_fails():
    blk = build("Mamba2")
    ref, prm = mlp_run(blk, False)
    r = MR.ratios("mlp", mlp_run(blk, True, mut="gate_value_swapped")[0], ref, prm, M)
    assert r["mlp_y"] > MR.TOL["mlp_y"], r


def test_dropped_residual_gradient_fails():
    blk = build("Mamba2")
    ref, prm = block_run(blk, False)
    r = MR.ratios("blk", block_run(blk, True, mut="residual_grad_dropped", chunk=128)[0], ref, prm, M)
    assert r["blk_dx"] > MR.TOL["blk_dx"], r


# --------------------------------------------------------------------- the node code delivers its gradients
def _node(kind, seed=0):
    """The real Block (bf16 parameters, CPU): (call, acts, weights, dos)."""
    blk = build(kind, regime="trained", seed=seed)
    t = inputs(blk.norm.weight.shape[0], seed)
    hidden = t["hidden"].view(B, S, -1).requires_grad_()
    res = t["res"].float().view(B, S, -1).requires_grad_()
    g = torch.Generator().manual_seed(seed + 21)
    dos = [(t["dh"].view(B, S, -1), t["dr"].float().view(B, S, -1)),
           (torch.randn(B, S, hidden.shape[-1], generator=g).to(BF16), torch.randn(B, S, hidden.shape[-1], generator=g))]
    return (lambda: blk(hidden, res)), {"hidden": hidden, "res": res}, dict(blk.named_parameters()), dos


@pytest.mark.parametrize("kind", ["Mamba2", "Mamba1"])
def test_node_code_delivers_every_gradient_to_every_destination(kind):
    call, acts, W, dos = _node(kind)
    _, _, ret = LR.run_node(call, acts, W, dos[:1], "returned")
    _, _, s32 = LR.run_node(call, acts, W, dos, "fp32")
    _, _, only2 = LR.run_node(call, acts, W, dos[1:], "fp32")
    _, _, s16 = LR.run_node(call, acts, W, dos, "bf16")
    for n, p in W.items():
        # returned: the fp32 value rounded once to the parameter's dtype; the same value an fp32 slot stores
        assert LR.one_rounding(ret[0][n], s32[0][n]) <= 1.0, n
        # an fp32 slot accumulates in fp32
        assert torch.equal(s32[1][n], s32[0][n] + only2[0][n]), n
        if MR.is_vector(n, p):
            # a bf16 slot: the stored value, then the old slot plus the fp32 contribution, each rounded once
            assert LR.one_rounding(s16[0][n], s32[0][n]) <= 1.0, n
            assert LR.one_rounding(s16[1][n], s16[0][n].to(F64) + only2[0][n].to(F64)) <= 1.0, n
    # the conv taps reach an fp32 slot in fp32, as the conv bias from the same kernel call does
    for n in ("mixer.conv1d.weight", "mixer.conv1d.bias"):
        v = s32[0][n]
        assert not torch.equal(v, v.to(BF16).float()), f"{n}: the fp32 slot holds bf16 values"
