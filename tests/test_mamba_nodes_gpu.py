"""GPU tier of the Mamba2-hybrid node check (``tests/mamba_node_reference.py``).

The real modules of ``models/mamba.py`` (``Mamba2``, ``Mamba1``, ``MHA``, ``GatedMLP``, ``Block`` and the model's ends)
run on the fused kernels with bf16 parameters at mamba_2.8b and mamba_9.8b shapes, with every weight gradient delivered
three ways (returned, an fp32 slot stored then accumulated, a bf16 slot stored then accumulated).  Outputs and
activation gradients are judged per token, weight matrices per output row, vector gradients element by element
against the sum of |per-token contributions|.  Each case prints its worst ratios as fractions of the tolerance
("MEASURE ... x tol"); the tolerances come from the CPU rounding emulation (tests/test_mamba_nodes_cpu.py).  The ATen
path's ratios are printed, not asserted.
"""
import subprocess
import time

import pytest
import torch

import llama_node_reference as LR
import mamba_node_reference as MR
from fms_fsdp_b200 import ops
from fms_fsdp_b200.models.mamba import MHA, Block, GatedMLP, Mamba1, Mamba2, MambaConfig, MambaLMHeadModel
from fms_fsdp_b200.ops import functional as FN

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64, F32, BF16 = torch.float64, torch.float32, torch.bfloat16


@pytest.fixture(scope="module")
def CK():
    from fms_fsdp_b200.ops import cuda_kernels as CK
    assert CK._C.__file__.endswith("_C.so")
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        card = torch.cuda.get_device_name()
    print(f"\nMEASURE card: {card}")
    t0 = time.time()
    yield CK
    print(f"\nMEASURE file wall time: {time.time() - t0:.1f} s")


class Judge:
    """Worst fraction of tolerance per quantity; ``done`` prints them with the run time and the allocator peak."""

    def __init__(self, tag):
        self.tag, self.w, self.t0 = tag, {}, time.time()
        torch.cuda.reset_peak_memory_stats()

    def __call__(self, name, frac):
        self.w[name] = max(self.w.get(name, 0.0), frac)

    def done(self, enforce=True):
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() / 2 ** 30
        print(f"MEASURE {self.tag}: " + " ".join(f"{n} {v:.3f}" for n, v in self.w.items())
              + f" x tol; {time.time() - self.t0:.1f} s, peak {peak:.1f} GiB")
        bad = {n: v for n, v in self.w.items() if not v <= 1.0}
        assert not (enforce and bad), (self.tag, bad)


def frac_rows(out, ref, key, rounded=False, scale=None):
    """Per-row ratio (rows: tokens of an activation, output rows of a weight; against the row's max of ``scale`` when
    given) as a fraction of TOL[key], plus one bf16 rounding of the row's max when ``rounded``."""
    n = ref.shape[-1]
    return MR.ratio(out.reshape(-1, n), ref.reshape(-1, n), scale) / (MR.TOL[key] + (LR.UBF if rounded else 0.0))


def frac_vec(out, ref, absum, key, rounded=()):
    bound = MR.TOL[key] * absum + sum(LR.UBF * r.to(F64).abs() for r in rounded)
    return LR.GR.ratio(out.reshape(-1), ref.to(F64).reshape(-1), bound.reshape(-1))


def deliveries(J, CK, tag, call, acts, weights, dos, check, fallbacks_per_call=0):
    """Every delivery on the fused kernels, then the ATen path (printed only).  Each fused forward + backward must add
    exactly ``fallbacks_per_call`` counted ATen fallbacks."""
    f0 = CK.fallback_count()
    ops.set_kernel_path("fused")
    try:
        out, dacts, after = LR.run_node(call, acts, weights, dos[:1], "returned")
        check(J, "returned", out, dacts, after[0], "returned", 1)
        _, dacts, after32 = LR.run_node(call, acts, weights, dos, "fp32")
        check(J, "fp32_store", None, None, after32[0], "fp32", 1)
        check(J, "fp32_accum", None, dacts, after32[1], "fp32", 2)
        _, _, only2 = LR.run_node(call, acts, weights, dos[1:], "fp32")
        _, _, again2 = LR.run_node(call, acts, weights, dos[1:], "fp32")
        _, _, after16 = LR.run_node(call, acts, weights, dos, "bf16")
        check(J, "bf16_store", None, None, after16[0], "bf16", 1)
        check(J, "bf16_accum", None, None, after16[1], "bf16", 2)
        for n, p in weights.items():
            # host-side adds: the old bf16 slot plus the fp32 value, rounded once.  Checkable only where the fp32
            # value is bit-reproducible from run to run (the conv and some norm gains sum over tokens in a varying
            # order); the CPU tier checks the rule for every parameter
            if MR.is_vector(n, p) and torch.equal(only2[0][n], again2[0][n]):
                J(f"{n}.bf16_accum_one_rounding", LR.one_rounding(
                    after16[1][n], after16[0][n].to(F64) + only2[0][n].to(F64)) / (1 + 2.0 ** -15))
            elif MR.is_vector(n, p):
                print(f"  {tag}: {n} is not bit-reproducible; one-rounding checked on the CPU tier only")
        assert CK.fallback_count() - f0 == 7 * fallbacks_per_call, f"{tag}: {CK.fallback_count() - f0} ATen fallbacks"
        ops.set_kernel_path("torch")
        out, dacts, after = LR.run_node(call, acts, weights, dos[:1], "returned")
        A = Judge(f"{tag} ATen path (not asserted)")
        check(A, "aten", out, dacts, after[0], "returned", 1)
        A.done(enforce=False)
    finally:
        ops.set_kernel_path("auto")


def rnd(g, *s, sc=1.0):
    return (torch.randn(*s, generator=g, device=DEV) * sc).to(BF16)


def judge_case(CK, tag, keyp, call, fn, acts, weights, dos, M, fallbacks_per_call=0, tied=False, post=None,
               dw_key=None):
    """Reference of dos[0] and of dos[0] + dos[1] (``fn(p, a)`` on float64 copies, then ``post(ref)``), then every
    delivery.  ``tied``: ``fn`` reads the head from a separate "lm_head.weight" holding the embedding's values."""
    params = {n: p.detach() for n, p in weights.items()}
    if tied:
        params["lm_head.weight"] = params["backbone.embedding.weight"]
    refs = {}
    for mb in (1, 2):
        d = tuple(sum(x[i].to(F64) for x in dos[:mb]) for i in range(len(dos[0])))
        refs[mb] = MR.evaluate(fn, params, {n: t.detach() for n, t in acts.items()}, d, M, device=DEV)
        if post is not None:
            post(refs[mb])
        torch.cuda.empty_cache()

    def check(J, label, out, dacts, grads, mode, mb):
        ref = refs[mb]
        if out is not None:
            for i, (o, q) in enumerate(zip(out, ref["out"])):
                J(f"out{i}", frac_rows(o.detach(), q, keyp + "_y") if q.dim() else
                  abs(float(o) - float(q)) / abs(float(q)) / MR.TOL[keyp + "_loss"])
        if dacts is not None:
            for n, t in dacts.items():
                J(f"d{n}", frac_rows(t, ref["d" + n], keyp + "_dx"))
        for n, p in weights.items():
            if MR.is_vector(n, p):
                rounded = () if mode == "fp32" else tuple(refs[i][n] for i in range(1, mb + 1))
                J(f"{n}.{label}", frac_vec(grads[n], ref[n], ref[n + "_abs"], keyp + "_dv", rounded))
            else:
                J(f"{n}.{label}", frac_rows(grads[n], ref[n], dw_key or keyp + "_dw", mode != "fp32",
                                            ref.get(n + "_scale")))

    J = Judge(tag)
    leaves = {n: t for n, t in acts.items() if t.is_floating_point()}
    deliveries(J, CK, tag, call, leaves, weights, dos, check, fallbacks_per_call)
    del refs
    J.done()


# ================================================================================================= the cases
M2 = {"2.8b": dict(d_model=2560, headdim=64, d_state=128, ngroups=1),
      "9.8b": dict(d_model=4096, headdim=64, d_state=128, ngroups=1),
      "9.8b_G8": dict(d_model=4096, headdim=64, d_state=128, ngroups=8)}


def slow_enough(mix, u):
    """exp(aL) > 0.5 in every 128-step chunk (the slow regime's promise), from the float64 dt."""
    H = mix.nheads
    dt = u.reshape(-1, u.shape[-1]).to(F64) @ mix.in_proj.weight[-H:].to(F64).t()
    a = MR.softplus(dt + mix.dt_bias.to(F64)) * -torch.exp(mix.A_log.to(F64))
    S = u.shape[1]
    aL = a.view(u.shape[0], S // 128, 128, H).sum(2) if S % 128 == 0 else a.sum(0, keepdim=True)
    return bool((torch.exp(aL) > 0.5).all())


M2_CASES = [("2.8b", 1, 4096, "init", 0), ("2.8b", 1, 4096, "slow", 0), ("2.8b", 1, 4096, "trained", 0),
            ("2.8b", 2, 1024, "trained", 0), ("9.8b", 1, 4096, "slow", 0),
            ("9.8b_G8", 1, 1024, "trained", 2),        # grouped gated norm: rmsnorm_gated_fwd / _bwd on ATen
            ("2.8b", 1, 1000, "trained", 2)]           # S % 128 != 0: ssd_scan_chunked / ssd_scan_bwd on ATen


@pytest.mark.parametrize("shape,B,S,regime,fb", M2_CASES, ids=[f"{s}-B{b}-S{n}-{r}" for s, b, n, r, _ in M2_CASES])
def test_mamba2_mixer_against_float64(CK, shape, B, S, regime, fb):
    torch.manual_seed(0)
    mix = Mamba2(**M2[shape], device=DEV, dtype=BF16)
    mix.reset_parameters()
    MR.set_regime(mix, regime)
    cfg = MR.mixer_cfg(mix)
    g = torch.Generator(device=DEV).manual_seed(1)
    u = rnd(g, B, S, mix.d_model).requires_grad_()
    if regime == "slow":
        assert slow_enough(mix, u.detach())
    dos = [(rnd(g, B, S, mix.d_model),), (rnd(g, B, S, mix.d_model),)]
    M = B * S
    judge_case(CK, f"Mamba2 {shape} B{B} S{S} {regime}", "m2", lambda: mix(u),
               lambda p, a: MR.mamba2(p, a["u"].reshape(M, -1), S, cfg, chunk=256).view(B, S, -1),
               {"u": u}, dict(mix.named_parameters()), dos, M, fb)


M1_CASES = [(1, 2048, "init"), (2, 1024, "trained")]


@pytest.mark.parametrize("B,S,regime", M1_CASES, ids=[f"B{b}-S{s}-{r}" for b, s, r in M1_CASES])
def test_mamba1_mixer_against_float64(CK, B, S, regime):
    torch.manual_seed(0)
    mix = Mamba1(2560, d_state=16, device=DEV, dtype=BF16)
    mix.reset_parameters()
    MR.set_regime(mix, regime)
    cfg = MR.mixer_cfg(mix)
    g = torch.Generator(device=DEV).manual_seed(2)
    u = rnd(g, B, S, 2560).requires_grad_()
    dos = [(rnd(g, B, S, 2560),), (rnd(g, B, S, 2560),)]
    M = B * S
    judge_case(CK, f"Mamba1 2.8b B{B} S{S} {regime}", "m1", lambda: mix(u),
               lambda p, a: MR.mamba1(p, a["u"].reshape(M, -1), S, cfg).view(B, S, -1),
               {"u": u}, dict(mix.named_parameters()), dos, M)


@pytest.mark.parametrize("B,S", [(1, 4096), (2, 1024)])
def test_mha_against_float64(CK, B, S):
    torch.manual_seed(0)
    mix = MHA(4096, 32, 8, 128, 64, device=DEV, dtype=BF16)
    mix.reset_parameters()
    cfg = MR.mixer_cfg(mix)
    g = torch.Generator(device=DEV).manual_seed(3)
    x = rnd(g, B, S, 4096).requires_grad_()
    dos = [(rnd(g, B, S, 4096),), (rnd(g, B, S, 4096),)]
    M = B * S
    judge_case(CK, f"MHA 9.8b B{B} S{S}", "mha", lambda: mix(x),
               lambda p, a: MR.mha(p, a["x"].reshape(M, -1), S, cfg).view(B, S, -1),
               {"x": x}, dict(mix.named_parameters()), dos, M)


def test_gated_mlp_against_float64(CK):
    torch.manual_seed(0)
    mlp = GatedMLP(4096, 14336, device=DEV, dtype=BF16)
    mlp.reset_parameters()
    g = torch.Generator(device=DEV).manual_seed(4)
    x = rnd(g, 1, 4096, 4096).requires_grad_()
    dos = [(rnd(g, 1, 4096, 4096),), (rnd(g, 1, 4096, 4096),)]
    judge_case(CK, "GatedMLP 9.8b B1 S4096", "mlp", lambda: mlp(x),
               lambda p, a: MR.gated_mlp(p, a["x"].reshape(4096, -1)).view(1, 4096, -1),
               {"x": x}, dict(mlp.named_parameters()), dos, 4096)


BLOCKS = {"mamba2_mlp": ("Mamba2", 4096, 14336), "attention_mlp": ("MHA", 4096, 14336), "mamba2_2.8b": ("Mamba2", 2560, 0)}


@pytest.mark.parametrize("which", list(BLOCKS))
def test_block_against_float64(CK, which):
    kind, D, F = BLOCKS[which]
    torch.manual_seed(0)
    mix = Mamba2(D, device=DEV, dtype=BF16) if kind == "Mamba2" else MHA(D, 32, 8, 128, 64, device=DEV, dtype=BF16)
    blk = Block(D, mix, GatedMLP(D, F, device=DEV, dtype=BF16) if F else None, device=DEV, dtype=BF16)
    blk.reset_parameters()
    mix.reset_parameters()
    if F:
        blk.mlp.reset_parameters()
    with torch.no_grad():
        for n, p in blk.named_parameters():
            if n in ("norm.weight", "norm2.weight", "mixer.norm.weight"):
                p.copy_(1 + 0.3 * torch.randn(p.shape, device=DEV))
    cfg = MR.mixer_cfg(mix)
    S = 4096
    g = torch.Generator(device=DEV).manual_seed(5)
    h = rnd(g, 1, S, D).requires_grad_()
    r = torch.randn(1, S, D, generator=g, device=DEV).requires_grad_()
    dos = [(rnd(g, 1, S, D), torch.randn(1, S, D, generator=g, device=DEV)) for _ in range(2)]
    judge_case(CK, f"Block {which} B1 S{S}", "blk", lambda: blk(h, r),
               lambda p, a: tuple(t.view(1, S, -1) for t in MR.block(p, a["h"].reshape(S, -1), a["r"].reshape(S, -1),
                                                                     S, cfg, chunk=256)),
               {"h": h, "r": r}, dict(blk.named_parameters()), dos, S)


@pytest.mark.parametrize("which", ["2.8b_tied", "9.8b_untied"])
def test_ends_against_float64(CK, which):
    D, V, tied = (2560, 50280, True) if which == "2.8b_tied" else (4096, 128256, False)
    torch.manual_seed(0)
    model = MambaLMHeadModel(MambaConfig(d_model=D, n_layer=0, vocab_size=V, tie_embeddings=tied), device=DEV, dtype=BF16)
    model.reset_parameters()
    with torch.no_grad():
        model.backbone.norm_f.weight.copy_(1 + 0.3 * torch.randn(D, device=DEV))
    S = 4096
    g = torch.Generator(device=DEV).manual_seed(6)
    Vp = model.config.padded_vocab
    tokens = torch.randint(0, Vp, (1, S), generator=g, device=DEV)
    labels = torch.randint(0, Vp, (S,), generator=g, device=DEV)
    labels[torch.rand(S, generator=g, device=DEV) < 0.1] = -100
    weights = dict(model.named_parameters())
    one = torch.ones((), device=DEV)
    stats = {}
    FN.set_unit_upstream(True)                   # as the engine runs the head: an upstream gradient of exactly 1
    try:
        judge_case(CK, f"ends {which} V{Vp} B1 S{S}", "end", lambda: model.engine_head(*model.engine_embed(tokens),
                                                                                      labels=labels),
                   lambda p, a: MR.ends(p, a["tokens"].reshape(-1), a["labels"], False, stats=stats),
                   {"tokens": tokens, "labels": labels}, weights, [(one,), (one,)], S, tied=tied,
                   post=lambda ref: MR.head_scales(ref, stats, tied), dw_key="end_tied_dw" if tied else None)
    finally:
        FN.set_unit_upstream(False)
