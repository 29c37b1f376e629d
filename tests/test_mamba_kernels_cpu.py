"""CPU tier of the Mamba kernel tests (``tests/test_mamba_kernels_gpu.py`` is the H100 tier).

* The chunked (state-space dual) SSD form, which the GPU tests use as the reference at S = 4096, equals the sequential
  recurrence in value and in every gradient, in float64, for chunk lengths that do and do not divide S.
* The selective-scan oracle's autograd gradients equal a written-out float64 adjoint recurrence.
* Sensitivity guards: each GPU probe, run here at a CPU-sized instance of the same input distribution, would notice the
  term it probes.  Removing that term from the reference (cutting the sequence at the chunk / block length, merging the
  sequences of a batch, dropping the dt = 0 term) changes the probed region by at least 10x the GPU tolerance.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from fms_fsdp_b200.ops import torch_kernels as TK

F64 = torch.float64
L_SSD = 128            # csrc/ssd.cu chunk length
L_SEL = 32             # csrc/selscan.cu block length (one warp lane per step)
# tolerances of the GPU tier (kept equal to the constants of tests/test_mamba_kernels_gpu.py)
TOL_FWD, TOL_GRAD = 2e-2, 3e-2


# ----------------------------------------------------------------------------------------------- inputs
def inv_softplus(v):
    return v + torch.log(-torch.expm1(-v))


def ssd_inputs(regime, Bsz, S, H, P, G, N, gen, use_D=True, use_bias=True):
    """The GPU tier's SSD input distributions.  fast: the historic test distribution (chunk decay exp(aL) ~ 0);
    init: ``Mamba2.reset_parameters`` (dt log-uniform in [1e-3, 0.1] through dt_bias, A in [-16, -1]);
    slow: exp(aL) > 0.5 in every chunk."""
    M = Bsz * S
    r = lambda *s: torch.randn(*s, generator=gen)
    u = lambda *s: torch.rand(*s, generator=gen)
    if regime == "fast":
        dt, A, bias = r(M, H) * 0.5 - 1.0, -(u(H) * 4 + 0.5), r(H) * 0.2
    elif regime == "init":
        dt0 = torch.exp(u(H) * (math.log(0.1) - math.log(1e-3)) + math.log(1e-3))
        dt, A, bias = r(M, H) * 0.1, -(1 + 15 * u(H)), inv_softplus(dt0)
    else:
        dt, A, bias = r(M, H) * 0.05, -(0.5 + 0.5 * u(H)), inv_softplus(1e-3 + 2e-3 * u(H))
    if not use_bias:
        dt, bias = dt + bias, None
    return dict(x=r(M, H, P), dt=dt, A=A, Bm=r(M, G, N) * 0.5, Cm=r(M, G, N) * 0.5, D=r(H) if use_D else None,
                dt_bias=bias)


def sel_inputs(regime, Bsz, S, Dm, gen, use_z=True, use_D=True, use_bias=True, softplus=True):
    """Selective-scan (Mamba1, N = 16) distributions; init = ``Mamba1.reset_parameters`` (A = -(1..16))."""
    M, N = Bsz * S, 16
    r = lambda *s: torch.randn(*s, generator=gen)
    u = lambda *s: torch.rand(*s, generator=gen)
    if regime == "fast":
        delta, A, bias = r(M, Dm) * 0.5 - 1.0, -(u(Dm, N) * 4 + 0.5), r(Dm) * 0.2
    elif regime == "init":
        dt0 = torch.exp(u(Dm) * (math.log(0.1) - math.log(1e-3)) + math.log(1e-3))
        delta, A, bias = r(M, Dm) * 0.1, -torch.arange(1, N + 1, dtype=torch.float32).expand(Dm, N).clone(), inv_softplus(dt0)
    else:
        delta, A, bias = r(M, Dm) * 0.05, -(0.5 + 0.5 * u(Dm, N)), inv_softplus(1e-3 + 2e-3 * u(Dm))
    if not softplus:                          # the raw delta is the step: fold bias and softplus into it
        delta, bias = F.softplus(delta + bias), (None if not use_bias else torch.zeros(Dm))
    elif not use_bias:
        delta, bias = delta + bias, None
    return dict(u=r(M, Dm), delta=delta, A=A, Bm=r(M, N) * 0.5, Cm=r(M, N) * 0.5, D=r(Dm) if use_D else None,
                z=r(M, Dm) if use_z else None, delta_bias=bias)


def f64(d):
    return {k: (None if v is None else v.to(F64)) for k, v in d.items()}


def chunk_decay(inp, seq_len, L=L_SSD, softplus=True):
    """exp(sum of dt * A over each L-step chunk), [batch * chunks, H]."""
    v = inp["dt"].double() + (0 if inp["dt_bias"] is None else inp["dt_bias"].double())
    v = F.softplus(v) if softplus else v
    return torch.exp((v * inp["A"].double()).view(-1, L, v.shape[-1]).sum(1))


def region_change(ref, cut, sl=None):
    """max-abs of (ref - cut) over the probed region, over the max-abs of ref there (the GPU tier's metric)."""
    a, b = (ref, cut) if sl is None else (ref[sl], cut[sl])
    return ((a - b).abs().max() / a.abs().max()).item()


def ssd_seq(d, seq_len, softplus=True):
    return TK.ssd_scan_fwd(d["x"], d["dt"], d["A"], d["Bm"], d["Cm"], d["D"], d["dt_bias"], seq_len, 0, softplus)


def rows(Bsz, S, lo, hi):
    """Row mask of steps [lo, hi) of every sequence of a [Bsz * S, ...] tensor."""
    m = torch.zeros(Bsz, S, dtype=torch.bool)
    m[:, lo:hi] = True
    return m.reshape(-1)


# ------------------------------------------------------------------- chunked SSD form vs the recurrence
def _grads(fn, d, dy):
    leaves = {k: v.clone().requires_grad_() for k, v in d.items() if v is not None}
    y = fn({**d, **leaves})
    return y, dict(zip(leaves, torch.autograd.grad(y, list(leaves.values()), dy)))


@pytest.mark.parametrize("S,L,G,opts", [
    (70, 16, 1, {}), (70, 32, 2, {}), (96, 7, 4, {}), (64, 64, 4, {}), (50, 128, 2, {}),
    (96, 32, 1, {"use_D": False}), (96, 40, 2, {"use_bias": False}), (96, 24, 4, {"softplus": False}),
])
def test_ssd_chunked_equals_sequential_fp64_value_and_grads(S, L, G, opts):
    gen = torch.Generator().manual_seed(S * 31 + L)
    opts = dict(opts)
    softplus = opts.pop("softplus", True)
    H, P, N, Bsz = 4, 8, 8, 2
    d = f64(ssd_inputs("slow", Bsz, S, H, P, G, N, gen, **opts))
    if not softplus:
        d["dt"] = F.softplus(d["dt"] + (0 if d["dt_bias"] is None else d["dt_bias"]))
        d["dt"].view(-1)[::5] = 0.0                   # steps with dt exactly 0
    dy = torch.randn(Bsz * S, H, P, generator=gen, dtype=F64)
    args = lambda e: (e["x"], e["dt"], e["A"], e["Bm"], e["Cm"], e["D"], e["dt_bias"], S, L, softplus)
    y0, g0 = _grads(lambda e: TK.ssd_scan_fwd(*args(e)), d, dy)
    y1, g1 = _grads(lambda e: TK.ssd_scan_chunked(*args(e)), d, dy)
    assert y0.dtype == F64 and y1.dtype == F64
    assert (y1 - y0).abs().max() <= 1e-11 * y0.abs().max()
    for k in g0:
        assert (g1[k] - g0[k]).abs().max() <= 1e-10 * g0[k].abs().max(), k


# ----------------------------------------------------------------- selective scan vs a written-out adjoint
def sel_adjoint(d, seq_len, dout, softplus=True):
    """Gradients of ``TK.selective_scan_fwd`` by the backward recurrence written out in float64."""
    u, A = d["u"], d["A"]
    M, Dm = u.shape
    Bsz, N = M // seq_len, A.shape[1]
    view = lambda t, w: t.reshape(Bsz, seq_len, w)
    uf, raw = view(u, Dm), view(d["delta"], Dm)
    pre = raw + (0 if d["delta_bias"] is None else d["delta_bias"])
    dl = F.softplus(pre) if softplus else pre
    Bf, Cf, g_out = view(d["Bm"], N), view(d["Cm"], N), view(dout, Dm)
    a = torch.exp(dl[..., None] * A)                                   # [b, t, d, n]
    hs, h = [], torch.zeros(Bsz, Dm, N, dtype=F64)
    for t in range(seq_len):
        h = a[:, t] * h + (dl[:, t] * uf[:, t])[..., None] * Bf[:, t, None, :]
        hs.append(h)
    y = torch.stack([(hh * Cf[:, t, None, :]).sum(-1) for t, hh in enumerate(hs)], 1)
    if d["D"] is not None:
        y = y + uf * d["D"]
    out = {}
    if d["z"] is not None:
        z = view(d["z"], Dm)
        sg = torch.sigmoid(z)
        out["z"] = (g_out * y * sg * (1 + z * (1 - sg))).reshape(M, Dm)
        gy = g_out * z * sg
    else:
        gy = g_out
    if d["D"] is not None:
        out["D"] = (gy * uf).sum((0, 1))
    du, ddl = torch.zeros_like(uf), torch.zeros_like(uf)
    dB, dC, dA = torch.zeros_like(Bf), torch.zeros_like(Cf), torch.zeros_like(A)
    g = torch.zeros(Bsz, Dm, N, dtype=F64)
    for t in reversed(range(seq_len)):
        g = g + gy[:, t, :, None] * Cf[:, t, None, :]                 # adjoint of h_t
        dC[:, t] = (gy[:, t, :, None] * hs[t]).sum(1)
        gB = (g * Bf[:, t, None, :]).sum(-1)
        dB[:, t] = (g * (dl[:, t] * uf[:, t])[..., None]).sum(1)
        du[:, t] = dl[:, t] * gB + (0 if d["D"] is None else gy[:, t] * d["D"])
        hprev = hs[t - 1] if t > 0 else torch.zeros_like(g)
        gda = g * hprev * a[:, t]                                      # adjoint of log a_t = dl_t * A
        ddl[:, t] = uf[:, t] * gB + (gda * A).sum(-1)
        dA += (gda * dl[:, t, :, None]).sum(0)
        g = a[:, t] * g
    dpre = ddl * torch.sigmoid(pre) if softplus else ddl
    out.update(u=du.reshape(M, Dm), delta=dpre.reshape(M, Dm), A=dA, Bm=dB.reshape(M, N), Cm=dC.reshape(M, N))
    if d["delta_bias"] is not None:
        out["delta_bias"] = dpre.sum((0, 1))
    return y, out


@pytest.mark.parametrize("regime", ["init", "slow", "fast"])
@pytest.mark.parametrize("use_z,use_D,use_bias,softplus", [
    (True, True, True, True), (False, True, True, True), (True, False, True, True), (True, True, False, True),
    (False, False, False, False), (True, True, True, False),
])
def test_selective_scan_oracle_grads_match_written_out_recurrence(regime, use_z, use_D, use_bias, softplus):
    gen = torch.Generator().manual_seed(7)
    Bsz, S, Dm = 2, 40, 6
    d = f64(sel_inputs(regime, Bsz, S, Dm, gen, use_z, use_D, use_bias, softplus))
    dout = torch.randn(Bsz * S, Dm, generator=gen, dtype=F64)
    keys = [k for k in ("u", "delta", "A", "Bm", "Cm", "D", "z", "delta_bias") if d[k] is not None]
    leaves = {k: d[k].clone().requires_grad_() for k in keys}
    e = {**d, **leaves}
    y = TK.selective_scan_fwd(e["u"], e["delta"], e["A"], e["Bm"], e["Cm"], e["D"], e["z"], e["delta_bias"], S, softplus)
    assert y.dtype == F64
    auto = dict(zip(keys, torch.autograd.grad(y, [leaves[k] for k in keys], dout)))
    _, mine = sel_adjoint(d, S, dout, softplus)
    assert set(mine) == set(keys)
    for k in keys:
        assert (mine[k] - auto[k]).abs().max() <= 1e-10 * auto[k].abs().max(), k


# --------------------------------------------------------------------------------------- sensitivity guards
def ssd_probe_case(regime, Bsz=1, nc=4, H=4, P=8, G=1, N=16, seed=0):
    gen = torch.Generator().manual_seed(seed)
    S = nc * L_SSD
    return S, f64(ssd_inputs(regime, Bsz, S, H, P, G, N, gen))


@pytest.mark.parametrize("regime", ["init", "slow"])
def test_guard_ssd_carry_probe_sees_the_chunk_to_chunk_state(regime):
    """GPU carry probe: x only in chunk 0, y checked over chunks 1..n.  Cutting the sequence at the chunk length (no carried
    state) changes every later chunk, the last one included, by the whole region."""
    S, d = ssd_probe_case(regime)
    d["x"][rows(1, S, L_SSD, S)] = 0
    ref = ssd_seq(d, S)
    cut = ssd_seq(d, L_SSD)
    last = rows(1, S, S - L_SSD, S)
    assert region_change(ref, cut, last) >= 10 * TOL_FWD
    assert region_change(ref, cut, rows(1, S, L_SSD, S)) >= 10 * TOL_FWD
    # the carried signal survives to the last chunk, far above the fp32 floor of the output (it is small next to the D x
    # skip term of chunk 0, and in the init regime the slow heads that carry it also take small steps)
    assert ref[last].abs().max() >= 1e-4 * ref.abs().max()
    if regime == "slow":
        assert chunk_decay(d, S).min() > 0.5


def test_guard_fast_regime_hides_the_carried_state():
    """Why the historic SSD test could not see the chunk-to-chunk recurrence: in its distribution the carried state is
    multiplied by exp(aL) < 1e-20, so the output beyond chunk 0 is numerically zero."""
    S, d = ssd_probe_case("fast")
    assert chunk_decay(d, S).max() < 1e-12
    d["x"][rows(1, S, L_SSD, S)] = 0
    ref = ssd_seq(d, S)
    # chunk 1 still reads chunk 0's final state; every later chunk reads it through at least one factor exp(aL)
    assert ref[rows(1, S, 2 * L_SSD, S)].abs().max() < 1e-12 * ref.abs().max()


@pytest.mark.parametrize("regime", ["init", "slow"])
def test_guard_ssd_adjoint_probe_sees_the_reverse_state_pass(regime):
    """GPU adjoint probe: dy only in the last chunk; dx, ddt, dB over the earlier chunks and dA, d(dt_bias) checked.  Without
    the reverse chunk recurrence (sequence cut at the chunk length) all of them change by >= 10x the gradient tolerance;
    dA and d(dt_bias) do in the slow regime (at init the fast heads, which carry nothing, set their scale)."""
    S, d = ssd_probe_case(regime, seed=1)
    gen = torch.Generator().manual_seed(5)
    dy = torch.randn(S, 4, 8, generator=gen, dtype=F64)
    dy[~rows(1, S, S - L_SSD, S)] = 0
    fn = lambda seq: (lambda e: TK.ssd_scan_fwd(e["x"], e["dt"], e["A"], e["Bm"], e["Cm"], e["D"], e["dt_bias"], seq, 0))
    _, g_ref = _grads(fn(S), d, dy)
    _, g_cut = _grads(fn(L_SSD), d, dy)
    early = rows(1, S, 0, S - L_SSD)
    first = rows(1, S, 0, L_SSD)
    for k in ("x", "dt", "Bm"):
        assert region_change(g_ref[k], g_cut[k], early) >= 10 * TOL_GRAD, k
        assert g_ref[k][first].abs().max() >= 1e-3 * g_ref[k].abs().max(), k    # reaches the first chunk
    for k in ("A", "dt_bias") if regime == "slow" else ():
        assert region_change(g_ref[k], g_cut[k]) >= 10 * TOL_GRAD, k


def ssd_intra_dt_term(d, dy, seq_len, L=L_SSD):
    """The direct intra-chunk part of d(loss)/d(dt_s) at steps with dt_s = 0 (no softplus, no bias): dt_s as the weight
    of x_s, not as a decay exponent.  Written out: sum over l >= s in the chunk of exp(acs_l - acs_s) (C_l . B_s) (dy_l . x_s)."""
    x, dt, A, Bm, Cm = d["x"], d["dt"], d["A"], d["Bm"], d["Cm"]
    M, H, P = x.shape
    Hg = H // Bm.shape[1]
    out = torch.zeros(M, H, dtype=F64)
    for s, h in (dt == 0).nonzero().tolist():
        c_end = (s // L + 1) * L
        acc, run = 0.0, 0.0
        for l in range(s, c_end):
            if l > s:
                run += float(dt[l, h] * A[h])
            acc += math.exp(run) * float(Cm[l, h // Hg] @ Bm[s, h // Hg]) * float(dy[l, h] @ x[s, h])
        out[s, h] = acc
    return out


def test_guard_ssd_dt_zero_probe_sees_the_intra_chunk_term():
    """GPU probe of dt_softplus=False with dt exactly 0 at some steps: the dt gradient there has a direct intra-chunk term
    that a column sum divided by dt cannot carry.  The written-out term equals autograd's dt gradient when A = 0 (no decay
    path), and dropping it changes the dt gradient at those steps by >= 10x the gradient tolerance."""
    gen = torch.Generator().manual_seed(3)
    S, H, P, N = L_SSD, 2, 8, 8
    d = f64(ssd_inputs("slow", 1, S, H, P, 1, N, gen, use_bias=False))
    d["dt"] = F.softplus(d["dt"])
    zero = torch.zeros(S, H, dtype=torch.bool)
    zero[3::11] = True
    d["dt"][zero] = 0.0
    dy = torch.randn(S, H, P, generator=gen, dtype=F64)
    fn = lambda e: TK.ssd_scan_fwd(e["x"], e["dt"], e["A"], e["Bm"], e["Cm"], e["D"], e["dt_bias"], S, 0, False)
    flat = dict(d, A=torch.zeros_like(d["A"]))
    _, g_flat = _grads(fn, flat, dy)
    assert (g_flat["dt"][zero] - ssd_intra_dt_term(flat, dy, S)[zero]).abs().max() <= 1e-10 * g_flat["dt"][zero].abs().max()
    _, g = _grads(fn, d, dy)
    without = g["dt"][zero] - ssd_intra_dt_term(d, dy, S)[zero]
    assert region_change(g["dt"][zero], without) >= 10 * TOL_GRAD


def test_guard_batch_isolation_probes_see_a_leak():
    """GPU batch-isolation probes: sequences 2 and 3 of a batch of 3 against the same sequences alone.  Merging the batch
    into one sequence (a leak of state, conv window or carry) changes those sequences by >= 10x the gradient tolerance."""
    gen = torch.Generator().manual_seed(11)
    S = 2 * L_SSD
    d = f64(ssd_inputs("slow", 3, S, 4, 8, 1, 16, gen, use_D=False))    # D x would hide the state in the metric
    later = torch.arange(3 * S) >= S
    assert region_change(ssd_seq(d, S), ssd_seq(d, 3 * S), later) >= 10 * TOL_GRAD
    s = f64(sel_inputs("slow", 3, 2 * L_SEL, 32, gen, use_D=False))
    sel = lambda seq: TK.selective_scan_fwd(s["u"], s["delta"], s["A"], s["Bm"], s["Cm"], s["D"], s["z"], s["delta_bias"], seq)
    later = torch.arange(3 * 2 * L_SEL) >= 2 * L_SEL
    assert region_change(sel(2 * L_SEL), sel(6 * L_SEL), later) >= 10 * TOL_GRAD
    Sc, C = 65, 16
    x = torch.randn(3 * Sc, C, generator=gen, dtype=F64)
    w = torch.randn(C, 4, generator=gen, dtype=F64)
    conv = lambda seq: TK.causal_conv1d_fwd(x, w, None, seq, True)
    head = (torch.arange(3 * Sc) % Sc < 3) & (torch.arange(3 * Sc) >= Sc)     # the K - 1 first steps of sequences 2, 3
    assert region_change(conv(Sc), conv(3 * Sc), head) >= 10 * TOL_GRAD


@pytest.mark.parametrize("regime", ["init", "slow"])
def test_guard_selective_scan_block_carry_and_adjoint(regime):
    """GPU selective-scan probes across 32-step blocks: u only in block 0 (y over the later blocks), dy only in the last
    block (du, ddelta, dB over the earlier blocks; dA, d(delta_bias)).  Cutting at the block length changes each by
    >= 10x the tolerance."""
    gen = torch.Generator().manual_seed(13)
    S, Dm = 4 * L_SEL, 8
    d = f64(sel_inputs(regime, 1, S, Dm, gen))
    fwd = lambda e, seq: TK.selective_scan_fwd(e["u"], e["delta"], e["A"], e["Bm"], e["Cm"], e["D"], e["z"],
                                               e["delta_bias"], seq)
    c = dict(d)
    c["u"] = d["u"].clone()
    c["u"][L_SEL:] = 0
    later = rows(1, S, L_SEL, S)
    ref = fwd(c, S)
    assert region_change(ref, fwd(c, L_SEL), rows(1, S, S - L_SEL, S)) >= 10 * TOL_FWD
    assert ref[later].abs().max() >= 1e-3 * ref.abs().max()
    dy = torch.randn(S, Dm, generator=gen, dtype=F64)
    dy[: S - L_SEL] = 0
    _, g_ref = _grads(lambda e: fwd(e, S), d, dy)
    _, g_cut = _grads(lambda e: fwd(e, L_SEL), d, dy)
    early = rows(1, S, 0, S - L_SEL)
    for k in ("u", "delta", "Bm"):
        assert region_change(g_ref[k], g_cut[k], early) >= 10 * TOL_GRAD, k
    for k in ("A", "delta_bias"):
        assert region_change(g_ref[k], g_cut[k]) >= 10 * TOL_GRAD, k
