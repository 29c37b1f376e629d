"""Mamba kernels on the H100 against plain fp32 references: the SSD scan (csrc/ssd.cu and the batched GEMMs it drives),
the selective scan (csrc/selscan.cu), the causal conv1d (csrc/mamba.cu) and the fp32-residual / gated RMSNorm kernels
(csrc/elementwise.cu).

Inputs are bf16-rounded; the references get them cast to fp32 and their outputs are never rounded.  Errors are
``|a - b| / |b|`` (2-norm) and max-abs over the reference's max-abs, over the region a probe isolates.  Three input
regimes (``tests/test_mamba_kernels_cpu.py`` shows each probe can fail at them):
  fast   the historic test distribution, chunk decay exp(aL) ~ 0;
  init   the ``reset_parameters`` distributions of Mamba2 (dt log-uniform in [1e-3, 0.1], A in [-16, -1]) and Mamba1
         (A = -(1..16));
  slow   exp(aL) > 0.5 in every 128-step chunk.
Probes: carry (x only in chunk / block 0, y checked over the later ones) and adjoint (dy only in the last chunk / block,
the gradients checked over the earlier ones).  Every kernel call must run our kernels (``launch_count`` rises) and take no
ATen fallback, except where a test asserts the counted fallback on purpose.
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
L_SSD, L_SEL = 128, 32
TOL_FWD, TOL_GRAD = 2e-2, 3e-2
TOL_ISO = 8e-3          # per-row gradients of one sequence, batched vs alone: atomics reorder fp32 sums (one bf16 ulp)


@pytest.fixture(scope="module")
def K():
    from fms_fsdp_b200.ops import cuda_kernels as CK
    from fms_fsdp_b200.ops import torch_kernels as TK
    assert CK._C.__file__.endswith("_C.so")
    return CK, TK


class Native:
    """Asserts the block launched our kernels and took no ATen fallback."""

    def __init__(self, CK):
        self.CK = CK

    def __enter__(self):
        self.n0, self.f0 = self.CK.launch_count(), self.CK.fallback_count()
        return self

    def __exit__(self, et, *_):
        if et is None:
            assert self.CK.launch_count() > self.n0, "no kernel of ours ran"
            assert self.CK.fallback_count() == self.f0, dict(self.CK.FALLBACKS)


class Errors:
    """Collects (norm, max) errors against tolerances, prints them all, fails at the end with every violation."""

    def __init__(self, tag):
        self.tag, self.bad = tag, []

    def __call__(self, name, a, b, tol, sl=None, scale=None):
        a, b = a.detach().double(), b.detach().double()
        if sl is not None:
            a, b = a[sl], b[sl]
        d = a - b
        den_n = b.norm().clamp(min=1e-30) if scale is None else scale
        den_m = b.abs().max().clamp(min=1e-30) if scale is None else scale
        en, em = (d.norm() / den_n).item(), (d.abs().max() / den_m).item()
        print(f"MEASURE {self.tag} {name}: norm {en:.2e} max {em:.2e} tol {tol:.0e}")
        if not (en <= tol and em <= tol):
            self.bad.append((name, en, em, tol))

    def done(self):
        assert not self.bad, self.bad


def bits_equal(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b)


# ----------------------------------------------------------------------------------------------- inputs
def inv_softplus(v):
    return v + torch.log(-torch.expm1(-v))


def ssd_inputs(regime, Bsz, S, H, P, G, N, seed, use_D=True, use_bias=True):
    """Same distributions as ``tests/test_mamba_kernels_cpu.py``; x, dt, B, C bf16 on the device, A, D, dt_bias fp32."""
    gen = torch.Generator().manual_seed(seed)
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
    b16 = lambda t: t.to(DEV).bfloat16()
    return dict(x=b16(r(M, H, P)), dt=b16(dt), A=A.to(DEV), Bm=b16(r(M, G, N) * 0.5), Cm=b16(r(M, G, N) * 0.5),
                D=r(H).to(DEV) if use_D else None, dt_bias=None if bias is None else bias.to(DEV))


def sel_inputs(regime, Bsz, S, Dm, seed, use_z=True, use_D=True, use_bias=True, softplus=True):
    gen = torch.Generator().manual_seed(seed)
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
    if not softplus:
        delta, bias = F.softplus(delta + bias), (None if not use_bias else torch.zeros(Dm))
    elif not use_bias:
        delta, bias = delta + bias, None
    b16 = lambda t: t.to(DEV).bfloat16()
    return dict(u=b16(r(M, Dm)), delta=b16(delta), A=A.to(DEV), Bm=b16(r(M, N) * 0.5), Cm=b16(r(M, N) * 0.5),
                D=r(Dm).to(DEV) if use_D else None, z=b16(r(M, Dm)) if use_z else None,
                delta_bias=None if bias is None else bias.to(DEV))


def rows(Bsz, S, lo, hi):
    m = torch.zeros(Bsz, S, dtype=torch.bool, device=DEV)
    m[:, lo:hi] = True
    return m.reshape(-1)


def ref_grads(fn, d, keys, dy):
    """fp32 reference output and gradients (autograd) for the inputs ``keys`` of ``d``."""
    leaves = {k: d[k].detach().float().requires_grad_() for k in keys}
    e = {k: (v.float() if v is not None else None) for k, v in d.items()}
    e.update(leaves)
    y = fn(e)
    if dy is None:
        return y.detach(), None
    return y.detach(), dict(zip(keys, torch.autograd.grad(y, list(leaves.values()), dy.float())))


# --------------------------------------------------------------------------------------------------- SSD
SSD_KEYS = ("x", "dt", "A", "Bm", "Cm", "D", "dt_bias")


def ssd_ref(TK, seq_len, softplus=True):
    """Sequential recurrence up to S = 1024; beyond, the chunked form at chunk length 256 (pinned to the recurrence in
    float64 by the CPU tier) -- never the kernel's own 128-step chunking."""
    def fn(e):
        a = (e["x"], e["dt"], e["A"], e["Bm"], e["Cm"], e["D"], e["dt_bias"], seq_len)
        if seq_len <= 1024:
            return TK.ssd_scan_fwd(*a, 0, softplus)
        return TK.ssd_scan_chunked(*a, 256, softplus)
    return fn


def ssd_kernel(CK, d, seq_len, dy=None, softplus=True):
    a = (d["x"], d["dt"], d["A"], d["Bm"], d["Cm"], d["D"], d["dt_bias"], seq_len, 256)
    if dy is None:
        return CK.ssd_scan_fwd(*a, dt_softplus=softplus)
    g = CK.ssd_scan_bwd(dy, *a, dt_softplus=softplus)
    return dict(zip(SSD_KEYS, g))


SSD_CASES = [   # regime, batch, S, H, P, G, N, options
    ("init", 1, 128, 4, 32, 1, 16, {}),
    ("slow", 3, 1024, 4, 64, 2, 32, {}),
    ("init", 1, 1024, 4, 128, 4, 128, {}),                 # G = H: one head per group
    ("fast", 3, 1024, 8, 64, 1, 128, {}),
    ("slow", 3, 1024, 4, 64, 1, 64, {"use_D": False}),
    ("init", 1, 1024, 4, 32, 2, 16, {"use_bias": False}),
    ("slow", 3, 4096, 4, 64, 2, 32, {}),
    ("init", 1, 4096, 80, 64, 1, 128, {}),                 # mamba_2.8b mixer
    ("slow", 1, 4096, 128, 64, 1, 128, {}),                # mamba_9.8b mixer
]


@pytest.mark.parametrize("case", SSD_CASES, ids=lambda c: f"{c[0]}-b{c[1]}-S{c[2]}-H{c[3]}-P{c[4]}-G{c[5]}-N{c[6]}"
                         + "".join(f"-{k}" for k in c[7]))
def test_ssd_scan_vs_reference_with_carry_and_adjoint_probes(K, case):
    CK, TK = K
    regime, Bsz, S, H, P, G, N, opts = case
    d = ssd_inputs(regime, Bsz, S, H, P, G, N, seed=S + H + P + G + N, **opts)
    keys = [k for k in SSD_KEYS if d[k] is not None]
    nc = S // L_SSD
    if regime == "slow":
        v = F.softplus(d["dt"].float() + (0 if d["dt_bias"] is None else d["dt_bias"]))
        assert torch.exp((v * d["A"]).view(-1, L_SSD, H).sum(1)).min() > 0.5
    err = Errors(f"ssd[{regime},b{Bsz},S{S},H{H},P{P},G{G},N{N}{''.join(opts)}]")
    gen = torch.Generator(device=DEV).manual_seed(1)
    dy = torch.randn(Bsz * S, H, P, device=DEV, generator=gen).bfloat16()
    with Native(CK):
        y = ssd_kernel(CK, d, S)
        g = ssd_kernel(CK, d, S, dy)
    y0, g0 = ref_grads(ssd_ref(TK, S), d, keys, dy)
    err("y", y, y0, TOL_FWD)
    for k in keys:
        err("d" + k, g[k], g0[k], TOL_GRAD)
    if nc > 1:
        # carry probe: x only in chunk 0, y over chunks 1..n comes from the chunk-to-chunk state alone
        c = dict(d, x=d["x"] * rows(Bsz, S, 0, L_SSD)[:, None, None])
        with Native(CK):
            yc = ssd_kernel(CK, c, S)
        yc0, _ = ref_grads(ssd_ref(TK, S), c, [], None)
        later = rows(Bsz, S, L_SSD, S)
        err("carry y[chunks 1..]", yc, yc0, TOL_FWD, later)
        if regime != "fast":                                 # fast: nothing survives that far
            err("carry y[last chunk]", yc, yc0, TOL_FWD, rows(Bsz, S, S - L_SSD, S))
        # adjoint probe: dy only in the last chunk, gradients over the earlier chunks come from the reverse state pass
        last = rows(Bsz, S, S - L_SSD, S)
        dya = dy * last[:, None, None]
        with Native(CK):
            ga = ssd_kernel(CK, d, S, dya)
        _, ga0 = ref_grads(ssd_ref(TK, S), d, keys, dya)
        early = ~last
        for k in ("x", "dt", "Bm"):
            err(f"adjoint d{k}[early chunks]", ga[k], ga0[k], TOL_GRAD, early)
        # dC = dy . h vanishes where dy does: the kernel must leave nothing there
        err("adjoint dCm[early chunks]", ga["Cm"], ga0["Cm"], TOL_GRAD, early, scale=ga0["Cm"].abs().max())
        for k in ("A", "dt_bias"):
            if k in keys:
                err(f"adjoint d{k}", ga[k], ga0[k], TOL_GRAD)
    err.done()


def test_ssd_dt_zero_without_softplus(K):
    """``dt_softplus=False`` with steps whose dt is exactly 0 runs the counted ATen path: the kernels' backward recovers
    the intra-chunk dt gradient as a column sum divided by dt and would lose it at those steps.  The dt gradient there
    is right."""
    CK, TK = K
    S, H, P, G, N = 256, 4, 32, 1, 16
    d = ssd_inputs("slow", 1, S, H, P, G, N, seed=9, use_bias=False)
    zero = torch.zeros(S, H, dtype=torch.bool, device=DEV)
    zero[5::13] = True
    d["dt"] = F.softplus(d["dt"].float()).masked_fill(zero, 0.0).bfloat16()
    keys = [k for k in SSD_KEYS if d[k] is not None]
    gen = torch.Generator(device=DEV).manual_seed(2)
    dy = torch.randn(S, H, P, device=DEV, generator=gen).bfloat16()
    err = Errors("ssd[dt_softplus=False]")
    n0 = dict(CK.FALLBACKS)
    y = ssd_kernel(CK, d, S, softplus=False)
    g = ssd_kernel(CK, d, S, dy, softplus=False)
    for op in ("ssd_scan_chunked", "ssd_scan_bwd"):
        assert CK.FALLBACKS.get(op, 0) == n0.get(op, 0) + 1, op
    y0, g0 = ref_grads(ssd_ref(TK, S, False), d, keys, dy)
    err("y", y, y0, TOL_FWD)
    err("ddt at dt = 0", g["dt"], g0["dt"], TOL_GRAD, zero)
    err.done()


def test_ssd_batch_isolation(K):
    """Each sequence of a batch of 3 equals the same sequence run alone: the forward bit for bit (every tile and the state
    pass are per sequence, no atomics); per-row gradients within ``TOL_ISO`` (fp32 atomics in the mask backward);
    dA / d(dt_bias) of the batch equal the sum of the three within fp32 reordering."""
    CK, TK = K
    S, H, P, G, N = 512, 4, 64, 1, 32
    d = ssd_inputs("slow", 3, S, H, P, G, N, seed=4, use_D=False)
    gen = torch.Generator(device=DEV).manual_seed(3)
    dy = torch.randn(3 * S, H, P, device=DEV, generator=gen).bfloat16()
    err = Errors("ssd[batch isolation]")
    with Native(CK):
        yb = ssd_kernel(CK, d, S)
        gb = ssd_kernel(CK, d, S, dy)
        sums = {"A": 0, "dt_bias": 0}
        for i in range(3):
            sl = slice(i * S, (i + 1) * S)
            di = {k: (v[sl] if k in ("x", "dt", "Bm", "Cm") else v) for k, v in d.items()}
            yi = ssd_kernel(CK, di, S)
            gi = ssd_kernel(CK, di, S, dy[sl])
            assert bits_equal(yb[sl], yi), f"sequence {i}: batched forward differs from the sequence alone"
            for k in ("x", "dt", "Bm", "Cm"):
                err(f"seq{i} d{k}", gb[k][sl], gi[k], TOL_ISO)
            for k in sums:
                sums[k] = sums[k] + gi[k]
    for k in sums:
        err(f"d{k} batch = sum of sequences", gb[k], sums[k], 1e-4)
    err.done()


# --------------------------------------------------------------------------------------------- selective scan
SEL_KEYS = ("u", "delta", "A", "Bm", "Cm", "D", "z", "delta_bias")


def sel_ref(TK, seq_len, softplus=True):
    return lambda e: TK.selective_scan_fwd(e["u"], e["delta"], e["A"], e["Bm"], e["Cm"], e["D"], e["z"], e["delta_bias"],
                                            seq_len, softplus)


def sel_kernel(CK, d, seq_len, dy=None, softplus=True):
    a = (d["u"], d["delta"], d["A"], d["Bm"], d["Cm"], d["D"], d["z"], d["delta_bias"], seq_len, softplus)
    if dy is None:
        return CK.selective_scan_fwd(*a)
    g = CK.selective_scan_bwd(dy, *a)
    assert g is not None, "native selective-scan backward was not taken"
    du, dd, dA, dB, dC, dD, dz, ddb = g
    return dict(u=du, delta=dd, A=dA, Bm=dB, Cm=dC, D=dD, z=dz, delta_bias=ddb)


SEL_CASES = [   # regime, batch, S, Dm, z, D, delta_bias, softplus
    ("init", 3, 96, 96, True, True, True, True),
    ("init", 1, 2048, 5120, True, True, True, True),
    ("fast", 3, 32, 32, False, False, False, False),
    ("slow", 1, 2048, 96, True, False, True, True),
    ("init", 3, 96, 32, False, True, False, True),
    ("slow", 3, 96, 5120, True, True, True, False),
    ("fast", 1, 2048, 32, True, True, True, True),
]


@pytest.mark.parametrize("case", SEL_CASES, ids=lambda c: f"{c[0]}-b{c[1]}-S{c[2]}-Dm{c[3]}"
                         + "".join(f"-{n}" for n, on in zip(("z", "D", "bias", "softplus"), c[4:]) if on))
def test_selective_scan_vs_reference_with_block_probes(K, case):
    CK, TK = K
    regime, Bsz, S, Dm, use_z, use_D, use_bias, sp = case
    d = sel_inputs(regime, Bsz, S, Dm, seed=S + Dm, use_z=use_z, use_D=use_D, use_bias=use_bias, softplus=sp)
    keys = [k for k in SEL_KEYS if d[k] is not None]
    err = Errors(f"selscan[{regime},b{Bsz},S{S},Dm{Dm},z{int(use_z)},D{int(use_D)},bias{int(use_bias)},sp{int(sp)}]")
    gen = torch.Generator(device=DEV).manual_seed(1)
    dy = torch.randn(Bsz * S, Dm, device=DEV, generator=gen).bfloat16()
    with Native(CK):
        y = sel_kernel(CK, d, S, softplus=sp)
        g = sel_kernel(CK, d, S, dy, softplus=sp)
    y0, g0 = ref_grads(sel_ref(TK, S, sp), d, keys, dy)
    err("y", y, y0, TOL_FWD)
    for k in keys:
        err("d" + k, g[k], g0[k], TOL_GRAD)
    if S > L_SEL and regime != "fast":
        c = dict(d, u=d["u"] * rows(Bsz, S, 0, L_SEL)[:, None])
        with Native(CK):
            yc = sel_kernel(CK, c, S, softplus=sp)
        yc0, _ = ref_grads(sel_ref(TK, S, sp), c, [], None)
        err("carry y[blocks 1..]", yc, yc0, TOL_FWD, rows(Bsz, S, L_SEL, S))
        last = rows(Bsz, S, S - L_SEL, S)
        dya = dy * last[:, None]
        with Native(CK):
            ga = sel_kernel(CK, d, S, dya, softplus=sp)
        _, ga0 = ref_grads(sel_ref(TK, S, sp), d, keys, dya)
        for k in ("u", "delta", "Bm"):
            err(f"adjoint d{k}[early blocks]", ga[k], ga0[k], TOL_GRAD, ~last)
        for k in ("A", "delta_bias"):
            if k in keys:
                err(f"adjoint d{k}", ga[k], ga0[k], TOL_GRAD)
    err.done()


def test_selective_scan_batch_isolation(K):
    CK, TK = K
    S, Dm = 128, 96
    d = sel_inputs("slow", 3, S, Dm, seed=6, use_D=False)
    gen = torch.Generator(device=DEV).manual_seed(4)
    dy = torch.randn(3 * S, Dm, device=DEV, generator=gen).bfloat16()
    err = Errors("selscan[batch isolation]")
    per_row = ("u", "delta", "Bm", "Cm", "z")
    with Native(CK):
        yb = sel_kernel(CK, d, S)
        gb = sel_kernel(CK, d, S, dy)
        sums = {"A": 0, "delta_bias": 0}
        for i in range(3):
            sl = slice(i * S, (i + 1) * S)
            di = {k: (v[sl] if k in per_row else v) for k, v in d.items()}
            yi = sel_kernel(CK, di, S)
            gi = sel_kernel(CK, di, S, dy[sl])
            assert bits_equal(yb[sl], yi), f"sequence {i}: batched forward differs from the sequence alone"
            for k in per_row:
                err(f"seq{i} d{k}", gb[k][sl], gi[k], TOL_ISO)
            for k in sums:
                sums[k] = sums[k] + gi[k]
    for k in sums:
        err(f"d{k} batch = sum of sequences", gb[k], sums[k], 1e-4)
    err.done()


# ------------------------------------------------------------------------------------------------- conv1d
@pytest.mark.parametrize("C", [8, 1032, 5376, 8448])
@pytest.mark.parametrize("S", [1, 3, 63, 64, 65, 4096])
def test_conv1d_kernel_widths_bias_activation(K, S, C):
    """K in {2, 3, 4}, bias on / off, SiLU on / off; S crosses the 64-step CTA chunks and the backward's K - 1 halo; C
    leaves the last CTA partly idle (5376 = mamba_2.8b conv_dim, 8448 = mamba_9.8b)."""
    CK, TK = K
    Bsz = 1 if S * C > 4096 * 1032 else 2
    gen = torch.Generator(device=DEV).manual_seed(S * 7 + C)
    x = torch.randn(Bsz * S, C, device=DEV, generator=gen).bfloat16()
    dy = torch.randn(Bsz * S, C, device=DEV, generator=gen).bfloat16()
    err = Errors(f"conv1d[S{S},C{C}]")
    for Kw in (2, 3, 4):
        w = (0.5 * torch.randn(C, Kw, device=DEV, generator=gen)).bfloat16()
        bias = (0.1 * torch.randn(C, device=DEV, generator=gen)).bfloat16()
        for b in (bias, None):
            for act in (True, False):
                tag = f"K{Kw}{'-bias' if b is not None else ''}{'-silu' if act else ''}"
                with Native(CK):
                    y = CK.causal_conv1d_fwd(x, w, b, S, act)
                    dx, dw, db = CK.causal_conv1d_bwd(dy, x, w, b, S, act)
                bf = None if b is None else b.float()
                y0 = TK.causal_conv1d_fwd(x.float(), w.float(), bf, S, act)
                dx0, dw0, db0 = TK.causal_conv1d_bwd(dy.float(), x.float(), w.float(), bf, S, act)
                err(f"{tag} y", y, y0, 1e-2)
                err(f"{tag} dx", dx, dx0, 1e-2)
                err(f"{tag} dw", dw, dw0, 1e-3)
                if b is not None:
                    err(f"{tag} db", db, db0, 1e-3)
                else:
                    assert db is None
    err.done()


def test_conv1d_batch_isolation(K):
    """Forward and dx of each sequence bit-identical to the sequence alone (no atomics; the window starts at zero at
    every sequence start, across a 64-step CTA boundary too)."""
    CK, _ = K
    S, C = 100, 1032
    gen = torch.Generator(device=DEV).manual_seed(8)
    x = torch.randn(3 * S, C, device=DEV, generator=gen).bfloat16()
    dy = torch.randn(3 * S, C, device=DEV, generator=gen).bfloat16()
    w = (0.5 * torch.randn(C, 4, device=DEV, generator=gen)).bfloat16()
    b = (0.1 * torch.randn(C, device=DEV, generator=gen)).bfloat16()
    with Native(CK):
        yb = CK.causal_conv1d_fwd(x, w, b, S, True)
        dxb, dwb, dbb = CK.causal_conv1d_bwd(dy, x, w, b, S, True)
        dws, dbs = 0, 0
        for i in range(3):
            sl = slice(i * S, (i + 1) * S)
            assert bits_equal(yb[sl], CK.causal_conv1d_fwd(x[sl], w, b, S, True)), i
            dxi, dwi, dbi = CK.causal_conv1d_bwd(dy[sl], x[sl], w, b, S, True)
            assert bits_equal(dxb[sl], dxi), i
            dws, dbs = dws + dwi, dbs + dbi
    assert (dwb - dws).abs().max() <= 1e-4 * dws.abs().max() and (dbb - dbs).abs().max() <= 1e-4 * dbs.abs().max()


# -------------------------------------------------------------------------------------------------- norms
def norm_rows(M, D, gen, scale=1.0):
    """Rows of N(0, scale); row 1 near zero (eps dominates its rstd)."""
    t = torch.randn(M, D, device=DEV, generator=gen) * scale
    if M >= 3:
        t[1] *= 1e-4
    return t


@pytest.mark.parametrize("M", [1, 3, 600, 4096])
@pytest.mark.parametrize("D", [8, 2560, 4096, 5120, 8192])
def test_add_rmsnorm_and_gated_rmsnorm_kernels(K, D, M):
    """fp32-residual add + RMSNorm forward (``res_out`` bit-exact), its fp32-input backward, and the gated RMSNorm
    forward / backward against float64 autograd of the formula.  D = 8192 fills every register chunk; M > 528 runs the
    grid-stride loop and several dw partial rows; a near-zero row and a row of |z| ~ 30 are included."""
    CK, _ = K
    eps = 1e-5
    gen = torch.Generator(device=DEV).manual_seed(D + M)
    x = norm_rows(M, D, gen).bfloat16()
    res = norm_rows(M, D, gen, 2.0)
    w = (1 + 0.1 * torch.randn(D, device=DEV, generator=gen)).bfloat16()
    dy = torch.randn(M, D, device=DEV, generator=gen).bfloat16()
    z = torch.randn(M, D, device=DEV, generator=gen)
    z[0] = 30 * torch.sign(z[0])
    z = z.bfloat16()
    err = Errors(f"norm[D{D},M{M}]")

    with Native(CK):
        y, res_out, rstd = CK.add_rmsnorm_fwd(x, res, w, eps)
        dx, dw = CK.rmsnorm_bwd(dy, res_out, w, rstd)
    assert bits_equal(res_out, res + x.float())
    r = (res.double() + x.double()).requires_grad_()
    w64 = w.double().requires_grad_()
    rs = torch.rsqrt(r.pow(2).mean(-1, keepdim=True) + eps)
    y0 = r * rs * w64
    dx0, dw0 = torch.autograd.grad(y0, [r, w64], dy.double())
    err("add_rmsnorm y", y, y0, 1e-2)
    err("add_rmsnorm rstd", rstd, rs.squeeze(-1), 1e-4)
    err("rmsnorm_bwd_f32 dx", dx, dx0, 1e-3)
    err("rmsnorm_bwd_f32 dw", dw, dw0, 1e-3)

    with Native(CK):
        yg, rg = CK.rmsnorm_gated_fwd(x, z, w, eps, D)
        dxg, dzg, dwg = CK.rmsnorm_gated_bwd(dy, x, z, w, rg, D)
    x64, z64, w64 = (t.double().requires_grad_() for t in (x, z, w))
    uu = x64 * F.silu(z64)
    rs = torch.rsqrt(uu.pow(2).mean(-1, keepdim=True) + eps)
    yg0 = uu * rs * w64
    dxg0, dzg0, dwg0 = torch.autograd.grad(yg0, [x64, z64, w64], dy.double())
    err("gated y", yg, yg0, 1e-2)
    err("gated rstd", rg.reshape(-1), rs.reshape(-1), 1e-4)
    err("gated dx", dxg, dxg0, 1e-2)
    err("gated dz", dzg, dzg0, 1e-2)
    err("gated dw", dwg, dwg0, 1e-3)
    err.done()


@pytest.mark.parametrize("D,M", [(2560, 600), (8192, 3), (8200, 5)])
def test_norm_ops_through_autograd(K, D, M):
    """``ops.add_rmsnorm`` and ``ops.rmsnorm_gated`` (the model's entry points) against float64 autograd; D = 8200 is past
    the register cache and must take the counted ATen fallback, still correct."""
    CK, _ = K
    from fms_fsdp_b200 import ops
    eps = 1e-5
    gen = torch.Generator(device=DEV).manual_seed(D)
    x = norm_rows(M, D, gen).bfloat16().requires_grad_()
    res = norm_rows(M, D, gen, 2.0).requires_grad_()
    z = torch.randn(M, D, device=DEV, generator=gen).bfloat16().requires_grad_()
    w = torch.nn.Parameter((1 + 0.1 * torch.randn(D, device=DEV, generator=gen)).bfloat16())
    wg = torch.nn.Parameter((1 + 0.1 * torch.randn(D, device=DEV, generator=gen)).bfloat16())
    gy, gr, gg = (torch.randn(M, D, device=DEV, generator=gen) for _ in range(3))
    f0, n0 = CK.fallback_count(), CK.launch_count()
    y, r_out = ops.add_rmsnorm(x, res, w, eps)
    yg = ops.rmsnorm_gated(x, z, wg, eps)
    ((y.float() * gy).sum() + (r_out * gr).sum() + (yg.float() * gg).sum()).backward()
    if D <= 8192:
        assert CK.fallback_count() == f0 and CK.launch_count() > n0
    else:
        assert CK.fallback_count() >= f0 + 4      # add_rmsnorm_fwd, rmsnorm_bwd, rmsnorm_gated_fwd / _bwd
    x64, r64, z64, w64, wg64 = (t.detach().double().requires_grad_() for t in (x, res, z, w, wg))
    ro = r64 + x64
    y0 = ro * torch.rsqrt(ro.pow(2).mean(-1, keepdim=True) + eps) * w64
    uu = x64 * F.silu(z64)
    yg0 = uu * torch.rsqrt(uu.pow(2).mean(-1, keepdim=True) + eps) * wg64
    loss = (y0 * gy.double()).sum() + (ro * gr.double()).sum() + (yg0 * gg.double()).sum()
    gx0, gr0, gz0, gw0, gwg0 = torch.autograd.grad(loss, [x64, r64, z64, w64, wg64])
    err = Errors(f"ops norms[D{D},M{M}]")
    err("y", y, y0, 1e-2)
    err("res_out", r_out, ro, 1e-6)
    err("yg", yg, yg0, 1e-2)
    err("dx", x.grad, gx0, 1e-2)
    err("dres", res.grad, gr0, 1e-2)
    err("dz", z.grad, gz0, 1e-2)
    err("dw", w.grad, gw0, 1e-2)
    err("dw gated", wg.grad, gwg0, 1e-2)
    err.done()


# ------------------------------------------------------------------------------------------------- engine
def test_engine_mamba1_fused_kernels_match_aten_path():
    """``mamba1_tiny`` (selective-scan mixers, conv1d, fp32 residual stream) trained through the sharded engine on the
    sm_90a kernels against the ATen kernel path: same losses and grad norms, and no ATen fallback on the fused path."""
    from fms_fsdp_b200.models.mamba import MambaConfig, MambaLMHeadModel
    from fms_fsdp_b200.ops import cuda_kernels as CK
    from fms_fsdp_b200.ops import set_kernel_path
    from fms_fsdp_b200.parallel import ShardedAdamW, ShardedModel
    from fms_fsdp_b200.policies import bfSixteen
    from fms_fsdp_b200.utils.config_utils import get_model_config

    def run(path):
        set_kernel_path(path)
        torch.manual_seed(0); torch.cuda.manual_seed(0)
        with torch.device("meta"):
            m = MambaLMHeadModel(MambaConfig(**get_model_config("mamba1_tiny")))
        eng = ShardedModel(m, mixed_precision=bfSixteen, device=torch.device("cuda", 0))
        opt = ShardedAdamW(eng, lr=1e-3)
        out = []
        for st in range(4):
            x = torch.randint(0, 512, (2, 256), generator=torch.Generator().manual_seed(3 + st)).cuda()
            l = eng.forward_backward(x, x); g = eng.clip_grad_norm_(1.0); opt.step(); out.append((l.item(), g.item()))
        return out
    try:
        f0, n0 = dict(CK.FALLBACKS), CK.launch_count()
        fused = run("fused")
        assert CK.launch_count() - n0 > 100
        assert dict(CK.FALLBACKS) == f0, {k: v for k, v in CK.FALLBACKS.items() if v != f0.get(k, 0)}
        aten = run("torch")
    finally:
        set_kernel_path("auto")
    for (lf, gf), (la, ga) in zip(fused, aten):
        print(f"MEASURE engine mamba1_tiny: loss {lf:.5f} vs {la:.5f}, grad norm {gf:.4f} vs {ga:.4f}")
        assert abs(lf - la) < 3e-2 * abs(la) and abs(gf - ga) < 6e-2 * abs(ga)
    assert fused[-1][0] < fused[0][0]
