"""Elementwise sweeps of the pointwise transcendentals against fp64, over every finite bf16 input where the op has one
input, and over dense ranges of the saturated tails where it has more.

The kernel tests elsewhere feed randn data and judge an error relative to the RMS of the whole tensor.  Almost no
unit-normal element lands where a sigmoid or an erf saturates, so a systematic error there (an absolute error the size
of the value itself, an overflow to inf or NaN at the ends of the range) does not move that measure.  Here every
element is held to

    |got - ref| <= 2 ulp_bf16(ref) + 2^-20

and where the fp64 value rounds to +-inf in bf16 the kernel must return the same inf.  Each test prints the worst
error as a multiple of that bound and in bf16 ulps.
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

F64 = torch.float64
BF16 = torch.bfloat16
ABS = 2.0 ** -20
QUICK = 1.702


def all_finite_bf16():
    """Every finite bf16 value (65 280 of them, both zeros included), padded with zeros to a multiple of 8."""
    bits = torch.arange(-(1 << 15), 1 << 15, dtype=torch.int32).to(torch.int16)
    x = bits.view(BF16)
    x = x[torch.isfinite(x)]
    pad = (-x.numel()) % 8
    return torch.cat([x, torch.zeros(pad, dtype=BF16)]).cuda()


def ulp_bf16(r):
    """The spacing of bf16 values at |r| (fp64 tensor): 2^(e - 7) with e = floor(log2 |r|), subnormals at 2^-133."""
    e = torch.floor(torch.log2(r.abs().clamp_min(2.0 ** -126)))
    return torch.exp2(e - 7)


def check(label, got, ref, extra=None):
    """Holds got (bf16) to ref (fp64) elementwise; extra (fp64, same shape) widens the bound where a derived input
    error applies.  Returns the worst error as a multiple of the bound."""
    got, ref = got.reshape(-1), ref.reshape(-1).to(F64)
    assert torch.isfinite(ref).all(), f"{label}: the fp64 reference is not finite"
    ref16 = ref.to(torch.float32).to(BF16)
    inf = torch.isinf(ref16)
    bad_inf = int((got[inf] != ref16[inf]).sum())
    g, r = got[~inf].to(F64), ref[~inf]
    bound = 2 * ulp_bf16(r) + ABS
    if extra is not None:
        bound = bound + extra.reshape(-1)[~inf]
    err = (g - r).abs()
    ratio = torch.where(torch.isfinite(g), err / bound, torch.full_like(err, math.inf))
    i = int(ratio.argmax())
    worst = ratio[i].item()
    big = torch.isfinite(g) & (r.abs() >= 2.0 ** -12)     # where the ulp term of the bound dominates
    ulps = ((g - r).abs() / ulp_bf16(r))[big].max().item() if bool(big.any()) else 0.0
    print(f"[{label}] worst {worst:.3f}x the bound ({ulps:.2f} bf16 ulps at most where |ref| >= 2^-12) at ref "
          f"{r[i].item():.6e} "
          f"got {g[i].item():.6e}; {int(inf.sum())} inf references, {bad_inf} mismatched")
    assert bad_inf == 0, f"{label}: {bad_inf} elements whose fp64 value rounds to inf in bf16 are not that inf"
    assert worst <= 1.0, (f"{label}: |got - ref| = {err[i].item():.3e} > bound {bound[i].item():.3e} at ref "
                          f"{r[i].item():.6e} (got {g[i].item():.6e})")
    return worst


# ---------------------------------------------------------------------------------------------------------------------
# GELU / quick-GELU / LeakyReLU (small_ops.cu act_*) and GEGLU (elementwise.cu)
# ---------------------------------------------------------------------------------------------------------------------
def act_ref(x, mode):
    if mode == 0:
        return 0.5 * x * (1 + torch.erf(x / math.sqrt(2)))
    if mode == 1:
        return x * torch.sigmoid(QUICK * x)
    return torch.where(x > 0, x, 0.01 * x)


def act_grad_ref(x, mode):
    if mode == 0:
        return 0.5 * (1 + torch.erf(x / math.sqrt(2))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)
    if mode == 1:
        s = torch.sigmoid(QUICK * x)
        # s + 1.702 x s (1 - s), written so that x * s * (1 - s) stays finite at the ends of the range
        return s + QUICK * x * (s * torch.sigmoid(-QUICK * x))
    return torch.where(x > 0, torch.ones_like(x), torch.full_like(x, 0.01))


@pytest.mark.parametrize("mode", [0, 1, 2], ids=["gelu", "quick_gelu", "leaky_relu"])
def test_act_every_bf16(mode):
    from e4t_b200 import ops
    x = all_finite_bf16()
    xd = x.to(F64)
    check(f"act_fwd mode {mode}", ops.act_fwd(x, mode), act_ref(xd, mode))
    one = torch.ones_like(x)
    check(f"act_bwd mode {mode}, dy = 1", ops.act_bwd(x, one, mode), act_grad_ref(xd, mode))
    g = torch.Generator(device="cuda").manual_seed(mode)
    dy = torch.randn(x.shape, generator=g, device="cuda").to(BF16)
    check(f"act_bwd mode {mode}, random dy", ops.act_bwd(x, dy, mode), dy.to(F64) * act_grad_ref(xd, mode))


@pytest.mark.parametrize("linear", ["one", "random"])
def test_geglu_every_bf16_gate(linear):
    from e4t_b200 import ops
    gate = all_finite_bf16()
    Fd = 1024
    n = gate.numel()
    rows = -(-n // Fd)
    gate = torch.cat([gate, torch.zeros(rows * Fd - n, dtype=BF16, device="cuda")]).view(rows, Fd)
    g = torch.Generator(device="cuda").manual_seed(7)
    if linear == "one":
        u = torch.ones_like(gate)
    else:
        u = torch.randn(gate.shape, generator=g, device="cuda").to(BF16)
    h = torch.cat([u, gate], -1).contiguous()
    dout = torch.randn(u.shape, generator=g, device="cuda").to(BF16)
    ud, gd, dd = u.to(F64), gate.to(F64), dout.to(F64)
    check(f"geglu_fwd, linear {linear}", ops.geglu_fwd(h), ud * act_ref(gd, 0))
    dh = ops.geglu_bwd(h, dout)
    check(f"geglu_bwd du, linear {linear}", dh[:, :Fd], dd * act_ref(gd, 0))
    check(f"geglu_bwd dgate, linear {linear}", dh[:, Fd:], dd * ud * act_grad_ref(gd, 0))


# ---------------------------------------------------------------------------------------------------------------------
# softmax_rows (softmax.cu): peaked, sink and ramp rows, register kernel (n <= 16384) and two-pass kernel (longer)
# ---------------------------------------------------------------------------------------------------------------------
def peaked_rows(n, g):
    """fp32 score rows: spreads of 1, 3 and 6 nats, each alone and with a sink Δ = 8, 24, 48 nats above the row's
    max at a random column (the first and last columns among them), plus rising and falling ramps that span 60 nats."""
    rows = []
    for sigma in (1.0, 3.0, 6.0):
        base = torch.randn(n, generator=g, device="cuda") * sigma
        rows.append(base.clone())
        for j, delta in enumerate((8.0, 24.0, 48.0)):
            r = base.clone()
            col = (0, n - 1, int(torch.randint(0, n, (1,), generator=g, device="cuda")))[j]
            r[col] = base.max() + delta
            rows.append(r)
    ramp = torch.linspace(-30.0, 30.0, n, device="cuda")
    rows += [ramp, ramp.flip(0)]
    return torch.stack(rows)


@pytest.mark.parametrize("n", [4, 4096, 16384, 16388, 17408, 24576, 36864])
def test_softmax_rows_peaked(n):
    from e4t_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(n)
    x = peaked_rows(n, g)
    ld = n + 12                                  # strided rows: the kernel must keep to its own n columns
    xs = torch.full((x.shape[0], ld), float("nan"), device="cuda")
    xs[:, :n] = x
    out = torch.full((x.shape[0], ld), float("nan"), device="cuda", dtype=BF16)
    ops.softmax_rows(xs[:, :n], out=out[:, :n])
    assert out[:, n:].isnan().all(), "softmax_rows wrote past its row"
    check(f"softmax_rows n={n}", out[:, :n], torch.softmax(x.to(F64), -1))


# ---------------------------------------------------------------------------------------------------------------------
# GroupNorm + SiLU (norm.cu)
# ---------------------------------------------------------------------------------------------------------------------
B, HW, C, G, EPS = 2, 64 * 64, 320, 32, 1e-5


def _gn_inputs(seed, gamma_lo, gamma_hi, beta_lo, beta_hi):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn((B, HW, C), generator=g, device="cuda").clamp(-3, 3) * 2.0 + 0.5).to(BF16)
    gamma = torch.rand(C, generator=g, device="cuda") * (gamma_hi - gamma_lo) + gamma_lo
    beta = torch.rand(C, generator=g, device="cuda") * (beta_hi - beta_lo) + beta_lo
    return x, gamma, beta


def _gn_exact(x, gamma, beta):
    """fp64 mean and rstd per (image, group), and y = x̂ γ + β, all (B, HW, C)."""
    xd = x.to(F64).view(B, HW, G, C // G)
    mean = xd.mean((1, 3), keepdim=True)
    rstd = (xd.var((1, 3), unbiased=False, keepdim=True) + EPS).rsqrt()
    xh = ((xd - mean) * rstd).view(B, HW, C)
    return mean, rstd, xh, xh * gamma.to(F64) + beta.to(F64)


def _silu_grad(y):
    s = torch.sigmoid(y)
    return s * (1 + y * (1 - s))


def test_groupnorm_silu_forward_tails():
    """y = x̂ γ + β covers about [-36, 36] densely; the output is held elementwise to silu(y) in fp64, widened by
    |silu'(y)| times the error of the fp32 y the kernel forms from its statistics."""
    from e4t_b200 import ops
    x, gamma, beta = _gn_inputs(3, 1.0, 8.0, -12.0, 12.0)
    out, stats = ops.groupnorm_fwd(x, gamma, beta, G, EPS, True)
    mean, rstd, xh, y = _gn_exact(x, gamma, beta)
    print(f"[groupnorm silu fwd] x̂ in [{xh.min().item():.2f}, {xh.max().item():.2f}], y in "
          f"[{y.min().item():.2f}, {y.max().item():.2f}]")
    # a priori error of the fp32 statistics: Σ(x - p) and Σ(x - p)² over n elements (p = the group's first element)
    # are fp32 sums, held to sqrt(n)·u32 times the sum of their terms' magnitudes (the statistical bound of accumulated
    # rounding, not the worst case n·u32); the kernel's mean and rstd
    # (from its stats as gn_mean_rstd, common.cuh, forms them) must be within that of fp64
    u32 = 2.0 ** -24
    n = HW * (C // G)
    xg = x.to(F64).view(B, HW, G, C // G)
    dlt = xg - xg[:, :1, :, :1]
    s1, s2 = dlt.abs().sum((1, 3), keepdim=True), dlt.pow(2).sum((1, 3), keepdim=True)
    dm_ap = math.sqrt(n) * u32 * s1 / n + 2 * u32 * mean.abs()
    dvar = math.sqrt(n) * u32 * s2 / n + 2 * (dlt.sum((1, 3), keepdim=True) / n).abs() * dm_ap
    dr_ap = dvar * rstd.pow(2) / 2 + 2 * u32                           # relative error of rstd = (var + eps)^-1/2
    st = stats.to(F64)
    d = st[..., 1] / n
    m_k = (st[..., 0] + d).view(B, 1, G, 1)
    r_k = ((st[..., 2] / n - d * d).clamp_min(0) + EPS).rsqrt().view(B, 1, G, 1)
    print(f"[groupnorm silu fwd] |Δmean| {((m_k - mean).abs() / dm_ap).max().item():.2f}x, |Δrstd|/rstd "
          f"{((r_k - rstd).abs() / rstd / dr_ap).max().item():.2f}x their a priori bounds")
    assert bool(((m_k - mean).abs() <= dm_ap).all()), "groupnorm mean outside its fp32 error bound"
    assert bool(((r_k - rstd).abs() <= dr_ap * rstd).all()), "groupnorm rstd outside its fp32 error bound"
    per_chan = lambda t: t.expand(B, HW, G, C // G).reshape(B, HW, C)
    g64, b64 = gamma.to(F64).abs(), beta.to(F64).abs()
    scale = per_chan(rstd) * g64
    # y = fma(x, scale, shift) with shift = β - mean·scale: the statistics' a priori error through x̂ γ, plus the fp32
    # roundings of scale, mean·scale, shift and the fma, each at most one unit in the last place of its operand
    y_err = (per_chan(dm_ap) * scale + xh.abs() * g64 * per_chan(dr_ap)
             + 4 * u32 * ((x.to(F64) * scale).abs() + b64 + (per_chan(mean) * scale).abs() + y.abs()))
    print(f"[groupnorm silu fwd] fp32 error of y ≤ {y_err.max().item():.2e}")
    check("groupnorm_fwd silu, y in [-36, 36]", out, F.silu(y), _silu_grad(y).abs() * y_err)


def test_groupnorm_silu_backward_saturated():
    """Every y in [-12, -3], where silu' is small and the sigmoid's tail decides dx: the 4e-3 RMS bound of the kernel
    tests, per (image, group), now measures that tail."""
    from e4t_b200 import ops
    x, gamma, beta = _gn_inputs(4, 0.5, 1.5, -7.5, -7.5)
    _, _, xh, y = _gn_exact(x, gamma, beta)
    assert y.min().item() >= -12.01 and y.max().item() <= -2.99, (y.min().item(), y.max().item())
    g = torch.Generator(device="cuda").manual_seed(5)
    dy = torch.randn(x.shape, generator=g, device="cuda").to(BF16)
    _, stats = ops.groupnorm_fwd(x, gamma, beta, G, EPS, True)
    dx = ops.groupnorm_bwd(x, dy, gamma, beta, stats, G, EPS, True)
    xr = x.to(F64).permute(0, 2, 1).requires_grad_(True)
    yr = F.silu(F.group_norm(xr, G, gamma.to(F64), beta.to(F64), EPS))
    yr.backward(dy.to(F64).permute(0, 2, 1))
    ref = xr.grad.permute(0, 2, 1)
    err = (dx.to(F64) - ref).view(B, HW, G, C // G)
    r = ref.view(B, HW, G, C // G)
    glob = (err.pow(2).mean().sqrt() / r.pow(2).mean().sqrt()).item()
    per_group = (err.pow(2).mean((1, 3)).sqrt() / r.pow(2).mean().sqrt()).max().item()
    print(f"[groupnorm silu bwd, y in [-12, -3]] rms error {glob:.2e} (bound 4e-3), worst (image, group) "
          f"{per_group:.2e} (bound 1.6e-2)")
    assert torch.isfinite(dx).all()
    assert glob <= 4e-3 and per_group <= 4 * 4e-3, (glob, per_group)
