"""GPU parity of the HBM-bound kernels and the attention core (through the C-ABI) against fp32 torch restatements of
the same ops evaluated on the same bf16-representable inputs.  Tolerances are relative to the output RMS:
bf16-stored outputs carry one rounding (2^-9 ~ 2e-3 rms), so 4e-3; fp32 outputs 1e-3 or tighter as written."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False


def _rel(a, b):
    a = a.float(); b = b.float()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt().clamp_min(1e-20)).item()


def _mk(shape, g, scale=1.0, shift=0.0):
    return (torch.randn(shape, generator=g, device="cuda") * scale + shift).to(torch.bfloat16)


@pytest.mark.parametrize("B,HW,C", [(2, 4096, 320), (2, 1024, 640), (3, 256, 1920), (2, 64, 2560), (2, 256, 64)])
@pytest.mark.parametrize("silu", [False, True])
def test_groupnorm(B, HW, C, silu):
    from e4t_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(C + HW)
    x = _mk((B, HW, C), g, 1.5, 0.3)
    gamma = torch.randn(C, generator=g, device="cuda") * 0.3 + 1
    beta = torch.randn(C, generator=g, device="cuda") * 0.2
    dy = _mk((B, HW, C), g)
    xr = x.float().permute(0, 2, 1).requires_grad_(True)
    yr = F.group_norm(xr, 32, gamma, beta, 1e-5)
    if silu:
        yr = F.silu(yr)
    yr.backward(dy.float().permute(0, 2, 1))
    y, stats = ops.groupnorm_fwd(x, gamma, beta, 32, 1e-5, silu)
    assert _rel(y.permute(0, 2, 1), yr) < 4e-3
    dx = ops.groupnorm_bwd(x, dy, gamma, beta, stats, 32, 1e-5, silu)
    assert _rel(dx.permute(0, 2, 1), xr.grad) < 4e-3


@pytest.mark.parametrize("rows,C", [(4096, 320), (777, 640), (300, 1280), (64, 768), (100, 64)])
def test_layernorm(rows, C):
    from e4t_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(C + rows)
    x = _mk((rows, C), g, 2.0, 0.5)
    gamma = torch.randn(C, generator=g, device="cuda") * 0.3 + 1
    beta = torch.randn(C, generator=g, device="cuda") * 0.2
    dy = _mk((rows, C), g)
    xr = x.float().requires_grad_(True)
    yr = F.layer_norm(xr, (C,), gamma, beta, 1e-5)
    yr.backward(dy.float())
    y, stats = ops.layernorm_fwd(x, gamma, beta, 1e-5)
    assert _rel(y, yr) < 4e-3
    dx = ops.layernorm_bwd(x, dy, gamma, stats, 1e-5)
    assert _rel(dx, xr.grad) < 4e-3


# Inputs bf16(mu + sd * randn) with a large mean against the spread, as trained checkpoints produce (SD's VAE decoder is
# known for them): mu / sd = 0, 16, 64, 256, and nearly constant groups (sd 0.01 around 3).  Past ~256 bf16 itself
# erases the spread (its spacing at 256 is 2).  The reference is fp64 on the same bf16 values.
_OFFSETS = [(0.0, 1.0), (16.0, 1.0), (64.0, 1.0), (256.0, 1.0), (3.0, 0.01)]
_OFFSET_IDS = ["mu0", "mu16", "mu64", "mu256", "const3"]


def _ratio(x, dims):
    """Largest |mean| / std of x's groups (reduced over dims), measured on the bf16 values."""
    xd = x.double()
    return (xd.mean(dims).abs() / xd.std(dims).clamp_min(1e-30)).max().item()


@pytest.mark.parametrize("mu,sd", _OFFSETS, ids=_OFFSET_IDS)
@pytest.mark.parametrize("B,HW,C", [(2, 4096, 320), (1, 512 * 512, 128), (2, 64, 1280)],
                         ids=["unet_level0", "vae_512", "c1280_8x8"])
@pytest.mark.parametrize("silu", [False, True])
def test_groupnorm_offset(B, HW, C, silu, mu, sd):
    """GroupNorm(+SiLU) forward, dx and the affine gradients against fp64 torch when a group's mean is large against
    its spread: the statistics must not cancel (E[x^2] - mean^2 in fp32 loses all digits at mu / sd ~ 256)."""
    from e4t_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(C + HW + int(mu))
    x = _mk((B, HW, C), g, sd, mu)
    gamma = torch.randn(C, generator=g, device="cuda") * 0.3 + 1
    beta = torch.randn(C, generator=g, device="cuda") * 0.2
    dy = _mk((B, HW, C), g)
    ratio = _ratio(x.view(B, HW, 32, C // 32), (1, 3))
    xr = x.double().permute(0, 2, 1).requires_grad_(True)
    gr, br = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    yr = F.group_norm(xr, 32, gr, br, 1e-5)
    if silu:
        yr = F.silu(yr)
    yr.backward(dy.double().permute(0, 2, 1))
    y, stats = ops.groupnorm_fwd(x, gamma, beta, 32, 1e-5, silu)
    dx = ops.groupnorm_bwd(x, dy, gamma, beta, stats, 32, 1e-5, silu)
    dg, db = ops.groupnorm_param_grad(x, dy, stats, gamma, beta, 32, 1e-5, silu)
    errs = dict(y=_rel(y.permute(0, 2, 1), yr), dx=_rel(dx.permute(0, 2, 1), xr.grad), dgamma=_rel(dg, gr.grad),
                dbeta=_rel(db, br.grad))
    print(f"[groupnorm {B}x{HW}x{C} silu={silu} mu/sd={ratio:.1f}] " + " ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    for k, v in errs.items():
        assert v < 4e-3, (k, v, ratio)


@pytest.mark.parametrize("mu,sd", _OFFSETS, ids=_OFFSET_IDS)
@pytest.mark.parametrize("rows,C", [(2 * 4096, 320), (128, 1280), (300, 1024)])
def test_layernorm_offset(rows, C, mu, sd):
    """LayerNorm forward, dx and the affine gradients against fp64 torch with large row means (two-pass statistics)."""
    from e4t_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(C + rows + int(mu))
    x = _mk((rows, C), g, sd, mu)
    gamma = torch.randn(C, generator=g, device="cuda") * 0.3 + 1
    beta = torch.randn(C, generator=g, device="cuda") * 0.2
    dy = _mk((rows, C), g)
    ratio = _ratio(x, (1,))
    xr = x.double().requires_grad_(True)
    gr, br = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    F.layer_norm(xr, (C,), gr, br, 1e-5).backward(dy.double())
    y, stats = ops.layernorm_fwd(x, gamma, beta, 1e-5)
    dx = ops.layernorm_bwd(x, dy, gamma, stats, 1e-5)
    dg, db = ops.layernorm_param_grad(x, dy, stats, gamma)
    errs = dict(y=_rel(y, F.layer_norm(x.double(), (C,), gamma.double(), beta.double(), 1e-5)), dx=_rel(dx, xr.grad),
                dgamma=_rel(dg, gr.grad), dbeta=_rel(db, br.grad))
    print(f"[layernorm {rows}x{C} mu/sd={ratio:.1f}] " + " ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    for k, v in errs.items():
        assert v < 4e-3, (k, v, ratio)


def test_geglu_and_resample():
    from e4t_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(3)
    h = _mk((500, 2 * 1280), g)
    dout = _mk((500, 1280), g)
    hr = h.float().requires_grad_(True)
    u, gate = hr.chunk(2, dim=-1)
    outr = u * F.gelu(gate)
    outr.backward(dout.float())
    assert _rel(ops.geglu_fwd(h), outr) < 4e-3
    assert _rel(ops.geglu_bwd(h, dout), hr.grad) < 4e-3
    x = _mk((2, 8, 8, 64), g)
    up = ops.resample2x(x, 0)
    assert torch.equal(up.float(), F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest").permute(0, 2, 3, 1))
    big = _mk((2, 16, 16, 64), g)
    s = ops.resample2x(big, 1)
    ref = F.avg_pool2d(big.float().permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1) * 4
    assert _rel(s, ref) < 4e-3
    assert torch.equal(ops.resample2x(big, 2), big[:, ::2, ::2].contiguous())
    z = ops.resample2x(x, 3)
    zr = torch.zeros(2, 16, 16, 64, device="cuda", dtype=torch.bfloat16)
    zr[:, ::2, ::2] = x
    assert torch.equal(z, zr)


@pytest.mark.parametrize("R,C", [(320, 320), (768, 640), (1280, 1280), (96, 64)])
def test_weight_offsets(R, C):
    """Closed form vs the literal e4t/weightoffsets.py:14-23 sequence, incl. all parameter gradients."""
    from e4t_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(R + C)
    dev = "cuda"
    def rnd(*s, k=1.0):
        return (torch.rand(*s, generator=g, device=dev) * 2 - 1) * k
    v = torch.ones(1, device=dev) * 0.9
    w1, b1 = rnd(R, k=1.0), rnd(R, k=1.0)
    w2, b2 = rnd(C, k=1.0), rnd(C, k=1.0)
    Wc, bc = rnd(R, R, k=R ** -0.5), rnd(R, k=R ** -0.5)
    Wr, br = rnd(C, C, k=C ** -0.5), rnd(C, k=C ** -0.5)
    W = rnd(C, R, k=R ** -0.5)
    ps = [t.double().requires_grad_(True) for t in (v, w1, b1, w2, b2, Wc, bc, Wr, br)]
    pv, pw1, pb1, pw2, pb2, pWc, pbc, pWr, pbr = ps
    vx = pw1 * pv + pb1
    vy = pw2 * pv + pb2
    m = vx[:, None] * vy[None, :]
    m = m.T @ pWc.T + pbc
    m = m.T @ pWr.T + pbr
    delta = m.T
    weff_ref = W.double() * (1 + delta)
    dWeff = rnd(C, R)
    (weff_ref * dWeff.double()).sum().backward()
    vx_, vy_, a, b, s = ops.wo_factors(v, w1, b1, w2, b2, Wc, Wr)
    weff = ops.wo_weff(W, a, bc, b, s, br)
    assert _rel(weff, weff_ref) < 4e-3
    grads = ops.wo_bwd(dWeff, W, v, w1, w2, Wc, Wr, bc, vx_, vy_, a, b, s)
    names = ["v", "w1", "b1", "w2", "b2", "Wc", "bc", "Wr", "br"]
    for nme, got, p in zip(names, grads, ps):
        assert _rel(got, p.grad) < 1e-3, nme


def test_meanpool_convio_adamw():
    from e4t_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(11)
    x = _mk((3, 256, 640), g, 1.0, 0.2)
    out = torch.zeros(3, 1000, device="cuda")
    ops.meanpool_fwd(x, out, 100)
    assert _rel(out[:, 100:740], x.float().mean(1)) < 1e-4
    dout = torch.randn(3, 1000, generator=g, device="cuda")
    dx = ops.meanpool_bwd(dout, (3, 256, 640), 100)
    assert _rel(dx, (dout[:, None, 100:740] / 256).expand(3, 256, 640)) < 4e-3
    lat = torch.randn(2, 4, 16, 16, generator=g, device="cuda")
    w = torch.randn(64, 4, 3, 3, generator=g, device="cuda") * 0.2
    b = torch.randn(64, generator=g, device="cuda")
    y = ops.conv_in_fwd(lat, w, b)
    assert _rel(y.permute(0, 3, 1, 2), F.conv2d(lat, w, b, padding=1)) < 4e-3
    xo = _mk((2, 16, 16, 64), g)
    wo = torch.randn(4, 64, 3, 3, generator=g, device="cuda") * 0.1
    bo = torch.randn(4, generator=g, device="cuda")
    xr = xo.float().permute(0, 3, 1, 2).requires_grad_(True)
    yr = F.conv2d(xr, wo, bo, padding=1)
    dy = torch.randn(2, 4, 16, 16, generator=g, device="cuda")
    yr.backward(dy)
    assert _rel(ops.conv_out_fwd(xo, wo, bo), yr) < 1e-4
    assert _rel(ops.conv_out_bwd(dy, wo, 64).permute(0, 3, 1, 2), xr.grad) < 4e-3
    n = 10007
    p = torch.randn(n, generator=g, device="cuda"); gr = torch.randn(n, generator=g, device="cuda")
    pr = p.clone().requires_grad_(True)
    opt = torch.optim.AdamW([pr], lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2)
    m = torch.zeros(n, device="cuda"); v = torch.zeros(n, device="cuda")
    for step in range(1, 4):
        pr.grad = gr.clone() * step
        opt.step()
        ops.adamw_step(p, gr * step, m, v, 1e-3, 0.9, 0.999, 1e-8, 1e-2, step)
    assert _rel(p, pr.detach()) < 1e-5


def _attn_ref(q, k, v, H):
    B, N, C = q.shape
    dh = C // H
    qh = q.view(B, N, H, dh).transpose(1, 2); kh = k.view(B, -1, H, dh).transpose(1, 2); vh = v.view(B, -1, H, dh).transpose(1, 2)
    s = (qh @ kh.transpose(-1, -2)) * dh ** -0.5
    p = s.softmax(-1)
    return (p @ vh).transpose(1, 2).reshape(B, N, C), torch.logsumexp(s, -1)


@pytest.mark.parametrize("B,H,N,M,dh", [(2, 8, 256, 256, 40), (1, 8, 1024, 1024, 80), (2, 8, 256, 256, 160),
                                        (2, 8, 64, 64, 160), (2, 8, 1024, 77, 40), (1, 4, 256, 77, 160),
                                        (1, 8, 300, 200, 80), (2, 4, 256, 256, 16), (2, 4, 64, 77, 32),
                                        (1, 8, 4096, 4096, 40)])
def test_attention(B, H, N, M, dh):
    from e4t_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(N + M + dh)
    C = H * dh
    q = _mk((B, N, C), g); k = _mk((B, M, C), g); v = _mk((B, M, C), g); do = _mk((B, N, C), g)
    qr, kr, vr = (t.float().requires_grad_(True) for t in (q, k, v))
    oref, lse_ref = _attn_ref(qr, kr, vr, H)
    oref.backward(do.float())
    o, lse = ops.attn_fwd(q, k, v, H)
    torch.cuda.synchronize()
    assert _rel(o, oref) < 6e-3, _rel(o, oref)
    assert (lse - lse_ref).abs().max().item() < 2e-2
    for fused in (True, False):       # single-pass (dh <= 80, N >= 128) and two-kernel backward
        dq, dk, dv = ops.attn_bwd(q, k, v, o, do, lse, H, fused=fused)
        torch.cuda.synchronize()
        assert _rel(dq, qr.grad) < 1e-2, ("dq", fused, _rel(dq, qr.grad))
        assert _rel(dk, kr.grad) < 1e-2, ("dk", fused, _rel(dk, kr.grad))
        assert _rel(dv, vr.grad) < 1e-2, ("dv", fused, _rel(dv, vr.grad))


def test_attention_fused_qkv_strides():
    """Q/K/V as column slices of one fused (B,N,3C) projection output."""
    from e4t_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(9)
    B, H, N, dh = 2, 8, 256, 40
    C = H * dh
    qkv = _mk((B, N, 3 * C), g)
    q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
    oref, _ = _attn_ref(q.float(), k.float(), v.float(), H)
    o, _ = ops.attn_fwd(q, k, v, H)
    assert _rel(o, oref) < 6e-3


def test_fp32_output_kernels_meet_1e3_at_baseline_shapes():
    """north_star's tolerance (1e-3 relative, fp32) per kernel at BASELINE shapes, where the kernel can write fp32: the
    wgmma GEMM and the implicit-GEMM convolution with fp32 outputs, and the attention core's fp32 output (LSE).  Inputs
    are bf16-representable, the reference is fp64 torch.  (bf16 OUTPUTS carry 2^-9 rounding by themselves; the attention
    O tensor is therefore compared with the reference ROUNDED to bf16, which isolates the kernel's own error.)"""
    from e4t_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(123)
    # QKV projection GEMM of level 0 at B=16: (65536, 320) x (960, 320)^T
    A = _mk((65536, 320), g, 1.0)
    W = _mk((960, 320), g, 0.05)
    y = ops.gemm(A, W, out_dtype=torch.float32)
    ref = A[:8192].double() @ W.double().t()
    e_gemm = _rel(y[:8192], ref)
    # ResnetBlock conv 320 -> 320 at 64x64, B=4
    x = _mk((4, 64, 64, 320), g, 1.0)
    w = torch.randn(320, 320, 3, 3, generator=g, device="cuda") * 0.02
    w9 = w.permute(2, 3, 0, 1).reshape(9, 320, 320).to(torch.bfloat16).contiguous()
    yc = ops.conv3x3(x, w9, out_dtype=torch.float32)
    refc = F.conv2d(x[:1].double().permute(0, 3, 1, 2), w9.double().view(3, 3, 320, 320).permute(2, 3, 0, 1), padding=1)
    e_conv = _rel(yc[:1].permute(0, 3, 1, 2), refc)
    # level-0 self-attention (N = M = 4096, 8 x 40), B=2
    q, k, v = _mk((2, 4096, 320), g), _mk((2, 4096, 320), g), _mk((2, 4096, 320), g)
    o, lse = ops.attn_fwd(q, k, v, 8)
    oref, lse_ref = _attn_ref(q.float(), k.float(), v.float(), 8)
    e_lse = ((lse - lse_ref).abs() / lse_ref.abs().clamp_min(1.0)).max().item()
    e_o = _rel(o.float(), oref.to(torch.bfloat16).float())
    print(f"[fp32 outputs] gemm {e_gemm:.2e}  conv {e_conv:.2e}  attention LSE {e_lse:.2e}  attention O vs bf16(ref) {e_o:.2e}")
    assert e_gemm < 1e-3 and e_conv < 1e-3 and e_lse < 1e-3
    assert e_o < 4e-3
