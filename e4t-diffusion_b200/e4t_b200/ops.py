"""Raw (non-autograd) wrappers over the C-ABI entry points declared in include/e4t_b200.h.

Every function takes CUDA tensors, launches hand-written sm_90a kernels on torch's current stream and
returns torch tensors that merely own the output memory.
"""
import ctypes

import torch

from . import _lib
from ._lib import c_float, c_int, c_ll, c_void_p, ptr, stream

c_double = ctypes.c_double

BF16 = torch.bfloat16
F32 = torch.float32


def _fp(t):
    return ptr(t)


def gemm(A, B, *, a_mn=False, b_mn=False, out=None, out_dtype=BF16, bias=None, rowgroup=None,
         rows_per_group=1, residual=None, alpha=1.0, splits=1, accumulate=False, force_bn=0):
    """out[b] = alpha * op(A[b]) @ op(B[b])^T (+bias +rowgroup +residual).

    K-major operands are (.., rows, K) with K contiguous; MN-major operands are (.., K, rows) with rows
    contiguous (i.e. the transposed storage).  A 2-D operand is shared across the batch.
    accumulate=True -> fp32 atomic accumulation into `out` (required for split-K, which takes no bias, rowgroup or
    residual).  out, residual, bias and rowgroup must cover (batch, M, N), N and ceil(M / rows_per_group) x N.
    """
    assert A.dtype == BF16 and B.dtype == BF16
    assert A.stride(-1) == 1 and B.stride(-1) == 1
    if A.dim() == 3 and B.dim() == 3 and A.shape[0] != B.shape[0]:
        raise ValueError(f"gemm: operands disagree on batch: A {tuple(A.shape)}, B {tuple(B.shape)}")
    batch = 1
    if A.dim() == 3:
        batch = A.shape[0]
    if B.dim() == 3:
        batch = B.shape[0]
    if a_mn:
        K, M = A.shape[-2], A.shape[-1]
    else:
        M, K = A.shape[-2], A.shape[-1]
    if b_mn:
        Kb, N = B.shape[-2], B.shape[-1]
    else:
        N, Kb = B.shape[-2], B.shape[-1]
    assert K == Kb, (A.shape, B.shape, a_mn, b_mn)
    # The library takes only pointers and strides: a tensor smaller than the call would be read or written past its end
    if out is not None and tuple(out.shape) != ((batch, M, N) if out.dim() == 3 else (M, N) if batch == 1 else None):
        raise ValueError(f"gemm: out {tuple(out.shape)} is not (batch, M, N) = ({batch}, {M}, {N})")
    if residual is not None and (tuple(residual.shape[-2:]) != (M, N) or residual.dim() not in (2, 3)
                                 or (residual.dim() == 3 and residual.shape[0] != batch)):
        raise ValueError(f"gemm: residual {tuple(residual.shape)} does not cover ({batch}, {M}, {N})")
    if bias is not None and bias.numel() != N:
        raise ValueError(f"gemm: bias has {bias.numel()} elements, N = {N}")
    if rowgroup is not None and (rows_per_group < 1 or rowgroup.numel() != -(-M // rows_per_group) * N):
        raise ValueError(f"gemm: rowgroup {tuple(rowgroup.shape)} is not ceil({M} / {rows_per_group}) rows of {N}")
    a_bs = A.stride(0) if A.dim() == 3 and batch > 1 else 0
    b_bs = B.stride(0) if B.dim() == 3 and batch > 1 else 0
    if accumulate:
        assert out is not None and out.dtype == F32
        out_mode = 2
    else:
        if out is None:
            shape = (batch, M, N) if (A.dim() == 3 or B.dim() == 3) else (M, N)
            out = torch.empty(shape, device=A.device, dtype=out_dtype)
        out_mode = 0 if out.dtype == BF16 else 1
    assert out.stride(-1) == 1
    o_bs = out.stride(0) if out.dim() == 3 and batch > 1 else 0
    r_bs = 0
    ldr = 0
    if residual is not None:
        assert residual.dtype == BF16 and residual.stride(-1) == 1
        ldr = residual.stride(-2)
        r_bs = residual.stride(0) if residual.dim() == 3 and batch > 1 else 0
    if bias is not None:
        assert bias.dtype == F32 and bias.is_contiguous()
    if rowgroup is not None:
        assert rowgroup.dtype == F32 and rowgroup.is_contiguous()
    _lib.call("e4t_gemm_bf16", ptr(A), ptr(B), ptr(out), c_int(M), c_int(N), c_int(K), c_int(batch),
              c_int(int(a_mn)), c_int(int(b_mn)), c_ll(A.stride(-2)), c_ll(B.stride(-2)), c_ll(a_bs), c_ll(b_bs),
              c_int(out_mode), c_ll(out.stride(-2)), c_ll(o_bs), ptr(bias), ptr(rowgroup), c_int(rows_per_group),
              ptr(residual), c_ll(ldr), c_ll(r_bs), c_float(alpha), c_int(splits), c_int(force_bn), stream())
    return out


def conv3x3(x, w9, *, bias=None, rowgroup=None, residual=None, out_dtype=BF16, force_bn=0):
    """3x3 stride-1 pad-1 convolution on NHWC bf16.  x: (B,H,W,Cin); w9: (9,Cout,Cin) bf16, tap = ky*3+kx."""
    assert x.dtype == BF16 and w9.dtype == BF16 and x.is_contiguous() and w9.is_contiguous()
    Bn, H, W, Cin = x.shape
    Cout = w9.shape[1]
    assert w9.shape == (9, Cout, Cin)
    out = torch.empty((Bn, H, W, Cout), device=x.device, dtype=out_dtype)
    if residual is not None:
        assert residual.dtype == BF16 and residual.is_contiguous() and residual.shape == out.shape
    _lib.call("e4t_conv3x3_bf16", ptr(x), ptr(w9), ptr(out), c_int(Bn), c_int(H), c_int(W), c_int(Cin), c_int(Cout),
              c_int(0 if out_dtype == BF16 else 1), ptr(bias), ptr(rowgroup), ptr(residual), c_int(force_bn),
              stream())
    return out


def conv3x3_tiled(H, W):
    """True when conv3x3 (the tiled-box A operand) accepts an H x W output: W divides 128 and the tile's 128 / W rows
    divide H (or H*W divides 128), or W is a multiple of 128.  Other sizes take conv3x3_im2col; the stride-2
    convolutions and conv3x3_wgrad choose by the same kind of rule inside the library."""
    if W > 128:
        return W % 128 == 0
    if 128 % W:
        return False
    return H % (128 // W) == 0 if H * W >= 128 else 128 % (H * W) == 0


def conv3x3_im2col(x, w9, *, bias=None, rowgroup=None, residual=None, out_dtype=BF16, force_bn=0):
    """conv3x3 with the A operand loaded by TMA in im2col mode (tiles of 128 consecutive pixels across rows and
    images): any H x W.  Same arguments and result as conv3x3."""
    assert x.dtype == BF16 and w9.dtype == BF16 and x.is_contiguous() and w9.is_contiguous()
    Bn, H, W, Cin = x.shape
    Cout = w9.shape[1]
    assert w9.shape == (9, Cout, Cin)
    out = torch.empty((Bn, H, W, Cout), device=x.device, dtype=out_dtype)
    if residual is not None:
        assert residual.dtype == BF16 and residual.is_contiguous() and residual.shape == out.shape
    _lib.call("e4t_conv3x3_im2col_bf16", ptr(x), ptr(w9), ptr(out), c_int(Bn), c_int(H), c_int(W), c_int(Cin),
              c_int(Cout), c_int(0 if out_dtype == BF16 else 1), ptr(bias), ptr(rowgroup), ptr(residual),
              c_int(force_bn), stream())
    return out


def conv3x3_s2(x, w9, *, bias=None, force_bn=0, pad_lo=1):
    """3x3 stride-2 convolution on NHWC bf16 (Downsample2D): (B,H,W,Cin) -> (B,ceil(H/2),ceil(W/2),Cout).
    pad_lo=1: pad 1 on every side (any H, W); pad_lo=0: one zero row / column on the bottom and right only (diffusers
    Downsample2D(padding=0), the VAE encoder; H, W even)."""
    assert x.dtype == BF16 and w9.dtype == BF16 and x.is_contiguous() and w9.is_contiguous()
    Bn, H, W, Cin = x.shape
    Cout = w9.shape[1]
    out = torch.empty((Bn, (H + 1) // 2, (W + 1) // 2, Cout), device=x.device, dtype=BF16)
    if pad_lo == 1:
        _lib.call("e4t_conv3x3_s2_bf16", ptr(x), ptr(w9), ptr(out), c_int(Bn), c_int(H), c_int(W), c_int(Cin),
                  c_int(Cout), ptr(bias), c_int(force_bn), stream())
    else:
        _lib.call("e4t_conv3x3_s2p_bf16", ptr(x), ptr(w9), ptr(out), c_int(Bn), c_int(H), c_int(W), c_int(Cin),
                  c_int(Cout), c_int(pad_lo), ptr(bias), c_int(force_bn), stream())
    return out


def softmax_rows(x, out=None):
    """bf16 softmax over the last dim of fp32 scores x (.., n); rows may be strided (last dim contiguous)."""
    assert x.dtype == F32 and x.stride(-1) == 1
    n = x.shape[-1]
    x2 = x if x.dim() == 2 else x.reshape(-1, n)
    if out is None:
        out = torch.empty(x.shape, device=x.device, dtype=BF16)
    assert out.dtype == BF16 and out.stride(-1) == 1 and out.shape == x.shape
    o2 = out if out.dim() == 2 else out.view(-1, n)
    _lib.call("e4t_softmax_rows", ptr(x2), ptr(o2), c_ll(x2.shape[0]), c_int(n), c_ll(x2.stride(0)), c_ll(o2.stride(0)),
              stream())
    return out


# ----------------------------------------------------------------------------------------------
# normalisation
# ----------------------------------------------------------------------------------------------
def groupnorm_fwd(x, gamma, beta, groups, eps, silu):
    """x: (B,HW,C) or (B,H,W,C) bf16 NHWC.  Returns (y, stats): stats fp32 [B,G,3] = (p, sum(x - p), sum((x - p)^2))
    per (image, group) around the pivot p = the group's first element, the form groupnorm_bwd and
    groupnorm_param_grad take (csrc/common.cuh, gn_mean_rstd, turns it into (mean, rstd))."""
    assert x.dtype == BF16 and x.is_contiguous()
    Bn, C = x.shape[0], x.shape[-1]
    HW = x.numel() // (Bn * C)
    y = torch.empty_like(x)
    stats = torch.empty((Bn, groups, 3), device=x.device, dtype=F32)
    _lib.call("e4t_groupnorm_fwd", ptr(x), ptr(gamma), ptr(beta), ptr(y), ptr(stats), c_int(Bn), c_int(HW), c_int(C),
              c_int(groups), c_float(eps), c_int(int(silu)), stream())
    return y, stats


def groupnorm_bwd(x, dy, gamma, beta, stats, groups, eps, silu):
    assert x.dtype == BF16 and dy.dtype == BF16 and x.is_contiguous() and dy.is_contiguous()
    Bn, C = x.shape[0], x.shape[-1]
    HW = x.numel() // (Bn * C)
    dx = torch.empty_like(x)
    scratch = torch.empty((Bn, groups, 2), device=x.device, dtype=F32)
    _lib.call("e4t_groupnorm_bwd", ptr(x), ptr(dy), ptr(gamma), ptr(beta), ptr(stats), ptr(dx), ptr(scratch),
              c_int(Bn), c_int(HW), c_int(C), c_int(groups), c_float(eps), c_int(int(silu)), stream())
    return dx


def layernorm_fwd(x, gamma, beta, eps):
    assert x.dtype == BF16 and x.is_contiguous()
    C = x.shape[-1]
    rows = x.numel() // C
    y = torch.empty_like(x)
    stats = torch.empty((rows, 2), device=x.device, dtype=F32)
    _lib.call("e4t_layernorm_fwd", ptr(x), ptr(gamma), ptr(beta), ptr(y), ptr(stats), c_ll(rows), c_int(C),
              c_float(eps), stream())
    return y, stats


def layernorm_bwd(x, dy, gamma, stats, eps):
    assert x.dtype == BF16 and dy.dtype == BF16 and x.is_contiguous() and dy.is_contiguous()
    C = x.shape[-1]
    rows = x.numel() // C
    dx = torch.empty_like(x)
    _lib.call("e4t_layernorm_bwd", ptr(x), ptr(dy), ptr(gamma), ptr(stats), ptr(dx), c_ll(rows), c_int(C),
              c_float(eps), stream())
    return dx


# ----------------------------------------------------------------------------------------------
# elementwise
# ----------------------------------------------------------------------------------------------
def geglu_fwd(h):
    assert h.dtype == BF16 and h.is_contiguous()
    F = h.shape[-1] // 2
    rows = h.numel() // (2 * F)
    out = torch.empty(h.shape[:-1] + (F,), device=h.device, dtype=BF16)
    _lib.call("e4t_geglu_fwd", ptr(h), ptr(out), c_ll(rows), c_int(F), stream())
    return out


def geglu_bwd(h, dout):
    assert h.dtype == BF16 and dout.dtype == BF16 and h.is_contiguous() and dout.is_contiguous()
    F = h.shape[-1] // 2
    rows = h.numel() // (2 * F)
    dh = torch.empty_like(h)
    _lib.call("e4t_geglu_bwd", ptr(h), ptr(dout), ptr(dh), c_ll(rows), c_int(F), stream())
    return dh


def resample2x(x, mode):
    """NHWC bf16.  mode 0 nearest-up, 1 its adjoint, 2 stride-2 pick, 3 zero-insertion (adjoint of 2)."""
    assert x.dtype == BF16 and x.is_contiguous() and x.dim() == 4
    Bn, Hx, Wx, C = x.shape
    if mode in (0, 3):
        H, W = Hx, Wx
        y = torch.empty((Bn, 2 * H, 2 * W, C), device=x.device, dtype=BF16)
    else:
        H, W = Hx // 2, Wx // 2
        y = torch.empty((Bn, H, W, C), device=x.device, dtype=BF16)
    _lib.call("e4t_resample2x", ptr(x), ptr(y), c_int(Bn), c_int(H), c_int(W), c_int(C), c_int(mode), stream())
    return y


def _resize_args(x, size):
    assert x.dtype == BF16 and x.is_contiguous() and x.dim() == 4
    Bn, Hx, Wx, C = x.shape
    Hy, Wy = (int(s) for s in size)
    y = torch.empty((Bn, Hy, Wy, C), device=x.device, dtype=BF16)
    return y, (ptr(x), ptr(y), c_int(Bn), c_int(Hx), c_int(Wx), c_int(Hy), c_int(Wy), c_int(C))


def resize_nearest(x, size):
    """Nearest resize of NHWC bf16 (B,Hi,Wi,C) to (B,*size,C) with torch's index rule: bit-identical to
    F.interpolate(size=size, mode="nearest") (diffusers Upsample2D with output_size)."""
    y, args = _resize_args(x, size)
    _lib.call("e4t_resize_nearest", *args, c_int(0), stream())
    return y


def resize_nearest_bwd(dy, in_size):
    """Adjoint of resize_nearest: dy (B,Ho,Wo,C) at the resized size -> (B,*in_size,C) (fp32 sums, deterministic)."""
    dx, args = _resize_args(dy, in_size)
    _lib.call("e4t_resize_nearest", *args, c_int(1), stream())
    return dx


def zero_insert(dy, size):
    """Zero insertion of (B,Ho,Wo,C) to (B,*size,C), y[2i, 2j] = dy[i, j]: the adjoint of the stride-2 pick of a pad-1
    stride-2 convolution whose input is `size` (either side may be odd; Ho = ceil(size[0] / 2))."""
    y, args = _resize_args(dy, size)
    _lib.call("e4t_resize_nearest", *args, c_int(2), stream())
    return y


def meanpool_fwd(x, out, c_off):
    """x (B,HW,C)/(B,H,W,C) bf16 -> out[:, c_off:c_off+C] (fp32, (B, ldo))."""
    assert x.dtype == BF16 and x.is_contiguous() and out.dtype == F32 and out.stride(1) == 1
    Bn, C = x.shape[0], x.shape[-1]
    HW = x.numel() // (Bn * C)
    _lib.call("e4t_meanpool_fwd", ptr(x), ptr(out), c_int(Bn), c_int(HW), c_int(C), c_int(out.stride(0)), c_int(c_off),
              stream())


def meanpool_bwd(dout, shape, c_off):
    assert dout.dtype == F32 and dout.stride(1) == 1
    Bn, C = shape[0], shape[-1]
    HW = 1
    for s in shape[1:-1]:
        HW *= s
    dx = torch.empty(shape, device=dout.device, dtype=BF16)
    _lib.call("e4t_meanpool_bwd", ptr(dout), ptr(dx), c_int(Bn), c_int(HW), c_int(C), c_int(dout.stride(0)),
              c_int(c_off), stream())
    return dx


def conv_in_fwd(x, w, bias):
    """x NCHW fp32 (B,Cin,H,W) -> NHWC bf16 (B,H,W,Cout).  w fp32 (Cout,Cin,3,3)."""
    assert x.dtype == F32 and x.is_contiguous() and w.dtype == F32 and w.is_contiguous()
    Bn, Cin, H, W = x.shape
    Cout = w.shape[0]
    y = torch.empty((Bn, H, W, Cout), device=x.device, dtype=BF16)
    _lib.call("e4t_conv_in_fwd", ptr(x), ptr(w), ptr(bias), ptr(y), c_int(Bn), c_int(Cin), c_int(H), c_int(W),
              c_int(Cout), stream())
    return y


def conv_out_fwd(x, w, bias):
    """x NHWC bf16 (B,H,W,C) -> NCHW fp32 (B,Cout,H,W)."""
    assert x.dtype == BF16 and x.is_contiguous() and w.dtype == F32 and w.is_contiguous()
    Bn, H, W, C = x.shape
    Cout = w.shape[0]
    y = torch.empty((Bn, Cout, H, W), device=x.device, dtype=F32)
    _lib.call("e4t_conv_out_fwd", ptr(x), ptr(w), ptr(bias), ptr(y), c_int(Bn), c_int(H), c_int(W), c_int(C),
              c_int(Cout), stream())
    return y


def conv_out_bwd(dy, w, C):
    assert dy.dtype == F32 and dy.is_contiguous()
    Bn, Cout, H, W = dy.shape
    dx = torch.empty((Bn, H, W, C), device=dy.device, dtype=BF16)
    _lib.call("e4t_conv_out_bwd", ptr(dy), ptr(w), ptr(dx), c_int(Bn), c_int(H), c_int(W), c_int(C), c_int(Cout),
              stream())
    return dx


# ----------------------------------------------------------------------------------------------
# WeightOffsets
# ----------------------------------------------------------------------------------------------
def wo_factors(v, w1, b1, w2, b2, Wc, Wr):
    R, C = Wc.shape[0], Wr.shape[0]
    buf = torch.empty(2 * R + 3 * C, device=v.device, dtype=F32)
    vx, a, vy, b, s = buf[:R], buf[R:2 * R], buf[2 * R:2 * R + C], buf[2 * R + C:2 * R + 2 * C], buf[2 * R + 2 * C:]
    _lib.call("e4t_wo_factors_fwd", ptr(v), ptr(w1), ptr(b1), ptr(w2), ptr(b2), ptr(Wc), ptr(Wr), ptr(vx), ptr(vy),
              ptr(a), ptr(b), ptr(s), c_int(R), c_int(C), stream())
    return vx, vy, a, b, s


def wo_weff(W, a, bc, b, s, br, out=None):
    C, R = W.shape
    if out is None:
        out = torch.empty((C, R), device=W.device, dtype=BF16)
    assert out.is_contiguous() and out.shape == (C, R) and out.dtype == BF16
    _lib.call("e4t_wo_weff_fwd", ptr(W), ptr(a), ptr(bc), ptr(b), ptr(s), ptr(br), ptr(out), c_int(C), c_int(R),
              stream())
    return out


def wo_bwd(dWeff, W, v, w1, w2, Wc, Wr, bc, vx, vy, a, b, s, outs=None):
    """outs: optional 9 preallocated gradient tensors (dv,dw1,db1,dw2,db2,dWc,dbc,dWr,dbr) that are WRITTEN."""
    C, R = W.shape
    dev = W.device
    scratch = torch.empty(3 * C + 2 * R + R + C, device=dev, dtype=F32)
    if outs is not None:
        dv, dw1, db1, dw2, db2, dWc, dbc, dWr, dbr = outs
        for t in outs:
            assert t.dtype == F32 and t.is_contiguous()
    else:
        dv = torch.empty(1, device=dev, dtype=F32)
        dw1 = torch.empty(R, device=dev, dtype=F32); db1 = torch.empty(R, device=dev, dtype=F32)
        dw2 = torch.empty(C, device=dev, dtype=F32); db2 = torch.empty(C, device=dev, dtype=F32)
        dWc = torch.empty((R, R), device=dev, dtype=F32); dbc = torch.empty(R, device=dev, dtype=F32)
        dWr = torch.empty((C, C), device=dev, dtype=F32); dbr = torch.empty(C, device=dev, dtype=F32)
    _lib.call("e4t_wo_bwd", ptr(dWeff), ptr(W), ptr(v), ptr(w1), ptr(w2), ptr(Wc), ptr(Wr), ptr(bc), ptr(vx), ptr(vy),
              ptr(a), ptr(b), ptr(s), ptr(scratch), ptr(dv), ptr(dw1), ptr(db1), ptr(dw2), ptr(db2), ptr(dWc),
              ptr(dbc), ptr(dWr), ptr(dbr), c_int(R), c_int(C), stream())
    return dv, dw1, db1, dw2, db2, dWc, dbc, dWr, dbr


def adamw_step(p, g, m, v, lr, beta1, beta2, eps, weight_decay, step, grad_scale=1.0):
    assert p.dtype == F32 and p.is_contiguous() and g.is_contiguous() and m.is_contiguous() and v.is_contiguous()
    _lib.call("e4t_adamw_step", ptr(p), ptr(g), ptr(m), ptr(v), c_ll(p.numel()), c_float(lr), c_float(beta1),
              c_float(beta2), c_float(eps), c_float(weight_decay), c_int(step), c_float(grad_scale), stream())


def adamw_step_dev(p, g, m, v, lr, beta1, beta2, eps, weight_decay, step_dev, grad_scale=1.0):
    """AdamW with the step counter in device memory (int32 tensor, incremented by the call): graph-replayable."""
    assert p.dtype == F32 and step_dev.dtype == torch.int32
    _lib.call("e4t_adamw_step_dev", ptr(p), ptr(g), ptr(m), ptr(v), c_ll(p.numel()), c_float(lr), c_float(beta1),
              c_float(beta2), c_float(eps), c_float(weight_decay), ptr(step_dev), c_float(grad_scale), stream())


def _sched_args(sched):
    kind, warmup, total, cycles, power, lr_end = sched
    return c_int(kind), c_int(warmup), c_int(total), c_double(cycles), c_double(power), c_double(lr_end)


def adamw_step_sched(p, g, m, v, lr, beta1, beta2, eps, weight_decay, step_dev, lr_dev, sched, grad_scale=1.0):
    """adamw_step_dev following a learning-rate schedule on the device: `sched` = (kind, warmup, total, num_cycles,
    power, lr_end) (e4t_b200.optim); the lr each call uses is written to `lr_dev` (fp32, 1 element)."""
    assert p.dtype == F32 and step_dev.dtype == torch.int32 and lr_dev.dtype == F32
    _lib.call("e4t_adamw_step_sched", ptr(p), ptr(g), ptr(m), ptr(v), c_ll(p.numel()), c_float(lr), c_float(beta1),
              c_float(beta2), c_float(eps), c_float(weight_decay), ptr(step_dev), ptr(lr_dev), *_sched_args(sched),
              c_float(grad_scale), stream())


def adamw8bit_step_sched(p, g, m_codes, v_codes, m_absmax, v_absmax, qmap_m, qmap_v, lr, beta1, beta2, eps,
                         weight_decay, step_dev, lr_dev, sched, grad_scale=1.0):
    """8-bit AdamW (block-wise quantised moments, one absmax per 256 elements) with a schedule as adamw_step_sched."""
    assert p.dtype == F32 and g.dtype == F32 and m_codes.dtype == torch.uint8 and v_codes.dtype == torch.uint8
    assert m_absmax.dtype == F32 and v_absmax.dtype == F32 and qmap_m.numel() == 256 and qmap_v.numel() == 256
    n = p.numel()
    if not (g.numel() == m_codes.numel() == v_codes.numel() == n and m_absmax.numel() == v_absmax.numel() == n // 256):
        raise ValueError(f"adamw8bit_step_sched: {n} parameters need {n} gradients and codes and {n // 256} absmax")
    _lib.call("e4t_adamw8bit_step_sched", ptr(p), ptr(g), ptr(m_codes), ptr(v_codes), ptr(m_absmax), ptr(v_absmax),
              ptr(qmap_m), ptr(qmap_v), c_ll(n), c_float(lr), c_float(beta1), c_float(beta2), c_float(eps),
              c_float(weight_decay), ptr(step_dev), ptr(lr_dev), *_sched_args(sched), c_float(grad_scale), stream())


# ----------------------------------------------------------------------------------------------
# sampling: one scheduler update from a coefficient table (e4t/schedulers.py)
# ----------------------------------------------------------------------------------------------
def sampler_history_buffer(n_hist, n, device):
    """History slots for `sampler_step`: (n_hist, n rounded up to 4) fp32, so every slot starts 16-byte aligned."""
    return torch.zeros(n_hist, (n + 3) // 4 * 4, dtype=F32, device=device)


def _need(cond, msg):
    if not cond:
        raise _lib.E4TError(f"sampler_step: {msg}")


def sampler_step(out, x, x_next, hist, saved, noise, table, step_dev, row, guidance=None, t_out=None, model_in=None):
    """e4t_sampler_step: publish row *step_dev of `table` into `row`, advance the counter and apply the row to the n
    elements of `x`, writing `x_next` (may be `x`), the history slot, the saved sample and, when given, the next step's
    model input (all G rows) and timestep.  `out` holds n (no guidance) or 2n (uncond rows first; `guidance` is then a
    1-element fp32 device tensor) elements.  Every check runs before any launch."""
    n = x.numel()
    bufs = dict(out=out, x=x, x_next=x_next, saved=saved, row=row, noise=noise, t_out=t_out, model_in=model_in,
                guidance=guidance, hist=hist)
    for k, t in bufs.items():
        if t is None:
            continue
        _need(t.is_cuda and t.dtype == F32 and t.is_contiguous(), f"{k} must be a contiguous fp32 CUDA tensor")
    _need(n > 0 and out.numel() in (n, 2 * n), f"out has {out.numel()} elements for {n} latents (need n or 2n)")
    G = out.numel() // n
    _need(G == 1 or (guidance is not None and guidance.numel() == 1), "guidance (1 element) is needed with 2n outputs")
    _need(x_next.numel() == n and saved.numel() == n and (noise is None or noise.numel() == n),
          "x_next, saved and noise must have as many elements as x")
    _need(model_in is None or model_in.numel() == G * n, f"model_in must have {G} x {n} elements")
    _need(t_out is None or t_out.numel() == 1, "t_out must have 1 element")
    _need(hist.dim() == 2 and hist.shape[0] <= 4 and (hist.shape[0] == 0 or hist.shape[1] >= n),
          "hist must be (slots <= 4, >= n)")
    _need(table.is_cuda and table.dtype == torch.float64 and table.is_contiguous() and table.dim() == 2
          and table.shape[1] == 14 and table.shape[0] >= 1, "table must be a contiguous (rows >= 1, 14) fp64 CUDA tensor")
    _need(step_dev.is_cuda and step_dev.dtype == torch.int32 and step_dev.numel() == 1, "step_dev must be 1 int32")
    _need(row.numel() >= 14, "row needs 14 elements")
    _lib.call("e4t_sampler_step", ptr(out), c_int(G), ptr(guidance), ptr(x), ptr(x_next), ptr(hist),
              c_int(hist.shape[0]), c_ll(hist.shape[1]), ptr(saved), ptr(noise), ptr(table), c_int(table.shape[0]),
              ptr(step_dev), ptr(row), ptr(t_out), ptr(model_in), c_ll(n), stream())


# ----------------------------------------------------------------------------------------------
# attention core
# ----------------------------------------------------------------------------------------------
def _bs(t):
    return t.stride(0)


def attn_fwd(q, k, v, heads, scale=None):
    """q (B,N,H*dh), k/v (B,M,H*dh) bf16 (last dim contiguous; may be column slices of a fused projection).
    Returns (o (B,N,H*dh) bf16, lse (B,H,N) fp32).
    dh == 40, 64 or 80 with N and M multiples of 128, >= 512 (the SD 1.x 4096-token and 1024-token self-attention, the
    SD 2.x self-attention with heads of 64; for dh == 64 and 80 only grids of at least half as many 128-query CTAs as
    SMs) runs the warpgroup (wgmma + TMA) kernel; every other shape, or E4T_ATTN_WGMMA=0, the mma.sync kernel."""
    assert q.dtype == BF16 and k.dtype == BF16 and v.dtype == BF16
    assert q.stride(-1) == 1 and k.stride(-1) == 1 and v.stride(-1) == 1
    Bn, N, C = q.shape
    M = k.shape[1]
    dh = C // heads
    scale = dh ** -0.5 if scale is None else scale
    o = torch.empty((Bn, N, C), device=q.device, dtype=BF16)
    lse = torch.empty((Bn, heads, N), device=q.device, dtype=F32)
    _lib.call("e4t_attn_fwd", ptr(q), ptr(k), ptr(v), ptr(o), ptr(lse), c_int(Bn), c_int(heads), c_int(N), c_int(M),
              c_int(dh), c_ll(q.stride(1)), c_ll(_bs(q)), c_ll(k.stride(1)), c_ll(_bs(k)), c_ll(v.stride(1)),
              c_ll(_bs(v)), c_ll(o.stride(1)), c_ll(_bs(o)), c_float(scale), stream())
    return o, lse


def attn_bwd(q, k, v, o, do, lse, heads, scale=None, dq=None, dk=None, dv=None, fused=True, causal=False):
    """dq/dk/dv may be preallocated (e.g. column slices of one fused (B,N,3C) gradient buffer).
    fused=True: single-pass backward (S/dP computed once per tile pair, dQ reduced in fp32) when dh <= 80 and N >= 128;
    otherwise / fused=False the two-kernel (dK/dV, dQ) path.  The single-pass backward of a non-causal call with
    the shapes attn_fwd gives to the warpgroup kernels runs the warpgroup (wgmma + TMA) kernel, which reduces dQ with
    bulk tensor adds instead of scalar atomics; every other shape, or E4T_ATTN_WGMMA=0, the mma.sync kernel.
    causal=True (N == M, dh <= 80): key j contributes to query i only if j <= i; o / lse must come from a forward that
    applied the same mask (attn_small_fwd)."""
    assert do.dtype == BF16 and do.stride(-1) == 1
    Bn, N, C = q.shape
    M = k.shape[1]
    dh = C // heads
    scale = dh ** -0.5 if scale is None else scale
    dq = torch.empty((Bn, N, C), device=q.device, dtype=BF16) if dq is None else dq
    dk = torch.empty((Bn, M, C), device=q.device, dtype=BF16) if dk is None else dk
    dv = torch.empty((Bn, M, C), device=q.device, dtype=BF16) if dv is None else dv
    assert dq.stride(-1) == 1 and dk.stride(-1) == 1 and dv.stride(-1) == 1
    dlt = torch.empty((Bn, heads, N), device=q.device, dtype=F32)
    assert not causal or (dh <= 80 and N == M), "causal attention backward: dh <= 80 and N == M"
    if causal or (fused and dh <= 80 and N >= 128):
        dqacc = torch.empty((Bn, N, C), device=q.device, dtype=F32)
        _lib.call("e4t_attn_bwd_fused_causal" if causal else "e4t_attn_bwd_fused", ptr(q), ptr(k), ptr(v), ptr(o), ptr(do), ptr(lse), ptr(dlt), ptr(dqacc),
                  ptr(dq), ptr(dk), ptr(dv), c_int(Bn), c_int(heads), c_int(N), c_int(M), c_int(dh),
                  c_ll(q.stride(1)), c_ll(_bs(q)), c_ll(k.stride(1)), c_ll(_bs(k)), c_ll(v.stride(1)), c_ll(_bs(v)),
                  c_ll(o.stride(1)), c_ll(_bs(o)), c_ll(do.stride(1)), c_ll(_bs(do)), c_ll(dq.stride(1)),
                  c_ll(_bs(dq)), c_ll(dk.stride(1)), c_ll(_bs(dk)), c_ll(dv.stride(1)), c_ll(_bs(dv)),
                  c_float(scale), stream())
        return dq, dk, dv
    _lib.call("e4t_attn_bwd", ptr(q), ptr(k), ptr(v), ptr(o), ptr(do), ptr(lse), ptr(dlt), ptr(dq), ptr(dk), ptr(dv),
              c_int(Bn), c_int(heads), c_int(N), c_int(M), c_int(dh), c_ll(q.stride(1)), c_ll(_bs(q)),
              c_ll(k.stride(1)), c_ll(_bs(k)), c_ll(v.stride(1)), c_ll(_bs(v)), c_ll(o.stride(1)), c_ll(_bs(o)),
              c_ll(do.stride(1)), c_ll(_bs(do)), c_ll(dq.stride(1)), c_ll(_bs(dq)), c_ll(dk.stride(1)), c_ll(_bs(dk)),
              c_ll(dv.stride(1)), c_ll(_bs(dv)), c_float(scale), stream())
    return dq, dk, dv


# ----------------------------------------------------------------------------------------------
# small operators (csrc/small_ops.cu) and weight gradients
# ----------------------------------------------------------------------------------------------
ACT_GELU, ACT_QUICK_GELU, ACT_LEAKY_RELU = 0, 1, 2


def act_fwd(x, mode):
    assert x.dtype == BF16 and x.is_contiguous()
    y = torch.empty_like(x)
    _lib.call("e4t_act_fwd", ptr(x), ptr(y), c_ll(x.numel()), c_int(mode), stream())
    return y


def act_bwd(x, dy, mode):
    assert x.dtype == BF16 and dy.dtype == BF16 and x.is_contiguous() and dy.is_contiguous()
    dx = torch.empty_like(x)
    _lib.call("e4t_act_bwd", ptr(x), ptr(dy), ptr(dx), c_ll(x.numel()), c_int(mode), stream())
    return dx


def colsum_acc(x2, out, rows_per_group=0):
    """out[g][n] += sum of the rows of group g of x2 (bf16 (M,N), row stride = x2.stride(0)); out fp32, pre-initialised."""
    assert x2.dtype == BF16 and x2.dim() == 2 and x2.stride(1) == 1 and out.dtype == F32 and out.is_contiguous()
    _lib.call("e4t_colsum_acc", ptr(x2), ptr(out), c_ll(x2.shape[0]), c_int(x2.shape[1]), c_ll(x2.stride(0)),
              c_ll(rows_per_group), stream())
    return out


def embedding_grad(ids, dx, out):
    """out[ids[p]] += dx[p] for every position p (out fp32 (V, D), e.g. a token table's .grad; dx fp32 or bf16 (..., D)
    over ids' positions).  Deterministic: each table row is summed by one block in position order."""
    D = out.shape[1]
    ids = ids.reshape(-1)
    dx = dx.contiguous().view(-1, D)
    assert ids.dtype == torch.int64 and dx.shape[0] == ids.numel()
    assert dx.dtype in (F32, BF16) and out.dtype == F32 and out.dim() == 2 and out.is_contiguous()
    _lib.call("e4t_embedding_grad", ptr(ids), ptr(dx), c_int(int(dx.dtype == F32)), ptr(out), c_ll(ids.numel()),
              c_int(D), c_ll(out.shape[0]), stream())
    return out


def attn_small_fwd(q, k, v, heads, scale=None, causal=False):
    """Short-sequence attention (N, M <= 128, dh <= 64) with optional causal mask; same layout as attn_fwd."""
    assert q.dtype == BF16 and k.dtype == BF16 and v.dtype == BF16
    assert q.stride(-1) == 1 and k.stride(-1) == 1 and v.stride(-1) == 1
    Bn, N, C = q.shape
    M = k.shape[1]
    dh = C // heads
    scale = dh ** -0.5 if scale is None else scale
    o = torch.empty((Bn, N, C), device=q.device, dtype=BF16)
    lse = torch.empty((Bn, heads, N), device=q.device, dtype=F32)
    _lib.call("e4t_attn_small_fwd", ptr(q), ptr(k), ptr(v), ptr(o), ptr(lse), c_int(Bn), c_int(heads), c_int(N),
              c_int(M), c_int(dh), c_ll(q.stride(1)), c_ll(_bs(q)), c_ll(k.stride(1)), c_ll(_bs(k)), c_ll(v.stride(1)),
              c_ll(_bs(v)), c_ll(o.stride(1)), c_ll(_bs(o)), c_float(scale), c_int(int(causal)), stream())
    return o, lse


def attn_small_bwd(q, k, v, o, do, lse, heads, scale=None, causal=False, dq=None, dk=None, dv=None):
    assert do.dtype == BF16 and do.stride(-1) == 1
    Bn, N, C = q.shape
    M = k.shape[1]
    dh = C // heads
    scale = dh ** -0.5 if scale is None else scale
    dq = torch.empty((Bn, N, C), device=q.device, dtype=BF16) if dq is None else dq
    dk = torch.empty((Bn, M, C), device=q.device, dtype=BF16) if dk is None else dk
    dv = torch.empty((Bn, M, C), device=q.device, dtype=BF16) if dv is None else dv
    _lib.call("e4t_attn_small_bwd", ptr(q), ptr(k), ptr(v), ptr(o), ptr(do), ptr(lse), ptr(dq), ptr(dk), ptr(dv),
              c_int(Bn), c_int(heads), c_int(N), c_int(M), c_int(dh), c_ll(q.stride(1)), c_ll(_bs(q)),
              c_ll(k.stride(1)), c_ll(_bs(k)), c_ll(v.stride(1)), c_ll(_bs(v)), c_ll(o.stride(1)), c_ll(_bs(o)),
              c_ll(do.stride(1)), c_ll(_bs(do)), c_ll(dq.stride(1)), c_ll(_bs(dq)), c_ll(dk.stride(1)), c_ll(_bs(dk)),
              c_ll(dv.stride(1)), c_ll(_bs(dv)), c_float(scale), c_int(int(causal)), stream())
    return dq, dk, dv


def layernorm_param_grad(x, dy, stats, gamma):
    """(dgamma, dbeta) fp32 of LayerNorm given the forward's (mean, rstd) stats."""
    C = x.shape[-1]
    rows = x.numel() // C
    dg = torch.zeros(C, device=x.device, dtype=F32)
    db = torch.zeros(C, device=x.device, dtype=F32)
    _lib.call("e4t_layernorm_param_grad", ptr(x), ptr(dy), ptr(stats), ptr(gamma), ptr(dg), ptr(db), c_ll(rows), c_int(C),
              stream())
    return dg, db


def groupnorm_param_grad(x, dy, stats, gamma, beta, groups, eps, silu):
    """(dgamma, dbeta) fp32 of GroupNorm(+SiLU); stats = groupnorm_fwd's stats of x."""
    assert x.is_contiguous() and dy.is_contiguous() and stats.is_contiguous()
    Bn, C = x.shape[0], x.shape[-1]
    HW = x.numel() // (Bn * C)
    assert stats.shape == (Bn, groups, 3)
    dg = torch.zeros(C, device=x.device, dtype=F32)
    db = torch.zeros(C, device=x.device, dtype=F32)
    _lib.call("e4t_groupnorm_param_grad", ptr(x), ptr(dy), ptr(stats), ptr(gamma), ptr(beta), ptr(dg), ptr(db),
              c_int(Bn), c_int(HW), c_int(C), c_int(groups), c_float(eps), c_int(int(silu)), stream())
    return dg, db


def narrow_conv_wgrad(wide, narrow, sgn):
    """acc[w][n][tap] = sum wide[b,y,x,w] * narrow[b,n,y+sgn*(ky-1),x+sgn*(kx-1)] (weight gradients of conv_in / conv_out)."""
    assert wide.dtype == BF16 and wide.is_contiguous() and narrow.dtype == F32 and narrow.is_contiguous()
    Bn, H, W, Cw = wide.shape
    Cn = narrow.shape[1]
    assert narrow.shape == (Bn, Cn, H, W)
    acc = torch.zeros((Cw, Cn, 9), device=wide.device, dtype=F32)
    _lib.call("e4t_narrow_conv_wgrad", ptr(wide), ptr(narrow), ptr(acc), c_int(Bn), c_int(H), c_int(W), c_int(Cw),
              c_int(Cn), c_int(sgn), stream())
    return acc


def conv3x3_wgrad(x, dy):
    """dW9 fp32 (9, Cout, Cin) of a 3x3/s1/p1 convolution on NHWC bf16 (x: (B,H,W,Cin), dy: (B,H,W,Cout))."""
    assert x.dtype == BF16 and dy.dtype == BF16 and x.is_contiguous() and dy.is_contiguous()
    Bn, H, W, Cin = x.shape
    Cout = dy.shape[-1]
    dw9 = torch.zeros((9, Cout, Cin), device=x.device, dtype=F32)
    _lib.call("e4t_conv3x3_wgrad", ptr(x), ptr(dy), ptr(dw9), c_int(Bn), c_int(H), c_int(W), c_int(Cin), c_int(Cout),
              stream())
    return dw9


# ----------------------------------------------------------------------------------------------
# token merging (csrc/tome.cu)
# ----------------------------------------------------------------------------------------------
TOME_MAX_TOKENS = 16384   # tokens per image the select kernel takes (a 128 x 128 latent)


def _tome_need(cond, msg):
    if not cond:
        raise _lib.E4TError(f"token merging: {msg}")


def tome_match(x, pattern, h, w, sy, sx):
    """Bipartite matching of x (B, h*w, C) bf16 (C % 64 == 0): one dst token per sy x sx cell at offset pattern[cy, cx]
    (int32 (h // sy, w // sx) CUDA tensor), every other token src.  Returns dict(slot (N,), src_idx (Ns,), dst_idx
    (Nd,), node_max (B, Ns) fp32, node_idx (B, Ns) int32 raster index of the best dst)."""
    _tome_need(x.is_cuda and x.dtype == BF16 and x.dim() == 3 and x.is_contiguous(), "x must be a contiguous (B, N, C) "
               "bf16 CUDA tensor")
    Bn, N, C = x.shape
    _tome_need(h > 0 and w > 0 and h * w == N, f"{N} tokens are not an {h} x {w} grid")
    _tome_need(C % 64 == 0, f"C = {C} is not a multiple of 64")
    _tome_need(sy >= 1 and sx >= 1, f"stride ({sy}, {sx}) must be >= 1")
    hc, wc = h // sy, w // sx
    _tome_need(pattern.is_cuda and pattern.dtype == torch.int32 and pattern.is_contiguous()
               and tuple(pattern.shape) == (hc, wc), f"pattern must be a contiguous int32 ({hc}, {wc}) CUDA tensor")
    Nd = hc * wc
    Ns = N - Nd
    i32 = dict(device=x.device, dtype=torch.int32)
    slot, src_idx, dst_idx = torch.empty(N, **i32), torch.empty(max(Ns, 1), **i32), torch.empty(max(Nd, 1), **i32)
    src_n = torch.empty((Bn, max(Ns, 1), C), device=x.device, dtype=BF16)
    dst_n = torch.empty((Bn, max(Nd, 1), C), device=x.device, dtype=BF16)
    node_max = torch.empty((Bn, Ns), device=x.device, dtype=F32)
    node_idx = torch.empty((Bn, Ns), **i32)
    _lib.call("e4t_tome_match", ptr(x), ptr(pattern), c_int(Bn), c_int(h), c_int(w), c_int(C), c_int(sy), c_int(sx),
              ptr(slot), ptr(src_idx), ptr(dst_idx), ptr(src_n), ptr(dst_n), ptr(node_max), ptr(node_idx), stream())
    return dict(slot=slot, src_idx=src_idx[:Ns], dst_idx=dst_idx[:Nd], node_max=node_max, node_idx=node_idx)


def tome_select(m, r):
    """Merge the r src tokens of each image with the largest node_max (ties to the lower raster index) given
    tome_match's result `m`.  Returns dict(pos (B, N), row_off (B, N - r + 1), members (B, N) int32, w (B, N - r)
    fp32 = 1 / row length)."""
    Bn, Ns = m["node_max"].shape
    N, Nd = m["slot"].numel(), m["dst_idx"].numel()
    _tome_need(N <= TOME_MAX_TOKENS, f"{N} tokens per image; the select kernel takes at most {TOME_MAX_TOKENS} "
               "(a 128 x 128 latent)")
    _tome_need(0 <= r <= Ns and (r == 0 or Nd > 0), f"r = {r} with {Ns} src and {Nd} dst tokens")
    dev = m["slot"].device
    i32 = dict(device=dev, dtype=torch.int32)
    seg = torch.empty((Bn, 2, max(Nd, 1)), **i32)
    pos, members = torch.empty((Bn, N), **i32), torch.empty((Bn, N), **i32)
    row_off = torch.empty((Bn, N - r + 1), **i32)
    w = torch.empty((Bn, N - r), device=dev, dtype=F32)
    _lib.call("e4t_tome_select", ptr(m["node_max"]), ptr(m["node_idx"]), ptr(m["slot"]), ptr(m["src_idx"]), c_int(Bn),
              c_int(N), c_int(Ns), c_int(Nd), c_int(r), ptr(seg), ptr(pos), ptr(row_off), ptr(members), ptr(w),
              stream())
    return dict(pos=pos, row_off=row_off, members=members, w=w)


def _tome_rows(t, name, Bn, n, C):
    _tome_need(t.is_cuda and t.dtype == BF16 and t.is_contiguous() and tuple(t.shape) == (Bn, n, C),
               f"{name} must be a contiguous bf16 ({Bn}, {n}, {C}) CUDA tensor, got {tuple(t.shape)} {t.dtype}")


def tome_gather_reduce(x, plan, weighted):
    """(B, N, C) -> (B, N', C): row p = (1 / len if weighted else 1) * sum of x over the members of merged row p."""
    Bn, N = plan["pos"].shape
    Nm = plan["w"].shape[1]
    C = x.shape[-1]
    _tome_rows(x, "x", Bn, N, C)
    _tome_need(C % 8 == 0, f"C = {C} is not a multiple of 8")
    out = torch.empty((Bn, Nm, C), device=x.device, dtype=BF16)
    _lib.call("e4t_tome_gather_reduce", ptr(x), ptr(plan["row_off"]), ptr(plan["members"]),
              ptr(plan["w"] if weighted else None), ptr(out), c_int(Bn), c_int(N), c_int(Nm), c_int(C), stream())
    return out


def tome_gather_expand(y, plan, weighted, residual=None):
    """(B, N', C) -> (B, N, C): out[i] = (w[pos i] if weighted else 1) * y[pos i] (+ residual[i])."""
    Bn, N = plan["pos"].shape
    Nm = plan["w"].shape[1]
    C = y.shape[-1]
    _tome_rows(y, "y", Bn, Nm, C)
    _tome_need(C % 8 == 0, f"C = {C} is not a multiple of 8")
    if residual is not None:
        _tome_rows(residual, "residual", Bn, N, C)
    out = torch.empty((Bn, N, C), device=y.device, dtype=BF16)
    _lib.call("e4t_tome_gather_expand", ptr(y), ptr(plan["pos"]), ptr(plan["w"] if weighted else None),
              ptr(residual), ptr(out), c_int(Bn), c_int(Nm), c_int(N), c_int(C), stream())
    return out
