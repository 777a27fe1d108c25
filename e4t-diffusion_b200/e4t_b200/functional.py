"""torch.autograd.Function adapters over the sm_90a kernels (e4t_b200.ops).

Conventions on the device path
  * activations: bf16, channels-last — images are (B,H,W,C) contiguous, tokens are (B,N,C) contiguous
  * parameters: fp32 masters (nn.Parameter); kernels read bf16 operand copies made by `prepared()` and refreshed
    whenever the master's version counter moves (optimizer step, load_state_dict)
  * gradients: every Function returns dX; weight gradients are produced only for the E4T-trainable set
    (WeightOffsets through W_eff, encoder head) — the base UNet weights are never updated by pretrain_e4t.py
    (only `"wo"` and encoder params reach the optimizer, pretrain_e4t.py:274-278), so their grads are not computed.
"""
import torch

from . import ops

BF16 = torch.bfloat16
F32 = torch.float32


PARAM_EPOCH = 0  # bumped by optimisers that update parameters behind torch's version counters (FlatAdamW)


def bump_param_epoch():
    global PARAM_EPOCH
    PARAM_EPOCH += 1


GRAD_READY_HOOKS = {}  # name -> callable, fired from inside backward when a group of gradients is final (engine.py)


def fire_grad_ready(name):
    h = GRAD_READY_HOOKS.get(name)
    if h is not None:
        h()


NOGRAD_FWD_EPOCH = 0  # bumped by every no-grad UNet forward: W_eff is then always rebuilt from the current parameters


def bump_nograd_fwd_epoch():
    global NOGRAD_FWD_EPOCH
    NOGRAD_FWD_EPOCH += 1


def prepared(param, key, fn):
    """Cached derived tensor of a parameter (e.g. its bf16 / re-laid-out copy), refreshed on version change."""
    cache = getattr(param, "_e4t_prep", None)
    if cache is None:
        cache = {}
        try:
            param._e4t_prep = cache
        except Exception:
            return fn(param.detach())
    ent = cache.get(key)
    # PARAM_EPOCH only matters for parameters an arena optimiser updates behind torch's version counter
    ver = (param._version, param.data_ptr(), param.device, PARAM_EPOCH if getattr(param, "_e4t_arena", False) else 0)
    if ent is None or ent[0] != ver:
        with torch.no_grad():
            ent = (ver, fn(param.detach()))
        cache[key] = ent
    return ent[1]


def _c(t):
    return t if t.is_contiguous() else t.contiguous()


def as_bf16(t):
    return t if t.dtype == BF16 else t.to(BF16)


# ----------------------------------------------------------------------------------------------
# dense layers
# ----------------------------------------------------------------------------------------------
def _wgrad_splits(m, C, R):
    """Split-K factor of a weight-gradient GEMM: 0 = chosen inside the library by its tile cost model (gemm.cu auto_splits)."""
    return 0


class LinearFn(torch.autograd.Function):
    """y = x @ Wᵀ (+bias) (+residual).  w: bf16 (N,K) operand copy of the fp32 master `wp` (an nn.Parameter of shape
    (N,K) or (N,K,1,1), or None).  Backward: dX (+ pass-through to residual); and — only when the master weight / bias
    require grad (tuning_e4t.py:139-146 trains every UNet weight, --unfreeze_clip_vision the ViT; pretrain_e4t.py leaves
    them un-optimised, engine.PretrainStep freezes them) — dW = dYᵀ·X as a split-K wgmma GEMM (fp32) and
    db = column sums of dY."""

    @staticmethod
    def forward(ctx, x, w, bias, residual, wp=None):
        shp = x.shape
        x2 = _c(x).view(-1, shp[-1])
        res2 = None if residual is None else _c(residual).view(-1, w.shape[0])
        y = ops.gemm(x2, w, bias=bias, residual=res2)
        need_dw = wp is not None and ctx.needs_input_grad[4]     # (grad mode is off inside forward: ask ctx)
        ctx.save_for_backward(w, x2 if need_dw else None)
        ctx.shp = shp
        ctx.has_res = residual is not None
        ctx.wshape = None if wp is None else tuple(wp.shape)
        return y.view(*shp[:-1], w.shape[0])

    @staticmethod
    def backward(ctx, dy):
        w, x2 = ctx.saved_tensors
        N, K = w.shape
        dy2 = _c(dy).view(-1, N)
        dx = ops.gemm(dy2, w, b_mn=True).view(ctx.shp) if ctx.needs_input_grad[0] else None
        db = dw = None
        if ctx.needs_input_grad[2]:
            db = ops.colsum_acc(dy2, torch.zeros(N, device=dy2.device, dtype=F32))
        if len(ctx.needs_input_grad) > 4 and ctx.needs_input_grad[4] and x2 is not None:
            dw = torch.zeros((N, K), device=dy2.device, dtype=F32)
            ops.gemm(dy2, x2, a_mn=True, b_mn=True, out=dw, accumulate=True, splits=_wgrad_splits(x2.shape[0], N, K))
            kw = 1
            for d in ctx.wshape[1:]:
                kw *= d
            dw = (dw if kw == K else dw[:, :kw]).reshape(ctx.wshape)     # operand copies may be K-padded (ViT patch embed)
        return dx, None, db, (dy if ctx.has_res else None), dw


class QKVLinearFn(torch.autograd.Function):
    """LinearFn for a q|k|v projection whose three weights and biases are separate fp32 masters (the CLIP text tower's
    q_proj / k_proj / v_proj): the forward is one GEMM with the row-concatenated bf16 operand `w` (3D, D) and fp32 bias.
    Backward: dX, and — only for the masters that require grad — ONE dW GEMM (3D x D) and ONE column sum, whose row
    blocks are returned as the three masters' gradients."""

    @staticmethod
    def forward(ctx, x, w, bias, wq, wk, wv, bq, bk, bv):
        shp = x.shape
        x2 = _c(x).view(-1, shp[-1])
        y = ops.gemm(x2, w, bias=bias)
        need_dw = any(ctx.needs_input_grad[3:6])
        ctx.save_for_backward(w, x2 if need_dw else None)
        ctx.shp = shp
        return y.view(*shp[:-1], w.shape[0])

    @staticmethod
    def backward(ctx, dy):
        w, x2 = ctx.saved_tensors
        N, K = w.shape
        D = N // 3
        dy2 = _c(dy).view(-1, N)
        dx = ops.gemm(dy2, w, b_mn=True).view(ctx.shp) if ctx.needs_input_grad[0] else None
        dws = dbs = (None, None, None)
        if x2 is not None:
            dw = torch.zeros((N, K), device=dy2.device, dtype=F32)
            ops.gemm(dy2, x2, a_mn=True, b_mn=True, out=dw, accumulate=True, splits=_wgrad_splits(x2.shape[0], N, K))
            dws = tuple(dw[i * D:(i + 1) * D] if ctx.needs_input_grad[3 + i] else None for i in range(3))
        if any(ctx.needs_input_grad[6:9]):
            db = ops.colsum_acc(dy2, torch.zeros(N, device=dy2.device, dtype=F32))
            dbs = tuple(db[i * D:(i + 1) * D] if ctx.needs_input_grad[6 + i] else None for i in range(3))
        return (dx, None, None) + dws + dbs


class TokenEmbeddingFn(torch.autograd.Function):
    """table[ids] (token-embedding lookup, tuning_e4t.py:297) with the table's gradient from the deterministic
    e4t_embedding_grad kernel.  When an arena optimiser owns the table's .grad (FlatAdamW), the kernel adds into that
    view directly instead of returning a dense (V, D) gradient for autograd to add."""

    @staticmethod
    def forward(ctx, ids, table):
        ctx.save_for_backward(ids)
        ctx.table = table
        return table.detach()[ids]

    @staticmethod
    def backward(ctx, dy):
        (ids,) = ctx.saved_tensors
        table = ctx.table
        if not ctx.needs_input_grad[1]:
            return None, None
        if DIRECT_GRAD_WRITE and getattr(table, "_e4t_arena", False) and table.grad is not None:
            ops.embedding_grad(ids, dy, table.grad)
            return None, None
        return None, ops.embedding_grad(ids, dy, torch.zeros(table.shape, device=dy.device, dtype=F32))


class PositionAddFn(torch.autograd.Function):
    """bf16(x + pos) for token embeddings x (B, N, D) and the position table rows pos (N, D), both fp32 — the CLIP text
    tower's embedding sum rounded to its bf16 activations.  Backward: dX = dY, dpos = sum over the batch of dY as one
    column sum of dY viewed as (B, N*D)."""

    @staticmethod
    def forward(ctx, x, pos):
        ctx.shp = x.shape
        return (x + pos).to(BF16)

    @staticmethod
    def backward(ctx, dy):
        dy = _c(dy)
        B, N, D = ctx.shp
        dx = dy.float() if ctx.needs_input_grad[0] else None
        dpos = None
        if ctx.needs_input_grad[1]:
            dpos = ops.colsum_acc(dy.view(B, N * D), torch.zeros(N * D, device=dy.device, dtype=F32)).view(N, D)
        return dx, dpos


class BatchedLinearFn(torch.autograd.Function):
    """Y[i] = X[i] @ W[i]ᵀ for a stack of independent linears (E4TEncoder's 129 first_linears, encoder.py:159-162, as ONE
    batched wgmma GEMM instead of 129 launches).  x (n,B,K) bf16; w16 (n,N,K) bf16 operand copy of the stacked fp32
    master `wst`.  Backward: dX (batched GEMM) and dW (n,N,K) fp32 = dY[i]ᵀ X[i] (batched, written once — no atomics)."""

    @staticmethod
    def forward(ctx, x, w16, wst):
        x = _c(x)
        y = ops.gemm(x, w16)
        ctx.save_for_backward(x, w16)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w16 = ctx.saved_tensors
        dy = _c(dy)
        dx = ops.gemm(dy, w16, b_mn=True) if ctx.needs_input_grad[0] else None
        dw = None
        if ctx.needs_input_grad[2]:
            dw = torch.empty(w16.shape, device=dy.device, dtype=F32)
            ops.gemm(dy, x, a_mn=True, b_mn=True, out=dw)
        return dx, None, dw


class WOLinearFn(torch.autograd.Function):
    """y = x @ W_effᵀ where W_eff (bf16) is the WeightOffsets-modulated projection (cross_attention.py:506,516,518).
    `carrier` is the fp32 (C,R) autograd handle produced next to W_eff by WOEffectiveFn: the weight gradient is
    returned for it so that it stays fp32 while it is summed over the two UNet passes of a step.
    Backward: dX and dW_eff (split-K wgmma GEMM over the token dim, fp32 atomics)."""

    @staticmethod
    def forward(ctx, x, w_eff, carrier):
        shp = x.shape
        x2 = _c(x).view(-1, shp[-1])
        y = ops.gemm(x2, w_eff)
        ctx.save_for_backward(x2, w_eff)
        ctx.shp = shp
        return y.view(*shp[:-1], w_eff.shape[0])

    @staticmethod
    def backward(ctx, dy):
        x2, w_eff = ctx.saved_tensors
        C, R = w_eff.shape
        dy2 = _c(dy).view(-1, C)
        dx = ops.gemm(dy2, w_eff, b_mn=True).view(ctx.shp) if ctx.needs_input_grad[0] else None
        dw = None
        if ctx.needs_input_grad[2]:
            m = x2.shape[0]
            dw = torch.zeros((C, R), device=x2.device, dtype=F32)
            ops.gemm(dy2, x2, a_mn=True, b_mn=True, out=dw, accumulate=True, splits=_wgrad_splits(m, C, R))
        return dx, None, dw


class WOLinearBankFn(torch.autograd.Function):
    """WOLinearFn for projections managed by a wobank.WOBank: the weight gradient is accumulated (fp32 atomics of the
    split-K GEMM) straight into the bank's dW_eff buffer; `token` only orders the bank's backward after this node."""

    @staticmethod
    def forward(ctx, x, w_eff, dweff, token):
        shp = x.shape
        x2 = _c(x).view(-1, shp[-1])
        y = ops.gemm(x2, w_eff)
        ctx.save_for_backward(x2, w_eff)
        ctx.dweff = dweff
        ctx.shp = shp
        return y.view(*shp[:-1], w_eff.shape[0])

    @staticmethod
    def backward(ctx, dy):
        x2, w_eff = ctx.saved_tensors
        C, R = w_eff.shape
        dy2 = _c(dy).view(-1, C)
        dx = ops.gemm(dy2, w_eff, b_mn=True).view(ctx.shp) if ctx.needs_input_grad[0] else None
        m = x2.shape[0]
        ops.gemm(dy2, x2, a_mn=True, b_mn=True, out=ctx.dweff, accumulate=True, splits=_wgrad_splits(m, C, R))
        return dx, None, None, None


def conv3x3_any(x, w9, **kw):
    """Stride-1 3x3 convolution at any H x W: ops.conv3x3 where its tiled A box covers the size (ops.conv3x3_tiled),
    ops.conv3x3_im2col elsewhere."""
    conv = ops.conv3x3 if ops.conv3x3_tiled(x.shape[1], x.shape[2]) else ops.conv3x3_im2col
    return conv(x, w9, **kw)


class Conv3x3Fn(torch.autograd.Function):
    """3x3/s1/p1 convolution on NHWC (+bias +per-image row add (time embedding) +residual).  Backward: dX via the same
    implicit-GEMM kernel with the flipped/transposed taps; pass-through to residual; and, when the fp32 master weight
    `wp` (Cout,Cin,3,3) / bias / row add require grad (tuning), dW by the implicit-GEMM weight-gradient mode of the
    engine (9 taps x split-K over the pixels), db = column sums of dY, d(row add) = per-image column sums of dY."""

    @staticmethod
    def forward(ctx, x, w9, w9_dgrad, bias, rowgroup, residual, wp=None):
        x = _c(x)
        y = conv3x3_any(x, w9, bias=bias, rowgroup=rowgroup, residual=None if residual is None else _c(residual))
        need_dw = wp is not None and ctx.needs_input_grad[6]
        ctx.save_for_backward(w9_dgrad, x if need_dw else None)
        ctx.has_res = residual is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        w9_dgrad, x = ctx.saved_tensors
        dy = _c(dy)
        Bn, H, W, Cout = dy.shape
        dx = conv3x3_any(dy, w9_dgrad) if ctx.needs_input_grad[0] else None
        db = drow = dw = None
        dy2 = dy.view(-1, Cout)
        if ctx.needs_input_grad[3]:
            db = ops.colsum_acc(dy2, torch.zeros(Cout, device=dy.device, dtype=F32))
        if ctx.needs_input_grad[4]:
            drow = ops.colsum_acc(dy2, torch.zeros((Bn, Cout), device=dy.device, dtype=F32), rows_per_group=H * W)
        if len(ctx.needs_input_grad) > 6 and ctx.needs_input_grad[6] and x is not None:
            dw9 = ops.conv3x3_wgrad(x, dy)                                      # (9, Cout, Cin), tap = ky*3+kx
            dw = dw9.view(3, 3, Cout, -1).permute(2, 3, 0, 1).contiguous()     # -> (Cout, Cin, 3, 3)
        return dx, None, None, db, drow, (dy if ctx.has_res else None), dw


class Conv3x3S2Fn(torch.autograd.Function):
    """3x3 / stride 2 / pad 1 convolution (diffusers Downsample2D) computed directly at the output resolution (the
    implicit-GEMM A operand is gathered with TMA element strides).  Backward: dY is zero-inserted to the input
    resolution (the adjoint of the stride-2 pick) and then follows the stride-1 paths: dX by the dgrad convolution,
    dW / db (only when trainable) by the weight-gradient kernels."""

    @staticmethod
    def forward(ctx, x, w9, w9_dgrad, bias, wp=None):
        x = _c(x)
        y = ops.conv3x3_s2(x, w9, bias=bias)
        need_dw = wp is not None and ctx.needs_input_grad[4]
        ctx.save_for_backward(w9_dgrad, x if need_dw else None)
        ctx.in_hw = tuple(x.shape[1:3])
        return y

    @staticmethod
    def backward(ctx, dy):
        w9_dgrad, x = ctx.saved_tensors
        dy = _c(dy)
        Cout = dy.shape[-1]
        if ctx.in_hw == (2 * dy.shape[1], 2 * dy.shape[2]):
            up = ops.resample2x(dy, 3)                                          # zero insertion
        else:
            up = ops.zero_insert(dy, ctx.in_hw)                                 # to an odd input side
        dx = conv3x3_any(up, w9_dgrad) if ctx.needs_input_grad[0] else None
        db = dw = None
        if ctx.needs_input_grad[3]:
            db = ops.colsum_acc(dy.view(-1, Cout), torch.zeros(Cout, device=dy.device, dtype=F32))
        if len(ctx.needs_input_grad) > 4 and ctx.needs_input_grad[4] and x is not None:
            dw = ops.conv3x3_wgrad(x, up).view(3, 3, Cout, -1).permute(2, 3, 0, 1).contiguous()
        return dx, None, None, db, dw


class ResampleFn(torch.autograd.Function):
    """mode 0: nearest x2 upsample; mode 2: stride-2 pick.  Backward is the adjoint kernel (modes 1 / 3)."""

    @staticmethod
    def forward(ctx, x, mode):
        ctx.mode = mode
        return ops.resample2x(_c(x), mode)

    @staticmethod
    def backward(ctx, dy):
        return ops.resample2x(_c(dy), 1 if ctx.mode == 0 else 3), None


class ResizeNearestFn(torch.autograd.Function):
    """Nearest resize of NHWC to an explicit size (diffusers Upsample2D with output_size); backward is the adjoint.
    An exact 2x size runs the x2 kernel (ResampleFn's modes 0 / 1), so sizes that need no explicit size record no
    new op."""

    @staticmethod
    def forward(ctx, x, size):
        size = tuple(int(s) for s in size)
        ctx.in_hw = tuple(x.shape[1:3])
        ctx.x2 = size == (2 * x.shape[1], 2 * x.shape[2])
        return ops.resample2x(_c(x), 0) if ctx.x2 else ops.resize_nearest(_c(x), size)

    @staticmethod
    def backward(ctx, dy):
        return (ops.resample2x(_c(dy), 1) if ctx.x2 else ops.resize_nearest_bwd(_c(dy), ctx.in_hw)), None


class ConvOutFn(torch.autograd.Function):
    """UNet conv_out: NHWC bf16 -> NCHW fp32 (unet_2d_condition.py:557).  Weight/bias gradients only when trainable."""

    @staticmethod
    def forward(ctx, x, w, bias):
        x = _c(x)
        need_dw = ctx.needs_input_grad[1]
        ctx.save_for_backward(w, x if need_dw else None)
        ctx.C = x.shape[-1]
        return ops.conv_out_fwd(x, w.detach(), bias.detach())

    @staticmethod
    def backward(ctx, dy):
        w, x = ctx.saved_tensors
        dy = _c(dy.float())
        dx = ops.conv_out_bwd(dy, w.detach(), ctx.C) if ctx.needs_input_grad[0] else None
        dw = db = None
        if ctx.needs_input_grad[1] and x is not None:
            acc = ops.narrow_conv_wgrad(x, dy, -1)                              # [ci][co][tap]
            dw = acc.permute(1, 0, 2).reshape(dy.shape[1], ctx.C, 3, 3).contiguous()
        if ctx.needs_input_grad[2]:
            db = dy.sum(dim=(0, 2, 3))
        return dx, dw, db


class ConvInFn(torch.autograd.Function):
    """UNet conv_in: NCHW fp32 latents -> NHWC bf16 (unet_2d_condition.py:481).  The latent input never needs a gradient;
    weight/bias gradients only when trainable."""

    @staticmethod
    def forward(ctx, sample, w, bias):
        sample = _c(sample.detach().float())
        need_dw = ctx.needs_input_grad[1]
        ctx.save_for_backward(sample if need_dw else None)
        ctx.wshape = tuple(w.shape)
        return ops.conv_in_fwd(sample, w.detach(), bias.detach())

    @staticmethod
    def backward(ctx, dy):
        (sample,) = ctx.saved_tensors
        dy = _c(dy)
        dw = db = None
        if ctx.needs_input_grad[1] and sample is not None:
            dw = ops.narrow_conv_wgrad(dy, sample, 1).view(ctx.wshape)          # [co][ci][tap]
        if ctx.needs_input_grad[2]:
            C = dy.shape[-1]
            db = ops.colsum_acc(dy.view(-1, C), torch.zeros(C, device=dy.device, dtype=F32))
        return None, dw, db


# ----------------------------------------------------------------------------------------------
# normalisation / activation
# ----------------------------------------------------------------------------------------------
class GroupNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, groups, eps, silu):
        x = _c(x)
        y, stats = ops.groupnorm_fwd(x, gamma, beta, groups, eps, silu)
        ctx.save_for_backward(x, gamma, beta, stats)
        ctx.cfg = (groups, eps, silu)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, gamma, beta, stats = ctx.saved_tensors
        groups, eps, silu = ctx.cfg
        dy = _c(dy)
        dx = ops.groupnorm_bwd(x, dy, gamma, beta, stats, groups, eps, silu) if ctx.needs_input_grad[0] else None
        dg = db = None
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:      # affine parameters trainable (tuning)
            dg, db = ops.groupnorm_param_grad(x, dy, stats, gamma.detach(), beta.detach(), groups, eps, silu)
        return dx, dg, db, None, None, None


class LayerNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, eps):
        x = _c(x)
        y, stats = ops.layernorm_fwd(x, gamma, beta, eps)
        ctx.save_for_backward(x, gamma, stats)
        ctx.eps = eps
        return y

    @staticmethod
    def backward(ctx, dy):
        x, gamma, stats = ctx.saved_tensors
        dy = _c(dy)
        dx = ops.layernorm_bwd(x, dy, gamma, stats, ctx.eps) if ctx.needs_input_grad[0] else None
        dg = db = None
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:      # affine parameters trainable (tuning / unfrozen ViT)
            dg, db = ops.layernorm_param_grad(x, dy, stats, gamma.detach())
        return dx, dg, db, None


class GEGLUFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, h):
        h = _c(h)
        ctx.save_for_backward(h)
        return ops.geglu_fwd(h)

    @staticmethod
    def backward(ctx, dout):
        (h,) = ctx.saved_tensors
        return ops.geglu_bwd(h, _c(dout))


class ActFn(torch.autograd.Function):
    """Elementwise activation on bf16: mode ops.ACT_GELU (open_clip ViT MLP), ops.ACT_QUICK_GELU (CLIP text MLP),
    ops.ACT_LEAKY_RELU (E4TEncoder head)."""

    @staticmethod
    def forward(ctx, x, mode):
        x = _c(x)
        ctx.save_for_backward(x)
        ctx.mode = mode
        return ops.act_fwd(x, mode)

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        return ops.act_bwd(x, _c(dy), ctx.mode), None


class SmallAttentionFn(torch.autograd.Function):
    """softmax(QKᵀ/sqrt(dh) [+ causal mask]) V for short sequences (N, M <= 128, dh <= 64) on the fused (B,N,3C)
    projection output — the CLIP text tower's causal self-attention (modeling_clip.py:45-51)."""

    @staticmethod
    def forward(ctx, qkv, heads, scale, causal):
        qkv = _c(qkv)
        C = qkv.shape[-1] // 3
        q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
        o, lse = ops.attn_small_fwd(q, k, v, heads, scale, causal)
        ctx.save_for_backward(qkv, o, lse)
        ctx.cfg = (heads, scale, causal)
        return o

    @staticmethod
    def backward(ctx, do):
        qkv, o, lse = ctx.saved_tensors
        heads, scale, causal = ctx.cfg
        C = qkv.shape[-1] // 3
        q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
        d = torch.empty_like(qkv)
        if causal and q.shape[1] == k.shape[1] and (C // heads) % 8 == 0 and C // heads <= 80 and (3 * C) % 8 == 0:
            # tensor-core fused backward with the causal mask (33 us against 129 us for the scalar kernel at the CLIP-L
            # text shape 16 x 12 x 77 x 64, r02 call 21)
            ops.attn_bwd(q, k, v, o, _c(do), lse, heads, scale, dq=d[..., :C], dk=d[..., C:2 * C], dv=d[..., 2 * C:],
                         causal=True)
        else:
            ops.attn_small_bwd(q, k, v, o, _c(do), lse, heads, scale, causal, dq=d[..., :C], dk=d[..., C:2 * C],
                               dv=d[..., 2 * C:])
        return d, None, None, None


# ----------------------------------------------------------------------------------------------
# attention core
# ----------------------------------------------------------------------------------------------
class AttentionFn(torch.autograd.Function):
    """softmax(QKᵀ/sqrt(dh))V on token-major tensors, taking the FUSED projection outputs so that the projection
    backward sees one contiguous gradient:
      self-attention : a = qkv (B,N,3C), b = None      -> grad (B,N,3C)
      cross-attention: a = q (B,N,C),  b = kv (B,M,2C) -> grads (B,N,C), (B,M,2C)"""

    @staticmethod
    def forward(ctx, a, b, heads, scale):
        a = _c(a)
        if b is None:
            C = a.shape[-1] // 3
            q, k, v = a[..., :C], a[..., C:2 * C], a[..., 2 * C:]
        else:
            b = _c(b)
            C = a.shape[-1]
            q, k, v = a, b[..., :C], b[..., C:]
        o, lse = ops.attn_fwd(q, k, v, heads, scale)
        ctx.save_for_backward(a, b, o, lse)
        ctx.cfg = (heads, scale)
        return o

    @staticmethod
    def backward(ctx, do):
        a, b, o, lse = ctx.saved_tensors
        heads, scale = ctx.cfg
        if b is None:
            C = a.shape[-1] // 3
            q, k, v = a[..., :C], a[..., C:2 * C], a[..., 2 * C:]
            da = torch.empty_like(a)
            ops.attn_bwd(q, k, v, o, _c(do), lse, heads, scale, dq=da[..., :C], dk=da[..., C:2 * C], dv=da[..., 2 * C:])
            return da, None, None, None
        C = a.shape[-1]
        q, k, v = a, b[..., :C], b[..., C:]
        da = torch.empty_like(a)
        db = torch.empty_like(b)
        ops.attn_bwd(q, k, v, o, _c(do), lse, heads, scale, dq=da, dk=db[..., :C], dv=db[..., C:])
        return da, db, None, None


# ----------------------------------------------------------------------------------------------
# WeightOffsets: fused effective projection weights of one attention module
# ----------------------------------------------------------------------------------------------
# When an arena optimiser owns the gradients (FlatAdamW: every trainable param's .grad is a zeroed view of one flat
# buffer and each WeightOffsets parameter receives exactly ONE contribution per step), the WO backward kernels write
# straight into those views instead of returning ~900 small tensors for autograd to add.
DIRECT_GRAD_WRITE = False

WO_EPOCH = 0  # bumped by every WOEffectiveFn.backward: cached W_eff graphs are single-use


_WO_FIELDS = ("v", "linear1.weight", "linear1.bias", "linear2.weight", "linear2.bias", "linear_column.weight",
              "linear_column.bias", "linear_row.weight", "linear_row.bias")


class WOEffectiveFn(torch.autograd.Function):
    """W_eff = W ⊙ (1 + Δ), Δ = b·aᵀ + s·b_cᵀ + b_r·1ᵀ (closed form of e4t/weightoffsets.py:14-23) for a GROUP of
    projections that share their input (q,k,v of self-attention; k,v of cross-attention), written into one
    row-concatenated bf16 matrix so that the projection is a single GEMM.

    apply(n, W_1..W_n, (v,w1,β1,w2,β2,Wc,bc,Wr,br)_1..n) -> (W_eff (ΣC_i, R) bf16 [non-differentiable],
                                                             carrier (ΣC_i, R) fp32 [uninitialised autograd handle]).
    Backward: five mat-vec reductions of G = dW_eff ⊙ W per projection -> all nine WeightOffsets parameter grads
    (SURVEY.md Appendix A); G is never materialised."""

    @staticmethod
    def forward(ctx, n, *args):
        Ws = args[:n]
        wo = [args[n + 9 * i:n + 9 * (i + 1)] for i in range(n)]
        R = Ws[0].shape[1]
        Ctot = sum(w.shape[0] for w in Ws)
        out = torch.empty((Ctot, R), device=Ws[0].device, dtype=BF16)
        saved = []
        r0 = 0
        for W, p in zip(Ws, wo):
            v, w1, b1, w2, b2, Wc, bc, Wr, br = p
            vx, vy, a, b, s = ops.wo_factors(v, w1, b1, w2, b2, Wc, Wr)
            ops.wo_weff(W, a, bc, b, s, br, out=out[r0:r0 + W.shape[0]])
            r0 += W.shape[0]
            saved += [vx, vy, a, b, s]
        ctx.n = n
        ctx.save_for_backward(*args, *saved)
        carrier = torch.empty((Ctot, R), device=out.device, dtype=F32)
        ctx.mark_non_differentiable(out)
        return out, carrier

    @staticmethod
    def backward(ctx, _unused, dW):
        global WO_EPOCH
        WO_EPOCH += 1
        n = ctx.n
        t = ctx.saved_tensors
        Ws = t[:n]
        wo = [t[n + 9 * i:n + 9 * (i + 1)] for i in range(n)]
        fac = t[n + 9 * n:]
        dW = _c(dW.float())
        grads, base_grads = [], []
        r0 = 0
        for i, (W, p) in enumerate(zip(Ws, wo)):
            v, w1, b1, w2, b2, Wc, bc, Wr, br = p
            vx, vy, a, b, s = fac[5 * i:5 * i + 5]
            C = W.shape[0]
            # gradients are RETURNED (autograd's AccumulateGrad adds them to .grad, arena view or not), so repeated
            # backward passes before an optimiser step accumulate; the batched WOBank path accumulates in its kernels
            dv, dw1, db1, dw2, db2, dWc, dbc, dWr, dbr = ops.wo_bwd(dW[r0:r0 + C], W, v, w1, w2, Wc, Wr, bc, vx,
                                                                  vy, a, b, s)
            grads += [dv, dw1.view_as(w1), db1, dw2.view_as(w2), db2, dWc, dbc, dWr, dbr]
            if ctx.needs_input_grad[1 + i]:     # base projection weight trainable (tuning): dW = dW_eff ⊙ (1 + Δ)
                delta = b[:, None] * a[None, :] + s[:, None] * bc[None, :] + br[:, None]
                base_grads.append(dW[r0:r0 + C] * (1.0 + delta))
            else:
                base_grads.append(None)
            r0 += C
        return (None,) + tuple(base_grads) + tuple(grads)


# ----------------------------------------------------------------------------------------------
# E4T encoder feature pooling (encoder.py:147-148)
# ----------------------------------------------------------------------------------------------
class MeanPoolCatFn(torch.autograd.Function):
    """cat_k mean_{HW}(map_k) -> (B, ΣC_k) fp32, maps are channels-last bf16 (B,H,W,C)."""

    @staticmethod
    def forward(ctx, *maps):
        B = maps[0].shape[0]
        total = sum(m.shape[-1] for m in maps)
        out = torch.empty((B, total), device=maps[0].device, dtype=F32)
        off = 0
        for m in maps:
            ops.meanpool_fwd(_c(m), out, off)
            off += m.shape[-1]
        ctx.shapes = [tuple(m.shape) for m in maps]
        return out

    @staticmethod
    def backward(ctx, dout):
        # every E4TEncoder-head gradient is final here (this is the head's first forward op, so its last backward op):
        # the data-parallel engine starts their all-reduce now, under the encoder-half UNet backward that follows
        fire_grad_ready("encoder_head")
        dout = _c(dout.float())
        outs = []
        off = 0
        for i, shp in enumerate(ctx.shapes):
            outs.append(ops.meanpool_bwd(dout, shp, off) if ctx.needs_input_grad[i] else None)
            off += shp[-1]
        return tuple(outs)


# ----------------------------------------------------------------------------------------------
# token merging (e4t_b200/tome.py): both maps are linear in the tokens; the plan (matching) carries no gradient
# ----------------------------------------------------------------------------------------------
class ToMeMergeFn(torch.autograd.Function):
    """(B, N, C) -> (B, N', C): each merged row is the mean of its members.  Backward: dx[i] = dy[pos i] / len."""

    @staticmethod
    def forward(ctx, x, plan):
        ctx.plan = plan
        return ops.tome_gather_reduce(_c(as_bf16(x)), plan, weighted=True)

    @staticmethod
    def backward(ctx, dy):
        return ops.tome_gather_expand(_c(dy), ctx.plan, weighted=True), None


class ToMeUnmergeFn(torch.autograd.Function):
    """(B, N', C) -> (B, N, C): out[i] = y[pos i] + residual[i].  Backward: dy[p] = sum of dout over row p's
    members; dresidual = dout."""

    @staticmethod
    def forward(ctx, y, plan, residual):
        ctx.plan = plan
        return ops.tome_gather_expand(_c(y), plan, weighted=False, residual=_c(residual))

    @staticmethod
    def backward(ctx, dout):
        dout = _c(dout)
        return ops.tome_gather_reduce(dout, ctx.plan, weighted=False), None, dout
