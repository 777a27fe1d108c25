"""BasicTransformerBlock / FeedForward / GEGLU — mirror of e4t/models/attention.py:181-430 on the sm_90a kernels.
LayerNorm -> attn1 (self) -> LayerNorm -> attn2 (cross) -> LayerNorm -> GEGLU feed-forward, residual adds fused into
the producing GEMM epilogues.  AttentionBlock (attention.py:37-178): the VAE mid-block's single-head attention,
forward only."""
import math
from typing import Optional

import torch
from torch import nn

from e4t.models.cross_attention import CrossAttention, _weight_bf16
from e4t_b200 import functional as FN


class GEGLU(nn.Module):
    """attention.py:409-430: proj: dim_in -> 2*dim_out, out = h * gelu(gate) (exact erf GELU)."""

    def __init__(self, dim_in: int, dim_out: int):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out * 2)

    def forward(self, hidden_states):
        h = FN.LinearFn.apply(hidden_states, _weight_bf16(self.proj), self.proj.bias, None, self.proj.weight)
        return FN.GEGLUFn.apply(h)


class FeedForward(nn.Module):
    """attention.py:335-384 (activation_fn='geglu', the only variant SD-v1.x builds)."""

    def __init__(self, dim: int, dim_out: Optional[int] = None, mult: int = 4, dropout: float = 0.0,
                 activation_fn: str = "geglu", final_dropout: bool = False):
        super().__init__()
        if activation_fn != "geglu":
            raise NotImplementedError("only GEGLU feed-forward is on the SD-v1.x path")
        inner_dim = int(dim * mult)
        dim_out = dim_out if dim_out is not None else dim
        self.net = nn.ModuleList([GEGLU(dim, inner_dim), nn.Dropout(dropout), nn.Linear(inner_dim, dim_out)])

    def forward(self, hidden_states, residual=None):
        h = self.net[0](hidden_states)
        return FN.LinearFn.apply(h, _weight_bf16(self.net[2]), self.net[2].bias, residual, self.net[2].weight)


class BasicTransformerBlock(nn.Module):
    """attention.py:181-332."""

    def __init__(self, dim: int, num_attention_heads: int, attention_head_dim: int, dropout=0.0,
                 cross_attention_dim: Optional[int] = None, activation_fn: str = "geglu",
                 num_embeds_ada_norm: Optional[int] = None, attention_bias: bool = False,
                 only_cross_attention: bool = False, upcast_attention: bool = False,
                 norm_elementwise_affine: bool = True, norm_type: str = "layer_norm", final_dropout: bool = False):
        super().__init__()
        if norm_type != "layer_norm" or num_embeds_ada_norm is not None or only_cross_attention:
            raise NotImplementedError("AdaLayerNorm / only_cross_attention are not on the SD-v1.x path")
        self.only_cross_attention = only_cross_attention
        self.attn1 = CrossAttention(query_dim=dim, heads=num_attention_heads, dim_head=attention_head_dim,
                                    dropout=dropout, bias=attention_bias, upcast_attention=upcast_attention)
        self.ff = FeedForward(dim, dropout=dropout, activation_fn=activation_fn, final_dropout=final_dropout)
        self.attn2 = CrossAttention(query_dim=dim, cross_attention_dim=cross_attention_dim, heads=num_attention_heads,
                                    dim_head=attention_head_dim, dropout=dropout, bias=attention_bias,
                                    upcast_attention=upcast_attention) if cross_attention_dim is not None else None
        self.norm1 = nn.LayerNorm(dim, elementwise_affine=norm_elementwise_affine)
        self.norm2 = nn.LayerNorm(dim, elementwise_affine=norm_elementwise_affine) if self.attn2 is not None else None
        self.norm3 = nn.LayerNorm(dim, elementwise_affine=norm_elementwise_affine)

    _tome = None   # the token-merging patch in force (e4t_b200.tome.apply_patch), shared by the UNet's blocks

    @staticmethod
    def _ln(norm, x):
        return FN.LayerNormFn.apply(x, norm.weight, norm.bias, norm.eps)

    def forward(self, hidden_states, encoder_hidden_states=None, timestep=None, attention_mask=None,
                cross_attention_kwargs=None, class_labels=None, hw=None):
        """hw: the (H, W) grid of the tokens, which token merging needs (Transformer2DModel passes it)."""
        kw = cross_attention_kwargs if cross_attention_kwargs is not None else {}
        x = FN.as_bf16(hidden_states)
        if self._tome is not None and hw is not None:
            from e4t_b200 import tome
            plan = tome.plan(self._tome, x, hw)
            if plan is not None:
                return self._forward_merged(x, plan, self._tome["args"], encoder_hidden_states, attention_mask, kw)
        x = self.attn1(self._ln(self.norm1, x), encoder_hidden_states=None, attention_mask=attention_mask,
                       residual=x, **kw)                                                   # attention.py:291-302
        if self.attn2 is not None:
            x = self.attn2(self._ln(self.norm2, x), encoder_hidden_states=encoder_hidden_states,
                           attention_mask=attention_mask, residual=x, **kw)                # :304-316
        return self.ff(self._ln(self.norm3, x), residual=x)                                # :318-330

    def _forward_merged(self, x, plan, a, encoder_hidden_states, attention_mask, kw):
        """tomesd's patched block: each sub-layer that merges runs on the N - r merged tokens and is unmerged with the
        residual added by the same kernel (its out-projection then runs without the fused residual)."""
        if a.merge_attn:
            h = FN.ToMeMergeFn.apply(self._ln(self.norm1, x), plan)
            x = FN.ToMeUnmergeFn.apply(self.attn1(h, encoder_hidden_states=None, attention_mask=attention_mask, **kw),
                                       plan, x)
        else:
            x = self.attn1(self._ln(self.norm1, x), encoder_hidden_states=None, attention_mask=attention_mask,
                           residual=x, **kw)
        if self.attn2 is not None:
            if a.merge_crossattn:
                h = FN.ToMeMergeFn.apply(self._ln(self.norm2, x), plan)
                x = FN.ToMeUnmergeFn.apply(self.attn2(h, encoder_hidden_states=encoder_hidden_states,
                                                      attention_mask=attention_mask, **kw), plan, x)
            else:
                x = self.attn2(self._ln(self.norm2, x), encoder_hidden_states=encoder_hidden_states,
                               attention_mask=attention_mask, residual=x, **kw)
        if a.merge_mlp:
            return FN.ToMeUnmergeFn.apply(self.ff(FN.ToMeMergeFn.apply(self._ln(self.norm3, x), plan)), plan, x)
        return self.ff(self._ln(self.norm3, x), residual=x)


# the fp32 score matrix of one image is N² · 4 bytes (64 MiB at a 64 x 64 latent); images are processed in chunks
# whose scores stay under this bound, and never fewer than one image per chunk: above 128 x 128 latent tokens one image
# is already over it (1.2 GB of scores + 0.6 GB of bf16 probabilities at 1088 x 1024 px, 2.4 + 1.2 GB at 1024 x 1536)
ATTN_SCORE_BYTES = 1 << 30


class AttentionBlock(nn.Module):
    """attention.py:37-178 — the single-head spatial self-attention of the VAE mid-block (diffusers 0.14, forward only).
    GroupNorm (no SiLU) -> q|k|v as ONE GEMM with bias (weights row-concatenated) -> S = scale·Q·Kᵀ in fp32 (batched
    GEMM) -> row softmax to bf16 -> O = P·V (V MN-major) -> proj_attn with bias and the residual in the epilogue.
    The reference order of operations (:152-177): scores in the working dtype, softmax in fp32, (h + residual) / 1."""

    def __init__(self, channels: int, num_head_channels: Optional[int] = None, norm_num_groups: int = 32,
                 rescale_output_factor: float = 1.0, eps: float = 1e-5):
        super().__init__()
        self.channels = channels
        self.num_heads = channels // num_head_channels if num_head_channels is not None else 1
        self.num_head_size = num_head_channels
        self.group_norm = nn.GroupNorm(num_channels=channels, num_groups=norm_num_groups, eps=eps, affine=True)
        self.query = nn.Linear(channels, channels)
        self.key = nn.Linear(channels, channels)
        self.value = nn.Linear(channels, channels)
        self.rescale_output_factor = rescale_output_factor
        self.proj_attn = nn.Linear(channels, channels, 1)

    def _qkv(self):
        """q|k|v weights row-concatenated into one bf16 GEMM operand + fp32 bias; cached on query's parameters and
        keyed on the versions and storage of key's and value's, so an update of any of the three rebuilds them."""
        ps = (self.query, self.key, self.value)
        kv = lambda n: tuple((getattr(p, n)._version, getattr(p, n).data_ptr()) for p in ps[1:])
        w = FN.prepared(self.query.weight, ("vae_qkv_w",) + kv("weight"),
                        lambda _: torch.cat([p.weight.detach() for p in ps], 0).to(torch.bfloat16).contiguous())
        b = FN.prepared(self.query.bias, ("vae_qkv_b",) + kv("bias"),
                        lambda _: torch.cat([p.bias.detach() for p in ps], 0).float().contiguous())
        return w, b

    def forward(self, hidden_states):
        """hidden_states: channels-last (B, H, W, C) bf16 CUDA tensor."""
        if self.num_heads != 1 or self.rescale_output_factor != 1.0:
            raise NotImplementedError("only the single-head, unscaled AttentionBlock of the VAE is supported")
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError("AttentionBlock runs inference only (no backward)")
        from e4t.models.resnet import f32
        from e4t_b200 import ops
        x = FN._c(FN.as_bf16(hidden_states))
        B, H, W, C = x.shape
        N = H * W
        gn = self.group_norm
        h = ops.groupnorm_fwd(x, f32(gn.weight), f32(gn.bias), gn.num_groups, gn.eps, False)[0]
        w_qkv, b_qkv = self._qkv()
        qkv = ops.gemm(h.view(B * N, C), w_qkv, bias=b_qkv).view(B, N, 3 * C)
        scale = 1.0 / math.sqrt(C / self.num_heads)
        o = torch.empty((B, N, C), device=x.device, dtype=torch.bfloat16)
        # N % 8 != 0 (a latent with an odd side): the score and probability rows get a pitch of Np = N rounded up to 8
        # elements, which TMA and the softmax's vector loads need.  The pad columns of the scores are set to -inf after
        # the GEMM, so their probabilities are exact zeros; P·V reads K = N columns of P (its K tail is TMA
        # out-of-bounds zero fill)
        Np = (N + 7) // 8 * 8
        chunk = max(1, ATTN_SCORE_BYTES // (N * Np * 4))
        for i in range(0, B, chunk):
            q, k, v = qkv[i:i + chunk, :, :C], qkv[i:i + chunk, :, C:2 * C], qkv[i:i + chunk, :, 2 * C:]
            if Np == N:
                s = ops.gemm(q, k, alpha=scale, out_dtype=torch.float32)           # (b, N, N) fp32
                p = ops.softmax_rows(s)
            else:
                s = torch.empty((q.shape[0], N, Np), device=x.device, dtype=torch.float32)
                ops.gemm(q, k, alpha=scale, out=s[..., :N])
                s[..., N:] = float("-inf")
                p = ops.softmax_rows(s)[..., :N]
            del s
            ops.gemm(p, v, b_mn=True, out=o[i:i + chunk])
        w_o = FN.prepared(self.proj_attn.weight, "bf16", lambda t: t.to(torch.bfloat16).contiguous())
        out = ops.gemm(o.view(B * N, C), w_o, bias=f32(self.proj_attn.bias), residual=x.view(B * N, C))
        return out.view(B, H, W, C)
