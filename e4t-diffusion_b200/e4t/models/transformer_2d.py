"""Transformer2DModel (continuous-input path) — mirror of e4t/models/transformer_2d.py:149-286.
The reference permutes NCHW -> (B,HW,C) and back around the blocks (two full HBM copies per instance); on
channels-last activations both reshapes are free views and the 1x1 proj_in/proj_out convs are plain GEMMs with the
residual add folded into proj_out's epilogue."""
from dataclasses import dataclass
from typing import Optional

import torch
from torch import nn

from e4t._mixins import BaseOutput, ConfigMixin, ModelMixin, register_to_config
from e4t.models.attention import BasicTransformerBlock
from e4t_b200 import functional as FN


@dataclass
class Transformer2DModelOutput(BaseOutput):
    sample: torch.Tensor = None


def _w1x1_bf16(conv):
    return FN.prepared(conv.weight, "bf16_1x1", lambda w: w.reshape(w.shape[0], w.shape[1]).to(torch.bfloat16).contiguous())


class Transformer2DModel(ModelMixin, ConfigMixin):
    @register_to_config
    def __init__(self, num_attention_heads: int = 16, attention_head_dim: int = 88, in_channels: Optional[int] = None,
                 out_channels: Optional[int] = None, num_layers: int = 1, dropout: float = 0.0, norm_num_groups: int = 32,
                 cross_attention_dim: Optional[int] = None, attention_bias: bool = False,
                 sample_size: Optional[int] = None, num_vector_embeds: Optional[int] = None,
                 patch_size: Optional[int] = None, activation_fn: str = "geglu",
                 num_embeds_ada_norm: Optional[int] = None, use_linear_projection: bool = False,
                 only_cross_attention: bool = False, upcast_attention: bool = False, norm_type: str = "layer_norm",
                 norm_elementwise_affine: bool = True):
        super().__init__()
        if num_vector_embeds is not None or patch_size is not None:
            raise NotImplementedError("vectorised / patched inputs are out of scope (SURVEY.md §2 #4)")
        self.use_linear_projection = use_linear_projection
        self.num_attention_heads = num_attention_heads
        self.attention_head_dim = attention_head_dim
        inner_dim = num_attention_heads * attention_head_dim
        self.is_input_continuous = True
        self.in_channels = in_channels
        self.norm = nn.GroupNorm(num_groups=norm_num_groups, num_channels=in_channels, eps=1e-6, affine=True)
        if use_linear_projection:
            self.proj_in = nn.Linear(in_channels, inner_dim)
        else:
            self.proj_in = nn.Conv2d(in_channels, inner_dim, kernel_size=1, stride=1, padding=0)
        self.transformer_blocks = nn.ModuleList([
            BasicTransformerBlock(inner_dim, num_attention_heads, attention_head_dim, dropout=dropout,
                                  cross_attention_dim=cross_attention_dim, activation_fn=activation_fn,
                                  num_embeds_ada_norm=num_embeds_ada_norm, attention_bias=attention_bias,
                                  only_cross_attention=only_cross_attention, upcast_attention=upcast_attention,
                                  norm_type=norm_type, norm_elementwise_affine=norm_elementwise_affine)
            for _ in range(num_layers)])
        self.out_channels = in_channels if out_channels is None else out_channels
        if use_linear_projection:
            self.proj_out = nn.Linear(inner_dim, in_channels)
        else:
            self.proj_out = nn.Conv2d(inner_dim, in_channels, kernel_size=1, stride=1, padding=0)

    def _w(self, lin):
        if isinstance(lin, nn.Conv2d):
            return _w1x1_bf16(lin)
        return FN.prepared(lin.weight, "bf16", lambda w: w.to(torch.bfloat16).contiguous())

    def forward(self, hidden_states, encoder_hidden_states=None, timestep=None, class_labels=None,
                cross_attention_kwargs=None, return_dict: bool = True):
        """hidden_states: channels-last (B,H,W,C) bf16."""
        x = hidden_states
        B, H, W, C = x.shape
        h = FN.GroupNormFn.apply(x, self.norm.weight, self.norm.bias, self.norm.num_groups, self.norm.eps, False)
        h = FN.LinearFn.apply(h.view(B, H * W, C), self._w(self.proj_in), self.proj_in.bias, None,
                              self.proj_in.weight)                                                   # :253-261
        for block in self.transformer_blocks:                                                           # :268-275
            h = block(h, encoder_hidden_states=encoder_hidden_states, timestep=timestep,
                      cross_attention_kwargs=cross_attention_kwargs, class_labels=class_labels, hw=(H, W))
        out = FN.LinearFn.apply(h, self._w(self.proj_out), self.proj_out.bias, x.view(B, H * W, C),
                                self.proj_out.weight)                                                # :279-286
        out = out.view(B, H, W, C)
        if not return_dict:
            return (out,)
        return Transformer2DModelOutput(sample=out)
