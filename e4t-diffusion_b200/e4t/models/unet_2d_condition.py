"""UNet2DConditionModel — mirror of e4t/models/unet_2d_condition.py:36-562 (diffusers 0.14.0 config surface plus the
E4T `return_encoder_outputs` early exit, 517-521), running channels-last bf16 on the sm_90a kernels.

Public tensors keep the reference's logical shapes: `sample` in/out is (B,4,H,W); the 13 encoder feature maps are
returned as (B,C,H,W) *views* of the channels-last bf16 buffers (torch.channels_last strides, no copy)."""
import math
from dataclasses import dataclass
from typing import Any, Dict, Optional, Tuple, Union

import torch
import torch.nn as nn
import torch.nn.functional as F

from e4t._mixins import BaseOutput, ConfigMixin, ModelMixin, register_to_config
from e4t.models.resnet import ResnetBlock2D
from e4t.models.unet_2d_blocks import (CrossAttnDownBlock2D, CrossAttnUpBlock2D, DownBlock2D, UNetMidBlock2DCrossAttn,
                                       UpBlock2D, get_down_block, get_up_block)
from e4t_b200 import functional as FN
from e4t_b200 import ops
from e4t_b200._lib import E4TError


@dataclass
class UNet2DConditionOutput(BaseOutput):
    sample: torch.Tensor = None


class Timesteps(nn.Module):
    """diffusers 0.14.0 Timesteps / get_timestep_embedding (sinusoid, [cos,sin] after flip)."""

    def __init__(self, num_channels, flip_sin_to_cos, downscale_freq_shift):
        super().__init__()
        self.num_channels = num_channels
        self.flip_sin_to_cos = flip_sin_to_cos
        self.downscale_freq_shift = downscale_freq_shift

    def forward(self, timesteps):
        half = self.num_channels // 2
        exponent = -math.log(10000) * torch.arange(half, dtype=torch.float32, device=timesteps.device)
        exponent = exponent / (half - self.downscale_freq_shift)
        emb = timesteps[:, None].float() * torch.exp(exponent)[None, :]
        emb = torch.cat([torch.sin(emb), torch.cos(emb)], dim=-1)
        if self.flip_sin_to_cos:
            emb = torch.cat([emb[:, half:], emb[:, :half]], dim=-1)
        return emb


class TimestepEmbedding(nn.Module):
    def __init__(self, in_channels, time_embed_dim, act_fn="silu", out_dim=None, post_act_fn=None, cond_proj_dim=None):
        super().__init__()
        if act_fn != "silu" or post_act_fn is not None or cond_proj_dim is not None:
            raise NotImplementedError("only the SD-v1.x TimestepEmbedding configuration is supported")
        self.linear_1 = nn.Linear(in_channels, time_embed_dim)
        self.act = nn.SiLU()
        self.linear_2 = nn.Linear(time_embed_dim, out_dim if out_dim is not None else time_embed_dim)

    def forward(self, sample, condition=None):
        return self.linear_2(self.act(self.linear_1(sample)))


class UNet2DConditionModel(ModelMixin, ConfigMixin):
    _supports_gradient_checkpointing = True

    @register_to_config
    def __init__(self, sample_size: Optional[int] = None, in_channels: int = 4, out_channels: int = 4,
                 center_input_sample: bool = False, flip_sin_to_cos: bool = True, freq_shift: int = 0,
                 down_block_types: Tuple[str] = ("CrossAttnDownBlock2D", "CrossAttnDownBlock2D",
                                                 "CrossAttnDownBlock2D", "DownBlock2D"),
                 mid_block_type: Optional[str] = "UNetMidBlock2DCrossAttn",
                 up_block_types: Tuple[str] = ("UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D",
                                               "CrossAttnUpBlock2D"),
                 only_cross_attention: Union[bool, Tuple[bool]] = False,
                 block_out_channels: Tuple[int] = (320, 640, 1280, 1280), layers_per_block: int = 2,
                 downsample_padding: int = 1, mid_block_scale_factor: float = 1, act_fn: str = "silu",
                 norm_num_groups: Optional[int] = 32, norm_eps: float = 1e-5, cross_attention_dim: int = 1280,
                 attention_head_dim: Union[int, Tuple[int]] = 8, dual_cross_attention: bool = False,
                 use_linear_projection: bool = False, class_embed_type: Optional[str] = None,
                 num_class_embeds: Optional[int] = None, upcast_attention: bool = False,
                 resnet_time_scale_shift: str = "default", time_embedding_type: str = "positional",
                 timestep_post_act: Optional[str] = None, time_cond_proj_dim: Optional[int] = None,
                 conv_in_kernel: int = 3, conv_out_kernel: int = 3,
                 projection_class_embeddings_input_dim: Optional[int] = None):
        super().__init__()
        self.sample_size = sample_size
        self.in_channels = in_channels
        if len(down_block_types) != len(up_block_types):
            raise ValueError(f"Must provide the same number of `down_block_types` as `up_block_types`. "
                             f"`down_block_types`: {down_block_types}. `up_block_types`: {up_block_types}.")
        if len(block_out_channels) != len(down_block_types):
            raise ValueError(f"Must provide the same number of `block_out_channels` as `down_block_types`. "
                             f"`block_out_channels`: {block_out_channels}. `down_block_types`: {down_block_types}.")
        if not isinstance(only_cross_attention, bool) and len(only_cross_attention) != len(down_block_types):
            raise ValueError("Must provide the same number of `only_cross_attention` as `down_block_types`.")
        if not isinstance(attention_head_dim, int) and len(attention_head_dim) != len(down_block_types):
            raise ValueError("Must provide the same number of `attention_head_dim` as `down_block_types`.")
        if (time_embedding_type != "positional" or class_embed_type is not None or num_class_embeds is not None
                or conv_in_kernel != 3 or conv_out_kernel != 3 or norm_num_groups is None
                or mid_block_type != "UNetMidBlock2DCrossAttn"):
            raise NotImplementedError("configuration outside the SD-v1.x E4T path (SURVEY.md §8)")

        self.conv_in = nn.Conv2d(in_channels, block_out_channels[0], kernel_size=3, padding=1)
        time_embed_dim = block_out_channels[0] * 4
        self.time_proj = Timesteps(block_out_channels[0], flip_sin_to_cos, freq_shift)
        self.time_embedding = TimestepEmbedding(block_out_channels[0], time_embed_dim, act_fn=act_fn,
                                                post_act_fn=timestep_post_act, cond_proj_dim=time_cond_proj_dim)
        self.class_embedding = None
        self.down_blocks = nn.ModuleList([])
        self.up_blocks = nn.ModuleList([])
        if isinstance(only_cross_attention, bool):
            only_cross_attention = [only_cross_attention] * len(down_block_types)
        if isinstance(attention_head_dim, int):
            attention_head_dim = (attention_head_dim,) * len(down_block_types)

        output_channel = block_out_channels[0]
        for i, down_block_type in enumerate(down_block_types):
            input_channel = output_channel
            output_channel = block_out_channels[i]
            is_final_block = i == len(block_out_channels) - 1
            self.down_blocks.append(get_down_block(
                down_block_type, num_layers=layers_per_block, in_channels=input_channel, out_channels=output_channel,
                temb_channels=time_embed_dim, add_downsample=not is_final_block, resnet_eps=norm_eps,
                resnet_act_fn=act_fn, resnet_groups=norm_num_groups, cross_attention_dim=cross_attention_dim,
                attn_num_head_channels=attention_head_dim[i], downsample_padding=downsample_padding,
                dual_cross_attention=dual_cross_attention, use_linear_projection=use_linear_projection,
                only_cross_attention=only_cross_attention[i], upcast_attention=upcast_attention,
                resnet_time_scale_shift=resnet_time_scale_shift))

        self.mid_block = UNetMidBlock2DCrossAttn(
            in_channels=block_out_channels[-1], temb_channels=time_embed_dim, resnet_eps=norm_eps,
            resnet_act_fn=act_fn, output_scale_factor=mid_block_scale_factor,
            resnet_time_scale_shift=resnet_time_scale_shift, cross_attention_dim=cross_attention_dim,
            attn_num_head_channels=attention_head_dim[-1], resnet_groups=norm_num_groups,
            dual_cross_attention=dual_cross_attention, use_linear_projection=use_linear_projection,
            upcast_attention=upcast_attention)

        self.num_upsamplers = 0
        reversed_block_out_channels = list(reversed(block_out_channels))
        reversed_attention_head_dim = list(reversed(attention_head_dim))
        only_cross_attention = list(reversed(only_cross_attention))
        output_channel = reversed_block_out_channels[0]
        for i, up_block_type in enumerate(up_block_types):
            is_final_block = i == len(block_out_channels) - 1
            prev_output_channel = output_channel
            output_channel = reversed_block_out_channels[i]
            input_channel = reversed_block_out_channels[min(i + 1, len(block_out_channels) - 1)]
            add_upsample = not is_final_block
            if add_upsample:
                self.num_upsamplers += 1
            self.up_blocks.append(get_up_block(
                up_block_type, num_layers=layers_per_block + 1, in_channels=input_channel, out_channels=output_channel,
                prev_output_channel=prev_output_channel, temb_channels=time_embed_dim, add_upsample=add_upsample,
                resnet_eps=norm_eps, resnet_act_fn=act_fn, resnet_groups=norm_num_groups,
                cross_attention_dim=cross_attention_dim, attn_num_head_channels=reversed_attention_head_dim[i],
                dual_cross_attention=dual_cross_attention, use_linear_projection=use_linear_projection,
                only_cross_attention=only_cross_attention[i], upcast_attention=upcast_attention,
                resnet_time_scale_shift=resnet_time_scale_shift))

        self.conv_norm_out = nn.GroupNorm(num_channels=block_out_channels[0], num_groups=norm_num_groups, eps=norm_eps)
        self.conv_act = nn.SiLU()
        self.conv_out = nn.Conv2d(block_out_channels[0], out_channels, kernel_size=3, padding=1)

    @property
    def latent_multiple(self) -> int:
        """Latent heights and widths must be multiples of this: the overall down-sampling factor 2^(levels - 1) (8 for
        SD-v1.4, i.e. images in multiples of 64 px), so every stride-2 convolution sees an even size and each up block
        meets its skip connections at their size.  1 while enable_any_latent_size() is in effect."""
        if getattr(self, "_any_latent_size", False):
            return 1
        return 2 ** (len(self.config.block_out_channels) - 1)

    @property
    def min_latent_size(self) -> int:
        """Smallest latent height and width the UNet takes: 2^(levels - 1), so the deepest level is at least 1 x 1."""
        return 2 ** (len(self.config.block_out_channels) - 1)

    def enable_any_latent_size(self):
        """Accept any latent height and width of at least `min_latent_size` (images in multiples of the VAE's factor,
        8 px for SD): stride-2 convolutions at odd sides give ceil(side / 2), and each up block resizes to its skip
        connection's size, as diffusers does when it forwards the up-sampling size.  Sizes that are multiples of
        2^(levels - 1) run exactly as with the switch off."""
        self._any_latent_size = True

    def disable_any_latent_size(self):
        """Back to the default: latent sides must be multiples of 2^(levels - 1)."""
        self._any_latent_size = False

    # ---- processor plumbing (unet_2d_condition.py:291-341) ---------------------------------------
    @property
    def attn_processors(self) -> Dict[str, Any]:
        procs = {}
        for name, module in self.named_modules():
            if hasattr(module, "set_processor"):
                procs[f"{name}.processor"] = module.processor
        return procs

    def set_attn_processor(self, processor):
        mods = [(n, m) for n, m in self.named_modules() if hasattr(m, "set_processor")]
        if isinstance(processor, dict) and len(processor) != len(mods):
            raise ValueError(f"A dict of processors was passed, but the number of processors {len(processor)} does not "
                             f"match the number of attention layers: {len(mods)}.")
        for n, m in mods:
            m.set_processor(processor[f"{n}.processor"] if isinstance(processor, dict) else processor)

    def set_attention_slice(self, slice_size):
        return None  # attention scores never leave the SM in the fused kernel

    def _set_gradient_checkpointing(self, module, value=False):
        if isinstance(module, (CrossAttnDownBlock2D, DownBlock2D, CrossAttnUpBlock2D, UpBlock2D)):
            module.gradient_checkpointing = value

    def enable_gradient_checkpointing(self):
        raise NotImplementedError("gradient checkpointing is not needed at 180 GB HBM and is not implemented")

    # ---- time embedding -----------------------------------------------------------------------------
    def _resnets(self):
        return [m for m in self.modules() if isinstance(m, ResnetBlock2D) and m.time_emb_proj is not None]

    def _time_embed(self, timesteps, batch, device):
        if not torch.is_tensor(timesteps):
            dtype = torch.float64 if isinstance(timesteps, float) else torch.int64
            timesteps = torch.tensor([timesteps], dtype=dtype, device=device)
        elif len(timesteps.shape) == 0:
            timesteps = timesteps[None].to(device)
        timesteps = timesteps.to(device).expand(batch)
        resnets = self._resnets()
        trainable = torch.is_grad_enabled() and (any(p.requires_grad for p in self.time_embedding.parameters())
                                                 or any(r.time_emb_proj.weight.requires_grad for r in resnets))
        if trainable:
            # tuning_e4t.py trains the whole UNet: the time-embedding MLP and the 22 per-block projections stay on
            # differentiable fp32 torch ops (a (B,320)->(B,1280)->(B,ΣCout) chain, negligible FLOPs); their gradients
            # arrive through the row-add operand of each block's first convolution (Conv3x3Fn returns d(row add))
            t_emb = self.time_proj(timesteps).to(torch.float32)
            emb = self.time_embedding(t_emb)
            w_cat = torch.cat([r.time_emb_proj.weight for r in resnets], dim=0)
            b_cat = torch.cat([r.time_emb_proj.bias for r in resnets], dim=0)
            rows = F.linear(F.silu(emb), w_cat, b_cat)
            off = 0
            for r in resnets:
                c = r.time_emb_proj.out_features
                r._temb_row = (emb, rows[:, off:off + c].contiguous())
                off += c
            return emb
        with torch.no_grad():
            t_emb = self.time_proj(timesteps).to(torch.float32)
            emb = self.time_embedding(t_emb)                                       # unet_2d_condition.py:461-468
            # all ResnetBlock2D time_emb_proj(silu(emb)) projections in ONE fp32 matmul
            ws = [r.time_emb_proj.weight for r in resnets]
            key = tuple((w._version, w.data_ptr()) for w in ws)
            cache = getattr(self, "_temb_cat", None)
            if cache is None or cache[0] != key:
                cache = (key, torch.cat([w.detach().float() for w in ws], dim=0),
                         torch.cat([r.time_emb_proj.bias.detach().float() for r in resnets], dim=0))
                self._temb_cat = cache
            rows = torch.addmm(cache[2], F.silu(emb), cache[1].t())
            off = 0
            for r in resnets:
                c = r.time_emb_proj.out_features
                r._temb_row = (emb, rows[:, off:off + c].contiguous())
                off += c
        return emb

    # ---- forward (unet_2d_condition.py:410-562) -----------------------------------------------------------
    def forward(self, sample, timestep, encoder_hidden_states, class_labels=None, timestep_cond=None,
                attention_mask=None, cross_attention_kwargs=None, down_block_additional_residuals=None,
                mid_block_additional_residual=None, return_dict=True, return_encoder_outputs=False):
        if not sample.is_cuda:
            raise E4TError("e4t UNet2DConditionModel runs on the sm_90a kernels only (no CPU fallback); "
                           "move the model and inputs to a CUDA device")
        if attention_mask is not None or class_labels is not None or down_block_additional_residuals is not None \
                or mid_block_additional_residual is not None:
            raise NotImplementedError("attention_mask / class_labels / ControlNet residuals are not on the E4T path")
        # upsample sizes are forwarded when a side is not a multiple of the overall up factor (:426-436)
        forward_upsample_size = any(s % (2 ** self.num_upsamplers) != 0 for s in sample.shape[-2:])
        if forward_upsample_size and not getattr(self, "_any_latent_size", False):
            raise NotImplementedError("latent size must be a multiple of 2**num_upsamplers "
                                      "(enable_any_latent_size() lifts this)")
        if min(sample.shape[-2:]) < self.min_latent_size:
            raise E4TError(f"latents of {sample.shape[-2]} x {sample.shape[-1]}: the sides must be at least "
                           f"{self.min_latent_size}")
        if not torch.is_grad_enabled():
            FN.bump_nograd_fwd_epoch()      # no-grad forwards always rebuild W_eff from the current parameters
        if self.config.center_input_sample:
            sample = 2 * sample - 1.0
        B = sample.shape[0]
        emb = self._time_embed(timestep, B, sample.device)
        ehs = FN.as_bf16(encoder_hidden_states).contiguous()
        x = FN.ConvInFn.apply(sample, self.conv_in.weight, self.conv_in.bias)       # :481 (the latent input has no grad)
        res = (x,)
        for blk in self.down_blocks:                                               # :485-496
            if getattr(blk, "has_cross_attention", False):
                x, r = blk(hidden_states=x, temb=emb, encoder_hidden_states=ehs,
                           cross_attention_kwargs=cross_attention_kwargs)
            else:
                x, r = blk(hidden_states=x, temb=emb)
            res += r
        x = self.mid_block(x, emb, encoder_hidden_states=ehs, cross_attention_kwargs=cross_attention_kwargs)  # :508
        if return_encoder_outputs:                                                 # :517-521
            res += (x,)
            return dict(down_block_samples=tuple(t.permute(0, 3, 1, 2) for t in res))
        upsample_size = None
        for i, blk in enumerate(self.up_blocks):                                   # :527-551
            n = len(blk.resnets)
            skips, res = res[-n:], res[:-n]
            if i < len(self.up_blocks) - 1 and forward_upsample_size:
                upsample_size = tuple(res[-1].shape[1:3])                          # NHWC: the next skip's (H, W)
            if getattr(blk, "has_cross_attention", False):
                x = blk(hidden_states=x, temb=emb, res_hidden_states_tuple=skips, encoder_hidden_states=ehs,
                        cross_attention_kwargs=cross_attention_kwargs, upsample_size=upsample_size)
            else:
                x = blk(hidden_states=x, temb=emb, res_hidden_states_tuple=skips, upsample_size=upsample_size)
        n = self.conv_norm_out
        x = FN.GroupNormFn.apply(x, n.weight, n.bias, n.num_groups, n.eps, True)  # :554-556
        out = FN.ConvOutFn.apply(x, self.conv_out.weight, self.conv_out.bias)       # :557 -> (B,4,H,W) fp32
        if not return_dict:
            return (out,)
        return UNet2DConditionOutput(sample=out)
