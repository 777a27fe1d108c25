"""Encoder / Decoder / DiagonalGaussianDistribution / DecoderOutput — the composition of diffusers 0.14 models/vae.py,
restated on the sm_90a kernels (forward only; the VAE is frozen in pre-training and runs under no_grad in inference).
Parameter names and shapes are diffusers'.  The ends take and return NCHW fp32 like the UNet's conv_in / conv_out
(narrow direct-convolution kernels); everything between runs on channels-last bf16 activations (B,H,W,C): GroupNorm(+SiLU)
kernels, the wgmma implicit-GEMM 3x3 convolution (stride 1, stride 2 with padding 0, wide rows) and the mid-block
AttentionBlock (GEMMs + row softmax)."""
from dataclasses import dataclass
from typing import Optional

import torch
import torch.nn.functional as F
from torch import nn

from e4t._mixins import BaseOutput
from e4t.models.resnet import f32
from e4t.models.unet_2d_blocks import UNetMidBlock2D, get_down_block, get_up_block
from e4t_b200 import functional as FN
from e4t_b200 import ops


@dataclass
class DecoderOutput(BaseOutput):
    sample: torch.FloatTensor = None


def _conv_in(conv, x):
    """NCHW (any float dtype) -> NHWC bf16 through the narrow direct 3x3 kernel (Cin <= 16)."""
    return ops.conv_in_fwd(FN._c(x.float()), f32(conv.weight).contiguous(), f32(conv.bias))


def _norm_act_out(norm, conv, h, engine=False):
    """conv_norm_out + SiLU + conv_out: NHWC bf16 -> NCHW fp32.
    engine=False: the narrow direct 3x3 kernel (CUDA cores, Cout <= 8).  engine=True: the wgmma implicit-GEMM conv with
    Cout zero-padded to 64 and an fp32 store, then the first Cout channels as NCHW (the decoder's 128 -> 3 at 512²: one
    warp per pixel took 16.1 ms of a 113 ms B = 16 decode on an H100, DESIGN §5)."""
    h = ops.groupnorm_fwd(FN._c(h), f32(norm.weight), f32(norm.bias), norm.num_groups, norm.eps, True)[0]
    if not engine:
        return ops.conv_out_fwd(h, f32(conv.weight).contiguous(), f32(conv.bias))
    co = conv.out_channels
    w9 = FN.prepared(conv.weight, "w9_pad64", lambda w: F.pad(w.float(), (0, 0, 0, 0, 0, 0, 0, 64 - co))
                     .permute(2, 3, 0, 1).reshape(9, 64, w.shape[1]).to(torch.bfloat16).contiguous())
    b = FN.prepared(conv.bias, "f32_pad64", lambda t: F.pad(t.float(), (0, 64 - co)).contiguous())
    y = FN.conv3x3_any(h, w9, bias=b, out_dtype=torch.float32)                    # (B, H, W, 64) fp32
    return y[..., :co].permute(0, 3, 1, 2).contiguous()


class Encoder(nn.Module):
    def __init__(self, in_channels=3, out_channels=3, down_block_types=("DownEncoderBlock2D",),
                 block_out_channels=(64,), layers_per_block=2, norm_num_groups=32, act_fn="silu", double_z=True):
        super().__init__()
        self.layers_per_block = layers_per_block
        self.conv_in = nn.Conv2d(in_channels, block_out_channels[0], kernel_size=3, stride=1, padding=1)
        self.mid_block = None
        self.down_blocks = nn.ModuleList([])
        output_channel = block_out_channels[0]
        for i, down_block_type in enumerate(down_block_types):
            input_channel = output_channel
            output_channel = block_out_channels[i]
            is_final_block = i == len(block_out_channels) - 1
            self.down_blocks.append(get_down_block(
                down_block_type, num_layers=self.layers_per_block, in_channels=input_channel,
                out_channels=output_channel, add_downsample=not is_final_block, resnet_eps=1e-6, downsample_padding=0,
                resnet_act_fn=act_fn, resnet_groups=norm_num_groups, attn_num_head_channels=None, temb_channels=None))
        self.mid_block = UNetMidBlock2D(in_channels=block_out_channels[-1], resnet_eps=1e-6, resnet_act_fn=act_fn,
                                        output_scale_factor=1, resnet_time_scale_shift="default",
                                        attn_num_head_channels=None, resnet_groups=norm_num_groups, temb_channels=None)
        self.conv_norm_out = nn.GroupNorm(num_channels=block_out_channels[-1], num_groups=norm_num_groups, eps=1e-6)
        self.conv_act = nn.SiLU()
        conv_out_channels = 2 * out_channels if double_z else out_channels
        self.conv_out = nn.Conv2d(block_out_channels[-1], conv_out_channels, 3, padding=1)

    def forward(self, x):
        """x: NCHW pixels (CUDA) -> NCHW fp32 moments (B, 2 * latent_channels, H / 2^(levels-1), ...)."""
        sample = _conv_in(self.conv_in, x)
        for down_block in self.down_blocks:
            sample = down_block(sample)
        sample = self.mid_block(sample)
        return _norm_act_out(self.conv_norm_out, self.conv_out, sample)


class Decoder(nn.Module):
    def __init__(self, in_channels=3, out_channels=3, up_block_types=("UpDecoderBlock2D",), block_out_channels=(64,),
                 layers_per_block=2, norm_num_groups=32, act_fn="silu"):
        super().__init__()
        self.layers_per_block = layers_per_block
        self.conv_in = nn.Conv2d(in_channels, block_out_channels[-1], kernel_size=3, stride=1, padding=1)
        self.mid_block = None
        self.up_blocks = nn.ModuleList([])
        self.mid_block = UNetMidBlock2D(in_channels=block_out_channels[-1], resnet_eps=1e-6, resnet_act_fn=act_fn,
                                        output_scale_factor=1, resnet_time_scale_shift="default",
                                        attn_num_head_channels=None, resnet_groups=norm_num_groups, temb_channels=None)
        reversed_block_out_channels = list(reversed(block_out_channels))
        output_channel = reversed_block_out_channels[0]
        for i, up_block_type in enumerate(up_block_types):
            prev_output_channel = output_channel
            output_channel = reversed_block_out_channels[i]
            is_final_block = i == len(block_out_channels) - 1
            self.up_blocks.append(get_up_block(
                up_block_type, num_layers=self.layers_per_block + 1, in_channels=prev_output_channel,
                out_channels=output_channel, prev_output_channel=None, add_upsample=not is_final_block,
                resnet_eps=1e-6, resnet_act_fn=act_fn, resnet_groups=norm_num_groups, attn_num_head_channels=None,
                temb_channels=None))
        self.conv_norm_out = nn.GroupNorm(num_channels=block_out_channels[0], num_groups=norm_num_groups, eps=1e-6)
        self.conv_act = nn.SiLU()
        self.conv_out = nn.Conv2d(block_out_channels[0], out_channels, 3, padding=1)

    def forward(self, z):
        """z: NCHW latents (CUDA) -> NCHW fp32 pixels."""
        sample = _conv_in(self.conv_in, z)
        sample = self.mid_block(sample)
        for up_block in self.up_blocks:
            sample = up_block(sample)
        # the engine when its operand fits (Cin % 64 == 0, Cout <= 64; the up blocks' convolutions already ran at this
        # resolution, so it tiles); the direct kernel otherwise
        engine = self.conv_out.in_channels % 64 == 0 and self.conv_out.out_channels <= 64
        return _norm_act_out(self.conv_norm_out, self.conv_out, sample, engine=engine)


class DiagonalGaussianDistribution:
    """diffusers vae.py DiagonalGaussianDistribution: moments = (mean, logvar) along dim 1, logvar clamped to [-30, 20]."""

    def __init__(self, parameters, deterministic=False):
        self.parameters = parameters
        self.mean, self.logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(self.logvar, -30.0, 20.0)
        self.deterministic = deterministic
        self.std = torch.exp(0.5 * self.logvar)
        self.var = torch.exp(self.logvar)
        if self.deterministic:
            self.var = self.std = torch.zeros_like(self.mean, device=self.parameters.device, dtype=self.parameters.dtype)

    def sample(self, generator: Optional[torch.Generator] = None, noise: Optional[torch.Tensor] = None):
        """mean + std * eps; eps ~ N(0, 1) from `generator` (or the given `noise`, same shape as the mean)."""
        if noise is None:
            noise = torch.randn(self.mean.shape, generator=generator, device=self.parameters.device,
                                dtype=self.parameters.dtype)
        return self.mean + self.std * noise.to(device=self.parameters.device, dtype=self.parameters.dtype)

    def kl(self, other=None):
        if self.deterministic:
            return torch.Tensor([0.0])
        if other is None:
            return 0.5 * torch.sum(torch.pow(self.mean, 2) + self.var - 1.0 - self.logvar, dim=[1, 2, 3])
        return 0.5 * torch.sum(torch.pow(self.mean - other.mean, 2) / other.var + self.var / other.var - 1.0
                               - self.logvar + other.logvar, dim=[1, 2, 3])

    def mode(self):
        return self.mean
