"""fp32 oracle of the Stable Diffusion VAE (diffusers 0.14 AutoencoderKL): parameter inventory and a functional
restatement of encode / decode with torch ops only.

It is pinned to the reference's own blocks (DownEncoderBlock2D, UpDecoderBlock2D, UNetMidBlock2D, AttentionBlock) by
tests/golden/vae.pt, which oracle/gen_golden_vae.py writes from them (tests/test_vae_cpu.py), and it is the parity
target of the CUDA path (tests/test_vae_gpu.py, tools/vae_ab.py).  Weights come from e4t_oracle.synth_state_dict, so
every consumer can rebuild the fixture's parameters from the seed alone."""
import hashlib
import math

import torch
import torch.nn.functional as F

TINY_VAE = dict(in_channels=3, out_channels=3, down_block_types=("DownEncoderBlock2D",) * 3,
                up_block_types=("UpDecoderBlock2D",) * 3, block_out_channels=(64, 128, 128), layers_per_block=1,
                act_fn="silu", latent_channels=4, norm_num_groups=32, sample_size=64, scaling_factor=0.18215)
SD_VAE = dict(in_channels=3, out_channels=3, down_block_types=("DownEncoderBlock2D",) * 4,
              up_block_types=("UpDecoderBlock2D",) * 4, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
              act_fn="silu", latent_channels=4, norm_num_groups=32, sample_size=512, scaling_factor=0.18215)


# ---- parameter inventory -------------------------------------------------------------------------------------------
def _conv_shapes(p, cout, cin, k):
    return {p + "weight": (cout, cin, k, k), p + "bias": (cout,)}


def _norm_shapes(p, c):
    return {p + "weight": (c,), p + "bias": (c,)}


def _res_shapes(p, cin, cout):
    s = {**_norm_shapes(p + "norm1.", cin), **_conv_shapes(p + "conv1.", cout, cin, 3),
         **_norm_shapes(p + "norm2.", cout), **_conv_shapes(p + "conv2.", cout, cout, 3)}
    if cin != cout:
        s.update(_conv_shapes(p + "conv_shortcut.", cout, cin, 1))
    return s


def _mid_shapes(p, c):
    s = {**_res_shapes(p + "resnets.0.", c, c), **_res_shapes(p + "resnets.1.", c, c),
         **_norm_shapes(p + "attentions.0.group_norm.", c)}
    for n in ("query", "key", "value", "proj_attn"):
        s[f"{p}attentions.0.{n}.weight"] = (c, c)
        s[f"{p}attentions.0.{n}.bias"] = (c,)
    return s


def vae_param_shapes(cfg):
    ch, lpb, lat = list(cfg["block_out_channels"]), cfg["layers_per_block"], cfg["latent_channels"]
    n = len(ch)
    s = {**_conv_shapes("encoder.conv_in.", ch[0], cfg["in_channels"], 3)}
    prev = ch[0]
    for i, c in enumerate(ch):
        for j in range(lpb):
            s.update(_res_shapes(f"encoder.down_blocks.{i}.resnets.{j}.", prev if j == 0 else c, c))
        if i < n - 1:
            s.update(_conv_shapes(f"encoder.down_blocks.{i}.downsamplers.0.conv.", c, c, 3))
        prev = c
    s.update(_mid_shapes("encoder.mid_block.", ch[-1]))
    s.update(_norm_shapes("encoder.conv_norm_out.", ch[-1]))
    s.update(_conv_shapes("encoder.conv_out.", 2 * lat, ch[-1], 3))
    s.update(_conv_shapes("quant_conv.", 2 * lat, 2 * lat, 1))
    s.update(_conv_shapes("post_quant_conv.", lat, lat, 1))
    s.update(_conv_shapes("decoder.conv_in.", ch[-1], lat, 3))
    s.update(_mid_shapes("decoder.mid_block.", ch[-1]))
    rev = ch[::-1]
    prev = rev[0]
    for i, c in enumerate(rev):
        for j in range(lpb + 1):
            s.update(_res_shapes(f"decoder.up_blocks.{i}.resnets.{j}.", prev if j == 0 else c, c))
        if i < n - 1:
            s.update(_conv_shapes(f"decoder.up_blocks.{i}.upsamplers.0.conv.", c, c, 3))
        prev = c
    s.update(_norm_shapes("decoder.conv_norm_out.", ch[0]))
    s.update(_conv_shapes("decoder.conv_out.", cfg["out_channels"], ch[0], 3))
    return s


def vae_inventory(shapes):
    """(number of keys, number of parameters, sha256 of the sorted `key:shape` lines) of a {key: shape} dict."""
    keys = sorted(shapes)
    sha = hashlib.sha256("\n".join(f"{k}:{tuple(shapes[k])}" for k in keys).encode()).hexdigest()
    return dict(n_keys=len(keys), n_params=sum(math.prod(shapes[k]) for k in keys), sha256=sha)


# ---- forward -------------------------------------------------------------------------------------------------------
def _gn(sd, p, x, silu, groups):
    y = F.group_norm(x, groups, sd[p + "weight"], sd[p + "bias"], 1e-6)
    return F.silu(y) if silu else y


def _conv(sd, p, x, **kw):
    return F.conv2d(x, sd[p + "weight"], sd[p + "bias"], **kw)


def _resnet(sd, p, x, g):
    h = _conv(sd, p + "conv1.", _gn(sd, p + "norm1.", x, True, g), padding=1)
    h = _conv(sd, p + "conv2.", _gn(sd, p + "norm2.", h, True, g), padding=1)
    if p + "conv_shortcut.weight" in sd:
        x = _conv(sd, p + "conv_shortcut.", x)
    return x + h


def _attn(sd, p, x, g):
    """AttentionBlock (one head): scores in the working dtype, softmax in fp32, (h + residual) / 1."""
    B, C, H, W = x.shape
    h = _gn(sd, p + "group_norm.", x, False, g).reshape(B, C, H * W).transpose(1, 2)
    q, k, v = (F.linear(h, sd[p + n + ".weight"], sd[p + n + ".bias"]) for n in ("query", "key", "value"))
    s = torch.baddbmm(torch.empty(B, H * W, H * W, dtype=q.dtype, device=q.device), q, k.transpose(-1, -2), beta=0,
                      alpha=1 / math.sqrt(C))
    o = torch.bmm(torch.softmax(s.float(), dim=-1).type(s.dtype), v)
    o = F.linear(o, sd[p + "proj_attn.weight"], sd[p + "proj_attn.bias"])
    return o.transpose(-1, -2).reshape(B, C, H, W) + x


def _mid(sd, p, x, g):
    x = _resnet(sd, p + "resnets.0.", x, g)
    x = _attn(sd, p + "attentions.0.", x, g)
    return _resnet(sd, p + "resnets.1.", x, g)


def vae_encode(sd, cfg, x):
    """NCHW pixels -> NCHW moments (mean | logvar) = quant_conv(encoder(x))."""
    n, lpb, g = len(cfg["block_out_channels"]), cfg["layers_per_block"], cfg["norm_num_groups"]
    h = _conv(sd, "encoder.conv_in.", x, padding=1)
    for i in range(n):
        for j in range(lpb):
            h = _resnet(sd, f"encoder.down_blocks.{i}.resnets.{j}.", h, g)
        if i < n - 1:   # Downsample2D(padding=0): zero row / column on the bottom and right, unpadded stride-2 conv
            h = _conv(sd, f"encoder.down_blocks.{i}.downsamplers.0.conv.", F.pad(h, (0, 1, 0, 1)), stride=2)
    h = _mid(sd, "encoder.mid_block.", h, g)
    h = _conv(sd, "encoder.conv_out.", _gn(sd, "encoder.conv_norm_out.", h, True, g), padding=1)
    return _conv(sd, "quant_conv.", h)


def vae_decode(sd, cfg, z):
    """NCHW latents -> NCHW pixels = decoder(post_quant_conv(z))."""
    n, lpb, g = len(cfg["block_out_channels"]), cfg["layers_per_block"], cfg["norm_num_groups"]
    h = _conv(sd, "decoder.conv_in.", _conv(sd, "post_quant_conv.", z), padding=1)
    h = _mid(sd, "decoder.mid_block.", h, g)
    for i in range(n):
        for j in range(lpb + 1):
            h = _resnet(sd, f"decoder.up_blocks.{i}.resnets.{j}.", h, g)
        if i < n - 1:
            h = _conv(sd, f"decoder.up_blocks.{i}.upsamplers.0.conv.",
                      F.interpolate(h, scale_factor=2.0, mode="nearest"), padding=1)
    return _conv(sd, "decoder.conv_out.", _gn(sd, "decoder.conv_norm_out.", h, True, g), padding=1)


def vae_sample(moments, noise):
    """DiagonalGaussianDistribution(moments).sample() with the given noise: mean + exp(0.5 clamp(logvar, -30, 20)) noise."""
    mean, logvar = torch.chunk(moments, 2, dim=1)
    return mean + torch.exp(0.5 * logvar.clamp(-30.0, 20.0)) * noise


def vae_latents(sd, cfg, pixel_values, noise):
    """pretrain_e4t.py:598-599: vae.encode(pixel_values).latent_dist.sample() * scaling_factor."""
    return vae_sample(vae_encode(sd, cfg, pixel_values), noise) * cfg["scaling_factor"]
