"""The CPU oracle at latent sizes that are not multiples of the UNet's down-sampling factor 2^(levels - 1).

The reference's UNet2DConditionModel forwards each up block's skip size to its upsampler when a latent side is not a
multiple of its overall up factor (e4t/models/unet_2d_condition.py:426-436, 535-536; diffusers' Upsample2D then runs
F.interpolate(size=..., mode="nearest")).  `unet_forward` restates that on e4t_oracle's blocks; at every other size it
is e4t_oracle.unet_forward itself.  `pretrain_step` and `pipeline_sample` are e4t_oracle's with this forward in place of
e4t_oracle.unet_forward.  The down path needs no change: F.conv2d(stride=2, padding=1) already gives ceil(side / 2).
Pinned by tests/golden/ragged.pt (oracle/gen_golden_ragged.py)."""
import contextlib

import torch
import torch.nn.functional as F

from oracle import e4t_oracle as O

_base_unet_forward = O.unet_forward


def unet_forward(sd, cfg, sample, timesteps, ehs, return_encoder_outputs=False):
    """UNet2DConditionModel.forward (unet_2d_condition.py:410-562) with the upsample sizes forwarded."""
    boc, L = cfg["block_out_channels"], cfg["layers_per_block"]
    n = len(boc)
    if return_encoder_outputs or not any(s % 2 ** (n - 1) for s in sample.shape[-2:]):
        return _base_unet_forward(sd, cfg, sample, timesteps, ehs, return_encoder_outputs)
    heads, groups, eps = cfg["attention_head_dim"], cfg["norm_num_groups"], cfg["norm_eps"]
    if not torch.is_tensor(timesteps):
        timesteps = torch.tensor([timesteps], dtype=torch.int64)
    elif timesteps.dim() == 0:
        timesteps = timesteps[None]
    timesteps = timesteps.expand(sample.shape[0])
    t_emb = O.timestep_embedding(timesteps, boc[0], cfg["flip_sin_to_cos"], cfg["freq_shift"]).to(sample.dtype)
    emb = F.linear(F.silu(F.linear(t_emb, sd["time_embedding.linear_1.weight"], sd["time_embedding.linear_1.bias"])),
                   sd["time_embedding.linear_2.weight"], sd["time_embedding.linear_2.bias"])
    x = F.conv2d(sample, sd["conv_in.weight"], sd["conv_in.bias"], padding=1)
    res = [x]
    for i in range(n):
        for j in range(L):
            x = O.resnet_block(sd, f"down_blocks.{i}.resnets.{j}.", x, emb, groups, eps)
            if i < n - 1:
                x = O.transformer_2d(sd, f"down_blocks.{i}.attentions.{j}.", x, ehs, heads, groups)
            res.append(x)
        if i < n - 1:
            x = F.conv2d(x, sd[f"down_blocks.{i}.downsamplers.0.conv.weight"],
                         sd[f"down_blocks.{i}.downsamplers.0.conv.bias"], stride=2, padding=1)
            res.append(x)
    x = O.resnet_block(sd, "mid_block.resnets.0.", x, emb, groups, eps)
    x = O.transformer_2d(sd, "mid_block.attentions.0.", x, ehs, heads, groups)
    x = O.resnet_block(sd, "mid_block.resnets.1.", x, emb, groups, eps)
    for i in range(n):
        for j in range(L + 1):
            x = torch.cat([x, res.pop()], dim=1)
            x = O.resnet_block(sd, f"up_blocks.{i}.resnets.{j}.", x, emb, groups, eps)
            if i > 0:
                x = O.transformer_2d(sd, f"up_blocks.{i}.attentions.{j}.", x, ehs, heads, groups)
        if i < n - 1:
            x = F.interpolate(x, size=res[-1].shape[2:], mode="nearest")                               # :535-536
            x = F.conv2d(x, sd[f"up_blocks.{i}.upsamplers.0.conv.weight"],
                         sd[f"up_blocks.{i}.upsamplers.0.conv.bias"], padding=1)
    x = F.silu(F.group_norm(x, groups, sd["conv_norm_out.weight"], sd["conv_norm_out.bias"], eps))
    return F.conv2d(x, sd["conv_out.weight"], sd["conv_out.bias"], padding=1)


@contextlib.contextmanager
def _forwarding_sizes():
    orig = O.unet_forward
    O.unet_forward = unet_forward
    try:
        yield
    finally:
        O.unet_forward = orig


def pretrain_step(*args, **kwargs):
    """e4t_oracle.pretrain_step with the upsample sizes forwarded."""
    with _forwarding_sizes():
        return O.pretrain_step(*args, **kwargs)


def pipeline_sample(*args, **kwargs):
    """e4t_oracle.pipeline_sample with the upsample sizes forwarded."""
    with _forwarding_sizes():
        return O.pipeline_sample(*args, **kwargs)
