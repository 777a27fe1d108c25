"""AutoencoderKL — drop-in for diffusers 0.14 models/autoencoder_kl.py (the Stable Diffusion VAE) on the sm_90a kernels.
Forward only: the VAE is frozen in pre-training (`vae.encode(pixel_values).latent_dist.sample() * scaling_factor`) and
in inference (`decode_latents`).  Same constructor, `config`, state-dict keys and shapes as diffusers.

Inputs are NCHW pixels / latents (fp32, bf16 or fp16) on a CUDA device; outputs are NCHW in the parameter dtype.  The
latent-sized 1x1 convolutions (quant_conv, post_quant_conv: B x 8 x 64 x 64 values) and the Gaussian sampling stay
torch glue.  post_quant_conv's bias is NOT folded into decoder.conv_in: the 3x3 conv's zero padding does not carry a
constant input offset at the border, so that fold would not be exact."""
from dataclasses import dataclass
import os
import json

import torch
import torch.nn.functional as F
from torch import nn

from e4t._mixins import BaseOutput, ConfigMixin, ModelMixin, register_to_config
from e4t.models.vae import Decoder, DecoderOutput, DiagonalGaussianDistribution, Encoder
from e4t_b200._lib import E4TError

# largest activation, in elements, one kernel call may see: the batch is split so that every channels-last activation
# of a chunk stays below 2^31 elements (a 16 x 512 x 512 x 256 bf16 decoder activation is 2^30 elements, 2 GiB)
MAX_ACTIVATION_ELEMS = (1 << 31) - 1


@dataclass
class AutoencoderKLOutput(BaseOutput):
    latent_dist: "DiagonalGaussianDistribution" = None


class AutoencoderKL(ModelMixin, ConfigMixin):
    @register_to_config
    def __init__(self, in_channels=3, out_channels=3, down_block_types=("DownEncoderBlock2D",),
                 up_block_types=("UpDecoderBlock2D",), block_out_channels=(64,), layers_per_block=1, act_fn="silu",
                 latent_channels=4, norm_num_groups=32, sample_size=32, scaling_factor=0.18215):
        super().__init__()
        self.encoder = Encoder(in_channels=in_channels, out_channels=latent_channels,
                               down_block_types=down_block_types, block_out_channels=block_out_channels,
                               layers_per_block=layers_per_block, act_fn=act_fn, norm_num_groups=norm_num_groups,
                               double_z=True)
        self.decoder = Decoder(in_channels=latent_channels, out_channels=out_channels, up_block_types=up_block_types,
                               block_out_channels=block_out_channels, layers_per_block=layers_per_block,
                               norm_num_groups=norm_num_groups, act_fn=act_fn)
        self.quant_conv = nn.Conv2d(2 * latent_channels, 2 * latent_channels, 1)
        self.post_quant_conv = nn.Conv2d(latent_channels, latent_channels, 1)

    # ------------------------------------------------------------------------------------------------------------
    def _check(self, x, what):
        if not x.is_cuda:
            raise E4TError(f"e4t AutoencoderKL.{what} runs on the sm_90a kernels only (no CPU fallback)")
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError(f"AutoencoderKL.{what} is inference only: call it under torch.no_grad() or "
                                      "freeze the VAE (requires_grad_(False))")

    def _chunk(self, hw_pixels):
        """Images per kernel call so that no activation exceeds MAX_ACTIVATION_ELEMS: level i has 1 / 4^i of the full
        resolution's pixels, and its activations (encoder and decoder) have at most the channels of levels i - 1 .. i + 1."""
        ch = list(self.config.block_out_channels)
        per_image = max(max(ch[max(i - 1, 0):i + 2]) * (hw_pixels >> (2 * i)) for i in range(len(ch)))
        return max(1, MAX_ACTIVATION_ELEMS // per_image)

    @staticmethod
    def _conv1x1(conv, x):
        return F.conv2d(x, conv.weight.float(), conv.bias.float())

    def _encode_moments(self, x):
        n = self._chunk(x.shape[2] * x.shape[3])
        h = torch.cat([self.encoder(x[i:i + n]) for i in range(0, x.shape[0], n)]) if x.shape[0] > n \
            else self.encoder(x)
        return self._conv1x1(self.quant_conv, h).to(self.dtype)

    def encode(self, x, return_dict: bool = True):
        self._check(x, "encode")
        posterior = DiagonalGaussianDistribution(self._encode_moments(x))
        if not return_dict:
            return (posterior,)
        return AutoencoderKLOutput(latent_dist=posterior)

    def _decode(self, z, return_dict: bool = True):
        z = self._conv1x1(self.post_quant_conv, z.float())
        f = 2 ** (len(self.config.block_out_channels) - 1)
        n = self._chunk(z.shape[2] * z.shape[3] * f * f)
        dec = torch.cat([self.decoder(z[i:i + n]) for i in range(0, z.shape[0], n)]) if z.shape[0] > n \
            else self.decoder(z)
        dec = dec.to(self.dtype)
        if not return_dict:
            return (dec,)
        return DecoderOutput(sample=dec)

    def decode(self, z, return_dict: bool = True):
        self._check(z, "decode")
        return self._decode(z, return_dict)

    def forward(self, sample, sample_posterior: bool = False, return_dict: bool = True, generator=None):
        posterior = self.encode(sample).latent_dist
        z = posterior.sample(generator=generator) if sample_posterior else posterior.mode()
        dec = self.decode(z).sample
        if not return_dict:
            return (dec,)
        return DecoderOutput(sample=dec)

    # ------------------------------------------------------------------------------------------------------------
    @classmethod
    def from_pretrained(cls, path, subfolder=None, torch_dtype=None, **kwargs):
        """Local diffusers-format directory only (<path>[/<subfolder>]/{config.json, diffusion_pytorch_model.*}):
        .bin, .safetensors or their sharded *.index.json forms.  Missing or unexpected keys are fatal."""
        from e4t.utils import _load_diffusers_weights
        d = os.path.join(path, subfolder) if subfolder else path
        if not os.path.isdir(d):
            raise FileNotFoundError(f"{d} (hub download is unavailable offline)")
        with open(os.path.join(d, cls.config_name)) as f:
            cfg = {k: v for k, v in json.load(f).items() if not k.startswith("_")}
        for k in ("down_block_types", "up_block_types", "block_out_channels"):
            if k in cfg:
                cfg[k] = tuple(cfg[k])
        model = cls(**cfg)
        sd = _load_diffusers_weights(d)
        if not sd:
            raise FileNotFoundError(f"no VAE weights under {d} (looked for diffusion_pytorch_model.{{bin,safetensors}} "
                                    f"and their sharded *.index.json forms)")
        m, u = model.load_state_dict(sd, strict=False)
        if m:
            raise RuntimeError(f"missing keys:\n{m}")
        if u:
            raise RuntimeError(f"unexpected keys:\n{u}")
        if torch_dtype is not None:
            model = model.to(torch_dtype)
        return model.eval()
