"""Generate tests/golden/rect.pt by running the REFERENCE's own modules (imported unchanged from a checkout of
mkshing/e4t-diffusion named by $E4T_REFERENCE_DIR, via oracle/shim) at a non-square size:

    E4T_REFERENCE_DIR=/path/to/e4t-diffusion python oracle/gen_golden_rect.py   # writes tests/golden/rect.pt

Every other fixture is square, so a transposed H / W in the oracle's token reshapes would pass against them.  Two cases:
  * the tiny UNet (e4t_oracle.TINY_UNET, B = 2) at 24 x 40 latents: output, pooled encoder outputs and the gradients of
    (out * w).sum() + sum (enc_i * wenc_i).sum() w.r.t. the encoder hidden states and every parameter (compacted by
    golden_format.compact_grads);
  * the tiny VAE (vae_oracle.TINY_VAE) encode at 96 x 160 pixels and decode of 24 x 40 latents.
Weights come from e4t_oracle.synth_state_dict.  The small inputs are stored; the encoder-output weights `wenc` (drawn
from the same generator after x, t, ehs, w, in encoder-output order) and the VAE's pixels are re-drawn from the seed.  It pins oracle/e4t_oracle.py and
oracle/vae_oracle.py (tests/test_resolution_cpu.py)."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REFERENCE = os.environ.get("E4T_REFERENCE_DIR", os.path.join(ROOT, "..", "e4t-diffusion"))
sys.path[:0] = [REFERENCE, os.path.join(HERE, "shim"), ROOT]

from oracle import e4t_oracle as O  # noqa: E402
from oracle import vae_oracle as V  # noqa: E402
from oracle.golden_format import compact_grads  # noqa: E402

import e4t.models.unet_2d_blocks as ref_blocks  # noqa: E402  (the reference's)
from e4t.models.attention import AttentionBlock  # noqa: E402  (the reference's)
from e4t.models.unet_2d_condition import UNet2DConditionModel  # noqa: E402  (the reference's)
from diffusers.models.vae import AutoencoderKL  # noqa: E402  (oracle/shim composition of the reference's blocks)

ref_blocks.AttentionBlock = AttentionBlock   # as in gen_golden_vae.py: the VAE mid-block uses the reference's

OUT = os.path.join(ROOT, "tests", "golden", "rect.pt")
UNET_HW = (24, 40)
VAE_HW = (96, 160)
SEED = 23


def unet_case():
    cfg, B, (H, W) = O.TINY_UNET, 2, UNET_HW
    m = UNet2DConditionModel(**O.ref_unet_kwargs(cfg))
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert shapes == O.unet_param_shapes(cfg)
    m.load_state_dict(O.synth_state_dict(shapes, SEED), strict=True)
    g = torch.Generator().manual_seed(SEED + 1)
    x = torch.randn(B, 4, H, W, generator=g)
    t = torch.randint(0, 1000, (B,), generator=g)
    ehs = torch.randn(B, 77, cfg["cross_attention_dim"], generator=g).requires_grad_(True)
    w = torch.randn(B, 4, H, W, generator=g)
    out = m(x, t, ehs).sample
    enc = m(x, t, ehs, return_encoder_outputs=True)["down_block_samples"]
    wenc = [torch.randn(e.shape, generator=g) for e in enc]
    ((out * w).sum() + sum((e * we).sum() for e, we in zip(enc, wenc))).backward()
    grads = {}
    for k, p in m.named_parameters():
        if p.grad.dim() >= 2 and p.grad.shape[0] > 8 and p.grad[0].numel() > 8:
            grads[k + "#corner"] = p.grad.reshape(p.grad.shape[0], -1)[:8, :8].clone()
            grads[k + "#norm"] = p.grad.norm()
        else:
            grads[k] = p.grad.clone()
    return dict(cfg=cfg, seed=SEED, x=x, t=t, ehs=ehs.detach().clone(), w=w, out=out.detach().clone(),
                enc_pooled=torch.cat([e.mean(dim=(2, 3)) for e in enc], dim=-1).detach().clone(),
                enc_shapes=[tuple(e.shape) for e in enc], d_ehs=ehs.grad.clone(), grads=compact_grads(grads))


def vae_case():
    cfg, (H, W) = V.TINY_VAE, VAE_HW
    f = 2 ** (len(cfg["block_out_channels"]) - 1)
    m = AutoencoderKL(**cfg).eval()
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert shapes == V.vae_param_shapes(cfg)
    m.load_state_dict(O.synth_state_dict(shapes, SEED + 2), strict=True)
    g = torch.Generator().manual_seed(SEED + 3)
    x = torch.rand(1, 3, H, W, generator=g) * 2 - 1
    z = torch.randn(1, 4, H // f, W // f, generator=g)
    with torch.no_grad():
        moments = m.encode(x).parameters.clone()
        decoded = m.decode(z).clone()
    return dict(cfg=cfg, seed=SEED + 2, z=z, moments=moments, decoded=decoded)


def main():
    torch.manual_seed(0)
    rec = dict(unet=unet_case(), vae=vae_case())
    torch.save(rec, OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main()
