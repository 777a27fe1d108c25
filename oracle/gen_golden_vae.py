"""Generate tests/golden/vae.pt by running the REFERENCE's own VAE blocks (DownEncoderBlock2D, UpDecoderBlock2D,
UNetMidBlock2D from e4t/models/unet_2d_blocks.py and AttentionBlock from e4t/models/attention.py, imported unchanged from
a checkout of mkshing/e4t-diffusion named by $E4T_REFERENCE_DIR) composed by oracle/shim/diffusers/models/vae.py:

    E4T_REFERENCE_DIR=/path/to/e4t-diffusion python oracle/gen_golden_vae.py   # writes tests/golden/vae.pt

The fixture holds a tiny fp32 encode / decode case (TINY_VAE, 64 x 64 pixels -> 16 x 16 latents, weights from
e4t_oracle.synth_state_dict) and the SD-config inventory (number of keys, number of parameters, sha256 of the sorted
`key:shape` lines).  It pins oracle/vae_oracle.py (tests/test_vae_cpu.py)."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REFERENCE = os.environ.get("E4T_REFERENCE_DIR", os.path.join(ROOT, "..", "e4t-diffusion"))
sys.path[:0] = [REFERENCE, os.path.join(HERE, "shim"), ROOT]

from oracle import e4t_oracle as O  # noqa: E402
from oracle import vae_oracle as V  # noqa: E402

import e4t.models.unet_2d_blocks as ref_blocks  # noqa: E402  (the reference's)
from e4t.models.attention import AttentionBlock  # noqa: E402  (the reference's)
from diffusers.models.vae import AutoencoderKL  # noqa: E402  (oracle/shim composition of the reference's blocks)

# the shim's diffusers.models.attention stubs AttentionBlock; the VAE mid-block must use the reference's
ref_blocks.AttentionBlock = AttentionBlock

OUT = os.path.join(ROOT, "tests", "golden", "vae.pt")
SEED = 11


def build(cfg):
    m = AutoencoderKL(**cfg).eval()
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    mine = V.vae_param_shapes(cfg)
    assert shapes == mine, (set(shapes) ^ set(mine), [k for k in shapes if k in mine and shapes[k] != mine[k]][:5])
    return m, shapes


def main():
    torch.manual_seed(0)
    m, shapes = build(V.TINY_VAE)
    m.load_state_dict(O.synth_state_dict(shapes, SEED), strict=True)
    g = torch.Generator().manual_seed(SEED + 1)
    x = torch.rand(1, 3, 64, 64, generator=g) * 2 - 1
    z = torch.randn(1, 4, 16, 16, generator=g)
    noise = torch.randn(1, 4, 16, 16, generator=g)
    with torch.no_grad():
        post = m.encode(x)
        rec = dict(cfg=V.TINY_VAE, seed=SEED, x=x, z=z, noise=noise, moments=post.parameters.clone(),
                   sample=post.sample(noise).clone(), decoded=m.decode(z).clone())
    _, sd_shapes = build(V.SD_VAE)
    rec["sd_inventory"] = V.vae_inventory(sd_shapes)
    print(rec["sd_inventory"])
    torch.save(rec, OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main()
