"""Generate tests/golden/ragged.pt by running the REFERENCE's own UNet2DConditionModel (imported unchanged from a
checkout of mkshing/e4t-diffusion named by $E4T_REFERENCE_DIR, via oracle/shim) at latent sizes that are not multiples
of its down-sampling factor:

    E4T_REFERENCE_DIR=/path/to/e4t-diffusion python oracle/gen_golden_ragged.py   # writes tests/golden/ragged.pt

The tiny UNet (e4t_oracle.TINY_UNET, B = 2) at 9 x 13 and 13 x 7 latents: its stride-2 convolutions see odd sides and
it forwards the skip sizes to its upsamplers (unet_2d_condition.py:426-436, 535-536).  Each case stores the output,
the pooled encoder outputs and the gradients of (out * w).sum() + sum (enc_i * wenc_i).sum() w.r.t. the encoder hidden
states and every parameter (compacted by golden_format.compact_grads), as gen_golden_rect.py does.  It pins
oracle/ragged_oracle.py (tests/test_ragged_cpu.py) and the e4t UNet with enable_any_latent_size() (tests/test_ragged_gpu.py)."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REFERENCE = os.environ.get("E4T_REFERENCE_DIR", os.path.join(ROOT, "..", "e4t-diffusion"))
sys.path[:0] = [REFERENCE, os.path.join(HERE, "shim"), ROOT]

from oracle import e4t_oracle as O  # noqa: E402
from oracle.golden_format import compact_grads  # noqa: E402

from e4t.models.unet_2d_condition import UNet2DConditionModel  # noqa: E402  (the reference's)

OUT = os.path.join(ROOT, "tests", "golden", "ragged.pt")
SIZES = ((9, 13), (13, 7))
SEED = 29


def unet_case(hw, seed):
    cfg, B, (H, W) = O.TINY_UNET, 2, hw
    m = UNet2DConditionModel(**O.ref_unet_kwargs(cfg))
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert shapes == O.unet_param_shapes(cfg)
    m.load_state_dict(O.synth_state_dict(shapes, seed), strict=True)
    g = torch.Generator().manual_seed(seed + 1)
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
    return dict(cfg=cfg, seed=seed, hw=hw, x=x, t=t, ehs=ehs.detach().clone(), w=w, out=out.detach().clone(),
                enc_pooled=torch.cat([e.mean(dim=(2, 3)) for e in enc], dim=-1).detach().clone(),
                enc_shapes=[tuple(e.shape) for e in enc], d_ehs=ehs.grad.clone(), grads=compact_grads(grads))


def main():
    torch.manual_seed(0)
    rec = {f"{h}x{w}": unet_case((h, w), SEED + 10 * i) for i, (h, w) in enumerate(SIZES)}
    torch.save(rec, OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main()
