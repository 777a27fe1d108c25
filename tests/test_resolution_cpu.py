"""Non-square sizes without a GPU: the CPU oracle against tests/golden/rect.pt (oracle/gen_golden_rect.py: the
reference's own tiny UNet at 24 x 40 latents and tiny VAE at 96 x 160 pixels), and the size rule of the pipeline,
the UNet and the training steps."""
import os
import types

import pytest
import torch

from oracle import e4t_oracle as O
from oracle import vae_oracle as V
from oracle.golden_format import base_name, golden_view, unpack_grads

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rect.pt")


def _rel(a, b):
    a = a.double(); b = b.double()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt().clamp_min(1e-30)).item()


def rect_unet_inputs(gold):
    """The generator's draws of oracle/gen_golden_rect.py:unet_case, in its order."""
    cfg, x = gold["cfg"], gold["x"]
    g = torch.Generator().manual_seed(gold["seed"] + 1)
    xs = torch.randn(x.shape, generator=g)
    t = torch.randint(0, 1000, (x.shape[0],), generator=g)
    ehs = torch.randn(x.shape[0], 77, cfg["cross_attention_dim"], generator=g)
    w = torch.randn(x.shape, generator=g)
    wenc = [torch.randn(tuple(s), generator=g) for s in gold["enc_shapes"]]
    return xs, t, ehs, w, wenc


def test_oracle_unet_matches_reference_at_24x40():
    gold = torch.load(GOLD)["unet"]
    cfg = gold["cfg"]
    x, t, ehs, w, wenc = rect_unet_inputs(gold)
    assert x.shape[-2:] == (24, 40)
    for a, b in ((x, "x"), (t, "t"), (ehs, "ehs"), (w, "w")):
        assert torch.equal(a, gold[b]), b
    sd = O.synth_state_dict(O.unet_param_shapes(cfg), gold["seed"])
    for p in sd.values():
        p.requires_grad_(True)
    ehs.requires_grad_(True)
    out = O.unet_forward(sd, cfg, x, t, ehs)
    enc = O.unet_forward(sd, cfg, x, t, ehs, return_encoder_outputs=True)["down_block_samples"]
    assert [tuple(e.shape) for e in enc] == gold["enc_shapes"]
    assert _rel(out, gold["out"]) < 1e-4
    assert _rel(torch.cat([e.mean(dim=(2, 3)) for e in enc], -1), gold["enc_pooled"]) < 1e-4
    ((out * w).sum() + sum((e * we).sum() for e, we in zip(enc, wenc))).backward()
    assert _rel(ehs.grad, gold["d_ehs"]) < 1e-4
    refs = unpack_grads(gold["grads"])
    assert {base_name(k) for k in refs} == set(sd)
    for k, ref in refs.items():
        assert _rel(golden_view(sd[base_name(k)].grad, k, ref), ref) < 1e-4, k


def test_oracle_vae_matches_reference_at_96x160():
    gold = torch.load(GOLD)["vae"]
    cfg = gold["cfg"]
    g = torch.Generator().manual_seed(gold["seed"] + 1)
    x = torch.rand(1, 3, 96, 160, generator=g) * 2 - 1
    sd = O.synth_state_dict(V.vae_param_shapes(cfg), gold["seed"])
    with torch.no_grad():
        moments = V.vae_encode(sd, cfg, x)
        decoded = V.vae_decode(sd, cfg, gold["z"])
    assert moments.shape == (1, 8, 24, 40) and decoded.shape == (1, 3, 96, 160)
    assert _rel(moments, gold["moments"]) < 1e-4
    assert _rel(decoded, gold["decoded"]) < 1e-4


def test_unet_latent_multiple():
    from e4t.models.unet_2d_condition import UNet2DConditionModel
    assert UNet2DConditionModel(**O.ref_unet_kwargs(O.TINY_UNET)).latent_multiple == 2
    sd14 = types.SimpleNamespace(config=types.SimpleNamespace(block_out_channels=O.SD14_UNET["block_out_channels"]))
    assert UNet2DConditionModel.latent_multiple.fget(sd14) == 8


def _fake_pipe(levels, vae_scale_factor):
    unet = types.SimpleNamespace(latent_multiple=2 ** (levels - 1), config=types.SimpleNamespace(sample_size=64))
    return types.SimpleNamespace(unet=unet, vae_scale_factor=vae_scale_factor, domain_embed_scale=0.1)


@pytest.mark.parametrize("h,w", [(520, 512), (512, 776), (544, 512), (96, 100)])
def test_pipeline_rejects_sizes_off_the_rule(h, w):
    """SD-v1.4 (4 levels, VAE factor 8): multiples of 64 px; raised before the pipeline touches a model."""
    from e4t.pipeline_stable_diffusion_e4t import StableDiffusionE4TPipeline
    with pytest.raises(ValueError, match="multiples of 64 px"):
        StableDiffusionE4TPipeline.__call__(_fake_pipe(4, 8), prompt="a photo of *s", height=h, width=w)


def test_pipeline_size_rule_follows_the_models():
    """A tiny UNet (2 levels) with the tiny VAE (factor 4) needs multiples of 8 px only."""
    from e4t.pipeline_stable_diffusion_e4t import StableDiffusionE4TPipeline
    with pytest.raises(ValueError, match="multiples of 8 px"):
        StableDiffusionE4TPipeline.__call__(_fake_pipe(2, 4), prompt="x", height=96, width=164)
    # a size on the rule passes the check and fails later, on the stand-in's missing parts
    with pytest.raises(AttributeError):
        StableDiffusionE4TPipeline.__call__(_fake_pipe(2, 4), prompt="x", height=96, width=160)


def test_step_rejects_latents_off_the_rule():
    from e4t_b200._lib import E4TError
    from e4t_b200.engine import PretrainStep
    step = types.SimpleNamespace(unet=types.SimpleNamespace(latent_multiple=8))
    batch = dict(pixel_values=None, latents=torch.zeros(1, 4, 64, 60), noise=None)
    with pytest.raises(E4TError, match="multiples of the UNet's down-sampling factor 8"):
        PretrainStep.forward_loss(step, batch)
