"""Latent sizes that are not multiples of the UNet's down-sampling factor, without a GPU: the CPU oracle against
tests/golden/ragged.pt (oracle/gen_golden_ragged.py: the reference's own tiny UNet at 9 x 13 and 13 x 7 latents, with
odd stride-2 inputs and the skip sizes forwarded to the upsamplers), and the size rules of the UNet, the pipeline and
the training steps with UNet2DConditionModel.enable_any_latent_size()."""
import os
import types

import pytest
import torch

from oracle import e4t_oracle as O
from oracle import ragged_oracle as RO
from oracle.golden_format import base_name, golden_view, unpack_grads

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ragged.pt")


def _rel(a, b):
    a = a.double(); b = b.double()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt().clamp_min(1e-30)).item()


def ragged_unet_inputs(gold):
    """The generator's draws of oracle/gen_golden_ragged.py:unet_case, in its order."""
    cfg, x = gold["cfg"], gold["x"]
    g = torch.Generator().manual_seed(gold["seed"] + 1)
    xs = torch.randn(x.shape, generator=g)
    t = torch.randint(0, 1000, (x.shape[0],), generator=g)
    ehs = torch.randn(x.shape[0], 77, cfg["cross_attention_dim"], generator=g)
    w = torch.randn(x.shape, generator=g)
    wenc = [torch.randn(tuple(s), generator=g) for s in gold["enc_shapes"]]
    return xs, t, ehs, w, wenc


@pytest.mark.parametrize("case", ["9x13", "13x7"])
def test_oracle_unet_matches_reference_at_ragged_latents(case):
    gold = torch.load(GOLD)[case]
    cfg = gold["cfg"]
    x, t, ehs, w, wenc = ragged_unet_inputs(gold)
    assert x.shape[-2:] == tuple(gold["hw"])
    for a, b in ((x, "x"), (t, "t"), (ehs, "ehs"), (w, "w")):
        assert torch.equal(a, gold[b]), b
    sd = O.synth_state_dict(O.unet_param_shapes(cfg), gold["seed"])
    for p in sd.values():
        p.requires_grad_(True)
    ehs.requires_grad_(True)
    out = RO.unet_forward(sd, cfg, x, t, ehs)
    enc = RO.unet_forward(sd, cfg, x, t, ehs, return_encoder_outputs=True)["down_block_samples"]
    assert [tuple(e.shape) for e in enc] == gold["enc_shapes"]
    assert out.shape == x.shape
    assert _rel(out, gold["out"]) < 1e-4
    assert _rel(torch.cat([e.mean(dim=(2, 3)) for e in enc], -1), gold["enc_pooled"]) < 1e-4
    ((out * w).sum() + sum((e * we).sum() for e, we in zip(enc, wenc))).backward()
    assert _rel(ehs.grad, gold["d_ehs"]) < 1e-4
    refs = unpack_grads(gold["grads"])
    assert {base_name(k) for k in refs} == set(sd)
    for k, ref in refs.items():
        assert _rel(golden_view(sd[base_name(k)].grad, k, ref), ref) < 1e-4, k


def test_golden_file_is_small():
    assert os.path.getsize(GOLD) < 1 << 20


def test_any_latent_size_switch():
    from e4t.models.unet_2d_condition import UNet2DConditionModel
    m = UNet2DConditionModel(**O.ref_unet_kwargs(O.TINY_UNET))
    assert m.latent_multiple == 2 and m.min_latent_size == 2
    m.enable_any_latent_size()
    assert m.latent_multiple == 1 and m.min_latent_size == 2
    m.disable_any_latent_size()
    assert m.latent_multiple == 2
    # the properties still work on an object that only has `config`
    sd14 = types.SimpleNamespace(config=types.SimpleNamespace(block_out_channels=O.SD14_UNET["block_out_channels"]))
    assert UNet2DConditionModel.latent_multiple.fget(sd14) == 8
    assert UNet2DConditionModel.min_latent_size.fget(sd14) == 8
    UNet2DConditionModel.enable_any_latent_size(sd14)
    assert UNet2DConditionModel.latent_multiple.fget(sd14) == 1


def _fake_pipe(latent_multiple, min_latent_size, vae_scale_factor):
    unet = types.SimpleNamespace(latent_multiple=latent_multiple, min_latent_size=min_latent_size,
                                 config=types.SimpleNamespace(sample_size=64))
    return types.SimpleNamespace(unet=unet, vae_scale_factor=vae_scale_factor, domain_embed_scale=0.1)


@pytest.mark.parametrize("h,w", [(520, 512), (504, 776), (64, 64), (600, 800)])
def test_pipeline_with_the_switch_takes_multiples_of_8_px(h, w):
    """SD-v1.4 with the switch on (latent multiple 1, VAE factor 8): a size on the rule passes the check and fails
    later, on the stand-in's missing parts."""
    from e4t.pipeline_stable_diffusion_e4t import StableDiffusionE4TPipeline
    with pytest.raises(AttributeError):
        StableDiffusionE4TPipeline.__call__(_fake_pipe(1, 8, 8), prompt="a photo of *s", height=h, width=w)


@pytest.mark.parametrize("h,w,match", [(516, 512, "multiples of 8 px"), (512, 56, "at least 64 px"),
                                       (56, 512, "at least 64 px"), (8, 8, "at least 64 px")])
def test_pipeline_with_the_switch_refuses(h, w, match):
    from e4t.pipeline_stable_diffusion_e4t import StableDiffusionE4TPipeline
    with pytest.raises(ValueError, match=match):
        StableDiffusionE4TPipeline.__call__(_fake_pipe(1, 8, 8), prompt="a photo of *s", height=h, width=w)


def _step_rule(latent_multiple, hw):
    from e4t_b200.engine import PretrainStep
    unet = types.SimpleNamespace(latent_multiple=latent_multiple, min_latent_size=8)
    step = types.SimpleNamespace(unet=unet)
    batch = dict(pixel_values=None, latents=torch.zeros((1, 4) + hw), noise=None)
    return PretrainStep.forward_loss(step, batch)


@pytest.mark.parametrize("hw", [(65, 65), (63, 97), (8, 9)])
def test_step_rule_with_the_switch_takes_any_side(hw):
    """The check passes; the stand-in then fails on its missing parts."""
    with pytest.raises(KeyError):
        _step_rule(1, hw)


@pytest.mark.parametrize("hw", [(7, 64), (64, 4), (1, 1)])
def test_step_rule_with_the_switch_refuses_small_sides(hw):
    from e4t_b200._lib import E4TError
    with pytest.raises(E4TError, match="at least 8"):
        _step_rule(1, hw)


def test_step_rule_without_the_switch_is_unchanged():
    from e4t_b200._lib import E4TError
    with pytest.raises(E4TError, match="multiples of the UNet's down-sampling factor 8"):
        _step_rule(8, (65, 64))
