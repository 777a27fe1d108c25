"""CPU tests of AutoencoderKL's module surface: diffusers 0.14 state-dict keys / shapes / parameter count for the
SD-v1.x config, config attributes, from_pretrained from local directories (bin, safetensors, sharded) with strict keys,
and the refusals (CPU input, hub names)."""
import json
import os

import pytest
import torch

SD_CFG = dict(in_channels=3, out_channels=3, down_block_types=["DownEncoderBlock2D"] * 4,
              up_block_types=["UpDecoderBlock2D"] * 4, block_out_channels=[128, 256, 512, 512], layers_per_block=2,
              act_fn="silu", latent_channels=4, norm_num_groups=32, sample_size=512, scaling_factor=0.18215)
TINY_CFG = dict(SD_CFG, down_block_types=["DownEncoderBlock2D"] * 3, up_block_types=["UpDecoderBlock2D"] * 3,
                block_out_channels=[64, 128, 128], layers_per_block=1, sample_size=64)


def _model(cfg):
    from e4t.models.autoencoder_kl import AutoencoderKL
    return AutoencoderKL(**{k: tuple(v) if isinstance(v, list) else v for k, v in cfg.items()})


def test_sd_vae_inventory():
    sd = _model(SD_CFG).state_dict()
    # the published size of the Stable Diffusion v1.x VAE
    assert len(sd) == 248
    assert sum(v.numel() for v in sd.values()) == 83_653_863
    shapes = {k: tuple(v.shape) for k, v in sd.items()}
    assert shapes["encoder.conv_in.weight"] == (128, 3, 3, 3)
    assert shapes["encoder.conv_out.weight"] == (8, 512, 3, 3)
    assert shapes["quant_conv.weight"] == (8, 8, 1, 1)
    assert shapes["post_quant_conv.weight"] == (4, 4, 1, 1)
    assert shapes["decoder.conv_in.weight"] == (512, 4, 3, 3)
    assert shapes["decoder.conv_out.weight"] == (3, 128, 3, 3)
    assert shapes["encoder.down_blocks.0.downsamplers.0.conv.weight"] == (128, 128, 3, 3)
    assert "encoder.down_blocks.3.downsamplers.0.conv.weight" not in shapes
    assert shapes["encoder.down_blocks.1.resnets.0.conv_shortcut.weight"] == (256, 128, 1, 1)
    assert shapes["decoder.up_blocks.2.resnets.0.conv_shortcut.weight"] == (256, 512, 1, 1)
    assert shapes["decoder.up_blocks.0.upsamplers.0.conv.weight"] == (512, 512, 3, 3)
    assert "decoder.up_blocks.3.upsamplers.0.conv.weight" not in shapes
    assert len([k for k in shapes if k.startswith("decoder.up_blocks.0.resnets.")]) == 3 * 8
    for side in ("encoder", "decoder"):
        p = f"{side}.mid_block.attentions.0."
        for n in ("query", "key", "value", "proj_attn"):
            assert shapes[p + n + ".weight"] == (512, 512) and shapes[p + n + ".bias"] == (512,)
        assert shapes[p + "group_norm.weight"] == (512,)


def test_config_surface():
    vae = _model(SD_CFG)
    assert vae.config.scaling_factor == 0.18215
    assert tuple(vae.config.block_out_channels) == (128, 256, 512, 512)
    assert vae.config["latent_channels"] == 4
    assert vae.dtype == torch.float32
    # the pipeline's latent-to-pixel factor
    assert 2 ** (len(vae.config.block_out_channels) - 1) == 8


def _save(vae, d, fmt):
    os.makedirs(d, exist_ok=True)
    vae.save_config(d)
    sd = {k: v.contiguous() for k, v in vae.state_dict().items()}
    if fmt == "bin":
        torch.save(sd, os.path.join(d, "diffusion_pytorch_model.bin"))
    elif fmt == "safetensors":
        from safetensors.torch import save_file
        save_file(sd, os.path.join(d, "diffusion_pytorch_model.safetensors"))
    else:
        keys = sorted(sd)
        halves = [keys[:len(keys) // 2], keys[len(keys) // 2:]]
        wm = {}
        for i, ks in enumerate(halves):
            name = f"diffusion_pytorch_model-0000{i + 1}-of-00002.bin"
            torch.save({k: sd[k] for k in ks}, os.path.join(d, name))
            wm.update({k: name for k in ks})
        with open(os.path.join(d, "diffusion_pytorch_model.bin.index.json"), "w") as f:
            json.dump({"weight_map": wm}, f)


@pytest.mark.parametrize("fmt", ["bin", "safetensors", "sharded"])
def test_from_pretrained_round_trip(tmp_path, fmt):
    from e4t.models.autoencoder_kl import AutoencoderKL
    if fmt == "safetensors":
        pytest.importorskip("safetensors")
    torch.manual_seed(0)
    vae = _model(TINY_CFG)
    _save(vae, str(tmp_path / "vae"), fmt)
    got = AutoencoderKL.from_pretrained(str(tmp_path), subfolder="vae")
    assert tuple(got.config.block_out_channels) == (64, 128, 128)
    a, b = vae.state_dict(), got.state_dict()
    assert a.keys() == b.keys()
    assert all(torch.equal(a[k], b[k]) for k in a)


def test_from_pretrained_is_strict(tmp_path):
    from e4t.models.autoencoder_kl import AutoencoderKL
    vae = _model(TINY_CFG)
    d = str(tmp_path / "vae")
    _save(vae, d, "bin")
    sd = torch.load(os.path.join(d, "diffusion_pytorch_model.bin"))
    sd["encoder.mid_block.attentions.0.to_q.weight"] = sd.pop("encoder.mid_block.attentions.0.query.weight")
    torch.save(sd, os.path.join(d, "diffusion_pytorch_model.bin"))
    with pytest.raises(RuntimeError, match="missing keys"):
        AutoencoderKL.from_pretrained(str(tmp_path), subfolder="vae")
    sd["encoder.mid_block.attentions.0.query.weight"] = sd["encoder.mid_block.attentions.0.to_q.weight"]
    torch.save(sd, os.path.join(d, "diffusion_pytorch_model.bin"))
    with pytest.raises(RuntimeError, match="unexpected keys"):
        AutoencoderKL.from_pretrained(str(tmp_path), subfolder="vae")


def test_from_pretrained_hub_name_raises():
    from e4t.models.autoencoder_kl import AutoencoderKL
    with pytest.raises(FileNotFoundError):
        AutoencoderKL.from_pretrained("CompVis/stable-diffusion-v1-4", subfolder="vae")


def test_cpu_input_raises():
    from e4t_b200._lib import E4TError
    vae = _model(TINY_CFG).requires_grad_(False)
    with pytest.raises(E4TError):
        vae.encode(torch.zeros(1, 3, 64, 64))
    with pytest.raises(E4TError):
        vae.decode(torch.zeros(1, 4, 16, 16))


def test_block_factories_and_padding():
    from e4t.models.resnet import Downsample2D
    from e4t.models.unet_2d_blocks import DownEncoderBlock2D, UpDecoderBlock2D, get_down_block, get_up_block
    b = get_down_block("DownEncoderBlock2D", num_layers=2, in_channels=64, out_channels=128, temb_channels=None,
                       add_downsample=True, resnet_eps=1e-6, resnet_act_fn="silu", attn_num_head_channels=None,
                       resnet_groups=32, downsample_padding=0)
    assert isinstance(b, DownEncoderBlock2D) and b.downsamplers[0].padding == 0
    assert b.downsamplers[0].conv.padding == (0, 0)
    u = get_up_block("UpDecoderBlock2D", num_layers=3, in_channels=128, out_channels=64, prev_output_channel=None,
                     temb_channels=None, add_upsample=False, resnet_eps=1e-6, resnet_act_fn="silu",
                     attn_num_head_channels=None, resnet_groups=32)
    assert isinstance(u, UpDecoderBlock2D) and u.upsamplers is None and len(u.resnets) == 3
    with pytest.raises(NotImplementedError):
        Downsample2D(64, use_conv=True, padding=2)


GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vae.pt")


def test_oracle_matches_reference_golden():
    """oracle/vae_oracle.py against the reference's own VAE blocks (tests/golden/vae.pt, oracle/gen_golden_vae.py)."""
    from oracle import e4t_oracle as O
    from oracle import vae_oracle as V
    gold = torch.load(GOLD)
    cfg = gold["cfg"]
    sd = O.synth_state_dict(V.vae_param_shapes(cfg), gold["seed"])
    with torch.no_grad():
        moments = V.vae_encode(sd, cfg, gold["x"])
        decoded = V.vae_decode(sd, cfg, gold["z"])
    torch.testing.assert_close(moments, gold["moments"], rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(V.vae_sample(moments, gold["noise"]), gold["sample"], rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(decoded, gold["decoded"], rtol=1e-4, atol=1e-5)


def test_sd_vae_inventory_matches_reference():
    from oracle import vae_oracle as V
    inv = torch.load(GOLD)["sd_inventory"]
    shapes = {k: tuple(v.shape) for k, v in _model(SD_CFG).state_dict().items()}
    assert V.vae_inventory(shapes) == inv
    assert V.vae_inventory(V.vae_param_shapes(V.SD_VAE)) == inv
    assert inv["n_keys"] == 248 and inv["n_params"] == 83_653_863
