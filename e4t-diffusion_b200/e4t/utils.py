"""Checkpoint / config helpers — the state-dict key contract of e4t/utils.py:76-159:
  weight_offsets.pt = {k: v for k in unet.state_dict() if "wo" in k}   (utils.py:129-131)
  encoder.pt        = encoder.state_dict()                               (utils.py:158-159)
  config.json       = argparse namespace, read back as AttributeDict     (utils.py:17-40,76-89)
Hub download (utils.py:43-73) needs network and is out of scope; local paths work the same way."""
import json
import os

import torch

from e4t.encoder import E4TEncoder
from e4t.models.unet_2d_condition import UNet2DConditionModel


class AttributeDict(dict):
    """dict with attribute access; a missing attribute reads as None (utils.py:17-40)."""

    def __getattr__(self, k):
        return self.get(k, None)

    def __setattr__(self, k, v):
        self[k] = v

    def __delattr__(self, k):
        del self[k]


def load_config_from_pretrained(pretrained_model_name_or_path):
    if not os.path.exists(pretrained_model_name_or_path):
        raise FileNotFoundError(f"{pretrained_model_name_or_path} (hub download is unavailable offline)")
    if "config.json" not in pretrained_model_name_or_path:
        pretrained_model_name_or_path = os.path.join(pretrained_model_name_or_path, "config.json")
    with open(pretrained_model_name_or_path, "r", encoding="utf-8") as f:
        return AttributeDict(json.load(f))


def load_e4t_unet(pretrained_model_name_or_path=None, ckpt_path=None, **kwargs):
    """Base SD UNet weights from a local diffusers-format directory (<path>/unet/{config.json,*.bin}) overlaid with
    weight_offsets.pt / unet.pt; missing keys are tolerated only for a fresh WO init, unexpected keys are fatal
    (utils.py:92-126)."""
    assert pretrained_model_name_or_path is not None or ckpt_path is not None
    if pretrained_model_name_or_path is None:
        assert os.path.basename(ckpt_path) in ("unet.pt", "weight_offsets.pt"), \
            "You must specify the filename! (`unet.pt` or `weight_offsets.pt`)"
        config = load_config_from_pretrained(os.path.dirname(ckpt_path))
        pretrained_model_name_or_path = config.pretrained_model_name_or_path if config.pretrained_args is None \
            else config.pretrained_args["pretrained_model_name_or_path"]
    d = os.path.join(pretrained_model_name_or_path, "unet")
    with open(os.path.join(d, "config.json")) as f:
        cfg = {k: v for k, v in json.load(f).items() if not k.startswith("_")}
    unet = UNet2DConditionModel(**cfg)
    state_dict = _load_diffusers_weights(d)
    if not state_dict:
        # the reference goes through OriginalUNet2DConditionModel.from_pretrained (utils.py:114) and therefore always
        # starts from real base weights; a directory without a weight file must not silently mean "random init"
        raise FileNotFoundError(f"no UNet weights under {d} (looked for diffusion_pytorch_model.{{bin,safetensors}} "
                                f"and their sharded *.index.json forms)")
    if ckpt_path:
        state_dict.update(torch.load(ckpt_path, map_location="cpu"))
        print(f"Resuming from {ckpt_path}")
    m, u = unet.load_state_dict(state_dict, strict=False)
    if ckpt_path is None:
        m = [k for k in m if "wo" not in k]      # a fresh run starts its WeightOffsets from their default init
    if len(m) > 0:
        raise RuntimeError(f"missing keys:\n{m}")
    if len(u) > 0:
        raise RuntimeError(f"unexpected keys:\n{u}")
    return unet


def _load_diffusers_weights(d, stem="diffusion_pytorch_model"):
    """state dict of a diffusers-format model directory: <stem>.bin / <stem>.safetensors or the sharded
    <stem>.{bin,safetensors}.index.json forms."""
    state_dict = {}

    def load_one(path):
        if path.endswith(".safetensors"):
            from safetensors.torch import load_file
            return load_file(path, device="cpu")
        return torch.load(path, map_location="cpu")

    for ext in ("safetensors", "bin"):
        single = os.path.join(d, f"{stem}.{ext}")
        index = single + ".index.json"
        if os.path.exists(single):
            state_dict.update(load_one(single))
            break
        if os.path.exists(index):
            with open(index) as f:
                shards = sorted(set(json.load(f)["weight_map"].values()))
            for sh in shards:
                state_dict.update(load_one(os.path.join(d, sh)))
            break
    return state_dict


def _detached(sd):
    """Clones: after FlatAdamW the trainable parameters are views of one 1.5 GB arena, and torch.save serialises the
    whole storage behind every view (ADVICE r1)."""
    return {k: v.detach().clone().contiguous() for k, v in sd.items()}


def save_e4t_unet(model, save_dir, save_all=False):
    """weight_offsets.pt = the "wo" entries (utils.py:129-131); save_all=True -> unet.pt = the full state dict
    (tuning_e4t.py:232)."""
    os.makedirs(save_dir, exist_ok=True)
    if save_all:
        torch.save(_detached(model.state_dict()), os.path.join(save_dir, "unet.pt"))
    else:
        torch.save(_detached({k: v for k, v in model.state_dict().items() if "wo" in k}),
                   os.path.join(save_dir, "weight_offsets.pt"))


def save_text_encoder(model, save_dir):
    """text_encoder.pt = the text encoder's state dict (tuning_e4t.py:236-237, --train_text_encoder), as clones: under
    the optimiser arena its parameters are views of one multi-GB storage.  inference.py:95-103 loads it with strict
    missing / unexpected key checks."""
    os.makedirs(save_dir, exist_ok=True)
    torch.save(_detached(model.state_dict()), os.path.join(save_dir, "text_encoder.pt"))


def save_config(args, save_dir, pretrained_args=None):
    """config.json as the training scripts write it (pretrain_e4t.py:230-234; nested `pretrained_args` when a run
    starts from an earlier E4T checkpoint, utils.py:76-89)."""
    os.makedirs(save_dir, exist_ok=True)
    cfg = dict(vars(args)) if not isinstance(args, dict) else dict(args)
    if pretrained_args is not None:
        cfg["pretrained_args"] = dict(pretrained_args)
    with open(os.path.join(save_dir, "config.json"), "w", encoding="utf-8") as f:
        json.dump(cfg, f, indent=2, default=str)
    return cfg


def load_e4t_encoder(ckpt_path=None, **kwargs):
    encoder = E4TEncoder(**kwargs)
    if ckpt_path:
        if not os.path.exists(ckpt_path):
            raise FileNotFoundError(f"{ckpt_path} (hub download is unavailable offline)")
        if "encoder.pt" not in ckpt_path:
            ckpt_path = os.path.join(ckpt_path, "encoder.pt")
        state_dict = torch.load(ckpt_path, map_location="cpu")
        print(f"Resuming from {ckpt_path}")
        m, u = encoder.load_state_dict(state_dict, strict=False)
        if len(m) > 0:
            raise RuntimeError(f"missing keys:\n{m}")
        if len(u) > 0:
            raise RuntimeError(f"unexpected keys:\n{u}")
    return encoder


def save_e4t_encoder(model, save_dir):
    os.makedirs(save_dir, exist_ok=True)
    torch.save(_detached(model.state_dict()), os.path.join(save_dir, "encoder.pt"))


def image_grid(imgs, rows, cols):
    from PIL import Image
    assert len(imgs) == rows * cols
    w, h = imgs[0].size
    grid = Image.new("RGB", size=(cols * w, rows * h))
    for i, img in enumerate(imgs):
        grid.paste(img, box=(i % cols * w, i // cols * h))
    return grid


def load_image(image_path, resolution=None):
    """PIL RGB image from a local path or URL; with `resolution`, the shorter side is resized to it (Lanczos,
    albumentations.SmallestMaxSize(interpolation=3) in the reference) and the centre square is cropped
    (utils.py:162-177)."""
    from PIL import Image, ImageOps
    if image_path.startswith("http://") or image_path.startswith("https://"):
        import requests
        img = Image.open(requests.get(image_path, stream=True).raw)
    else:
        img = Image.open(image_path)
    img = ImageOps.exif_transpose(img).convert("RGB")
    if resolution:
        w, h = img.size
        s = resolution / min(w, h)
        img = img.resize((max(resolution, round(w * s)), max(resolution, round(h * s))), resample=Image.LANCZOS)
        w, h = img.size
        left, top = (w - resolution) // 2, (h - resolution) // 2
        img = img.crop((left, top, left + resolution, top + resolution))
    return img
