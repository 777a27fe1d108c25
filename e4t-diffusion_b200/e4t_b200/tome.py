"""Token merging (ToMe) for the UNet's transformer blocks, the equivalent of `tomesd.apply_patch(pipe, ratio=0.5)`.

    from e4t_b200 import tome
    tome.apply_patch(pipe, ratio=0.5)      # or a UNet2DConditionModel; PretrainStep / TuningStep built on it train so
    ...
    tome.remove_patch(pipe)

The rules are those of tomesd 0.1.x (bipartite_soft_matching_random2d and its patched diffusers block):
  * the UNet's latent is H0 x W0 (N0 tokens); a block whose input has N tokens merges when
    downsample = ceil(sqrt(N0 // N)) <= max_downsample; its grid is h = ceil(H0 / downsample), w = ceil(W0 / downsample)
    (checked against the block's real size) and it merges r = min(int(N * ratio), N_src) tokens;
  * per block call, from the block input x (before norm1) and without gradient: one dst token per sy x sx cell at an
    offset drawn uniformly per cell (shared by the batch; the top-left token when use_rand=False or the batch is odd),
    every other token src; each src token's best dst by cosine similarity (ties to the lowest raster index); the r src
    tokens with the largest similarity are merged into their dst (ties to the lower raster index);
  * merge ("mean"): a dst row becomes (x_dst + sum of its merged src) / (1 + count), a kept src row is copied; kept
    tokens stay in raster order.  Unmerge: every token reads the row of its representative, then the residual is added;
  * merge_attn: x = unmerge(attn1(merge(norm1(x)))) + x; merge_crossattn / merge_mlp do the same for attn2 / ff, all
    with the one matching of the block input.

Everything runs on the kernels of csrc/tome.cu; the patterns are drawn on the device from torch's CUDA generator, so a
captured CUDA graph draws fresh ones at every replay.
"""
import math
from dataclasses import dataclass

import torch

from . import ops
from ._lib import E4TError

_SERIAL = [0]


@dataclass(frozen=True)
class ToMeArgs:
    ratio: float = 0.5
    max_downsample: int = 1
    sx: int = 2
    sy: int = 2
    use_rand: bool = True
    merge_attn: bool = True
    merge_crossattn: bool = False
    merge_mlp: bool = False


def check_args(ratio, max_downsample, sx, sy):
    if not (isinstance(ratio, (int, float)) and 0.0 <= ratio < 1.0):
        raise E4TError(f"ToMe ratio must be in [0, 1), got {ratio!r}")
    if max_downsample not in (1, 2, 4, 8):
        raise E4TError(f"ToMe max_downsample must be 1, 2, 4 or 8, got {max_downsample!r}")
    if not (isinstance(sx, int) and isinstance(sy, int) and sx >= 1 and sy >= 1):
        raise E4TError(f"ToMe strides sx, sy must be integers >= 1, got ({sx!r}, {sy!r})")


def block_geometry(H0, W0, N, args):
    """(downsample, h, w, r) of a block with N input tokens under a latent of H0 x W0, or None when it does not merge."""
    ds = int(math.ceil(math.sqrt((H0 * W0) // N)))
    if ds > args.max_downsample:
        return None
    h, w = int(math.ceil(H0 / ds)), int(math.ceil(W0 / ds))
    n_dst = (h // args.sy) * (w // args.sx)
    r = min(int(N * args.ratio), N - n_dst) if n_dst > 0 else 0
    return ds, h, w, r


def _unet_of(model):
    from e4t.models.unet_2d_condition import UNet2DConditionModel
    if isinstance(model, UNet2DConditionModel):
        return model
    unet = getattr(model, "unet", None)
    if isinstance(unet, UNet2DConditionModel):
        return unet
    raise TypeError(f"ToMe patches a UNet2DConditionModel or a pipeline holding one, not {type(model).__name__}")


def apply_patch(model, ratio=0.5, max_downsample=1, sx=2, sy=2, use_rand=True, merge_attn=True, merge_crossattn=False,
                merge_mlp=False):
    """Merge tokens in the transformer blocks of `model` (a UNet2DConditionModel or a StableDiffusionE4TPipeline).
    Replaces an earlier patch; ratio = 0 leaves the model unpatched."""
    check_args(ratio, max_downsample, sx, sy)
    unet = _unet_of(model)
    remove_patch(unet)
    if ratio == 0:
        return model
    from e4t.models.attention import BasicTransformerBlock
    _SERIAL[0] += 1
    info = dict(args=ToMeArgs(float(ratio), max_downsample, sx, sy, bool(use_rand), bool(merge_attn),
                              bool(merge_crossattn), bool(merge_mlp)),
                size=None, serial=_SERIAL[0], record=None)

    def size_hook(module, args, kwargs):
        sample = args[0] if args else kwargs["sample"]
        info["size"] = tuple(sample.shape[-2:])

    info["hook"] = unet.register_forward_pre_hook(size_hook, with_kwargs=True)
    unet._tome_info = info
    for m in unet.modules():
        if isinstance(m, BasicTransformerBlock):
            m._tome = info
    return model


def remove_patch(model):
    """Undo apply_patch: the blocks run their unpatched path again."""
    unet = _unet_of(model)
    info = getattr(unet, "_tome_info", None)
    if info is not None:
        info["hook"].remove()
        unet._tome_info = None
    for m in unet.modules():
        if getattr(m, "_tome", None) is not None:
            m._tome = None
    return model


def signature(model):
    """Identifies the patch in force (None when unpatched): captured CUDA graphs are keyed and checked by it."""
    info = getattr(_unet_of(model), "_tome_info", None)
    return None if info is None else info["serial"]


class record_plans:
    """Context manager: every merging block call of the patched `model` appends its plan (the dict of `plan`) to
    the list it yields, in call order."""

    def __init__(self, model):
        self.info = getattr(_unet_of(model), "_tome_info", None)
        if self.info is None:
            raise E4TError("record_plans: the model has no ToMe patch")

    def __enter__(self):
        self.info["record"] = []
        return self.info["record"]

    def __exit__(self, *exc):
        self.info["record"] = None
        return False


def plan(info, x, hw):
    """The matching of one block call: None when the block does not merge, else the dict of ops.tome_match and
    ops.tome_select (plus the grid and r) that ToMeMergeFn / ToMeUnmergeFn take."""
    if info["size"] is None:
        raise E4TError("ToMe: the patched UNet's forward has not recorded the latent size")
    a = info["args"]
    H0, W0 = info["size"]
    N = x.shape[1]
    geo = block_geometry(H0, W0, N, a)
    if geo is None:
        return None
    ds, h, w, r = geo
    if (h, w) != tuple(hw):
        raise E4TError(f"ToMe: a block of {hw[0]} x {hw[1]} tokens under a {H0} x {W0} latent does not have the "
                       f"{h} x {w} grid of downsample {ds}")
    if r <= 0:
        return None
    B = x.shape[0]
    with torch.no_grad():
        shape = (h // a.sy, w // a.sx)
        if a.use_rand and B % 2 == 0:
            pattern = torch.randint(0, a.sy * a.sx, shape, device=x.device, dtype=torch.int32)
        else:
            pattern = torch.zeros(shape, device=x.device, dtype=torch.int32)
        m = ops.tome_match(x.detach().contiguous(), pattern, h, w, a.sy, a.sx)
        p = ops.tome_select(m, r)
    p.update(m, pattern=pattern, grid=(h, w), r=r)
    if info["record"] is not None:
        info["record"].append(p)
    return p
