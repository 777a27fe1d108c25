"""A/B timing at image sizes other than 512²: e4t (sm_90a kernels) against stock torch on the same weights (the
oracle's composition on torch ops under bf16 autocast, channels_last 4-D weights and activations, cuDNN convolutions,
SDPA attention).

    python tools/resolution_ab.py [--iters 10] [--sizes 512x512,768x512,...] [--skip-conv] [--ragged]

1. Per image size (H x W pixels): one SD-v1.4 classifier-free-guidance denoising step (encoder-half UNet on one
   latent, E4T encoder head with CLIP ViT-H/14, CLIP-L text encoder, full UNet on two latents) and the SD VAE decode of
   one latent, the two paths timed alternately with CUDA events: median and min - max in ms.
2. ops.conv3x3_im2col against ops.conv3x3 (tiled A box) on the 512² UNet (B = 2, the CFG batch) and VAE (B = 1)
   convolution shapes, where both accept the input.
3. e4t_conv3x3_wgrad picks its load by shape, so its tiled load is timed at 512² training shapes (B = 16) and its
   im2col load on the same batch with every row one pixel shorter, compared per pixel.
--ragged: sizes that are multiples of 8 px but not of 64 (520², 544 x 672, 504 x 776), each followed by the nearest
multiple-of-64 size, with UNet2DConditionModel.enable_any_latent_size(): the difference is the cost of the im2col
loads, the explicit-size resize and zero insertion, and the mma.sync attention at ragged token counts.
The card, its power limit and SM clock are read in the same run.  Synthetic weights (PyTorch's default init)."""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "e4t-diffusion_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from oracle import e4t_oracle as O  # noqa: E402
from oracle import ragged_oracle as RO  # noqa: E402
from oracle import vae_oracle as V  # noqa: E402

SIZES = "512x512,768x512,512x768,576x576,640x640,768x768"
# each ragged size, then its nearest multiple-of-64 size (ties round down)
RAGGED = "520x520,512x512,544x672,512x640,504x776,512x768"


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def stats(ts):
    s = sorted(ts)
    return s[len(s) // 2], s[0], s[-1]


def alternate(fns, iters):
    """{name: [ms, ...]}: each function once per round, in turn, CUDA events around it."""
    out = {n: [] for n in fns}
    for n, f in fns.items():      # warm-up: module loads, cuDNN / tensor-map choices
        f(); f()
    torch.cuda.synchronize()
    for _ in range(iters):
        for n, f in fns.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            b.synchronize()
            out[n].append(a.elapsed_time(b))
    return out


def cl(sd):
    return {k: (v.contiguous(memory_format=torch.channels_last) if v.dim() == 4 else v) for k, v in sd.items()}


def e4t_cfg_step(unet, enc, text, lat, pix, ids, idx, t, ehs_e4t, class_embed):
    with torch.no_grad():
        e = unet(lat, t, ehs_e4t, return_encoder_outputs=True)
        dom = class_embed + 0.1 * enc(x=pix, unet_down_block_samples=e["down_block_samples"]).float()
        emb = text.get_input_embeddings()(ids).clone()
        emb[:, idx, :] = dom.to(emb.dtype)
        ehs = text(inputs_embeds=emb)[0].to(torch.bfloat16)
        pred = unet(torch.cat([lat, lat]), t.expand(2), torch.cat([ehs_e4t, ehs])).sample
        u, c = pred.chunk(2)
        return u + 7.5 * (c - u)


def torch_cfg_step(sd_u, sd_e, sd_t, lat, pix, ids, idx, t, ehs_e4t, class_embed):
    tok = sd_t["text_model.embeddings.token_embedding.weight"]
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        e = RO.unet_forward(sd_u, O.SD14_UNET, lat, t, ehs_e4t, return_encoder_outputs=True)
        dom = class_embed + 0.1 * O.encoder_forward(sd_e, O.VIT_H14, pix, e["down_block_samples"]).float()
        emb = tok[ids].clone()
        emb[:, idx, :] = dom.to(emb.dtype)
        ehs = O.text_forward(sd_t, O.CLIP_TEXT_L, inputs_embeds=emb)
        pred = RO.unet_forward(sd_u, O.SD14_UNET, torch.cat([lat, lat]), t.expand(2), torch.cat([ehs_e4t, ehs]))
        u, c = pred.float().chunk(2)
        return u + 7.5 * (c - u)


def conv_table(iters):
    from e4t_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(0)
    rows = []
    # (B, H, W, Cin, Cout): 512² UNet levels 0-3 (CFG batch 2) and the SD VAE decoder levels (B = 1)
    shapes = [(2, 64, 64, 320, 320), (2, 32, 32, 640, 640), (2, 16, 16, 1280, 1280), (2, 8, 8, 1280, 1280),
              (2, 64, 64, 640, 320), (1, 64, 64, 512, 512), (1, 128, 128, 512, 512), (1, 256, 256, 256, 256),
              (1, 512, 512, 128, 128)]
    for B, H, W, Ci, Co in shapes:
        x = (torch.randn(B, H, W, Ci, generator=g, device="cuda")).to(torch.bfloat16)
        w = (torch.randn(9, Co, Ci, generator=g, device="cuda") * 0.05).to(torch.bfloat16)
        same = torch.equal(ops.conv3x3(x, w), ops.conv3x3_im2col(x, w))
        r = alternate({"tiled": lambda: ops.conv3x3(x, w), "im2col": lambda: ops.conv3x3_im2col(x, w)}, iters)
        rows.append((f"conv3x3 {B}x{H}x{W} {Ci}->{Co}", stats(r["tiled"]), stats(r["im2col"]), same))
    return rows


def wgrad_table(iters):
    """e4t_conv3x3_wgrad chooses its load by shape, so the tiled and im2col loads are compared on a 512² training shape
    and on the same pixel count laid out so that only im2col applies (the rows of one image are one pixel narrower)."""
    from e4t_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(1)
    rows = []
    for (B, H, W), (H2, W2), Ci, Co in [((16, 64, 64), (64, 63), 320, 320), ((16, 32, 32), (32, 31), 640, 640),
                                        ((16, 16, 16), (16, 15), 1280, 1280), ((16, 8, 8), (8, 7), 1280, 1280)]:
        x = torch.randn(B, H, W, Ci, generator=g, device="cuda").to(torch.bfloat16)
        dy = torch.randn(B, H, W, Co, generator=g, device="cuda").to(torch.bfloat16)
        x2, dy2 = x[:, :H2, :W2].contiguous(), dy[:, :H2, :W2].contiguous()
        r = alternate({"tiled": lambda: ops.conv3x3_wgrad(x, dy), "im2col": lambda: ops.conv3x3_wgrad(x2, dy2)}, iters)
        rows.append((f"wgrad {B}x{H}x{W} vs {B}x{H2}x{W2} {Ci}->{Co}", stats(r["tiled"]), stats(r["im2col"]),
                     (H2 * W2) / (H * W)))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--sizes", default=SIZES)
    ap.add_argument("--skip-conv", action="store_true")
    ap.add_argument("--ragged", action="store_true", help=f"time {RAGGED} (sizes that are multiples of 8 px)")
    args = ap.parse_args()
    if args.ragged:
        args.sizes = RAGGED
    print("card:", card())
    import bench
    from e4t.models.autoencoder_kl import AutoencoderKL
    torch.backends.cudnn.benchmark = True
    unet, enc, text = bench.build_models("cuda")
    if args.ragged:
        unet.enable_any_latent_size()
    sd_u, sd_e, sd_t = (cl({k: v for k, v in m.state_dict().items()}) for m in (unet, enc, text))
    sd_t = {k: v.float() for k, v in sd_t.items()}
    b = bench.to_device(bench.host_batch(1, 3, pinned=False), "cuda")
    ids, idx, t, pix = b["input_ids"], int(b["placeholder_idxs"][0]), b["timesteps"], b["pixel_values"]
    with torch.no_grad():
        ehs_e4t = text(input_ids=torch.tensor([[49406] + [49407] * 76], device="cuda"))[0].to(torch.bfloat16)
        class_embed = text.get_input_embeddings()(torch.tensor([320], device="cuda")).float()
    torch.manual_seed(0)
    vae = AutoencoderKL(**V.SD_VAE).cuda().eval().requires_grad_(False)
    sd_v = cl({k: v.float() for k, v in vae.state_dict().items()})
    print(f"{'image':>9} | {'CFG step e4t ms (min-max)':>26} | {'torch ms (min-max)':>22} | {'ratio':>5} | "
          f"{'VAE decode e4t ms':>24} | {'torch ms':>22} | ratio | diff step / decode")
    for s in args.sizes.split(","):
        Hp, Wp = (int(v) for v in s.split("x"))
        g = torch.Generator(device="cuda").manual_seed(Hp * Wp)
        lat = torch.randn(1, 4, Hp // 8, Wp // 8, generator=g, device="cuda")
        latc = lat.contiguous(memory_format=torch.channels_last)
        z = torch.randn(1, 4, Hp // 8, Wp // 8, generator=g, device="cuda")
        zc = z.contiguous(memory_format=torch.channels_last)

        def ours_step():
            return e4t_cfg_step(unet, enc, text, lat, pix, ids, idx, t, ehs_e4t, class_embed)

        def torch_step():
            return torch_cfg_step(sd_u, sd_e, sd_t, latc, pix, ids, idx, t, ehs_e4t, class_embed)

        def ours_dec():
            with torch.no_grad():
                return vae.decode(z).sample

        def torch_dec():
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                return V.vae_decode(sd_v, V.SD_VAE, zc)
        r = alternate({"os": ours_step, "ts": torch_step}, args.iters)
        d = alternate({"od": ours_dec, "td": torch_dec}, args.iters)
        rel = lambda a, c: ((a.float() - c.float()).pow(2).mean().sqrt() / c.float().pow(2).mean().sqrt()).item()
        e_s, e_d = rel(ours_step(), torch_step()), rel(ours_dec(), torch_dec())
        (om, olo, ohi), (tm, tlo, thi) = stats(r["os"]), stats(r["ts"])
        (dm, dlo, dhi), (vm, vlo, vhi) = stats(d["od"]), stats(d["td"])
        print(f"{Hp:>4}x{Wp:<4} | {om:8.2f} ({olo:6.2f}-{ohi:6.2f}) | {tm:8.2f} ({tlo:6.2f}-{thi:6.2f}) | "
              f"{tm / om:5.2f} | {dm:8.2f} ({dlo:6.2f}-{dhi:6.2f}) | {vm:8.2f} ({vlo:6.2f}-{vhi:6.2f}) | "
              f"{vm / dm:5.2f} | {e_s:.2e} / {e_d:.2e}", flush=True)
        torch.cuda.empty_cache()
    if not args.skip_conv:
        print("\nsame input, both loads (ms median (min-max)); identical = bit-identical outputs")
        for name, a, c, same in conv_table(max(args.iters, 20)):
            print(f"{name:>34}: tiled {a[0]:.3f} ({a[1]:.3f}-{a[2]:.3f})  im2col {c[0]:.3f} ({c[1]:.3f}-{c[2]:.3f})"
                  f"  {c[0] / a[0] - 1:+.1%}  identical={same}")
        print("\nweight gradient: tiled box at 512² shapes vs im2col at the same batch one column narrower")
        for name, a, c, frac in wgrad_table(max(args.iters, 20)):
            print(f"{name:>44}: tiled {a[0]:.3f} ({a[1]:.3f}-{a[2]:.3f})  im2col {c[0]:.3f} ({c[1]:.3f}-{c[2]:.3f})"
                  f"  per pixel {c[0] / frac / a[0] - 1:+.1%}")
    print("card:", card())


if __name__ == "__main__":
    main()
