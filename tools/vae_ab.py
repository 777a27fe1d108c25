"""A/B timing of the VAE: e4t's AutoencoderKL (sm_90a kernels) against stock torch on the same weights (the oracle's
diffusers 0.14 composition on torch ops under bf16 autocast, channels_last activations and weights, cuDNN convolutions).

    python tools/vae_ab.py [--batch 16] [--res 512] [--iters 10] [--step-iters 5]

1. Both directions (encode B x 3 x res², decode B x 4 x (res/8)²) timed alternately in one process with CUDA events, the
   L2 cache flushed before every timed call: median and min - max, images/s, TFLOP/s (FLOPs counted from the torch
   path's shapes by torch.utils.flop_counter), and the relative RMS difference between the two outputs.
2. A per-layer breakdown of our path (CUDA events around every block, median of three runs).
3. The SD-v1.4 pre-training step (bench.py's models and batches, eager launches) given latents, against the same step
   encoding pixel_values into latents on the device with the VAE attached, alternately.
The card, its power limit and SM clock are read before and after.  Synthetic weights (PyTorch's default init)."""
import argparse
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "e4t-diffusion_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

from oracle import vae_oracle as V  # noqa: E402


# ---- stock torch path: the fp32 oracle's composition (oracle/vae_oracle.py) under bf16 autocast ---------------------
def torch_encode(sd, x):
    with torch.autocast("cuda", dtype=torch.bfloat16):
        return V.vae_encode(sd, V.SD_VAE, x)


def torch_decode(sd, z):
    with torch.autocast("cuda", dtype=torch.bfloat16):
        return V.vae_decode(sd, V.SD_VAE, z)


# ---- measurement ---------------------------------------------------------------------------------------------------
def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks_event_reasons.active"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt()).item()


def breakdown(vae, x, z, reps=3):
    """Per-block device time of our encode and decode (CUDA events around each block)."""
    from e4t.models.resnet import f32
    from e4t.models.vae import _conv_in
    from e4t_b200 import functional as FN
    from e4t_b200 import ops
    import torch.nn.functional as F

    def run():
        rows = []

        def timed(name, fn):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            out = fn()
            b.record()
            rows.append((name, a, b))
            return out

        def ends(prefix, m, h):
            n = m.conv_norm_out
            h = timed(f"{prefix}.conv_norm_out+silu", lambda: ops.groupnorm_fwd(h, f32(n.weight), f32(n.bias),
                                                                                n.num_groups, n.eps, True)[0])
            c = m.conv_out
            rows.append(_direct(f"{prefix}.conv_out {c.in_channels}->{c.out_channels} direct", c, h))
            if prefix == "dec":     # what the decoder runs: the engine with Cout padded to 64 (vae.py _norm_act_out)
                timed(f"{prefix}.conv_out {c.in_channels}->{c.out_channels} engine",
                      lambda: _norm_act_out_conv_only(c, h))

        def _direct(name, c, h):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            ops.conv_out_fwd(h, f32(c.weight).contiguous(), f32(c.bias))
            b.record()
            return (name, a, b)

        def _norm_act_out_conv_only(c, h):
            co = c.out_channels
            w9 = FN.prepared(c.weight, "w9_pad64", None)
            bias = FN.prepared(c.bias, "f32_pad64", None)
            return ops.conv3x3(h, w9, bias=bias, out_dtype=torch.float32)[..., :co].permute(0, 3, 1, 2).contiguous()

        def mid(prefix, m, h):
            h = timed(f"{prefix}.mid.resnet0", lambda: m.resnets[0](h, None))
            h = timed(f"{prefix}.mid.attention", lambda: m.attentions[0](h))
            return timed(f"{prefix}.mid.resnet1", lambda: m.resnets[1](h, None))

        e = vae.encoder
        h = timed("enc.conv_in 3->128", lambda: _conv_in(e.conv_in, x))
        for i, blk in enumerate(e.down_blocks):
            for j, r in enumerate(blk.resnets):
                h = timed(f"enc.down{i}.resnet{j} {r.in_channels}->{r.out_channels} @{h.shape[1]}",
                          lambda r=r, h=h: r(h, None))
            if blk.downsamplers is not None:
                h = timed(f"enc.down{i}.downsample @{h.shape[1]}", lambda blk=blk, h=h: blk.downsamplers[0](h))
        h = mid("enc", e.mid_block, h)
        ends("enc", e, h)
        d = vae.decoder
        zz = F.conv2d(z, vae.post_quant_conv.weight, vae.post_quant_conv.bias)
        h = timed("dec.conv_in 4->512", lambda: _conv_in(d.conv_in, zz))
        h = mid("dec", d.mid_block, h)
        for i, blk in enumerate(d.up_blocks):
            for j, r in enumerate(blk.resnets):
                h = timed(f"dec.up{i}.resnet{j} {r.in_channels}->{r.out_channels} @{h.shape[1]}",
                          lambda r=r, h=h: r(h, None))
            if blk.upsamplers is not None:
                h = timed(f"dec.up{i}.upsample @{h.shape[1]}->{2 * h.shape[1]}", lambda blk=blk, h=h: blk.upsamplers[0](h))
        ends("dec", d, h)
        torch.cuda.synchronize()
        return [(n, a.elapsed_time(b)) for n, a, b in rows]

    run()
    runs = [run() for _ in range(reps)]
    med = [(runs[0][i][0], sorted(r[i][1] for r in runs)[reps // 2]) for i in range(len(runs[0]))]
    for side in ("enc", "dec"):
        # the decoder runs the engine conv_out; its direct-kernel row is shown for comparison only
        tot = sum(t for n, t in med if n.startswith(side) and not (side == "dec" and n.endswith(" direct")))
        print(f"per-layer breakdown, {'encode' if side == 'enc' else 'decode'} (B = {x.shape[0]}, median of {reps}): "
              f"{tot:.2f} ms in all")
        for n, t in med:
            if n.startswith(side):
                print(f"  {n:44s} {t:8.3f} ms  {100 * t / tot:5.1f} %")


def step_timing(vae, iters):
    """bench.py's SD-v1.4 pre-training step, eager, given latents vs encoding pixel_values with the VAE."""
    import importlib.util
    from e4t_b200.engine import PretrainStep
    spec = importlib.util.spec_from_file_location("e4t_bench", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    unet, enc, text = bench.build_models("cuda")
    step = PretrainStep(unet, enc, text, placeholder_token_id=49408, class_token_id=320, lr=1.6e-5,
                        weight_dtype=torch.bfloat16, vae=vae)
    hb = bench.to_device(bench.host_batch(16, 42, pinned=False), "cuda")
    cases = {"given latents": hb, "pixels -> latents (VAE)": {k: v for k, v in hb.items() if k != "latents"}}
    B = hb["latents"].shape[0]
    for b in cases.values():
        step(b)
    times = {k: [] for k in cases}
    for _ in range(iters):
        for k, b in cases.items():
            a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            step(b)
            e.record()
            e.synchronize()
            times[k].append(a.elapsed_time(e))
    for k, ts in times.items():
        ts = sorted(ts)
        med = ts[len(ts) // 2]
        print(f"pretrain step (eager) {k:26s} median {med:8.2f} ms (min {ts[0]:.2f}, max {ts[-1]:.2f})  "
              f"{B / med * 1e3:6.1f} images/s")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--step-iters", type=int, default=5)
    args = ap.parse_args()
    from torch.utils.flop_counter import FlopCounterMode
    from e4t.models.autoencoder_kl import AutoencoderKL
    torch.backends.cudnn.benchmark = True
    torch.manual_seed(0)
    vae = AutoencoderKL(**V.SD_VAE).cuda().eval().requires_grad_(False)
    sd = {k: (v.contiguous(memory_format=torch.channels_last) if v.dim() == 4 else v)
          for k, v in vae.state_dict().items()}
    B, R = args.batch, args.res
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.rand((B, 3, R, R), generator=g, device="cuda") * 2 - 1
    z = torch.randn((B, 4, R // 8, R // 8), generator=g, device="cuda")
    xb = x.contiguous(memory_format=torch.channels_last)
    zb = z.contiguous(memory_format=torch.channels_last)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    cases = {
        "encode/e4t": lambda: vae.encode(x).latent_dist.parameters,
        "encode/torch": lambda: torch_encode(sd, xb),
        "decode/e4t": lambda: vae.decode(z).sample,
        "decode/torch": lambda: torch_decode(sd, zb),
    }
    flops = {}
    with torch.no_grad():
        for d, fn, inp in (("encode", torch_encode, xb[:1]), ("decode", torch_decode, zb[:1])):
            with FlopCounterMode(display=False) as fc:
                fn(sd, inp)
            flops[d] = fc.get_total_flops() * B
        outs = {k: f() for k, f in cases.items()}
        for _ in range(2):
            for f in cases.values():
                f()
        torch.cuda.synchronize()
        times = {k: [] for k in cases}
        for _ in range(args.iters):
            for k, f in cases.items():
                flush.zero_()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                f()
                b.record()
                b.synchronize()
                times[k].append(a.elapsed_time(b))
    print(f"card: {card()}")
    print(f"B = {B}, {R}x{R} pixels / {R // 8}x{R // 8} latents, {args.iters} alternating iterations, L2 flushed")
    for k, ts in times.items():
        ts = sorted(ts)
        med = ts[len(ts) // 2]
        d = k.split("/")[0]
        print(f"{k:14s} median {med:8.2f} ms  (min {ts[0]:.2f}, max {ts[-1]:.2f})  {B / med * 1e3:7.1f} images/s  "
              f"{flops[d] / med / 1e9:6.1f} TFLOP/s  [{flops[d] / B / 1e12:.2f} TFLOP per image]")
    print(f"encode output e4t vs torch: rel RMS {rel(outs['encode/e4t'], outs['encode/torch']):.3e}")
    print(f"decode output e4t vs torch: rel RMS {rel(outs['decode/e4t'], outs['decode/torch']):.3e}")
    del outs
    torch.cuda.empty_cache()
    with torch.no_grad():
        breakdown(vae, x, z)
    step_timing(vae, args.step_iters)
    print(f"card (after): {card()}")


if __name__ == "__main__":
    main()
