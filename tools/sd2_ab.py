"""Stable Diffusion 2.x on the H100: dh = 64 self-attention and the graphed 768² training steps, with the warpgroup
(wgmma) attention kernels against the mma.sync kernels (E4T_ATTN_WGMMA=0).

    python tools/sd2_ab.py [--iters 12] [--steps 5]

1. Self-attention core, heads of 64: level 0 and level 1 of the SD 2.x UNet at 768² (9216 tokens x 5 heads, 2304 x 10)
   and 512² (4096 x 5, 1024 x 10), B = 16 and B = 1.  Forward and single-pass backward timed with CUDA events, L2
   flushed before every launch, the two paths alternating in one process (the library reads the switch on every
   call); median and min-max over --iters launches.  Outputs of the two paths are compared on the same inputs.
2. The graphed SD 2.x PretrainStep and TuningStep (v-prediction, pad id 0) at 768² (96 x 96 latents) on synthetic
   weights, once per attention path (a graph keeps the kernels it was captured with, so each path is captured on its
   own).  The batch is the largest of 16, 8, 4, 2, 1 that fits; its peak memory is reported.
Card name, power limit and SM clock are read in the same run.  Needs a GPU; fails without one.
"""
import argparse
import gc
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "e4t-diffusion_b200"), os.path.join(ROOT, "tools")]

from attn_ab import card, rel, stats  # noqa: E402

ATTN = {"768_L0": (9216, 5), "768_L1": (2304, 10), "512_L0": (4096, 5), "512_L1": (1024, 10)}
DH = 64


def attention(args, report):
    from e4t_b200 import ops
    dev = torch.device("cuda")
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)   # > 50 MB L2

    def timed(fn):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1)

    for name, (N, H) in ATTN.items():
        for B in (16, 1):
            C = H * DH
            g = torch.Generator(device=dev).manual_seed(N + B)
            qkv = (torch.randn(B, N, 3 * C, device=dev, generator=g) * 0.5).to(torch.bfloat16)
            q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
            do = (torch.randn(B, N, C, device=dev, generator=g) * 0.5).to(torch.bfloat16)
            outs = {}
            for sw in ("0", "1"):
                os.environ["E4T_ATTN_WGMMA"] = sw
                o, lse = ops.attn_fwd(q, k, v, H)
                outs[sw] = (o, lse) + tuple(ops.attn_bwd(q, k, v, o, do, lse, H))
            torch.cuda.synchronize()
            agree = {n: rel(a, b) for n, a, b in zip(("o", "lse", "dq", "dk", "dv"), outs["1"], outs["0"])}
            o, lse = outs["0"][:2]
            times = {"fwd": {"0": [], "1": []}, "bwd": {"0": [], "1": []}}
            for it in range(args.iters + 2):          # the first two rounds warm up
                for sw in ("0", "1"):
                    os.environ["E4T_ATTN_WGMMA"] = sw
                    tf = timed(lambda: ops.attn_fwd(q, k, v, H))
                    tb = timed(lambda: ops.attn_bwd(q, k, v, o, do, lse, H))
                    if it >= 2:
                        times["fwd"][sw].append(tf)
                        times["bwd"][sw].append(tb)
            fl = 4.0 * N * N * C * B
            res = {"N": N, "heads": H, "B": B, "ctas": (N // 128) * H * B, "wgmma_vs_mma_sync_rel": agree}
            for kind, mult in (("fwd", 1.0), ("bwd", 2.5)):
                for sw, label in (("0", "mma_sync"), ("1", "wgmma")):
                    st = stats(times[kind][sw])
                    st["tflops_at_median"] = round(mult * fl / (st["median_ms"] * 1e-3) / 1e12, 1)
                    res[f"{kind}_{label}"] = st
                res[f"{kind}_speedup"] = round(res[f"{kind}_mma_sync"]["median_ms"] / res[f"{kind}_wgmma"]["median_ms"], 2)
            report["attention"][f"{name}_B{B}"] = res
            print(json.dumps({f"{name}_B{B}": res}), flush=True)
            del qkv, do, outs, o, lse
    os.environ.pop("E4T_ATTN_WGMMA", None)
    del flush
    torch.cuda.empty_cache()


def build():
    from e4t.encoder import E4TEncoder
    from e4t.models.modeling_clip import CLIPTextConfig, CLIPTextModel
    from e4t.models.unet_2d_condition import UNet2DConditionModel
    from oracle import e4t_oracle as O
    from oracle import sd2_oracle as S
    torch.manual_seed(0)
    with torch.device("cuda"):
        unet = UNet2DConditionModel(**O.ref_unet_kwargs(S.SD2_UNET))
        enc = E4TEncoder(word_embedding_dim=1024, arch="ViT-H-14", freeze_clip_vision=True)
        t = S.CLIP_TEXT_SD2
        text = CLIPTextModel(CLIPTextConfig(vocab_size=t["vocab"], hidden_size=t["width"], intermediate_size=t["mlp"],
                                            num_hidden_layers=t["layers"], num_attention_heads=t["heads"],
                                            hidden_act=t["act"]))
    text.to(torch.bfloat16)
    return unet, enc, text


def batch(B, seed):
    from oracle import e4t_oracle as O
    from oracle import sd2_oracle as S
    b = O.synth_batch(B, seed, latent_hw=96, image_hw=768)
    b["input_ids"], idxs = S.synth_input_ids([i % 10 for i in range(B)], pad_id=0)
    b["placeholder_idxs"] = torch.tensor(idxs)
    return {k: v.cuda() for k, v in b.items()}


def steps(args, report):
    from e4t_b200.engine import PretrainStep, TuningStep
    for kind in ("pretrain", "tuning"):
        B_fit = None
        for sw in ("1", "0"):
            os.environ["E4T_ATTN_WGMMA"] = sw
            for B in ((16, 8, 4, 2, 1) if B_fit is None else (B_fit,)):
                step = None
                try:
                    gc.collect()
                    torch.cuda.empty_cache()
                    torch.cuda.reset_peak_memory_stats()
                    unet, enc, text = build()
                    ctor = TuningStep if kind == "tuning" else PretrainStep
                    step = ctor(unet, enc, text, 49408, class_token_id=320, prediction_type="v_prediction", pad_id=0)
                    b0 = batch(B, 1)
                    step.enable_cuda_graph(b0, warmup=2)
                    bs = [batch(B, 2 + i) for i in range(2)]
                    for i in range(2):
                        step(bs[i % 2])
                    torch.cuda.synchronize()
                    ts, losses = [], []
                    for i in range(args.steps):
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        out = step(bs[i % 2])
                        e1.record()
                        e1.synchronize()
                        ts.append(e0.elapsed_time(e1))
                        losses.append(out["loss"].item())
                    st = stats(ts)
                    st.update(B=B, images_per_s=round(B / (st["median_ms"] * 1e-3), 2),
                              peak_mem_gib=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
                              losses=[round(v, 5) for v in losses])
                    B_fit = B
                    label = "wgmma" if sw == "1" else "mma_sync"
                    report["steps"][f"{kind}_768_{label}"] = st
                    print(json.dumps({f"{kind}_768_{label}": st}), flush=True)
                    break
                except torch.OutOfMemoryError:
                    report["steps"].setdefault(f"{kind}_768_oom", []).append(B)
                    print(f"{kind} B={B}: out of memory", flush=True)
                finally:
                    step = unet = enc = text = None
                    gc.collect()
                    torch.cuda.empty_cache()
        a, b = report["steps"].get(f"{kind}_768_mma_sync"), report["steps"].get(f"{kind}_768_wgmma")
        if a and b:
            report["steps"][f"{kind}_768_speedup"] = round(a["median_ms"] / b["median_ms"], 3)
    os.environ.pop("E4T_ATTN_WGMMA", None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=12)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON report to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("sd2_ab.py needs a GPU")
    t0 = time.time()
    report = {"card_before": card(), "attention": {}, "steps": {}}
    attention(args, report)
    steps(args, report)
    report["card_after"] = card()
    report["wall_s"] = round(time.time() - t0, 1)
    text = json.dumps(report, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)
    bad = [(n, k, r) for n, s in report["attention"].items() for k, r in s["wgmma_vs_mma_sync_rel"].items()
           if not r < 2e-3]
    if bad:
        sys.exit(f"paths disagree: {bad}")


if __name__ == "__main__":
    main()
