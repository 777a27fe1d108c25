"""Token merging on the H100: the same graphed workloads without a patch (ratio 0) and with tomesd's defaults
(ratio 0.5, max_downsample 1: the level-0 self-attention runs on half the tokens), alternating in one process.

    python tools/tome_ab.py [--rounds 2] [--steps 6] [--out report.json]

1. Graphed steps on synthetic weights, B = 16 (or the largest of 16, 8, 4 that fits): SD 1.4 PretrainStep and
   TuningStep at 512², SD 2.x PretrainStep (v-prediction) at 768².  A captured graph keeps the patch it was captured
   with, so each round captures once per ratio, times --steps replays with CUDA events and releases the graph; the
   ratios alternate over --rounds rounds.  Peak memory per ratio.
2. One graphed sampling step at 512², B = 1, guidance 7.5 (SD 1.4 pipeline, DDIM): per-step time from CUDA events
   recorded in the step callback.
3. The ToMe kernels at SD 1.4 level 0, 512², B = 16 (4096 tokens x 320): match (partition, normalise, wgmma),
   select, merge (gather-reduce) and unmerge (gather-expand), CUDA events over many launches.
Card name, power limit and SM clock are read in the same run.  Needs a GPU; fails without one.
"""
import argparse
import gc
import json
import os
import sys
import time
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "e4t-diffusion_b200"), os.path.join(ROOT, "tools")]

from attn_ab import card, stats  # noqa: E402

RATIOS = (0.0, 0.5)


def events_ms(fn, n):
    ts = []
    for _ in range(n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return ts


def build(kind):
    import bench
    if kind != "sd2":
        return bench.build_models("cuda")
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


def batch(kind, B, seed):
    from oracle import e4t_oracle as O
    if kind == "sd2":
        from oracle import sd2_oracle as S
        b = O.synth_batch(B, seed, latent_hw=96, image_hw=768)
        b["input_ids"], idxs = S.synth_input_ids([i % 10 for i in range(B)], pad_id=0)
    else:
        b = O.synth_batch(B, seed, latent_hw=64, image_hw=512)
        idxs = [row.index(O.PLACEHOLDER_ID) for row in b["input_ids"].tolist()]
    b["placeholder_idxs"] = torch.tensor(idxs)
    return {k: v.cuda() for k, v in b.items()}


def steps(args, report):
    from e4t_b200 import tome
    from e4t_b200.engine import PretrainStep, TuningStep
    for name, kind, ctor in (("sd14_pretrain_512", "sd1", PretrainStep), ("sd14_tuning_512", "sd1", TuningStep),
                             ("sd2_pretrain_768", "sd2", PretrainStep)):
        kw = dict(prediction_type="v_prediction", pad_id=0) if kind == "sd2" else {}
        res = {r: dict(ms=[], peak_gib=0.0, losses=[]) for r in RATIOS}
        B_fit = None
        for rnd in range(args.rounds):
            for ratio in RATIOS:
                for B in ((16, 8, 4) if B_fit is None else (B_fit,)):
                    step = unet = enc = text = None
                    try:
                        gc.collect()
                        torch.cuda.empty_cache()
                        torch.cuda.reset_peak_memory_stats()
                        unet, enc, text = build(kind)
                        tome.apply_patch(unet, ratio=ratio)
                        step = ctor(unet, enc, text, 49408, class_token_id=320, **kw)
                        step.enable_cuda_graph(batch(kind, B, 1), warmup=2)
                        bs = [batch(kind, B, 2 + i) for i in range(2)]
                        for i in range(2):
                            step(bs[i % 2])
                        out = {}

                        def one(i=[0]):
                            out.update(step(bs[i[0] % 2]))
                            i[0] += 1

                        res[ratio]["ms"] += events_ms(one, args.steps)
                        res[ratio]["losses"].append(round(out["loss"].item(), 5))
                        res[ratio]["peak_gib"] = max(res[ratio]["peak_gib"],
                                                     round(torch.cuda.max_memory_allocated() / 2 ** 30, 2))
                        B_fit = B
                        break
                    except torch.OutOfMemoryError:
                        print(f"{name} ratio {ratio} B={B}: out of memory", flush=True)
                    finally:
                        if step is not None:
                            step.release_cuda_graph()
                        step = unet = enc = text = None
                        gc.collect()
                        torch.cuda.empty_cache()
        entry = {"B": B_fit}
        for ratio in RATIOS:
            st = stats(res[ratio]["ms"]) if res[ratio]["ms"] else {}
            st.update(peak_mem_gib=res[ratio]["peak_gib"], losses=res[ratio]["losses"])
            entry[f"ratio_{ratio}"] = st
        if res[0.0]["ms"] and res[0.5]["ms"]:
            entry["speedup"] = round(entry["ratio_0.0"]["median_ms"] / entry["ratio_0.5"]["median_ms"], 3)
            entry["saved_ms"] = round(entry["ratio_0.0"]["median_ms"] - entry["ratio_0.5"]["median_ms"], 2)
        report["steps"][name] = entry
        print(json.dumps({name: entry}), flush=True)


def sampling(args, report):
    import bench
    from sample_ab import WordTokenizer
    from e4t.pipeline_stable_diffusion_e4t import SCHEDULER_MAPPING, StableDiffusionE4TPipeline
    from e4t_b200 import tome
    unet, enc, text = bench.build_models("cuda")
    conf = types.SimpleNamespace(placeholder_token="*s", domain_class_token="a", domain_embed_scale=1.0)
    pipe = StableDiffusionE4TPipeline(None, text, WordTokenizer(), unet, enc, SCHEDULER_MAPPING["ddim"](),
                                      e4t_config=conf, already_added_placeholder_token=True).enable_cuda_graph()
    g = torch.Generator().manual_seed(0)
    image = torch.rand(1, 3, 512, 512, generator=g) * 2 - 1
    latents = torch.randn(1, 4, 64, 64, generator=g)
    res = {r: [] for r in RATIOS}
    for rnd in range(args.rounds + 1):
        for ratio in RATIOS:
            tome.apply_patch(pipe, ratio=ratio)
            ev = []

            def cb(i, t, x):
                e = torch.cuda.Event(enable_timing=True)
                e.record()
                ev.append(e)

            pipe(["a photo of *s"], num_inference_steps=args.sample_steps, guidance_scale=7.5, latents=latents.clone(),
                 image=image, output_type="latent", callback=cb)
            torch.cuda.synchronize()
            if rnd > 0:        # round 0 captures both graphs
                res[ratio] += [a.elapsed_time(b) for a, b in zip(ev[:-1], ev[1:])]
    entry = {f"ratio_{r}": stats(res[r]) for r in RATIOS}
    entry["speedup"] = round(entry["ratio_0.0"]["median_ms"] / entry["ratio_0.5"]["median_ms"], 3)
    report["sampling_512_B1_cfg"] = entry
    print(json.dumps({"sampling_512_B1_cfg": entry}), flush=True)
    del pipe, unet, enc, text
    gc.collect()
    torch.cuda.empty_cache()


def kernels(args, report):
    from e4t_b200 import ops
    B, h, w, C = 16, 64, 64, 320
    N, r = h * w, 2048
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(B, N, C, device="cuda", generator=g).to(torch.bfloat16)
    pattern = torch.randint(0, 4, (h // 2, w // 2), device="cuda", generator=g, dtype=torch.int32)
    m = ops.tome_match(x, pattern, h, w, 2, 2)
    plan = ops.tome_select(m, r)
    y = ops.tome_gather_reduce(x, plan, True)
    calls = {"match": lambda: ops.tome_match(x, pattern, h, w, 2, 2), "select": lambda: ops.tome_select(m, r),
             "merge_gather_reduce": lambda: ops.tome_gather_reduce(x, plan, True),
             "unmerge_gather_expand": lambda: ops.tome_gather_expand(y, plan, False, residual=x)}
    out = {"shape": dict(B=B, N=N, C=C, r=r)}
    for name, fn in calls.items():
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        out[name] = stats(events_ms(fn, args.kernel_iters))
    report["kernels_sd14_level0_B16"] = out
    print(json.dumps({"kernels_sd14_level0_B16": out}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--sample-steps", type=int, default=12)
    ap.add_argument("--kernel-iters", type=int, default=50)
    ap.add_argument("--out", default=None, help="also write the JSON report to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("tome_ab.py needs a GPU")
    t0 = time.time()
    report = {"card_before": card(), "steps": {}}
    kernels(args, report)
    sampling(args, report)
    steps(args, report)
    report["card_after"] = card()
    report["wall_s"] = round(time.time() - t0, 1)
    text = json.dumps(report, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
