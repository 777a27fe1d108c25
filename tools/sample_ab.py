"""Eager against CUDA-graph sampling: StableDiffusionE4TPipeline at SD v1.4 shapes (UNet, CLIP-L text tower) with the
E4T encoder on CLIP ViT-H/14, synthetic weights, 512² images, guidance 7.5, 50 steps, B = 1 and B = 4, for DDIM and
PLMS.  The eager loop and the graphed loop (`pipe.enable_cuda_graph()`) run alternately, one whole call each per
round, on the same prompt, image and starting latents.

Per-step time: CUDA events recorded from the step callback, consecutive events differenced (median (min-max) over every
step of every round).  Seconds per image: host clock around a whole call ending in a device synchronise, over B.  The
relative RMS difference of the graphed latents from the eager ones is printed per configuration.  The card, its power
limit and SM clock are read in the same run.

    python tools/sample_ab.py [--rounds 3] [--steps 50] [--batches 1,4] [--schedulers ddim,plms]"""
import argparse
import os
import subprocess
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "e4t-diffusion_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


class WordTokenizer:
    """Whitespace tokenizer over a few fixed CLIP word ids; `*s` is the placeholder (id 49408)."""
    model_max_length = 77
    WORDS = {"a": 320, "photo": 1125, "of": 539, "*s": 49408}

    def add_tokens(self, tok):
        return 0

    def __len__(self):
        return 49409

    def convert_tokens_to_ids(self, tok):
        return self.WORDS[tok]

    def __call__(self, text, padding=None, truncation=None, max_length=77, return_tensors=None, add_special_tokens=True):
        rows = []
        for s in [text] if isinstance(text, str) else text:
            ids = [self.WORDS[w] for w in s.split()]
            if add_special_tokens:
                ids = [49406] + ids + [49407] * (max_length - 1 - len(ids))
            rows.append(ids)
        return types.SimpleNamespace(input_ids=torch.tensor(rows, dtype=torch.int64))


def stats(ts):
    s = sorted(ts)
    return s[len(s) // 2], s[0], s[-1]


def run(pipe, graph, B, steps, latents, image):
    (pipe.enable_cuda_graph if graph else pipe.disable_cuda_graph)()
    events = []

    def cb(i, t, x):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        events.append(e)

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = pipe(["a photo of *s"] * B, num_inference_steps=steps, guidance_scale=7.5, latents=latents.clone(),
               image=image, output_type="latent", callback=cb).images
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    ms = [a.elapsed_time(b) for a, b in zip(events[:-1], events[1:])]
    return out, ms, wall


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--batches", default="1,4")
    ap.add_argument("--schedulers", default="ddim,plms")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "sample_ab.py measures on a CUDA device"
    print("card:", card())
    import bench
    from e4t.pipeline_stable_diffusion_e4t import SCHEDULER_MAPPING, StableDiffusionE4TPipeline
    unet, enc, text = bench.build_models("cuda")
    conf = types.SimpleNamespace(placeholder_token="*s", domain_class_token="a", domain_embed_scale=1.0)
    pipe = StableDiffusionE4TPipeline(None, text, WordTokenizer(), unet, enc, SCHEDULER_MAPPING["ddim"](),
                                      e4t_config=conf, already_added_placeholder_token=True)
    g = torch.Generator().manual_seed(0)
    image = torch.rand(1, 3, 512, 512, generator=g) * 2 - 1
    print(f"{'scheduler':>9} {'B':>2} | {'eager ms/step (min-max)':>26} | {'graph ms/step (min-max)':>26} | "
          f"{'eager s/img':>11} | {'graph s/img':>11} | graph vs eager rel RMS")
    for name in args.schedulers.split(","):
        pipe.scheduler = SCHEDULER_MAPPING[name]()
        for B in (int(b) for b in args.batches.split(",")):
            latents = torch.randn(B, 4, 64, 64, generator=g)
            run(pipe, True, B, 3, latents, image)        # capture + warm-up of both paths
            run(pipe, False, B, 3, latents, image)
            res = {False: ([], []), True: ([], [])}
            outs = {}
            for _ in range(args.rounds):
                for graph in (False, True):
                    out, ms, wall = run(pipe, graph, B, args.steps, latents, image)
                    res[graph][0].extend(ms)
                    res[graph][1].append(wall / B)
                    outs[graph] = out
            d = ((outs[True] - outs[False]).pow(2).mean().sqrt() / outs[False].pow(2).mean().sqrt()).item()
            (em, elo, ehi), (gm, glo, ghi) = stats(res[False][0]), stats(res[True][0])
            es, gs = stats(res[False][1])[0], stats(res[True][1])[0]
            print(f"{name:>9} {B:>2} | {em:8.2f} ({elo:7.2f}-{ehi:7.2f}) | {gm:8.2f} ({glo:7.2f}-{ghi:7.2f}) | "
                  f"{es:11.3f} | {gs:11.3f} | {d:.2e}", flush=True)
            pipe.disable_cuda_graph()
            torch.cuda.empty_cache()
    print("card:", card())


if __name__ == "__main__":
    main()
