"""A/B timing of the domain-tuning step (TuningStep == tuning_e4t.py:270-338) with and without --train_text_encoder,
at the real size: SD-v1.4 UNet, E4T encoder on ViT-H/14, CLIP-L text tower (bench.py's models, synthetic weights and
bench.py's batches), B = 16 by default.

    python tools/tuning_text_ab.py [--batch 16] [--steps 5] [--warmup 2] [--rounds 2]

Each round builds the frozen-text and the text-training step in turn (both do not fit on one card together at B = 16),
and times each one eagerly and as one replayed CUDA graph, with a host clock around work that ends in a device
synchronise: median ms/step with min - max over the timed steps.  It also reports the e4t kernel launches of one eager
step and the peak allocated memory of the variant.  The card, its power limit and SM clocks are read before and after."""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "e4t-diffusion_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks_event_reasons.active"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def timed(fn, batches, steps):
    ts = []
    for i in range(steps):
        b = batches[i % len(batches)]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn(b)
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
        assert torch.isfinite(out["loss"]).item()
    return ts


def run_variant(train_text, B, steps, warmup):
    import bench
    from e4t_b200 import _lib
    from e4t_b200.engine import TuningStep
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    unet, enc, text = bench.build_models("cuda")
    if train_text:
        text.float()          # the text tower trains on fp32 masters (tuning_e4t.py --train_text_encoder)
    batches = [bench.to_device(bench.host_batch(B, seed=s, pinned=False), "cuda") for s in range(2)]
    step = TuningStep(unet, enc, text, 49408, class_token_id=320, train_text_encoder=train_text)
    res = dict(train_text_encoder=train_text, arena_params=step.opt.numel)
    # capture first: eager steps on the default stream before the capture would leave autograd nodes bound to it
    step.enable_cuda_graph(batches[0], warmup=warmup)
    timed(step, batches, warmup)
    ts = timed(step, batches, steps)
    res["graph_ms"] = [statistics.median(ts), min(ts), max(ts)]
    eager = step._eager_step
    timed(eager, batches, warmup)
    _lib.reset_launch_count()
    eager(batches[0])
    torch.cuda.synchronize()
    res["launches_per_step"] = _lib.launch_count()
    ts = timed(eager, batches, steps)
    res["eager_ms"] = [statistics.median(ts), min(ts), max(ts)]
    res["peak_gib"] = torch.cuda.max_memory_allocated() / 2 ** 30
    step.release_cuda_graph()
    del step, unet, enc, text, batches
    gc.collect()
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tuning_text_ab.py measures on a CUDA device; none found")
    print("card before:", card())
    results = []
    for r in range(a.rounds):
        for train_text in (False, True):
            res = run_variant(train_text, a.batch, a.steps, a.warmup)
            res["round"] = r
            results.append(res)
            print(json.dumps(res), flush=True)
    print("card after:", card())
    for tt in (False, True):
        rs = [r for r in results if r["train_text_encoder"] == tt]
        print(f"train_text_encoder={tt}: eager {[round(r['eager_ms'][0], 1) for r in rs]} ms/step, graphed "
              f"{[round(r['graph_ms'][0], 1) for r in rs]} ms/step, {rs[0]['launches_per_step']} launches/step, "
              f"peak {max(r['peak_gib'] for r in rs):.1f} GiB, arena {rs[0]['arena_params'] / 1e6:.1f} M params")


if __name__ == "__main__":
    main()
