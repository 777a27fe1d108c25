"""A/B timing of the optimiser: fp32 AdamW (28 B per parameter per step) against the block-wise 8-bit AdamW (16 B),
--use_8bit_adam of pretrain_e4t.py / tuning_e4t.py.

    python tools/optimizer_ab.py [--iters 20] [--batch 16] [--steps 5] [--warmup 2] [--skip-step]

1. The optimiser launch alone over an arena of the pre-training (374.6 M), domain-tuning (1234.1 M) and
   tuning + text encoder (1357.2 M) sizes: CUDA events around `iters` launches after two warm-up launches, ms per launch
   and the bytes the algorithm moves over that time as GB/s and as a share of the H100 SXM's 3.35 TB/s.
2. The graphed TuningStep at B = 16 (bench.py's models and batches) with use_8bit_adam off and on: median ms per
   replayed step (host clock around work that ends in a device synchronise) and peak allocated GiB.
The card, its power limit and SM clocks are read before and after."""
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

HBM = 3.35e12
SIZES = {"pretrain": 374.6e6, "tuning": 1234.1e6, "tuning+text": 1357.2e6}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks_event_reasons.active"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def time_launch(fn, iters):
    for _ in range(2):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def optimizer_launches(iters):
    from e4t_b200 import ops, optim
    out = []
    for name, size in SIZES.items():
        n = int(round(size / 256)) * 256
        sd = torch.zeros(1, device="cuda", dtype=torch.int32)
        lr_dev = torch.zeros(1, device="cuda")
        p = torch.randn(n, device="cuda") * 0.02
        g = torch.randn(n, device="cuda") * 1e-3
        m, v = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
        ms32 = time_launch(lambda: ops.adamw_step_dev(p, g, m, v, 1e-5, 0.9, 0.999, 1e-8, 1e-2, sd), iters)
        del m, v
        torch.cuda.empty_cache()
        mc, vc = torch.zeros(n, device="cuda", dtype=torch.uint8), torch.zeros(n, device="cuda", dtype=torch.uint8)
        ma, va = torch.zeros(n // 256, device="cuda"), torch.zeros(n // 256, device="cuda")
        qm, qv = optim.dynamic_map(True).cuda(), optim.dynamic_map(False).cuda()
        sched = (0, 0, 0, 0.0, optim.POWER, optim.LR_END)
        ms8 = time_launch(lambda: ops.adamw8bit_step_sched(p, g, mc, vc, ma, va, qm, qv, 1e-5, 0.9, 0.999, 1e-8, 1e-2,
                                                            sd, lr_dev, sched), iters)
        b32, b8 = 28.0 * n, 16.0 * n + 16.0 * (n // 256)
        res = dict(arena=name, params_M=n / 1e6, fp32_ms=ms32, fp32_GBps=b32 / ms32 / 1e6, fp32_hbm=b32 / (ms32 * 1e-3) / HBM,
                   int8_ms=ms8, int8_GBps=b8 / ms8 / 1e6, int8_hbm=b8 / (ms8 * 1e-3) / HBM,
                   floor_fp32_ms=b32 / HBM * 1e3, floor_int8_ms=b8 / HBM * 1e3,
                   moments_saved_GiB=(8.0 * n - 2.0 * n - 8.0 * (n // 256)) / 2 ** 30)
        print(json.dumps(res), flush=True)
        out.append(res)
        del p, g, mc, vc, ma, va
        gc.collect()
        torch.cuda.empty_cache()
    return out


def graphed_tuning_step(use_8bit, B, steps, warmup):
    import bench
    from e4t_b200.engine import TuningStep
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    unet, enc, text = bench.build_models("cuda")
    batches = [bench.to_device(bench.host_batch(B, seed=s, pinned=False), "cuda") for s in range(2)]
    step = TuningStep(unet, enc, text, 49408, class_token_id=320, use_8bit_adam=use_8bit)
    step.enable_cuda_graph(batches[0], warmup=warmup)
    ts = []
    for i in range(warmup + steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = step(batches[i % 2])
        torch.cuda.synchronize()
        if i >= warmup:
            ts.append((time.perf_counter() - t0) * 1e3)
        assert torch.isfinite(out["loss"]).item()
    res = dict(use_8bit_adam=use_8bit, arena_M=step.opt.numel / 1e6, graph_ms=[statistics.median(ts), min(ts), max(ts)],
               peak_gib=torch.cuda.max_memory_allocated() / 2 ** 30, loss=out["loss"].item())
    step.release_cuda_graph()
    del step, unet, enc, text, batches, out
    gc.collect()
    torch.cuda.empty_cache()
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--skip-step", action="store_true", help="time the optimiser launches only")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("optimizer_ab.py measures on a CUDA device; none found")
    print("card before:", card())
    launches = optimizer_launches(a.iters)
    steps = [] if a.skip_step else [graphed_tuning_step(u, a.batch, a.steps, a.warmup) for u in (False, True)]
    print("card after:", card())
    for r in launches:
        print(f"{r['arena']:>12} {r['params_M']:7.1f} M: fp32 {r['fp32_ms']:6.2f} ms ({r['fp32_GBps']:5.0f} GB/s, "
              f"{100 * r['fp32_hbm']:3.0f} % of 3.35 TB/s)   8-bit {r['int8_ms']:6.2f} ms ({r['int8_GBps']:5.0f} GB/s, "
              f"{100 * r['int8_hbm']:3.0f} %)   moments -{r['moments_saved_GiB']:.2f} GiB")
    for u in (False, True):
        rs = [r for r in steps if r["use_8bit_adam"] == u]
        if rs:
            print(f"graphed TuningStep B={a.batch} use_8bit_adam={u}: {[round(r['graph_ms'][0], 1) for r in rs]} ms/step, "
                  f"peak {max(r['peak_gib'] for r in rs):.1f} GiB")


if __name__ == "__main__":
    main()
