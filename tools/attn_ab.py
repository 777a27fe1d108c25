"""A/B timing of the self-attention core: warpgroup (wgmma) kernels against the mma.sync kernels.

    python tools/attn_ab.py [--batch 16] [--iters 24]

For the level-0 (N = M = 4096, 8 heads x 40) and level-1 (N = M = 1024, 8 heads x 80) self-attention shapes of the
SD-v1.4 UNet it times forward and single-pass backward with E4T_ATTN_WGMMA=0 and =1, alternating in one process (the
library reads the switch on every call).  CUDA events, L2 flushed before every launch, median and min-max over
--iters launches.  The backward figure includes its delta pre-pass, the dQ scratch memset and the bf16 conversion.
O / LSE / dQ / dK / dV of the two paths are compared on the same seeded inputs.  Card name, power limit and SM clock
are read in the same run and printed with the numbers.  Shapes the warpgroup kernels do not take run the same kernel
under both settings, which shows the noise floor.  Needs a GPU; fails without one.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "e4t-diffusion_b200"))

SHAPES = {"L0_self": (4096, 8, 40), "L1_self": (1024, 8, 80)}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--id={torch.cuda.current_device()}", f"--query-gpu={q}",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=20).stdout.strip()
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except (OSError, subprocess.SubprocessError) as e:
        return {"name": torch.cuda.get_device_name(), "error": repr(e)}


def rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


def stats(ts):
    ts = sorted(ts)
    return {"median_ms": round(ts[len(ts) // 2], 4), "min_ms": round(ts[0], 4), "max_ms": round(ts[-1], 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--iters", type=int, default=24)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("attn_ab.py needs a GPU")
    from e4t_b200 import ops
    dev = torch.device("cuda")
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)   # > 50 MB L2
    report = {"card_before": card(), "batch": args.batch, "iters": args.iters, "shapes": {}}

    def timed(fn):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1)

    for name, (N, H, dh) in SHAPES.items():
        C = H * dh
        g = torch.Generator(device=dev).manual_seed(N + dh)
        qkv = (torch.randn(args.batch, N, 3 * C, device=dev, generator=g) * 0.5).to(torch.bfloat16)
        q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
        do = (torch.randn(args.batch, N, C, device=dev, generator=g) * 0.5).to(torch.bfloat16)
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
        fl = 4.0 * N * N * C * args.batch
        res = {"N": N, "heads": H, "dh": dh, "new_vs_old_rel": agree}
        for kind, mult in (("fwd", 1.0), ("bwd", 2.5)):
            for sw, label in (("0", "mma_sync"), ("1", "default")):
                st = stats(times[kind][sw])
                st["tflops_at_median"] = round(mult * fl / (st["median_ms"] * 1e-3) / 1e12, 1)
                res[f"{kind}_{label}"] = st
            a, b = res[f"{kind}_mma_sync"], res[f"{kind}_default"]
            res[f"{kind}_ranges_overlap"] = not (b["max_ms"] < a["min_ms"] or a["max_ms"] < b["min_ms"])
        report["shapes"][name] = res
    os.environ.pop("E4T_ATTN_WGMMA", None)
    report["card_after"] = card()
    print(json.dumps(report, indent=1))
    bad = [(n, k, r) for n, s in report["shapes"].items() for k, r in s["new_vs_old_rel"].items() if not r < 2e-3]
    if bad:
        sys.exit(f"paths disagree: {bad}")


if __name__ == "__main__":
    main()
