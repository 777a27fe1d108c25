"""Per-call inventory and A/B timing of the GEMM / implicit-convolution engine over one pre-training step.

    python tools/gemm_ab.py [--lib PATH ...] [--batch 16] [--iters 15] [--without-residual] [--out FILE]
    python tools/gemm_ab.py --tile-cost [--tile-m 16384] [--lib PATH] [--iters 7] [--out FILE]

Runs one eager pre-training step (bench.py's models and inputs, after one warm-up step) with ops.gemm, ops.conv3x3,
ops.conv3x3_s2 and ops.conv3x3_wgrad wrapped, and records every call: shapes, operand majors, output dtype and mode,
bias / rowgroup / residual, alpha, splits and the number of calls per step.  Each distinct call is then replayed alone
on fresh seeded tensors of the same shapes, strides and alignment (CUDA events, L2 flushed before every launch, median
over --iters launches) and weighted by its call count.

Every --lib names a libe4t_b200.so; the first one runs the step.  With several, the libraries are loaded side by side
and timed alternately, launch by launch, and their outputs are compared on the same inputs.  Card name, power limit and
SM clock are read in the same run.  Needs a GPU; fails without one.

--without-residual replays every call that adds a residual a second time with residual=None, alternating with the
original call on the same inputs, and reports per call and call-weighted per step what adding the residual costs.

--tile-cost [--tile-m 16384] skips the step and times the engine alone (L2 flushed, median of --iters launches) at
M = --tile-m for N in 320 ... 5120, every tile width BN the tile-width choice can take (forced with force_bn), K from 64
to 2880, and bf16, bf16 + residual and fp32 outputs.  Per BN and output mode it fits time = rounds * (a + b * kchunks)
by least squares (rounds = persistent-grid rounds, ceil(tiles / SMs); kchunks = K / 64) and reports a, the fixed cost
per tile, and b, the cost per 64-deep k-chunk, in microseconds, with the worst relative residual of the fit.  Every
sample goes into the --out report.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
from collections import OrderedDict

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "e4t-diffusion_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

WRAPPED = ("gemm", "conv3x3", "conv3x3_s2", "conv3x3_wgrad")


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--id={torch.cuda.current_device()}", f"--query-gpu={q}",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=20).stdout.strip()
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except (OSError, subprocess.SubprocessError) as e:
        return {"name": torch.cuda.get_device_name(), "error": repr(e)}


def open_lib(path):
    h = ctypes.CDLL(os.path.abspath(path))
    h.e4t_last_error.restype = ctypes.c_char_p
    h.e4t_version.restype = ctypes.c_int
    h.e4t_launch_count.restype = ctypes.c_ulonglong
    h.e4t_reset_launch_count.restype = None
    return h


def spec(v):
    """Hashable description of one argument; tensors by shape, stride, dtype and 16-byte misalignment of the base."""
    if isinstance(v, torch.Tensor):
        return ("T", tuple(v.shape), tuple(v.stride()), str(v.dtype).replace("torch.", ""),
                (v.data_ptr() % 16) // v.element_size())
    return ("V", v)


def make(sp, g):
    """A fresh seeded tensor laid out as described by spec()."""
    _, shape, stride, dt, mis = sp
    dtype = getattr(torch, dt)
    need = 1 + sum((s - 1) * st for s, st in zip(shape, stride)) if shape else 1
    buf = torch.randn(need + 16, device="cuda", generator=g).mul_(0.2).to(dtype)
    return buf.as_strided(shape, stride, mis)


def inventory(batch):
    import bench
    from e4t_b200 import ops
    from e4t_b200.engine import PretrainStep
    dev = torch.device("cuda")
    unet, enc, text = bench.build_models(dev)
    step = PretrainStep(unet, enc, text, placeholder_token_id=49408, class_token_id=320, lr=1.6e-5,
                        weight_dtype=torch.bfloat16)
    b = bench.to_device(bench.host_batch(batch, 42), dev)
    step(b)
    torch.cuda.synchronize()
    calls = OrderedDict()
    orig = {n: getattr(ops, n) for n in WRAPPED}

    def wrap(name):
        fn = orig[name]

        def w(*args, **kw):
            key = (name, tuple(spec(a) for a in args), tuple(sorted((k, spec(v)) for k, v in kw.items())))
            calls[key] = calls.get(key, 0) + 1
            return fn(*args, **kw)
        return w

    for n in WRAPPED:
        setattr(ops, n, wrap(n))
    try:
        step(b)
        torch.cuda.synchronize()
    finally:
        for n in WRAPPED:
            setattr(ops, n, orig[n])
    del step, unet, enc, text, b
    torch.cuda.empty_cache()
    return calls


def describe(key):
    name, args, kw = key
    ts = [a for a in args if a[0] == "T"]
    kwd = dict(kw)
    d = {"op": name}
    if name == "gemm":
        A, B = ts[0], ts[1]
        a_mn = kwd.get("a_mn", ("V", False))[1]
        b_mn = kwd.get("b_mn", ("V", False))[1]
        M = A[1][-1] if a_mn else A[1][-2]
        K = A[1][-2] if a_mn else A[1][-1]
        N = B[1][-1] if b_mn else B[1][-2]
        bt = max(A[1][0] if len(A[1]) == 3 else 1, B[1][0] if len(B[1]) == 3 else 1)
        d.update(M=M, N=N, K=K, batch=bt, a_mn=bool(a_mn), b_mn=bool(b_mn))
        d["flops"] = 2.0 * M * N * K * bt
        acc = kwd.get("accumulate", ("V", False))[1]
        out = kwd.get("out")
        d["out"] = "fp32_atomic" if acc else (out[3] if out and out[0] == "T" else
                                              str(kwd.get("out_dtype", ("V", torch.bfloat16))[1]).replace("torch.", ""))
        if out and out[0] == "T" and out[4]:
            d["out_misaligned"] = True
        for k in ("bias", "rowgroup", "residual"):
            if kwd.get(k, ("V", None))[0] == "T":
                d[k] = True
        for k in ("alpha", "splits", "force_bn"):
            if k in kwd:
                d[k] = kwd[k][1]
    else:
        x, w = ts[0], ts[1]
        Bn, H, W, Cin = x[1]
        Cout = w[1][1] if name != "conv3x3_wgrad" else w[1][-1]
        s = 2 if name == "conv3x3_s2" else 1
        d.update(B=Bn, H=H, W=W, Cin=Cin, Cout=Cout)
        d["flops"] = 2.0 * Bn * (H // s) * (W // s) * 9 * Cin * Cout
        for k in ("bias", "rowgroup", "residual"):
            if kwd.get(k, ("V", None))[0] == "T":
                d[k] = True
    return d


def out_elems(row):
    """Elements of the call's output (and of its residual)."""
    if row["op"] == "gemm":
        return row["M"] * row["N"] * row["batch"]
    s = 2 if row["op"] == "conv3x3_s2" else 1
    return row["B"] * (row["H"] // s) * (row["W"] // s) * row["Cout"]


def replay_fn(key, g):
    """run(drop=()) replays the call on fresh seeded inputs, leaving out the keyword arguments named in drop."""
    from e4t_b200 import ops
    name, args, kw = key
    a = [make(s, g) if s[0] == "T" else s[1] for s in args]
    k = {n: (make(s, g) if s[0] == "T" else s[1]) for n, s in kw}
    out = k.get("out")
    fn = getattr(ops, name)

    def run(drop=()):
        if out is not None and k.get("accumulate"):
            out.zero_()
        r = fn(*a, **{n: v for n, v in k.items() if n not in drop})
        return out if r is None else r
    return run


def stats(ts):
    ts = sorted(ts)
    return {"median_ms": round(ts[len(ts) // 2], 4), "min_ms": round(ts[0], 4), "max_ms": round(ts[-1], 4)}


TILE_N = (320, 640, 960, 1280, 2560, 5120)
TILE_K = (64, 128, 320, 640, 1280, 2880)
TILE_MODES = ("bf16", "bf16_residual", "fp32")


def tile_cost(args, handle):
    """Fixed and per-chunk cost of an engine tile, fitted from a K sweep at fixed M x N (see the module docstring)."""
    import numpy as np
    from e4t_b200 import _lib, ops
    _lib._lib = handle
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    M = args.tile_m
    g = torch.Generator(device="cuda").manual_seed(7)
    A = torch.randn(M, max(TILE_K), device="cuda", generator=g).mul_(0.2).bfloat16()
    Bw = torch.randn(max(TILE_N), max(TILE_K), device="cuda", generator=g).mul_(0.2).bfloat16()
    R = torch.randn(M, max(TILE_N), device="cuda", generator=g).mul_(0.2).bfloat16()
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    samples = {}
    for N in TILE_N:
        for bn in range(64, 257, 32):
            if bn > 2 * N:
                continue
            rounds = -(-(-(-M // 128) * -(-N // bn)) // sms)
            for K in TILE_K:
                a, b = A[:, :K].contiguous(), Bw[:N, :K].contiguous()
                for mode in TILE_MODES:
                    kw = dict(force_bn=bn, out_dtype=torch.float32 if mode == "fp32" else torch.bfloat16,
                              residual=R[:, :N] if mode == "bf16_residual" else None)
                    ts = []
                    for it in range(args.iters + 1):             # the first launch warms up
                        flush.zero_()
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        ops.gemm(a, b, **kw)
                        e1.record()
                        e1.synchronize()
                        if it:
                            ts.append(e0.elapsed_time(e1))
                    ts.sort()
                    samples.setdefault((bn, mode), []).append(
                        dict(N=N, K=K, rounds=rounds, kchunks=K // 64, ms=ts[len(ts) // 2]))
    fits = []
    for (bn, mode), rows in sorted(samples.items()):
        X = np.array([[r["rounds"], r["rounds"] * r["kchunks"]] for r in rows], dtype=np.float64)
        y = np.array([r["ms"] * 1e3 for r in rows])
        (ca, cb), *_ = np.linalg.lstsq(X, y, rcond=None)
        worst = float(np.max(np.abs(X @ np.array([ca, cb]) - y) / y))
        fits.append(dict(BN=bn, mode=mode, a_us=round(float(ca), 3), b_us=round(float(cb), 4), points=len(rows),
                         worst_rel_resid=round(worst, 3)))
    print(f"{'BN':>4s} {'mode':14s} {'a us':>8s} {'b us':>8s} {'pts':>4s} {'worst':>6s}")
    for f in fits:
        print(f"{f['BN']:4d} {f['mode']:14s} {f['a_us']:8.3f} {f['b_us']:8.4f} {f['points']:4d} "
              f"{f['worst_rel_resid']:6.3f}")
    return {"tile_m": M, "sms": sms, "fits": fits, "samples": {f"{k[0]}/{k[1]}": v for k, v in samples.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tile-cost", action="store_true", help="fit the per-tile and per-chunk cost instead of the step")
    ap.add_argument("--tile-m", type=int, default=16384)
    ap.add_argument("--lib", action="append", default=[], help="libe4t_b200.so to time (repeat to A/B; first runs the step)")
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--iters", type=int, default=15)
    ap.add_argument("--without-residual", action="store_true",
                    help="also time every residual call with residual=None and report what the residual costs")
    ap.add_argument("--out", default=None, help="also write the JSON report here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gemm_ab.py needs a GPU")
    from e4t_b200 import _lib
    libs = args.lib or [_lib.lib_path()]
    _lib._LIB_PATH = os.path.abspath(libs[0])
    handles = [open_lib(p) for p in libs]
    _lib._lib = handles[0]
    report = {"card_before": card(), "batch": args.batch, "iters": args.iters, "libs": libs}
    if args.tile_cost:
        report["tile_cost"] = tile_cost(args, handles[0])
        report["card_after"] = card()
        print(json.dumps({"card_before": report["card_before"], "card_after": report["card_after"]}))
        if args.out:
            os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
            with open(args.out, "w") as f:
                json.dump(report, f, indent=1)
        return
    calls = inventory(args.batch)
    report["distinct_calls"] = len(calls)
    report["calls_per_step"] = sum(calls.values())

    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")

    def timed(fn):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1)

    rows = []
    for i, (key, count) in enumerate(calls.items()):
        g = torch.Generator(device="cuda").manual_seed(1000 + i)
        run = replay_fn(key, g)
        row = describe(key)
        row["count"] = count
        nores = args.without_residual and row.get("residual", False)
        outs, times, times_nores = [], [[] for _ in handles], [[] for _ in handles]
        for h in handles:
            _lib._lib = h
            outs.append(run().clone())
        for it in range(args.iters + 1):             # the first round warms up
            for li, h in enumerate(handles):
                _lib._lib = h
                t = timed(run)
                if it:
                    times[li].append(t)
                if nores:
                    t = timed(lambda: run(drop=("residual",)))
                    if it:
                        times_nores[li].append(t)
        for li in range(len(handles)):
            row[f"lib{li}"] = stats(times[li])
            if nores:
                row[f"lib{li}_without_residual"] = stats(times_nores[li])
                row[f"lib{li}_residual_cost_ms"] = round(row[f"lib{li}"]["median_ms"]
                                                         - row[f"lib{li}_without_residual"]["median_ms"], 4)
        if len(handles) > 1:
            a, b = outs[0].float(), outs[1].float()
            row["max_abs_diff_vs_lib0"] = (a - b).abs().max().item()
            row["rel_diff_vs_lib0"] = ((a - b).norm() / (a.norm() + 1e-12)).item()
            row["bit_identical"] = bool(torch.equal(outs[0], outs[1]))
            r0, r1 = row["lib0"], row["lib1"]
            row["ranges_overlap"] = not (r1["max_ms"] < r0["min_ms"] or r0["max_ms"] < r1["min_ms"])
        rows.append(row)
        del run, outs
    _lib._lib = handles[0]
    report["calls"] = rows
    tot = {}
    for li in range(len(handles)):
        tot[f"lib{li}_ms_per_step"] = round(sum(r["count"] * r[f"lib{li}"]["median_ms"] for r in rows), 3)
        k640 = [r for r in rows if r["op"] == "gemm" and r["K"] <= 640]
        tot[f"lib{li}_gemm_K_le_640_ms_per_step"] = round(sum(r["count"] * r[f"lib{li}"]["median_ms"] for r in k640), 3)
        if args.without_residual:
            res = [r for r in rows if r.get("residual")]
            tot[f"lib{li}_residual_calls_ms_per_step"] = round(
                sum(r["count"] * r[f"lib{li}"]["median_ms"] for r in res), 3)
            tot[f"lib{li}_residual_cost_ms_per_step"] = round(
                sum(r["count"] * r[f"lib{li}_residual_cost_ms"] for r in res), 3)
    if args.without_residual:
        res = [r for r in rows if r.get("residual")]
        tot["residual_calls_per_step"] = sum(r["count"] for r in res)
        tot["residual_elements_per_step"] = sum(r["count"] * out_elems(r) for r in res)
    tot["flops_per_step"] = sum(r["count"] * r["flops"] for r in rows)
    report["totals"] = tot
    report["card_after"] = card()
    txt = json.dumps(report, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(txt)
    # table: one line per distinct call, heaviest first
    print(f"{'op':14s} {'shape':44s} {'epi':22s} {'n':>3s} " + " ".join(f"{'lib%d ms' % i:>9s}" for i in range(len(handles)))
          + ("".join(f" {'lib%d res' % i:>9s}" for i in range(len(handles))) if args.without_residual else ""))
    for r in sorted(rows, key=lambda r: -r["count"] * r["lib0"]["median_ms"]):
        shp = (f"{r['M']}x{r['N']}x{r['K']} b{r['batch']} {'T' if r['a_mn'] else 'N'}{'T' if r['b_mn'] else 'N'}"
               if r["op"] == "gemm" else f"{r['B']}x{r['H']}x{r['W']} {r['Cin']}->{r['Cout']}")
        epi = ",".join(k for k in ("bias", "rowgroup", "residual", "out_misaligned") if r.get(k))
        epi = (r.get("out", "") + (" " + epi if epi else ""))[:22]
        print(f"{r['op']:14s} {shp:44s} {epi:22s} {r['count']:3d} "
              + " ".join(f"{r['lib%d' % i]['median_ms']:9.4f}" for i in range(len(handles)))
              + ("" if len(handles) == 1 else f"  {'' if r['ranges_overlap'] else '*'}"
                 f"{'=' if r['bit_identical'] else '%.1e' % r['rel_diff_vs_lib0']}"))
    print(json.dumps({"card": report["card_before"], "totals": tot}))
    bad = [r for r in rows if len(handles) > 1 and not r["rel_diff_vs_lib0"] < 1e-5]
    if bad:
        sys.exit(f"libraries disagree on {len(bad)} calls")


if __name__ == "__main__":
    main()
