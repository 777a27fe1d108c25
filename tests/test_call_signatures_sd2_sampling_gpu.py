"""Every distinct kernel call of SD 2.x training and of full-size sampling, replayed alone against an fp64 reference.

The harness of test_call_signatures_gpu.py (NaN guard bands, NaN-filled torch.empty inside ops, a global bound per
output and 4x that bound per block of the kernel's tiling) over four workloads the SD 1.4 and VAE replays do not record:
  sd2_pretrain_768_b16         eager SD 2.x PretrainStep at 768² (96 x 96 latents), B = 16: v prediction, pad id 0,
                               cosine schedule with warm-up; heads of 64 on the wgmma and the mma.sync attention, the
                               1024-wide context, linear proj_in / proj_out, adamw_step_sched;
  sd2_tuning_text_768_b4_8bit  eager SD 2.x TuningStep, text encoder trained in fp32, 8-bit AdamW with
                               constant_with_warmup, B = 4: adamw8bit_step_sched on the real 1.6 G-element arena;
  sd14_sample_512              the SD 1.4 pipeline with the SD VAE, 2 steps each: B = 1 DPM-Solver++ graphed (warm-up
                               and capture recorded), B = 4 Euler ancestral eager with a CUDA generator, B = 1 LMS
                               without guidance eager;
  sd2_sample_768               the SD 2.x pipeline with the SD VAE, PNDM with v prediction, B = 1, graphed; the VAE
                               decode at 768² runs softmax_rows over 9216 columns.

Alias groups: arguments of one call that are the same tensor (same data_ptr, shape and stride) are recorded as part of
the signature and replayed as one guarded tensor, so a call such as the graphed step's in-place update
sampler_step(..., x, x_next=x, ...) is replayed as it runs.  References read the values from before the call, checks
read the tensor after it, and an aliased output is not NaN-filled before the call (it is also an input).

New references against fp64: adamw_step_sched (the schedule at a step where its factor is neither 0 nor 1),
adamw8bit_step_sched (random codes, absmax over 1e-8 .. 1e2, whole 256-element blocks sampled) and sampler_step (a
table row with every term live).  The attention and softmax signatures are replayed again at peaked scores."""
import inspect
import math
import os
import sys
import time
import types
from collections import Counter, OrderedDict

import pytest
import torch

from oracle import vae_oracle as V

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_call_signatures_gpu as H  # noqa: E402
import test_optimizer_options_gpu as OO  # noqa: E402
import test_ragged_gpu as RG  # noqa: E402
from test_call_signatures_gpu import (LOCAL, Call, Check, Guarded, Recorder, _free, describe,  # noqa: E402
                                      evaluate, spec)

pytestmark = pytest.mark.gpu
F64 = torch.float64
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BLOCK = 256                 # elements per absmax block of the 8-bit moments
U8_SENTINEL = 0xA5          # guard value of uint8 buffers (the 8-bit moment codes)


@pytest.fixture(scope="module", autouse=True)
def _keep_direct_grad_write():
    """FlatAdamW sets functional.DIRECT_GRAD_WRITE for the whole process; put it back after this file."""
    from e4t_b200 import functional as FN
    saved = FN.DIRECT_GRAD_WRITE
    yield
    FN.DIRECT_GRAD_WRITE = saved


# ---------------------------------------------------------------------------------------------------------------------
# alias-aware recording and replay
# ---------------------------------------------------------------------------------------------------------------------
def alias_groups(items):
    """Names of the tensor arguments that are one tensor (data_ptr, shape, stride), in argument order; groups of 2+."""
    by = OrderedDict()
    for n, v in items:
        if isinstance(v, torch.Tensor) and v.numel():
            by.setdefault((v.data_ptr(), tuple(v.shape), tuple(v.stride())), []).append(n)
    return tuple(tuple(g) for g in by.values() if len(g) > 1)


class AliasRecorder(Recorder):
    """Recorder whose keys are (op, ((param, spec), ...), alias groups)."""

    def _wrap(self, name, fn):
        sig = inspect.signature(fn)

        def w(*args, **kw):
            b = sig.bind(*args, **kw)
            b.apply_defaults()
            items = tuple(b.arguments.items())
            key = (name, tuple((k, spec(v)) for k, v in items), alias_groups(items))
            self.calls[key] = self.calls.get(key, 0) + 1
            return fn(*args, **kw)
        return w


class GuardedU8(Guarded):
    """Guarded for uint8 buffers, whose guard value is U8_SENTINEL."""

    def __init__(self, sp, device="cuda"):
        _, shape, stride, dt, mis = sp
        self.dtype = torch.uint8
        self.off = H.GUARD + mis
        self.span = (1 + sum((s - 1) * st for s, st in zip(shape, stride))) if all(shape) else 0
        self.fill = U8_SENTINEL
        self.buf = torch.full((self.off + self.span + H.GUARD,), U8_SENTINEL, device=device, dtype=torch.uint8)
        self.t = self.buf.as_strided(shape, stride, self.off)
        self.numel = self.t.numel()

    def outside_intact(self):
        mask = torch.ones_like(self.buf, dtype=torch.bool)
        mask.as_strided(self.t.shape, self.t.stride(), self.off).fill_(False)
        return bool((self.buf[mask] == U8_SENTINEL).all())


def _guarded(sp):
    return GuardedU8(sp) if sp[3] == "uint8" else Guarded(sp)


class ACall(Call):
    """Call with one guarded tensor per alias group: every name of the group is that tensor."""

    def __init__(self, key, g):
        self.name, self.g = key[0], g
        self.kw, self.guarded = {}, {}
        self.aliases = key[2] if len(key) > 2 else ()
        head = {n: grp[0] for grp in self.aliases for n in grp}
        for n, sp in key[1]:
            if head.get(n, n) != n:
                self.kw[n] = self.kw[head[n]]
            elif sp[0] == "T":
                gt = _guarded(sp)
                if gt.dtype.is_floating_point:
                    gt.t.copy_(torch.randn(gt.t.shape, generator=g, device="cuda"))
                self.guarded[n] = gt
                self.kw[n] = gt.t
            elif sp[0] == "L":
                gts = [_guarded(s) for s in sp[1]]
                for i, gt in enumerate(gts):
                    self.guarded[f"{n}[{i}]"] = gt
                self.kw[n] = [gt.t for gt in gts]
            else:
                self.kw[n] = sp[1]

    def aliased(self, n):
        return any(n in grp for grp in self.aliases)

    def nan_(self, n):
        if not self.aliased(n):          # an aliased output is also an input: it keeps its values
            super().nan_(n)


def describe_key(key):
    groups = key[2] if len(key) > 2 else ()
    return describe(key) + "".join(f" [{' = '.join(grp)}]" for grp in groups)


# ---------------------------------------------------------------------------------------------------------------------
# workloads
# ---------------------------------------------------------------------------------------------------------------------
def _sd2_ab():
    tools = os.path.join(ROOT, "tools")
    if tools not in sys.path:
        sys.path.insert(0, tools)
    import sd2_ab
    return sd2_ab


def workload_sd2_pretrain():
    from e4t_b200.engine import PretrainStep
    A = _sd2_ab()
    unet, enc, text = A.build()
    step = PretrainStep(unet, enc, text, 49408, class_token_id=320, prediction_type="v_prediction", pad_id=0,
                        lr_scheduler="cosine", lr_warmup_steps=100, max_train_steps=1000)
    b = A.batch(16, 1)
    step(b)
    torch.cuda.synchronize()
    with AliasRecorder() as r:
        step(b)
        torch.cuda.synchronize()
    return r.calls


def workload_sd2_tuning_8bit():
    from e4t_b200.engine import TuningStep
    A = _sd2_ab()
    unet, enc, text = A.build()
    text.float()
    step = TuningStep(unet, enc, text, 49408, class_token_id=320, train_text_encoder=True, use_8bit_adam=True,
                      lr_scheduler="constant_with_warmup", lr_warmup_steps=100, prediction_type="v_prediction",
                      pad_id=0)
    b = A.batch(4, 2)
    step(b)
    torch.cuda.synchronize()
    with AliasRecorder() as r:
        step(b)
        torch.cuda.synchronize()
    return r.calls


def _pipeline(unet, enc, text, scheduler):
    from test_pipeline_gpu import _Tok
    from e4t.models.autoencoder_kl import AutoencoderKL
    from e4t.pipeline_stable_diffusion_e4t import StableDiffusionE4TPipeline
    torch.manual_seed(0)
    vae = AutoencoderKL(**V.SD_VAE).cuda().eval().requires_grad_(False)
    cfg = types.SimpleNamespace(placeholder_token="*s", domain_class_token="a", domain_embed_scale=0.1)
    return StableDiffusionE4TPipeline(vae, text, _Tok(), unet, enc, scheduler, e4t_config=cfg)


def _sample(pipe, B, guidance, image_px, seed):
    g = torch.Generator().manual_seed(seed)
    image = torch.rand(1, 3, image_px, image_px, generator=g) * 2 - 1
    out = pipe(["a photo of *s"] * B, num_inference_steps=2, guidance_scale=guidance, image=image, output_type="np",
               generator=torch.Generator(device="cuda").manual_seed(seed)).images
    side = pipe.unet.config.sample_size * 8
    assert out.shape == (B, side, side, 3) and bool(torch.isfinite(torch.from_numpy(out)).all())


def workload_sd14_sample():
    import bench
    from e4t.schedulers import DPMSolverMultistepScheduler, EulerAncestralDiscreteScheduler, LMSDiscreteScheduler
    unet, enc, text = bench.build_models("cuda")
    pipe = _pipeline(unet, enc, text, DPMSolverMultistepScheduler())
    with AliasRecorder() as r:
        pipe.enable_cuda_graph()
        _sample(pipe, 1, 7.5, 512, 1)
        pipe.disable_cuda_graph()
        pipe.scheduler = EulerAncestralDiscreteScheduler()
        _sample(pipe, 4, 7.5, 512, 2)
        pipe.scheduler = LMSDiscreteScheduler()
        _sample(pipe, 1, 1.0, 512, 3)
        torch.cuda.synchronize()
    return r.calls


def workload_sd2_sample():
    from e4t.schedulers import PNDMScheduler
    unet, enc, text = _sd2_ab().build()
    pipe = _pipeline(unet, enc, text, PNDMScheduler(prediction_type="v_prediction"))
    pipe.enable_cuda_graph()
    with AliasRecorder() as r:
        _sample(pipe, 1, 7.5, 768, 4)
        torch.cuda.synchronize()
    return r.calls


WORKLOADS = [("sd2_pretrain_768_b16", workload_sd2_pretrain),
             ("sd2_tuning_text_768_b4_8bit", workload_sd2_tuning_8bit),
             ("sd14_sample_512", workload_sd14_sample), ("sd2_sample_768", workload_sd2_sample)]


def record_all():
    """OrderedDict key -> {workload: calls}, and per workload (distinct calls, wall time, peak allocated bytes)."""
    inv, stats = OrderedDict(), {}
    for wname, fn in WORKLOADS:
        _free()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.time()
        calls = fn()
        peak = torch.cuda.max_memory_allocated()
        _free()
        stats[wname] = (len(calls), time.time() - t0, peak)
        for k, n in calls.items():
            inv.setdefault(k, {})[wname] = n
    return inv, stats


# ---------------------------------------------------------------------------------------------------------------------
# fp64 references of the three ops the SD 1.4 replay does not reach
# ---------------------------------------------------------------------------------------------------------------------
def _schedule_point(sched, lr):
    """(schedule name, steps taken t0, factor λ(t0)): inside the warm-up for constant_with_warmup, past it for the
    decaying schedules, so the factor the kernel applies is neither 0 nor 1."""
    from e4t_b200 import optim
    kind, W, T = sched[:3]
    name = optim.SCHEDULES[kind]
    if name == "constant":
        t0 = 4
    elif name == "constant_with_warmup" or T <= W:
        t0 = max(1, W // 2)
    else:
        t0 = W + max(1, (T - W) // 3)
    lam = optim.lr_lambda(name, t0, W, T or None, lr)
    assert name == "constant" or 0 < lam < 1, f"{name}: the factor at step {t0} is {lam}: pick another step"
    return name, t0, lam


def _lr_and_step_checks(c, t0, lr_k):
    got = c["lr_dev"].item()
    assert abs(got - lr_k) <= 1e-6 * abs(lr_k), f"lr_dev {got!r}, schedule gives {lr_k!r}"
    assert int(c["step_dev"].item()) == t0 + 1, f"step_dev {int(c['step_dev'].item())}, expected {t0 + 1}"


def h_adamw_step_sched(c):
    p, g, m, v = c["p"], c["g"], c["m"], c["v"]
    n = p.numel()
    v.copy_(torch.rand(v.shape, generator=c.g, device="cuda") * 1e-2)
    m.mul_(0.1)
    _, t0, lam = _schedule_point(c["sched"], c["lr"])
    lr_k = c["lr"] * lam
    c["step_dev"].fill_(t0)
    c.nan_("lr_dev")
    # the seeded sample of h_adamw_step_dev: the first and last 4-float vector blocks, the tail, 2^20 random indices
    head = torch.arange(min(n, 4096), device="cuda")
    tail = torch.arange(max(0, n - 4099), n, device="cuda")
    mid = torch.randint(0, n, (1 << 20,), generator=c.g, device="cuda")
    idx = torch.cat([head, mid, tail]).unique()
    before = [H._d(t.reshape(-1)[idx]) for t in (p, g, m, v)]
    f = OO._f32
    pr, mr, vr = H._adamw_ref(*before, f(lr_k), f(c["beta1"]), f(c["beta2"]), f(c["eps"]), f(c["weight_decay"]),
                              t0 + 1, c["grad_scale"])
    c.run()
    _lr_and_step_checks(c, t0, lr_k)
    return [Check("p", p.reshape(-1)[idx], pr, 1e-5), Check("m", m.reshape(-1)[idx], mr, 1e-5),
            Check("v", v.reshape(-1)[idx], vr, 1e-5)]


def _worst_block(bad_elems, blocks):
    """Arena block index of the first flagged element of the sampled blocks (bad_elems: bool over the sample)."""
    return int(blocks[int(bad_elems.nonzero()[0, 0]) // BLOCK])


def _codes_problem(got, want, x, q, blocks, what):
    """test_optimizer_options_gpu._check_codes with the failing block named: codes equal, except where x's fp64
    distances to two neighbouring map entries tie to 1e-6."""
    got, want = got.long(), want.long()
    bad = got != want
    tie = ((got - want).abs() == 1) & (((x - q[got]).abs() - (x - q[want]).abs()).abs() <= 1e-6)
    wrong = bad & ~tie
    if bool(wrong.any()):
        return (f"{what}: {int(wrong.sum())} codes differ beyond a tie, first in block {_worst_block(wrong, blocks)} "
                f"(got {got[wrong][:4].tolist()}, want {want[wrong][:4].tolist()})")
    return None


def h_adamw8bit_step_sched(c):
    from e4t_b200 import optim
    p, g = c["p"], c["g"]
    n = p.numel()
    nb = n // BLOCK
    gen = c.g
    # state: random codes, one absmax per block spread over 1e-8 .. 1e2, the dynamic maps the optimiser codes with
    for name in ("m_codes", "v_codes"):
        c[name].copy_(torch.randint(0, 256, c[name].shape, generator=gen, device="cuda", dtype=torch.uint8))
    for name in ("m_absmax", "v_absmax"):
        c[name].copy_(10.0 ** (torch.rand(nb, generator=gen, device="cuda") * 10 - 8))
    c["qmap_m"].copy_(optim.dynamic_map(True))
    c["qmap_v"].copy_(optim.dynamic_map(False))
    # gradients: per-block scales 1e-8 .. 1e2; every 16th block all zero; every 16th (offset 8) spans 1e-8 .. 1e2 inside
    gv = g.view(nb, BLOCK)
    gv.mul_(10.0 ** (torch.rand(nb, generator=gen, device="cuda") * 10 - 8)[:, None])
    mixed = torch.arange(8, nb, 16, device="cuda")
    gv[mixed] = (torch.randn(mixed.numel(), BLOCK, generator=gen, device="cuda")
                 * 10.0 ** (torch.rand(mixed.numel(), BLOCK, generator=gen, device="cuda") * 10 - 8))
    gv[0::16] = 0
    _, t0, lam = _schedule_point(c["sched"], c["lr"])
    lr_k = c["lr"] * lam
    c["step_dev"].fill_(t0)
    c.nan_("lr_dev")
    # a seeded sample of whole blocks, always with the first and the last
    blocks = torch.cat([torch.tensor([0, nb - 1], device="cuda"),
                        torch.randint(0, nb, (4096,), generator=gen, device="cuda")]).unique()
    idx = (blocks[:, None] * BLOCK + torch.arange(BLOCK, device="cuda")).reshape(-1)
    qm64, qv64 = c["qmap_m"].double(), c["qmap_v"].double()
    f = OO._f32
    ref = OO.adamw8bit_ref(H._d(p[idx]), H._d(g[idx]), c["m_codes"][idx], c["v_codes"][idx],
                           H._d(c["m_absmax"][blocks]), H._d(c["v_absmax"][blocks]), qm64, qv64, f(lr_k),
                           f(c["beta1"]), f(c["beta2"]), f(c["eps"]), f(c["weight_decay"]), t0 + 1, c["grad_scale"])
    c.run()
    _lr_and_step_checks(c, t0, lr_k)
    problems = [f"{name} has non-finite elements" for name in ("p", "m_absmax", "v_absmax")
                if not bool(torch.isfinite(c[name]).all())]
    # p: 1e-5 relative plus 1e-4 of the Adam update (the kernel's fp32 bias corrections, test_optimizer_options_gpu)
    tol = 1e-5 * ref["p"].abs() + 1e-4 * ref["upd"].abs() + 1e-30
    err = (p[idx].double() - ref["p"]).abs()
    if not bool((err <= tol).all()):
        problems.append(f"p: {(err / tol).max().item():.2f}x its element bound, first in block "
                        f"{_worst_block(err > tol, blocks)}")
    for what, got, want in (("m absmax", c["m_absmax"][blocks], ref["ma"]),
                            ("v absmax", c["v_absmax"][blocks], ref["va"])):
        e = ((got.double() - want).abs() / want.abs().clamp_min(1e-300)).where(want != 0, got.double().abs())
        if e.max().item() > 1e-6:
            problems.append(f"{what}: relative error {e.max().item():.2e} (bound 1e-6) in block "
                            f"{int(blocks[int(e.argmax())])}")
    for what, got, want, x, q in (("m codes", c["m_codes"][idx], ref["mc"], ref["xm"], qm64),
                                  ("v codes", c["v_codes"][idx], ref["vc"], ref["xv"], qv64)):
        msg = _codes_problem(got, want, x, q, blocks, what)
        if msg:
            problems.append(msg)
    assert not problems, "; ".join(problems)
    return [Check("p", p[idx], ref["p"], 1e-5, block=(1, BLOCK), unit="sampled 256-element block")]


def h_sampler_step(c):
    """One table row with every term live: sample, guided output, each history slot below n_hist, saved sample, noise
    (when given); an in-range history slot written; the sample saved; the next model input and timestep published."""
    import e4t.schedulers as SC
    from test_schedulers_cpu import apply_row
    x, out, hist, table = c["x"], c["out"], c["hist"], c["table"]
    n = x.numel()
    G, n_hist, rows = out.numel() // n, hist.shape[0], table.shape[0]
    gen = torch.Generator().manual_seed(int(torch.randint(0, 1 << 30, (1,), generator=c.g, device="cuda")))
    coef = lambda: 0.25 + 0.75 * torch.rand(1, generator=gen).item()                    # noqa: E731
    i = int(torch.randint(0, rows, (1,), generator=gen))
    r = torch.zeros(SC.ROW, dtype=F64)
    r[SC.X], r[SC.E], r[SC.S] = coef(), -coef(), coef()
    for k in range(n_hist):
        r[SC.H0 + k] = coef() * (-1) ** k
    r[SC.Z] = coef() if c["noise"] is not None else 0.0
    r[SC.SLOT] = int(torch.randint(0, n_hist, (1,), generator=gen)) if n_hist else -1
    r[SC.HA], r[SC.HB], r[SC.SAVE] = coef(), -coef(), 1.0
    r[SC.S_NEXT], r[SC.T_NEXT] = 1.0 + coef(), float(int(torch.randint(1, 1000, (1,), generator=gen)))
    table[i].copy_(r)
    c["step_dev"].fill_(i)
    if c["guidance"] is not None:
        c["guidance"].fill_(7.5)
    for name in ("x_next", "row", "t_out", "model_in"):
        c.nan_(name)
    # fp64 reference from the values before the call (x_next may be x)
    x0 = H._d(x).reshape(-1)
    o = H._d(out).reshape(G, n)
    e = o[0] + 7.5 * (o[1] - o[0]) if G == 2 else o[0]
    hist0 = H._d(hist)
    hl = [hist0[k, :n].clone() if k < n_hist else torch.zeros(n, dtype=F64, device="cuda")
          for k in range(SC.MAX_HISTORY)]
    z = H._d(c["noise"]).reshape(-1) if c["noise"] is not None else None
    xn, saved = apply_row(r.cuda(), e, x0, hl, H._d(c["saved"]).reshape(-1), z)
    c.run()
    blk = dict(view2d=lambda t: t.reshape(1, -1), block=(1, 1024), unit="1024-element block")
    checks = [Check("x_next", c["x_next"], xn, 1e-5, **blk),
              Check("saved (the old x, exact)", c["saved"], saved, 0.0, **blk)]
    if n_hist:
        s = int(r[SC.SLOT])
        keep = torch.ones(hist.shape, dtype=torch.bool, device="cuda")
        keep[s, :n] = False
        checks += [Check(f"hist[{s}]", hist[s, :n], hl[s], 1e-5, **blk),
                   Check("hist outside the written slot (unchanged, exact)", hist[keep], hist0[keep], 0.0, **blk)]
    if c["model_in"] is not None:
        mi = c["model_in"].reshape(G, n)
        checks += [Check(f"model_in[{h}]", mi[h], xn * r[SC.S_NEXT].item(), 1e-5, **blk) for h in range(G)]
    want_row = r.float().cuda()
    assert torch.equal(c["row"][:SC.ROW], want_row), f"published row {c['row'][:SC.ROW].tolist()} != {want_row.tolist()}"
    if c["t_out"] is not None:
        assert c["t_out"].item() == want_row[SC.T_NEXT].item(), f"t_out {c['t_out'].item()} != {r[SC.T_NEXT].item()}"
    assert int(c["step_dev"].item()) == i + 1, f"step_dev {int(c['step_dev'].item())}, expected {i + 1}"
    return checks


HANDLERS = dict(RG.HANDLERS, adamw_step_sched=h_adamw_step_sched, adamw8bit_step_sched=h_adamw8bit_step_sched,
                sampler_step=h_sampler_step)


# ---------------------------------------------------------------------------------------------------------------------
# the inventory, and what the workloads exist for
# ---------------------------------------------------------------------------------------------------------------------
def _shape(key, name):
    sp = H._arg(key, name)
    return sp[1] if sp[0] == "T" else None


def _attn_shapes(inv, op):
    """(B, N, M, dh) of every recorded call of an attention op."""
    out = set()
    for k in inv:
        if k[0] == op:
            (B, N, C), M = _shape(k, "q"), _shape(k, "k")[1]
            out.add((B, N, M, C // H._arg(k, "heads")[1]))
    return out


def check_inventory(inv, stats):
    """Prints the inventory and asserts that the workloads reached what they exist for."""
    for w, (n, secs, peak) in stats.items():
        ops = Counter(k[0] for k, ws in inv.items() if w in ws)
        print(f"[inventory {w}] {n} distinct calls, recorded in {secs:.0f} s, peak {peak / 2 ** 30:.1f} GiB: "
              + ", ".join(f"{op} {c}" for op, c in sorted(ops.items())))
    groups = Counter((k[0], grp) for k in inv for grp in k[2])
    print("[inventory] alias groups: " + (", ".join(f"{op} {' = '.join(g)} ({c} signatures)"
                                                    for (op, g), c in sorted(groups.items())) or "none"))
    ops_seen = {k[0] for k in inv}
    assert not ops_seen - set(HANDLERS), f"recorded but not replayed: {sorted(ops_seen - set(HANDLERS))}"
    # heads of 64 at the B = 16 shapes the wgmma rule of ops.attn_fwd takes, and at shapes it leaves to mma.sync
    for op in ("attn_fwd", "attn_bwd"):
        sh = _attn_shapes(inv, op)
        assert {(16, 9216, 9216, 64), (16, 2304, 2304, 64)} <= sh, (op, sorted(sh))
        assert any(dh == 64 and (N in (576, 144) or M == 77) for _, N, M, dh in sh), (op, sorted(sh))
    n8 = [math.prod(_shape(k, "p")) for k in inv if k[0] == "adamw8bit_step_sched"]
    assert any(n > 10 ** 9 for n in n8), f"adamw8bit_step_sched arenas {n8}: none above 1e9 elements"
    assert any(k[0] == "adamw_step_sched" for k in inv)
    ss = [k for k in inv if k[0] == "sampler_step"]
    hist = {_shape(k, "hist")[0] for k in ss}
    noise = {_shape(k, "noise") is not None for k in ss}
    G = {math.prod(_shape(k, "out")) // math.prod(_shape(k, "x")) for k in ss}
    assert {2, 4} <= hist and noise == {True, False} and G == {1, 2}, (hist, noise, G)
    assert any(("x", "x_next") in k[2] for k in ss), "no sampler_step with x_next aliasing x"
    assert any(_shape(k, "x")[-1] == 9216 for k in inv if k[0] == "softmax_rows"), "no softmax_rows over 9216 columns"
    missing = [op for op in OPS if op not in ops_seen]
    assert not missing, f"the workloads no longer reach {missing}: a refactor routes around ops or a workload broke"
    assert ops_seen <= set(OPS), f"recorded but not in OPS (not replayed): {sorted(ops_seen - set(OPS))}"


@pytest.fixture(scope="module")
def inventory():
    t0 = time.time()
    inv, stats = record_all()
    check_inventory(inv, stats)
    print(f"[inventory] {len(inv)} distinct calls, recorded in {time.time() - t0:.0f} s")
    return inv


# every op the four workloads reach; each is replayed by its own test
OPS = sorted(set(H.REQUIRED) - {"adamw_step_dev"}
             | {"adamw_step_sched", "adamw8bit_step_sched", "sampler_step", "conv3x3_im2col", "wo_factors", "wo_weff"})


def replay(key, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    c = ACall(key, g)
    err = None
    try:
        results = [(chk,) + evaluate(chk) for chk in HANDLERS[key[0]](c)]
    except AssertionError as e:
        results, err = [], str(e)
    bad = c.guards_intact()
    del c
    return results, bad, err


@pytest.mark.parametrize("op", OPS)
def test_replay_every_recorded_call(inventory, op):
    keys = [k for k in inventory if k[0] == op]
    assert keys, f"no recorded call of {op}"
    t0 = time.time()
    failures, worst_g, worst_b = [], 0.0, 0.0
    for i, key in enumerate(keys):
        results, bad, err = replay(key, 3000 + i)
        sig = describe_key(key)
        if err:
            failures.append(f"{sig}: {err}")
        if bad:
            failures.append(f"{sig}: wrote outside the logical extent of {bad}")
        for chk, finite, glob, worst, where in results:
            if chk.bound:
                worst_g, worst_b = max(worst_g, glob / chk.bound), max(worst_b, worst / chk.bound)
            if not finite:
                failures.append(f"{sig}: {chk.label} has non-finite elements (unwritten or poisoned by a NaN read)")
            elif glob > chk.bound or worst > LOCAL * chk.bound:
                failures.append(f"{sig}: {chk.label} error {glob:.2e} (bound {chk.bound:.1e}); worst {chk.unit} "
                                f"at {where}: {worst:.2e} (bound {LOCAL * chk.bound:.1e})")
        _free()
    per = Counter(w for k in keys for w in inventory[k])
    print(f"[replay {op}] {len(keys)} signatures ({', '.join(f'{w} {n}' for w, n in sorted(per.items()))}); worst "
          f"global error {worst_g:.2f}x its bound, worst block {worst_b:.2f}x the global bound "
          f"({time.time() - t0:.0f} s)")
    assert not failures, "\n".join(failures)


def test_replay_attention_peaked(inventory):
    """test_call_signatures_gpu.test_replay_attention_peaked over these workloads' attention and softmax_rows
    signatures (none of them has an alias group)."""
    keys = [k for k in inventory if k[0] in H.PEAKED_OPS]
    assert not any(k[2] for k in keys), [describe_key(k) for k in keys if k[2]]
    t0 = time.time()
    H.test_replay_attention_peaked(inventory)
    print(f"[peaked replay] {len(keys)} signatures ({time.time() - t0:.0f} s)")
