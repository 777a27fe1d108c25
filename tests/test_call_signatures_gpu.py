"""Every distinct kernel call of the real training and VAE paths, replayed alone against an fp64 reference.

A module-scoped fixture wraps every public function of e4t_b200.ops that calls into the library and records each
distinct call (op, shape / stride / dtype / 16-byte misalignment of every tensor, every scalar, call count) over:
  (a) one eager SD-v1.4 PretrainStep at B = 16 (bench.py's models and inputs, after one warm-up step);
  (b) one eager TuningStep(train_text_encoder=True) on the same models at B = 16;
  (c) SD-config AutoencoderKL encode and decode at 512 x 512.
The kernel tests elsewhere check hand-picked shapes; this file checks exactly the tile widths, split-K factors and
epilogue paths that pick_bn / auto_splits choose for the shapes the product launches.

Replay: each distinct call runs alone on fresh seeded inputs laid out with the recorded strides and misalignment,
inside buffers whose elements outside the logical extent (column-slice gaps, guard bands before and after) are NaN,
so a read outside the tensor poisons the result and a write outside it is seen.  Outputs start NaN (read-write
arguments start random and the reference adds to them), and while the call runs the torch.empty / torch.empty_like
that ops uses return NaN-filled memory, so an unwritten output element or uninitialised internal scratch shows up.

Per output: everything in the logical extent is finite, everything outside it is still NaN, the RMS error relative to
the reference RMS is within the bound the op's own kernel test uses, and every block of the kernel's tiling (128 x 64
for the GEMM engine, (image, head, 64 queries) for attention, (image, group) for GroupNorm, rows for the row kernels)
has an RMS error of at most 4x that bound (relative to the RMS of the whole reference), so one wrong tile cannot hide in
a large tensor.  The WeightOffsets bank (_lib.call directly) is checked against fp64 by test_wo_bank_gpu.py.
"""
import gc
import inspect
import math
import time
from collections import OrderedDict

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

GUARD = 64            # NaN elements before and after every tensor (a multiple of 16 bytes for every dtype used)
LOCAL = 4.0           # block bound = LOCAL x the global bound
INT_SENTINEL = -7777  # guard value of integer buffers
NAN = float("nan")
F64 = torch.float64

# every op the three workloads must reach
REQUIRED = ["gemm", "conv3x3", "conv3x3_s2", "conv3x3_wgrad", "narrow_conv_wgrad", "softmax_rows",
            "groupnorm_fwd", "groupnorm_bwd", "groupnorm_param_grad", "layernorm_fwd", "layernorm_bwd",
            "layernorm_param_grad", "geglu_fwd", "geglu_bwd", "resample2x", "meanpool_fwd", "meanpool_bwd",
            "conv_in_fwd", "conv_out_fwd", "conv_out_bwd", "adamw_step_dev", "attn_fwd", "attn_bwd", "attn_small_fwd",
            "act_fwd", "act_bwd", "colsum_acc", "embedding_grad"]
# (the text tower's causal backward runs on attn_bwd(causal=True); the WeightOffsets projections go through the bank)


# ---------------------------------------------------------------------------------------------------------------------
# recording
# ---------------------------------------------------------------------------------------------------------------------
def lib_ops():
    """Names of the public functions of e4t_b200.ops that call into the library."""
    from e4t_b200 import ops
    return sorted(n for n, f in vars(ops).items() if inspect.isfunction(f) and f.__module__ == ops.__name__
                  and not n.startswith("_") and "_lib.call" in inspect.getsource(f))


def spec(v):
    """Hashable description of one argument: tensors by shape, stride, dtype and 16-byte misalignment of the base."""
    if isinstance(v, torch.Tensor):
        return ("T", tuple(v.shape), tuple(v.stride()), str(v.dtype).replace("torch.", ""),
                (v.data_ptr() % 16) // v.element_size())
    if isinstance(v, (list, tuple)) and any(isinstance(x, torch.Tensor) for x in v):
        return ("L", tuple(spec(x) for x in v))
    return ("V", v)


class Recorder:
    """Wraps ops' library-calling functions; calls[(op, ((param, spec), ...))] = count."""

    def __init__(self):
        self.calls = OrderedDict()

    def __enter__(self):
        from e4t_b200 import ops
        self.orig = {n: getattr(ops, n) for n in lib_ops()}
        for n, fn in self.orig.items():
            setattr(ops, n, self._wrap(n, fn))
        return self

    def _wrap(self, name, fn):
        sig = inspect.signature(fn)

        def w(*args, **kw):
            b = sig.bind(*args, **kw)
            b.apply_defaults()
            key = (name, tuple((k, spec(v)) for k, v in b.arguments.items()))
            self.calls[key] = self.calls.get(key, 0) + 1
            return fn(*args, **kw)
        return w

    def __exit__(self, *exc):
        from e4t_b200 import ops
        for n, fn in self.orig.items():
            setattr(ops, n, fn)


def _free():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def workload_pretrain():
    import bench
    from e4t_b200.engine import PretrainStep
    unet, enc, text = bench.build_models(torch.device("cuda"))
    step = PretrainStep(unet, enc, text, placeholder_token_id=49408, class_token_id=320, lr=1.6e-5,
                        weight_dtype=torch.bfloat16)
    b = bench.to_device(bench.host_batch(16, 42, pinned=False), "cuda")
    step(b)
    torch.cuda.synchronize()
    with Recorder() as r:
        step(b)
        torch.cuda.synchronize()
    return r.calls


def workload_tuning_text():
    import bench
    from e4t_b200.engine import TuningStep
    unet, enc, text = bench.build_models("cuda")
    text.float()
    b = bench.to_device(bench.host_batch(16, seed=1, pinned=False), "cuda")
    step = TuningStep(unet, enc, text, 49408, class_token_id=320, train_text_encoder=True)
    step(b)
    torch.cuda.synchronize()
    with Recorder() as r:
        step(b)
        torch.cuda.synchronize()
    return r.calls


def workload_vae():
    from oracle import vae_oracle as V
    from e4t.models.autoencoder_kl import AutoencoderKL
    torch.manual_seed(0)
    vae = AutoencoderKL(**V.SD_VAE).cuda().eval().requires_grad_(False)
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.rand((1, 3, 512, 512), generator=g, device="cuda") * 2 - 1
    with torch.no_grad(), Recorder() as r:
        z = vae.encode(x).latent_dist.mean
        vae.decode(z)
        torch.cuda.synchronize()
    return r.calls


WORKLOADS = [("pretrain_b16", workload_pretrain), ("tuning_text_b16", workload_tuning_text),
             ("vae_sd_512", workload_vae)]


def record_all():
    """OrderedDict key -> {workload: calls}, and per-workload wall times."""
    inv, times = OrderedDict(), {}
    for wname, fn in WORKLOADS:
        t0 = time.time()
        calls = fn()
        _free()
        times[wname] = time.time() - t0
        for k, n in calls.items():
            inv.setdefault(k, {})[wname] = n
    return inv, times


def _arg(key, name):
    return dict(key[1])[name]


@pytest.fixture(scope="module")
def inventory():
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    inv, times = record_all()
    per = {}
    for k, ws in inv.items():
        for w in ws:
            per.setdefault(w, {}).setdefault(k[0], 0)
            per[w][k[0]] += 1
    for w, d in per.items():
        print(f"[inventory {w}] {sum(d.values())} distinct calls ({times[w]:.0f} s): "
              + ", ".join(f"{op} {n}" for op, n in sorted(d.items())))
    ops_seen = {k[0] for k in inv}
    missing = [op for op in REQUIRED if op not in ops_seen]
    assert not missing, f"the workloads no longer reach {missing}: a refactor routes around ops or a workload broke"
    s2_pads = {_arg(k, "pad_lo")[1] for k in inv if k[0] == "conv3x3_s2"}
    assert s2_pads == {0, 1}, s2_pads
    causal = {_arg(k, "causal")[1] for k in inv if k[0] == "attn_bwd"}
    assert causal == {False, True}, causal
    unreplayed = ops_seen - set(REQUIRED)
    assert not unreplayed, f"recorded but not replayed (add them to REQUIRED with a reference): {sorted(unreplayed)}"
    print(f"[inventory] {len(inv)} distinct calls, recorded in {time.time() - t0:.0f} s, peak "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")
    return inv


# ---------------------------------------------------------------------------------------------------------------------
# replay: NaN-guarded tensors and NaN-filled torch.empty
# ---------------------------------------------------------------------------------------------------------------------
class Guarded:
    """A tensor with the recorded shape / stride / misalignment inside a buffer whose other elements are NaN."""

    def __init__(self, sp, device="cuda"):
        _, shape, stride, dt, mis = sp
        self.dtype = getattr(torch, dt)
        self.off = GUARD + mis
        self.span = (1 + sum((s - 1) * st for s, st in zip(shape, stride))) if all(shape) else 0
        self.buf = torch.empty(self.off + self.span + GUARD, device=device, dtype=self.dtype)
        self.fill = NAN if self.dtype.is_floating_point else INT_SENTINEL
        self.buf.fill_(self.fill)
        self.t = self.buf.as_strided(shape, stride, self.off)
        self.numel = self.t.numel()

    def outside_intact(self):
        """True if every element outside the logical extent still holds its guard value."""
        if self.span == self.numel:           # dense: only the guard bands
            parts = [self.buf[:self.off], self.buf[self.off + self.span:]]
        else:
            mask = torch.ones_like(self.buf, dtype=torch.bool)
            mask.as_strided(self.t.shape, self.t.stride(), self.off).fill_(False)
            parts = [self.buf[mask]]
        for p in parts:
            ok = p.isnan().all() if self.dtype.is_floating_point else (p == INT_SENTINEL).all()
            if not bool(ok):
                return False
        return True


class _NaNTorch:
    """Stands in for `torch` inside ops while a replayed call runs: empty / empty_like return NaN-filled memory."""

    def __init__(self, real):
        self._real = real

    def __getattr__(self, n):
        return getattr(self._real, n)

    def empty(self, *a, **k):
        t = self._real.empty(*a, **k)
        return t.fill_(NAN) if t.is_floating_point() else t

    def empty_like(self, *a, **k):
        t = self._real.empty_like(*a, **k)
        return t.fill_(NAN) if t.is_floating_point() else t


def run_poisoned(name, kw):
    from e4t_b200 import ops
    real = ops.torch
    ops.torch = _NaNTorch(real)
    try:
        r = getattr(ops, name)(**kw)
        torch.cuda.synchronize()
    finally:
        ops.torch = real
    return r


class Call:
    """The arguments of one recorded call, rebuilt.  Tensors start random (bf16 / fp32: randn * scale); handlers
    re-fill inputs that must be consistent, and mark outputs with nan_()."""

    def __init__(self, key, g):
        self.name = key[0]
        self.g = g
        self.kw, self.guarded = {}, {}
        for n, sp in key[1]:
            if sp[0] == "T":
                gt = Guarded(sp)
                if gt.dtype.is_floating_point:
                    gt.t.copy_(torch.randn(gt.t.shape, generator=g, device="cuda"))
                self.guarded[n] = gt
                self.kw[n] = gt.t
            elif sp[0] == "L":
                gts = [Guarded(s) for s in sp[1]]
                for i, gt in enumerate(gts):
                    self.guarded[f"{n}[{i}]"] = gt
                self.kw[n] = [gt.t for gt in gts]
            else:
                self.kw[n] = sp[1]

    def __getitem__(self, n):
        return self.kw[n]

    def rnd(self, n, scale=1.0, shift=0.0):
        t = self.kw[n]
        t.copy_(torch.randn(t.shape, generator=self.g, device="cuda") * scale + shift)
        return t

    def nan_(self, n):
        t = self.kw[n]
        if isinstance(t, torch.Tensor):
            t.fill_(NAN)

    def run(self):
        return run_poisoned(self.name, self.kw)

    def guards_intact(self):
        return [n for n, gt in self.guarded.items() if not gt.outside_intact()]


# ---------------------------------------------------------------------------------------------------------------------
# error measures
# ---------------------------------------------------------------------------------------------------------------------
class Check:
    """One output: got vs ref (same shape), global RMS-relative error bound, and its block tiling: `view2d` maps a
    tensor to 2-D (rows, cols) and (br, bc) is the block size in that view."""

    def __init__(self, label, got, ref, bound, view2d=None, block=(1, 1 << 30), per_block_rms=False, unit=None):
        self.label, self.got, self.ref, self.bound = label, got, ref, bound
        self.unit = unit or ("row" if block[1] >= 1 << 30 else f"{block[0]} x {block[1]} block")
        self.per_block_rms = per_block_rms     # block error relative to the block's own reference RMS
        self.view2d = view2d or (lambda t: t.reshape(-1, t.shape[-1]) if t.dim() > 1 else t.reshape(1, -1))
        self.block = block


def block_errors(err2, ref_rms, br, bc):
    """Per-block RMS of err2 (2-D) / ref_rms (a scalar, or per block); returns (worst, (block row, block col))."""
    R, C = err2.shape
    br, bc = min(br, R), min(bc, C)
    Rp, Cp = -(-R // br) * br, -(-C // bc) * bc
    sq = torch.zeros(Rp, Cp, dtype=F64, device=err2.device)
    sq[:R, :C] = err2.double() ** 2
    cnt = torch.zeros(Rp, Cp, dtype=F64, device=err2.device)
    cnt[:R, :C] = 1
    s = sq.view(Rp // br, br, Cp // bc, bc).sum((1, 3))
    n = cnt.view(Rp // br, br, Cp // bc, bc).sum((1, 3))
    rms = (s / n.clamp_min(1)).sqrt() / ref_rms
    i = int(rms.argmax())
    return rms.max().item(), divmod(i, rms.shape[1])


def evaluate(chk):
    """(finite, global error, worst block error, worst block coordinates)."""
    got = chk.got.detach()
    finite = bool(torch.isfinite(got).all())
    ref = chk.ref.to(got.device, F64)
    g2, r2 = chk.view2d(got.double()), chk.view2d(ref)
    err = g2 - r2
    ref_rms = r2.pow(2).mean().sqrt().clamp_min(1e-30)
    glob = (err.pow(2).mean().sqrt() / ref_rms).item()
    if chk.per_block_rms:
        br, bc = chk.block
        R, C = r2.shape
        assert R % br == 0 and C % bc == 0
        ref_rms = r2.reshape(R // br, br, C // bc, bc).pow(2).mean((1, 3)).sqrt().clamp_min(1e-30)
    worst, where = block_errors(err.nan_to_num(nan=1e30), ref_rms, *chk.block)
    return finite, glob, worst, where


# ---------------------------------------------------------------------------------------------------------------------
# fp64 references, one per op (restating the contracts in ops.py's docstrings)
# ---------------------------------------------------------------------------------------------------------------------
TILE = (128, 64)      # the engine's output tile


def _d(t):
    return t.detach().to(F64).contiguous()


def h_gemm(c):
    A, B = _d(c["A"]), _d(c["B"])
    if c["a_mn"]:
        A = A.transpose(-1, -2)
    if not c["b_mn"]:
        B = B.transpose(-1, -2)
    acc = c["accumulate"]
    out = c["out"]
    if acc:
        c.rnd("out")
        init = _d(out).clone()
    elif out is not None:
        c.nan_("out")
    ref = c["alpha"] * torch.matmul(A, B)
    if c["bias"] is not None:
        ref = ref + _d(c["bias"])
    if c["rowgroup"] is not None:
        M = ref.shape[-2]
        rg = _d(c["rowgroup"]).view(-1, ref.shape[-1])
        ref = ref + rg[torch.arange(M, device=ref.device) // max(c["rows_per_group"], 1)]
    if c["residual"] is not None:
        ref = ref + _d(c["residual"])
    if acc:
        ref = ref.reshape(init.shape) + init
    r = c.run()
    got = out if out is not None else r
    bound = 4e-3 if got.dtype == torch.bfloat16 else 2e-3
    return [Check("out", got, ref.reshape(got.shape), bound, block=TILE)]


def _w9_to_oihw(w9):
    _, Co, Ci = w9.shape
    return _d(w9).view(3, 3, Co, Ci).permute(2, 3, 0, 1)


def _nchw(t):
    return _d(t).permute(0, 3, 1, 2)


def h_conv3x3(c):
    ref = F.conv2d(_nchw(c["x"]), _w9_to_oihw(c["w9"]), padding=1).permute(0, 2, 3, 1)
    if c["bias"] is not None:
        ref = ref + _d(c["bias"])
    if c["rowgroup"] is not None:
        ref = ref + _d(c["rowgroup"]).view(ref.shape[0], 1, 1, -1)
    if c["residual"] is not None:
        ref = ref + _d(c["residual"])
    got = c.run()
    return [Check("out", got, ref, 4e-3 if got.dtype == torch.bfloat16 else 2e-3, block=TILE)]


def h_conv3x3_s2(c):
    x = _nchw(c["x"])
    if c["pad_lo"] == 1:
        ref = F.conv2d(x, _w9_to_oihw(c["w9"]), stride=2, padding=1)
    else:
        ref = F.conv2d(F.pad(x, (0, 1, 0, 1)), _w9_to_oihw(c["w9"]), stride=2)
    ref = ref.permute(0, 2, 3, 1)
    if c["bias"] is not None:
        ref = ref + _d(c["bias"])
    return [Check("out", c.run(), ref, 4e-3, block=TILE)]


def h_conv3x3_wgrad(c):
    x, dy = _nchw(c["x"]), _nchw(c["dy"])
    w = torch.nn.grad.conv2d_weight(x, (dy.shape[1], x.shape[1], 3, 3), dy, padding=1)
    ref = w.permute(2, 3, 0, 1).reshape(9, dy.shape[1], x.shape[1])
    return [Check("dw9", c.run(), ref, 2e-3, block=TILE)]


def h_narrow_conv_wgrad(c):
    wide, narrow, sgn = _d(c["wide"]), _d(c["narrow"]), c["sgn"]
    Bn, H, W, Cw = wide.shape
    npad = F.pad(narrow, (1, 1, 1, 1))
    taps = []
    for ky in range(3):
        for kx in range(3):
            oy, ox = 1 + sgn * (ky - 1), 1 + sgn * (kx - 1)
            taps.append(torch.einsum("byxw,bnyx->wn", wide, npad[:, :, oy:oy + H, ox:ox + W]))
    ref = torch.stack(taps, -1)
    return [Check("acc", c.run(), ref, 2e-3, view2d=lambda t: t.reshape(t.shape[0], -1), block=(128, 64))]


def h_softmax_rows(c):
    c.rnd("x", 3.0)
    if c["out"] is not None:
        c.nan_("out")
    ref = torch.softmax(_d(c["x"]), -1)
    r = c.run()
    return [Check("out", r, ref, 4e-3, block=(1, 1 << 30))]


def _gn_setup(c):
    x = c.rnd("x", 1.5, 0.3)
    C = x.shape[-1]
    gamma = c.rnd("gamma", 0.3, 1.0)
    beta = c.rnd("beta", 0.2)
    return x, C, gamma, beta


def _gn_ref(c, x, gamma, beta, dy=None):
    Bn, C, G = x.shape[0], x.shape[-1], c["groups"]
    xr = _d(x).reshape(Bn, -1, C).permute(0, 2, 1).requires_grad_(True)
    gr, br = _d(gamma).requires_grad_(True), _d(beta).requires_grad_(True)
    y = F.group_norm(xr, G, gr, br, c["eps"])
    if c["silu"]:
        y = F.silu(y)
    if dy is not None:
        y.backward(_d(dy).reshape(Bn, -1, C).permute(0, 2, 1))
    return y.detach().permute(0, 2, 1), xr.grad, gr.grad, br.grad


def _gn_view(G):
    # (image, group) blocks: (B, HW, C) -> (B * G, HW * C/G)
    def v(t):
        Bn, C = t.shape[0], t.shape[-1]
        return t.reshape(Bn, -1, G, C // G).permute(0, 2, 1, 3).reshape(Bn * G, -1)
    return v


def _gn_stats(c, x, gamma, beta):
    from e4t_b200 import ops
    _, st = ops.groupnorm_fwd(x, gamma, beta, c["groups"], c["eps"], c["silu"])
    c["stats"].copy_(st)


def h_groupnorm_fwd(c):
    x, C, gamma, beta = _gn_setup(c)
    y_ref = _gn_ref(c, x, gamma, beta)[0]
    y, stats = c.run()
    Bn = x.shape[0]
    assert bool(torch.isfinite(stats).all()), "groupnorm stats not finite"
    return [Check("y", y.reshape(Bn, -1, C), y_ref, 4e-3, view2d=_gn_view(c["groups"]), block=(1, 1 << 40),
                  unit="(image * G + group)")]


def h_groupnorm_bwd(c):
    x, C, gamma, beta = _gn_setup(c)
    dy = c.rnd("dy")
    _gn_stats(c, x, gamma, beta)
    _, dx_ref, _, _ = _gn_ref(c, x, gamma, beta, dy)
    dx = c.run()
    return [Check("dx", dx.reshape(x.shape[0], -1, C), dx_ref.permute(0, 2, 1), 4e-3, view2d=_gn_view(c["groups"]),
                  block=(1, 1 << 40), unit="(image * G + group)")]


def h_groupnorm_param_grad(c):
    x, C, gamma, beta = _gn_setup(c)
    dy = c.rnd("dy")
    _gn_stats(c, x, gamma, beta)
    _, _, dg_ref, db_ref = _gn_ref(c, x, gamma, beta, dy)
    dg, db = c.run()
    return [Check("dgamma", dg, dg_ref, 4e-3, block=(1, 64)), Check("dbeta", db, db_ref, 4e-3, block=(1, 64))]


def _ln_ref(c, x, gamma, beta, dy=None):
    C = x.shape[-1]
    xr = _d(x).requires_grad_(True)
    gr, br = _d(gamma).requires_grad_(True), _d(beta).requires_grad_(True)
    y = F.layer_norm(xr, (C,), gr, br, c["eps"] if "eps" in c.kw else 1e-5)
    if dy is not None:
        y.backward(_d(dy))
    return y.detach(), xr.grad, gr.grad, br.grad


def _ln_stats(c, x, gamma, eps):
    from e4t_b200 import ops
    _, st = ops.layernorm_fwd(x, gamma, torch.zeros_like(gamma), eps)
    c["stats"].copy_(st)


def h_layernorm_fwd(c):
    x = c.rnd("x", 2.0, 0.5)
    gamma, beta = c.rnd("gamma", 0.3, 1.0), c.rnd("beta", 0.2)
    y_ref = _ln_ref(c, x, gamma, beta)[0]
    y, stats = c.run()
    assert bool(torch.isfinite(stats).all()), "layernorm stats not finite"
    return [Check("y", y, y_ref, 4e-3)]


def h_layernorm_bwd(c):
    x, dy = c.rnd("x", 2.0, 0.5), c.rnd("dy")
    gamma = c.rnd("gamma", 0.3, 1.0)
    _ln_stats(c, x, gamma, c["eps"])
    dx_ref = _ln_ref(c, x, gamma, torch.zeros_like(gamma), dy)[1]
    return [Check("dx", c.run(), dx_ref, 4e-3)]


def h_layernorm_param_grad(c):
    x, dy = c.rnd("x", 2.0, 0.5), c.rnd("dy")
    gamma = c.rnd("gamma", 0.3, 1.0)
    _ln_stats(c, x, gamma, 1e-5)
    _, _, dg_ref, db_ref = _ln_ref(c, x, gamma, torch.zeros_like(gamma), dy)
    dg, db = c.run()
    return [Check("dgamma", dg, dg_ref, 4e-3, block=(1, 64)), Check("dbeta", db, db_ref, 4e-3, block=(1, 64))]


def h_geglu_fwd(c):
    h = _d(c["h"])
    u, gate = h.chunk(2, -1)
    return [Check("out", c.run(), u * F.gelu(gate), 4e-3)]


def h_geglu_bwd(c):
    h = _d(c["h"]).requires_grad_(True)
    u, gate = h.chunk(2, -1)
    (u * F.gelu(gate)).backward(_d(c["dout"]))
    return [Check("dh", c.run(), h.grad, 4e-3)]


def _act(x, mode):
    if mode == 0:
        return F.gelu(x)
    if mode == 1:
        return x * torch.sigmoid(1.702 * x)
    return F.leaky_relu(x, 0.01)


def h_act_fwd(c):
    return [Check("y", c.run(), _act(_d(c["x"]), c["mode"]), 4e-3)]


def h_act_bwd(c):
    x = _d(c["x"]).requires_grad_(True)
    _act(x, c["mode"]).backward(_d(c["dy"]))
    return [Check("dx", c.run(), x.grad, 4e-3)]


def h_resample2x(c):
    x, mode = _d(c["x"]), c["mode"]
    if mode == 0:
        ref = x.repeat_interleave(2, 1).repeat_interleave(2, 2)
    elif mode == 1:
        Bn, H, W, C = x.shape
        ref = x.view(Bn, H // 2, 2, W // 2, 2, C).sum((2, 4))
    elif mode == 2:
        ref = x[:, ::2, ::2]
    else:
        Bn, H, W, C = x.shape
        ref = torch.zeros(Bn, 2 * H, 2 * W, C, dtype=F64, device=x.device)
        ref[:, ::2, ::2] = x
    return [Check("y", c.run(), ref, 4e-3)]


def h_meanpool_fwd(c):
    x = _d(c["x"])
    Bn, C = x.shape[0], x.shape[-1]
    init = _d(c["out"]).clone()        # read-write: columns outside [c_off, c_off + C) must be left alone
    ref = init.clone()
    ref[:, c["c_off"]:c["c_off"] + C] = x.reshape(Bn, -1, C).mean(1)
    c.run()
    return [Check("out", c["out"], ref, 1e-4)]


def h_meanpool_bwd(c):
    shape, off = c["shape"], c["c_off"]
    Bn, C = shape[0], shape[-1]
    HW = math.prod(shape[1:-1])
    ref = (_d(c["dout"])[:, None, off:off + C] / HW).expand(Bn, HW, C).reshape(shape)
    return [Check("dx", c.run(), ref, 4e-3)]


def h_conv_in_fwd(c):
    c.rnd("w", 0.2)
    ref = F.conv2d(_d(c["x"]), _d(c["w"]), _d(c["bias"]), padding=1).permute(0, 2, 3, 1)
    return [Check("y", c.run(), ref, 4e-3)]


def h_conv_out_fwd(c):
    c.rnd("w", 0.1)
    ref = F.conv2d(_nchw(c["x"]), _d(c["w"]), _d(c["bias"]), padding=1)
    return [Check("y", c.run(), ref, 1e-4, view2d=lambda t: t.reshape(-1, t.shape[-1]))]


def h_conv_out_bwd(c):
    c.rnd("w", 0.1)
    dy, w = _d(c["dy"]), _d(c["w"])
    Bn, Co, H, W = dy.shape
    ref = torch.nn.grad.conv2d_input((Bn, c["C"], H, W), w, dy, padding=1).permute(0, 2, 3, 1)
    return [Check("dx", c.run(), ref, 4e-3)]


def _adamw_ref(p, g, m, v, lr, b1, b2, eps, wd, t, gs):
    g = g * gs
    p = p * (1 - lr * wd)
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    denom = (v.sqrt() / math.sqrt(1 - b2 ** t)) + eps
    return p - (lr / (1 - b1 ** t)) * m / denom, m, v


def h_adamw_step_dev(c):
    p, g, m, v = c["p"], c["g"], c["m"], c["v"]
    n = p.numel()
    v.copy_(torch.rand(v.shape, generator=c.g, device="cuda") * 1e-2)
    m.mul_(0.1)
    t0 = 4
    c["step_dev"].fill_(t0)
    # a seeded sample that always holds the first and last 4-float vector blocks and the tail
    head = torch.arange(min(n, 4096), device="cuda")
    tail = torch.arange(max(0, n - 4099), n, device="cuda")
    mid = torch.randint(0, n, (1 << 20,), generator=c.g, device="cuda")
    idx = torch.cat([head, mid, tail]).unique()
    before = [_d(t.reshape(-1)[idx]) for t in (p, g, m, v)]
    pr, mr, vr = _adamw_ref(*before, c["lr"], c["beta1"], c["beta2"], c["eps"], c["weight_decay"], t0 + 1,
                            c["grad_scale"])
    c.run()
    assert int(c["step_dev"].item()) == t0 + 1
    return [Check("p", p.reshape(-1)[idx], pr, 1e-5), Check("m", m.reshape(-1)[idx], mr, 1e-5),
            Check("v", v.reshape(-1)[idx], vr, 1e-5)]


def _attn_ref_fwd(q, k, v, H, scale, causal):
    """o (B,N,C), lse (B,H,N), P (B,H,N,M) in fp64 for one image chunk."""
    B, N, C = q.shape
    M, dh = k.shape[1], C // H
    qh, kh, vh = (t.reshape(B, -1, H, dh).transpose(1, 2) for t in (q, k, v))
    s = (qh @ kh.transpose(-1, -2)) * scale
    if causal:
        s = s.masked_fill(torch.ones(N, M, dtype=torch.bool, device=q.device).triu(1), float("-inf"))
    lse = torch.logsumexp(s, -1)
    p = torch.exp(s - lse[..., None])
    return (p @ vh).transpose(1, 2).reshape(B, N, C), lse, p


def _attn_ref_bwd(q, k, v, o, do, p, H, scale):
    B, N, C = q.shape
    dh = C // H
    qh, kh, vh, oh, doh = (t.reshape(B, -1, H, dh).transpose(1, 2) for t in (q, k, v, o, do))
    dp = doh @ vh.transpose(-1, -2)
    ds = p * (dp - (doh * oh).sum(-1, keepdim=True))
    dq = (ds @ kh) * scale
    dk = (ds.transpose(-1, -2) @ qh) * scale
    dv = p.transpose(-1, -2) @ doh
    return tuple(t.transpose(1, 2).reshape(B, -1, C) for t in (dq, dk, dv))


def _attn_chunks(B, N, M, H):
    per = max(1, int(2 ** 28 // max(1, H * N * M)))        # <= 2 GiB of fp64 scores per chunk
    return [(i, min(B, i + per)) for i in range(0, B, per)]


def _attn_scale(c, C, H):
    return (C // H) ** -0.5 if c["scale"] is None else c["scale"]


def h_attn_fwd(c, causal=False):
    q, k, v, H = c["q"], c["k"], c["v"], c["heads"]
    B, N, C = q.shape
    M = k.shape[1]
    scale = _attn_scale(c, C, H)
    causal = causal or bool(c.kw.get("causal", False))
    o_ref = torch.empty(B, N, C, dtype=F64, device="cuda")
    lse_ref = torch.empty(B, H, N, dtype=F64, device="cuda")
    for i, j in _attn_chunks(B, N, M, H):
        o_ref[i:j], lse_ref[i:j], _ = _attn_ref_fwd(_d(q[i:j]), _d(k[i:j]), _d(v[i:j]), H, scale, causal)
    o, lse = c.run()
    dh = C // H
    lse_err = (lse.double() - lse_ref).abs().max().item()
    assert lse_err < 2e-2, f"lse max abs error {lse_err:.2e}"
    return [Check("o", o, o_ref, 6e-3, block=(64, dh), unit="(image * N / 64 + query block, head)")]


def h_attn_bwd(c):
    q, k, v, H = c["q"], c["k"], c["v"], c["heads"]
    B, N, C = q.shape
    M = k.shape[1]
    dh = C // H
    scale = _attn_scale(c, C, H)
    causal = bool(c["causal"])
    for n in ("dq", "dk", "dv"):
        c.nan_(n)
    refs = [torch.empty(t.shape, dtype=F64, device="cuda") for t in (q, k, v)]
    for i, j in _attn_chunks(B, N, M, H):
        qd, kd, vd = _d(q[i:j]), _d(k[i:j]), _d(v[i:j])
        o, lse, p = _attn_ref_fwd(qd, kd, vd, H, scale, causal)
        c["o"][i:j].copy_(o)
        c["lse"][i:j].copy_(lse)
        o16 = _d(c["o"][i:j])            # the kernel sees bf16 O
        gq, gk, gv = _attn_ref_bwd(qd, kd, vd, o16, _d(c["do"][i:j]), p, H, scale)
        refs[0][i:j], refs[1][i:j], refs[2][i:j] = gq, gk, gv
        del o, lse, p
    dq, dk, dv = c.run()
    return [Check(n, t, r, 1e-2, block=(64, dh), unit="(image * tokens / 64 + token block, head)")
            for n, t, r in zip(("dq", "dk", "dv"), (dq, dk, dv), refs)]


def h_attn_small_fwd(c):
    return h_attn_fwd(c)


def h_colsum_acc(c):
    x2, out, rpg = _d(c["x2"]), c["out"], c["rows_per_group"]
    init = _d(out).clone()
    M, N = x2.shape
    if rpg <= 0:
        ref = init.view(-1, N) + x2.sum(0)
    else:
        ref = init.view(-1, N) + x2.view(-1, rpg, N).sum(1)
    c.run()
    return [Check("out", out, ref.view(out.shape), 2e-3, block=(1, 64))]


def h_embedding_grad(c):
    ids, out = c["ids"], c["out"]
    V = out.shape[0]
    r = torch.randint(0, V, ids.shape, generator=c.g, device="cuda")
    r[torch.rand(ids.shape, generator=c.g, device="cuda") < 0.6] = V - 1      # the pad / EOS id dominates
    ids.copy_(r)
    D = out.shape[1]
    init = _d(out).clone()
    ref = init.index_add(0, ids.reshape(-1), _d(c["dx"]).reshape(-1, D))
    c.run()
    # rows: each table row is an fp32 sum in position order, so its error scales with the row (the pad / EOS row sums
    # ~740 positions and is ~27x the table's RMS); it is held to the bound relative to its own magnitude
    return [Check("out", out, ref, 1e-6, block=(1, D), per_block_rms=True)]


HANDLERS = {n[2:]: f for n, f in globals().items() if n.startswith("h_") and callable(f)}


# ---------------------------------------------------------------------------------------------------------------------
# the tests
# ---------------------------------------------------------------------------------------------------------------------
def describe(key):
    parts = []
    for n, sp in key[1]:
        if sp[0] == "T":
            parts.append(f"{n}={sp[3]}{list(sp[1])}" + (f"/s{list(sp[2])}" if sp[2] != _contig(sp[1]) else "")
                         + (f"+{sp[4]}" if sp[4] else ""))
        elif sp[0] == "L":
            parts.append(f"{n}=[{len(sp[1])} tensors]")
        elif sp[1] is not None and sp[1] is not False:
            parts.append(f"{n}={sp[1]}")
    return f"{key[0]}({', '.join(parts)})"


def _contig(shape):
    st, acc = [], 1
    for s in reversed(shape):
        st.append(acc)
        acc *= s
    return tuple(reversed(st))


def replay(key, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    c = Call(key, g)
    checks = HANDLERS[key[0]](c)
    results = []
    bad_guards = c.guards_intact()
    for chk in checks:
        finite, glob, worst, where = evaluate(chk)
        results.append((chk, finite, glob, worst, where))
    del c
    return results, bad_guards


@pytest.mark.parametrize("op", REQUIRED)
def test_replay_every_recorded_call(inventory, op):
    keys = [k for k in inventory if k[0] == op]
    assert keys, f"no recorded call of {op}"
    t0 = time.time()
    failures, worst_g, worst_b = [], 0.0, 0.0
    for i, key in enumerate(keys):
        results, bad_guards = replay(key, 1000 + i)
        sig = describe(key)
        if bad_guards:
            failures.append(f"{sig}: wrote outside the logical extent of {bad_guards}")
        for chk, finite, glob, worst, where in results:
            worst_g, worst_b = max(worst_g, glob / chk.bound), max(worst_b, worst / chk.bound)
            if not finite:
                failures.append(f"{sig}: {chk.label} has non-finite elements (unwritten or poisoned by a NaN read)")
            elif glob > chk.bound or worst > LOCAL * chk.bound:
                failures.append(f"{sig}: {chk.label} error {glob:.2e} (bound {chk.bound:.1e}); worst {chk.unit} "
                                f"at {where}: {worst:.2e} (bound {LOCAL * chk.bound:.1e})")
        _free()
    print(f"[replay {op}] {len(keys)} signatures; worst global error {worst_g:.2f}x its bound, worst block "
          f"{worst_b:.2f}x the global bound ({time.time() - t0:.0f} s)")
    assert not failures, "\n".join(failures)


# ---------------------------------------------------------------------------------------------------------------------
# the attention and softmax signatures again, at peaked scores
# ---------------------------------------------------------------------------------------------------------------------
PEAKED_OPS = ("attn_fwd", "attn_bwd", "attn_small_fwd", "attn_small_bwd", "softmax_rows")


def _refill_peaked(c, g):
    """q / k of an attention call (or the fp32 scores of a softmax_rows call) refilled by the peaked-score generator of
    test_attention_numerics_gpu.py, the sink keys' V rows zeroed; returns a line with the Δ / σ reached."""
    import test_attention_numerics_gpu as AN
    if c.name == "softmax_rows":
        # the rows spread over 9 generator slots: every (Δ, σ) pair of the generator's cycles
        x = c["x"]
        n = x.shape[-1]
        x2 = x.view(-1, n) if x.dim() > 2 else x
        rows, slots, dh = x2.shape[0], 9, 64
        per = -(-rows // slots)
        q, k, peaked, sinks = AN.peaked_qk(slots, per, n, 1, dh, dh ** -0.5, g)
        q, k = q.to(torch.bfloat16), k.to(torch.bfloat16)
        x2.copy_(((q.double() @ k.double().transpose(1, 2)) * dh ** -0.5).reshape(-1, n)[:rows])
        dmin, sig = AN.achieved(q, k, 1, dh ** -0.5, peaked, sinks)
        return f"Δ ≥ {dmin:.1f} nats, flat-row σ {sig[0]:.2f} to {sig[1]:.2f}"
    q, k, v, heads = c["q"], c["k"], c["v"], c["heads"]
    B, N, C = q.shape
    M = k.shape[1]
    dh = C // heads
    scale = _attn_scale(c, C, heads)
    qg, kg, peaked, sinks = AN.peaked_qk(B, N, M, heads, dh, scale, g)
    q.copy_(qg)
    k.copy_(kg)
    for i, j in enumerate(sinks):
        b, h = divmod(i, heads)
        v[b, j, h * dh:(h + 1) * dh] = 0
    dmin, sig = AN.achieved(q, k, heads, scale, peaked, sinks, bool(c.kw.get("causal", False)))
    return f"Δ ≥ {dmin:.1f} nats, flat-row σ {sig[0]:.2f} to {sig[1]:.2f}"


def _peaked_attention(c, sig, failures):
    """Runs one attention call against test_attention_numerics_gpu.reference: O elementwise and the LSE per row to
    their derived bounds (forward), the per-row gradient bound (backward), plus the replay's tensor and block bounds."""
    import test_attention_numerics_gpu as AN
    q, k, v, heads = c["q"], c["k"], c["v"], c["heads"]
    B, N, C = q.shape
    dh = C // heads
    scale = _attn_scale(c, C, heads)
    causal = bool(c.kw.get("causal", False))
    bwd = c.name in ("attn_bwd", "attn_small_bwd")
    refs, (o_bound, lse_bound), noise = AN.reference(q, k, v, c["do"] if bwd else None, heads, scale, causal)
    checks, rows = [], []
    if bwd:
        c["o"].copy_(refs[0])
        c["lse"].copy_(refs[1])
        for n in ("dq", "dk", "dv"):
            c.nan_(n)
        got = c.run()
        for n, t, r in zip(("dq", "dk", "dv"), got, refs[2:]):
            checks.append(Check(n, t, r, 1e-2, block=(64, dh), unit="(image * tokens / 64 + token block, head)"))
            rw, nrows, at = AN.row_error(t, r, heads, noise[n], 1e-2)
            rows.append((n, rw / 1e-2, f"{n}: worst row {rw / 1e-2:.2f}x over the {nrows} of {t.numel() // dh} rows "
                                       f"above their noise (at {at})"))
            if rw > LOCAL * 1e-2:
                failures.append(f"{sig}: {n} row (token, head) {at} error {rw:.2e} (bound {LOCAL * 1e-2:.1e})")
    else:
        o, lse = c.run()
        checks.append(Check("o", o, refs[0], 6e-3, block=(64, dh), unit="(image * N / 64 + query block, head)"))
        for n, t, r, bnd in (("o elementwise", o, refs[0], o_bound), ("lse per row", lse, refs[1], lse_bound)):
            w, _ = AN.elementwise(t, r, bnd)
            rows.append((n, w, f"{n}: worst {w:.2f}x its derived bound"))
            if w > 1:
                failures.append(f"{sig}: {n} {w:.2f}x its derived bound")
    return checks, rows


def test_replay_attention_peaked(inventory):
    """Every recorded attention and softmax_rows signature with q / k (or the scores) from the peaked-score generator:
    sinks Δ = 8 / 24 / 48 nats above the row, other logits spread by σ = 1 / 3 / 6 nats, half the query rows flat, the
    sinks' V rows zero.  The replay's bounds, plus O elementwise and the LSE per row to derived bounds, and each query
    row of dQ and key row of dK / dV within 4x the bound of its own fp64 RMS where its derived noise allows
    (test_attention_numerics_gpu.py)."""
    keys = [k for k in inventory if k[0] in PEAKED_OPS]
    assert {k[0] for k in keys} >= {"attn_fwd", "attn_bwd", "attn_small_fwd", "softmax_rows"}
    failures, worst = [], {}
    for i, key in enumerate(keys):
        g = torch.Generator(device="cuda").manual_seed(5000 + i)
        c = Call(key, g)
        reached = _refill_peaked(c, g)
        sig = describe(key)
        if key[0] == "softmax_rows":        # (its handler would redraw the scores)
            if c["out"] is not None:
                c.nan_("out")
            checks, rows = [Check("out", c.run(), torch.softmax(_d(c["x"]), -1), 4e-3)], []
        else:
            checks, rows = _peaked_attention(c, sig, failures)
        bad = c.guards_intact()
        if bad:
            failures.append(f"{sig}: wrote outside the logical extent of {bad}")
        line = [reached]
        for chk in checks:
            finite, glob, wb, where = evaluate(chk)
            w = worst.setdefault((key[0], chk.label), [0.0, 0.0])
            w[0], w[1] = max(w[0], glob / chk.bound), max(w[1], wb / chk.bound)
            line.append(f"{chk.label}: global {glob / chk.bound:.2f}x, block {wb / chk.bound:.2f}x")
            if not finite:
                failures.append(f"{sig}: {chk.label} has non-finite elements")
            elif glob > chk.bound or wb > LOCAL * chk.bound:
                failures.append(f"{sig}: {chk.label} error {glob:.2e} (bound {chk.bound:.1e}); worst {chk.unit} "
                                f"at {where}: {wb:.2e} (bound {LOCAL * chk.bound:.1e})")
        for n, r, text in rows:
            w = worst.setdefault((key[0], n), [0.0, 0.0])
            w[1] = max(w[1], r)
            line.append(text)
        print(f"[peaked {sig}] " + "; ".join(line))
        del c
        _free()
    for (op, label), (gw, bw) in sorted(worst.items()):
        print(f"[peaked replay {op} {label}] worst " + (f"global {gw:.2f}x, block / row / element {bw:.2f}x" if gw
                                                        else f"{bw:.2f}x") + " the bound")
    assert not failures, "\n".join(failures)
