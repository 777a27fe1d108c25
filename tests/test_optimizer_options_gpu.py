"""The optimiser flags of pretrain_e4t.py / tuning_e4t.py on the device: --lr_scheduler / --lr_warmup_steps evaluated
by the optimiser launch from the device step counter (so CUDA-graph replays follow the schedule), and --use_8bit_adam as
the block-wise 8-bit AdamW (DESIGN.md, "Optimiser options"), each against an fp64 restatement, inside the graphed
TuningStep against the oracle, through a checkpoint round trip, and their refusals."""
import math

import pytest
import torch

from oracle import e4t_oracle as O

pytestmark = pytest.mark.gpu

F64 = torch.float64
BLOCK = 256


@pytest.fixture(scope="module", autouse=True)
def _keep_direct_grad_write():
    """FlatAdamW sets functional.DIRECT_GRAD_WRITE for the whole process; put it back after this file."""
    from e4t_b200 import functional as FN
    saved = FN.DIRECT_GRAD_WRITE
    yield
    FN.DIRECT_GRAD_WRITE = saved


def _f32(x):
    """The kernels take their scalars as fp32: the restatements use the same values."""
    return float(torch.tensor(x, dtype=torch.float32))


def _sched(name, W, T, lr=1e-3):
    from e4t_b200 import optim
    kind = optim.check_schedule(name, W, T, lr)
    return (kind, W, T or 0, optim.NUM_CYCLES.get(name, 0.0), optim.POWER, optim.LR_END)


def _host_lr(name, t, W, T, lr):
    from e4t_b200 import optim
    return lr * optim.lr_lambda(name, t, W, T, lr)


# ---- fp64 restatements -----------------------------------------------------------------------------------------------
def _adamw_ref(p, g, m, v, lr, b1, b2, eps, wd, t, gs):
    """fp64 AdamW step (torch.optim.AdamW, amsgrad=False); also returns the Adam update it subtracted."""
    g = g * gs
    p = p * (1 - lr * wd)
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    upd = (lr / (1 - b1 ** t)) * m / (v.sqrt() / math.sqrt(1 - b2 ** t) + eps)
    return p - upd, m, v, upd


def _nearest(x, q):
    """Index of the map entry nearest to each x (fp64 distances, ties to the lower index)."""
    hi = torch.searchsorted(q, x.contiguous()).clamp(1, q.numel() - 1)
    lo = hi - 1
    return torch.where((x - q[hi]).abs() < (x - q[lo]).abs(), hi, lo)


def adamw8bit_ref(p, g, mc, vc, ma, va, qm, qv, lr, b1, b2, eps, wd, t, gs):
    """The block-wise 8-bit AdamW step in fp64: decode m, v with the old absmax; AdamW on the decoded moments; the new
    block absmax of |m| and v; codes = nearest map entry of m / absmax_m and v / absmax_v (ties to the lower index, an
    all-zero block codes 0).  Returns p, codes, absmax, and the normalised moments and Adam update for the checks."""
    m = (qm[mc.long()].view(-1, BLOCK) * ma[:, None]).reshape(-1)
    v = (qv[vc.long()].view(-1, BLOCK) * va[:, None]).reshape(-1)
    p, m, v, upd = _adamw_ref(p, g, m, v, lr, b1, b2, eps, wd, t, gs)
    am = m.abs().view(-1, BLOCK).amax(1)
    av = v.view(-1, BLOCK).amax(1)
    xm = (m.view(-1, BLOCK) / torch.where(am > 0, am, 1.0)[:, None]).reshape(-1)
    xv = (v.view(-1, BLOCK) / torch.where(av > 0, av, 1.0)[:, None]).reshape(-1)
    return dict(p=p, mc=_nearest(xm, qm), vc=_nearest(xv, qv), ma=am, va=av, xm=xm, xv=xv, upd=upd)


def _check_codes(got, want, x, q, what):
    """Codes equal, except where x's fp64 distances to two neighbouring map entries tie to 1e-6."""
    got, want = got.long(), want.long()
    bad = got != want
    if bool(bad.any()):
        xb, gb, wb = x[bad], got[bad], want[bad]
        tie = ((gb - wb).abs() == 1) & (((xb - q[gb]).abs() - (xb - q[wb]).abs()).abs() <= 1e-6)
        assert bool(tie.all()), (f"{what}: {int((~tie).sum())} codes differ beyond a tie, e.g. x {xb[~tie][:4].tolist()} "
                                 f"got {gb[~tie][:4].tolist()} want {wb[~tie][:4].tolist()}")
    return int(bad.sum())


def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return ((a - b).norm() / (b.norm() + 1e-300)).item()


# ---- 1. the schedule inside a replayed graph ---------------------------------------------------------------------
@pytest.mark.parametrize("bits", [32, 8])
@pytest.mark.parametrize("name", ["constant", "constant_with_warmup", "linear", "cosine", "cosine_with_restarts",
                                  "polynomial"])
def test_graph_replays_follow_the_schedule(name, bits):
    from e4t_b200.engine import FlatAdamW
    lr, W, T = 3e-4, 7, 50
    prm = torch.nn.Parameter(torch.randn(4096, device="cuda"))
    opt = FlatAdamW([prm], lr=lr, lr_scheduler=name, lr_warmup_steps=W, max_train_steps=T, optim_bits=bits)
    opt.grad.normal_()
    opt.step()                                   # loads the kernels outside the capture
    torch.cuda.synchronize()
    opt.step_dev.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        opt.step()
    for k in range(1, 61):
        graph.replay()
        got = opt.lr_dev.item()
        want = _host_lr(name, k - 1, W, T, lr)
        assert abs(got - want) <= 1e-6 * abs(want) + 1e-30, (k, got, want)
        assert int(opt.step_dev.item()) == k
        assert math.isclose(opt.get_last_lr()[0], _host_lr(name, k, W, T, lr), rel_tol=1e-12, abs_tol=1e-30)
    assert torch.isfinite(opt.arena).all()


# ---- 2. scheduled fp32 AdamW against fp64 --------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["constant", "constant_with_warmup", "linear", "cosine", "cosine_with_restarts",
                                  "polynomial"])
def test_scheduled_adamw_vs_fp64(name):
    from e4t_b200 import ops
    gen = torch.Generator(device="cuda").manual_seed(11)
    n, lr, W, T = (1 << 22) + 3, 1e-3, 2, 4
    b1, b2, eps, wd, gs = 0.9, 0.999, 1e-8, 1e-2, 0.5
    p = torch.randn(n, device="cuda", generator=gen)
    m = torch.randn(n, device="cuda", generator=gen) * 0.1
    v = torch.rand(n, device="cuda", generator=gen) * 1e-2
    step_dev = torch.zeros(1, device="cuda", dtype=torch.int32)
    lr_dev = torch.zeros(1, device="cuda")
    # a seeded sample that always holds the first and last 4-float vector blocks and the tail (as h_adamw_step_dev)
    head = torch.arange(min(n, 4096), device="cuda")
    tail = torch.arange(max(0, n - 4099), n, device="cuda")
    mid = torch.randint(0, n, (1 << 20,), generator=gen, device="cuda")
    idx = torch.cat([head, mid, tail]).unique()
    for k in range(1, 6):
        g = torch.randn(n, device="cuda", generator=gen)
        before = [t[idx].double() for t in (p, g, m, v)]
        lr_k = _host_lr(name, k - 1, W, T, lr)
        pr, mr, vr, _ = _adamw_ref(*before, _f32(lr_k), _f32(b1), _f32(b2), _f32(eps), _f32(wd), k, gs)
        ops.adamw_step_sched(p, g, m, v, lr, b1, b2, eps, wd, step_dev, lr_dev, _sched(name, W, T, lr), gs)
        torch.cuda.synchronize()
        assert int(step_dev.item()) == k
        assert abs(lr_dev.item() - lr_k) <= 1e-6 * lr_k + 1e-30
        for what, got, want in (("p", p, pr), ("m", m, mr), ("v", v, vr)):
            assert _rel(got[idx], want) <= 1e-5, (name, k, what, _rel(got[idx], want))


# ---- 3. the 8-bit kernel against its fp64 restatement -------------------------------------------------------------
def test_adamw8bit_kernel_vs_fp64_restatement():
    from e4t_b200 import ops, optim
    gen = torch.Generator(device="cuda").manual_seed(12)
    nb = 3 * 4096                                         # 12288 blocks, 3.1 M elements
    n = nb * BLOCK
    lr, W, T = 1e-3, 1, 8
    b1, b2, eps, wd, gs = 0.9, 0.999, 1e-8, 1e-2, 1.0
    qm, qv = optim.dynamic_map(True).cuda(), optim.dynamic_map(False).cuda()
    qm64, qv64 = qm.double(), qv.double()
    p = torch.randn(n, device="cuda", generator=gen)
    mc = torch.zeros(n, device="cuda", dtype=torch.uint8)
    vc = torch.zeros(n, device="cuda", dtype=torch.uint8)
    ma = torch.zeros(nb, device="cuda")
    va = torch.zeros(nb, device="cuda")
    step_dev = torch.zeros(1, device="cuda", dtype=torch.int32)
    lr_dev = torch.zeros(1, device="cuda")
    # per-block gradient scales 1e-8 .. 1e2; every 16th block all zero; every 16th (offset 8) spans 1e-8 .. 1e2 inside
    scale = 10.0 ** (torch.rand(nb, device="cuda", generator=gen) * 10 - 8)
    zero = torch.arange(nb, device="cuda") % 16 == 0
    mixed = torch.arange(nb, device="cuda") % 16 == 8
    ties = 0
    for k in range(1, 6):
        g = torch.randn(nb, BLOCK, device="cuda", generator=gen) * scale[:, None]
        inner = 10.0 ** (torch.rand(nb, BLOCK, device="cuda", generator=gen) * 10 - 8)
        g = torch.where(mixed[:, None], torch.randn(nb, BLOCK, device="cuda", generator=gen) * inner, g)
        g = torch.where(zero[:, None], 0.0, g).reshape(-1).contiguous()
        lr_k = _host_lr("linear", k - 1, W, T, lr)
        ref = adamw8bit_ref(p.double(), g.double(), mc, vc, ma.double(), va.double(), qm64, qv64, _f32(lr_k),
                            _f32(b1), _f32(b2), _f32(eps), _f32(wd), k, gs)
        ops.adamw8bit_step_sched(p, g, mc, vc, ma, va, qm, qv, lr, b1, b2, eps, wd, step_dev, lr_dev,
                                 _sched("linear", W, T, lr), gs)
        torch.cuda.synchronize()
        for t in (p, ma, va):
            assert torch.isfinite(t).all()
        assert bool((ma[zero] == 0).all() and (va[zero] == 0).all())
        assert bool((mc.view(nb, BLOCK)[zero] == 127).all() and (vc.view(nb, BLOCK)[zero] == 0).all())
        for what, got, want in (("absmax m", ma, ref["ma"]), ("absmax v", va, ref["va"])):
            err = ((got.double() - want).abs() / want.abs().clamp_min(1e-300)).where(want != 0, got.double().abs())
            assert err.max().item() <= 1e-6, (k, what, err.max().item())
        ties += _check_codes(mc, ref["mc"], ref["xm"], qm64, f"step {k} m codes")
        ties += _check_codes(vc, ref["vc"], ref["xv"], qv64, f"step {k} v codes")
        # p: 1e-5 relative; the kernel's fp32 bias corrections (powf of beta near 1) move the Adam update by up to 1e-4
        tol = 1e-5 * ref["p"].abs() + 1e-4 * ref["upd"].abs() + 1e-30
        err = (p.double() - ref["p"]).abs()
        assert bool((err <= tol).all()), (k, (err / tol).max().item())
        assert _rel(p, ref["p"]) <= 1e-5
    print(f"[8-bit adamw] {n} elements x 5 steps: {ties} codes on fp64 ties")


# ---- 4. determinism: graph replays == eager calls, bit for bit ------------------------------------------------------
@pytest.mark.parametrize("bits", [32, 8])
def test_graph_replays_equal_eager_calls_bitwise(bits):
    from e4t_b200.engine import FlatAdamW
    gen = torch.Generator(device="cuda").manual_seed(13)
    x = torch.randn(1 << 20, device="cuda", generator=gen)
    y = torch.randn(5000, device="cuda", generator=gen)
    G = torch.randn(x.numel() + y.numel() + 2 * BLOCK, device="cuda", generator=gen)
    kw = dict(lr=1e-3, lr_scheduler="cosine", lr_warmup_steps=1, max_train_steps=6, optim_bits=bits)
    A = FlatAdamW([torch.nn.Parameter(x.clone()), torch.nn.Parameter(y.clone())], **kw)
    B = FlatAdamW([torch.nn.Parameter(x.clone()), torch.nn.Parameter(y.clone())], **kw)
    for o in (A, B):
        o.grad.copy_(G[:o.numel])
    A.step()                                     # loads the kernels outside the capture; B takes the same first step
    B.step()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        A.step()
    for _ in range(4):
        graph.replay()
        B.step()
    torch.cuda.synchronize()
    names = ("arena", "step_dev", "lr_dev") + (("m_codes", "v_codes", "m_absmax", "v_absmax") if bits == 8
                                              else ("exp_avg", "exp_avg_sq"))
    for k in names:
        assert torch.equal(getattr(A, k), getattr(B, k)), k
    assert int(A.step_dev.item()) == 5


# ---- 5. the graphed TuningStep against the oracle -------------------------------------------------------------------
def _tiny_models(seed=21):
    from e4t.encoder import E4TEncoder
    from e4t.models.modeling_clip import CLIPTextConfig, CLIPTextModel
    from e4t.models.unet_2d_condition import UNet2DConditionModel
    ucfg, vcfg, tcfg = O.TINY_UNET, O.VIT_TINY, O.CLIP_TEXT_TINY
    fd = O.pooled_feature_dim(ucfg)
    sd_u = O.synth_state_dict(O.unet_param_shapes(ucfg), seed)
    sd_e = O.synth_state_dict(O.encoder_param_shapes(vcfg, fd, tcfg["width"], 129), seed + 1)
    sd_t = O.synth_state_dict(O.text_param_shapes(tcfg), seed + 2)
    unet = UNet2DConditionModel(**O.ref_unet_kwargs(ucfg)); unet.load_state_dict(sd_u)
    enc = E4TEncoder(arch="ViT-tiny-test", word_embedding_dim=tcfg["width"], n_odd_layers=129, unet_feature_dim=fd)
    enc.load_state_dict(sd_e)
    text = CLIPTextModel(CLIPTextConfig(vocab_size=tcfg["vocab"], hidden_size=tcfg["width"],
                                        intermediate_size=tcfg["mlp"], num_hidden_layers=tcfg["layers"],
                                        num_attention_heads=tcfg["heads"]))
    text.load_state_dict(sd_t)
    return (unet.cuda(), enc.cuda(), text.cuda()), (sd_u, sd_e, sd_t)


def _batches(step, n):
    """test_tuning_step_tiny_vs_oracle_adamw_with_clipping's inputs: one image batch, re-noised every step."""
    base = O.synth_batch(2, seed=77, latent_hw=16, image_hw=64)
    out = []
    for it in range(n):
        gen = torch.Generator().manual_seed(900 + it)
        out.append(dict(base, noise=torch.randn(base["latents"].shape, generator=gen),
                        timesteps=torch.randint(0, 1000, (2,), generator=gen)))
    idx = torch.tensor(step.placeholder_idxs(out[0]["input_ids"]), device="cuda")
    dev = [dict({k: v.cuda() for k, v in b.items()}, placeholder_idxs=idx) for b in out]
    return out, dev


@pytest.mark.parametrize("option", ["cosine", "8bit"])
def test_graphed_tuning_step_tiny_vs_oracle(option):
    from e4t_b200 import optim
    from e4t_b200.engine import TuningStep
    (unet, enc, text), (sd_u, sd_e, sd_t) = _tiny_models()
    lr, W, T = 2e-4, 2, 5
    kw = dict(lr_scheduler="cosine", lr_warmup_steps=W, max_train_steps=T) if option == "cosine" else \
        dict(use_8bit_adam=True)
    step = TuningStep(unet, enc, text, O.PLACEHOLDER_ID, class_token_id=320, lr=lr, weight_dtype=torch.float32, **kw)
    keys = [k for k in sd_u] + [k for k in sd_e if not k.startswith("clip_vision.")]
    plist = [sd_u[k].requires_grad_(True) for k in sd_u] + [sd_e[k].requires_grad_(True) for k in sd_e
                                                            if not k.startswith("clip_vision.")]
    named = dict(unet.named_parameters())
    named.update(dict(enc.named_parameters()))
    b1, b2, eps, wd = 0.9, 0.999, 1e-8, 1e-2
    if option == "cosine":
        opt = torch.optim.AdamW(plist, lr=lr, betas=(b1, b2), weight_decay=wd, eps=eps)
        sch = torch.optim.lr_scheduler.LambdaLR(opt, lambda t: optim.lr_lambda("cosine", t, W, T, lr))
    else:
        # the restatement's arena is the device arena: same offsets, so its blocks hold the same elements
        offs = [step.opt.offsets[id(named[k])] for k in keys]
        N, nb = step.opt.numel, step.opt.numel // BLOCK
        st = dict(mc=torch.zeros(N, dtype=torch.uint8), vc=torch.zeros(N, dtype=torch.uint8),
                  ma=torch.zeros(nb, dtype=F64), va=torch.zeros(nb, dtype=F64))
        qm64, qv64 = optim.dynamic_map(True).double(), optim.dynamic_map(False).double()
    host, dev = _batches(step, 6)
    step.enable_cuda_graph(dev[0], warmup=1)      # one real optimiser step on batch 0, then capture
    lo, lg = [], []
    for it in range(6):
        ref = O.pretrain_step(sd_u, O.TINY_UNET, sd_e, O.VIT_TINY, sd_t, O.CLIP_TEXT_TINY, host[it],
                              class_token_id=320, reg_lambda=1e-4)
        for prm in plist:
            prm.grad = None
        ref["loss"].backward()
        torch.nn.utils.clip_grad_norm_(plist, 1.0)
        if option == "cosine":
            opt.step()
            sch.step()
        else:
            P = torch.zeros(N, dtype=F64)
            G = torch.zeros(N, dtype=F64)
            for prm, (o, n) in zip(plist, offs):
                P[o:o + n] = prm.detach().reshape(-1).double()
                G[o:o + n] = prm.grad.reshape(-1).double()
            r = adamw8bit_ref(P, G, st["mc"], st["vc"], st["ma"], st["va"], qm64, qv64, _f32(lr), _f32(b1), _f32(b2),
                              _f32(eps), _f32(wd), it + 1, 1.0)
            st = dict(mc=r["mc"].to(torch.uint8), vc=r["vc"].to(torch.uint8), ma=r["ma"], va=r["va"])
            with torch.no_grad():
                for prm, (o, n) in zip(plist, offs):
                    prm.copy_(r["p"][o:o + n].view_as(prm))
        if it > 0:                                 # steps 2..6 are graph replays
            out = step(dev[it])
            lo.append(ref["loss"].item()); lg.append(out["loss"].item())
    assert int(step.opt.step_dev.item()) == 6
    print(f"[graphed tuning step, {option}] oracle", [round(v, 5) for v in lo], "cuda", [round(v, 5) for v in lg])
    for a, b in zip(lo, lg):
        assert abs(a - b) <= 3e-2 * abs(a) + 1e-4, (lo, lg)
    if option == "cosine":
        assert math.isclose(step.opt.get_last_lr()[0], sch.get_last_lr()[0], rel_tol=1e-12, abs_tol=1e-30)


# ---- 6. checkpoint round trip after graphed steps ---------------------------------------------------------------------
def test_8bit_scheduled_state_dict_after_graphed_steps_resumes_bitwise():
    from e4t_b200 import optim
    from e4t_b200.engine import TuningStep
    kw = dict(class_token_id=320, lr=2e-4, weight_dtype=torch.float32, use_8bit_adam=True, lr_scheduler="cosine",
              lr_warmup_steps=2, max_train_steps=10)
    (ua, ea, ta), _ = _tiny_models(31)
    A = TuningStep(ua, ea, ta, O.PLACEHOLDER_ID, **kw)
    _, dev = _batches(A, 4)
    A.enable_cuda_graph(dev[0], warmup=1)
    for it in range(1, 4):
        A(dev[it])
    sd = A.opt.state_dict()
    assert sd["step"] == 4                                   # enable_cuda_graph's warm-up step + 3 replays
    assert sd["optim_bits"] == 8 and sd["lr_scheduler"] == "cosine"
    params = A.opt.arena.clone()
    # the next step from a fixed gradient (the forward / backward's split-K atomics are not bit-reproducible)
    G = torch.randn(A.opt.numel, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5)) * 1e-3
    A.opt.grad.copy_(G)
    A.opt.step()
    (ub, eb, tb), _ = _tiny_models(31)
    Bs = TuningStep(ub, eb, tb, O.PLACEHOLDER_ID, **dict(kw, lr_scheduler="constant", max_train_steps=None))
    Bs.opt.arena.copy_(params)
    Bs.opt.load_state_dict(sd)
    assert Bs.opt.lr_scheduler == "cosine" and Bs.opt.max_train_steps == 10
    assert math.isclose(Bs.opt.get_last_lr()[0], 2e-4 * optim.lr_lambda("cosine", 4, 2, 10, 2e-4), rel_tol=1e-12)
    Bs.opt.grad.copy_(G)
    Bs.opt.step()
    torch.cuda.synchronize()
    for k in ("arena", "m_codes", "v_codes", "m_absmax", "v_absmax", "step_dev", "lr_dev"):
        assert torch.equal(getattr(A.opt, k), getattr(Bs.opt, k)), k
    A.release_cuda_graph()


# ---- 7. memory of the 8-bit state ---------------------------------------------------------------------------------
def test_8bit_state_has_no_fp32_moments():
    from e4t_b200.engine import TuningStep
    (unet, enc, text), _ = _tiny_models(41)
    step = TuningStep(unet, enc, text, O.PLACEHOLDER_ID, class_token_id=320, lr=2e-4, weight_dtype=torch.float32,
                      use_8bit_adam=True)
    opt = step.opt
    n = opt.numel
    assert n % BLOCK == 0 and opt.exp_avg is None and opt.exp_avg_sq is None
    state = [opt.m_codes, opt.v_codes, opt.m_absmax, opt.v_absmax]
    assert sum(t.numel() * t.element_size() for t in state) == 2 * n + 8 * n // BLOCK
    # every parameter storage starts on a block boundary: no absmax block mixes two storages
    spans = {}
    for prm in opt.params:
        o, k = opt.offsets[id(prm)]
        lo, hi = spans.get(prm.untyped_storage().data_ptr(), (o, o + k))
        spans[prm.untyped_storage().data_ptr()] = (min(lo, o), max(hi, o + k))
    ivs = sorted(spans.values())
    assert all(lo % BLOCK == 0 for lo, _ in ivs)
    assert all(-(-a_hi // BLOCK) <= b_lo // BLOCK for (_, a_hi), (b_lo, _) in zip(ivs, ivs[1:]))


# ---- 8. refusals -------------------------------------------------------------------------------------------------------
def test_refusals():
    from e4t_b200 import ops, optim
    from e4t_b200._lib import E4TError
    from e4t_b200.engine import FlatAdamW, PretrainStep
    with pytest.raises(ValueError, match="constant, constant_with_warmup, linear, cosine, cosine_with_restarts"):
        PretrainStep(None, None, None, 0, 0, lr_scheduler="warmup_cosine")
    with pytest.raises(ValueError, match="needs max_train_steps"):
        PretrainStep(None, None, None, 0, 0, lr_scheduler="cosine", lr_warmup_steps=10)
    with pytest.raises(ValueError, match="must be smaller than the initial lr"):
        FlatAdamW([torch.nn.Parameter(torch.zeros(8, device="cuda"))], lr=1e-8, lr_scheduler="polynomial",
                  max_train_steps=10)
    with pytest.raises(ValueError, match="optim_bits"):
        FlatAdamW([torch.nn.Parameter(torch.zeros(8, device="cuda"))], optim_bits=16)
    o32 = FlatAdamW([torch.nn.Parameter(torch.zeros(300, device="cuda"))])
    o8 = FlatAdamW([torch.nn.Parameter(torch.zeros(300, device="cuda"))], optim_bits=8)
    with pytest.raises(ValueError, match="32-bit moments, this optimizer keeps 8-bit"):
        o8.load_state_dict(o32.state_dict())
    with pytest.raises(ValueError, match="8-bit moments, this optimizer keeps 32-bit"):
        o32.load_state_dict(o8.state_dict())
    # the C-ABI: n a multiple of 256, 16-byte aligned buffers, a known schedule
    qm, qv = optim.dynamic_map(True).cuda(), optim.dynamic_map(False).cuda()
    sd, lrd = torch.zeros(1, device="cuda", dtype=torch.int32), torch.zeros(1, device="cuda")

    def call8(n, off=0):
        buf = torch.zeros(n + 4, device="cuda")
        cb = torch.zeros(n + 16, device="cuda", dtype=torch.uint8)
        ops.adamw8bit_step_sched(buf[off:off + n], buf[off:off + n].clone() if off == 0 else buf[off:off + n],
                                 cb[:n], cb[:n].clone(), torch.zeros(n // 256, device="cuda"),
                                 torch.zeros(n // 256, device="cuda"), qm, qv, 1e-3, 0.9, 0.999, 1e-8, 0.0, sd, lrd,
                                 _sched("constant", 0, None))
    with pytest.raises(E4TError, match="is not a multiple of 256"):
        call8(1000)
    with pytest.raises(E4TError, match="16-byte aligned"):
        call8(512, off=1)
    p = torch.zeros(64, device="cuda")
    with pytest.raises(E4TError, match="unknown schedule kind"):
        ops.adamw_step_sched(p, p.clone(), p.clone(), p.clone(), 1e-3, 0.9, 0.999, 1e-8, 0.0, sd, lrd,
                             (9, 0, 10, 0.5, 1.0, 1e-7))
    with pytest.raises(E4TError, match="16-byte aligned"):
        q = torch.zeros(65, device="cuda")[1:]
        ops.adamw_step_sched(q, p, p.clone(), p.clone(), 1e-3, 0.9, 0.999, 1e-8, 0.0, sd, lrd,
                             _sched("linear", 0, 10))
    torch.cuda.synchronize()
    assert int(sd.item()) == 0                     # nothing was launched
