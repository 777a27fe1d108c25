"""Token merging (ToMe) on the sm_90a kernels: matching and selection against the rules and fp64, the gathers forward
and backward, the patched UNet, training step and sampling pipeline against the oracle (oracle/tome_oracle.py)
replaying the plans recorded from the GPU, and every refusal."""
import ctypes

import pytest
import torch

from oracle import e4t_oracle as O
from oracle import tome_oracle as T

pytestmark = pytest.mark.gpu

# Bound on |node_max - cos64| of one src/dst pair: the kernel multiplies the unit-norm rows rounded to bf16, a
# relative perturbation of at most u = 2^-9 per row, so |â·b̂ - a·b| <= 2u + u² for unit a, b; fp32 norms, products and
# sums add < 1e-5 at C <= 1280.
U = 2.0 ** -9
EPS = 2 * U + U * U + 1e-5

MATCH_SHAPES = [(16, 64, 64, 320), (2, 96, 96, 320), (2, 65, 67, 320), (3, 64, 64, 320), (2, 32, 32, 640),
                (2, 16, 16, 1280)]


def _x(B, N, C, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, N, C, generator=g).to(torch.bfloat16).cuda()


def _pattern(h, w, rand, seed=0):
    shape = (h // 2, w // 2)
    if not rand:
        return torch.zeros(shape, dtype=torch.int32, device="cuda")
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 4, shape, generator=g, dtype=torch.int32).cuda()


def _run(x, pattern, h, w, r):
    from e4t_b200 import ops
    m = ops.tome_match(x, pattern, h, w, 2, 2)
    p = ops.tome_select(m, r)
    p.update(m)
    return p


def _check_plan_against_own_node_max(p, r):
    """The selection and the CSR maps follow exactly from the kernel's node_max / node_idx and the tie rule."""
    src_idx = p["src_idx"].cpu().long()
    node_max = p["node_max"].cpu().double()
    merged = T.select(node_max, src_idx, r)
    ref = T.build_plan(p["pos"].shape[1], src_idx, p["node_idx"].cpu().long(), merged)
    for k in ("pos", "row_off", "members"):
        assert torch.equal(p[k].cpu().long(), ref[k]), k
    assert torch.equal(p["w"].cpu().double(), ref["w"].float().double())
    return merged


@pytest.mark.parametrize("rand", [True, False], ids=["rand", "zero"])
@pytest.mark.parametrize("B,h,w,C", MATCH_SHAPES)
def test_match_and_select(B, h, w, C, rand):
    N = h * w
    r = T.block_geometry(h, w, N, 0.5, 1, 2, 2)[3]
    x = _x(B, N, C, seed=B * 1000 + h + C)
    pattern = _pattern(h, w, rand, seed=h * w)
    p = _run(x, pattern, h, w, r)
    src_idx, dst_idx = T.partition(h, w, 2, 2, pattern.cpu())
    assert torch.equal(p["src_idx"].cpu().long(), src_idx) and torch.equal(p["dst_idx"].cpu().long(), dst_idx)
    merged = _check_plan_against_own_node_max(p, r)
    # fp64: node_max is the similarity to the dst it names, and the true maximum, within EPS
    xd = x.cpu().double()
    xn = xd / xd.norm(dim=-1, keepdim=True)
    cos = xn[:, src_idx] @ xn[:, dst_idx].transpose(1, 2)                   # (B, Ns, Nd)
    true_max = cos.max(-1).values
    nm = p["node_max"].cpu().double()
    col = torch.searchsorted(dst_idx, p["node_idx"].cpu().long())
    assert torch.equal(dst_idx[col], p["node_idx"].cpu().long())
    named = cos.gather(2, col[..., None])[..., 0]
    assert (nm - named).abs().max().item() <= EPS
    assert (nm - true_max).abs().max().item() <= EPS
    # every merged token is at least as similar (fp64) as every kept src token, up to the two roundings
    for b in range(B):
        assert true_max[b][merged[b]].min().item() >= true_max[b][~merged[b]].max().item() - 2 * EPS
    # bitwise repeatable
    q = _run(x, pattern, h, w, r)
    for k in ("node_max", "node_idx", "pos", "row_off", "members", "w"):
        assert torch.equal(p[k], q[k]), k


@pytest.mark.parametrize("kind", ["duplicates", "constant"])
def test_exact_ties(kind):
    B, h, w, C = 2, 64, 64, 320
    N = h * w
    r = T.block_geometry(h, w, N, 0.5, 1, 2, 2)[3]
    g = torch.Generator().manual_seed(7)
    if kind == "constant":
        vid = torch.zeros(B, N, dtype=torch.long)
        base = torch.randn(1, C, generator=g)
    else:
        vid = torch.randint(0, 6, (B, N), generator=g)
        base = torch.randn(6, C, generator=g)
    x = base[vid].to(torch.bfloat16).cuda()
    pattern = _pattern(h, w, True, seed=3)
    p = _run(x, pattern, h, w, r)
    _check_plan_against_own_node_max(p, r)
    src_idx, dst_idx = T.partition(h, w, 2, 2, pattern.cpu())
    ni = p["node_idx"].cpu().long()
    for b in range(B):
        # the named dst is the lowest raster dst holding the same vector (identical rows give identical products)
        first = {}
        for j in dst_idx.tolist():
            first.setdefault(int(vid[b, j]), j)
        assert all(first[int(vid[b, j])] == j for j in ni[b].tolist())
    if kind == "constant":
        assert (ni == int(dst_idx[0])).all()
        merged = _check_plan_against_own_node_max(p, r)
        assert torch.equal(torch.nonzero(merged[0]).reshape(-1), torch.arange(r))
    q = _run(x, pattern, h, w, r)
    for k in ("node_max", "node_idx", "pos", "row_off", "members", "w"):
        assert torch.equal(p[k], q[k]), k


# ---- gathers ---------------------------------------------------------------------------------------------------------
def _guarded(n, dtype=torch.bfloat16, g=64):
    buf = torch.full((n + 2 * g,), float("nan"), device="cuda", dtype=dtype)
    return buf, buf[g:g + n]


def _guards_intact(buf, n, g=64):
    return buf[:g].isnan().all().item() and buf[g + n:].isnan().all().item()


@pytest.mark.parametrize("B,h,w,C", [(2, 64, 64, 320), (3, 65, 67, 640), (2, 16, 16, 1280)])
def test_merge_unmerge_forward_backward(B, h, w, C):
    from e4t_b200 import _lib, functional as FN
    from e4t_b200._lib import c_int, ptr, stream
    N = h * w
    r = T.block_geometry(h, w, N, 0.5, 1, 2, 2)[3]
    x = _x(B, N, C, seed=11)
    p = _run(x, _pattern(h, w, True, 5), h, w, r)
    plan = T.as_cpu_plan(dict(p, r=r))
    Nm = N - r
    # raw kernels into NaN-guarded buffers
    buf, out = _guarded(B * Nm * C)
    _lib.call("e4t_tome_gather_reduce", ptr(x), ptr(p["row_off"]), ptr(p["members"]), ptr(p["w"]), ptr(out), c_int(B),
              c_int(N), c_int(Nm), c_int(C), stream())
    y = out.view(B, Nm, C)
    ref_y = T.merge(x.cpu().double(), plan)
    assert _guards_intact(buf, B * Nm * C) and not y.isnan().any()
    torch.testing.assert_close(y.cpu().double(), ref_y, rtol=2 ** -8, atol=1e-6)
    res = _x(B, N, C, seed=12)
    buf2, out2 = _guarded(B * N * C)
    _lib.call("e4t_tome_gather_expand", ptr(y), ptr(p["pos"]), ctypes.c_void_p(0), ptr(res), ptr(out2), c_int(B),
              c_int(Nm), c_int(N), c_int(C), stream())
    ref_o = T.unmerge(y.cpu().double(), plan, res.cpu().double())
    assert _guards_intact(buf2, B * N * C) and not out2.isnan().any()
    torch.testing.assert_close(out2.view(B, N, C).cpu().double(), ref_o, rtol=2 ** -8, atol=1e-6)
    # autograd functions against fp64 autograd of the oracle maps
    xg = x.clone().requires_grad_(True)
    rg = res.clone().requires_grad_(True)
    o = FN.ToMeUnmergeFn.apply(FN.ToMeMergeFn.apply(xg, p) * 2, p, rg)
    dout = _x(B, N, C, seed=13)
    dx, dres = torch.autograd.grad(o, (xg, rg), dout)
    x64 = x.cpu().double().requires_grad_(True)
    r64 = res.cpu().double().requires_grad_(True)
    o64 = T.unmerge(T.merge(x64, plan) * 2, plan, r64)
    dx64, dr64 = torch.autograd.grad(o64, (x64, r64), dout.cpu().double())
    torch.testing.assert_close(dx.cpu().double(), dx64, rtol=2 ** -7, atol=1e-5)
    assert torch.equal(dres, dout)
    dx2, _ = torch.autograd.grad(FN.ToMeUnmergeFn.apply(FN.ToMeMergeFn.apply(xg, p) * 2, p, rg), (xg, rg), dout)
    assert torch.equal(dx, dx2)


# ---- patched UNet forward ----------------------------------------------------------------------------------------------
def _rel(a, b):
    a = a.detach().double().cpu(); b = b.detach().double().cpu()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt().clamp_min(1e-30)).item()


def _unet(cfg, seed):
    from e4t.models.unet_2d_condition import UNet2DConditionModel
    m = UNet2DConditionModel(**O.ref_unet_kwargs(cfg))
    sd = O.synth_state_dict(O.unet_param_shapes(cfg), seed)
    m.load_state_dict(sd, strict=True)
    return m.cuda(), sd


@pytest.mark.parametrize("name,cfg,hw", [("tiny", O.TINY_UNET, 16), ("sd14", O.SD14_UNET, 64)])
def test_patched_unet_forward_vs_oracle(name, cfg, hw):
    from e4t_b200 import tome
    m, sd = _unet(cfg, 21)
    g = torch.Generator().manual_seed(22)
    B = 2
    x = torch.randn(B, 4, hw, hw, generator=g)
    t = torch.randint(0, 1000, (B,), generator=g)
    ehs = torch.randn(B, 77, cfg["cross_attention_dim"], generator=g)
    tome.apply_patch(m, ratio=0.5)
    try:
        with torch.no_grad(), tome.record_plans(m) as rec:
            if name == "sd14":
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    out = m(x.cuda(), t.cuda(), ehs.cuda()).sample
                    torch.cuda.synchronize()
                names = [e.name for e in prof.events()]
                assert any("attn_wgmma_fwd_kernel" in n for n in names)
                assert any("tome_match_kernel" in n for n in names)
            else:
                out = m(x.cuda(), t.cuda(), ehs.cuda()).sample
        plans = [T.as_cpu_plan(p) for p in rec]
    finally:
        tome.remove_patch(m)
    n0 = hw * hw
    # level 0: the attentions of down block 0 and of the last up block
    n_blocks = cfg["layers_per_block"] + (cfg["layers_per_block"] + 1)
    assert len(plans) == n_blocks and all(pl["w"].shape == (B, n0 - n0 // 2) for pl in plans)
    ref = T.unet_forward(sd, cfg, x, t, ehs, plans=plans)
    e = _rel(out, ref)
    print(f"[{name}] patched UNet vs oracle with the recorded plans: {e:.3e}")
    assert e < 3e-2


# ---- training ----------------------------------------------------------------------------------------------------------
def _models(seed=1):
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
    return (unet.cuda(), enc.cuda(), text.cuda()), (sd_u, ucfg, sd_e, vcfg, sd_t, tcfg)


def _step(mods, **kw):
    from e4t_b200.engine import PretrainStep
    unet, enc, text = mods
    return PretrainStep(unet, enc, text, O.PLACEHOLDER_ID, class_token_id=320, lr=1e-3, weight_dtype=torch.float32,
                        **kw)


def test_training_step_vs_oracle():
    from e4t_b200 import tome
    mods, (sd_u, ucfg, sd_e, vcfg, sd_t, tcfg) = _models()
    tome.apply_patch(mods[0], ratio=0.5)
    step = _step(mods)
    enc_params = {k: p.detach().clone() for k, p in mods[1].named_parameters() if p.requires_grad}
    batch = O.synth_batch(2, seed=42, latent_hw=16, image_hw=64)
    with tome.record_plans(mods[0]) as rec:
        out = step({k: v.cuda() for k, v in batch.items()})
        torch.cuda.synchronize()
    plans = [T.as_cpu_plan(p) for p in rec]
    assert len(plans) == 4        # encoder pass: down block 0; full pass: down block 0 and the last up block's two
    sd_e_g = {k: (v.clone().requires_grad_(True) if k in enc_params else v) for k, v in sd_e.items()}
    with T.patched((16, 16), plans=plans):
        ref = O.pretrain_step(sd_u, ucfg, sd_e_g, vcfg, sd_t, tcfg, batch, class_token_id=320)
    lo, lg = ref["loss"].item(), out["loss"].item()
    print(f"ToMe pre-training step: loss {lg:.6f} vs oracle {lo:.6f}")
    assert abs(lo - lg) <= 3e-2 * abs(lo) + 1e-4
    ref["loss"].backward()
    # AdamW's first step moves each parameter by lr * g / |g| (+ decay): its sign follows the gradient where the
    # gradient is well above the bf16 noise
    agree = total = 0
    for k, p in mods[1].named_parameters():
        if k not in enc_params:
            continue
        gref = sd_e_g[k].grad
        if gref is None:
            continue
        d = (p.detach().cpu() - enc_params[k].cpu()) + 1e-3 * 1e-2 * enc_params[k].cpu()
        big = gref.abs() > gref.abs().median() * 2
        agree += (torch.sign(-d[big]) == torch.sign(gref[big])).sum().item()
        total += big.sum().item()
    assert total > 0 and agree >= 0.95 * total, (agree, total)
    tome.remove_patch(mods[0])


def test_graphed_training_matches_eager_and_redraws():
    from e4t_b200 import tome
    batch = O.synth_batch(2, seed=42, latent_hw=16, image_hw=64)
    dev = {k: v.cuda() for k, v in batch.items()}
    dev["placeholder_idxs"] = torch.tensor([row.index(O.PLACEHOLDER_ID) for row in batch["input_ids"].tolist()],
                                           device="cuda")
    losses = []
    for graphed in (False, True):
        mods, _ = _models(seed=5)
        tome.apply_patch(mods[0], ratio=0.5, use_rand=False)
        step = _step(mods)
        if graphed:
            step.enable_cuda_graph(dev, warmup=3)
            out = step(dev)
        else:
            for _ in range(3):
                step(dev)
            out = step(dev)
        losses.append(out["loss"].item())
    assert abs(losses[0] - losses[1]) <= 1e-3 * abs(losses[0]), losses
    # use_rand: every replay draws new patterns
    mods, _ = _models(seed=5)
    tome.apply_patch(mods[0], ratio=0.5, use_rand=True)
    step = _step(mods)
    with tome.record_plans(mods[0]) as rec:
        step.enable_cuda_graph(dev, warmup=1)
    captured = rec[-1]["pattern"]
    step(dev)
    torch.cuda.synchronize()
    a = captured.clone()
    step(dev)
    torch.cuda.synchronize()
    assert not torch.equal(a, captured)
    # a patch change after capture is refused
    from e4t_b200._lib import E4TError
    tome.apply_patch(mods[0], ratio=0.25)
    with pytest.raises(E4TError, match="token-merging patch changed"):
        step(dev)
    tome.remove_patch(mods[0])
    with pytest.raises(E4TError, match="token-merging patch changed"):
        step(dev)


# ---- sampling pipeline -------------------------------------------------------------------------------------------------
from test_sampling_gpu import GRAPH_VS_EAGER, _run as _sample, sd1  # noqa: E402,F401

# Two sampling runs of the same pipeline are not bitwise equal (GroupNorm statistics accumulate with atomics, see
# test_sampling_gpu.py), so "unpatched" is checked as: the same kernel launches as an unpatched run, no ToMe kernel, and
# a result as close to the unpatched one as a second unpatched run is.


def _launches(sd1, graph):
    from e4t_b200 import _lib
    _lib.reset_launch_count()
    out, _ = _sample(sd1, "ddim", "epsilon", 7.5, steps=3, graph=graph)
    torch.cuda.synchronize()
    return out, _lib.launch_count()


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_pipeline_unpatched_equivalents(sd1, graph):
    from e4t_b200 import tome
    _launches(sd1, graph)                       # capture / warm-up
    base, n_base = _launches(sd1, graph)
    again, _ = _launches(sd1, graph)
    tome.apply_patch(sd1.pipe, ratio=0.0)
    zero, n_zero = _launches(sd1, graph)
    tome.apply_patch(sd1.pipe, ratio=0.5)
    merged, _ = _launches(sd1, graph)
    merged, n_merged = _launches(sd1, graph)
    tome.remove_patch(sd1.pipe)
    _launches(sd1, graph)
    removed, n_removed = _launches(sd1, graph)
    sd1.pipe.disable_cuda_graph()
    spread = _rel(again, base)
    print(f"[{'graph' if graph else 'eager'}] unpatched rerun {spread:.2e}, ratio 0 {_rel(zero, base):.2e}, removed "
          f"{_rel(removed, base):.2e}, merged {_rel(merged, base):.2e}")
    assert n_zero == n_base and n_removed == n_base and (graph or n_merged > n_base)
    assert _rel(zero, base) < GRAPH_VS_EAGER and _rel(removed, base) < GRAPH_VS_EAGER
    assert torch.isfinite(merged).all()


def test_pipeline_patched_graph_matches_eager(sd1):
    from e4t_b200 import tome
    tome.apply_patch(sd1.pipe, ratio=0.5, use_rand=False)
    try:
        eager, _ = _sample(sd1, "ddim", "epsilon", 7.5, steps=3, graph=False)
        graphed, _ = _sample(sd1, "ddim", "epsilon", 7.5, steps=3, graph=True)
        key = sd1.pipe._graph["key"]
        tome.apply_patch(sd1.pipe, ratio=0.5, use_rand=False)     # a new patch recaptures
        _sample(sd1, "ddim", "epsilon", 7.5, steps=3, graph=True)
        assert sd1.pipe._graph["key"] != key
    finally:
        tome.remove_patch(sd1.pipe)
        sd1.pipe.disable_cuda_graph()
    print(f"patched sampling, graph vs eager {_rel(graphed, eager):.2e}")
    assert _rel(graphed, eager) < GRAPH_VS_EAGER


# ---- refusals --------------------------------------------------------------------------------------------------------
def test_refusals():
    from e4t_b200 import ops, tome
    from e4t_b200._lib import E4TError
    m, _ = _unet(O.TINY_UNET, 3)
    for kw in (dict(ratio=1.0), dict(ratio=-0.5), dict(max_downsample=3), dict(sx=0), dict(sy=0)):
        with pytest.raises(E4TError):
            tome.apply_patch(m, **kw)
    # over the select kernel's limit: 129 x 128 tokens
    h, w, C = 129, 128, 64
    x = _x(1, h * w, C, seed=1)
    mt = ops.tome_match(x, _pattern(h, w, False), h, w, 2, 2)
    with pytest.raises(E4TError, match="16384"):
        ops.tome_select(mt, 100)
    tome.apply_patch(m, ratio=0.5)
    try:
        with pytest.raises(E4TError, match="16384"), torch.no_grad():
            m(torch.randn(1, 4, 136, 136, device="cuda"), torch.tensor([5], device="cuda"),
              torch.randn(1, 77, O.TINY_UNET["cross_attention_dim"], device="cuda"))
    finally:
        tome.remove_patch(m)
