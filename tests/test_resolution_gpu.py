"""Resolutions other than 512²: the im2col-mode implicit-GEMM convolutions against fp64 torch, every kernel call of
SD-v1.4 denoising, VAE and tuning at non-square sizes replayed alone, and the models end to end against the oracle.

Kernel bounds are those of test_gemm_gpu.test_conv3x3 / test_vae_gpu.test_conv3x3_s2_pads (RMS error relative to the
reference RMS), and every 128 x 64 output tile of the engine is held to 4x that bound, so one tile that spans two
images or two rows and reads the wrong pixels cannot hide in a large tensor."""
import os
import sys
import types

import pytest
import torch
import torch.nn.functional as F

from oracle import e4t_oracle as O
from oracle import vae_oracle as V

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_call_signatures_gpu as H  # noqa: E402

pytestmark = pytest.mark.gpu
F64 = torch.float64


def _rel(a, b):
    a = a.detach().double().cpu(); b = b.detach().double().cpu()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt().clamp_min(1e-30)).item()


def _mk(shape, g, scale=1.0):
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


def _check(label, got, ref, bound):
    finite, glob, worst, where = H.evaluate(H.Check(label, got, ref, bound, block=H.TILE))
    assert finite, f"{label}: non-finite output"
    assert glob <= bound, f"{label}: error {glob:.2e} > {bound:.1e}"
    assert worst <= H.LOCAL * bound, f"{label}: 128 x 64 tile {where} error {worst:.2e} > {H.LOCAL * bound:.1e}"
    return glob, worst


# ---------------------------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("B,Hh,W,Cin,Cout", [(2, 12, 8, 2560, 1280), (2, 8, 12, 640, 96), (2, 9, 9, 64, 160),
                                             (1, 64, 96, 320, 320), (2, 72, 72, 128, 100), (1, 8, 192, 64, 64),
                                             (1, 128, 192, 128, 128)])
def test_conv3x3_im2col(B, Hh, W, Cin, Cout, out_dtype):
    from e4t_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(B + Hh * W + Cin)
    x = _mk((B, Hh, W, Cin), g)
    w9 = _mk((9, Cout, Cin), g, scale=0.05)
    bias = torch.randn(Cout, generator=g, device="cuda")
    temb = torch.randn(B, Cout, generator=g, device="cuda")
    res = _mk((B, Hh, W, Cout), g)
    ref = F.conv2d(x.double().permute(0, 3, 1, 2), H._w9_to_oihw(w9), padding=1).permute(0, 2, 3, 1)
    ref = ref + bias.double() + temb.double()[:, None, None, :] + res.double()
    out = ops.conv3x3_im2col(x, w9, bias=bias, rowgroup=temb, residual=res, out_dtype=out_dtype)
    assert out.shape == (B, Hh, W, Cout) and out.dtype == out_dtype
    _check(f"conv3x3_im2col {B}x{Hh}x{W}", out, ref, 2e-3 if out_dtype == torch.float32 else 4e-3)


@pytest.mark.parametrize("B,Hh,W,Cin,Cout", [(2, 64, 64, 320, 320), (4, 8, 8, 1280, 1280), (3, 8, 8, 64, 96),
                                             (1, 16, 256, 128, 128)])
def test_conv3x3_im2col_equals_tiled_box(B, Hh, W, Cin, Cout):
    """Where both loads apply, the shared-memory tiles are byte-identical, so the results are bit-identical."""
    from e4t_b200 import ops
    assert ops.conv3x3_tiled(Hh, W)
    g = torch.Generator(device="cuda").manual_seed(Hh + Cout)
    x = _mk((B, Hh, W, Cin), g)
    w9 = _mk((9, Cout, Cin), g, scale=0.05)
    bias = torch.randn(Cout, generator=g, device="cuda")
    assert torch.equal(ops.conv3x3_im2col(x, w9, bias=bias), ops.conv3x3(x, w9, bias=bias))


def test_conv3x3_tiled_predicate():
    from e4t_b200 import ops
    ok = [(64, 64), (32, 32), (8, 8), (4, 4), (8, 16), (16, 256), (512, 512), (96, 64), (24, 16)]
    no = [(12, 8), (9, 9), (64, 96), (72, 72), (8, 192), (8, 12), (3, 32), (12, 16)]
    assert all(ops.conv3x3_tiled(*s) for s in ok) and not any(ops.conv3x3_tiled(*s) for s in no)


@pytest.mark.parametrize("pad_lo", [0, 1])
@pytest.mark.parametrize("B,Hh,W,Cin,Cout", [(2, 24, 16, 320, 320), (2, 18, 18, 640, 640), (1, 256, 384, 128, 128)])
def test_conv3x3_s2_im2col(B, Hh, W, Cin, Cout, pad_lo):
    from e4t_b200 import ops
    assert not ops.conv3x3_tiled(Hh // 2, W // 2)
    g = torch.Generator(device="cuda").manual_seed(Hh * W + Cin + pad_lo)
    x = _mk((B, Hh, W, Cin), g)
    w9 = _mk((9, Cout, Cin), g, scale=0.05)
    bias = torch.randn(Cout, generator=g, device="cuda")
    xd = x.double().permute(0, 3, 1, 2)
    if pad_lo == 0:
        ref = F.conv2d(F.pad(xd, (0, 1, 0, 1)), H._w9_to_oihw(w9), stride=2)
    else:
        ref = F.conv2d(xd, H._w9_to_oihw(w9), stride=2, padding=1)
    ref = ref.permute(0, 2, 3, 1) + bias.double()
    out = ops.conv3x3_s2(x, w9, bias=bias, pad_lo=pad_lo)
    assert out.shape == (B, Hh // 2, W // 2, Cout)
    _check(f"conv3x3_s2 pad {pad_lo} {Hh}x{W}", out, ref, 4e-3)


@pytest.mark.parametrize("B,Hh,W,Cin,Cout", [(1, 12, 8, 1280, 1280), (2, 12, 8, 640, 320), (1, 9, 9, 64, 128),
                                             (2, 9, 9, 320, 64), (2, 72, 72, 320, 320), (1, 64, 96, 128, 64)])
def test_conv3x3_wgrad_im2col(B, Hh, W, Cin, Cout):
    """Pixel counts 96, 81, 162 are not multiples of 64: the last K chunk reads past the end as zeros."""
    from e4t_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(Hh * W + Cout)
    x = _mk((B, Hh, W, Cin), g)
    dy = _mk((B, Hh, W, Cout), g)
    xd, dyd = x.double().permute(0, 3, 1, 2), dy.double().permute(0, 3, 1, 2)
    w = torch.nn.grad.conv2d_weight(xd, (Cout, Cin, 3, 3), dyd, padding=1)
    ref = w.permute(2, 3, 0, 1).reshape(9, Cout, Cin)
    _check(f"conv3x3_wgrad {B}x{Hh}x{W}", ops.conv3x3_wgrad(x, dy), ref, 2e-3)


# ---------------------------------------------------------------------------------------------------------------------
# every kernel call of SD-v1.4 denoising, the SD VAE and a tuning step at non-square sizes, replayed alone
# ---------------------------------------------------------------------------------------------------------------------
def h_wo_factors(c):
    """WeightOffsets factors (inference: the UNet's attention builds W_eff per call): vx = w1 v + b1, vy = w2 v + b2,
    a = Wc vx, b = Wr vy, s = Wr 1."""
    v, w1, b1, w2, b2, Wc, Wr = (H._d(c[n]) for n in ("v", "w1", "b1", "w2", "b2", "Wc", "Wr"))
    vx, vy = w1[:, 0] * v + b1, w2[:, 0] * v + b2
    ref = (vx, vy, Wc @ vx, Wr @ vy, Wr.sum(1))
    return [H.Check(n, g, r, 2e-3) for n, g, r in zip(("vx", "vy", "a", "b", "s"), c.run(), ref)]


def h_wo_weff(c):
    """W_eff = bf16(W * (1 + b a^T + s bc^T + br 1^T))."""
    W, a, bc, b, s, br = (H._d(c[n]) for n in ("W", "a", "bc", "b", "s", "br"))
    ref = W * (1 + b[:, None] * a[None, :] + s[:, None] * bc[None, :] + br[:, None])
    if c["out"] is not None:
        c.nan_("out")
    r = c.run()
    return [H.Check("out", r if c["out"] is None else c["out"], ref, 4e-3, block=H.TILE)]


HANDLERS = dict(H.HANDLERS, conv3x3_im2col=H.h_conv3x3, wo_factors=h_wo_factors, wo_weff=h_wo_weff)


def cfg_denoise_step(unet, enc, text, lat, pixel_values, input_ids, idx, t, guidance_scale=7.5):
    """One classifier-free-guidance step of StableDiffusionE4TPipeline.__call__ on one latent: the encoder-half UNet,
    the E4T encoder head, the text encoder with the domain embedding in the placeholder row, the full UNet on
    [unconditional, conditional]."""
    ids_e4t = torch.tensor([[49406] + [49407] * 76], device="cuda")
    with torch.no_grad():
        ehs_e4t = text(input_ids=ids_e4t)[0].to(torch.bfloat16)
        class_embed = text.get_input_embeddings()(torch.tensor([320], device="cuda")).float()
        e = unet(lat, t, ehs_e4t, return_encoder_outputs=True)
        dom = class_embed + 0.1 * enc(x=pixel_values, unet_down_block_samples=e["down_block_samples"]).float()
        emb = text.get_input_embeddings()(input_ids).clone()
        emb[:, idx, :] = dom.to(emb.dtype)
        ehs = text(inputs_embeds=emb)[0].to(torch.bfloat16)
        pred = unet(torch.cat([lat, lat]), t.expand(2), torch.cat([ehs_e4t, ehs])).sample
        u, c = pred.chunk(2)
        return u + guidance_scale * (c - u)


def _record_sd_workloads():
    import bench
    from e4t.models.autoencoder_kl import AutoencoderKL
    from e4t_b200.engine import TuningStep
    calls = {}

    def add(name, rec):
        for k, n in rec.calls.items():
            calls.setdefault(k, {})[name] = n
    unet, enc, text = bench.build_models("cuda")
    b = bench.to_device(bench.host_batch(1, 3, pinned=False), "cuda")
    idx = int(b["placeholder_idxs"][0])
    for hw in ((96, 64), (72, 72)):
        g = torch.Generator(device="cuda").manual_seed(hw[0])
        lat = torch.randn((1, 4) + hw, generator=g, device="cuda")
        with H.Recorder() as r:
            cfg_denoise_step(unet, enc, text, lat, b["pixel_values"], b["input_ids"], idx, b["timesteps"])
            torch.cuda.synchronize()
        add(f"cfg_step_{hw[0] * 8}x{hw[1] * 8}", r)
    step = TuningStep(unet, enc, text, 49408, class_token_id=320)
    tb = bench.to_device(bench.host_batch(2, 4, pinned=False), "cuda")
    g = torch.Generator(device="cuda").manual_seed(9)
    tb["latents"] = torch.randn(2, 4, 96, 64, generator=g, device="cuda") * 0.18215
    tb["noise"] = torch.randn(2, 4, 96, 64, generator=g, device="cuda")
    with H.Recorder() as r:
        step(tb)
        torch.cuda.synchronize()
    add("tuning_768x512", r)
    del step, unet, enc, text
    H._free()
    torch.manual_seed(0)
    vae = AutoencoderKL(**V.SD_VAE).cuda().eval().requires_grad_(False)
    for hw in ((512, 768), (576, 576)):
        g = torch.Generator(device="cuda").manual_seed(hw[1])
        x = torch.rand((1, 3) + hw, generator=g, device="cuda") * 2 - 1
        with torch.no_grad(), H.Recorder() as r:
            vae.decode(vae.encode(x).latent_dist.mean)
            torch.cuda.synchronize()
        add(f"vae_{hw[0]}x{hw[1]}", r)
    del vae
    H._free()
    return calls


def _old_wgrad_rule(Hh, W):
    return W <= 64 and 64 % W == 0 and (Hh * W) % 64 == 0 and Hh % (64 // W) == 0


@pytest.fixture(scope="module")
def inventory():
    from e4t_b200 import ops
    inv = _record_sd_workloads()
    ops_seen = {k[0] for k in inv}
    assert not ops_seen - set(HANDLERS), f"recorded but not replayed: {sorted(ops_seen - set(HANDLERS))}"
    im2col = [k for k in inv if k[0] == "conv3x3_im2col"]
    s2 = [k for k in inv if k[0] == "conv3x3_s2" and not ops.conv3x3_tiled(*[n // 2 for n in H._arg(k, "x")[1][1:3]])]
    wg = [k for k in inv if k[0] == "conv3x3_wgrad" and not _old_wgrad_rule(*H._arg(k, "x")[1][1:3])]
    print(f"[inventory] {len(inv)} distinct calls: {len(im2col)} conv3x3_im2col, {len(s2)} im2col stride-2, "
          f"{len(wg)} im2col wgrad")
    assert im2col and s2 and wg
    # the tiled conv3x3 still serves every size it covers
    assert all(ops.conv3x3_tiled(*H._arg(k, "x")[1][1:3]) for k in inv if k[0] == "conv3x3")
    return inv


def _replay(key, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    c = H.Call(key, g)
    checks = HANDLERS[key[0]](c)
    results = [(chk,) + H.evaluate(chk) for chk in checks]
    bad = c.guards_intact()
    del c
    return results, bad


def test_replay_every_call_at_other_resolutions(inventory):
    failures, worst_g, worst_b = [], 0.0, 0.0
    for i, key in enumerate(inventory):
        results, bad = _replay(key, 5000 + i)
        sig = H.describe(key)
        if bad:
            failures.append(f"{sig}: wrote outside the logical extent of {bad}")
        for chk, finite, glob, worst, where in results:
            worst_g, worst_b = max(worst_g, glob / chk.bound), max(worst_b, worst / chk.bound)
            if not finite:
                failures.append(f"{sig}: {chk.label} has non-finite elements")
            elif glob > chk.bound or worst > H.LOCAL * chk.bound:
                failures.append(f"{sig}: {chk.label} error {glob:.2e} (bound {chk.bound:.1e}); worst {chk.unit} at "
                                f"{where}: {worst:.2e}")
        H._free()
    print(f"[replay] {len(inventory)} signatures; worst global error {worst_g:.2f}x its bound, worst block "
          f"{worst_b:.2f}x the global bound")
    assert not failures, "\n".join(failures)


# ---------------------------------------------------------------------------------------------------------------------
# end to end, tiny configurations, 24 x 40 latents (every convolution of the tiny UNet takes the im2col path)
# ---------------------------------------------------------------------------------------------------------------------
def _rect_inputs(cfg, B, seed, hw):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn((B, 4) + hw, generator=g), torch.randint(0, 1000, (B,), generator=g),
            torch.randn(B, 77, cfg["cross_attention_dim"], generator=g), torch.randn((B, 4) + hw, generator=g))


@pytest.mark.parametrize("hw", [(24, 40), (40, 24)], ids=["24x40", "40x24"])
def test_tiny_unet_every_parameter_gradient_at_non_square_latents(hw):
    from e4t.models.unet_2d_condition import UNet2DConditionModel
    cfg = O.TINY_UNET
    m = UNet2DConditionModel(**O.ref_unet_kwargs(cfg))
    sd = O.synth_state_dict(O.unet_param_shapes(cfg), 7)
    m.load_state_dict(sd, strict=True)
    m = m.cuda()
    x, t, ehs, w = _rect_inputs(cfg, 2, 8, hw)
    out = m(x.cuda(), t.cuda(), ehs.cuda()).sample
    (out * w.cuda()).sum().backward()
    sdg = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    ref = O.unet_forward(sdg, cfg, x, t, ehs)
    (ref * w).sum().backward()
    e_out = _rel(out, ref)
    named = dict(m.named_parameters())
    assert all(p.grad is not None for p in named.values())
    errs = {k: _rel(named[k].grad, sdg[k].grad) for k in sd if "wo" not in k and sdg[k].grad is not None}
    srt = sorted(errs.values())
    print(f"[tiny unet {hw}] out {e_out:.3e}; {len(srt)} base params: median {srt[len(srt) // 2]:.3e} "
          f"max {srt[-1]:.3e} ({max(errs, key=errs.get)})")
    assert e_out < 3e-2
    assert srt[len(srt) // 2] < 3e-2 and srt[-1] < 0.15


def _rect_batch(seed, hw=(24, 40)):
    b = O.synth_batch(2, seed=seed, latent_hw=16, image_hw=64)
    g = torch.Generator().manual_seed(seed + 1)
    b["latents"] = torch.randn((2, 4) + hw, generator=g) * 0.18215
    b["noise"] = torch.randn((2, 4) + hw, generator=g)
    return b


def _tiny_models(seed):
    import test_vae_gpu as TV
    return TV._tiny_models(seed, seed + 1, seed + 2)


def test_pretrain_step_tiny_at_24x40_vs_oracle():
    from e4t_b200.engine import PretrainStep
    (unet, enc, text), (sd_u, sd_e, sd_t) = _tiny_models(11)
    step = PretrainStep(unet, enc, text, O.PLACEHOLDER_ID, class_token_id=320, lr=1e-3, weight_dtype=torch.float32,
                        optimizer=False)
    batch = _rect_batch(42)
    ref = O.pretrain_step(sd_u, O.TINY_UNET, sd_e, O.VIT_TINY, sd_t, O.CLIP_TEXT_TINY, batch, class_token_id=320)
    out = step.forward_loss({k: v.cuda() for k, v in batch.items()})
    e_pred, e_dom = _rel(out["pred"], ref["pred"]), _rel(out["domain_embed"], ref["domain_embed"])
    lo, lg = ref["loss"].item(), out["loss"].item()
    print(f"[pretrain 24x40] pred {e_pred:.3e} domain_embed {e_dom:.3e} loss {lg:.5f} vs {lo:.5f}")
    assert out["pred"].shape == (2, 4, 24, 40)
    assert e_pred < 3e-2 and e_dom < 3e-2
    assert abs(lo - lg) <= 3e-2 * abs(lo) + 1e-4


def test_tuning_step_tiny_at_24x40_vs_oracle_adamw_with_clipping():
    from e4t_b200.engine import TuningStep
    (unet, enc, text), (sd_u, sd_e, sd_t) = _tiny_models(21)
    step = TuningStep(unet, enc, text, O.PLACEHOLDER_ID, class_token_id=320, lr=2e-4, weight_dtype=torch.float32)
    plist = [sd_u[k].requires_grad_(True) for k in sd_u] + [sd_e[k].requires_grad_(True) for k in sd_e
                                                            if not k.startswith("clip_vision.")]
    opt = torch.optim.AdamW(plist, lr=2e-4, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8)
    base = _rect_batch(77)
    lo, lg = [], []
    for it in range(4):
        gen = torch.Generator().manual_seed(900 + it)
        batch = dict(base, noise=torch.randn(base["latents"].shape, generator=gen),
                     timesteps=torch.randint(0, 1000, (2,), generator=gen))
        ref = O.pretrain_step(sd_u, O.TINY_UNET, sd_e, O.VIT_TINY, sd_t, O.CLIP_TEXT_TINY, batch, class_token_id=320,
                              reg_lambda=1e-4)
        opt.zero_grad()
        ref["loss"].backward()
        torch.nn.utils.clip_grad_norm_(plist, 1.0)
        opt.step()
        lg.append(step({k: v.cuda() for k, v in batch.items()})["loss"].item())
        lo.append(ref["loss"].item())
    print("[tuning 24x40] oracle", [round(v, 5) for v in lo], "cuda", [round(v, 5) for v in lg])
    for a, b in zip(lo, lg):
        assert abs(a - b) <= 3e-2 * abs(a) + 1e-4, (lo, lg)


def _graph_vs_eager(make_step, lr):
    (ua, ea, ta), _ = _tiny_models(5)
    (ub, eb, tb), _ = _tiny_models(5)
    A = make_step(ua, ea, ta, O.PLACEHOLDER_ID, class_token_id=320, lr=lr, weight_dtype=torch.float32)
    Bs = make_step(ub, eb, tb, O.PLACEHOLDER_ID, class_token_id=320, lr=lr, weight_dtype=torch.float32)

    def mk(seed):
        b = {k: v.cuda() for k, v in _rect_batch(seed).items()}
        b["placeholder_idxs"] = torch.tensor(A.placeholder_idxs(b["input_ids"]), device="cuda")
        return b
    b0 = mk(100)
    Bs.enable_cuda_graph(b0, warmup=2)
    for _ in range(2):
        A(b0)
    la, lb = [], []
    for s in (101, 102, 103):
        b = mk(s)
        la.append(A(b)["loss"].item())
        lb.append(Bs(b)["loss"].item())
    return la, lb


def test_cuda_graph_step_at_24x40_matches_eager():
    """test_e2e_gpu.test_cuda_graph_step_matches_eager at 24 x 40 latents."""
    from e4t_b200.engine import PretrainStep
    la, lb = _graph_vs_eager(PretrainStep, 1e-3)
    print("[graph 24x40] eager", la, "graph", lb)
    for x, y in zip(la, lb):
        assert abs(x - y) <= 2e-3 * abs(x) + 1e-5


def test_cuda_graph_tuning_step_at_24x40_captures_im2col_weight_gradients():
    """The tuning step (every UNet convolution's weight gradient through the im2col load) captured whole; lr = 0 keeps
    the weights fixed, so eager and replayed losses agree although the split-K weight-gradient sums of the two runs
    are added in different orders."""
    from e4t_b200.engine import TuningStep
    la, lb = _graph_vs_eager(TuningStep, 0.0)
    print("[graph tuning 24x40] eager", la, "graph", lb)
    for x, y in zip(la, lb):
        assert abs(x - y) <= 2e-3 * abs(x) + 1e-5


def test_pipeline_with_vae_np_at_96x160_vs_oracle():
    import test_vae_gpu as TV
    from e4t.pipeline_stable_diffusion_e4t import DDIMScheduler, StableDiffusionE4TPipeline
    tcfg = O.CLIP_TEXT_TINY
    (unet, enc, text), (sd_u, sd_e, sd_t) = TV._tiny_models(41, 42, 43, text_vocab=tcfg["vocab"] - 1)
    vae, sd_v = TV._oracle_vae(44)
    cfg = types.SimpleNamespace(placeholder_token="*s", domain_class_token="a", domain_embed_scale=0.1)
    pipe = StableDiffusionE4TPipeline(vae, text, TV._Tok(), unet, enc, DDIMScheduler(), e4t_config=cfg)
    with torch.no_grad():
        text.get_input_embeddings().weight[-1] = sd_t["text_model.embeddings.token_embedding.weight"][-1].cuda()
    g = torch.Generator().manual_seed(3)
    image = torch.rand(1, 3, 64, 64, generator=g) * 2 - 1
    latents = torch.randn(2, 4, 24, 40, generator=g)
    prompt = ["a photo of *s", "a photo of *s"]
    with pytest.raises(ValueError, match="multiples of 8 px"):
        pipe(prompt, height=100, width=160, num_inference_steps=4, image=image, output_type="np")
    out = pipe(prompt, height=96, width=160, num_inference_steps=4, guidance_scale=1.0, latents=latents.clone(),
               image=image, output_type="np").images
    ids = pipe.tokenizer(prompt, max_length=77).input_ids
    ref_lat = O.pipeline_sample(sd_u, O.TINY_UNET, sd_e, O.VIT_TINY, sd_t, tcfg, image, ids, latents,
                                num_inference_steps=4, guidance_scale=1.0, class_token_id=O._WORD_IDS["a"])
    with torch.no_grad():
        ref = (V.vae_decode(sd_v, V.TINY_VAE, ref_lat / 0.18215) / 2 + 0.5).clamp(0, 1).permute(0, 2, 3, 1)
    out = torch.from_numpy(out)
    assert out.shape == (2, 96, 160, 3)
    e = _rel(out, ref)
    print(f"[pipeline np 96x160] rel err {e:.3e}")
    assert e < 4e-2


def test_step_rejects_latents_off_the_rule_on_device():
    from e4t_b200._lib import E4TError
    from e4t_b200.engine import PretrainStep
    (unet, enc, text), _ = _tiny_models(31)
    step = PretrainStep(unet, enc, text, O.PLACEHOLDER_ID, class_token_id=320, optimizer=False,
                        weight_dtype=torch.float32)
    b = {k: v.cuda() for k, v in _rect_batch(1, (24, 41)).items()}
    with pytest.raises(E4TError, match="multiples of the UNet's down-sampling factor 2"):
        step.forward_loss(b)


# ---------------------------------------------------------------------------------------------------------------------
# SD-v1.4 UNet and SD VAE at real sizes, against the oracle run on the GPU in fp32
# ---------------------------------------------------------------------------------------------------------------------
def _against_oracle(ours, ref_fn):
    with torch.no_grad():
        ref = ref_fn()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ref16 = ref_fn().float()
    e_ours, e_ref = _rel(ours, ref), _rel(ref16, ref)
    return e_ours, e_ref


@pytest.fixture(scope="module")
def sd14_unet():
    from e4t.models.unet_2d_condition import UNet2DConditionModel
    cfg = O.SD14_UNET
    sd = {k: v.cuda() for k, v in O.synth_state_dict(O.unet_param_shapes(cfg), 2).items()}
    m = UNet2DConditionModel(**O.ref_unet_kwargs(cfg)).cuda()
    m.load_state_dict(sd, strict=True)
    yield m, sd
    del m, sd
    H._free()


@pytest.mark.parametrize("hw", [(96, 64), (64, 96), (72, 72)], ids=["96x64", "64x96", "72x72"])
def test_sd14_unet_forward_vs_oracle(sd14_unet, hw):
    m, sd = sd14_unet
    cfg = O.SD14_UNET
    x, t, ehs, _ = (v.cuda() for v in _rect_inputs(cfg, 1, 3, hw))
    with torch.no_grad():
        out = m(x, t, ehs).sample
    assert out.shape == (1, 4) + hw
    e, e_ref = _against_oracle(out, lambda: O.unet_forward(sd, cfg, x, t, ehs))
    print(f"[sd14 unet {hw}] ours {e:.3e}  oracle under bf16 autocast {e_ref:.3e}")
    assert e <= 2.0 * e_ref + 1e-3, (e, e_ref)


# 1088 x 1024 and 1024 x 1536 put 17408 and 24576 tokens in each row of the mid-block attention's softmax, past the
# 16384 columns its register kernel holds
@pytest.mark.parametrize("hw", [(512, 768), (576, 576), (1088, 1024), (1024, 1536)],
                         ids=["512x768", "576x576", "1088x1024", "1024x1536"])
def test_sd_vae_decode_vs_oracle(hw):
    from e4t.models.autoencoder_kl import AutoencoderKL
    torch.manual_seed(0)
    vae = AutoencoderKL(**V.SD_VAE).cuda().eval().requires_grad_(False)
    sd = {k: v.float() for k, v in vae.state_dict().items()}
    g = torch.Generator(device="cuda").manual_seed(hw[1])
    z = torch.randn((1, 4, hw[0] // 8, hw[1] // 8), generator=g, device="cuda")
    with torch.no_grad():
        dec = vae.decode(z).sample
    assert dec.shape == (1, 3) + hw
    e, e_ref = _against_oracle(dec, lambda: V.vae_decode(sd, V.SD_VAE, z))
    print(f"[sd vae decode {hw}] ours {e:.3e}  oracle under bf16 autocast {e_ref:.3e}")
    assert e <= 2.0 * e_ref + 1e-3, (e, e_ref)
