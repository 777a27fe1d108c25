"""Latent sizes that are not multiples of the UNet's down-sampling factor (images in multiples of 8 px), with
UNet2DConditionModel.enable_any_latent_size(): the nearest resize to an explicit size, its adjoint and zero insertion
against torch, the stride-2 convolution at odd input sides and conv_in at any width against fp64, the VAE attention at
token counts that are not multiples of 8, the models end to end against the reference golden and the oracle, and the
switch leaving today's sizes exactly as they were."""
import os
import random
import sys
import types

import pytest
import torch
import torch.nn.functional as F

from oracle import e4t_oracle as O
from oracle import ragged_oracle as RO
from oracle import vae_oracle as V
from oracle.golden_format import base_name, golden_view, unpack_grads

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_call_signatures_gpu as H  # noqa: E402
import test_resolution_gpu as R  # noqa: E402
from test_ragged_cpu import GOLD, ragged_unet_inputs  # noqa: E402

pytestmark = pytest.mark.gpu
F64 = torch.float64
BF16 = torch.bfloat16
_rel, _check, _mk = R._rel, R._check, R._mk


def _nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def _nchw(t):
    return t.permute(0, 3, 1, 2)


# ---------------------------------------------------------------------------------------------------------------------
# nearest resize, its adjoint, zero insertion
# ---------------------------------------------------------------------------------------------------------------------
def _resize_pairs():
    rnd = random.Random(5)
    pairs = []
    for n in range(1, 41):
        outs = {2 * n - 1, 2 * n, 2 * n + 1} | {rnd.randint(1, 96) for _ in range(3)}
        pairs += [(n, o) for o in sorted(outs) if o > 0]
    return pairs


@pytest.mark.parametrize("C", [64, 320, 1280])
def test_resize_nearest_is_bit_exact_against_interpolate(C):
    from e4t_b200 import ops
    pairs = _resize_pairs()
    g = torch.Generator(device="cuda").manual_seed(C)
    bad = []
    for i, (hi, ho) in enumerate(pairs):
        wi, wo = pairs[-1 - i]                     # a different pair on the other axis
        x = torch.randn(2, C, hi, wi, generator=g, device="cuda").to(BF16)
        ref = F.interpolate(x, size=(ho, wo), mode="nearest")
        got = ops.resize_nearest(_nhwc(x), (ho, wo))
        if got.shape != (2, ho, wo, C) or not torch.equal(_nchw(got), ref):
            bad.append(((hi, wi), (ho, wo)))
    assert not bad, f"{len(bad)} of {len(pairs)} pairs differ, e.g. {bad[:5]}"


def test_resize_nearest_adjoint_against_fp64_autograd():
    from e4t_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(1)
    pairs = _resize_pairs()
    for i, (hi, ho) in enumerate(pairs[::3]):
        wi, wo = pairs[::3][-1 - i]
        x = torch.zeros(2, 64, hi, wi, dtype=F64, device="cuda", requires_grad=True)
        dy = torch.randn(2, 64, ho, wo, generator=g, device="cuda").to(BF16)
        F.interpolate(x, size=(ho, wo), mode="nearest").backward(dy.double())
        got = ops.resize_nearest_bwd(_nhwc(dy), (hi, wi))
        assert got.shape == (2, hi, wi, 64)
        err = (_nchw(got).double() - x.grad).abs()
        # fp32 sums of at most 2 x 2 ... 96 x 96 bf16 values, rounded once to bf16
        assert bool((err <= 2 ** -8 * x.grad.abs() + 1e-4).all()), ((hi, wi), (ho, wo), err.max().item())


def test_resize_nearest_and_adjoint_are_deterministic():
    from e4t_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(2)
    x = _mk((2, 33, 17, 320), g)
    dy = _mk((2, 65, 33, 320), g)
    assert torch.equal(ops.resize_nearest(x, (65, 33)), ops.resize_nearest(x, (65, 33)))
    assert torch.equal(ops.resize_nearest_bwd(dy, (33, 17)), ops.resize_nearest_bwd(dy, (33, 17)))


@pytest.mark.parametrize("size", [(65, 65), (33, 16), (16, 17), (9, 5), (1, 1), (2, 3)])
def test_zero_insert_to_odd_size_is_exact(size):
    from e4t_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(size[0] * 100 + size[1])
    dy = _mk((2, (size[0] + 1) // 2, (size[1] + 1) // 2, 64), g)
    ref = torch.zeros((2,) + size + (64,), dtype=BF16, device="cuda")
    ref[:, ::2, ::2] = dy
    assert torch.equal(ops.zero_insert(dy, size), ref)


def test_resize_fn_at_2x_runs_the_2x_kernel():
    from e4t_b200 import functional as FN
    g = torch.Generator(device="cuda").manual_seed(3)
    x = _mk((2, 12, 20, 64), g).requires_grad_(True)
    with H.Recorder() as r:
        y = FN.ResizeNearestFn.apply(x, (24, 40))
        y.backward(torch.ones_like(y))
    assert [k[0] for k in r.calls] == ["resample2x", "resample2x"]


# ---------------------------------------------------------------------------------------------------------------------
# stride-2 convolution at odd input sides, conv_in at any width
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,Hh,W,Cin,Cout", [(2, 65, 65, 320, 320), (2, 33, 17, 640, 640), (2, 17, 9, 1280, 1280),
                                             (2, 9, 5, 1280, 1280), (1, 65, 64, 320, 320), (1, 64, 33, 640, 640)])
def test_conv3x3_s2_at_odd_inputs_forward_dx_dw(B, Hh, W, Cin, Cout):
    from e4t_b200 import functional as FN
    from e4t.models.resnet import conv_w9, conv_w9_dgrad
    g = torch.Generator(device="cuda").manual_seed(Hh * W + Cin)
    conv = torch.nn.Conv2d(Cin, Cout, 3, stride=2, padding=1).cuda()
    with torch.no_grad():
        conv.weight.copy_(torch.randn(conv.weight.shape, generator=g, device="cuda") * 0.02)
        conv.bias.copy_(torch.randn(Cout, generator=g, device="cuda"))
    x = _mk((B, Hh, W, Cin), g).requires_grad_(True)
    y = FN.Conv3x3S2Fn.apply(x, conv_w9(conv), conv_w9_dgrad(conv), conv.bias, conv.weight)
    Ho, Wo = (Hh + 1) // 2, (W + 1) // 2
    assert y.shape == (B, Ho, Wo, Cout)
    dy = _mk((B, Ho, Wo, Cout), g)
    y.backward(dy)
    xd = _nchw(x.detach()).double().requires_grad_(True)
    wd = conv_w9(conv).double().view(3, 3, Cout, Cin).permute(2, 3, 0, 1).contiguous().requires_grad_(True)
    ref = F.conv2d(xd, wd, conv.bias.detach().double(), stride=2, padding=1)
    ref.backward(_nchw(dy).double())
    _check(f"conv3x3_s2 {Hh}x{W} y", y, ref.permute(0, 2, 3, 1), 4e-3)
    _check(f"conv3x3_s2 {Hh}x{W} dx", x.grad, xd.grad.permute(0, 2, 3, 1), 4e-3)
    _check(f"conv3x3_s2 {Hh}x{W} dw", conv.weight.grad.permute(2, 3, 0, 1).reshape(9, Cout, Cin),
           wd.grad.permute(2, 3, 0, 1).reshape(9, Cout, Cin), 4e-3)
    assert _rel(conv.bias.grad, _nchw(dy).double().sum((0, 2, 3))) < 1e-3


def test_conv3x3_s2_pad0_still_refuses_odd_inputs():
    from e4t_b200 import ops
    from e4t_b200._lib import E4TError
    g = torch.Generator(device="cuda").manual_seed(4)
    with pytest.raises(E4TError):
        ops.conv3x3_s2(_mk((1, 9, 8, 64), g), _mk((9, 64, 64), g), pad_lo=0)


@pytest.mark.parametrize("W", [1, 2, 3, 4, 5, 6, 7, 9, 63, 65, 97])
def test_conv_in_at_any_width(W):
    from e4t_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(W)
    x = torch.randn(2, 4, 13, W, generator=g, device="cuda")
    w = torch.randn(320, 4, 3, 3, generator=g, device="cuda") * 0.2
    b = torch.randn(320, generator=g, device="cuda")
    ref = F.conv2d(x.double(), w.double(), b.double(), padding=1).permute(0, 2, 3, 1)
    got = ops.conv_in_fwd(x, w, b)
    assert got.shape == (2, 13, W, 320)
    assert _rel(got, ref) < 4e-3


# ---------------------------------------------------------------------------------------------------------------------
# the VAE mid-block attention at token counts that are not multiples of 8
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,hw", [(2, (9, 13)), (1, (65, 65))], ids=["9x13", "65x65"])
def test_vae_attention_block_at_ragged_token_counts(B, hw):
    from e4t.models.attention import AttentionBlock
    torch.manual_seed(hw[0])
    blk = AttentionBlock(512, norm_num_groups=32, eps=1e-6).cuda().eval().requires_grad_(False)
    sd = {"a." + k: v.double() for k, v in blk.state_dict().items()}
    g = torch.Generator(device="cuda").manual_seed(7)
    x = _mk((B,) + hw + (512,), g)
    with torch.no_grad():
        got = blk(x)
        ref = V._attn(sd, "a.", _nchw(x).double(), 32).permute(0, 2, 3, 1)
    assert got.shape == x.shape
    e = _rel(got, ref)
    print(f"[vae attention {hw}] {e:.3e}")
    assert e < 1e-2


# ---------------------------------------------------------------------------------------------------------------------
# end to end, tiny configurations, against the reference's own UNet (tests/golden/ragged.pt)
# ---------------------------------------------------------------------------------------------------------------------
def _tiny_unet(sd):
    from e4t.models.unet_2d_condition import UNet2DConditionModel
    m = UNet2DConditionModel(**O.ref_unet_kwargs(O.TINY_UNET))
    m.load_state_dict(sd, strict=True)
    m.enable_any_latent_size()
    return m.cuda()


@pytest.mark.parametrize("case", ["9x13", "13x7"])
def test_tiny_unet_against_reference_golden(case):
    gold = torch.load(GOLD)[case]
    cfg = gold["cfg"]
    x, t, ehs, w, wenc = ragged_unet_inputs(gold)
    m = _tiny_unet(O.synth_state_dict(O.unet_param_shapes(cfg), gold["seed"]))
    ehs = ehs.cuda().requires_grad_(True)
    out = m(x.cuda(), t.cuda(), ehs).sample
    enc = m(x.cuda(), t.cuda(), ehs, return_encoder_outputs=True)["down_block_samples"]
    assert [tuple(e.shape) for e in enc] == gold["enc_shapes"]
    ((out * w.cuda()).sum() + sum((e.float() * we.cuda()).sum() for e, we in zip(enc, wenc))).backward()
    e_out = _rel(out, gold["out"])
    e_enc = _rel(torch.cat([e.float().mean(dim=(2, 3)) for e in enc], -1), gold["enc_pooled"])
    e_ehs = _rel(ehs.grad, gold["d_ehs"])
    named = dict(m.named_parameters())
    errs = {}
    for k, ref in unpack_grads(gold["grads"]).items():
        p = named[base_name(k)]
        assert p.grad is not None, k
        if "wo" not in k:
            errs[k] = _rel(golden_view(p.grad, k, ref), ref)
    srt = sorted(errs.values())
    print(f"[tiny unet {case}] out {e_out:.3e} enc {e_enc:.3e} d_ehs {e_ehs:.3e}; {len(srt)} gradient entries: "
          f"median {srt[len(srt) // 2]:.3e} max {srt[-1]:.3e} ({max(errs, key=errs.get)})")
    assert e_out < 3e-2 and e_enc < 3e-2 and e_ehs < 3e-2
    assert srt[len(srt) // 2] < 3e-2 and srt[-1] < 0.15


def _ragged_batch(seed, hw):
    b = O.synth_batch(2, seed=seed, latent_hw=16, image_hw=64)
    g = torch.Generator().manual_seed(seed + 1)
    b["latents"] = torch.randn((2, 4) + hw, generator=g) * 0.18215
    b["noise"] = torch.randn((2, 4) + hw, generator=g)
    return b


def _tiny_models(seed):
    (unet, enc, text), sds = R._tiny_models(seed)
    unet.enable_any_latent_size()
    return (unet, enc, text), sds


@pytest.mark.parametrize("hw", [(9, 13), (13, 7)], ids=["9x13", "13x7"])
def test_pretrain_step_tiny_at_ragged_latents_vs_oracle(hw):
    from e4t_b200.engine import PretrainStep
    (unet, enc, text), (sd_u, sd_e, sd_t) = _tiny_models(11)
    step = PretrainStep(unet, enc, text, O.PLACEHOLDER_ID, class_token_id=320, lr=1e-3, weight_dtype=torch.float32,
                        optimizer=False)
    batch = _ragged_batch(42, hw)
    ref = RO.pretrain_step(sd_u, O.TINY_UNET, sd_e, O.VIT_TINY, sd_t, O.CLIP_TEXT_TINY, batch, class_token_id=320)
    out = step.forward_loss({k: v.cuda() for k, v in batch.items()})
    e_pred, e_dom = _rel(out["pred"], ref["pred"]), _rel(out["domain_embed"], ref["domain_embed"])
    lo, lg = ref["loss"].item(), out["loss"].item()
    print(f"[pretrain {hw}] pred {e_pred:.3e} domain_embed {e_dom:.3e} loss {lg:.5f} vs {lo:.5f}")
    assert out["pred"].shape == (2, 4) + hw
    assert e_pred < 3e-2 and e_dom < 3e-2
    assert abs(lo - lg) <= 3e-2 * abs(lo) + 1e-4


def test_tuning_step_tiny_at_ragged_latents_vs_oracle():
    from e4t_b200.engine import TuningStep
    (unet, enc, text), (sd_u, sd_e, sd_t) = _tiny_models(21)
    step = TuningStep(unet, enc, text, O.PLACEHOLDER_ID, class_token_id=320, lr=2e-4, weight_dtype=torch.float32)
    plist = [sd_u[k].requires_grad_(True) for k in sd_u] + [sd_e[k].requires_grad_(True) for k in sd_e
                                                            if not k.startswith("clip_vision.")]
    opt = torch.optim.AdamW(plist, lr=2e-4, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8)
    base = _ragged_batch(77, (13, 9))
    lo, lg = [], []
    for it in range(3):
        gen = torch.Generator().manual_seed(900 + it)
        batch = dict(base, noise=torch.randn(base["latents"].shape, generator=gen),
                     timesteps=torch.randint(0, 1000, (2,), generator=gen))
        ref = RO.pretrain_step(sd_u, O.TINY_UNET, sd_e, O.VIT_TINY, sd_t, O.CLIP_TEXT_TINY, batch, class_token_id=320,
                              reg_lambda=1e-4)
        opt.zero_grad()
        ref["loss"].backward()
        torch.nn.utils.clip_grad_norm_(plist, 1.0)
        opt.step()
        lg.append(step({k: v.cuda() for k, v in batch.items()})["loss"].item())
        lo.append(ref["loss"].item())
    print("[tuning 13x9] oracle", [round(v, 5) for v in lo], "cuda", [round(v, 5) for v in lg])
    for a, b in zip(lo, lg):
        assert abs(a - b) <= 3e-2 * abs(a) + 1e-4, (lo, lg)


def _graph_vs_eager(make_step, lr, hw):
    (ua, ea, ta), _ = _tiny_models(5)
    (ub, eb, tb), _ = _tiny_models(5)
    A = make_step(ua, ea, ta, O.PLACEHOLDER_ID, class_token_id=320, lr=lr, weight_dtype=torch.float32)
    Bs = make_step(ub, eb, tb, O.PLACEHOLDER_ID, class_token_id=320, lr=lr, weight_dtype=torch.float32)

    def mk(seed):
        b = {k: v.cuda() for k, v in _ragged_batch(seed, hw).items()}
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


@pytest.mark.parametrize("kind", ["pretrain", "tuning"])
def test_cuda_graph_step_at_ragged_latents_matches_eager(kind):
    from e4t_b200.engine import PretrainStep, TuningStep
    la, lb = _graph_vs_eager(PretrainStep if kind == "pretrain" else TuningStep, 1e-3 if kind == "pretrain" else 0.0,
                             (9, 13))
    print(f"[graph {kind} 9x13] eager", la, "graph", lb)
    for x, y in zip(la, lb):
        assert abs(x - y) <= 2e-3 * abs(x) + 1e-5


def test_pipeline_with_vae_np_at_ragged_latents_vs_oracle():
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
    latents = torch.randn(2, 4, 13, 9, generator=g)
    prompt = ["a photo of *s", "a photo of *s"]
    with pytest.raises(ValueError, match="multiples of 8 px"):
        pipe(prompt, height=52, width=36, num_inference_steps=4, image=image, output_type="np")
    pipe.unet.enable_any_latent_size()
    out = pipe(prompt, height=52, width=36, num_inference_steps=4, guidance_scale=1.0, latents=latents.clone(),
               image=image, output_type="np").images
    ids = pipe.tokenizer(prompt, max_length=77).input_ids
    ref_lat = RO.pipeline_sample(sd_u, O.TINY_UNET, sd_e, O.VIT_TINY, sd_t, tcfg, image, ids, latents,
                                num_inference_steps=4, guidance_scale=1.0, class_token_id=O._WORD_IDS["a"])
    with torch.no_grad():
        ref = (V.vae_decode(sd_v, V.TINY_VAE, ref_lat / 0.18215) / 2 + 0.5).clamp(0, 1).permute(0, 2, 3, 1)
    out = torch.from_numpy(out)
    assert out.shape == (2, 52, 36, 3)
    e = _rel(out, ref)
    print(f"[pipeline np 52x36] rel err {e:.3e}")
    assert e < 4e-2


def test_step_refuses_latents_below_the_minimum_on_device():
    from e4t_b200._lib import E4TError
    from e4t_b200.engine import PretrainStep
    (unet, enc, text), _ = _tiny_models(31)
    step = PretrainStep(unet, enc, text, O.PLACEHOLDER_ID, class_token_id=320, optimizer=False,
                        weight_dtype=torch.float32)
    b = {k: v.cuda() for k, v in _ragged_batch(1, (1, 13)).items()}
    with pytest.raises(E4TError, match="at least 2"):
        step.forward_loss(b)


# ---------------------------------------------------------------------------------------------------------------------
# the switch leaves today's sizes alone
# ---------------------------------------------------------------------------------------------------------------------
def _on_off(m, x, t, ehs):
    """Outputs and recorded calls with the switch off, on, and off again: GroupNorm's statistics are summed across CTAs
    with fp32 atomics, so two forwards of the same UNet differ in the last bits; the switch may differ from off by no
    more than off differs from itself, and must issue the same calls with the same arguments."""
    with torch.no_grad():
        m(x, t, ehs)                 # the first forward also builds the cached operand copies
    outs, calls = [], []
    for on in (False, True, False):
        (m.enable_any_latent_size if on else m.disable_any_latent_size)()
        with torch.no_grad(), H.Recorder() as r:
            outs.append(m(x, t, ehs).sample.clone())
            torch.cuda.synchronize()
        calls.append(list(r.calls.items()))
    m.disable_any_latent_size()
    return outs, calls


def test_switch_changes_nothing_at_todays_sizes_tiny():
    m = _tiny_unet(O.synth_state_dict(O.unet_param_shapes(O.TINY_UNET), 7))
    x, t, ehs, _ = (v.cuda() for v in R._rect_inputs(O.TINY_UNET, 2, 8, (24, 40)))
    _check_on_off(*_on_off(m, x, t, ehs))


def _check_on_off(outs, calls):
    off, on, off2 = outs
    assert calls[0] == calls[1] == calls[2]
    e_on, e_off = _rel(on, off), _rel(off2, off)
    print(f"[switch at today's size] on vs off {e_on:.2e}, off vs off {e_off:.2e}")
    if e_off == 0:
        assert torch.equal(on, off)
    assert e_on <= 4 * e_off + 1e-3, (e_on, e_off)


# ---------------------------------------------------------------------------------------------------------------------
# SD-v1.4 UNet and SD VAE at ragged sizes, against the oracle run on the GPU in fp32
# ---------------------------------------------------------------------------------------------------------------------
sd14_unet = R.sd14_unet


def test_switch_changes_nothing_at_todays_sizes_sd14(sd14_unet):
    m, _ = sd14_unet
    x, t, ehs, _ = (v.cuda() for v in R._rect_inputs(O.SD14_UNET, 1, 3, (64, 64)))
    _check_on_off(*_on_off(m, x, t, ehs))


@pytest.mark.parametrize("hw", [(65, 65), (68, 84), (63, 97)], ids=["65x65", "68x84", "63x97"])
def test_sd14_unet_forward_at_ragged_latents_vs_oracle(sd14_unet, hw):
    m, sd = sd14_unet
    cfg = O.SD14_UNET
    x, t, ehs, _ = (v.cuda() for v in R._rect_inputs(cfg, 1, 3, hw))
    m.enable_any_latent_size()
    try:
        with torch.no_grad():
            out = m(x, t, ehs).sample
    finally:
        m.disable_any_latent_size()
    assert out.shape == (1, 4) + hw
    e, e_ref = R._against_oracle(out, lambda: RO.unet_forward(sd, cfg, x, t, ehs))
    print(f"[sd14 unet {hw}] ours {e:.3e}  oracle under bf16 autocast {e_ref:.3e}")
    assert e <= 2.0 * e_ref + 1e-3, (e, e_ref)


def test_sd_vae_encode_520x664_and_decode_65x65_vs_oracle():
    from e4t.models.autoencoder_kl import AutoencoderKL
    torch.manual_seed(0)
    vae = AutoencoderKL(**V.SD_VAE).cuda().eval().requires_grad_(False)
    sd = {k: v.float() for k, v in vae.state_dict().items()}
    g = torch.Generator(device="cuda").manual_seed(664)
    x = torch.rand((1, 3, 520, 664), generator=g, device="cuda") * 2 - 1
    z = torch.randn((1, 4, 65, 65), generator=g, device="cuda")
    with torch.no_grad():
        moments = vae.encode(x).latent_dist.parameters
        dec = vae.decode(z).sample
    assert moments.shape == (1, 8, 65, 83) and dec.shape == (1, 3, 520, 520)
    e, e_ref = R._against_oracle(moments, lambda: V.vae_encode(sd, V.SD_VAE, x))
    print(f"[sd vae encode 520x664] ours {e:.3e}  oracle under bf16 autocast {e_ref:.3e}")
    assert e <= 2.0 * e_ref + 1e-3, (e, e_ref)
    e, e_ref = R._against_oracle(dec, lambda: V.vae_decode(sd, V.SD_VAE, z))
    print(f"[sd vae decode 65x65] ours {e:.3e}  oracle under bf16 autocast {e_ref:.3e}")
    assert e <= 2.0 * e_ref + 1e-3, (e, e_ref)


# ---------------------------------------------------------------------------------------------------------------------
# every kernel call of an SD-v1.4 tuning step and an SD VAE encode + decode at ragged sizes, replayed alone
# ---------------------------------------------------------------------------------------------------------------------
def h_resize_nearest(c):
    ref = F.interpolate(_nchw(H._d(c["x"])), size=tuple(c["size"]), mode="nearest").permute(0, 2, 3, 1)
    return [H.Check("y", c.run(), ref, 1e-6)]


def h_resize_nearest_bwd(c):
    dy = H._d(c["dy"])
    x = torch.zeros((dy.shape[0], dy.shape[-1]) + tuple(c["in_size"]), dtype=F64, device="cuda", requires_grad=True)
    F.interpolate(x, size=dy.shape[1:3], mode="nearest").backward(_nchw(dy))
    return [H.Check("dx", c.run(), x.grad.permute(0, 2, 3, 1), 4e-3)]


def h_zero_insert(c):
    dy = H._d(c["dy"])
    ref = torch.zeros((dy.shape[0],) + tuple(c["size"]) + (dy.shape[-1],), dtype=F64, device="cuda")
    ref[:, ::2, ::2] = dy
    return [H.Check("y", c.run(), ref, 1e-6)]


HANDLERS = dict(R.HANDLERS, resize_nearest=h_resize_nearest, resize_nearest_bwd=h_resize_nearest_bwd,
                zero_insert=h_zero_insert)


def _guards_intact(c):
    """Call.guards_intact, except that a GEMM whose output rows are padded (the VAE attention's scores at token counts
    that are not multiples of 8) may write its TMA epilogue's last 16-byte chunk of each row past N: those pad columns
    are inside the row pitch, and the attention overwrites them before the softmax reads them.  Anything further out
    must still hold its guard value."""
    bad = c.guards_intact()
    if c.name != "gemm" or bad != ["out"]:
        return bad
    gt = c.guarded["out"]
    n = gt.t.shape[-1]
    per16 = 16 // gt.t.element_size()
    extra = min(-(-n // per16) * per16, gt.t.stride(-2)) - n
    mask = torch.ones_like(gt.buf, dtype=torch.bool)
    mask.as_strided(gt.t.shape, gt.t.stride(), gt.off).fill_(False)
    if extra:
        mask.as_strided(gt.t.shape[:-1] + (extra,), gt.t.stride(), gt.off + n).fill_(False)
    return [] if bool(gt.buf[mask].isnan().all()) else bad


def _record_ragged_workloads():
    import bench
    from e4t.models.autoencoder_kl import AutoencoderKL
    from e4t_b200.engine import TuningStep
    calls = {}

    def add(name, rec):
        for k, n in rec.calls.items():
            calls.setdefault(k, {})[name] = n
    unet, enc, text = bench.build_models("cuda")
    unet.enable_any_latent_size()
    step = TuningStep(unet, enc, text, 49408, class_token_id=320)
    tb = bench.to_device(bench.host_batch(2, 4, pinned=False), "cuda")
    g = torch.Generator(device="cuda").manual_seed(9)
    tb["latents"] = torch.randn(2, 4, 65, 83, generator=g, device="cuda") * 0.18215
    tb["noise"] = torch.randn(2, 4, 65, 83, generator=g, device="cuda")
    with H.Recorder() as r:
        step(tb)
        torch.cuda.synchronize()
    add("tuning_520x664", r)
    del step, unet, enc, text
    H._free()
    torch.manual_seed(0)
    vae = AutoencoderKL(**V.SD_VAE).cuda().eval().requires_grad_(False)
    g = torch.Generator(device="cuda").manual_seed(664)
    x = torch.rand((1, 3, 520, 664), generator=g, device="cuda") * 2 - 1
    with torch.no_grad(), H.Recorder() as r:
        vae.decode(vae.encode(x).latent_dist.mean)
        torch.cuda.synchronize()
    add("vae_520x664", r)
    del vae
    H._free()
    return calls


def test_replay_every_call_at_ragged_sizes():
    inv = _record_ragged_workloads()
    ops_seen = {k[0] for k in inv}
    assert not ops_seen - set(HANDLERS), f"recorded but not replayed: {sorted(ops_seen - set(HANDLERS))}"
    assert {"resize_nearest", "resize_nearest_bwd", "zero_insert"} <= ops_seen, sorted(ops_seen)
    failures, worst_g, worst_b = [], 0.0, 0.0
    for i, key in enumerate(inv):
        g = torch.Generator(device="cuda").manual_seed(7000 + i)
        c = H.Call(key, g)
        checks = HANDLERS[key[0]](c)
        results = [(chk,) + H.evaluate(chk) for chk in checks]
        bad = _guards_intact(c)
        del c
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
    print(f"[replay ragged] {len(inv)} signatures ({sorted(ops_seen)}); worst global error {worst_g:.2f}x its bound, "
          f"worst block {worst_b:.2f}x the global bound")
    assert not failures, "\n".join(failures)
