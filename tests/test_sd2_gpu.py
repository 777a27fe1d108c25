"""Stable Diffusion 2.x on the sm_90a kernels: the SD2 model shapes (linear proj_in / proj_out, heads of 64 on the
warpgroup attention, exact-GELU text tower), the v-prediction objective of the pre-training and tuning steps, the
v-prediction DDIM sampler and the SD 2.x empty prompt (pad id 0), against tests/golden/sd2.pt and the fp32 oracle.

Bands are the ones of the SD 1.x tests (test_e2e_gpu.py, test_tuning_gpu.py, test_pipeline_gpu.py): the CUDA path
computes with bf16 operands and fp32 accumulation, the oracle in fp32."""
import os

import pytest
import torch

from oracle import e4t_oracle as O
from oracle import sd2_oracle as S
from oracle.golden_format import base_name, golden_view, unpack_grads

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sd2.pt")


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt().clamp_min(1e-30)).item()


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD, weights_only=False)


def _unet(cfg, seed):
    from e4t.models.unet_2d_condition import UNet2DConditionModel
    m = UNet2DConditionModel(**O.ref_unet_kwargs(cfg))
    sd = O.synth_state_dict(S.unet_param_shapes(cfg), seed)
    m.load_state_dict(sd, strict=True)
    return m.cuda(), sd


def _text(t, seed):
    from e4t.models.modeling_clip import CLIPTextConfig, CLIPTextModel
    m = CLIPTextModel(CLIPTextConfig(vocab_size=t["vocab"], hidden_size=t["width"], intermediate_size=t["mlp"],
                                     num_hidden_layers=t["layers"], num_attention_heads=t["heads"],
                                     hidden_act=t.get("act", "quick_gelu")))
    sd = O.synth_state_dict(O.text_param_shapes(t), seed)
    m.load_state_dict(sd, strict=True)
    return m.cuda(), sd


def _models(cfgs, seeds):
    from e4t.encoder import E4TEncoder
    ucfg, vcfg, tcfg = cfgs
    fd = O.pooled_feature_dim(ucfg)
    unet, sd_u = _unet(ucfg, seeds[0])
    enc = E4TEncoder(arch="ViT-tiny-test", word_embedding_dim=tcfg["width"], n_odd_layers=129, unet_feature_dim=fd)
    sd_e = O.synth_state_dict(O.encoder_param_shapes(vcfg, fd, tcfg["width"], 129), seeds[1])
    enc.load_state_dict(sd_e, strict=True)
    text, sd_t = _text(tcfg, seeds[2])
    return (unet, enc.cuda(), text), (sd_u, sd_e, sd_t)


def test_tiny_sd2_unet_forward_and_every_gradient(gold):
    """Forward, encoder outputs and WeightOffsets gradients against the reference's golden; every other parameter
    gradient against autograd of the fp32 oracle."""
    g = gold["unet"]
    cfg = g["cfg"]
    m, sd = _unet(cfg, g["seed"])
    m.requires_grad_(True)
    x, t, ehs, w, wenc = O.golden_unet_inputs(cfg, g["B"], g["seed"], g["x"].shape[-1], g["enc_shapes"])
    ehs_c = ehs.cuda().requires_grad_(True)
    out = m(x.cuda(), t.cuda(), ehs_c).sample
    enc = m(x.cuda(), t.cuda(), ehs_c, return_encoder_outputs=True)["down_block_samples"]
    e_out = _rel(out, g["out"])
    e_enc = _rel(torch.cat([e.float().mean(dim=(2, 3)) for e in enc], -1), g["enc_pooled"])
    ((out * w.cuda()).sum() + sum((e.float() * we.cuda()).sum() for e, we in zip(enc, wenc))).backward()
    named = dict(m.named_parameters())
    wo = {k: _rel(golden_view(named[base_name(k)].grad, k, ref), ref) for k, ref in unpack_grads(g["wo_grads"]).items()}
    vec = sorted(v for k, v in wo.items() if not k.endswith(".v"))
    sdg = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    eg = ehs.clone().requires_grad_(True)
    o_ref = S.unet_forward(sdg, cfg, x, t, eg)
    e_ref = S.unet_forward(sdg, cfg, x, t, eg, return_encoder_outputs=True)["down_block_samples"]
    ((o_ref * w).sum() + sum((e * we).sum() for e, we in zip(e_ref, wenc))).backward()
    base = sorted(_rel(named[k].grad, sdg[k].grad) for k in sd if "wo" not in k)
    print(f"[sd2 tiny unet] out {e_out:.3e} enc {e_enc:.3e} d_ehs {_rel(ehs_c.grad, g['d_ehs']):.3e} wo median "
          f"{vec[len(vec) // 2]:.3e} max {vec[-1]:.3e}; base grads median {base[len(base) // 2]:.3e} "
          f"max {base[-1]:.3e}")
    assert e_out < 3e-2 and e_enc < 3e-2 and _rel(ehs_c.grad, g["d_ehs"]) < 6e-2
    assert vec[len(vec) // 2] < 6e-2 and vec[-1] < 0.15
    assert len(base) == sum(1 for k in sd if "wo" not in k) and base[len(base) // 2] < 6e-2 and base[-1] < 0.15


def test_full_sd2_unet_at_96x96_latents_vs_fp32_oracle():
    """The SD 2.x UNet (5 / 10 / 20 / 20 heads of 64, linear projections, 1024-wide context) at 768² pixels, B = 1:
    against the fp32 oracle on the GPU, within 2x the oracle's own error under bf16 autocast (floor 3e-2, as the
    SD 1.x UNet tests)."""
    cfg = S.SD2_UNET
    m, sd = _unet(cfg, 61)
    g = torch.Generator().manual_seed(62)
    x = torch.randn(1, 4, 96, 96, generator=g).cuda()
    t = torch.tensor([437]).cuda()
    ehs = torch.randn(1, 77, 1024, generator=g).cuda()
    with torch.no_grad():
        out = m(x, t, ehs).sample.float()
        del m
        sdc = {k: v.cuda() for k, v in sd.items()}
        tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
        try:
            ref = S.unet_forward(sdc, cfg, x, t, ehs)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                ref16 = S.unet_forward(sdc, cfg, x, t, ehs).float()
        finally:
            torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    e, calib = _rel(out, ref), _rel(ref16, ref)
    print(f"[sd2 unet 96x96] cuda vs fp32 oracle {e:.3e}; oracle under bf16 autocast {calib:.3e}")
    assert torch.isfinite(out).all() and e < max(3e-2, 2 * calib)


def _tiny_cfgs(gold):
    c = gold["step"]["cfg"]
    return c["unet"], c["vit"], c["text"]


def _oracle_run(sds, cfgs, batches, tune, prediction_type, pad_id):
    sd_u, sd_e, sd_t = ({k: v.clone() for k, v in sd.items()} for sd in sds)
    ucfg, vcfg, tcfg = cfgs
    train = [v.requires_grad_(True) for k, v in sd_u.items() if tune or "wo" in k]
    train += [v.requires_grad_(True) for k, v in sd_e.items() if not k.startswith("clip_vision.")]
    lr, reg = (2e-4, 1e-4) if tune else (1e-3, 1e-2)
    opt = torch.optim.AdamW(train, lr=lr, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8)
    losses = []
    for b in batches:
        ref = S.pretrain_step(sd_u, ucfg, sd_e, vcfg, sd_t, tcfg, b, class_token_id=320, reg_lambda=reg,
                              prediction_type=prediction_type, pad_id=pad_id)
        opt.zero_grad()
        ref["loss"].backward()
        if tune:
            torch.nn.utils.clip_grad_norm_(train, 1.0)
        opt.step()
        losses.append(ref["loss"].item())
    return losses


def _step(gold, tune, **kw):
    from e4t_b200.engine import PretrainStep, TuningStep
    (unet, enc, text), sds = _models(_tiny_cfgs(gold), gold["step"]["seeds"])
    if tune:
        s = TuningStep(unet, enc, text, O.PLACEHOLDER_ID, class_token_id=320, lr=2e-4, weight_dtype=torch.float32, **kw)
    else:
        s = PretrainStep(unet, enc, text, O.PLACEHOLDER_ID, class_token_id=320, lr=1e-3, weight_dtype=torch.float32,
                         **kw)
    return s, sds


def _batches(n, pad_id):
    out = []
    for i in range(n):
        b = O.synth_batch(2, seed=300 + i, latent_hw=16, image_hw=64)
        b["input_ids"], _ = S.synth_input_ids([i % 10, (3 * i + 1) % 10], pad_id=pad_id)
        out.append(b)
    return out


@pytest.mark.parametrize("tune", [False, True], ids=["pretrain", "tuning"])
def test_v_prediction_steps_eager_and_graphed_vs_oracle(gold, tune):
    """Five tiny SD2-shaped v-prediction steps (pad id 0), eager and as a replayed CUDA graph, against the oracle with
    torch AdamW (and clip_grad_norm_ for tuning).  The epsilon loss of the same first batch lies outside the band, so
    a prediction type that is ignored fails."""
    cfgs = _tiny_cfgs(gold)
    batches = _batches(5, 0)
    lo = _oracle_run(_models(cfgs, gold["step"]["seeds"])[1], cfgs, batches, tune, "v_prediction", 0)
    lo_eps = _oracle_run(_models(cfgs, gold["step"]["seeds"])[1], cfgs, batches[:1], tune, "epsilon", 0)
    band = lambda a: 3e-2 * abs(a) + 1e-4   # noqa: E731
    assert abs(lo_eps[0] - lo[0]) > band(lo[0]), (lo_eps[0], lo[0])
    eager, _ = _step(gold, tune, prediction_type="v_prediction", pad_id=0)
    le = [eager({k: v.cuda() for k, v in b.items()})["loss"].item() for b in batches]
    graphed, _ = _step(gold, tune, prediction_type="v_prediction", pad_id=0)

    def dev(b):
        d = {k: v.cuda() for k, v in b.items()}
        d["placeholder_idxs"] = torch.tensor(graphed.placeholder_idxs(d["input_ids"]), device="cuda")
        return d
    graphed.enable_cuda_graph(dev(batches[0]), warmup=1)     # one optimiser step on batch 0, then capture
    lg = [graphed(dev(b))["loss"].item() for b in batches[1:]]
    print(f"[v-prediction {'tuning' if tune else 'pretrain'}] oracle {[round(v, 5) for v in lo]} eager "
          f"{[round(v, 5) for v in le]} graphed {[round(v, 5) for v in lg]} (epsilon would be {lo_eps[0]:.5f})")
    for a, b in zip(lo, le):
        assert abs(a - b) <= band(a), (lo, le)
    for a, b in zip(lo[1:], lg):
        assert abs(a - b) <= band(a), (lo, lg)


def test_empty_prompt_with_pad_id_0_vs_oracle(gold):
    from e4t_b200.engine import PretrainStep
    cfgs = _tiny_cfgs(gold)
    (unet, enc, text), (_, _, sd_t) = _models(cfgs, gold["step"]["seeds"])
    s0 = PretrainStep(unet, enc, text, O.PLACEHOLDER_ID, class_token_id=320, weight_dtype=torch.float32,
                      optimizer=False, pad_id=0)
    s1 = PretrainStep(unet, enc, text, O.PLACEHOLDER_ID, class_token_id=320, weight_dtype=torch.float32,
                      optimizer=False)
    assert s0.ids_e4t.tolist() == [S.empty_prompt_ids(0)]
    with torch.no_grad():
        ref0 = S.text_forward(sd_t, cfgs[2], input_ids=torch.tensor([S.empty_prompt_ids(0)]))
        ref1 = S.text_forward(sd_t, cfgs[2], input_ids=torch.tensor([S.empty_prompt_ids()]))
    e0, e1 = _rel(s0.ehs_e4t.float(), ref0), _rel(s1.ehs_e4t.float(), ref1)
    print(f"[pad id] ehs_e4t pad 0 {e0:.3e}, pad EOS {e1:.3e}, the two oracles apart {_rel(ref0, ref1):.3e}")
    assert e0 < 3e-2 and e1 < 3e-2 and _rel(ref0, ref1) > 10 * e0


def test_default_ids_and_ops_calls_unchanged():
    """At the defaults the empty prompt is today's [BOS] + [EOS] * 76, and a tiny SD 1.x step makes exactly the same
    library calls with prediction_type / pad_id passed at their defaults as without them."""
    import test_e2e_gpu as E
    from test_call_signatures_gpu import Recorder
    calls = []
    for kw in ({}, dict(prediction_type="epsilon", pad_id=49407)):
        unet, enc, text, _, _, PretrainStep = E._build_step(seed=9)
        s = PretrainStep(unet, enc, text, O.PLACEHOLDER_ID, class_token_id=320, lr=1e-3, weight_dtype=torch.float32,
                         **kw)
        assert torch.equal(s.ids_e4t.cpu(), torch.tensor([[49406] + [49407] * 76]))
        b = {k: v.cuda() for k, v in O.synth_batch(2, 11, 16, 64).items()}
        s(b)
        torch.cuda.synchronize()
        with Recorder() as r:
            out = s(b)
            torch.cuda.synchronize()
        assert torch.isfinite(out["loss"])
        calls.append(r.calls)
    assert len(calls[0]) > 50 and calls[0] == calls[1]


def test_pipeline_v_prediction_vs_oracle(gold):
    import types
    from test_pipeline_gpu import _Tok
    from e4t.pipeline_stable_diffusion_e4t import DDIMScheduler, StableDiffusionE4TPipeline
    ucfg, vcfg, tcfg = cfgs = _tiny_cfgs(gold)
    (unet, enc, _), (sd_u, sd_e, _) = _models(cfgs, (71, 72, 73))
    small = dict(tcfg, vocab=tcfg["vocab"] - 1)
    text, _ = _text(small, 73)
    full = O.synth_state_dict(O.text_param_shapes(tcfg), 73)
    cfg = types.SimpleNamespace(placeholder_token="*s", domain_class_token="a", domain_embed_scale=0.1)
    sched = DDIMScheduler.from_config({"prediction_type": "v_prediction", "beta_schedule": "scaled_linear"})
    pipe = StableDiffusionE4TPipeline(None, text, _Tok(), unet, enc, sched, e4t_config=cfg)
    with torch.no_grad():
        text.get_input_embeddings().weight.copy_(full["text_model.embeddings.token_embedding.weight"].cuda())
    g = torch.Generator().manual_seed(3)
    image = torch.rand(1, 3, 64, 64, generator=g) * 2 - 1
    latents = torch.randn(2, 4, 16, 16, generator=g)
    prompt = ["a photo of *s", "a photo of *s"]
    out = pipe(prompt, num_inference_steps=4, guidance_scale=7.5, latents=latents.clone(), image=image,
               output_type="latent").images
    ids = pipe.tokenizer(prompt, max_length=77).input_ids
    kw = dict(num_inference_steps=4, guidance_scale=7.5, class_token_id=O._WORD_IDS["a"])
    ref = S.pipeline_sample(sd_u, ucfg, sd_e, vcfg, full, tcfg, image, ids, latents, prediction_type="v_prediction",
                            **kw)
    ref_eps = S.pipeline_sample(sd_u, ucfg, sd_e, vcfg, full, tcfg, image, ids, latents, **kw)
    e = _rel(out, ref)
    print(f"[pipeline v-prediction] latents after 4 DDIM steps rel err {e:.3e} "
          f"(epsilon sampler {_rel(ref_eps, ref):.3e})")
    assert out.shape == (2, 4, 16, 16) and e < 8e-2 and _rel(ref_eps, ref) > 8e-2
