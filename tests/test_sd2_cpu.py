"""Stable Diffusion 2.x without a GPU: the oracle's SD2 model shapes (linear projections, per-level head counts, exact-GELU
text tower, v-prediction, pad id 0) against tests/golden/sd2.pt, which the reference's own modules produced
(oracle/gen_golden_sd2.py); the v-prediction target and DDIM step against literal restatements of the diffusers 0.14
formulas; and the refusals of unknown prediction types and unsupported scheduler configs."""
import hashlib
import json
import os

import pytest
import torch

from oracle import e4t_oracle as O
from oracle import sd2_oracle as S
from oracle.golden_format import base_name, golden_view, unpack_grads

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sd2.pt")


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD, weights_only=False)


def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt().clamp_min(1e-30)).item()


def _grad_errs(grads, packed):
    return {k: _rel(golden_view(grads[base_name(k)], k, ref), ref) for k, ref in unpack_grads(packed).items()}


def test_tiny_sd2_unet_oracle_vs_reference(gold):
    g = gold["unet"]
    cfg = g["cfg"]
    assert cfg["use_linear_projection"] and cfg["attention_head_dim"] == (2, 4) and cfg["cross_attention_dim"] == 96
    sd = O.synth_state_dict(S.unet_param_shapes(cfg), g["seed"])
    assert sd["down_blocks.0.attentions.0.proj_in.weight"].shape == (64, 64)
    for k in sd:
        if "wo" in k:
            sd[k].requires_grad_(True)
    x, t, ehs, w, wenc = O.golden_unet_inputs(cfg, g["B"], g["seed"], g["x"].shape[-1], g["enc_shapes"])
    assert torch.equal(x, g["x"]) and torch.equal(ehs, g["ehs"])
    ehs.requires_grad_(True)
    out = S.unet_forward(sd, cfg, x, t, ehs)
    enc = S.unet_forward(sd, cfg, x, t, ehs, return_encoder_outputs=True)["down_block_samples"]
    assert _rel(out, g["out"]) < 1e-4
    assert _rel(torch.cat([e.mean(dim=(2, 3)) for e in enc], -1), g["enc_pooled"]) < 1e-4
    ((out * w).sum() + sum((e * we).sum() for e, we in zip(enc, wenc))).backward()
    assert _rel(ehs.grad, g["d_ehs"]) < 1e-4
    errs = _grad_errs({k: v.grad for k, v in sd.items() if "wo" in k}, g["wo_grads"])
    assert len(errs) > 100 and max(errs.values()) < 1e-4, max(errs.items(), key=lambda kv: kv[1])


def test_sd2_unet_inventory(gold):
    inv = gold["inventory"]
    shapes = S.unet_param_shapes(S.SD2_UNET)
    keys = sorted(shapes)
    digest = hashlib.sha256("\n".join(f"{k}:{tuple(shapes[k])}" for k in keys).encode()).hexdigest()
    numel = {k: int(torch.Size(s).numel()) for k, s in shapes.items()}
    assert digest == inv["sha256"] and len(keys) == inv["n_keys"]
    assert sum(n for k, n in numel.items() if "wo" not in k) == inv["n_base"] == 865910724
    assert sum(n for k, n in numel.items() if "wo" in k) == inv["n_wo"]
    assert sum(1 for k in shapes if "wo" in k) == inv["n_wo_tensors"]


def test_v_prediction_step_oracle_vs_reference(gold):
    g = gold["step"]
    ucfg, vcfg, tcfg = g["cfg"]["unet"], g["cfg"]["vit"], g["cfg"]["text"]
    su, se, st = g["seeds"]
    sd_u = O.synth_state_dict(S.unet_param_shapes(ucfg), su)
    sd_e = O.synth_state_dict(O.encoder_param_shapes(vcfg, O.pooled_feature_dim(ucfg), tcfg["width"], 129), se)
    sd_t = O.synth_state_dict(O.text_param_shapes(tcfg), st)
    for k in sd_u:
        if "wo" in k:
            sd_u[k].requires_grad_(True)
    batch = O.synth_batch(g["B"], seed=g["batch_seed"], latent_hw=16, image_hw=64)
    batch["input_ids"] = g["input_ids"]
    assert (g["input_ids"] == 0).any(), "the prompts are padded with id 0"
    ref = S.pretrain_step(sd_u, ucfg, sd_e, vcfg, sd_t, tcfg, batch, prediction_type="v_prediction", pad_id=g["pad_id"])
    for k in ("loss", "loss_diff", "loss_reg"):
        assert abs(ref[k].item() - g[k]) <= 1e-4 * abs(g[k]), k
    assert _rel(ref["pred"], g["pred"]) < 1e-4 and _rel(ref["domain_embed"], g["domain_embed"]) < 1e-4
    ref["loss"].backward()
    errs = _grad_errs({k: v.grad for k, v in sd_u.items() if "wo" in k}, g["wo_grads"])
    vec = [e for k, e in errs.items() if not k.endswith(".v")]
    assert max(vec) < 1e-4, max(errs.items(), key=lambda kv: kv[1])
    eps = S.pretrain_step(sd_u, ucfg, sd_e, vcfg, sd_t, tcfg, batch, pad_id=g["pad_id"])
    assert abs(eps["loss_diff"].item() - g["loss_diff"]) > 1e-2 * g["loss_diff"]


def test_gelu_text_tower_pinned_to_transformers(gold):
    from transformers import CLIPTextConfig, CLIPTextModel
    p = gold["pin_text_gelu"]
    t = gold["step"]["cfg"]["text"]
    assert t["act"] == "gelu" and p["rel"] < 1e-5
    sd = O.synth_state_dict(O.text_param_shapes(t), gold["step"]["seeds"][2])
    cfg = CLIPTextConfig(vocab_size=t["vocab"], hidden_size=t["width"], intermediate_size=t["mlp"],
                         num_hidden_layers=t["layers"], num_attention_heads=t["heads"],
                         max_position_embeddings=t["positions"], hidden_act="gelu", layer_norm_eps=1e-5)
    hf = CLIPTextModel(cfg).eval()
    missing, unexpected = hf.load_state_dict(sd, strict=False)
    assert not unexpected and all("position_ids" in k for k in missing)
    with torch.no_grad():
        mine = S.text_forward(sd, t, input_ids=p["ids"])
        theirs = hf(input_ids=p["ids"]).last_hidden_state
        quick = S.text_forward(sd, dict(t, act="quick_gelu"), input_ids=p["ids"])
    assert _rel(mine, theirs) < 1e-5
    assert _rel(mine[:, :8], p["out_first8"]) < 1e-5
    assert _rel(quick, theirs) > 1e-3, "the activation switch changes nothing"


def test_get_velocity_matches_diffusers_formula():
    from e4t_b200.engine import add_noise, ddpm_alphas_cumprod, get_velocity
    g = torch.Generator().manual_seed(0)
    lat, noise = torch.randn(3, 4, 8, 8, generator=g), torch.randn(3, 4, 8, 8, generator=g)
    t = torch.tensor([0, 500, 999])
    acp = ddpm_alphas_cumprod()
    # diffusers 0.14 DDPMScheduler.get_velocity, literally
    sqrt_alpha_prod = (acp[t] ** 0.5).flatten()[:, None, None, None]
    sqrt_one_minus_alpha_prod = ((1 - acp[t]) ** 0.5).flatten()[:, None, None, None]
    want = sqrt_alpha_prod * noise - sqrt_one_minus_alpha_prod * lat
    assert torch.equal(get_velocity(lat, noise, t, acp), want)
    assert torch.equal(S.get_velocity(lat, noise, t), want)
    # v and the noisy sample give back x0 = √ᾱ·x_t − √(1−ᾱ)·v
    x_t = add_noise(lat, noise, t, acp)
    torch.testing.assert_close(sqrt_alpha_prod * x_t - sqrt_one_minus_alpha_prod * want, lat, atol=1e-5, rtol=0)


@pytest.mark.parametrize("eta", [0.0, 0.5])
def test_v_prediction_ddim_step_matches_diffusers_formula(eta):
    from e4t.pipeline_stable_diffusion_e4t import DDIMScheduler
    s = DDIMScheduler(prediction_type="v_prediction")
    s.set_timesteps(10)
    g = torch.Generator().manual_seed(1)
    x, v = torch.randn(2, 4, 8, 8, generator=g), torch.randn(2, 4, 8, 8, generator=g)
    for t in (int(s.timesteps[0]), int(s.timesteps[-1])):
        prev_t = t - 1000 // 10
        alpha_prod_t = s.alphas_cumprod[t]
        alpha_prod_t_prev = s.alphas_cumprod[prev_t] if prev_t >= 0 else s.final_alpha_cumprod
        beta_prod_t = 1 - alpha_prod_t
        # diffusers 0.14 DDIMScheduler.step, v_prediction branch, literally
        pred_original_sample = (alpha_prod_t ** 0.5) * x - (beta_prod_t ** 0.5) * v
        pred_epsilon = (alpha_prod_t ** 0.5) * v + (beta_prod_t ** 0.5) * x
        variance = (1 - alpha_prod_t_prev) / (1 - alpha_prod_t) * (1 - alpha_prod_t / alpha_prod_t_prev)
        std_dev_t = eta * variance ** 0.5
        pred_sample_direction = (1 - alpha_prod_t_prev - std_dev_t ** 2) ** 0.5 * pred_epsilon
        want = alpha_prod_t_prev ** 0.5 * pred_original_sample + pred_sample_direction
        gen = torch.Generator().manual_seed(5)
        out = s.step(v, t, x, eta=eta, generator=gen)
        if eta > 0:
            want = want + std_dev_t * torch.randn(x.shape, generator=torch.Generator().manual_seed(5))
        torch.testing.assert_close(out.prev_sample, want, atol=1e-6, rtol=1e-6)
        torch.testing.assert_close(out.pred_original_sample, pred_original_sample, atol=1e-6, rtol=1e-6)
        if eta == 0:
            torch.testing.assert_close(S.ddim_step(v, t, x, 10, prediction_type="v_prediction"), want,
                                       atol=1e-5, rtol=1e-5)


def test_epsilon_ddim_step_unchanged_by_default():
    from e4t.pipeline_stable_diffusion_e4t import DDIMScheduler
    a, b = DDIMScheduler(), DDIMScheduler(prediction_type="epsilon")
    a.set_timesteps(5); b.set_timesteps(5)
    g = torch.Generator().manual_seed(2)
    x, e = torch.randn(1, 4, 8, 8, generator=g), torch.randn(1, 4, 8, 8, generator=g)
    t = int(a.timesteps[1])
    assert torch.equal(a.step(e, t, x).prev_sample, b.step(e, t, x).prev_sample)
    torch.testing.assert_close(a.step(e, t, x).prev_sample, S.ddim_step(e, t, x, 5), atol=1e-6, rtol=1e-6)


def test_scheduler_from_config_and_from_pretrained(tmp_path):
    from e4t.pipeline_stable_diffusion_e4t import DDIMScheduler
    # the published SD 2.1 scheduler_config.json values (extra keys such as _class_name, trained_betas are ignored)
    cfg = {"_class_name": "DDIMScheduler", "beta_end": 0.012, "beta_schedule": "scaled_linear", "beta_start": 0.00085,
           "clip_sample": False, "num_train_timesteps": 1000, "prediction_type": "v_prediction",
           "set_alpha_to_one": False, "steps_offset": 1, "trained_betas": None}
    s = DDIMScheduler.from_config(cfg)
    assert s.prediction_type == "v_prediction" and s.steps_offset == 1
    assert torch.equal(s.alphas_cumprod, DDIMScheduler().alphas_cumprod)
    (tmp_path / "scheduler").mkdir()
    (tmp_path / "scheduler" / "scheduler_config.json").write_text(json.dumps(cfg))
    p = DDIMScheduler.from_pretrained(str(tmp_path), subfolder="scheduler")
    assert p.prediction_type == "v_prediction" and torch.equal(p.alphas_cumprod, s.alphas_cumprod)
    assert DDIMScheduler.from_config({}).prediction_type == "epsilon"
    s1 = DDIMScheduler.from_config(dict(cfg, set_alpha_to_one=True, beta_end=0.02))
    assert s1.final_alpha_cumprod.item() == 1.0 and not torch.equal(s1.alphas_cumprod, s.alphas_cumprod)


@pytest.mark.parametrize("bad", [dict(beta_schedule="linear"), dict(beta_schedule="squaredcos_cap_v2"),
                                 dict(clip_sample=True), dict(prediction_type="sample")])
def test_scheduler_refuses_unsupported_config(bad):
    from e4t.pipeline_stable_diffusion_e4t import DDIMScheduler
    with pytest.raises(ValueError):
        DDIMScheduler.from_config(dict({"beta_schedule": "scaled_linear"}, **bad))


@pytest.mark.parametrize("kind", ["sample", "eps", None])
def test_pretrain_step_refuses_unknown_prediction_type(kind):
    from e4t_b200.engine import PretrainStep, TuningStep
    # refused before any model is touched: the models here are placeholders
    for ctor in (PretrainStep, TuningStep):
        with pytest.raises(ValueError, match="'epsilon' or 'v_prediction'"):
            ctor(None, None, None, 49408, 320, prediction_type=kind)


def test_synth_ids_pad_id():
    ids, idxs = S.synth_input_ids([0, 5])
    ids0, idxs0 = S.synth_input_ids([0, 5], pad_id=0)
    assert idxs == idxs0 and torch.equal(ids, torch.where(ids0 == 0, O.EOS, ids0))
    assert ids0[0, idxs0[0] + 1] == O.EOS and ids0[0, idxs0[0] + 2] == 0
    assert S.empty_prompt_ids() == [O.BOS] + [O.EOS] * 76
    assert S.empty_prompt_ids(0) == [O.BOS, O.EOS] + [0] * 75
