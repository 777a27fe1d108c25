"""The CPU oracle for Stable Diffusion 2.x base models (stabilityai/stable-diffusion-2-1, 768-v) -- TEST INFRASTRUCTURE.

What differs from SD 1.x, restated on e4t_oracle's blocks:
  * UNet: `attention_head_dim` is the head COUNT (unet_2d_condition.py:123,132,153), one int or one per level with the
    mid block taking the last; `use_linear_projection` makes proj_in / proj_out nn.Linear, applied after / before the
    token reshape (transformer_2d.py:150-153,206-209,254-261).  `upcast_attention` changes nothing in fp32.
  * Text tower: `act` ("quick_gelu" or "gelu") is CLIPTextConfig.hidden_act.
  * Objective: prediction_type "v_prediction" trains against diffusers 0.14 DDPMScheduler.get_velocity
    (pretrain_e4t.py:638-643) and samples with the v branch of DDIMScheduler.step.
  * Empty prompt: the SD 2.x tokenizer pads with id 0 (`pad_id`), after [BOS, EOS].
With an int head count, no linear projection, quick_gelu, epsilon and pad id EOS every function here computes what its
e4t_oracle namesake computes.  Pinned by tests/golden/sd2.pt (oracle/gen_golden_sd2.py)."""
import torch
import torch.nn.functional as F

from oracle import e4t_oracle as O

# Stable Diffusion 2.x (768-v): 5 / 10 / 20 / 20 heads of 64, linear proj_in / proj_out, OpenCLIP ViT-H text tower
# (23 layers of 1024, exact GELU), v-prediction; E4T word_embedding_dim=1024
SD2_UNET = dict(in_channels=4, out_channels=4, block_out_channels=(320, 640, 1280, 1280), layers_per_block=2,
                attention_head_dim=(5, 10, 20, 20), cross_attention_dim=1024, norm_num_groups=32, norm_eps=1e-5,
                sample_size=96, flip_sin_to_cos=True, freq_shift=0, use_linear_projection=True, upcast_attention=True)
CLIP_TEXT_SD2 = dict(width=1024, layers=23, heads=16, mlp=4096, vocab=49409, positions=77, act="gelu")
PREDICTION_TYPES = ("epsilon", "v_prediction")


def unet_param_shapes(cfg):
    """e4t_oracle.unet_param_shapes with nn.Linear proj_in / proj_out under use_linear_projection."""
    s = O.unet_param_shapes(cfg)
    if cfg.get("use_linear_projection", False):
        for k, shp in s.items():
            if k.endswith(("proj_in.weight", "proj_out.weight")) and len(shp) == 4:
                s[k] = shp[:2]
    return s


def transformer_2d(sd, p, x, ctx, heads, groups, linear=False):
    """Transformer2DModel.forward, continuous path (transformer_2d.py:248-286)."""
    if not linear:
        return O.transformer_2d(sd, p, x, ctx, heads, groups)
    B, C, H, W = x.shape
    h = F.group_norm(x, groups, sd[p + "norm.weight"], sd[p + "norm.bias"], 1e-6)
    h = F.linear(h.permute(0, 2, 3, 1).reshape(B, H * W, C), sd[p + "proj_in.weight"], sd[p + "proj_in.bias"])
    h = O.transformer_block(sd, p + "transformer_blocks.0.", h, ctx, heads)
    h = F.linear(h, sd[p + "proj_out.weight"], sd[p + "proj_out.bias"])
    return h.reshape(B, H, W, C).permute(0, 3, 1, 2) + x


def unet_forward(sd, cfg, sample, timesteps, ehs, return_encoder_outputs=False):
    """UNet2DConditionModel.forward (unet_2d_condition.py:410-562) with per-level heads and linear projections."""
    boc, L = cfg["block_out_channels"], cfg["layers_per_block"]
    groups, eps = cfg["norm_num_groups"], cfg["norm_eps"]
    n = len(boc)
    heads = cfg["attention_head_dim"]
    heads = (heads,) * n if isinstance(heads, int) else tuple(heads)
    lin = cfg.get("use_linear_projection", False)
    if not torch.is_tensor(timesteps):
        timesteps = torch.tensor([timesteps], dtype=torch.int64)
    elif timesteps.dim() == 0:
        timesteps = timesteps[None]
    timesteps = timesteps.expand(sample.shape[0])
    t_emb = O.timestep_embedding(timesteps, boc[0], cfg["flip_sin_to_cos"], cfg["freq_shift"]).to(sample.dtype)
    emb = F.linear(F.silu(F.linear(t_emb, sd["time_embedding.linear_1.weight"], sd["time_embedding.linear_1.bias"])),
                   sd["time_embedding.linear_2.weight"], sd["time_embedding.linear_2.bias"])
    x = F.conv2d(sample, sd["conv_in.weight"], sd["conv_in.bias"], padding=1)
    res = [x]
    for i in range(n):
        for j in range(L):
            x = O.resnet_block(sd, f"down_blocks.{i}.resnets.{j}.", x, emb, groups, eps)
            if i < n - 1:
                x = transformer_2d(sd, f"down_blocks.{i}.attentions.{j}.", x, ehs, heads[i], groups, lin)
            res.append(x)
        if i < n - 1:
            x = F.conv2d(x, sd[f"down_blocks.{i}.downsamplers.0.conv.weight"],
                         sd[f"down_blocks.{i}.downsamplers.0.conv.bias"], stride=2, padding=1)
            res.append(x)
    x = O.resnet_block(sd, "mid_block.resnets.0.", x, emb, groups, eps)
    x = transformer_2d(sd, "mid_block.attentions.0.", x, ehs, heads[-1], groups, lin)
    x = O.resnet_block(sd, "mid_block.resnets.1.", x, emb, groups, eps)
    if return_encoder_outputs:
        return dict(down_block_samples=tuple(res) + (x,))
    for i in range(n):
        for j in range(L + 1):
            x = torch.cat([x, res.pop()], dim=1)
            x = O.resnet_block(sd, f"up_blocks.{i}.resnets.{j}.", x, emb, groups, eps)
            if i > 0:
                x = transformer_2d(sd, f"up_blocks.{i}.attentions.{j}.", x, ehs, heads[n - 1 - i], groups, lin)
        if i < n - 1:
            x = F.interpolate(x, scale_factor=2.0, mode="nearest")
            x = F.conv2d(x, sd[f"up_blocks.{i}.upsamplers.0.conv.weight"],
                         sd[f"up_blocks.{i}.upsamplers.0.conv.bias"], padding=1)
    x = F.silu(F.group_norm(x, groups, sd["conv_norm_out.weight"], sd["conv_norm_out.bias"], eps))
    return F.conv2d(x, sd["conv_out.weight"], sd["conv_out.bias"], padding=1)


def text_forward(sd, t, inputs_embeds=None, input_ids=None, p="text_model."):
    """e4t_oracle.text_forward with the MLP activation of t["act"] (CLIPTextConfig.hidden_act)."""
    if t.get("act", "quick_gelu") == "quick_gelu":
        return O.text_forward(sd, t, inputs_embeds, input_ids, p)
    if inputs_embeds is None:
        inputs_embeds = sd[p + "embeddings.token_embedding.weight"][input_ids]
    W = t["width"]
    x = inputs_embeds + sd[p + "embeddings.position_embedding.weight"][:inputs_embeds.shape[1]]
    for i in range(t["layers"]):
        b = p + f"encoder.layers.{i}."
        h = F.layer_norm(x, (W,), sd[b + "layer_norm1.weight"], sd[b + "layer_norm1.bias"], 1e-5)
        w_in = torch.cat([sd[b + f"self_attn.{n}.weight"] for n in ("q_proj", "k_proj", "v_proj")])
        b_in = torch.cat([sd[b + f"self_attn.{n}.bias"] for n in ("q_proj", "k_proj", "v_proj")])
        x = x + O._mha(h, w_in, b_in, sd[b + "self_attn.out_proj.weight"], sd[b + "self_attn.out_proj.bias"],
                       t["heads"], causal=True)
        h = F.layer_norm(x, (W,), sd[b + "layer_norm2.weight"], sd[b + "layer_norm2.bias"], 1e-5)
        h = F.gelu(F.linear(h, sd[b + "mlp.fc1.weight"], sd[b + "mlp.fc1.bias"]))
        x = x + F.linear(h, sd[b + "mlp.fc2.weight"], sd[b + "mlp.fc2.bias"])
    return F.layer_norm(x, (W,), sd[p + "final_layer_norm.weight"], sd[p + "final_layer_norm.bias"], 1e-5)


def empty_prompt_ids(pad_id=O.EOS):
    """Token ids of the empty prompt padded to 77: [BOS, EOS, pad, ...]."""
    return [O.BOS, O.EOS] + [pad_id] * 75


def synth_input_ids(template_idxs, max_len=77, pad_id=O.EOS):
    """e4t_oracle.synth_input_ids with the positions after each row's first EOS set to pad_id."""
    ids, idxs = O.synth_input_ids(template_idxs, max_len)
    for row, idx in zip(ids, idxs):
        row[idx + 2:] = pad_id
    return ids, idxs


def get_velocity(latents, noise, timesteps, acp=None):
    """diffusers 0.14 DDPMScheduler.get_velocity (restated), indexed as e4t_oracle.add_noise is."""
    acp = (O.ddpm_alphas_cumprod() if acp is None else acp).to(latents.device)
    a = acp[timesteps].to(latents.dtype) ** 0.5
    s = (1 - acp[timesteps].to(latents.dtype)) ** 0.5
    return a.view(-1, 1, 1, 1) * noise - s.view(-1, 1, 1, 1) * latents


def pretrain_step(sd_unet, ucfg, sd_enc, vcfg, sd_text, tcfg, batch, class_token_id=320, domain_embed_scale=0.1,
                  reg_lambda=0.01, prediction_type="epsilon", pad_id=O.EOS):
    """Loop body pretrain_e4t.py:616-647, with the :638-643 prediction-type branch."""
    if prediction_type not in PREDICTION_TYPES:
        raise ValueError(f"Unknown prediction type {prediction_type}")
    pixel_values, latents, noise = batch["pixel_values"], batch["latents"], batch["noise"]
    timesteps, input_ids = batch["timesteps"], batch["input_ids"]
    B = latents.shape[0]
    emb_w = sd_text["text_model.embeddings.token_embedding.weight"]
    class_embed = emb_w[class_token_id].detach()
    with torch.no_grad():
        ehs_e4t = text_forward(sd_text, tcfg, input_ids=torch.tensor([empty_prompt_ids(pad_id)], device=latents.device))
    inputs_embeds = emb_w[input_ids].detach().clone()
    idxs = [row.index(O.PLACEHOLDER_ID) for row in input_ids.tolist()]
    noisy = O.add_noise(latents, noise, timesteps)
    enc = unet_forward(sd_unet, ucfg, noisy, timesteps, ehs_e4t.expand(B, -1, -1), return_encoder_outputs=True)
    domain_embed = O.encoder_forward(sd_enc, vcfg, pixel_values, enc["down_block_samples"])
    domain_embed = class_embed.clone().expand(B, -1) + domain_embed_scale * domain_embed
    for i, idx in enumerate(idxs):
        inputs_embeds[i, idx, :] = domain_embed[i]
    ehs = text_forward(sd_text, tcfg, inputs_embeds=inputs_embeds)
    pred = unet_forward(sd_unet, ucfg, noisy, timesteps, ehs)
    target = noise if prediction_type == "epsilon" else get_velocity(latents, noise, timesteps)
    loss_diff = F.mse_loss(pred.float(), target.float(), reduction="mean")
    loss_reg = reg_lambda * domain_embed.pow(2).sum()
    return dict(loss=loss_diff + loss_reg, loss_diff=loss_diff, loss_reg=loss_reg, pred=pred,
                domain_embed=domain_embed, placeholder_idxs=idxs)


def ddim_step(out, t, x, num_inference_steps, acp=None, num_train=1000, prediction_type="epsilon"):
    """e4t_oracle.ddim_step (eta = 0); with "v_prediction" `out` is the model's v and x₀ = √a_t·x − √(1−a_t)·v,
    ε = √a_t·v + √(1−a_t)·x (diffusers 0.14 DDIMScheduler.step)."""
    if prediction_type == "epsilon":
        return O.ddim_step(out, t, x, num_inference_steps, acp, num_train)
    acp = O.ddpm_alphas_cumprod() if acp is None else acp
    prev_t = t - num_train // num_inference_steps
    a_t = acp[t]
    a_prev = acp[prev_t] if prev_t >= 0 else acp[0]
    pred_x0 = a_t ** 0.5 * x - (1 - a_t) ** 0.5 * out
    eps = a_t ** 0.5 * out + (1 - a_t) ** 0.5 * x
    return a_prev ** 0.5 * pred_x0 + (1 - a_prev) ** 0.5 * eps


def pipeline_sample(sd_unet, ucfg, sd_enc, vcfg, sd_text, tcfg, image, input_ids, latents, num_inference_steps=4,
                    guidance_scale=7.5, class_token_id=320, domain_embed_scale=0.1, prediction_type="epsilon",
                    pad_id=O.EOS):
    """e4t_oracle.pipeline_sample (pipeline_stable_diffusion_e4t.py:181-216) on this file's UNet, text tower and
    DDIM step."""
    emb_w = sd_text["text_model.embeddings.token_embedding.weight"]
    bsz = latents.shape[0]
    idx = input_ids[0].tolist().index(O.PLACEHOLDER_ID)
    with torch.no_grad():
        ehs_e4t = text_forward(sd_text, tcfg, input_ids=torch.tensor([empty_prompt_ids(pad_id)])).expand(bsz, -1, -1)
        base_embeds = emb_w[input_ids]
        class_embed = emb_w[class_token_id]
        pix = image.expand(bsz, -1, -1, -1)
        x = latents.clone()
        for t in O.ddim_timesteps(num_inference_steps):
            tt = torch.full((bsz,), t, dtype=torch.int64)
            enc = unet_forward(sd_unet, ucfg, x, tt, ehs_e4t, return_encoder_outputs=True)
            dom = class_embed.expand(bsz, -1) + domain_embed_scale * O.encoder_forward(sd_enc, vcfg, pix,
                                                                                        enc["down_block_samples"])
            emb = base_embeds.expand(bsz, -1, -1).clone()
            emb[:, idx, :] = dom
            ehs = text_forward(sd_text, tcfg, inputs_embeds=emb)
            if guidance_scale > 1.0:
                out = unet_forward(sd_unet, ucfg, torch.cat([x, x]), torch.cat([tt, tt]), torch.cat([ehs_e4t, ehs]))
                u, c = out.chunk(2)
                out = u + guidance_scale * (c - u)
            else:
                out = unet_forward(sd_unet, ucfg, x, tt, ehs)
            x = ddim_step(out, t, x, num_inference_steps, prediction_type=prediction_type)
    return x
