"""Oracle of the domain-tuning step with a trainable text encoder (tuning_e4t.py:280-314, --train_text_encoder), in
fp32 torch on the restated modules of oracle/e4t_oracle.py.  It differs from `e4t_oracle.pretrain_step` in two places
only: the token-embedding lookup keeps its gradient, and class_embed / ehs_e4t are read, without gradient, from the
text weights as they are at this step."""
import torch
import torch.nn.functional as F

from oracle import e4t_oracle as O


def tuning_step_text(sd_unet, ucfg, sd_enc, vcfg, sd_text, tcfg, batch, class_token_id=320, domain_embed_scale=0.1,
                     reg_lambda=1e-4):
    pixel_values, latents, noise = batch["pixel_values"], batch["latents"], batch["noise"]
    timesteps, input_ids = batch["timesteps"], batch["input_ids"]
    B = latents.shape[0]
    emb_w = sd_text["text_model.embeddings.token_embedding.weight"]
    class_embed = emb_w[class_token_id].detach()                                                      # :280-281
    ids_e4t = torch.tensor([[O.BOS] + [O.EOS] * 76], dtype=torch.int64, device=latents.device)
    with torch.no_grad():
        ehs_e4t = O.text_forward(sd_text, tcfg, input_ids=ids_e4t)                                    # :282-287
    inputs_embeds = emb_w[input_ids]                                                                  # :297, with grad
    idxs = [row.index(O.PLACEHOLDER_ID) for row in input_ids.tolist()]
    noisy = O.add_noise(latents, noise, timesteps)
    enc = O.unet_forward(sd_unet, ucfg, noisy, timesteps, ehs_e4t.expand(B, -1, -1), return_encoder_outputs=True)
    domain_embed = O.encoder_forward(sd_enc, vcfg, pixel_values, enc["down_block_samples"])
    domain_embed = class_embed.clone().expand(B, -1) + domain_embed_scale * domain_embed
    for i, idx in enumerate(idxs):                                                                    # :310-311
        inputs_embeds[i, idx, :] = domain_embed[i]
    ehs = O.text_forward(sd_text, tcfg, inputs_embeds=inputs_embeds)                                  # :314
    pred = O.unet_forward(sd_unet, ucfg, noisy, timesteps, ehs)
    loss_diff = F.mse_loss(pred.float(), noise.float(), reduction="mean")
    loss_reg = reg_lambda * domain_embed.pow(2).sum()
    return dict(loss=loss_diff + loss_reg, loss_diff=loss_diff, loss_reg=loss_reg, pred=pred,
                domain_embed=domain_embed, placeholder_idxs=idxs)
