"""Golden fixture of the Stable Diffusion 2.x model shapes, made by running the REFERENCE's own modules (imported
unchanged from a checkout of mkshing/e4t-diffusion named by $E4T_REFERENCE_DIR, via oracle/shim) on seeded synthetic
weights:

    E4T_REFERENCE_DIR=/path/to/e4t-diffusion python oracle/gen_golden_sd2.py   # writes tests/golden/sd2.pt (< 1 MB)

It holds
  * `unet`: a tiny SD2-shaped UNet (linear proj_in / proj_out, 2 and 4 heads of 32, upcast_attention, 96-wide context)
    -- forward, pooled encoder outputs and every WeightOffsets gradient of a weighted sum of both (as gen_golden.py);
  * `inventory`: keys, shapes, parameter counts and sha256 of the full SD 2.x UNet (sd2_oracle.SD2_UNET);
  * `step`: one tiny v-prediction pre-training step (pretrain_e4t.py:616-647 with the :638-643 v_prediction branch and
    the SD 2.x empty prompt padded with id 0): losses, pred, domain embedding and the WeightOffsets gradients;
  * `pin_text_gelu`: the oracle's exact-GELU text tower against transformers.CLIPTextModel(hidden_act="gelu").
Everything is fp32 on CPU.
"""
import hashlib
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
# a checkout of mkshing/e4t-diffusion (its modules are imported unchanged; nothing of it is stored in this repository)
REFERENCE = os.environ.get("E4T_REFERENCE_DIR", os.path.join(ROOT, "..", "e4t-diffusion"))
sys.path[:0] = [REFERENCE, os.path.join(HERE, "shim"), ROOT]

from oracle import e4t_oracle as O  # noqa: E402
from oracle import sd2_oracle as S  # noqa: E402
from oracle.golden_format import compact_grads  # noqa: E402

from e4t.models.unet_2d_condition import UNet2DConditionModel  # noqa: E402  (the reference's)

OUT = os.path.join(ROOT, "tests", "golden")

# tiny SD2-shaped configurations (tests/test_sd2_cpu.py and tests/test_sd2_gpu.py rebuild the same models from them)
TINY_SD2_UNET = dict(in_channels=4, out_channels=4, block_out_channels=(64, 128), layers_per_block=1,
                     attention_head_dim=(2, 4), cross_attention_dim=96, norm_num_groups=32, norm_eps=1e-5,
                     sample_size=16, flip_sin_to_cos=True, freq_shift=0, use_linear_projection=True,
                     upcast_attention=True)
TINY_SD2_TEXT = dict(width=96, layers=2, heads=4, mlp=192, vocab=49409, positions=77, act="gelu")
SEED_U, SEED_E, SEED_T = 21, 22, 23
STEP_B, STEP_SEED, STEP_TEMPLATES, PAD_ID = 2, 7, (3, 8), 0


def hf_text(sd, t):
    from transformers import CLIPTextConfig, CLIPTextModel
    cfg = CLIPTextConfig(vocab_size=t["vocab"], hidden_size=t["width"], intermediate_size=t["mlp"],
                         num_hidden_layers=t["layers"], num_attention_heads=t["heads"],
                         max_position_embeddings=t["positions"], hidden_act=t["act"], layer_norm_eps=1e-5,
                         eos_token_id=O.EOS, bos_token_id=O.BOS, pad_token_id=PAD_ID)
    hf = CLIPTextModel(cfg).eval()
    missing, unexpected = hf.load_state_dict(sd, strict=False)
    assert not unexpected and all("position_ids" in k for k in missing), (missing, unexpected)
    return hf


def rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt().clamp_min(1e-30)).item()


def wo_summary(named, limit):
    """WeightOffsets gradients: whole up to `limit` entries, else a 16 x 16 corner and the norm."""
    out = {}
    for k, p in named.items():
        if p.grad.numel() <= limit:
            out[k] = p.grad.clone()
        else:
            out[k + "#corner"] = p.grad[:16, :16].clone()
            out[k + "#norm"] = p.grad.norm()
    return compact_grads(out)


def build_ref_unet(cfg, seed):
    m = UNet2DConditionModel(**O.ref_unet_kwargs(cfg))
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == S.unet_param_shapes(cfg)
    sd = O.synth_state_dict(S.unet_param_shapes(cfg), seed)
    m.load_state_dict(sd, strict=True)
    return m


def unet_case(cfg, B, seed, hw):
    """As oracle/gen_golden.py:unet_case (same input draws, so O.golden_unet_inputs re-draws them)."""
    g = torch.Generator().manual_seed(seed + 17)
    m = build_ref_unet(cfg, seed)
    x = torch.randn(B, 4, hw, hw, generator=g)
    t = torch.randint(0, 1000, (B,), generator=g)
    ehs = torch.randn(B, 77, cfg["cross_attention_dim"], generator=g).requires_grad_(True)
    w = torch.randn(B, 4, hw, hw, generator=g)
    out = m(x, t, ehs).sample
    enc = m(x, t, ehs, return_encoder_outputs=True)["down_block_samples"]
    wenc = [torch.randn(e.shape, generator=g) for e in enc]
    ((out * w).sum() + sum((e * we).sum() for e, we in zip(enc, wenc))).backward()
    return dict(cfg=cfg, seed=seed, B=B, x=x, t=t, ehs=ehs.detach().clone(), w=w, out=out.detach().clone(),
                enc_pooled=torch.cat([e.mean(dim=(2, 3)) for e in enc], dim=-1).detach().clone(),
                enc_shapes=[tuple(e.shape) for e in enc], d_ehs=ehs.grad.clone(),
                wo_grads=wo_summary({k: p for k, p in m.named_parameters() if "wo" in k}, 4096))


def inventory(cfg):
    m = UNet2DConditionModel(**O.ref_unet_kwargs(cfg))
    sd = m.state_dict()
    shapes = {k: tuple(v.shape) for k, v in sd.items()}
    assert shapes == S.unet_param_shapes(cfg)
    keys = sorted(shapes)
    return dict(sha256=hashlib.sha256("\n".join(f"{k}:{shapes[k]}" for k in keys).encode()).hexdigest(),
                n_keys=len(keys), n_base=sum(p.numel() for k, p in m.named_parameters() if "wo" not in k),
                n_wo=sum(p.numel() for k, p in m.named_parameters() if "wo" in k),
                n_wo_tensors=sum(1 for k, _ in m.named_parameters() if "wo" in k))


def step_case():
    """One v-prediction step: the reference UNet for both passes, the oracle's encoder and text tower (pinned
    elsewhere), autograd for the WeightOffsets gradients."""
    ucfg, vcfg, tcfg = TINY_SD2_UNET, O.VIT_TINY, TINY_SD2_TEXT
    unet = build_ref_unet(ucfg, SEED_U)
    wo = {}
    for k, p in unet.named_parameters():
        p.requires_grad_("wo" in k)
        if "wo" in k:
            wo[k] = p
    sd_e = O.synth_state_dict(O.encoder_param_shapes(vcfg, O.pooled_feature_dim(ucfg), tcfg["width"], 129), SEED_E)
    sd_t = O.synth_state_dict(O.text_param_shapes(tcfg), SEED_T)
    batch = O.synth_batch(STEP_B, seed=STEP_SEED, latent_hw=16, image_hw=64)
    batch["input_ids"], _ = S.synth_input_ids(STEP_TEMPLATES, pad_id=PAD_ID)
    B = STEP_B
    emb_w = sd_t["text_model.embeddings.token_embedding.weight"]
    with torch.no_grad():
        ehs_e4t = S.text_forward(sd_t, tcfg, input_ids=torch.tensor([S.empty_prompt_ids(PAD_ID)]))
    latents, noise, t = batch["latents"], batch["noise"], batch["timesteps"]
    inputs_embeds = emb_w[batch["input_ids"]].detach().clone()
    idxs = [row.index(O.PLACEHOLDER_ID) for row in batch["input_ids"].tolist()]
    noisy = O.add_noise(latents, noise, t)
    enc = unet(noisy, t, ehs_e4t.expand(B, -1, -1), return_encoder_outputs=True)
    dom = O.encoder_forward(sd_e, vcfg, batch["pixel_values"], enc["down_block_samples"])
    dom = emb_w[320].detach().clone().expand(B, -1) + 0.1 * dom
    for i, idx in enumerate(idxs):
        inputs_embeds[i, idx, :] = dom[i]
    ehs = S.text_forward(sd_t, tcfg, inputs_embeds=inputs_embeds)
    pred = unet(noisy, t, ehs).sample
    target = S.get_velocity(latents, noise, t)                                  # pretrain_e4t.py:641-643
    loss_diff = torch.nn.functional.mse_loss(pred.float(), target.float(), reduction="mean")
    loss_reg = 0.01 * dom.pow(2).sum()
    (loss_diff + loss_reg).backward()
    return dict(cfg=dict(unet=ucfg, vit=vcfg, text=tcfg), seeds=(SEED_U, SEED_E, SEED_T), B=B, batch_seed=STEP_SEED,
                pad_id=PAD_ID, input_ids=batch["input_ids"], loss=(loss_diff + loss_reg).item(),
                loss_diff=loss_diff.item(), loss_reg=loss_reg.item(), pred=pred.detach().clone(),
                domain_embed=dom.detach().clone(), wo_grads=wo_summary(wo, 256))


def main():
    torch.manual_seed(0)
    torch.set_num_threads(os.cpu_count())
    rec = {}
    print("tiny sd2 unet")
    rec["unet"] = unet_case(TINY_SD2_UNET, 2, 5, 16)
    print("sd2 inventory")
    rec["inventory"] = inventory(S.SD2_UNET)
    print(rec["inventory"])
    print("v-prediction step")
    rec["step"] = step_case()
    print({k: rec["step"][k] for k in ("loss", "loss_diff", "loss_reg")})
    sd_t = O.synth_state_dict(O.text_param_shapes(TINY_SD2_TEXT), SEED_T)
    ids, _ = S.synth_input_ids([0, 5, 9], pad_id=PAD_ID)
    with torch.no_grad():
        hf = hf_text(sd_t, TINY_SD2_TEXT)(input_ids=ids).last_hidden_state
        rec["pin_text_gelu"] = dict(ids=ids, out_first8=hf[:, :8].clone(),
                                    rel=rel(S.text_forward(sd_t, TINY_SD2_TEXT, input_ids=ids), hf))
    print("pin_text_gelu", rec["pin_text_gelu"]["rel"])
    assert rec["pin_text_gelu"]["rel"] < 1e-5
    path = os.path.join(OUT, "sd2.pt")
    torch.save(rec, path)
    print("wrote", path, os.path.getsize(path))


if __name__ == "__main__":
    main()
