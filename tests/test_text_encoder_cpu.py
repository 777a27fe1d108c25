"""Domain tuning with a trainable CLIP text encoder (tuning_e4t.py --train_text_encoder), host side: the oracle's text
gradients pinned to transformers' CLIPTextModel, the oracle step's text-training path, and the text_encoder.pt
checkpoint written from parameters that are views of one large storage (the optimiser arena)."""
import os
import sys

import torch

from oracle import e4t_oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from text_tuning_oracle import tuning_step_text  # noqa: E402


def _rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def test_oracle_text_gradients_match_transformers_clip_text():
    from transformers import CLIPTextConfig, CLIPTextModel
    t = O.CLIP_TEXT_TINY
    cfg = CLIPTextConfig(vocab_size=t["vocab"], hidden_size=t["width"], intermediate_size=t["mlp"],
                         num_hidden_layers=t["layers"], num_attention_heads=t["heads"],
                         max_position_embeddings=t["positions"], hidden_act="quick_gelu", layer_norm_eps=1e-5,
                         eos_token_id=O.EOS, bos_token_id=O.BOS, pad_token_id=O.EOS)
    hf = CLIPTextModel(cfg).eval()
    sd = O.synth_state_dict(O.text_param_shapes(t), 9)
    missing, unexpected = hf.load_state_dict(sd, strict=False)
    assert not unexpected and all("position_ids" in k for k in missing), (missing, unexpected)
    ids, _ = O.synth_input_ids([0, 5, 9])
    w = torch.randn(3, 77, t["width"], generator=torch.Generator().manual_seed(2))
    (hf(input_ids=ids).last_hidden_state * w).sum().backward()
    sdg = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    (O.text_forward(sdg, t, input_ids=ids) * w).sum().backward()
    named = dict(hf.named_parameters())
    assert set(sd) <= set(named)
    for k in sd:
        assert sdg[k].grad is not None and named[k].grad is not None, k
        if k.endswith("k_proj.bias"):      # softmax is invariant to a key bias: both gradients are rounding noise
            scale = named[k.replace("k_proj", "v_proj")].grad.norm()
            assert sdg[k].grad.norm() < 1e-5 * scale and named[k].grad.norm() < 1e-5 * scale, k
            continue
        assert _rel(sdg[k].grad, named[k].grad) <= 1e-4, (k, _rel(sdg[k].grad, named[k].grad))


def _tiny_step_inputs():
    ucfg, vcfg, tcfg = O.TINY_UNET, O.VIT_TINY, O.CLIP_TEXT_TINY
    fd = O.pooled_feature_dim(ucfg)
    sd_u = O.synth_state_dict(O.unet_param_shapes(ucfg), 1)
    sd_e = O.synth_state_dict(O.encoder_param_shapes(vcfg, fd, tcfg["width"], 129), 2)
    sd_t = O.synth_state_dict(O.text_param_shapes(tcfg), 3)
    return (ucfg, vcfg, tcfg), (sd_u, sd_e, sd_t), O.synth_batch(2, seed=42, latent_hw=16, image_hw=64)


def test_oracle_step_text_training_path():
    """Same forward as the frozen path; gradients reach every text parameter, and the overwritten placeholder
    positions send none to the token table (tuning_e4t.py:297-314)."""
    (ucfg, vcfg, tcfg), (sd_u, sd_e, sd_t), batch = _tiny_step_inputs()
    frozen = O.pretrain_step(sd_u, ucfg, sd_e, vcfg, sd_t, tcfg, batch, reg_lambda=1e-4)
    sdg = {k: v.clone().requires_grad_(True) for k, v in sd_t.items()}
    out = tuning_step_text(sd_u, ucfg, sd_e, vcfg, sdg, tcfg, batch, reg_lambda=1e-4)
    assert torch.equal(out["loss"].detach(), frozen["loss"])
    out["loss"].backward()
    assert all(v.grad is not None for v in sdg.values())
    g = sdg["text_model.embeddings.token_embedding.weight"].grad
    assert torch.count_nonzero(g[O.PLACEHOLDER_ID]) == 0                         # only ever at overwritten positions
    for i in torch.unique(batch["input_ids"]).tolist():
        if i != O.PLACEHOLDER_ID:
            assert torch.count_nonzero(g[i]) > 0, i


def test_text_checkpoint_roundtrip_from_arena_views(tmp_path):
    from e4t import utils
    from e4t.models.modeling_clip import CLIPTextConfig, CLIPTextModel

    def fresh():
        m = CLIPTextModel(CLIPTextConfig(vocab_size=49408, hidden_size=64, intermediate_size=128, num_hidden_layers=2,
                                         num_attention_heads=4))
        m.resize_token_embeddings(49409)                                         # + the placeholder token
        return m
    m = fresh()
    ps = list(m.parameters())
    arena = torch.zeros(sum(p.numel() for p in ps) + 1000)                      # parameters as views of one storage
    o = 0
    with torch.no_grad():
        for p in ps:
            arena[o:o + p.numel()].copy_(p.reshape(-1))
            p.data = arena[o:o + p.numel()].view(p.shape)
            o += p.numel()
    utils.save_text_encoder(m, str(tmp_path))
    sd = torch.load(tmp_path / "text_encoder.pt", map_location="cpu")
    assert all(v.untyped_storage().nbytes() == v.numel() * v.element_size() for v in sd.values())
    m2 = fresh()
    assert set(sd) == set(m2.state_dict())
    missing, unexpected = m2.load_state_dict(sd, strict=False)                  # inference.py:95-103
    assert not missing and not unexpected
    assert all(torch.equal(v, sd[k]) for k, v in m2.state_dict().items())
    assert all(torch.equal(v, m.state_dict()[k]) for k, v in sd.items())
