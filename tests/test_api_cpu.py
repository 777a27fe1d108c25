"""CPU checks of the drop-in boundary: module API / state-dict key contract of the `e4t` mirror, the C-ABI library
(loads, exports every symbol include/e4t_b200.h declares — no compute calls), host-side helpers."""
import ctypes
import os
import re

import pytest
import torch

from oracle import e4t_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from e4t_b200 import _lib
    if not os.path.exists(_lib.lib_path()):
        import importlib.util
        spec = importlib.util.spec_from_file_location("build", os.path.join(ROOT, "e4t-diffusion_b200", "csrc", "build.py"))
        b = importlib.util.module_from_spec(spec); spec.loader.exec_module(b); b.build()
    lib = ctypes.CDLL(_lib.lib_path())
    hdr = open(os.path.join(ROOT, "include", "e4t_b200.h")).read()
    names = re.findall(r"\b(e4t_[a-z0-9_]+)\s*\(", hdr)
    assert len(names) >= 20
    for n in set(names):
        assert hasattr(lib, n), f"{n} declared in include/e4t_b200.h but not exported"
    lib.e4t_version.restype = ctypes.c_int
    assert lib.e4t_version() >= 100


def test_unet_state_dict_keys_match_reference_inventory():
    import hashlib
    from e4t.models.unet_2d_condition import UNet2DConditionModel
    m = UNet2DConditionModel(**O.ref_unet_kwargs(O.TINY_UNET))
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == O.unet_param_shapes(O.TINY_UNET)
    # "wo" selects exactly the WeightOffsets parameters (pretrain_e4t.py:276-278, utils.py:130)
    for n, _ in m.named_parameters():
        assert ("wo" in n) == (".wo_" in n)
    # SD-v1.4 inventory hash vs the reference's state_dict (tests/golden/inventory.pt) without building 1 B params
    inv = torch.load(os.path.join(ROOT, "tests", "golden", "inventory.pt"))
    with torch.device("meta"):
        big = UNet2DConditionModel(**O.ref_unet_kwargs(O.SD14_UNET))
    sd = big.state_dict()
    keys = sorted(sd)
    sha = hashlib.sha256("\n".join(f"{k}:{tuple(sd[k].shape)}" for k in keys).encode()).hexdigest()
    assert sha == inv["sha256"]
    assert sum(p.numel() for n, p in big.named_parameters() if "wo" not in n) == 859520964
    assert sum(p.numel() for n, p in big.named_parameters() if "wo" in n) == 143226592


def test_config_surface_and_api():
    from e4t.models.unet_2d_condition import UNet2DConditionModel
    from e4t.models.cross_attention import CrossAttention, B200AttnProcessor
    m = UNet2DConditionModel(**O.ref_unet_kwargs(O.TINY_UNET))
    assert m.config.cross_attention_dim == 64 and m.config["layers_per_block"] == 1 and m.in_channels == 4
    assert m.dtype == torch.float32 and m.device.type == "cpu" and m.sample_size == 16
    procs = m.attn_processors
    assert len(procs) == 2 * 4 and all(k.endswith(".processor") for k in procs)
    m.set_attn_processor(B200AttnProcessor())
    m.enable_xformers_memory_efficient_attention()     # must exist (pretrain_e4t.py:269), no-op
    m.set_attention_slice("auto")
    a = CrossAttention(query_dim=64, cross_attention_dim=96, heads=4, dim_head=16)
    assert a.wo_k.linear_column.weight.shape == (96, 96) and a.wo_k.linear_row.weight.shape == (64, 64)
    assert a.to_q.bias is None and a.to_out[0].bias is not None and a.scale == 16 ** -0.5


def test_weightoffsets_forward_matches_literal_reference_sequence():
    from e4t.weightoffsets import WeightOffsets
    w = WeightOffsets(24, 16).double()
    sd = {"p." + k: v for k, v in w.state_dict().items()}
    assert tuple(w().shape) == (16, 24)
    assert torch.allclose(w(), O.wo_delta(sd, "p."), atol=1e-12)


def test_encoder_and_text_module_contract():
    from e4t.encoder import E4TEncoder
    from e4t.models.modeling_clip import CLIPTextConfig, CLIPTextModel
    with torch.device("meta"):
        e = E4TEncoder.__new__(E4TEncoder)
    e = E4TEncoder(arch="ViT-tiny-test", word_embedding_dim=64, n_odd_layers=129, unet_feature_dim=448, clip_model="ignored")
    assert {k: tuple(v.shape) for k, v in e.state_dict().items()} == O.encoder_param_shapes(O.VIT_TINY, 448, 64, 129)
    assert not any(p.requires_grad for p in e.clip_vision.parameters())
    assert "mean" not in e.state_dict() and e.dtype == torch.float32
    assert e.first_linears[7].weight.data_ptr() == e._fl_w[7].data_ptr()
    t = O.CLIP_TEXT_TINY
    m = CLIPTextModel(CLIPTextConfig(vocab_size=49408, hidden_size=t["width"], intermediate_size=t["mlp"],
                                     num_hidden_layers=t["layers"], num_attention_heads=t["heads"]))
    m.resize_token_embeddings(49409)                      # pretrain_e4t.py:254-259
    assert m.get_input_embeddings().weight.shape[0] == 49409
    sd = O.synth_state_dict(O.text_param_shapes(t), 5)
    m.load_state_dict(sd)
    ids, idxs = O.synth_input_ids([0, 7])
    with torch.no_grad():
        a = m(inputs_embeds=m.get_input_embeddings()(ids))[0]
        b = O.text_forward(sd, t, input_ids=ids)
    assert torch.allclose(a, b, atol=2e-5)


def test_attribute_dict_and_checkpoint_filters(tmp_path):
    from e4t.utils import AttributeDict, load_config_from_pretrained
    import json
    (tmp_path / "config.json").write_text(json.dumps({"pretrained_model_name_or_path": "x", "reg_lambda": 0.01}))
    cfg = load_config_from_pretrained(str(tmp_path))
    assert cfg.reg_lambda == 0.01 and cfg.not_there is None and isinstance(cfg, AttributeDict)


def test_wo_bank_record_layout_matches_library():
    """The ctypes mirror of the device table record (e4t_b200/wobank.py) matches csrc/elementwise.cu's WOProj."""
    from e4t_b200 import _lib
    from e4t_b200.wobank import _WOProj
    lib = _lib.load()
    lib.e4t_wo_bank_record_size.restype = ctypes.c_int
    assert lib.e4t_wo_bank_record_size() == ctypes.sizeof(_WOProj) == 23 * 8 + 8


@pytest.mark.parametrize("query_dim,cross_dim,heads,dim_head,bad", [
    (64, 30, 4, 16, "to_k: 30 in-"),         # kv in-features not a multiple of 8
    (36, None, 4, 16, "to_q: 36 in-"),       # self-attention, query_dim 36 (a multiple of 4, not of 8)
    (64, 96, 3, 4, "to_q: 64 in- and 12 out-"),  # inner dim 12
])
def test_wo_bank_refuses_sides_that_are_not_multiples_of_8(query_dim, cross_dim, heads, dim_head, bad):
    """The bank's vector loads and the projection GEMMs need R and C to be multiples of 8: WOBank refuses other shapes
    when it is built, before it allocates anything or calls the library (so this runs on the CPU)."""
    from e4t.models.cross_attention import CrossAttention
    from e4t_b200.wobank import WOBank
    ok = CrossAttention(query_dim=64, cross_attention_dim=768, heads=8, dim_head=8)
    badm = CrossAttention(query_dim=query_dim, cross_attention_dim=cross_dim, heads=heads, dim_head=dim_head)
    with pytest.raises(ValueError, match=r"attention module 1 \(CrossAttention\), " + re.escape(bad)):
        WOBank([ok, badm])


@pytest.mark.parametrize("R,C", [(8, 8), (24, 16), (40, 72)])
def test_wo_closed_form_gradients_match_autograd(R, C):
    """SURVEY.md Appendix A backward identities (what wo_bank_*_kernel implement) vs autograd of the literal module."""
    torch.manual_seed(R * 100 + C)
    sd = {k: torch.randn(s, dtype=torch.float64) for k, s in O._wo_shapes("p.", R, C).items()}
    for v in sd.values():
        v.requires_grad_(True)
    W = torch.randn(C, R, dtype=torch.float64)
    dWeff = torch.randn(C, R, dtype=torch.float64)
    ((W * (1 + O.wo_delta(sd, "p."))) * dWeff).sum().backward()
    with torch.no_grad():
        v, w1, b1 = sd["p.v"], sd["p.linear1.weight"][:, 0], sd["p.linear1.bias"]
        w2, b2 = sd["p.linear2.weight"][:, 0], sd["p.linear2.bias"]
        Wc, bc, Wr = sd["p.linear_column.weight"], sd["p.linear_column.bias"], sd["p.linear_row.weight"]
        vx, vy = w1 * v + b1, w2 * v + b2
        a, b, s = Wc @ vx, Wr @ vy, Wr.sum(1)
        G = dWeff * W
        Ga, Gbc, G1, GTb, GTs = G @ a, G @ bc, G.sum(1), G.t() @ b, G.t() @ s
        dvy, dvx = Wr.t() @ Ga, Wc.t() @ GTb
        exp = {"p.linear_row.weight": Ga[:, None] * vy[None, :] + Gbc[:, None], "p.linear_row.bias": G1,
               "p.linear_column.weight": GTb[:, None] * vx[None, :], "p.linear_column.bias": GTs,
               "p.linear2.weight": (dvy * v)[:, None], "p.linear2.bias": dvy, "p.linear1.weight": (dvx * v)[:, None],
               "p.linear1.bias": dvx, "p.v": (w1 @ dvx + w2 @ dvy).reshape(1)}
    for k, e in exp.items():
        assert torch.allclose(sd[k].grad, e, rtol=1e-10, atol=1e-10), k
