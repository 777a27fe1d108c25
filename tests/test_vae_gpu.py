"""GPU tests of the VAE path: the conv engine's wide rows and bottom/right-only padding, the row softmax, and
AutoencoderKL encode / decode (tiny and full SD-v1.x size) against an fp32 functional restatement of diffusers 0.14's
AutoencoderKL written below with torch ops only.

Tolerance rule for the models (DESIGN §4): the error of our bf16 path against the fp32 reference must be at most twice
the reference's own error when it runs under bf16 autocast (plus a small floor)."""

import math
import types

import pytest
import torch
import torch.nn.functional as F

from oracle import e4t_oracle as O
from oracle import vae_oracle as V

pytestmark = pytest.mark.gpu
torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False

TINY, SD = V.TINY_VAE, V.SD_VAE


def _rel(a, b):
    a = a.float(); b = b.float()
    return ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt().clamp_min(1e-12)).item()


def _mk(shape, g, scale=1.0):
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W,Cin,Cout", [(1, 512, 512, 128, 128), (2, 256, 256, 256, 256), (1, 64, 384, 64, 64)])
def test_conv3x3_wide_rows(B, H, W, Cin, Cout):
    from e4t_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(H + W + Cin)
    x = _mk((B, H, W, Cin), g)
    w = _mk((Cout, Cin, 3, 3), g, scale=0.05)
    bias = torch.randn(Cout, generator=g, device="cuda")
    res = _mk((B, H, W, Cout), g)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), bias, padding=1) + res.float().permute(0, 3, 1, 2)
    w9 = w.permute(2, 3, 0, 1).reshape(9, Cout, Cin).contiguous()
    out = ops.conv3x3(x, w9, bias=bias, residual=res, out_dtype=torch.float32)
    assert _rel(out.permute(0, 3, 1, 2), ref) < 2e-3


@pytest.mark.parametrize("pad_lo", [0, 1])
@pytest.mark.parametrize("B,H,W,Cin,Cout", [(1, 512, 512, 128, 128), (2, 64, 64, 256, 256), (2, 256, 256, 256, 128)])
def test_conv3x3_s2_pads(B, H, W, Cin, Cout, pad_lo):
    from e4t_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(H + Cin + pad_lo)
    x = _mk((B, H, W, Cin), g)
    w = _mk((Cout, Cin, 3, 3), g, scale=0.05)
    bias = torch.randn(Cout, generator=g, device="cuda")
    xf = x.float().permute(0, 3, 1, 2)
    if pad_lo == 0:   # diffusers Downsample2D(padding=0)
        ref = F.conv2d(F.pad(xf, (0, 1, 0, 1)), w.float(), bias, stride=2)
    else:
        ref = F.conv2d(xf, w.float(), bias, stride=2, padding=1)
    w9 = w.permute(2, 3, 0, 1).reshape(9, Cout, Cin).contiguous()
    out = ops.conv3x3_s2(x, w9, bias=bias, pad_lo=pad_lo)
    assert out.shape == (B, H // 2, W // 2, Cout)
    assert _rel(out.permute(0, 3, 1, 2), ref) < 4e-3


def test_conv3x3_unsupported_width_names_it():
    from e4t_b200 import ops
    from e4t_b200._lib import E4TError
    x = torch.zeros((1, 8, 192, 64), device="cuda", dtype=torch.bfloat16)
    w9 = torch.zeros((9, 64, 64), device="cuda", dtype=torch.bfloat16)
    with pytest.raises(E4TError, match="192"):
        ops.conv3x3(x, w9)


@pytest.mark.parametrize("rows,n,ld", [(4096, 4096, 4096), (77, 1000, 1024), (3, 16384, 16384), (5, 256, 260)])
def test_softmax_rows(rows, n, ld):
    from e4t_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(n + rows)
    x = (torch.randn((rows, ld), generator=g, device="cuda") * 8.0)[:, :n]
    out = ops.softmax_rows(x)
    ref = torch.softmax(x, dim=-1)
    assert out.dtype == torch.bfloat16
    assert (out.float() - ref).abs().max().item() <= 2.0 ** -8 * ref.max().item() + 1e-6
    assert torch.allclose(out.float().sum(-1), torch.ones(rows, device="cuda"), atol=2e-2)


# ------------------------------------------------------------------------------------------------------------------
# models, against the fp32 oracle (oracle/vae_oracle.py, pinned to the reference's blocks by tests/golden/vae.pt)
# ------------------------------------------------------------------------------------------------------------------
ref_encode, ref_decode = V.vae_encode, V.vae_decode


def _vae(cfg, seed):
    from e4t.models.autoencoder_kl import AutoencoderKL
    torch.manual_seed(seed)
    vae = AutoencoderKL(**cfg).cuda().eval().requires_grad_(False)
    sd = {k: v.float() for k, v in vae.state_dict().items()}
    return vae, sd


def _check_against_ref(ours, ref_fn, sd, cfg, inp):
    with torch.no_grad():
        ref = ref_fn(sd, cfg, inp)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ref16 = ref_fn(sd, cfg, inp).float()
    e_ours, e_ref = _rel(ours, ref), _rel(ref16, ref)
    assert e_ours <= 2.0 * e_ref + 1e-3, (e_ours, e_ref)
    return e_ours, e_ref


@pytest.mark.parametrize("cfg,hw", [(TINY, 64), (SD, 512)], ids=["tiny", "sd512"])
def test_vae_encode_decode(cfg, hw):
    vae, sd = _vae(cfg, 0)
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.rand((1, 3, hw, hw), generator=g, device="cuda") * 2 - 1
    with torch.no_grad():
        post = vae.encode(x).latent_dist
        moments = post.parameters
    lat = hw // 2 ** (len(cfg["block_out_channels"]) - 1)
    assert moments.shape == (1, 8, lat, lat)
    e = _check_against_ref(moments, ref_encode, sd, cfg, x)
    print(f"encode {hw}: ours {e[0]:.3e}  autocast {e[1]:.3e}")
    mean, logvar = torch.chunk(moments, 2, dim=1)
    assert torch.equal(post.mean, mean) and torch.equal(post.std, torch.exp(0.5 * logvar.clamp(-30, 20)))
    z = torch.randn(moments[:, :4].shape, generator=g, device="cuda")
    with torch.no_grad():
        dec = vae.decode(z).sample
    assert dec.shape == (1, 3, hw, hw) and dec.dtype == torch.float32
    e = _check_against_ref(dec, ref_decode, sd, cfg, z)
    print(f"decode {hw}: ours {e[0]:.3e}  autocast {e[1]:.3e}")


def test_vae_batch_sampling_and_dtype():
    vae, sd = _vae(TINY, 3)
    g = torch.Generator(device="cuda").manual_seed(4)
    x = torch.rand((3, 3, 64, 64), generator=g, device="cuda") * 2 - 1
    with torch.no_grad():
        post = vae.encode(x).latent_dist
        one = vae.encode(x[1:2]).latent_dist
        # per-image results do not depend on the batch
        assert _rel(one.mean, post.mean[1:2]) < 1e-2
        s1 = post.sample(generator=torch.Generator(device="cuda").manual_seed(7))
        s2 = post.mean + post.std * torch.randn(post.mean.shape, generator=torch.Generator(device="cuda").manual_seed(7),
                                                device="cuda")
        assert torch.equal(s1, s2)
        assert torch.equal(post.mode(), post.mean)
        out = vae(x, sample_posterior=False).sample
        assert out.shape == x.shape
        vae16 = vae.to(torch.bfloat16)
        dec16 = vae16.decode(post.mean.to(torch.bfloat16)).sample
        assert dec16.dtype == torch.bfloat16
        dec32 = vae16.decode(post.mean).sample
        assert _rel(dec16, dec32) < 5e-2     # the latents differ by their bf16 rounding


def test_vae_rejects_grad_and_cpu():
    from e4t.models.autoencoder_kl import AutoencoderKL
    from e4t_b200._lib import E4TError
    vae = AutoencoderKL(**TINY).cuda()
    x = torch.zeros((1, 3, 64, 64), device="cuda")
    with pytest.raises(NotImplementedError):
        vae.encode(x)
    vae.requires_grad_(False)
    with pytest.raises(E4TError):
        vae.encode(x.cpu())


def _tiny_models(seed_u=1, seed_e=2, seed_t=3, text_vocab=None):
    from e4t.encoder import E4TEncoder
    from e4t.models.modeling_clip import CLIPTextConfig, CLIPTextModel
    from e4t.models.unet_2d_condition import UNet2DConditionModel
    ucfg, vcfg, tcfg = O.TINY_UNET, O.VIT_TINY, O.CLIP_TEXT_TINY
    fd = O.pooled_feature_dim(ucfg)
    sd_u = O.synth_state_dict(O.unet_param_shapes(ucfg), seed_u)
    sd_e = O.synth_state_dict(O.encoder_param_shapes(vcfg, fd, tcfg["width"], 129), seed_e)
    sd_t = O.synth_state_dict(O.text_param_shapes(tcfg), seed_t)
    unet = UNet2DConditionModel(**O.ref_unet_kwargs(ucfg)); unet.load_state_dict(sd_u)
    enc = E4TEncoder(arch="ViT-tiny-test", word_embedding_dim=tcfg["width"], n_odd_layers=129, unet_feature_dim=fd)
    enc.load_state_dict(sd_e)
    vocab = tcfg["vocab"] if text_vocab is None else text_vocab
    text = CLIPTextModel(CLIPTextConfig(vocab_size=vocab, hidden_size=tcfg["width"], intermediate_size=tcfg["mlp"],
                                        num_hidden_layers=tcfg["layers"], num_attention_heads=tcfg["heads"]))
    sd_t_load = dict(sd_t)
    key = "text_model.embeddings.token_embedding.weight"
    sd_t_load[key] = sd_t[key][:vocab]
    text.load_state_dict(sd_t_load)
    return (unet.cuda(), enc.cuda(), text.cuda()), (sd_u, sd_e, sd_t)


def _oracle_vae(seed):
    """AutoencoderKL(TINY) on cuda with the oracle's synthetic weights, and those weights (fp32, CPU)."""
    from e4t.models.autoencoder_kl import AutoencoderKL
    sd = O.synth_state_dict(V.vae_param_shapes(TINY), seed)
    vae = AutoencoderKL(**TINY)
    vae.load_state_dict(sd)
    return vae.cuda().eval().requires_grad_(False), sd


def _step(vae, optimizer, seed=1):
    from e4t_b200.engine import PretrainStep
    (unet, enc, text), sds = _tiny_models(seed, seed + 1, seed + 2)
    return PretrainStep(unet, enc, text, O.PLACEHOLDER_ID, class_token_id=320, lr=1e-3, weight_dtype=torch.float32,
                        optimizer=optimizer, vae=vae), sds


def _pixel_batch(seed):
    b = O.synth_batch(2, seed=seed, latent_hw=16, image_hw=64)
    g = torch.Generator().manual_seed(seed + 1000)
    b["vae_noise"] = torch.randn(b["latents"].shape, generator=g)
    return b


def test_pretrain_step_with_vae_matches_oracle():
    """Loss of a step whose latents the VAE computes from pixels on the device, against the oracle step given the
    oracle VAE's latents for the same pixels and latent noise (the smoke() tolerance)."""
    vae, sd_v = _oracle_vae(21)
    step, (sd_u, sd_e, sd_t) = _step(vae, optimizer=False)
    batch = _pixel_batch(42)
    with torch.no_grad():
        ref_lat = V.vae_latents(sd_v, TINY, batch["pixel_values"], batch["vae_noise"])
        lat = step.encode_latents(batch["pixel_values"].cuda(), batch["vae_noise"].cuda())
    assert _rel(lat.cpu(), ref_lat) < 3e-2
    ref = O.pretrain_step(sd_u, O.TINY_UNET, sd_e, O.VIT_TINY, sd_t, O.CLIP_TEXT_TINY,
                          dict(batch, latents=ref_lat), class_token_id=320)
    out = step.forward_loss({k: v.cuda() for k, v in batch.items() if k != "latents"})
    lo, lg = ref["loss"].item(), out["loss"].item()
    print(f"[vae step] loss cuda {lg:.5f} vs oracle {lo:.5f}")
    assert abs(lo - lg) <= 3e-2 * abs(lo) + 1e-4, (lo, lg)
    step_plain, _ = _step(None, optimizer=False)
    with pytest.raises(KeyError):
        step_plain.forward_loss({k: v.cuda() for k, v in batch.items() if k not in ("latents", "vae_noise")})


@pytest.mark.parametrize("with_noise", [True, False], ids=["vae_noise", "device_randn"])
def test_pretrain_step_with_vae_cuda_graph_matches_eager(with_noise):
    """The VAE encode runs inside the captured whole-step graph: replays give the losses of eager steps.  Without
    `vae_noise` the latent noise is drawn on the device inside the graph, so the two runs are compared in
    distribution only (same RNG stream is not guaranteed): the loss must stay finite and close."""
    va, _ = _oracle_vae(21)
    vb, _ = _oracle_vae(21)
    A, _ = _step(va, optimizer=True, seed=5)
    Bs, _ = _step(vb, optimizer=True, seed=5)

    def mk(seed):
        b = {k: v.cuda() for k, v in _pixel_batch(seed).items() if k != "latents"}
        if not with_noise:
            b.pop("vae_noise")
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
    print(f"[vae graph, {'vae_noise' if with_noise else 'device randn'}] eager", la, "graph", lb)
    for x, y in zip(la, lb):
        assert math.isfinite(y)
        if with_noise:
            assert abs(x - y) <= 2e-3 * abs(x) + 1e-5
        else:
            assert abs(x - y) <= 0.25 * abs(x)


class _Tok:
    """Whitespace tokenizer over the oracle's fixed word ids."""
    model_max_length = 77

    def __init__(self):
        self.extra = {}

    def add_tokens(self, tok):
        if tok in self.extra:
            return 0
        self.extra[tok] = O.PLACEHOLDER_ID
        return 1

    def __len__(self):
        return 49408 + len(self.extra)

    def convert_tokens_to_ids(self, tok):
        return self.extra[tok]

    def __call__(self, text, padding=None, truncation=None, max_length=77, return_tensors=None, add_special_tokens=True):
        texts = [text] if isinstance(text, str) else text
        rows = []
        for s in texts:
            ids = [self.extra.get(w, O._WORD_IDS.get(w)) for w in s.split()]
            if add_special_tokens:
                ids = [O.BOS] + ids
                ids = ids + [O.EOS] * (max_length - len(ids))
            rows.append(ids)
        return types.SimpleNamespace(input_ids=torch.tensor(rows, dtype=torch.int64))


def test_pipeline_with_vae_np_vs_oracle():
    """StableDiffusionE4TPipeline with an AutoencoderKL attached, output_type="np", against the oracle decode of the
    oracle's denoising loop."""
    from e4t.pipeline_stable_diffusion_e4t import DDIMScheduler, StableDiffusionE4TPipeline
    tcfg = O.CLIP_TEXT_TINY
    (unet, enc, text), (sd_u, sd_e, sd_t) = _tiny_models(41, 42, 43, text_vocab=tcfg["vocab"] - 1)
    vae, sd_v = _oracle_vae(44)
    cfg = types.SimpleNamespace(placeholder_token="*s", domain_class_token="a", domain_embed_scale=0.1)
    pipe = StableDiffusionE4TPipeline(vae, text, _Tok(), unet, enc, DDIMScheduler(), e4t_config=cfg)
    assert pipe.vae_scale_factor == 4          # TINY_VAE has three levels
    with torch.no_grad():
        text.get_input_embeddings().weight[-1] = sd_t["text_model.embeddings.token_embedding.weight"][-1].cuda()
    g = torch.Generator().manual_seed(3)
    image = torch.rand(1, 3, 64, 64, generator=g) * 2 - 1
    latents = torch.randn(2, 4, 16, 16, generator=g)
    prompt = ["a photo of *s", "a photo of *s"]
    out = pipe(prompt, height=64, width=64, num_inference_steps=4, guidance_scale=1.0, latents=latents.clone(),
               image=image, output_type="np").images
    ids = pipe.tokenizer(prompt, max_length=77).input_ids
    ref_lat = O.pipeline_sample(sd_u, O.TINY_UNET, sd_e, O.VIT_TINY, sd_t, tcfg, image, ids, latents,
                                num_inference_steps=4, guidance_scale=1.0, class_token_id=O._WORD_IDS["a"])
    with torch.no_grad():
        ref = (V.vae_decode(sd_v, TINY, ref_lat / 0.18215) / 2 + 0.5).clamp(0, 1).permute(0, 2, 3, 1)
    out = torch.from_numpy(out)
    assert out.shape == (2, 64, 64, 3)
    e = _rel(out, ref)
    print(f"[pipeline np] rel err {e:.3e}")
    assert e < 4e-2
