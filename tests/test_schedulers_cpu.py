"""Sampling schedulers (e4t/schedulers.py, --scheduler_type of inference.py:65-72): the coefficient tables that the
sampler kernel applies, against the fp64 diffusers-structured restatements of oracle/sampler_oracle.py; the constants
of the SD v1.x config; config handling; and the pipeline's from_pretrained."""
import json
import os
import types

import pytest
import torch

from oracle import sampler_oracle as SO

import e4t.schedulers as SC
from e4t.schedulers import (SCHEDULER_MAPPING, DDIMScheduler, DPMSolverMultistepScheduler,
                            EulerAncestralDiscreteScheduler, EulerDiscreteScheduler, LMSDiscreteScheduler,
                            PNDMScheduler)

NAMES = ["ddim", "plms", "lms", "euler", "euler_ancestral", "dpm_solver++"]
# the SD v1.4 scheduler/scheduler_config.json (a PNDM config)
SD14_CONFIG = {"_class_name": "PNDMScheduler", "_diffusers_version": "0.7.0.dev0", "beta_end": 0.012,
               "beta_schedule": "scaled_linear", "beta_start": 0.00085, "num_train_timesteps": 1000,
               "set_alpha_to_one": False, "skip_prk_steps": True, "steps_offset": 1, "trained_betas": None,
               "clip_sample": False}


def apply_row(row, out, x, hist, saved, z):
    """fp64 restatement of e4t_sampler_step's per-element update for one table row (csrc/sampler.cu)."""
    xn = row[SC.X] * x + row[SC.E] * out + row[SC.S] * saved
    for k in range(SC.MAX_HISTORY):
        if row[SC.H0 + k] != 0:
            xn = xn + row[SC.H0 + k] * hist[k]
    if row[SC.Z] != 0:
        xn = xn + row[SC.Z] * z
    slot = int(row[SC.SLOT])
    if slot >= 0:
        hist[slot] = row[SC.HA] * x + row[SC.HB] * out
    if row[SC.SAVE] != 0:
        saved = x.clone()
    return xn, saved


def _rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def _trajectory_errors(name, prediction_type, n, eta=0.0):
    sched = SCHEDULER_MAPPING[name].from_config({"prediction_type": prediction_type})
    sched.set_timesteps(n)
    table = sched.sampler_table(eta=eta).double()
    ref = SO.make(name, prediction_type)
    ref.set_timesteps(n)
    ts = [float(t) for t in sched.timesteps]
    assert ts == [float(t) for t in ref.timesteps] and table.shape == (len(ts), SC.ROW)
    g = torch.Generator().manual_seed(n)
    shape = (2, 4, 5, 7)
    x = torch.randn(shape, generator=g, dtype=torch.float64) * ref.init_noise_sigma
    x_ref = x.clone()
    hist = [torch.zeros(shape, dtype=torch.float64) for _ in range(SC.MAX_HISTORY)]
    saved = torch.zeros(shape, dtype=torch.float64)
    errs = []
    for i, t in enumerate(ref.timesteps):
        e = torch.randn(shape, generator=g, dtype=torch.float64)
        z = torch.randn(shape, generator=g, dtype=torch.float64)
        assert (table[i, SC.Z] != 0) == SO.needs_noise(ref, i), f"step {i}: noise use differs"
        x, saved = apply_row(table[i], e, x, hist, saved, z)
        x_ref = ref.step(e, t, x_ref, noise=z)
        errs.append(_rel(x, x_ref))
        if i + 1 < len(ts):     # the next model input scale and timestep the kernel publishes
            scaled = ref.scale_model_input(torch.ones(1, dtype=torch.float64), ref.timesteps[i + 1]).item()
            assert abs(table[i, SC.S_NEXT].item() - scaled) <= 1e-12 and table[i, SC.T_NEXT].item() == ts[i + 1]
    return errs


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 14, 15, 16, 50])
@pytest.mark.parametrize("prediction_type", ["epsilon", "v_prediction"])
@pytest.mark.parametrize("name", NAMES)
def test_table_reproduces_oracle_trajectory(name, prediction_type, n):
    errs = _trajectory_errors(name, prediction_type, n)
    assert max(errs) <= 1e-10, errs


def test_ddim_table_with_eta_matches_eager_step_arithmetic():
    """DDIM with eta > 0: every row carries the noise coefficient std = eta·√((1−ᾱ_prev)/(1−ᾱ_t)·(1−ᾱ_t/ᾱ_prev))."""
    s = DDIMScheduler()
    s.set_timesteps(10)
    tab = s.sampler_table(eta=0.5)
    assert (tab[:, SC.Z] > 0).all()
    acp = s.alphas_cumprod.double()
    t, p = int(s.timesteps[3]), int(s.timesteps[4])
    std = 0.5 * ((1 - acp[p]) / (1 - acp[t]) * (1 - acp[t] / acp[p])) ** 0.5
    assert abs(tab[3, SC.Z].item() - std.item()) < 1e-15
    assert (s.sampler_table()[:, SC.Z] == 0).all()


def test_sd14_pinned_constants():
    lms = LMSDiscreteScheduler.from_config(SD14_CONFIG)
    eul = EulerDiscreteScheduler.from_config(SD14_CONFIG)
    for s in (lms, eul, EulerAncestralDiscreteScheduler.from_config(SD14_CONFIG)):
        assert abs(s.init_noise_sigma - 14.614641) < 1e-5
    p = PNDMScheduler.from_config(SD14_CONFIG)
    p.set_timesteps(50)
    assert len(p.timesteps) == 51 and p.timesteps[:4].tolist() == [981, 961, 961, 941]
    assert p.timesteps[-1].item() == 1
    d = DPMSolverMultistepScheduler.from_config(SD14_CONFIG)
    d.set_timesteps(50)
    assert d.timesteps[:4].tolist() == [999, 979, 959, 939] and d.timesteps.dtype == torch.int64
    eul.set_timesteps(50)
    assert eul.timesteps[0].item() == 999.0 and abs(eul.timesteps[1].item() - 978.6122) < 1e-4
    assert eul.timesteps.dtype == torch.float64
    x = torch.ones(3)
    assert torch.allclose(eul.scale_model_input(x, eul.timesteps[0]), x / (14.614641 ** 2 + 1) ** 0.5)
    assert p.scale_model_input(x, p.timesteps[0]) is x and p.init_noise_sigma == 1.0


@pytest.mark.parametrize("name", NAMES)
def test_from_config_refusals_and_ignored_keys(name):
    cls = SCHEDULER_MAPPING[name]
    with pytest.raises(ValueError):
        cls.from_config({"beta_schedule": "linear"})
    with pytest.raises(ValueError):
        cls.from_config({"prediction_type": "sample"})
    if name != "ddim":    # DDIMScheduler.from_config is unchanged
        with pytest.raises(ValueError):
            cls.from_config({"trained_betas": [0.1] * 1000})
    s = cls.from_config(dict(SD14_CONFIG, some_future_key=3, _class_name="Whatever"))
    s.set_timesteps(5)
    assert len(s.timesteps) >= 5


def test_from_pretrained_reads_a_local_directory(tmp_path):
    d = tmp_path / "scheduler"
    d.mkdir()
    (d / "scheduler_config.json").write_text(json.dumps(dict(SD14_CONFIG, prediction_type="v_prediction")))
    for name in NAMES:
        s = SCHEDULER_MAPPING[name].from_pretrained(str(tmp_path), subfolder="scheduler")
        assert s.prediction_type == "v_prediction"
    s = EulerDiscreteScheduler.from_pretrained(str(tmp_path), subfolder="scheduler", prediction_type="epsilon")
    assert s.prediction_type == "epsilon"
    with pytest.raises(ValueError):
        PNDMScheduler.from_pretrained(str(tmp_path), subfolder="scheduler", beta_schedule="squaredcos_cap_v2")


def test_scheduler_mapping_keys_are_inference_py_choices():
    assert list(SCHEDULER_MAPPING) == ["ddim", "plms", "lms", "euler", "euler_ancestral", "dpm_solver++"]
    import e4t.pipeline_stable_diffusion_e4t as P
    assert SCHEDULER_MAPPING["ddim"] is P.DDIMScheduler
    for cls in SCHEDULER_MAPPING.values():
        assert getattr(P, cls.__name__) is cls and hasattr(cls, "sampler_table")


def test_history_slots_never_read_and_written_in_one_step():
    for name in NAMES:
        for n in (1, 2, 5, 16):
            s = SCHEDULER_MAPPING[name]()
            s.set_timesteps(n)
            for r in s.sampler_table():
                slot = int(r[SC.SLOT])
                assert -1 <= slot < s.sampler_history
                if slot >= 0:
                    assert r[SC.H0 + slot] == 0
                assert (r[SC.H0 + s.sampler_history:SC.H0 + SC.MAX_HISTORY] == 0).all()


def test_pipeline_from_pretrained_loads_pndm_and_vae_strictly(tmp_path):
    from e4t.models.autoencoder_kl import AutoencoderKL
    from e4t.pipeline_stable_diffusion_e4t import StableDiffusionE4TPipeline
    from test_pipeline_gpu import _Tok
    vae = _tiny_vae_dir(tmp_path)
    pipe = _pipe_from(tmp_path)
    assert type(pipe.scheduler) is PNDMScheduler and isinstance(pipe.vae, AutoencoderKL)
    ref = vae.state_dict()
    got = pipe.vae.state_dict()
    assert set(got) == set(ref) and all(torch.equal(got[k], ref[k]) for k in ref)
    own = DDIMScheduler()
    text = types.SimpleNamespace(device=torch.device("cpu"), resize_token_embeddings=lambda n: None,
                                 get_input_embeddings=lambda: torch.nn.Embedding(49409, 8))
    conf = types.SimpleNamespace(placeholder_token="*s", domain_class_token="a", domain_embed_scale=0.1)
    pipe2 = StableDiffusionE4TPipeline.from_pretrained(str(tmp_path), vae=None, scheduler=own, text_encoder=text,
                                                       tokenizer=_Tok(), unet=None, e4t_encoder=None, e4t_config=conf)
    assert pipe2.scheduler is own and pipe2.vae is None
    assert pipe2.enable_xformers_memory_efficient_attention() is None


def _tiny_vae_dir(tmp_path):
    from e4t.models.autoencoder_kl import AutoencoderKL
    (tmp_path / "scheduler").mkdir()
    (tmp_path / "scheduler" / "scheduler_config.json").write_text(json.dumps(SD14_CONFIG))
    vae = AutoencoderKL(in_channels=3, out_channels=3, down_block_types=["DownEncoderBlock2D"] * 2,
                        up_block_types=["UpDecoderBlock2D"] * 2, block_out_channels=[64, 64], layers_per_block=1,
                        latent_channels=4, norm_num_groups=32, sample_size=32)
    vae.save_pretrained(str(tmp_path / "vae"))
    return vae


def _pipe_from(tmp_path):
    from e4t.pipeline_stable_diffusion_e4t import StableDiffusionE4TPipeline
    from test_pipeline_gpu import _Tok
    text = types.SimpleNamespace(device=torch.device("cpu"), resize_token_embeddings=lambda n: None,
                                 get_input_embeddings=lambda: torch.nn.Embedding(49409, 8))
    conf = types.SimpleNamespace(placeholder_token="*s", domain_class_token="a", domain_embed_scale=0.1)
    return StableDiffusionE4TPipeline.from_pretrained(str(tmp_path), text_encoder=text, tokenizer=_Tok(), unet=None,
                                                      e4t_encoder=None, e4t_config=conf)


def test_pipeline_from_pretrained_reads_a_sharded_vae_without_a_plain_bin(tmp_path):
    """A VAE directory whose weights are only a sharded index (no diffusion_pytorch_model.bin) loads, every weight
    read once from its shard; a shard set that misses a weight is refused."""
    vae = _tiny_vae_dir(tmp_path)
    d = tmp_path / "vae"
    os.remove(d / "diffusion_pytorch_model.bin")
    ref = vae.state_dict()
    keys = sorted(ref)
    half = len(keys) // 2
    shards = {"diffusion_pytorch_model-00001-of-00002.bin": keys[:half],
              "diffusion_pytorch_model-00002-of-00002.bin": keys[half:]}
    for name, ks in shards.items():
        torch.save({k: ref[k] for k in ks}, d / name)
    index = {"metadata": {}, "weight_map": {k: name for name, ks in shards.items() for k in ks}}
    (d / "diffusion_pytorch_model.bin.index.json").write_text(json.dumps(index))
    pipe = _pipe_from(tmp_path)
    got = pipe.vae.state_dict()
    assert type(pipe.scheduler) is PNDMScheduler
    assert set(got) == set(ref) and all(torch.equal(got[k], ref[k]) for k in ref)
    # drop one weight from the second shard: the load must fail, not leave a randomly initialised tensor
    torch.save({k: ref[k] for k in keys[half:-1]}, d / "diffusion_pytorch_model-00002-of-00002.bin")
    with pytest.raises(RuntimeError, match="missing keys"):
        _pipe_from(tmp_path)
