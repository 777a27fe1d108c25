"""Sampling schedulers of the reference's inference.py (--scheduler_type, inference.py:44,65-72,118), following
diffusers 0.14.0 with the defaults the SD v1.x / 2.x scheduler configs leave in place: scaled-linear betas, epsilon or
v prediction.  diffusers is not a dependency.

Every one of these schedulers moves the latents by a linear combination of the current sample x, the current (guided)
model output e, a few earlier outputs, a saved sample and fresh noise z, with coefficients that depend only on the step
index.  `sampler_table()` writes those coefficients for the whole trajectory as one fp64 row per entry of `timesteps`;
the sm_90a kernel `e4t_sampler_step` (csrc/sampler.cu) applies row *step_dev of it, so a whole denoising step needs no
host-side branching and can be replayed from a CUDA graph.  The table format is defined here and nowhere else:

    x_next = T[X]·x + T[E]·e + Σ_k T[H0 + k]·hist[k] + T[S]·saved + T[Z]·z
    hist[T[SLOT]] = T[HA]·x + T[HB]·e              (T[SLOT] < 0: no history entry this step)
    saved = x                                       (T[SAVE] != 0)
    next model input = T[S_NEXT]·x_next at timestep T[T_NEXT]

All right-hand sides read the values from before the step; no slot is read and written in the same step.  The host
resolves the ring positions of the history, so the kernel reads named slots and does no index arithmetic.
`step()` of the table schedulers runs the same kernel on the current row (one code path for eager and graphed use)."""
import json
import math
import os
from dataclasses import dataclass

import numpy as np
import torch

from e4t._mixins import BaseOutput

# ---- the table format (mirrored by the kernel's column indices in csrc/sampler.cu) --------------------------------
X, E, H0, S, Z, SLOT, HA, HB, SAVE, S_NEXT, T_NEXT = 0, 1, 2, 6, 7, 8, 9, 10, 11, 12, 13
ROW = 14
MAX_HISTORY = 4


@dataclass
class _StepOutput(BaseOutput):
    prev_sample: torch.Tensor = None
    pred_original_sample: torch.Tensor = None


def _scaled_linear_acp(num_train_timesteps, beta_start, beta_end):
    betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
    return torch.cumprod(1.0 - betas, dim=0)


def _check_config(config):
    if config.get("beta_schedule", "scaled_linear") != "scaled_linear":
        raise ValueError(f"beta_schedule {config['beta_schedule']!r} is not supported (only 'scaled_linear')")
    if config.get("trained_betas") is not None:
        raise ValueError("trained_betas is not supported (only the scaled_linear beta schedule)")


def _read_config(path, subfolder, overrides):
    d = os.path.join(path, subfolder) if subfolder else path
    with open(os.path.join(d, "scheduler_config.json")) as f:
        config = json.load(f)
    config.update(overrides)
    return config


def draw_noise(shape, generator, device):
    """One latent-shaped fp32 N(0, 1) draw from the caller's generator (a list: one image per generator), on
    `device`.  The eager and the graphed sampling paths both draw through here, once per step whose noise coefficient
    is non-zero, in step order."""
    if isinstance(generator, (list, tuple)):
        return torch.cat([torch.randn((1,) + tuple(shape[1:]), generator=g, device=g.device, dtype=torch.float32)
                          for g in generator]).to(device)
    gdev = generator.device if generator is not None else device
    return torch.randn(tuple(shape), generator=generator, device=gdev, dtype=torch.float32).to(device)


class _Lin:
    """A linear combination of the step's named inputs ('x', 'e', 'h0'..'h3', 's', 'z'), built in fp64 while a
    scheduler's update is restated; `row()` lays it out in the table format."""
    __slots__ = ("c",)

    def __init__(self, c=None):
        self.c = dict(c or {})

    @classmethod
    def of(cls, name):
        return cls({name: 1.0})

    def __add__(self, o):
        c = dict(self.c)
        for k, v in o.c.items():
            c[k] = c.get(k, 0.0) + v
        return _Lin(c)

    def __sub__(self, o):
        return self + (-1.0) * o

    def __rmul__(self, a):
        return _Lin({k: float(a) * v for k, v in self.c.items()})

    def __truediv__(self, a):
        return (1.0 / float(a)) * self

    def get(self, k):
        return self.c.get(k, 0.0)


def _row(x_next, slot=-1, h=None, save=False):
    r = np.zeros(ROW, dtype=np.float64)
    bad = set(x_next.c) - {"x", "e", "s", "z"} - {f"h{k}" for k in range(MAX_HISTORY)}
    assert not bad, bad
    r[X], r[E], r[S], r[Z] = x_next.get("x"), x_next.get("e"), x_next.get("s"), x_next.get("z")
    for k in range(MAX_HISTORY):
        r[H0 + k] = x_next.get(f"h{k}")
    r[SLOT] = slot
    if slot >= 0:
        assert set(h.c) <= {"x", "e"} and x_next.get(f"h{slot}") == 0.0
        r[HA], r[HB] = h.get("x"), h.get("e")
    r[SAVE] = 1.0 if save else 0.0
    return r


class _Ring:
    """Host-side ring of history slots: `entries` are the slots of the kept values, oldest first."""

    def __init__(self, n_slots, keep):
        self.n, self.keep, self.entries = n_slots, keep, []

    def kept(self):
        """Slots of the values kept before this step's entry is added (the newest `keep - 1`)."""
        return self.entries[-(self.keep - 1):] if self.keep > 1 else []

    def push(self):
        """Slot for this step's entry: one that holds no kept value (so none is read and written in one step)."""
        kept = self.kept()
        slot = next(k for k in range(self.n) if k not in kept)
        self.entries = kept + [slot]
        return slot


def _finish(rows, scales, timesteps):
    """Fill each row's next-step model-input scale and timestep (the last row repeats its own: nothing reads it)."""
    T = len(rows)
    for i, r in enumerate(rows):
        r[S_NEXT] = scales[i + 1] if i + 1 < T else 1.0
        r[T_NEXT] = float(timesteps[i + 1] if i + 1 < T else timesteps[i])
    return torch.from_numpy(np.stack(rows)) if rows else torch.zeros(0, ROW, dtype=torch.float64)


# ---- DDIM ----------------------------------------------------------------------------------------------------------
class DDIMScheduler:
    """diffusers 0.14 DDIMScheduler as configured by SD-v1.x (scheduler/scheduler_config.json): scaled_linear betas
    0.00085..0.012, 1000 train steps, clip_sample False, set_alpha_to_one False, steps_offset 1, epsilon prediction.
    prediction_type="v_prediction" is the SD 2.x 768-v configuration: the model predicts v = √ᾱ_t·ε − √(1−ᾱ_t)·x₀."""
    order = 1
    init_noise_sigma = 1.0
    sampler_history = 0

    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, steps_offset=1,
                 set_alpha_to_one=False, prediction_type="epsilon"):
        if prediction_type not in ("epsilon", "v_prediction"):
            raise ValueError(f"prediction_type must be 'epsilon' or 'v_prediction', got {prediction_type!r}")
        betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        self.final_alpha_cumprod = torch.tensor(1.0) if set_alpha_to_one else self.alphas_cumprod[0]
        self.num_train_timesteps = num_train_timesteps
        self.steps_offset = steps_offset
        self.prediction_type = prediction_type
        self.num_inference_steps = None
        self.timesteps = torch.arange(num_train_timesteps - 1, -1, -1)

    # scheduler_config.json keys this class follows; the others must hold the values it implements
    _CONFIG_KEYS = ("num_train_timesteps", "beta_start", "beta_end", "steps_offset", "set_alpha_to_one",
                    "prediction_type")

    @classmethod
    def from_config(cls, config):
        """DDIMScheduler from a diffusers scheduler config (a dict, e.g. a model's scheduler_config.json).  Only the
        scaled_linear beta schedule without sample clipping is implemented; any other is refused."""
        if config.get("beta_schedule", "scaled_linear") != "scaled_linear":
            raise ValueError(f"beta_schedule {config['beta_schedule']!r} is not supported (only 'scaled_linear')")
        if config.get("clip_sample", False):
            raise ValueError("clip_sample=True is not supported")
        return cls(**{k: config[k] for k in cls._CONFIG_KEYS if k in config})

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, subfolder=None, **kw):
        """DDIMScheduler.from_pretrained(path, subfolder="scheduler") on a local model directory (inference.py:118);
        nothing is downloaded."""
        import json
        import os
        d = os.path.join(pretrained_model_name_or_path, subfolder) if subfolder else pretrained_model_name_or_path
        with open(os.path.join(d, "scheduler_config.json")) as f:
            config = json.load(f)
        config.update(kw)
        return cls.from_config(config)

    def set_timesteps(self, num_inference_steps, device=None):
        self.num_inference_steps = num_inference_steps
        ratio = self.num_train_timesteps // num_inference_steps
        ts = (torch.arange(0, num_inference_steps) * ratio).round().flip(0).to(torch.int64) + self.steps_offset
        self.timesteps = ts.to(device) if device is not None else ts

    def scale_model_input(self, sample, timestep=None):
        return sample

    def step(self, model_output, timestep, sample, eta=0.0, generator=None, **kw):
        t = int(timestep)
        prev_t = t - self.num_train_timesteps // self.num_inference_steps
        a_t = self.alphas_cumprod[t].to(sample.device)
        a_prev = (self.alphas_cumprod[prev_t] if prev_t >= 0 else self.final_alpha_cumprod).to(sample.device)
        out = model_output.to(torch.float32)
        x = sample.to(torch.float32)
        if self.prediction_type == "epsilon":
            eps = out
            pred_x0 = (x - (1 - a_t) ** 0.5 * eps) / a_t ** 0.5
        else:
            pred_x0 = a_t ** 0.5 * x - (1 - a_t) ** 0.5 * out
            eps = a_t ** 0.5 * out + (1 - a_t) ** 0.5 * x
        var = (1 - a_prev) / (1 - a_t) * (1 - a_t / a_prev)
        std = eta * var ** 0.5
        prev = a_prev ** 0.5 * pred_x0 + (1 - a_prev - std ** 2) ** 0.5 * eps
        if eta > 0:
            prev = prev + std * torch.randn(x.shape, generator=generator, device=x.device, dtype=x.dtype)
        return _StepOutput(prev_sample=prev.to(sample.dtype), pred_original_sample=pred_x0.to(sample.dtype))

    def sampler_table(self, eta=0.0):
        """The step above as table rows (the graphed sampling path); `eta` > 0 gives each row a noise coefficient."""
        acp = self.alphas_cumprod.double()
        ts = [int(t) for t in self.timesteps.cpu()]
        ratio = self.num_train_timesteps // self.num_inference_steps
        x, e, z = _Lin.of("x"), _Lin.of("e"), _Lin.of("z")
        rows = []
        for t in ts:
            prev_t = t - ratio
            a_t = float(acp[t])
            a_prev = float(acp[prev_t]) if prev_t >= 0 else float(self.final_alpha_cumprod)
            if self.prediction_type == "epsilon":
                eps, x0 = e, (x - math.sqrt(1 - a_t) * e) / math.sqrt(a_t)
            else:
                x0 = math.sqrt(a_t) * x - math.sqrt(1 - a_t) * e
                eps = math.sqrt(a_t) * e + math.sqrt(1 - a_t) * x
            std = eta * math.sqrt((1 - a_prev) / (1 - a_t) * (1 - a_t / a_prev))
            xn = math.sqrt(a_prev) * x0 + math.sqrt(1 - a_prev - std ** 2) * eps
            if eta > 0:
                xn = xn + std * z
            rows.append(_row(xn))
        return _finish(rows, [1.0] * len(ts), ts)


# ---- the table schedulers ------------------------------------------------------------------------------------------
class _TableScheduler:
    """Common surface: config handling, fp64 ᾱ / σ, eager `step()` on the sampler kernel."""
    order = 1
    init_noise_sigma = 1.0
    sampler_history = 0
    _CONFIG_KEYS = ("num_train_timesteps", "beta_start", "beta_end", "prediction_type")

    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, prediction_type="epsilon"):
        if prediction_type not in ("epsilon", "v_prediction"):
            raise ValueError(f"prediction_type must be 'epsilon' or 'v_prediction', got {prediction_type!r}")
        self.alphas_cumprod = _scaled_linear_acp(num_train_timesteps, beta_start, beta_end)
        self.num_train_timesteps = num_train_timesteps
        self.prediction_type = prediction_type
        self.num_inference_steps = None
        self.timesteps = None
        self._table = None
        self._eager = None

    @classmethod
    def from_config(cls, config):
        """From a diffusers scheduler config dict.  Keys the scheduler does not use are ignored (as diffusers ignores
        them); a beta schedule other than scaled_linear, trained betas or an unknown prediction type is refused."""
        _check_config(config)
        return cls(**{k: config[k] for k in cls._CONFIG_KEYS if k in config})

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, subfolder=None, **kw):
        """`from_pretrained(model_dir, subfolder="scheduler", **overrides)` on a local directory; nothing is
        downloaded."""
        return cls.from_config(_read_config(pretrained_model_name_or_path, subfolder, kw))

    def set_timesteps(self, num_inference_steps, device=None):
        self.num_inference_steps = num_inference_steps
        ts, rows, scales = self._trajectory(num_inference_steps)
        self._host_ts = [float(t) for t in ts]
        self._table = _finish(rows, scales, ts)
        t = torch.tensor(ts) if len(ts) else torch.zeros(0)
        self.timesteps = t.to(device) if device is not None else t
        self._eager = None

    def sampler_table(self, eta=0.0):
        """fp64 (len(timesteps), ROW) table of the trajectory set by `set_timesteps` (`eta` is DDIM's only)."""
        if self._table is None:
            raise ValueError("call set_timesteps() before sampler_table()")
        return self._table.clone()

    def _index(self, timestep):
        t = float(timestep)
        try:
            return self._host_ts.index(t)
        except ValueError:
            raise ValueError(f"timestep {t} is not in this scheduler's timesteps") from None

    def scale_model_input(self, sample, timestep):
        return sample

    def step(self, model_output, timestep, sample, eta=0.0, generator=None, return_dict=True, **kw):
        """One step on the sampler kernel with this step's table row; steps must follow `timesteps` in order."""
        from e4t_b200 import ops
        st = self._eager
        n = sample.numel()
        if st is None or st["n"] != n or st["device"] != sample.device:
            dev = sample.device
            st = self._eager = dict(n=n, device=dev, i=0, table=self._table.to(dev),
                                    step=torch.zeros(1, dtype=torch.int32, device=dev),
                                    hist=ops.sampler_history_buffer(self.sampler_history, n, dev),
                                    saved=torch.zeros(n, dtype=torch.float32, device=dev),
                                    row=torch.zeros(ROW, dtype=torch.float32, device=dev))
        i = st["i"]
        if i >= len(self._host_ts) or float(timestep) != self._host_ts[i]:
            raise ValueError(f"step {i}: timestep {float(timestep)} does not follow this scheduler's timesteps "
                             "(call set_timesteps() to start a new trajectory)")
        z = draw_noise(sample.shape, generator, sample.device) if self._table[i, Z] != 0 else None
        x = sample.to(torch.float32).contiguous()
        x_next = torch.empty_like(x)
        ops.sampler_step(model_output.to(torch.float32).contiguous(), x, x_next, st["hist"], st["saved"], z,
                         st["table"], st["step"], st["row"])
        st["i"] = i + 1
        out = _StepOutput(prev_sample=x_next.to(sample.dtype))
        return out if return_dict else (out.prev_sample,)

    def _alpha(self, t):
        return float(self.alphas_cumprod[int(t)].double())


def _x0(prediction_type, x, e, sigma):
    """x₀ from the model output in σ-space (diffusers' Euler / LMS: epsilon x − σ·e, v −σ/√(σ²+1)·e + x/(σ²+1))."""
    if prediction_type == "epsilon":
        return x - sigma * e
    return (-sigma / math.sqrt(sigma ** 2 + 1)) * e + (1.0 / (sigma ** 2 + 1)) * x


class _SigmaScheduler(_TableScheduler):
    """LMS / Euler / Euler ancestral: float timesteps linspace(0, T−1, n) reversed, σ interpolated on them, the
    model input scaled by 1/√(σ²+1), `init_noise_sigma` = max σ."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        acp = self.alphas_cumprod
        self._train_sigmas = (((1 - acp) / acp) ** 0.5).numpy()          # fp32, as diffusers computes it
        self.init_noise_sigma = float(np.float32(self._train_sigmas.max()))

    def _sigmas(self, n):
        ts = np.linspace(0, self.num_train_timesteps - 1, n, dtype=float)[::-1].copy()
        sig = np.interp(ts, np.arange(0, len(self._train_sigmas)), self._train_sigmas)
        sig = np.concatenate([sig, [0.0]]).astype(np.float32).astype(np.float64)
        return ts, sig

    def _trajectory(self, n):
        ts, sig = self._sigmas(n)
        x, e = _Lin.of("x"), _Lin.of("e")
        rows = []
        self._begin()
        for i in range(n):
            d = (x - _x0(self.prediction_type, x, e, sig[i])) / sig[i]
            rows.append(self._update(i, d, sig))
        self._sig = sig
        return ts, rows, [1.0 / math.sqrt(s ** 2 + 1) for s in sig[:n]]

    def scale_model_input(self, sample, timestep):
        return sample / math.sqrt(self._sig[self._index(timestep)] ** 2 + 1)

    def _begin(self):
        pass


class EulerDiscreteScheduler(_SigmaScheduler):
    """diffusers 0.14 EulerDiscreteScheduler with s_churn = 0: x_next = x + d·(σ_{i+1} − σ_i), d = (x − x₀)/σ_i."""

    def _update(self, i, d, sig):
        return _row(_Lin.of("x") + (sig[i + 1] - sig[i]) * d)


class EulerAncestralDiscreteScheduler(_SigmaScheduler):
    """diffusers 0.14 EulerAncestralDiscreteScheduler: x_next = x + d·(σ_down − σ_i) + σ_up·z."""

    def _update(self, i, d, sig):
        s, sn = sig[i], sig[i + 1]
        up = math.sqrt(sn ** 2 * (s ** 2 - sn ** 2) / s ** 2)
        down = math.sqrt(sn ** 2 - up ** 2)
        xn = _Lin.of("x") + (down - s) * d
        if up != 0.0:
            xn = xn + up * _Lin.of("z")
        return _row(xn)


def _lms_coefficient(sig, i, order, j):
    """∫_{σ_i}^{σ_{i+1}} Π_{k≠j, k<order} (τ − σ_{i−k}) / (σ_{i−j} − σ_{i−k}) dτ, exactly (the integrand is a
    polynomial; diffusers integrates it numerically with scipy's quad)."""
    p = np.polynomial.Polynomial([1.0])
    for k in range(order):
        if k != j:
            p = p * np.polynomial.Polynomial([-sig[i - k], 1.0]) / (sig[i - j] - sig[i - k])
    q = p.integ()
    return q(sig[i + 1]) - q(sig[i])


class LMSDiscreteScheduler(_SigmaScheduler):
    """diffusers 0.14 LMSDiscreteScheduler, order 4: x_next = x + Σ_j c_j·d_{i−j} over the last min(i+1, 4)
    derivatives, which are kept in four history slots."""
    sampler_history = 4
    lms_order = 4

    def _begin(self):
        self._ring = _Ring(self.sampler_history, self.lms_order)

    def _update(self, i, d, sig):
        kept = self._ring.kept()
        seq = [_Lin.of(f"h{k}") for k in kept] + [d]           # the derivatives, oldest first
        order = min(i + 1, self.lms_order)
        xn = _Lin.of("x")
        for j in range(order):
            xn = xn + _lms_coefficient(sig, i, order, j) * seq[-1 - j]
        slot = self._ring.push()
        return _row(xn, slot, d)


class PNDMScheduler(_TableScheduler):
    """diffusers 0.14 PNDMScheduler with skip_prk_steps=True (PLMS), set_alpha_to_one=False, steps_offset=1: the
    default scheduler of the SD v1.x / 2.x scheduler configs and of the reference pipeline."""
    sampler_history = 4
    _CONFIG_KEYS = _TableScheduler._CONFIG_KEYS + ("steps_offset", "set_alpha_to_one", "skip_prk_steps")

    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, prediction_type="epsilon",
                 steps_offset=1, set_alpha_to_one=False, skip_prk_steps=True):
        super().__init__(num_train_timesteps, beta_start, beta_end, prediction_type)
        if not skip_prk_steps:
            raise ValueError("skip_prk_steps=False (Runge-Kutta warm-up steps) is not supported")
        self.steps_offset = steps_offset
        self.final_alpha_cumprod = 1.0 if set_alpha_to_one else float(self.alphas_cumprod[0].double())

    def _trajectory(self, n):
        r = self.num_train_timesteps // n
        _t = np.arange(0, n) * r + self.steps_offset
        ts = np.concatenate([_t[:-1], _t[-2:-1], _t[-1:]])[::-1].astype(np.int64).copy()
        x, e = _Lin.of("x"), _Lin.of("e")
        ring = _Ring(self.sampler_history, 4)
        rows = []
        for counter, t in enumerate(int(v) for v in ts):
            prev_t = t - r
            slot = -1
            if counter != 1:
                seq = [_Lin.of(f"h{k}") for k in ring.kept()] + [e]     # ets after appending e, oldest first
                slot = ring.push()
            else:
                seq = [_Lin.of(f"h{k}") for k in ring.entries]
                prev_t, t = t, t + r
            sample, save = x, False
            if len(seq) == 1 and counter == 0:
                eh, save = e, True
            elif len(seq) == 1 and counter == 1:
                eh, sample = (e + seq[-1]) / 2, _Lin.of("s")
            elif len(seq) == 2:
                eh = (3 * seq[-1] - seq[-2]) / 2
            elif len(seq) == 3:
                eh = (23 * seq[-1] - 16 * seq[-2] + 5 * seq[-3]) / 12
            else:
                eh = (55 * seq[-1] - 59 * seq[-2] + 37 * seq[-3] - 9 * seq[-4]) / 24
            a_t = self._alpha(t)
            a_prev = self._alpha(prev_t) if prev_t >= 0 else self.final_alpha_cumprod
            if self.prediction_type == "v_prediction":
                eh = math.sqrt(a_t) * eh + math.sqrt(1 - a_t) * sample
            denom = a_t * math.sqrt(1 - a_prev) + math.sqrt(a_t * (1 - a_t) * a_prev)
            xn = math.sqrt(a_prev / a_t) * sample - ((a_prev - a_t) / denom) * eh
            rows.append(_row(xn, slot, e, save))
        return ts, rows, [1.0] * len(ts)


class DPMSolverMultistepScheduler(_TableScheduler):
    """diffusers 0.14 DPMSolverMultistepScheduler: solver_order 2, algorithm_type dpmsolver++, solver_type midpoint,
    lower_order_final True, no thresholding.  The data prediction m of the previous step lives in a history slot."""
    sampler_history = 2
    _CONFIG_KEYS = _TableScheduler._CONFIG_KEYS + ("solver_order", "algorithm_type", "solver_type",
                                                   "lower_order_final", "thresholding")

    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, prediction_type="epsilon",
                 solver_order=2, algorithm_type="dpmsolver++", solver_type="midpoint", lower_order_final=True,
                 thresholding=False):
        super().__init__(num_train_timesteps, beta_start, beta_end, prediction_type)
        if (solver_order, algorithm_type, solver_type, thresholding) != (2, "dpmsolver++", "midpoint", False):
            raise ValueError("only solver_order=2, algorithm_type='dpmsolver++', solver_type='midpoint' without "
                             "thresholding is supported")
        self.lower_order_final = lower_order_final

    def _trajectory(self, n):
        ts = np.linspace(0, self.num_train_timesteps - 1, n + 1).round()[::-1][:-1].copy().astype(np.int64)
        x, e = _Lin.of("x"), _Lin.of("e")

        def als(t):
            a = self._alpha(t)
            al, sg = math.sqrt(a), math.sqrt(1 - a)
            return al, sg, math.log(al) - math.log(sg)

        ring = _Ring(self.sampler_history, 2)
        rows = []
        for i, s0 in enumerate(int(v) for v in ts):
            t = 0 if i == n - 1 else int(ts[i + 1])
            a_s, sg_s, l_s = als(s0)
            m = (x - sg_s * e) / a_s if self.prediction_type == "epsilon" else a_s * x - sg_s * e
            kept = ring.kept()
            slot = ring.push()
            a_t, sg_t, l_t = als(t)
            h = l_t - l_s
            k = a_t * (math.exp(-h) - 1.0)
            if i == 0 or (i == n - 1 and self.lower_order_final and n < 15):
                xn = (sg_t / sg_s) * x - k * m
            else:
                m1 = _Lin.of(f"h{kept[-1]}")
                l_s1 = als(int(ts[i - 1]))[2]
                r0 = (l_s - l_s1) / h
                d1 = (m - m1) / r0
                xn = (sg_t / sg_s) * x - k * m - (0.5 * k) * d1
            rows.append(_row(xn, slot, m))
        return ts, rows, [1.0] * len(ts)


# inference.py:65-72 (--scheduler_type)
SCHEDULER_MAPPING = {
    "ddim": DDIMScheduler,
    "plms": PNDMScheduler,
    "lms": LMSDiscreteScheduler,
    "euler": EulerDiscreteScheduler,
    "euler_ancestral": EulerAncestralDiscreteScheduler,
    "dpm_solver++": DPMSolverMultistepScheduler,
}
