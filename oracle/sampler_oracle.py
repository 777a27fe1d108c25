"""fp64 restatements of the diffusers 0.14.0 sampling schedulers behind the reference's --scheduler_type
(inference.py:65-72): PNDM (PLMS), LMS, Euler, Euler ancestral and DPM-Solver++ multistep, with the defaults the SD
scheduler configs leave in place, and the pipeline denoising loop over any of them (and DDIM).

These follow diffusers' own structure: lists of `ets`, `derivatives` and `model_outputs`, counters and per-step
branches.  They deliberately do not use the coefficient-table formulation of e4t/schedulers.py, so that the tables
are checked against an independent statement of the same arithmetic.  LMS integrates its coefficients with
scipy's quad, as diffusers does."""
import numpy as np
import torch

from oracle import e4t_oracle as O

F64 = torch.float64


def _acp(num_train=1000, beta_start=0.00085, beta_end=0.012):
    betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train, dtype=torch.float32) ** 2
    return torch.cumprod(1.0 - betas, dim=0)


class PNDM:
    """PNDMScheduler(skip_prk_steps=True, set_alpha_to_one=False, steps_offset=1).step_plms."""
    needs_noise = False

    def __init__(self, prediction_type="epsilon", num_train=1000):
        self.acp = _acp(num_train).double()
        self.final = self.acp[0]
        self.num_train, self.prediction_type = num_train, prediction_type
        self.init_noise_sigma = 1.0

    def set_timesteps(self, n):
        self.n = n
        r = self.num_train // n
        _t = np.arange(0, n) * r + 1
        self.timesteps = np.concatenate([_t[:-1], _t[-2:-1], _t[-1:]])[::-1].tolist()
        self.ets, self.counter, self.cur_sample = [], 0, None

    def scale_model_input(self, x, t):
        return x

    def step(self, model_output, timestep, sample, noise=None):
        prev_timestep = timestep - self.num_train // self.n
        if self.counter != 1:
            self.ets = self.ets[-3:]
            self.ets.append(model_output)
        else:
            prev_timestep = timestep
            timestep = timestep + self.num_train // self.n
        if len(self.ets) == 1 and self.counter == 0:
            self.cur_sample = sample
        elif len(self.ets) == 1 and self.counter == 1:
            model_output = (model_output + self.ets[-1]) / 2
            sample = self.cur_sample
            self.cur_sample = None
        elif len(self.ets) == 2:
            model_output = (3 * self.ets[-1] - self.ets[-2]) / 2
        elif len(self.ets) == 3:
            model_output = (23 * self.ets[-1] - 16 * self.ets[-2] + 5 * self.ets[-3]) / 12
        else:
            model_output = (1 / 24) * (55 * self.ets[-1] - 59 * self.ets[-2] + 37 * self.ets[-3] - 9 * self.ets[-4])
        a_t = self.acp[timestep]
        a_prev = self.acp[prev_timestep] if prev_timestep >= 0 else self.final
        b_t, b_prev = 1 - a_t, 1 - a_prev
        if self.prediction_type == "v_prediction":
            model_output = a_t ** 0.5 * model_output + b_t ** 0.5 * sample
        sample_coeff = (a_prev / a_t) ** 0.5
        denom = a_t * b_prev ** 0.5 + (a_t * b_t * a_prev) ** 0.5
        self.counter += 1
        return sample_coeff * sample - (a_prev - a_t) * model_output / denom


class _Sigmas:
    needs_noise = False

    def __init__(self, prediction_type="epsilon", num_train=1000):
        acp = _acp(num_train)
        self.train_sigmas = (((1 - acp) / acp) ** 0.5).numpy()
        self.num_train, self.prediction_type = num_train, prediction_type
        self.init_noise_sigma = float(np.float32(self.train_sigmas.max()))

    def set_timesteps(self, n):
        ts = np.linspace(0, self.num_train - 1, n, dtype=float)[::-1].copy()
        sig = np.interp(ts, np.arange(0, len(self.train_sigmas)), self.train_sigmas)
        self.sigmas = np.concatenate([sig, [0.0]]).astype(np.float32).astype(np.float64)
        self.timesteps = ts.tolist()
        self.derivatives = []

    def index(self, t):
        return self.timesteps.index(t)

    def scale_model_input(self, x, t):
        return x / (self.sigmas[self.index(t)] ** 2 + 1) ** 0.5

    def x0(self, e, x, sigma):
        if self.prediction_type == "epsilon":
            return x - sigma * e
        return e * (-sigma / (sigma ** 2 + 1) ** 0.5) + x / (sigma ** 2 + 1)


class Euler(_Sigmas):
    def step(self, model_output, timestep, sample, noise=None):
        i = self.index(timestep)
        sigma = self.sigmas[i]
        derivative = (sample - self.x0(model_output, sample, sigma)) / sigma
        return sample + derivative * (self.sigmas[i + 1] - sigma)


class EulerAncestral(_Sigmas):
    def needs_noise_at(self, i):
        return self.sigmas[i + 1] != 0.0

    def step(self, model_output, timestep, sample, noise=None):
        i = self.index(timestep)
        sigma_from, sigma_to = self.sigmas[i], self.sigmas[i + 1]
        pred = self.x0(model_output, sample, sigma_from)
        sigma_up = (sigma_to ** 2 * (sigma_from ** 2 - sigma_to ** 2) / sigma_from ** 2) ** 0.5
        sigma_down = (sigma_to ** 2 - sigma_up ** 2) ** 0.5
        derivative = (sample - pred) / sigma_from
        prev = sample + derivative * (sigma_down - sigma_from)
        if sigma_up != 0.0:
            prev = prev + noise * sigma_up
        return prev


class LMS(_Sigmas):
    def coefficient(self, order, t, current_order):
        from scipy import integrate

        def lms_derivative(tau):
            prod = 1.0
            for k in range(order):
                if current_order == k:
                    continue
                prod *= (tau - self.sigmas[t - k]) / (self.sigmas[t - current_order] - self.sigmas[t - k])
            return prod

        return integrate.quad(lms_derivative, self.sigmas[t], self.sigmas[t + 1], epsrel=1e-4)[0]

    def step(self, model_output, timestep, sample, noise=None, order=4):
        i = self.index(timestep)
        sigma = self.sigmas[i]
        self.derivatives.append((sample - self.x0(model_output, sample, sigma)) / sigma)
        if len(self.derivatives) > order:
            self.derivatives.pop(0)
        order = min(i + 1, order)
        coeffs = [self.coefficient(order, i, co) for co in range(order)]
        return sample + sum(c * d for c, d in zip(coeffs, reversed(self.derivatives)))


class DPMSolverPP:
    """DPMSolverMultistepScheduler(solver_order=2, dpmsolver++, midpoint, lower_order_final=True)."""
    needs_noise = False

    def __init__(self, prediction_type="epsilon", num_train=1000):
        acp = _acp(num_train).double()
        self.alpha_t, self.sigma_t = acp ** 0.5, (1 - acp) ** 0.5
        self.lambda_t = torch.log(self.alpha_t) - torch.log(self.sigma_t)
        self.num_train, self.prediction_type = num_train, prediction_type
        self.init_noise_sigma = 1.0

    def set_timesteps(self, n):
        self.timesteps = (np.linspace(0, self.num_train - 1, n + 1).round()[::-1][:-1].copy()
                          .astype(np.int64).tolist())
        self.model_outputs = [None, None]
        self.lower_order_nums = 0

    def scale_model_input(self, x, t):
        return x

    def step(self, model_output, timestep, sample, noise=None):
        n = len(self.timesteps)
        step_index = self.timesteps.index(timestep)
        prev_timestep = 0 if step_index == n - 1 else self.timesteps[step_index + 1]
        lower_order_final = step_index == n - 1 and n < 15
        a, s = self.alpha_t[timestep], self.sigma_t[timestep]
        if self.prediction_type == "epsilon":
            m = (sample - s * model_output) / a
        else:
            m = a * sample - s * model_output
        self.model_outputs[0] = self.model_outputs[1]
        self.model_outputs[-1] = m
        lt, at, st = self.lambda_t[prev_timestep], self.alpha_t[prev_timestep], self.sigma_t[prev_timestep]
        if self.lower_order_nums < 1 or lower_order_final:
            h = lt - self.lambda_t[timestep]
            prev = (st / s) * sample - (at * (torch.exp(-h) - 1.0)) * m
        else:
            s0, s1 = timestep, self.timesteps[step_index - 1]
            m0, m1 = self.model_outputs[-1], self.model_outputs[-2]
            h, h_0 = lt - self.lambda_t[s0], self.lambda_t[s0] - self.lambda_t[s1]
            r0 = h_0 / h
            D0, D1 = m0, (1.0 / r0) * (m0 - m1)
            prev = ((st / self.sigma_t[s0]) * sample - (at * (torch.exp(-h) - 1.0)) * D0
                    - 0.5 * (at * (torch.exp(-h) - 1.0)) * D1)
        if self.lower_order_nums < 2:
            self.lower_order_nums += 1
        return prev


class DDIM:
    """e4t_oracle.ddim_step / sd2_oracle.ddim_step (eta = 0) behind the same interface."""
    needs_noise = False

    def __init__(self, prediction_type="epsilon", num_train=1000):
        self.prediction_type, self.num_train = prediction_type, num_train
        self.init_noise_sigma = 1.0

    def set_timesteps(self, n):
        self.n = n
        self.timesteps = O.ddim_timesteps(n)

    def scale_model_input(self, x, t):
        return x

    def step(self, model_output, timestep, sample, noise=None):
        from oracle import sd2_oracle as S
        acp = O.ddpm_alphas_cumprod().to(sample.dtype)
        return S.ddim_step(model_output, timestep, sample, self.n, acp, prediction_type=self.prediction_type)


SCHEDULERS = {"ddim": DDIM, "plms": PNDM, "lms": LMS, "euler": Euler, "euler_ancestral": EulerAncestral,
              "dpm_solver++": DPMSolverPP}


def make(name, prediction_type="epsilon"):
    return SCHEDULERS[name](prediction_type)


def needs_noise(sched, i):
    f = getattr(sched, "needs_noise_at", None)
    return f(i) if f is not None else sched.needs_noise


def pipeline_sample(sd_unet, ucfg, sd_enc, vcfg, sd_text, tcfg, image, input_ids, latents, num_inference_steps=4,
                    guidance_scale=7.5, class_token_id=320, domain_embed_scale=0.1, scheduler="ddim",
                    prediction_type="epsilon", pad_id=O.EOS, generator=None, sd2=False):
    """e4t_oracle.pipeline_sample / sd2_oracle.pipeline_sample (pipeline_stable_diffusion_e4t.py:181-216) over any
    scheduler above: `latents` are the unscaled N(0, 1) draw (multiplied by init_noise_sigma here), the model input is
    scale_model_input(x, t), timesteps may be fractional, and step noise is drawn from `generator` (fp32, latent-shaped)
    only on the steps that use it.  sd2=True runs sd2_oracle's UNet and text tower (SD 2.x shapes)."""
    from oracle import sd2_oracle as S2
    M = S2 if sd2 else O
    sched = make(scheduler, prediction_type) if isinstance(scheduler, str) else scheduler
    emb_w = sd_text["text_model.embeddings.token_embedding.weight"]
    bsz = latents.shape[0]
    idx = input_ids[0].tolist().index(O.PLACEHOLDER_ID)
    empty = S2.empty_prompt_ids(pad_id) if sd2 else [O.BOS] + [O.EOS] * 76
    with torch.no_grad():
        ehs_e4t = M.text_forward(sd_text, tcfg, input_ids=torch.tensor([empty])).expand(bsz, -1, -1)
        base_embeds = emb_w[input_ids]
        class_embed = emb_w[class_token_id]
        pix = image.expand(bsz, -1, -1, -1)
        sched.set_timesteps(num_inference_steps)
        x = latents.clone() * sched.init_noise_sigma
        for i, t in enumerate(sched.timesteps):
            tt = torch.full((bsz,), t, dtype=torch.float64 if isinstance(t, float) else torch.int64)
            xin = sched.scale_model_input(x, t).to(latents.dtype)
            enc = M.unet_forward(sd_unet, ucfg, xin, tt, ehs_e4t, return_encoder_outputs=True)
            dom = class_embed.expand(bsz, -1) + domain_embed_scale * O.encoder_forward(sd_enc, vcfg, pix,
                                                                                        enc["down_block_samples"])
            emb = base_embeds.expand(bsz, -1, -1).clone()
            emb[:, idx, :] = dom
            ehs = M.text_forward(sd_text, tcfg, inputs_embeds=emb)
            if guidance_scale > 1.0:
                out = M.unet_forward(sd_unet, ucfg, torch.cat([xin, xin]), torch.cat([tt, tt]),
                                     torch.cat([ehs_e4t, ehs]))
                u, c = out.chunk(2)
                out = u + guidance_scale * (c - u)
            else:
                out = M.unet_forward(sd_unet, ucfg, xin, tt, ehs)
            z = None
            if needs_noise(sched, i):
                z = torch.randn(tuple(x.shape), generator=generator, dtype=torch.float32)
            x = sched.step(out, t, x, noise=z).to(latents.dtype)
    return x
