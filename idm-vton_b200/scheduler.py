"""DDPM ancestral scheduler with the reference pipeline's configuration (host side, plain torch fp32).

Restates diffusers==0.25.0 DDPMScheduler as used by src/tryon_pipeline.py:1561,1823 (set_timesteps / step) for:
scaled_linear betas 0.00085..0.012, 1000 train steps, epsilon prediction, fixed_small variance, leading spacing with
steps_offset 1, optional zero-terminal-SNR rescale (train_xl.py:317). The per-step arithmetic itself runs in
b200vton_cfg_ddpm_step; this class produces the timestep list (or takes a custom one), the per-step scalar coefficients
and the forward-process noising of add_noise (strength < 1).
"""
import torch


def _rescale_zero_terminal_snr(betas):
    alphas = 1.0 - betas
    alphas_cumprod = torch.cumprod(alphas, dim=0)
    alphas_bar_sqrt = alphas_cumprod.sqrt()
    a0 = alphas_bar_sqrt[0].clone()
    aT = alphas_bar_sqrt[-1].clone()
    alphas_bar_sqrt = alphas_bar_sqrt - aT
    alphas_bar_sqrt = alphas_bar_sqrt * (a0 / (a0 - aT))
    alphas_bar = alphas_bar_sqrt ** 2
    alphas = alphas_bar[1:] / alphas_bar[:-1]
    alphas = torch.cat([alphas_bar[0:1], alphas])
    return 1 - alphas


class DDPMScheduler:
    order = 1
    init_noise_sigma = 1.0

    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                 timestep_spacing="leading", steps_offset=1, rescale_betas_zero_snr=False,
                 prediction_type="epsilon", variance_type="fixed_small", clip_sample=False):
        if beta_schedule != "scaled_linear" or prediction_type != "epsilon" or variance_type != "fixed_small" or clip_sample:
            raise NotImplementedError("only the IDM-VTON scheduler configuration is supported")
        if timestep_spacing not in ("leading", "trailing", "linspace"):
            raise ValueError(timestep_spacing)
        self.config = type("Cfg", (), dict(num_train_timesteps=num_train_timesteps, beta_start=beta_start,
                                           beta_end=beta_end, beta_schedule=beta_schedule,
                                           timestep_spacing=timestep_spacing, steps_offset=steps_offset,
                                           rescale_betas_zero_snr=rescale_betas_zero_snr,
                                           prediction_type=prediction_type, variance_type=variance_type,
                                           clip_sample=clip_sample))()
        betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
        if rescale_betas_zero_snr:
            betas = _rescale_zero_terminal_snr(betas)
        self.betas = betas
        self.alphas = 1.0 - betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        self.one = torch.tensor(1.0)
        self.num_inference_steps = None
        self.custom_timesteps = False
        self.timesteps = torch.arange(num_train_timesteps - 1, -1, -1)

    def set_timesteps(self, num_inference_steps=None, device=None, timesteps=None):
        """diffusers 0.25 semantics: either a step count (spaced by `timestep_spacing`) or a custom list of train
        timesteps, strictly descending and below num_train_timesteps (`custom_timesteps` is then set)."""
        n = self.config.num_train_timesteps
        if num_inference_steps is not None and timesteps is not None:
            raise ValueError("Can only pass one of `num_inference_steps` or `custom_timesteps`.")
        if timesteps is not None:
            ts = [int(t) for t in timesteps]
            if any(a <= b for a, b in zip(ts, ts[1:])):
                raise ValueError("`custom_timesteps` must be in descending order.")
            if ts[0] >= n:
                raise ValueError(f"`timesteps` must start before `self.config.train_timesteps`: {n}.")
            self.custom_timesteps = True
            ts = torch.tensor(ts, dtype=torch.int64)
            self.timesteps = ts.to(device) if device is not None else ts
            return
        if num_inference_steps > n:
            raise ValueError(f"num_inference_steps {num_inference_steps} > num_train_timesteps {n}")
        self.custom_timesteps = False
        self.num_inference_steps = num_inference_steps
        sp = self.config.timestep_spacing
        if sp == "leading":
            ratio = n // num_inference_steps
            ts = (torch.arange(0, num_inference_steps, dtype=torch.float64) * ratio).round().flip(0).to(torch.int64)
            ts = ts + self.config.steps_offset
        elif sp == "trailing":
            ratio = n / num_inference_steps
            ts = (torch.arange(n, 0, -ratio, dtype=torch.float64)).round().to(torch.int64) - 1
        else:
            ts = torch.linspace(0, n - 1, num_inference_steps, dtype=torch.float64).round().flip(0).to(torch.int64)
        self.timesteps = ts.to(device) if device is not None else ts

    def add_noise(self, original_samples, noise, timesteps):
        """sqrt(abar_t) * x0 + sqrt(1 - abar_t) * noise per sample, with alphas_cumprod cast to the samples' dtype and
        device first (diffusers DDPMScheduler.add_noise)."""
        ac = self.alphas_cumprod.to(device=original_samples.device, dtype=original_samples.dtype)
        timesteps = timesteps.to(original_samples.device)
        sqrt_a = ac[timesteps] ** 0.5
        sqrt_1ma = (1 - ac[timesteps]) ** 0.5
        shape = (-1,) + (1,) * (original_samples.ndim - 1)
        return sqrt_a.reshape(shape) * original_samples + sqrt_1ma.reshape(shape) * noise

    def scale_model_input(self, sample, timestep=None):
        return sample

    def previous_timestep(self, t):
        if self.custom_timesteps:
            ts = self.timesteps.tolist()
            i = ts.index(int(t))
            return ts[i + 1] if i + 1 < len(ts) else -1
        steps = self.num_inference_steps if self.num_inference_steps else self.config.num_train_timesteps
        return t - self.config.num_train_timesteps // steps

    def step(self, model_output, timestep, sample, generator=None, return_dict=True):
        """diffusers DDPMScheduler.step (epsilon prediction, fixed_small variance) on the host in plain torch — the
        arithmetic the reference loop runs at src/tryon_pipeline.py:1823. The engine does NOT call this (its per-step
        update is the fused `b200vton_cfg_ddpm_step` kernel fed by `step_coefficients`); it exists so this object is a
        complete scheduler for callers that step it themselves (e.g. the reference pipeline in oracle/make_golden_pipeline.py)."""
        t = int(timestep)
        prev_t = self.previous_timestep(t)
        a_t = self.alphas_cumprod[t]
        a_prev = self.alphas_cumprod[prev_t] if prev_t >= 0 else self.one
        b_t, b_prev = 1 - a_t, 1 - a_prev
        cur_a = a_t / a_prev
        cur_b = 1 - cur_a
        pred_original_sample = (sample - b_t ** 0.5 * model_output) / a_t ** 0.5
        pred_prev_sample = (a_prev ** 0.5 * cur_b) / b_t * pred_original_sample + cur_a ** 0.5 * b_prev / b_t * sample
        self._last_noise = None
        if t > 0:
            dev = model_output.device
            rand_dev = "cpu" if (generator is not None and generator.device.type == "cpu" and dev.type != "cpu") else dev
            noise = torch.randn(model_output.shape, generator=generator, device=rand_dev, dtype=model_output.dtype).to(dev)
            var = torch.clamp((1 - a_prev) / (1 - a_t) * cur_b, min=1e-20)
            pred_prev_sample = pred_prev_sample + (var ** 0.5) * noise
            self._last_noise = noise
        if not return_dict:
            return (pred_prev_sample,)
        return type("DDPMSchedulerOutput", (), dict(prev_sample=pred_prev_sample, pred_original_sample=pred_original_sample))()

    def step_coefficients(self, t):
        """(sqrt(1-abar_t), 1/sqrt(abar_t), x0 coeff, x_t coeff, sigma_t) as python floats, computed in fp32 torch
        exactly like DDPMScheduler.step / _get_variance."""
        t = int(t)
        prev_t = self.previous_timestep(t)
        a_t = self.alphas_cumprod[t]
        a_prev = self.alphas_cumprod[prev_t] if prev_t >= 0 else self.one
        b_t = 1 - a_t
        b_prev = 1 - a_prev
        cur_a = a_t / a_prev
        cur_b = 1 - cur_a
        c0 = (a_prev ** 0.5 * cur_b) / b_t
        c1 = cur_a ** 0.5 * b_prev / b_t
        var = torch.clamp((1 - a_prev) / (1 - a_t) * cur_b, min=1e-20)
        sigma = var ** 0.5 if t > 0 else torch.tensor(0.0)
        inv_sa = torch.tensor(1.0, dtype=torch.float32) / (a_t ** 0.5)
        return float(b_t ** 0.5), float(inv_sa), float(c0), float(c1), float(sigma)
