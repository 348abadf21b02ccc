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


# ----------------------------------------------------------------------------------------------------------------------
# DDIM, Euler and DPM-Solver++ (multistep), restated from diffusers==0.25.0 for the engine. The diffusers source was
# not at hand when these were written: each docstring says which details are restated from memory of that release
# and could not be checked against it. The engine only reads the generic attributes (alphas_cumprod, sigmas,
# timesteps, config, ...), so a caller's own diffusers scheduler takes the same path (denoise.solver_step_tables).
# ----------------------------------------------------------------------------------------------------------------------
import inspect

import numpy as np


class _Config(dict):
    """A diffusers FrozenDict-like config: a dict whose keys are also attributes."""

    __getattr__ = dict.__getitem__


def _config_dict(config):
    if isinstance(config, dict):
        return dict(config)
    return {k: v for k, v in vars(type(config)).items() if not k.startswith("_")} | dict(vars(config))


class _FromConfig:
    @classmethod
    def from_config(cls, config, **kwargs):
        """diffusers `SchedulerMixin.from_config`: the keys of `config` (a dict, a FrozenDict or another scheduler's
        `config`) that this constructor takes, overridden by `kwargs`; other keys are ignored."""
        params = inspect.signature(cls.__init__).parameters
        kw = {k: v for k, v in _config_dict(config).items() if k in params and k != "self"}
        kw.update(kwargs)
        return cls(**kw)


def _betas(num_train_timesteps, beta_start, beta_end, beta_schedule, rescale_betas_zero_snr):
    if beta_schedule != "scaled_linear":
        raise NotImplementedError("only the scaled_linear beta schedule of the IDM-VTON scheduler config is restated")
    betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
    return _rescale_zero_terminal_snr(betas) if rescale_betas_zero_snr else betas


def _spaced_int_timesteps(n, steps, spacing, steps_offset):
    """DDPM / DDIM set_timesteps: `leading`, `trailing` or `linspace`, as int64, descending."""
    if steps > n:
        raise ValueError(f"num_inference_steps {steps} > num_train_timesteps {n}")
    if spacing == "leading":
        ratio = n // steps
        ts = (np.arange(0, steps) * ratio).round()[::-1].copy().astype(np.int64) + steps_offset
    elif spacing == "trailing":
        ts = np.round(np.arange(n, 0, -n / steps)).astype(np.int64) - 1
    elif spacing == "linspace":
        ts = np.linspace(0, n - 1, steps).round()[::-1].copy().astype(np.int64)
    else:
        raise ValueError(f"{spacing} is not supported. Please make sure to choose one of 'leading', 'trailing' or 'linspace'.")
    return torch.from_numpy(ts)


def _ddpm_add_noise(alphas_cumprod, original_samples, noise, timesteps):
    ac = alphas_cumprod.to(device=original_samples.device, dtype=original_samples.dtype)
    timesteps = timesteps.to(original_samples.device)
    shape = (-1,) + (1,) * (original_samples.ndim - 1)
    return (ac[timesteps] ** 0.5).reshape(shape) * original_samples + ((1 - ac[timesteps]) ** 0.5).reshape(shape) * noise


def _randn_like(x, generator):
    dev = x.device
    rand_dev = "cpu" if (generator is not None and generator.device.type == "cpu" and dev.type != "cpu") else dev
    return torch.randn(x.shape, generator=generator, device=rand_dev, dtype=x.dtype).to(dev)


def _init_step_index(timesteps, t):
    """diffusers `_init_step_index`: the position of `t` in the schedule; the second match when `t` occurs twice."""
    idx = (timesteps == t).nonzero()
    if len(idx) == 0:
        raise ValueError(f"timestep {float(t)} is not in the scheduler's timesteps")
    return int(idx[1 if len(idx) > 1 else 0])


class DDIMScheduler(_FromConfig):
    """diffusers 0.25 DDIMScheduler, epsilon prediction without clipping or thresholding.

    set_timesteps: the leading / trailing / linspace spacings of DDPMScheduler (int64). step(t) goes from t to
    prev_t = t - T_train // num_inference_steps (for every spacing, as diffusers does); at prev_t < 0, alpha_prev is
    `final_alpha_cumprod` (1 with `set_alpha_to_one`, else alphas_cumprod[0]). With a = alphas_cumprod[t]:
        x0 = (x - sqrt(1 - a) eps) / sqrt(a);   var = (1 - a_prev) / (1 - a) * (1 - a / a_prev);   sigma = eta sqrt(var)
        prev = sqrt(a_prev) x0 + sqrt(1 - a_prev - sigma^2) eps  [+ sigma * noise, drawn in the model output's dtype
        from `generator` only when eta > 0]
    The coefficients are fp32 CPU tensors and the arithmetic runs in the dtype of the model output: on fp16 tensors
    each product and sum rounds to fp16 (the rounding points of b200vton_cfg_solver_step kind 0). `set_alpha_to_one`
    defaults to True, and the engine's DDPMScheduler config has no such key, so `from_config` of it ends the last step at
    alpha = 1; a checkpoint scheduler config that sets it to False (as SDXL-derived configs commonly do) ends at
    alphas_cumprod[0]. The engine reads `final_alpha_cumprod` from the caller's object, so both are stepped as
    configured. Restated from memory of
    the 0.25 source, not checked against it: `step` has no fp32 upcast; `use_clipped_model_output` only matters with
    clipping or thresholding, both of which raise here."""

    order = 1
    init_noise_sigma = 1.0

    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                 trained_betas=None, clip_sample=True, set_alpha_to_one=True, steps_offset=0, prediction_type="epsilon",
                 thresholding=False, dynamic_thresholding_ratio=0.995, clip_sample_range=1.0, sample_max_value=1.0,
                 timestep_spacing="leading", rescale_betas_zero_snr=False):
        if trained_betas is not None:
            raise NotImplementedError("trained_betas is not restated")
        self.config = _Config(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                              beta_schedule=beta_schedule, trained_betas=trained_betas, clip_sample=clip_sample,
                              set_alpha_to_one=set_alpha_to_one, steps_offset=steps_offset,
                              prediction_type=prediction_type, thresholding=thresholding,
                              dynamic_thresholding_ratio=dynamic_thresholding_ratio,
                              clip_sample_range=clip_sample_range, sample_max_value=sample_max_value,
                              timestep_spacing=timestep_spacing, rescale_betas_zero_snr=rescale_betas_zero_snr)
        self.betas = _betas(num_train_timesteps, beta_start, beta_end, beta_schedule, rescale_betas_zero_snr)
        self.alphas = 1.0 - self.betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        self.final_alpha_cumprod = torch.tensor(1.0) if set_alpha_to_one else self.alphas_cumprod[0]
        self.num_inference_steps = None
        self.timesteps = torch.from_numpy(np.arange(0, num_train_timesteps)[::-1].copy().astype(np.int64))

    def set_timesteps(self, num_inference_steps, device=None):
        self.num_inference_steps = num_inference_steps
        ts = _spaced_int_timesteps(self.config.num_train_timesteps, num_inference_steps, self.config.timestep_spacing,
                                   self.config.steps_offset)
        self.timesteps = ts.to(device) if device is not None else ts

    def scale_model_input(self, sample, timestep=None):
        return sample

    def add_noise(self, original_samples, noise, timesteps):
        return _ddpm_add_noise(self.alphas_cumprod, original_samples, noise, timesteps)

    def _get_variance(self, t, prev_t):
        a = self.alphas_cumprod[t]
        a_prev = self.alphas_cumprod[prev_t] if prev_t >= 0 else self.final_alpha_cumprod
        return (1 - a_prev) / (1 - a) * (1 - a / a_prev)

    def step(self, model_output, timestep, sample, eta=0.0, use_clipped_model_output=False, generator=None,
             variance_noise=None, return_dict=True):
        if self.config.prediction_type != "epsilon" or self.config.clip_sample or self.config.thresholding:
            raise NotImplementedError("epsilon prediction without clip_sample / thresholding is restated")
        t = int(timestep)
        prev_t = t - self.config.num_train_timesteps // self.num_inference_steps
        a = self.alphas_cumprod[t]
        a_prev = self.alphas_cumprod[prev_t] if prev_t >= 0 else self.final_alpha_cumprod
        pred_original_sample = (sample - (1 - a) ** 0.5 * model_output) / a ** 0.5
        std_dev_t = eta * self._get_variance(t, prev_t) ** 0.5
        prev_sample = a_prev ** 0.5 * pred_original_sample + (1 - a_prev - std_dev_t ** 2) ** 0.5 * model_output
        self._last_noise = None
        if eta > 0:
            if variance_noise is None:
                variance_noise = _randn_like(model_output, generator)
            prev_sample = prev_sample + std_dev_t * variance_noise
            self._last_noise = variance_noise
        if not return_dict:
            return (prev_sample,)
        return type("DDIMSchedulerOutput", (), dict(prev_sample=prev_sample,
                                                    pred_original_sample=pred_original_sample))()


class EulerDiscreteScheduler(_FromConfig):
    """diffusers 0.25 EulerDiscreteScheduler, epsilon prediction, linear interpolation, s_churn = 0.

    set_timesteps: float32 timesteps, `linspace` = linspace(0, T - 1, N) reversed (fractional), `leading` =
    arange(N) * (T // N) reversed + steps_offset, `trailing` = round(arange(T, 0, -T / N)) - 1; sigmas =
    sqrt((1 - a) / a) interpolated linearly at the timesteps, then a final 0 (N + 1 values, fp32).
    init_noise_sigma = max sigma for linspace / trailing, sqrt(max sigma^2 + 1) for leading.
    scale_model_input(x, t) = x / sqrt(sigma^2 + 1) with sigma at the step index.
    step: x0 = x - sigma * eps;  d = (x - x0) / sigma;  prev = x + d * (sigma_next - sigma).
    Restated from memory of the 0.25 source, not checked against it: `step` draws one variance-noise tensor from
    `generator` on every call even at s_churn = 0 (it is multiplied by zero and unused), in the model output's dtype;
    `step` upcasts the sample to fp32 first and casts the result back to the model output's dtype, while
    `sigma * eps` is a CPU fp32 scalar times the model output (so it rounds to fp16 on fp16 tensors); the sigmas live
    on the CPU, so every divisor is a CPU scalar; the step index is set by the first `scale_model_input` / `step` call
    at the position of that timestep in `timesteps` (the second match if it occurs twice) and advances by one per step;
    `add_noise` is x0 + sigma_t * noise with sigma_t at the position of t in `timesteps`. Karras sigmas, other
    interpolation types and s_churn > 0 are not restated and raise."""

    order = 1

    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                 trained_betas=None, prediction_type="epsilon", interpolation_type="linear", use_karras_sigmas=False,
                 timestep_spacing="linspace", steps_offset=0, rescale_betas_zero_snr=False):
        if trained_betas is not None or use_karras_sigmas or interpolation_type != "linear":
            raise NotImplementedError("trained_betas, use_karras_sigmas and interpolation types other than linear are "
                                      "not restated")
        self.config = _Config(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                              beta_schedule=beta_schedule, trained_betas=trained_betas, prediction_type=prediction_type,
                              interpolation_type=interpolation_type, use_karras_sigmas=use_karras_sigmas,
                              timestep_spacing=timestep_spacing, steps_offset=steps_offset,
                              rescale_betas_zero_snr=rescale_betas_zero_snr)
        self.betas = _betas(num_train_timesteps, beta_start, beta_end, beta_schedule, rescale_betas_zero_snr)
        self.alphas = 1.0 - self.betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        self.num_inference_steps = None
        self.set_timesteps(num_train_timesteps)
        self.num_inference_steps = None

    @property
    def init_noise_sigma(self):
        max_sigma = self.sigmas.max()
        if self.config.timestep_spacing in ("linspace", "trailing"):
            return max_sigma
        return (max_sigma ** 2 + 1) ** 0.5

    @property
    def step_index(self):
        return self._step_index

    def set_timesteps(self, num_inference_steps, device=None):
        self.num_inference_steps = num_inference_steps
        n = self.config.num_train_timesteps
        sp = self.config.timestep_spacing
        if sp == "linspace":
            ts = np.linspace(0, n - 1, num_inference_steps, dtype=np.float32)[::-1].copy()
        elif sp == "leading":
            ratio = n // num_inference_steps
            ts = (np.arange(0, num_inference_steps) * ratio).round()[::-1].copy().astype(np.float32)
            ts += self.config.steps_offset
        elif sp == "trailing":
            ratio = n / num_inference_steps
            ts = (np.arange(n, 0, -ratio)).round().copy().astype(np.float32)
            ts -= 1
        else:
            raise ValueError(f"{sp} is not supported. Please make sure to choose one of 'linspace', 'leading' or 'trailing'.")
        sigmas = np.array(((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5)
        sigmas = np.interp(ts, np.arange(0, len(sigmas)), sigmas)
        sigmas = np.concatenate([sigmas, [0.0]]).astype(np.float32)
        self.sigmas = torch.from_numpy(sigmas)
        ts = torch.from_numpy(ts)
        self.timesteps = ts.to(device) if device is not None else ts
        self._step_index = None

    def _index(self, timestep):
        if self._step_index is None:
            self._step_index = _init_step_index(self.timesteps.cpu(), timestep)
        return self._step_index

    def scale_model_input(self, sample, timestep):
        sigma = self.sigmas[self._index(timestep)]
        return sample / ((sigma ** 2 + 1) ** 0.5)

    def add_noise(self, original_samples, noise, timesteps):
        sigmas = self.sigmas.to(device=original_samples.device, dtype=original_samples.dtype)
        sched = self.timesteps.to(original_samples.device)
        idx = [(sched == t).nonzero().item() for t in timesteps.to(original_samples.device)]
        sigma = sigmas[idx].flatten()
        while sigma.ndim < original_samples.ndim:
            sigma = sigma.unsqueeze(-1)
        return original_samples + noise * sigma

    def step(self, model_output, timestep, sample, s_churn=0.0, s_tmin=0.0, s_tmax=float("inf"), s_noise=1.0,
             generator=None, return_dict=True):
        if s_churn > 0 or self.config.prediction_type != "epsilon":
            raise NotImplementedError("s_churn > 0 and non-epsilon prediction are not restated")
        i = self._index(timestep)
        sample = sample.to(torch.float32)
        sigma = self.sigmas[i]
        self._last_noise = _randn_like(model_output, generator)          # drawn and unused at s_churn = 0
        pred_original_sample = sample - sigma * model_output
        derivative = (sample - pred_original_sample) / sigma
        prev_sample = sample + derivative * (self.sigmas[i + 1] - sigma)
        prev_sample = prev_sample.to(model_output.dtype)
        self._step_index += 1
        if not return_dict:
            return (prev_sample,)
        return type("EulerDiscreteSchedulerOutput", (), dict(prev_sample=prev_sample,
                                                             pred_original_sample=pred_original_sample))()


class DPMSolverMultistepScheduler(_FromConfig):
    """diffusers 0.25 DPMSolverMultistepScheduler, algorithm_type `dpmsolver++`, solver_type `midpoint`, solver_order 1 or
    2, epsilon prediction (DPM-Solver++(2M), Lu et al. 2022, Alg. 2).

    set_timesteps: int64 timesteps from linspace(0, T - 1, N + 1) (`linspace`), arange(N + 1) * (T // (N + 1)) +
    steps_offset (`leading`) or round(arange(T, 0, -T / N)) - 1 (`trailing`), each descending without its last entry
    where diffusers drops it; sigmas = sqrt((1 - a) / a) interpolated at the timesteps. With use_karras_sigmas the
    sigmas are Karras et al.'s rho = 7 ramp between the largest and smallest training sigma and the timesteps are
    those sigmas mapped back by log-sigma interpolation, rounded. On the solver's scale, alpha_t = 1 / sqrt(sigma^2 + 1)
    and sigma_t = sigma * alpha_t, lambda = log alpha_t - log sigma_t, h = lambda_next - lambda.
    step at index i: x0 = (x - sigma_t eps) / alpha_t (fp16 on fp16 tensors), then with the sample upcast to fp32
        order 1:  prev = (sigma_t' / sigma_t) x - alpha_t' (e^-h - 1) x0
        order 2:  prev = (sigma_t' / sigma_t) x - alpha_t' (e^-h - 1) x0 - 0.5 alpha_t' (e^-h - 1) (1 / r0) (x0 - x0_prev),
                  r0 = h_prev / h
    cast back to the model output's dtype. The first step of a run is order 1; with lower_order_final and fewer than 15
    timesteps (or euler_at_final) the last one is too. Restated from memory of the 0.25 source, not checked against it:
    the final sigma is sqrt((1 - a_0) / a_0) without Karras sigmas and a repeat of the last sigma with them (so the last
    Karras step is the identity); `add_noise` uses the alphas_cumprod parametrisation of DDPM even with Karras sigmas;
    the sigmas live on the CPU; `step` upcasts the sample to fp32 after the data prediction is formed; no draw from
    `generator` happens; Karras timesteps are not de-duplicated; the step index is found and advanced as for Euler."""

    order = 1
    init_noise_sigma = 1.0

    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                 trained_betas=None, solver_order=2, prediction_type="epsilon", thresholding=False,
                 dynamic_thresholding_ratio=0.995, sample_max_value=1.0, algorithm_type="dpmsolver++",
                 solver_type="midpoint", lower_order_final=True, euler_at_final=False, use_karras_sigmas=False,
                 use_lu_lambdas=False, lambda_min_clipped=-float("inf"), variance_type=None,
                 timestep_spacing="linspace", steps_offset=0):
        if trained_betas is not None:
            raise NotImplementedError("trained_betas is not restated")
        if algorithm_type not in ("dpmsolver", "dpmsolver++", "sde-dpmsolver", "sde-dpmsolver++"):
            raise NotImplementedError(f"{algorithm_type} does is not implemented for {self.__class__}")
        if solver_type not in ("midpoint", "heun"):
            raise NotImplementedError(f"{solver_type} does is not implemented for {self.__class__}")
        self.config = _Config(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                              beta_schedule=beta_schedule, trained_betas=trained_betas, solver_order=solver_order,
                              prediction_type=prediction_type, thresholding=thresholding,
                              dynamic_thresholding_ratio=dynamic_thresholding_ratio, sample_max_value=sample_max_value,
                              algorithm_type=algorithm_type, solver_type=solver_type,
                              lower_order_final=lower_order_final, euler_at_final=euler_at_final,
                              use_karras_sigmas=use_karras_sigmas, use_lu_lambdas=use_lu_lambdas,
                              lambda_min_clipped=lambda_min_clipped, variance_type=variance_type,
                              timestep_spacing=timestep_spacing, steps_offset=steps_offset)
        self.betas = _betas(num_train_timesteps, beta_start, beta_end, beta_schedule, False)
        self.alphas = 1.0 - self.betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        self.num_inference_steps = None
        self.timesteps = torch.from_numpy(np.linspace(0, num_train_timesteps - 1, num_train_timesteps,
                                                      dtype=np.float32)[::-1].copy())
        self.model_outputs = [None] * solver_order
        self.lower_order_nums = 0
        self._step_index = None

    @property
    def step_index(self):
        return self._step_index

    def _supported(self):
        c = self.config
        if (c.solver_order not in (1, 2) or c.algorithm_type != "dpmsolver++" or c.solver_type != "midpoint"
                or c.thresholding or c.prediction_type != "epsilon" or c.use_lu_lambdas):
            raise NotImplementedError("dpmsolver++ / midpoint at solver_order 1 or 2 with epsilon prediction, no "
                                      "thresholding and no use_lu_lambdas is restated")

    @staticmethod
    def _sigma_to_t(sigma, log_sigmas):
        log_sigma = np.log(np.maximum(sigma, 1e-10))
        dists = log_sigma - log_sigmas[:, np.newaxis]
        low_idx = np.cumsum((dists >= 0), axis=0).argmax(axis=0).clip(max=log_sigmas.shape[0] - 2)
        high_idx = low_idx + 1
        low, high = log_sigmas[low_idx], log_sigmas[high_idx]
        w = np.clip((low - log_sigma) / (low - high), 0, 1)
        t = (1 - w) * low_idx + w * high_idx
        return t.reshape(sigma.shape)

    @staticmethod
    def _convert_to_karras(in_sigmas, num_inference_steps):
        sigma_min, sigma_max = in_sigmas[-1].item(), in_sigmas[0].item()
        rho = 7.0
        ramp = np.linspace(0, 1, num_inference_steps)
        min_inv_rho, max_inv_rho = sigma_min ** (1 / rho), sigma_max ** (1 / rho)
        return (max_inv_rho + ramp * (min_inv_rho - max_inv_rho)) ** rho

    def set_timesteps(self, num_inference_steps=None, device=None):
        self._supported()
        n = self.config.num_train_timesteps
        last = n          # lambda_min_clipped = -inf clips nothing
        sp = self.config.timestep_spacing
        if sp == "linspace":
            ts = np.linspace(0, last - 1, num_inference_steps + 1).round()[::-1][:-1].copy().astype(np.int64)
        elif sp == "leading":
            ratio = last // (num_inference_steps + 1)
            ts = (np.arange(0, num_inference_steps + 1) * ratio).round()[::-1][:-1].copy().astype(np.int64)
            ts += self.config.steps_offset
        elif sp == "trailing":
            ratio = n / num_inference_steps
            ts = np.arange(last, 0, -ratio).round().copy().astype(np.int64)
            ts -= 1
        else:
            raise ValueError(f"{sp} is not supported. Please make sure to choose one of 'linspace', 'leading' or 'trailing'.")
        sigmas = np.array(((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5)
        log_sigmas = np.log(sigmas)
        if self.config.use_karras_sigmas:
            sigmas = np.flip(sigmas).copy()
            sigmas = self._convert_to_karras(sigmas, num_inference_steps)
            ts = np.array([self._sigma_to_t(s, log_sigmas) for s in sigmas]).round()
            sigmas = np.concatenate([sigmas, sigmas[-1:]]).astype(np.float32)
        else:
            sigmas = np.interp(ts, np.arange(0, len(sigmas)), sigmas)
            sigma_last = (((1 - self.alphas_cumprod[0]) / self.alphas_cumprod[0]) ** 0.5).item()
            sigmas = np.concatenate([sigmas, [sigma_last]]).astype(np.float32)
        self.sigmas = torch.from_numpy(sigmas)
        ts = torch.from_numpy(ts).to(torch.int64)
        self.timesteps = ts.to(device) if device is not None else ts
        self.num_inference_steps = len(ts)
        self.model_outputs = [None] * self.config.solver_order
        self.lower_order_nums = 0
        self._step_index = None

    @staticmethod
    def _sigma_to_alpha_sigma_t(sigma):
        alpha_t = 1 / ((sigma ** 2 + 1) ** 0.5)
        return alpha_t, sigma * alpha_t

    def scale_model_input(self, sample, timestep=None):
        return sample

    def add_noise(self, original_samples, noise, timesteps):
        return _ddpm_add_noise(self.alphas_cumprod, original_samples, noise, timesteps)

    def step_orders(self, start, count):
        """Solver order of the `count` steps a run takes from step index `start` (the first step of a run is order 1)."""
        n = len(self.timesteps)
        return [solver_order_at(j, start + j, n, self.config) for j in range(count)]

    def step(self, model_output, timestep, sample, generator=None, return_dict=True):
        self._supported()
        if self._step_index is None:
            self._step_index = _init_step_index(self.timesteps.cpu(), timestep)
        i = self._step_index
        alpha_t, sigma_t = self._sigma_to_alpha_sigma_t(self.sigmas[i])
        x0 = (sample - sigma_t * model_output) / alpha_t                                 # convert_model_output
        self.model_outputs = self.model_outputs[1:] + [x0]
        sample = sample.to(torch.float32)
        order = solver_order_at(self.lower_order_nums, i, len(self.timesteps), self.config)
        alpha_n, sigma_n = self._sigma_to_alpha_sigma_t(self.sigmas[i + 1])
        lam_n, lam = torch.log(alpha_n) - torch.log(sigma_n), torch.log(alpha_t) - torch.log(sigma_t)
        h = lam_n - lam
        c = alpha_n * (torch.exp(-h) - 1.0)
        prev_sample = (sigma_n / sigma_t) * sample - c * x0
        if order == 2:
            alpha_p, sigma_p = self._sigma_to_alpha_sigma_t(self.sigmas[i - 1])
            r0 = (lam - (torch.log(alpha_p) - torch.log(sigma_p))) / h
            prev_sample = prev_sample - 0.5 * c * ((1.0 / r0) * (x0 - self.model_outputs[-2]))
        prev_sample = prev_sample.to(model_output.dtype)
        if self.lower_order_nums < self.config.solver_order:
            self.lower_order_nums += 1
        self._step_index += 1
        self._last_noise = None
        if not return_dict:
            return (prev_sample,)
        return type("SchedulerOutput", (), dict(prev_sample=prev_sample))()


def config_getter(config):
    """get(key, default) on a scheduler config: a dict (diffusers' FrozenDict) or an object with attributes (or None)."""
    return (lambda k, d=None: config.get(k, d)) if isinstance(config, dict) else (lambda k, d=None: getattr(config, k, d))


def solver_order_at(steps_taken, step_index, n_timesteps, config):
    """Order of DPMSolverMultistepScheduler.step at `step_index` of a schedule of `n_timesteps`, after `steps_taken`
    steps of this run: 1 for the run's first step, for solver_order 1, and for the last step of the schedule when
    euler_at_final is set or lower_order_final is set with fewer than 15 timesteps; 2 otherwise."""
    get = config_getter(config)
    final = step_index == n_timesteps - 1 and (get("euler_at_final", False)
                                               or (get("lower_order_final", True) and n_timesteps < 15))
    if get("solver_order", 2) == 1 or steps_taken < 1 or final:
        return 1
    return 2
