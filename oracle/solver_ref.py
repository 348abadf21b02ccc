"""ORACLE (test infrastructure, not product): float64 update rules of the three fast samplers the engine runs, written
from the papers rather than from idm_vton_b200/scheduler.py, and the denoising loop of src/tryon_pipeline.py:1765-1866
driven by any of them (`scale_model_input` before the channel concat at :1772-1777, `step` at :1823).

  DDIM            Song et al. 2020, eq. 12 (sigma of eq. 16 times eta)
  Euler           Karras et al. 2022, Alg. 1 without churn, on the probability-flow ODE dx/dsigma = (x - D(x)) / sigma
  DPM-Solver++(2M) Lu et al. 2022, Alg. 2 (data prediction, multistep, second order; first order at the first step)

Built on oracle/unet_ref.py like oracle/schedule_ref.py; loop_ref.py and schedule_ref.py are unchanged. Only tests/
imports this module.
"""
import math

import torch

from . import unet_ref as R


def ddim_update(x, eps, a_t, a_prev, eta=0.0, noise=None):
    """Song et al. eq. 12: x_prev = sqrt(a_prev) x0 + sqrt(1 - a_prev - s^2) eps + s z, x0 = (x - sqrt(1 - a_t) eps) /
    sqrt(a_t), s = eta sqrt((1 - a_prev) / (1 - a_t)) sqrt(1 - a_t / a_prev) (eq. 16)."""
    s = eta * math.sqrt((1 - a_prev) / (1 - a_t)) * math.sqrt(1 - a_t / a_prev)
    x0 = (x - math.sqrt(1 - a_t) * eps) / math.sqrt(a_t)
    out = math.sqrt(a_prev) * x0 + math.sqrt(1 - a_prev - s * s) * eps
    if noise is not None and s > 0:
        out = out + s * noise
    return out


def euler_update(x, eps, sigma, sigma_next):
    """Karras et al. Alg. 1 (S_churn = 0): D = x - sigma eps, d = (x - D) / sigma, x_next = x + (sigma_next - sigma) d;
    x lives on the sigma scale x = x0 + sigma n."""
    denoised = x - sigma * eps
    return x + (sigma_next - sigma) * (x - denoised) / sigma


def dpmpp_update(x, x0, alpha_t, sigma_t, alpha_n, sigma_n, x0_prev=None, lam_prev=None):
    """Lu et al. Alg. 2: h = lambda_n - lambda_t (lambda = log(alpha / sigma)); first order
    x_n = (sigma_n / sigma_t) x - alpha_n (e^-h - 1) x0; second order with r = (lambda_t - lambda_prev) / h,
    D = (1 + 1 / (2 r)) x0 - 1 / (2 r) x0_prev in place of x0."""
    lam_t, lam_n = math.log(alpha_t / sigma_t), math.log(alpha_n / sigma_n)
    h = lam_n - lam_t
    d = x0
    if x0_prev is not None:
        r = (lam_t - lam_prev) / h
        d = (1 + 1 / (2 * r)) * x0 - 1 / (2 * r) * x0_prev
    return (sigma_n / sigma_t) * x - alpha_n * math.expm1(-h) * d


class SolverRef:
    """The per-step arithmetic of a scheduler object in float64, from its generic attributes (alphas_cumprod, sigmas,
    timesteps, num_inference_steps, config). kind: "ddim" | "euler" | "dpmpp"."""

    def __init__(self, scheduler, kind, eta=0.0):
        self.kind, self.eta = kind, eta
        self.sch = scheduler
        self.ac = scheduler.alphas_cumprod.double().cpu()
        self.x0_prev = self.lam_prev = None
        self.taken = 0
        if kind != "ddim":
            self.sig = scheduler.sigmas.double().cpu()
            ts = scheduler.timesteps.double().cpu()
            self.index_of = {}
            for i, t in enumerate(ts.tolist()):
                self.index_of.setdefault(t, i)

    def scale(self, t):
        if self.kind != "euler":
            return 1.0
        return 1.0 / math.sqrt(self.sig[self.index_of[float(t)]].item() ** 2 + 1)

    def step(self, eps, t, x, noise=None):
        cfg = self.sch.config
        get = (lambda k, d=None: cfg.get(k, d)) if isinstance(cfg, dict) else (lambda k, d=None: getattr(cfg, k, d))
        if self.kind == "ddim":
            t = int(t)
            prev = t - get("num_train_timesteps") // self.sch.num_inference_steps
            a_prev = self.ac[prev].item() if prev >= 0 else (1.0 if get("set_alpha_to_one", True) else self.ac[0].item())
            return ddim_update(x, eps, self.ac[t].item(), a_prev, self.eta, noise)
        i = self.index_of[float(t)]
        s, s_next = self.sig[i].item(), self.sig[i + 1].item()
        if self.kind == "euler":
            return euler_update(x, eps, s, s_next)
        a_t, a_n = 1 / math.sqrt(s * s + 1), 1 / math.sqrt(s_next * s_next + 1)
        sigma_t, sigma_n = s * a_t, s_next * a_n
        x0 = (x - sigma_t * eps) / a_t
        n = len(self.sch.timesteps)
        last = i == n - 1 and (get("euler_at_final", False) or (get("lower_order_final", True) and n < 15))
        second = self.taken > 0 and get("solver_order", 2) == 2 and not last
        out = dpmpp_update(x, x0, a_t, sigma_t, a_n, sigma_n, self.x0_prev if second else None, self.lam_prev)
        self.x0_prev, self.lam_prev = x0, math.log(a_t / sigma_t)
        self.taken += 1
        return out


def denoise_loop(sd_t, cfg_t, sd_g, cfg_g, inp, scheduler, kind, timesteps, guidance_scale=2.0, eta=0.0, noises=None,
                 max_steps=None):
    """src/tryon_pipeline.py:1765-1866 with `scheduler` (set_timesteps already called) stepped by SolverRef over the
    run's `timesteps` (floats for Euler's linspace spacing). inp: the loop_ref.denoise_loop inputs, latents already
    multiplied by init_noise_sigma. noises: per step, DDIM's variance noise (eta > 0) or None."""
    ref = SolverRef(scheduler, kind, eta)
    latents = inp["latents"]
    for i, t in enumerate(timesteps):
        if max_steps is not None and i >= max_steps:
            break
        x_in = torch.cat([latents] * 2) * ref.scale(t)                                          # :1769, :1772
        x_in = torch.cat([x_in, inp["mask"], inp["masked_image_latents"], inp["pose_latents"]], dim=1)   # :1777
        tt = torch.as_tensor(float(t), dtype=torch.float32, device=latents.device)
        feats = R.unet_garment_forward(sd_g, cfg_g, inp["cloth_latents"], tt, inp["text_embeds_cloth"])  # :1787
        if feats[0].shape[0] != latents.shape[0]:
            feats = [f.expand(latents.shape[0], -1, -1) for f in feats]
        feats = [torch.cat([torch.zeros_like(d), d]) for d in feats]
        added = {"text_embeds": inp["add_text_embeds"], "time_ids": inp["add_time_ids"], "image_embeds": inp["image_embeds"]}
        noise_pred = R.unet_tryon_forward(sd_t, cfg_t, x_in, tt, inp["prompt_embeds"], added, feats)
        u, c = noise_pred.chunk(2)
        eps = u + guidance_scale * (c - u)                                                       # :1815-1816
        latents = ref.step(eps, t, latents, None if noises is None else noises[i])              # :1823
    return latents
