"""ORACLE (test infrastructure, not product): the denoising loop of src/tryon_pipeline.py:1765-1866 with the schedule
arguments of the reference `__call__` — a part of the spaced schedule (strength, denoising_start / denoising_end), a custom
timestep list (diffusers==0.25.0 DDPMScheduler.set_timesteps(timesteps=...) / previous_timestep) and guidance rescale
(rescale_noise_cfg, :101-113, applied at :1818-1820). Built on oracle/loop_ref.py, whose defaults it reproduces.

Only tests/ and oracle/make_golden_schedule.py import this module.
"""
import torch

from . import loop_ref as LR
from . import unet_ref as R


class DDPMScheduleRef(LR.DDPMRef):
    """DDPMRef that also takes a custom descending timestep list: each custom timestep steps to the next one, the last
    to -1 (diffusers DDPMScheduler.previous_timestep with custom_timesteps)."""

    custom = None

    def set_timesteps(self, num_inference_steps=None, timesteps=None):
        if timesteps is None:
            self.custom = None
            return super().set_timesteps(num_inference_steps)
        self.custom = [int(t) for t in timesteps]
        self.timesteps = torch.tensor(self.custom)
        return self.timesteps

    def step(self, model_output, t, sample, generator=None, noise=None):
        if self.custom is None:
            return super().step(model_output, t, sample, generator=generator, noise=noise)
        i = self.custom.index(int(t))
        # the parent's step derives prev_t from an even spacing, which a custom list does not have
        return _ddpm_step(self, model_output, int(t), self.custom[i + 1] if i + 1 < len(self.custom) else -1, sample,
                          generator, noise)


def _ddpm_step(sch, model_output, t, prev_t, sample, generator, noise):
    """loop_ref.DDPMRef.step with an explicit previous timestep."""
    alpha_prod_t = sch.alphas_cumprod[t]
    alpha_prod_t_prev = sch.alphas_cumprod[prev_t] if prev_t >= 0 else sch.one
    beta_prod_t = 1 - alpha_prod_t
    beta_prod_t_prev = 1 - alpha_prod_t_prev
    current_alpha_t = alpha_prod_t / alpha_prod_t_prev
    current_beta_t = 1 - current_alpha_t
    pred_original_sample = (sample - beta_prod_t ** 0.5 * model_output) / alpha_prod_t ** 0.5
    pred_original_sample_coeff = (alpha_prod_t_prev ** 0.5 * current_beta_t) / beta_prod_t
    current_sample_coeff = current_alpha_t ** 0.5 * beta_prod_t_prev / beta_prod_t
    pred_prev_sample = pred_original_sample_coeff * pred_original_sample + current_sample_coeff * sample
    variance = 0
    if t > 0:
        if noise is None:
            noise = torch.randn(model_output.shape, generator=generator, device=model_output.device,
                                dtype=model_output.dtype)
        var = torch.clamp((1 - alpha_prod_t_prev) / (1 - alpha_prod_t) * current_beta_t, min=1e-20)
        variance = (var ** 0.5) * noise
    return pred_prev_sample + variance


def rescale_noise_cfg(noise_cfg, noise_pred_text, guidance_rescale):
    """src/tryon_pipeline.py:101-113: blend of the CFG result and the CFG result rescaled to the cond prediction's
    per-sample std (unbiased, over C*H*W), in the dtype of the inputs."""
    std_text = noise_pred_text.std(dim=list(range(1, noise_pred_text.ndim)), keepdim=True)
    std_cfg = noise_cfg.std(dim=list(range(1, noise_cfg.ndim)), keepdim=True)
    noise_pred_rescaled = noise_cfg * (std_text / std_cfg)
    return guidance_rescale * noise_pred_rescaled + (1 - guidance_rescale) * noise_cfg


def denoise_loop(sd_t, cfg_t, sd_g, cfg_g, inp, num_steps, guidance_scale=2.0, noises=None, max_steps=None,
                 timesteps=None, guidance_rescale=0.0):
    """loop_ref.denoise_loop with the schedule arguments. timesteps: the timesteps to run. With num_steps set they are a
    part of the num_steps-step schedule (each steps to t - T_train // num_steps); with num_steps=None they are a custom
    schedule. guidance_rescale: rescale_noise_cfg after CFG when > 0. inp / noises as in loop_ref.denoise_loop."""
    sch = DDPMScheduleRef()
    if num_steps is None:
        timesteps = sch.set_timesteps(timesteps=timesteps)
    else:
        full = sch.set_timesteps(num_steps)
        timesteps = full if timesteps is None else torch.as_tensor(timesteps)
    latents = inp["latents"]
    for i, t in enumerate(timesteps):
        if max_steps is not None and i >= max_steps:
            break
        latent_model_input = torch.cat([latents] * 2)                                            # :1769
        latent_model_input = torch.cat([latent_model_input, inp["mask"], inp["masked_image_latents"],
                                        inp["pose_latents"]], dim=1)                             # :1777
        tt = torch.as_tensor(int(t), device=latents.device)
        feats = R.unet_garment_forward(sd_g, cfg_g, inp["cloth_latents"], tt, inp["text_embeds_cloth"])  # :1787
        if feats[0].shape[0] != latents.shape[0]:
            feats = [f.expand(latents.shape[0], -1, -1) for f in feats]
        feats = [torch.cat([torch.zeros_like(d), d]) for d in feats]                              # :1796
        added = {"text_embeds": inp["add_text_embeds"], "time_ids": inp["add_time_ids"],
                 "image_embeds": inp["image_embeds"]}
        noise_pred = R.unet_tryon_forward(sd_t, cfg_t, latent_model_input, tt, inp["prompt_embeds"], added, feats)
        u, c = noise_pred.chunk(2)
        noise_pred = u + guidance_scale * (c - u)                                                 # :1815-1816
        if guidance_rescale > 0.0:
            noise_pred = rescale_noise_cfg(noise_pred, c, guidance_rescale)                       # :1818-1820
        latents = sch.step(noise_pred, t, latents, noise=None if noises is None else noises[i])   # :1823
    return latents
