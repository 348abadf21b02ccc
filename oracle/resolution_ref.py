"""ORACLE (test infrastructure, not product): the two UNets and the denoising loop of oracle/unet_ref.py and
oracle/loop_ref.py at ANY latent size, with the garment at a size of its own.

Only tests/, __graft_entry__.smoke() and scripts may import this module.

What it adds to unet_ref (which it reuses for every leaf op and block):
  * `upsample_size` (src/unet_hacked_tryon.py:1081-1091,1357-1379; src/unet_hacked_garmnet.py:994-1000,1264-1274): when
    either dimension of a UNet's own input is not a multiple of 2^num_upsamplers, every non-final up block's Upsample2D
    runs F.interpolate(size=<H,W of the next skip>, mode="nearest") instead of scale 2 (diffusers 0.25 Upsample2D);
  * the garment UNet decides this from the cloth latents, the try-on UNet from the person latents; the try-on attention
    concatenates the garment's Ng tokens whatever N is (src/attentionhacked_tryon.py:334).
At sizes that are multiples of 2^num_upsamplers these functions compute exactly what unet_ref / loop_ref compute.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from . import loop_ref as LR
from . import unet_ref as R


def nearest_index(d, n_in, n_out):
    """Source index of output index d of ATen's `nearest` interpolation to a given size (aten/src/ATen/native/UpSample.h
    nearest_idx; the CUDA kernel uses the general branch, which gives the same indices): identity when the size is
    kept, d >> 1 when it doubles, otherwise min(floor(d * float32(n_in / n_out)), n_in - 1) in float32."""
    if n_out == n_in:
        return d
    if n_out == 2 * n_in:
        return d >> 1
    scale = np.float32(n_in) / np.float32(n_out)
    return min(int(math.floor(np.float32(d) * scale)), n_in - 1)


def upsample(sd, p, x, size=None):
    """diffusers Upsample2D: nearest x2 or, with `size` (the forwarded upsample_size), nearest to that size; then conv3x3."""
    if size is None:
        x = F.interpolate(x, scale_factor=2.0, mode="nearest")
    else:
        x = F.interpolate(x, size=tuple(size), mode="nearest")
    return F.conv2d(x, sd[f"{p}.conv.weight"], sd[f"{p}.conv.bias"], padding=1)


def forwards_upsample_size(cfg, sample):
    """src/unet_hacked_tryon.py:1081-1091: any latent dimension not a multiple of 2^num_upsamplers."""
    div = 2 ** (len(cfg["block_out_channels"]) - 1)
    return any(d % div for d in sample.shape[-2:])


def _trunk(sd, cfg, sample, emb, enc, garment_features, collect, stop_after_up):
    """unet_ref._trunk with the reference's upsample_size rule."""
    ch = cfg["block_out_channels"]
    tl = cfg["transformer_layers_per_block"]
    nh = cfg["num_heads"]
    ip = cfg["ip_tokens"]
    ips = cfg.get("ip_scale", 1.0)
    sized = forwards_upsample_size(cfg, sample)
    idx = 0
    x = F.conv2d(sample, sd["conv_in.weight"], sd["conv_in.bias"], padding=1)
    skips = [x]
    for i in range(len(ch)):
        for j in range(cfg["layers_per_block"]):
            x = R.resnet_block(sd, f"down_blocks.{i}.resnets.{j}", x, emb)
            if i > 0:
                x, idx = R.transformer_2d(sd, f"down_blocks.{i}.attentions.{j}", x, enc, nh[i], tl[i], ip,
                                          garment_features, idx, collect, ips)
            skips.append(x)
        if i < len(ch) - 1:
            x = R.downsample(sd, f"down_blocks.{i}.downsamplers.0", x)
            skips.append(x)
    x = R.resnet_block(sd, "mid_block.resnets.0", x, emb)
    x, idx = R.transformer_2d(sd, "mid_block.attentions.0", x, enc, nh[-1], tl[-1], ip, garment_features, idx, collect,
                              ips)
    x = R.resnet_block(sd, "mid_block.resnets.1", x, emb)
    rnh, rtl = list(reversed(nh)), list(reversed(tl))
    for i in range(len(ch)):
        if i >= stop_after_up:
            break
        for j in range(cfg["layers_per_block"] + 1):
            x = torch.cat([x, skips.pop()], dim=1)
            x = R.resnet_block(sd, f"up_blocks.{i}.resnets.{j}", x, emb)
            if i < len(ch) - 1:
                x, idx = R.transformer_2d(sd, f"up_blocks.{i}.attentions.{j}", x, enc, rnh[i], rtl[i], ip,
                                          garment_features, idx, collect, ips)
        if i < len(ch) - 1:
            x = upsample(sd, f"up_blocks.{i}.upsamplers.0", x, skips[-1].shape[2:] if sized else None)
    return x


def unet_tryon_forward(sd, cfg, sample, timestep, encoder_hidden_states, added_cond_kwargs, garment_features):
    """unet_ref.unet_tryon_forward at any latent size."""
    emb = R._time_embed(sd, cfg, sample, timestep, added_cond_kwargs)
    enc = torch.cat([encoder_hidden_states, added_cond_kwargs["image_embeds"]], dim=1)
    x = _trunk(sd, cfg, sample, emb, enc, garment_features, None, stop_after_up=len(cfg["block_out_channels"]))
    x = F.group_norm(x, 32, sd["conv_norm_out.weight"], sd["conv_norm_out.bias"], 1e-5)
    x = F.silu(x)
    return F.conv2d(x, sd["conv_out.weight"], sd["conv_out.bias"], padding=1)


def unet_garment_forward(sd, cfg, sample, timestep, encoder_hidden_states):
    """unet_ref.unet_garment_forward at any latent size (the cloth's own)."""
    emb = R._time_embed(sd, cfg, sample, timestep, None)
    feats = []
    _trunk(sd, cfg, sample, emb, encoder_hidden_states, None, feats, stop_after_up=len(cfg["block_out_channels"]) - 1)
    return feats


def denoise_loop(sd_t, cfg_t, sd_g, cfg_g, inp, num_steps, guidance_scale=2.0, scheduler=None, noises=None,
                 max_steps=None):
    """loop_ref.denoise_loop (src/tryon_pipeline.py:1765-1823) with both UNets at their own input sizes:
    cloth_latents [Bg,4,hg,wg] may differ in size from latents [B,4,h,w]."""
    sch = scheduler or LR.DDPMRef()
    timesteps = sch.set_timesteps(num_steps)
    latents = inp["latents"]
    for i, t in enumerate(timesteps):
        if max_steps is not None and i >= max_steps:
            break
        latent_model_input = torch.cat([latents] * 2)                                            # :1769
        latent_model_input = torch.cat([latent_model_input, inp["mask"], inp["masked_image_latents"],
                                        inp["pose_latents"]], dim=1)                             # :1777
        tt = torch.as_tensor(int(t), device=latents.device)
        feats = unet_garment_forward(sd_g, cfg_g, inp["cloth_latents"], tt, inp["text_embeds_cloth"])  # :1787
        if feats[0].shape[0] != latents.shape[0]:
            feats = [f.expand(latents.shape[0], -1, -1) for f in feats]
        feats = [torch.cat([torch.zeros_like(d), d]) for d in feats]                              # :1796
        added = {"text_embeds": inp["add_text_embeds"], "time_ids": inp["add_time_ids"],
                 "image_embeds": inp["image_embeds"]}
        noise_pred = unet_tryon_forward(sd_t, cfg_t, latent_model_input, tt, inp["prompt_embeds"], added, feats)
        u, c = noise_pred.chunk(2)
        noise_pred = u + guidance_scale * (c - u)                                                 # :1815-1816
        latents = sch.step(noise_pred, t, latents, noise=None if noises is None else noises[i])   # :1823
    return latents
