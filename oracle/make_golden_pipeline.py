"""Golden vectors of the REFERENCE pipeline `StableDiffusionXLInpaintPipeline.__call__` (src/tryon_pipeline.py:1254-1896)
at BASELINE config 1 (256x256 px, 2 denoise steps, batch 1, CPU fp32).

Needs a checkout of the original project (IDM_VTON_REFERENCE). `src/tryon_pipeline.py`, `src/unet_hacked_tryon.py`,
`src/unet_hacked_garmnet.py` and `ip_adapter/*.py` are imported UNMODIFIED and in place on the diffusers shim; the
components diffusers / the HF hub would supply (not available offline) are stand-ins with seeded weights:
  unet / unet_encoder   the reference's own UNet2DConditionModel classes, tiny SDXL-topology config (oracle.unet_ref.tiny_config)
  vae                   idm-vton_b200.vae.AutoencoderKL (small geometry), posterior log-variance forced to the clamp
                        minimum (std = e^-15) so that `latent_dist.sample()` on the GLOBAL RNG (the pose image,
                        src/tryon_pipeline.py:1646) is reproducible across devices; every draw still advances its generator
  image_encoder         transformers.CLIPVisionModelWithProjection, 2 layers, width 192
  scheduler             idm-vton_b200.scheduler.DDPMScheduler (restated diffusers DDPM; step() on the host)
What this pins for the product pipeline and for oracle/loop_ref.py: RNG draw order (:889, 964 via 911-932, 1646, 1654,
1823), the [latents | mask | masked-image | pose] channel order (:1777), [uncond ; cond] batch order (:1711-1714,
1769, 1796), mask preprocessing / nearest resize (:934-980), the CFG formula (:1815-1816), the timestep list, and that
the loop restated in loop_ref.denoise_loop reproduces the reference loop to fp32 round-off.

Usage:  python oracle/make_golden_pipeline.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("IDM_VTON_REFERENCE", "")   # checkout of the original IDM-VTON project
GOLDEN = os.path.join(ROOT, "tests", "golden")
H = W = 256
STEPS = 2
GUIDANCE = 2.0


def seeded_fill_(module, seed, gain=1.0):
    """Deterministic weights independent of any framework init routine: every parameter, in state-dict order, from one
    seeded CPU generator (matrices uniform +-sqrt(3/fan_in), vectors N(0, 0.05), norm scales 1 +- 0.1)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in module.state_dict().items():
            if not torch.is_floating_point(p):
                continue
            if p.ndim >= 2:
                fan_in = p[0].numel()
                w = (torch.rand(p.shape, generator=g) * 2 - 1) * (3.0 / fan_in) ** 0.5 * gain
            elif name.endswith("weight") and ("norm" in name.lower() or "ln" in name.lower()):
                w = 1.0 + 0.1 * torch.randn(p.shape, generator=g)
            else:
                w = 0.05 * torch.randn(p.shape, generator=g)
            p.copy_(w.half().float().to(p.dtype))
    return module


def make_vae():
    from idm_vton_b200.vae import AutoencoderKL
    vae = seeded_fill_(AutoencoderKL(block_out_channels=(32, 64, 64, 64)), seed=31).eval()
    with torch.no_grad():      # posterior log-variance = clamp minimum (see module docstring)
        vae.quant_conv.weight[4:].zero_()
        vae.quant_conv.bias[4:].fill_(-30.0)
    return vae


def make_image_encoder(width):
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection
    cfg = CLIPVisionConfig(hidden_size=width, intermediate_size=2 * width, num_hidden_layers=2, num_attention_heads=3,
                           patch_size=14, image_size=224, projection_dim=64)
    return seeded_fill_(CLIPVisionModelWithProjection(cfg), seed=32).eval()


def make_call_inputs(cfg_t, B=1, seed=33):
    g = torch.Generator().manual_seed(seed)
    cross = cfg_t["cross_attention_dim"]
    pooled = cfg_t["projection_class_embeddings_input_dim"] - 6 * cfg_t["addition_time_embed_dim"]
    r = lambda *s: torch.randn(*s, generator=g).half().float()  # noqa: E731
    mask = torch.zeros(B, 1, H, W)
    mask[:, :, H // 4: 3 * H // 4, W // 8: 5 * W // 8] = 1.0          # off-centre rectangle: catches x/y swaps
    return dict(
        image=torch.rand(B, 3, H, W, generator=g).half().float(), mask_image=mask,
        pose_img=(torch.rand(B, 3, H, W, generator=g) * 2 - 1).half().float(),
        cloth=(torch.rand(B, 3, H, W, generator=g) * 2 - 1).half().float(),
        ip_adapter_image=r(B, 3, 224, 224),
        prompt_embeds=r(B, 77, cross), negative_prompt_embeds=r(B, 77, cross),
        pooled_prompt_embeds=r(B, pooled), negative_pooled_prompt_embeds=r(B, pooled),
        text_embeds_cloth=r(B, 77, cross),
    )


def call_kwargs(inp, generator):
    """The keyword set of inference.py:397-414."""
    return dict(prompt_embeds=inp["prompt_embeds"], negative_prompt_embeds=inp["negative_prompt_embeds"],
                pooled_prompt_embeds=inp["pooled_prompt_embeds"],
                negative_pooled_prompt_embeds=inp["negative_pooled_prompt_embeds"], num_inference_steps=STEPS,
                generator=generator, strength=1.0, pose_img=inp["pose_img"], text_embeds_cloth=inp["text_embeds_cloth"],
                cloth=inp["cloth"], mask_image=inp["mask_image"], image=inp["image"], height=H, width=W,
                ip_adapter_image=inp["ip_adapter_image"], guidance_scale=GUIDANCE)


def main():
    sys.path.insert(0, os.path.join(ROOT, "oracle", "shim"))
    sys.path.insert(0, REF)
    sys.path.insert(0, ROOT)
    from oracle import unet_ref as R
    from oracle import loop_ref as LR
    from oracle.make_golden import build_reference_unet
    from idm_vton_b200.scheduler import DDPMScheduler
    import src.tryon_pipeline as tp
    import src.unet_hacked_garmnet as ug
    import src.unet_hacked_tryon as ut
    cfg_t, cfg_g = R.tiny_config("tryon"), R.tiny_config("garment")
    sd_t, sd_g = R.make_state_dict(cfg_t, seed=11), R.make_state_dict(cfg_g, seed=22)
    sd_t = {k: v.half().float() for k, v in sd_t.items()}
    sd_g = {k: v.half().float() for k, v in sd_g.items()}
    unet, unet_enc = build_reference_unet(ut, cfg_t), build_reference_unet(ug, cfg_g)
    unet.load_state_dict(sd_t, strict=True)
    unet_enc.load_state_dict(sd_g, strict=True)
    sch = DDPMScheduler()
    pipe = tp.StableDiffusionXLInpaintPipeline(
        vae=make_vae(), text_encoder=None, text_encoder_2=None, tokenizer=None, tokenizer_2=None, unet=unet,
        unet_encoder=unet_enc, scheduler=sch, image_encoder=make_image_encoder(cfg_t["resampler"]["embedding_dim"]))
    inp = make_call_inputs(cfg_t)

    # record what the reference hands to its UNets at step 0 and the variance noise of every step
    rec = {"noises": [], "latents": []}
    orig_unet_forward, orig_enc_forward, orig_step = unet.forward, unet_enc.forward, sch.step

    def unet_forward(sample, t, **kw):
        if "x13" not in rec:
            rec.update(x13=sample.clone(), prompt_embeds=kw["encoder_hidden_states"].clone(),
                       added={k: v.clone() for k, v in kw["added_cond_kwargs"].items()},
                       n_features=len(kw["garment_features"]))
        return orig_unet_forward(sample, t, **kw)

    def enc_forward(sample, t, text, **kw):
        rec.setdefault("cloth_latents", sample.clone())
        return orig_enc_forward(sample, t, text, **kw)

    def step(*a, **kw):
        out = orig_step(*a, **kw)
        rec["noises"].append(None if sch._last_noise is None else sch._last_noise.clone())
        return out

    unet.forward, unet_enc.forward, sch.step = unet_forward, enc_forward, step

    def on_step_end(p, i, t, kw):
        rec["latents"].append(kw["latents"].clone())
        return {}

    torch.manual_seed(1234)                          # the pose draw uses the global RNG (:1646)
    with torch.no_grad():
        images = pipe(**call_kwargs(inp, torch.Generator().manual_seed(42)), output_type="pt",
                      callback_on_step_end=on_step_end)[0]
    x13 = rec["x13"]
    B = inp["image"].shape[0]
    assert x13.shape == (2 * B, 13, H // 8, W // 8) and len(rec["latents"]) == STEPS
    assert torch.equal(x13[:B], x13[B:]) or not torch.equal(x13[:B, 4:], x13[B:, 4:])
    print("timesteps", sch.timesteps.tolist(), "| latents absmax per step", [float(l.abs().max()) for l in rec["latents"]],
          "| image range", float(images.min()), float(images.max()))

    # ---- pin oracle/loop_ref.py against the reference loop: same prepared tensors in, same latents out
    loop_in = dict(latents=x13[B:, :4], mask=x13[:, 4:5], masked_image_latents=x13[:, 5:9], pose_latents=x13[:, 9:13],
                   cloth_latents=rec["cloth_latents"], prompt_embeds=rec["prompt_embeds"],
                   add_text_embeds=rec["added"]["text_embeds"], add_time_ids=rec["added"]["time_ids"],
                   image_embeds=rec["added"]["image_embeds"], text_embeds_cloth=inp["text_embeds_cloth"])
    with torch.no_grad():
        lat_oracle = LR.denoise_loop(sd_t, cfg_t, sd_g, cfg_g, loop_in, STEPS, guidance_scale=GUIDANCE,
                                     noises=rec["noises"])
    d = (lat_oracle - rec["latents"][-1]).abs().max().item()
    print("loop_ref.denoise_loop vs reference loop: max|d| =", d)
    assert d < 1e-4 * max(1.0, rec["latents"][-1].abs().max().item())

    torch.save({
        "note": "REFERENCE StableDiffusionXLInpaintPipeline.__call__ (src/tryon_pipeline.py) on the diffusers shim, CPU fp32, "
                "config 1: 256x256 px, 2 steps, B=1, guidance 2.0, generator seed 42, global seed 1234; components and "
                "inputs from oracle/make_golden_pipeline.py (make_vae, make_image_encoder, make_call_inputs, tiny UNets "
                "seeds 11/22 rounded to fp16)",
        "timesteps": sch.timesteps.clone(), "images": images.half(),
        "latents_per_step": [l.clone() for l in rec["latents"]],
        "loop_inputs": {k: v.clone() for k, v in loop_in.items()},
        "noises": [None if n is None else n.clone() for n in rec["noises"]],
        "n_features": rec["n_features"],
    }, os.path.join(GOLDEN, "pipeline_call_ref.pt"))
    print("wrote", os.path.join(GOLDEN, "pipeline_call_ref.pt"))


if __name__ == "__main__":
    main()
