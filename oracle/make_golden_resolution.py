"""Golden vectors of the REFERENCE pipeline `StableDiffusionXLInpaintPipeline.__call__` (src/tryon_pipeline.py) at image
sizes that are multiples of 8 but not of 32, and with the garment at a size of its own.

Same components, seeds and 2-step schedule as oracle/make_golden_pipeline.py (config 1: CPU fp32, B=1, guidance 2.0,
generator seed 42, global seed 1234); per case the person images (image, mask, pose) are H x W and the cloth image is
Hc x Wc (CASES). What this pins: the reference's `upsample_size` path (src/unet_hacked_tryon.py:1081-1091,1357-1379 and
src/unet_hacked_garmnet.py:994-1000,1264-1274) in both UNets, the garment UNet run at the cloth's own latent size
(:1654,1787) and the try-on attention over Ng != N garment tokens (src/attentionhacked_tryon.py:334). For every case it
asserts that oracle/resolution_ref.denoise_loop reproduces the reference loop on the tensors the reference handed to it.

To keep the file small (about 0.6 MB) it stores only what cannot be recomputed: per case the latents, mask, masked-image
and pose latents of the conditional half (the uncond half is the same tensor, :1769,1796), the cloth latents, the
Resampler output, the time ids, the step noises, the latents after every step and the timesteps. The prompt, pooled and
garment-text embeddings are the call inputs (rebuilt by loop_inputs(), checked here), and the images are the VAE decode of
the final latents (rebuilt by decode_images(), checked here).

Usage:  IDM_VTON_REFERENCE=<checkout of the original project> python oracle/make_golden_resolution.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "pipeline_resolution_ref.pt")

# name -> ((person H, W), (cloth H, W)) in pixels
CASES = {
    "odd_both": ((264, 200), (264, 200)),          # latents 33x25 -> 17x13 -> 9x7: both UNets forward upsample_size
    "even_not_x4": ((240, 176), (240, 176)),       # 30x22 -> 15x11 -> 8x6: upsample 8 -> 15 and 6 -> 11
    "cloth_larger": ((256, 192), (264, 200)),      # Ng > N; only the garment UNet forwards upsample_size
    "cloth_smaller": ((264, 200), (192, 144)),     # Ng < N; 24x18 -> 12x9 -> 6x5: garment forwards upsample_size too
}
STORED = ("latents", "mask", "masked_image_latents", "pose_latents", "cloth_latents", "image_embeds", "add_time_ids")


def make_case_inputs(cfg_t, name, B=1, seed=33):
    """make_golden_pipeline.make_call_inputs with the person images at the case's H x W and the cloth at Hc x Wc."""
    (H, W), (Hc, Wc) = CASES[name]
    g = torch.Generator().manual_seed(seed)
    cross = cfg_t["cross_attention_dim"]
    pooled = cfg_t["projection_class_embeddings_input_dim"] - 6 * cfg_t["addition_time_embed_dim"]
    r = lambda *s: torch.randn(*s, generator=g).half().float()  # noqa: E731
    mask = torch.zeros(B, 1, H, W)
    mask[:, :, H // 4: 3 * H // 4, W // 8: 5 * W // 8] = 1.0
    return dict(
        image=torch.rand(B, 3, H, W, generator=g).half().float(), mask_image=mask,
        pose_img=(torch.rand(B, 3, H, W, generator=g) * 2 - 1).half().float(),
        cloth=(torch.rand(B, 3, Hc, Wc, generator=g) * 2 - 1).half().float(),
        ip_adapter_image=r(B, 3, 224, 224),
        prompt_embeds=r(B, 77, cross), negative_prompt_embeds=r(B, 77, cross),
        pooled_prompt_embeds=r(B, pooled), negative_pooled_prompt_embeds=r(B, pooled),
        text_embeds_cloth=r(B, 77, cross),
    )


def call_kwargs(MG, inp, generator, name):
    """make_golden_pipeline.call_kwargs (the keyword set of inference.py:397-414) at the case's size."""
    kw = MG.call_kwargs(inp, generator)
    kw["height"], kw["width"] = CASES[name][0]
    return kw


def loop_inputs(case, call_inputs):
    """The tensors the reference handed to its loop (resolution_ref.denoise_loop's `inp`) from a golden case and
    make_case_inputs() (CPU fp32)."""
    s = case["stored"]
    dup = lambda t: torch.cat([t, t])  # noqa: E731
    return dict(
        latents=s["latents"].clone(), mask=dup(s["mask"]), masked_image_latents=dup(s["masked_image_latents"]),
        pose_latents=dup(s["pose_latents"]), cloth_latents=s["cloth_latents"].clone(),
        prompt_embeds=torch.cat([call_inputs["negative_prompt_embeds"], call_inputs["prompt_embeds"]]),
        add_text_embeds=torch.cat([call_inputs["negative_pooled_prompt_embeds"], call_inputs["pooled_prompt_embeds"]]),
        add_time_ids=s["add_time_ids"].clone(), image_embeds=s["image_embeds"].clone(),
        text_embeds_cloth=call_inputs["text_embeds_cloth"].clone())


def decode_images(vae, latents):
    """The reference's output_type="pt" images from its final latents: vae.decode(latents / scaling_factor), then
    VaeImageProcessor.postprocess (denormalize, clamp to [0, 1])."""
    with torch.no_grad():
        x = vae.decode(latents / vae.config.scaling_factor, return_dict=False)[0]
    return (x / 2 + 0.5).clamp(0, 1)


def main():
    sys.path.insert(0, os.path.join(ROOT, "oracle", "shim"))
    sys.path.insert(0, os.environ.get("IDM_VTON_REFERENCE", ""))
    sys.path.insert(0, ROOT)
    import idm_vton_b200  # noqa: F401
    from oracle import unet_ref as R
    from oracle import resolution_ref as RR
    from oracle import make_golden_pipeline as MG
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
    vae = MG.make_vae()
    pipe = tp.StableDiffusionXLInpaintPipeline(
        vae=vae, text_encoder=None, text_encoder_2=None, tokenizer=None, tokenizer_2=None, unet=unet,
        unet_encoder=unet_enc, scheduler=sch, image_encoder=MG.make_image_encoder(cfg_t["resampler"]["embedding_dim"]))
    orig_unet_forward, orig_enc_forward, orig_step = unet.forward, unet_enc.forward, sch.step
    rec = {}

    def unet_forward(sample, t, **kw):
        if "x13" not in rec:
            rec.update(x13=sample.clone(), prompt_embeds=kw["encoder_hidden_states"].clone(),
                       added={k: v.clone() for k, v in kw["added_cond_kwargs"].items()})
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
        rec["timesteps"].append(int(t))
        rec["latents"].append(kw["latents"].clone())
        return {}

    cases = {}
    for name, ((H, W), (Hc, Wc)) in CASES.items():
        rec.clear()
        rec.update(noises=[], latents=[], timesteps=[])
        inp = make_case_inputs(cfg_t, name)
        B = inp["image"].shape[0]
        torch.manual_seed(1234)                      # the pose draw uses the global RNG (:1646)
        with torch.no_grad():
            images = pipe(**call_kwargs(MG, inp, torch.Generator().manual_seed(42), name), output_type="pt",
                          callback_on_step_end=on_step_end)[0]
        x13 = rec["x13"]
        assert x13.shape == (2 * B, 13, H // 8, W // 8) and rec["cloth_latents"].shape[-2:] == (Hc // 8, Wc // 8)
        assert torch.equal(x13[:B], x13[B:])          # [latents]*2 and the duplicated conditioning
        loop_in = dict(latents=x13[B:, :4], mask=x13[:, 4:5], masked_image_latents=x13[:, 5:9], pose_latents=x13[:, 9:13],
                       cloth_latents=rec["cloth_latents"], prompt_embeds=rec["prompt_embeds"],
                       add_text_embeds=rec["added"]["text_embeds"], add_time_ids=rec["added"]["time_ids"],
                       image_embeds=rec["added"]["image_embeds"], text_embeds_cloth=inp["text_embeds_cloth"])
        with torch.no_grad():
            lat_oracle = RR.denoise_loop(sd_t, cfg_t, sd_g, cfg_g, loop_in, MG.STEPS, guidance_scale=MG.GUIDANCE,
                                         noises=rec["noises"])
        d = (lat_oracle - rec["latents"][-1]).abs().max().item()
        print(f"{name}: person {H}x{W} cloth {Hc}x{Wc} | timesteps {rec['timesteps']} | resolution_ref.denoise_loop vs "
              f"reference loop: max|d| = {d:.3e}")
        assert d < 1e-4 * max(1.0, rec["latents"][-1].abs().max().item())
        stored = {k: (loop_in[k][B:] if k in ("mask", "masked_image_latents", "pose_latents") else loop_in[k]).clone()
                  for k in STORED}
        case = {"person": (H, W), "cloth": (Hc, Wc), "timesteps": torch.tensor(rec["timesteps"]), "stored": stored,
                "noises": [None if n is None else n.clone() for n in rec["noises"]],
                "latents_per_step": [l.clone() for l in rec["latents"]]}
        rebuilt = loop_inputs(case, inp)
        assert all(torch.equal(rebuilt[k], loop_in[k]) for k in loop_in), "loop_inputs() does not rebuild the loop inputs"
        d_img = (decode_images(vae, rec["latents"][-1]) - images).abs().max().item()
        assert d_img == 0.0, f"decode_images() differs from the reference's images by {d_img}"
        cases[name] = case
    torch.save({
        "note": "REFERENCE StableDiffusionXLInpaintPipeline.__call__ (src/tryon_pipeline.py) on the diffusers shim, CPU fp32, "
                f"num_inference_steps={MG.STEPS}, B=1, guidance 2.0, generator seed 42, global seed 1234; components from "
                "oracle/make_golden_pipeline.py, inputs from make_golden_resolution.make_case_inputs (person and cloth "
                "sizes per case); make_golden_resolution.loop_inputs() and decode_images() rebuild the rest",
        "steps": MG.STEPS, "cases": cases,
    }, OUT)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
