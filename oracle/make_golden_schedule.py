"""Golden vectors of the REFERENCE pipeline `StableDiffusionXLInpaintPipeline.__call__` (src/tryon_pipeline.py) with its
denoising-schedule arguments: strength, custom timesteps, denoising_start / denoising_end and guidance_rescale.

Same components, inputs and seeds as oracle/make_golden_pipeline.py (CPU fp32, 256x256 px, B=1, guidance 2.0, generator
seed 42, global seed 1234), with num_inference_steps=4 and, per case, the arguments in CASES. For every case this records
what the reference hands to its loop, the variance noise of every step, the latents after every step and the timesteps
it runs, and asserts that oracle/schedule_ref.denoise_loop reproduces the reference loop on those tensors. What this pins:
get_timesteps (:987-1020), retrieve_timesteps with a custom list (:265-300), the prepare_latents branches (:850-909:
image encoded before the noise is drawn, add_noise at the first timestep, add_noise=False under denoising_start), the
denoising_end truncation (:1732-1752), the denoising_start quirk of :1558-1566 and rescale_noise_cfg (:101-113,1818-1820).

To keep the file small (about 0.4 MB) it stores what depends on the schedule and nothing that can be recomputed: the
prompt and garment-text embeddings the loop receives are the call inputs themselves (checked here) and are rebuilt by
loop_inputs(); the VAE samples of the masked image, pose and garment are stored once (their posterior std is e^-15, so
every case draws them equal to 1e-6, checked here); per case the timesteps, the initial and the final latents, and the
step noises for the cases in REPLAY_CASES, on which tests/test_schedule_cpu.py replays the oracle loop.

Usage:  IDM_VTON_REFERENCE=<checkout of the original project> python oracle/make_golden_schedule.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STEPS = 4
OUT = os.path.join(ROOT, "tests", "golden", "pipeline_schedule_ref.pt")

# name -> keyword arguments on top of make_golden_pipeline.call_kwargs (whose strength=1.0 is dropped: "default" leaves
# strength at the signature's 0.9999)
CASES = {
    "default": dict(),
    "strength_rescale": dict(strength=0.5, guidance_rescale=0.7),
    "custom_timesteps": dict(strength=1.0, timesteps=[901, 601, 301, 1]),
    "denoising_end": dict(strength=1.0, denoising_end=0.5),
    "start_end": dict(denoising_start=0.25, denoising_end=0.75),
    "start_only": dict(denoising_start=0.5),
}
REPLAY_CASES = ("strength_rescale", "custom_timesteps")
SHARED = ("mask", "add_text_embeds", "add_time_ids", "image_embeds", "masked_image_latents", "pose_latents", "cloth_latents")


def case_kwargs(MG, inp, generator, name):
    kw = MG.call_kwargs(inp, generator)
    kw.pop("strength")
    kw.update(CASES[name])
    if "timesteps" in kw:
        kw["num_inference_steps"] = None
    else:
        kw["num_inference_steps"] = STEPS
    return kw


def oracle_schedule(name, run_timesteps):
    """(num_steps, timesteps) arguments of schedule_ref.denoise_loop for the schedule a case runs."""
    if "timesteps" in CASES[name]:
        return None, CASES[name]["timesteps"]
    return STEPS, run_timesteps


def loop_inputs(golden, name, call_inputs):
    """The tensors the reference handed to its loop in case `name` (schedule_ref.denoise_loop's `inp`), from the golden
    and make_golden_pipeline.make_call_inputs() (CPU fp32)."""
    d = {k: v.clone() for k, v in golden["shared"].items()}
    d["prompt_embeds"] = torch.cat([call_inputs["negative_prompt_embeds"], call_inputs["prompt_embeds"]])
    d["text_embeds_cloth"] = call_inputs["text_embeds_cloth"].clone()
    d["latents"] = golden["cases"][name]["latents"].clone()
    return d


def main():
    sys.path.insert(0, os.path.join(ROOT, "oracle", "shim"))
    sys.path.insert(0, os.environ.get("IDM_VTON_REFERENCE", ""))
    sys.path.insert(0, ROOT)
    import idm_vton_b200  # noqa: F401
    from oracle import unet_ref as R
    from oracle import schedule_ref as SR
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
    pipe = tp.StableDiffusionXLInpaintPipeline(
        vae=MG.make_vae(), text_encoder=None, text_encoder_2=None, tokenizer=None, tokenizer_2=None, unet=unet,
        unet_encoder=unet_enc, scheduler=sch, image_encoder=MG.make_image_encoder(cfg_t["resampler"]["embedding_dim"]))
    inp = MG.make_call_inputs(cfg_t)
    B = inp["image"].shape[0]
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

    shared, cases = None, {}
    for name in CASES:
        rec.clear()
        rec.update(noises=[], latents=[], timesteps=[])
        torch.manual_seed(1234)                      # the pose draw uses the global RNG (:1646)
        with torch.no_grad():
            pipe(**case_kwargs(MG, inp, torch.Generator().manual_seed(42), name), output_type="pt",
                 callback_on_step_end=on_step_end)
        x13 = rec["x13"]
        loop_in = dict(latents=x13[B:, :4], mask=x13[:, 4:5], masked_image_latents=x13[:, 5:9], pose_latents=x13[:, 9:13],
                       cloth_latents=rec["cloth_latents"], prompt_embeds=rec["prompt_embeds"],
                       add_text_embeds=rec["added"]["text_embeds"], add_time_ids=rec["added"]["time_ids"],
                       image_embeds=rec["added"]["image_embeds"], text_embeds_cloth=inp["text_embeds_cloth"])
        num_steps, ts = oracle_schedule(name, rec["timesteps"])
        with torch.no_grad():
            lat_oracle = SR.denoise_loop(sd_t, cfg_t, sd_g, cfg_g, loop_in, num_steps, guidance_scale=MG.GUIDANCE,
                                         noises=rec["noises"], timesteps=ts,
                                         guidance_rescale=CASES[name].get("guidance_rescale", 0.0))
        d = (lat_oracle - rec["latents"][-1]).abs().max().item()
        print(f"{name}: timesteps {rec['timesteps']} | schedule_ref.denoise_loop vs reference loop: max|d| = {d:.3e}")
        assert d < 1e-4 * max(1.0, rec["latents"][-1].abs().max().item())
        if shared is None:
            shared = {k: loop_in[k].clone() for k in SHARED}
        assert all(torch.allclose(loop_in[k], shared[k], rtol=0, atol=1e-6) for k in SHARED)
        cases[name] = {
            "kwargs": CASES[name], "timesteps": torch.tensor(rec["timesteps"]), "latents": loop_in["latents"].clone(),
            "final_latents": rec["latents"][-1].clone(),
            "noises": [None if n is None else n.clone() for n in rec["noises"]] if name in REPLAY_CASES else None,
        }
        rebuilt = loop_inputs({"shared": shared, "cases": cases}, name, inp)
        assert all(torch.equal(rebuilt[k], loop_in[k]) for k in ("prompt_embeds", "text_embeds_cloth", "latents"))
    torch.save({
        "note": "REFERENCE StableDiffusionXLInpaintPipeline.__call__ (src/tryon_pipeline.py) on the diffusers shim, CPU fp32, "
                f"256x256 px, num_inference_steps={STEPS}, B=1, guidance 2.0, generator seed 42, global seed 1234, per case "
                "the keyword arguments in 'kwargs'; components and inputs from oracle/make_golden_pipeline.py; "
                "make_golden_schedule.loop_inputs() rebuilds each case's loop inputs",
        "steps": STEPS, "shared": shared, "cases": cases,
    }, OUT)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
