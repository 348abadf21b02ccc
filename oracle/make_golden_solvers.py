"""Golden vectors of the REFERENCE pipeline `StableDiffusionXLInpaintPipeline.__call__` (src/tryon_pipeline.py) driven by
DDIMScheduler, EulerDiscreteScheduler and DPMSolverMultistepScheduler (the restatements in idm_vton_b200/scheduler.py,
each built with `from_config` of the IDM-VTON DDPM config).

Same components, inputs and seeds as oracle/make_golden_schedule.py (CPU fp32, 256x256 px, B=1, guidance 2.0, generator
seed 42, global seed 1234), num_inference_steps=5, per case the scheduler and call arguments in CASES. What this pins is
how the reference's own loop drives a scheduler: `init_noise_sigma` (and `add_noise` with strength < 1), the timesteps
after get_timesteps, `scale_model_input` before the channel concat (:1772-1777), `eta` and `generator` passed to `step`
only when its signature takes them (:746-761). For every case it records the latents the loop starts from, the timesteps,
DDIM's variance noises at eta > 0 and the final latents, and asserts that oracle/solver_ref.denoise_loop (the papers'
update rules in float64 on the scheduler's own alphas / sigmas) reproduces the reference loop on those tensors.

The file keeps only what depends on the scheduler: the VAE samples of the masked image, pose and garment are stored once
(shared; loop_inputs() of make_golden_schedule rebuilds each case's loop inputs from them and the call inputs), and per
case the scheduler arguments, timesteps, initial and final latents and step noises.

Usage:  IDM_VTON_REFERENCE=<checkout of the original project> python oracle/make_golden_solvers.py
"""
import functools
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STEPS = 5
OUT = os.path.join(ROOT, "tests", "golden", "pipeline_solvers_ref.pt")

# name -> (scheduler class, from_config overrides, extra call keyword arguments)
CASES = {
    "ddim_eta0": ("DDIMScheduler", {}, dict(eta=0.0)),
    "ddim_eta1": ("DDIMScheduler", {}, dict(eta=1.0)),
    "euler_leading": ("EulerDiscreteScheduler", {}, {}),
    "euler_linspace": ("EulerDiscreteScheduler", dict(timestep_spacing="linspace"), {}),
    "dpmpp_2m": ("DPMSolverMultistepScheduler", {}, {}),
    "dpmpp_2m_karras": ("DPMSolverMultistepScheduler", dict(use_karras_sigmas=True), {}),
    "dpmpp_2m_strength": ("DPMSolverMultistepScheduler", {}, dict(strength=0.5)),
}
KIND = {"DDIMScheduler": "ddim", "EulerDiscreteScheduler": "euler", "DPMSolverMultistepScheduler": "dpmpp"}
DETERMINISTIC = ("ddim_eta0", "euler_leading", "euler_linspace", "dpmpp_2m", "dpmpp_2m_karras", "dpmpp_2m_strength")
SHARED = ("mask", "add_text_embeds", "add_time_ids", "image_embeds", "masked_image_latents", "pose_latents", "cloth_latents")


def make_scheduler(name):
    """A fresh restated scheduler of case `name`, from the IDM-VTON DDPM config."""
    from idm_vton_b200 import scheduler as S
    cls, over, _ = CASES[name]
    return getattr(S, cls).from_config(S.DDPMScheduler().config, **over)


def case_kwargs(MG, inp, generator, name):
    kw = MG.call_kwargs(inp, generator)              # strength 1.0 unless the case sets it
    kw.update(CASES[name][2], num_inference_steps=STEPS)
    return kw


def main():
    sys.path.insert(0, os.path.join(ROOT, "oracle", "shim"))
    sys.path.insert(0, os.environ.get("IDM_VTON_REFERENCE", ""))
    sys.path.insert(0, ROOT)
    import idm_vton_b200  # noqa: F401
    from oracle import unet_ref as R
    from oracle import solver_ref as SV
    from oracle import make_golden_pipeline as MG
    from oracle import make_golden_schedule as MS
    from oracle.make_golden import build_reference_unet
    import src.tryon_pipeline as tp
    import src.unet_hacked_garmnet as ug
    import src.unet_hacked_tryon as ut
    torch.use_deterministic_algorithms(True)
    cfg_t, cfg_g = R.tiny_config("tryon"), R.tiny_config("garment")
    sd_t = {k: v.half().float() for k, v in R.make_state_dict(cfg_t, seed=11).items()}
    sd_g = {k: v.half().float() for k, v in R.make_state_dict(cfg_g, seed=22).items()}
    unet, unet_enc = build_reference_unet(ut, cfg_t), build_reference_unet(ug, cfg_g)
    unet.load_state_dict(sd_t, strict=True)
    unet_enc.load_state_dict(sd_g, strict=True)
    inp = MG.make_call_inputs(cfg_t)
    B = inp["image"].shape[0]
    shared, cases = None, {}
    for name in CASES:
        sch = make_scheduler(name)
        pipe = tp.StableDiffusionXLInpaintPipeline(
            vae=MG.make_vae(), text_encoder=None, text_encoder_2=None, tokenizer=None, tokenizer_2=None, unet=unet,
            unet_encoder=unet_enc, scheduler=sch, image_encoder=MG.make_image_encoder(cfg_t["resampler"]["embedding_dim"]))
        rec = dict(noises=[], latents=[], timesteps=[])
        orig_unet, orig_enc, orig_step, orig_scale = unet.forward, unet_enc.forward, sch.step, sch.scale_model_input

        def unet_forward(sample, t, **kw):
            if "x13" not in rec:
                rec.update(x13=sample.clone(), prompt_embeds=kw["encoder_hidden_states"].clone(),
                           added={k: v.clone() for k, v in kw["added_cond_kwargs"].items()})
            return orig_unet(sample, t, **kw)

        def enc_forward(sample, t, text, **kw):
            rec.setdefault("cloth_latents", sample.clone())
            return orig_enc(sample, t, text, **kw)

        @functools.wraps(orig_scale)
        def scale_model_input(sample, t):
            rec.setdefault("latents0", sample[B:].clone())        # the loop's latents, before scaling
            return orig_scale(sample, t)

        @functools.wraps(orig_step)           # keeps step's signature: the reference introspects it for eta / generator
        def step(*a, **kw):
            rec.setdefault("step_kwargs", sorted(kw))
            out = orig_step(*a, **kw)
            rec["noises"].append(None if sch._last_noise is None else sch._last_noise.clone())
            return out

        def on_step_end(p, i, t, kw):
            rec["timesteps"].append(float(t))
            rec["latents"].append(kw["latents"].clone())
            return {}

        unet.forward, unet_enc.forward, sch.step, sch.scale_model_input = unet_forward, enc_forward, step, scale_model_input
        torch.manual_seed(1234)                     # the pose draw uses the global RNG (:1646)
        try:
            with torch.no_grad():
                pipe(**case_kwargs(MG, inp, torch.Generator().manual_seed(42), name), output_type="pt",
                     callback_on_step_end=on_step_end)
        finally:
            unet.forward, unet_enc.forward = orig_unet, orig_enc
        x13 = rec["x13"]
        loop_in = dict(latents=rec["latents0"], mask=x13[:, 4:5], masked_image_latents=x13[:, 5:9],
                       pose_latents=x13[:, 9:13], cloth_latents=rec["cloth_latents"], prompt_embeds=rec["prompt_embeds"],
                       add_text_embeds=rec["added"]["text_embeds"], add_time_ids=rec["added"]["time_ids"],
                       image_embeds=rec["added"]["image_embeds"], text_embeds_cloth=inp["text_embeds_cloth"])
        eta = CASES[name][2].get("eta", 0.0)
        noises = rec["noises"] if name == "ddim_eta1" else None
        ref_sch = make_scheduler(name)
        ref_sch.set_timesteps(STEPS)
        with torch.no_grad():
            lat_oracle = SV.denoise_loop(sd_t, cfg_t, sd_g, cfg_g, loop_in, ref_sch, KIND[CASES[name][0]],
                                         torch.tensor(rec["timesteps"]), guidance_scale=MG.GUIDANCE, eta=eta,
                                         noises=noises)
        d = (lat_oracle - rec["latents"][-1]).abs().max().item()
        print(f"{name}: timesteps {rec['timesteps']} step kwargs {rec['step_kwargs']} | solver_ref.denoise_loop vs "
              f"reference loop: max|d| = {d:.3e}")
        assert d < 1e-4 * max(1.0, rec["latents"][-1].abs().max().item())
        if shared is None:
            shared = {k: loop_in[k].clone() for k in SHARED}
        assert all(torch.allclose(loop_in[k], shared[k], rtol=0, atol=1e-6) for k in SHARED)
        cases[name] = {
            "scheduler": CASES[name][0], "config": CASES[name][1], "kwargs": CASES[name][2],
            "timesteps": torch.tensor(rec["timesteps"], dtype=torch.float64), "latents": loop_in["latents"].clone(),
            "final_latents": rec["latents"][-1].clone(),
            "noises": [n.clone() for n in rec["noises"]] if name == "ddim_eta1" else None,
        }
        rebuilt = MS.loop_inputs({"shared": shared, "cases": cases}, name, inp)
        assert all(torch.equal(rebuilt[k], loop_in[k]) for k in ("prompt_embeds", "text_embeds_cloth", "latents"))
    torch.save({
        "note": "REFERENCE StableDiffusionXLInpaintPipeline.__call__ (src/tryon_pipeline.py) on the diffusers shim, CPU fp32, "
                f"256x256 px, num_inference_steps={STEPS}, B=1, guidance 2.0, generator seed 42, global seed 1234, per case "
                "the restated scheduler (from_config of the DDPM config with 'config') and the keyword arguments in "
                "'kwargs'; components and inputs from oracle/make_golden_pipeline.py; make_golden_schedule.loop_inputs() "
                "rebuilds each case's loop inputs",
        "steps": STEPS, "shared": shared, "cases": cases,
    }, OUT)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
