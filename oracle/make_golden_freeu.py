"""Golden vectors of FreeU on the REFERENCE's own modules: its tiny try-on UNet and its pipeline at config 1, with
`enable_freeu`, and the signatures of the reference's `enable_freeu` / `disable_freeu`. Writes tests/golden/freeu_ref.pt.

Needs a checkout of the original project (IDM_VTON_REFERENCE). The reference's up blocks call diffusers'
`apply_freeu`, which the test-only shim leaves unimplemented; oracle/freeu_ref.apply_freeu (diffusers 0.25.0 restated,
FFT form) is installed in the shim before the reference is imported. Everything else is oracle/make_golden.py's and
oracle/make_golden_pipeline.py's set-up: same seeded weights, inputs, components and seeds.

Cases: the SDXL values (b1 1.3, b2 1.4, s1 0.9, s2 0.2), a set that differs between the stages, and s1 = 0, which the
reference's truthiness rule turns into FreeU off. The UNet runs at latent 24 x 16, so its FreeU stages (6 x 4 and
12 x 8) are not powers of two and take the fp32 branch of `fourier_filter`.

Usage:  python oracle/make_golden_freeu.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
CASES = {
    "sdxl": dict(s1=0.9, s2=0.2, b1=1.3, b2=1.4),
    "asym": dict(s1=0.3, s2=0.95, b1=1.05, b2=1.6),
    "s1_zero": dict(s1=0.0, s2=0.2, b1=1.3, b2=1.4),
}
UNET_SIZE = (24, 16)


def install_apply_freeu():
    """Puts oracle.freeu_ref.apply_freeu into the diffusers shim, before the reference's up blocks import it."""
    sys.path.insert(0, os.path.join(ROOT, "oracle", "shim"))
    import diffusers.utils.torch_utils as tu
    from oracle import freeu_ref as FR
    tu.apply_freeu = FR.apply_freeu


def unet_cases(ut):
    from oracle import unet_ref as R
    from oracle.make_golden import build_reference_unet, synth_inputs
    cfg_t, cfg_g = R.tiny_config("tryon"), R.tiny_config("garment")
    sd_t, sd_g = R.make_state_dict(cfg_t, seed=11), R.make_state_dict(cfg_g, seed=22)
    net = build_reference_unet(ut, cfg_t)
    net.load_state_dict(sd_t, strict=True)
    h, w = UNET_SIZE
    x = synth_inputs(cfg_t, cfg_g, 1, h, w)
    out = {}
    with torch.no_grad():
        feats = R.unet_garment_forward(sd_g, cfg_g, x["cloth"], x["timestep"], x["text_embeds_cloth"])
        fc = [torch.cat([torch.zeros_like(d), d]) for d in feats]
        img = R.resampler_forward(sd_t, "encoder_hid_proj", cfg_t["resampler"], x["clip_tokens"])
        added = {"text_embeds": x["text_embeds"], "time_ids": x["time_ids"], "image_embeds": img}

        def run():
            return net(x["sample"], x["timestep"], encoder_hidden_states=x["prompt_embeds"], added_cond_kwargs=added,
                       return_dict=False, garment_features=fc)[0]

        out["off"] = run()
        for name, kw in CASES.items():
            net.enable_freeu(**kw)
            out[name] = run()
            net.disable_freeu()
        assert torch.equal(run(), out["off"]), "disable_freeu must restore the plain forward"
    for name in CASES:
        print(f"unet {name:8s} FreeU effect max|on - off| = {(out[name] - out['off']).abs().max().item():.3e}")
    assert torch.equal(out["s1_zero"], out["off"])
    return {"B": 1, "h": h, "w": w, "noise_pred": {k: v.clone() for k, v in out.items()}}


def pipeline_case(tp, ut, ug, kw):
    """The reference pipeline at config 1 with enable_freeu(**kw): per-step latents, images, the loop's inputs and
    the step noises (as oracle/make_golden_pipeline.py records them)."""
    from oracle import make_golden_pipeline as MG
    from oracle import unet_ref as R
    from oracle.make_golden import build_reference_unet
    from idm_vton_b200.scheduler import DDPMScheduler
    cfg_t, cfg_g = R.tiny_config("tryon"), R.tiny_config("garment")
    sd_t = {k: v.half().float() for k, v in R.make_state_dict(cfg_t, seed=11).items()}
    sd_g = {k: v.half().float() for k, v in R.make_state_dict(cfg_g, seed=22).items()}
    unet, unet_enc = build_reference_unet(ut, cfg_t), build_reference_unet(ug, cfg_g)
    unet.load_state_dict(sd_t, strict=True)
    unet_enc.load_state_dict(sd_g, strict=True)
    sch = DDPMScheduler()
    pipe = tp.StableDiffusionXLInpaintPipeline(
        vae=MG.make_vae(), text_encoder=None, text_encoder_2=None, tokenizer=None, tokenizer_2=None, unet=unet,
        unet_encoder=unet_enc, scheduler=sch, image_encoder=MG.make_image_encoder(cfg_t["resampler"]["embedding_dim"]))
    pipe.enable_freeu(**kw)
    inp = MG.make_call_inputs(cfg_t)
    rec = {"noises": [], "latents": []}
    orig_unet_forward, orig_enc_forward, orig_step = unet.forward, unet_enc.forward, sch.step

    def unet_forward(sample, t, **k):
        if "x13" not in rec:
            rec.update(x13=sample.clone(), prompt_embeds=k["encoder_hidden_states"].clone(),
                       added={n: v.clone() for n, v in k["added_cond_kwargs"].items()})
        return orig_unet_forward(sample, t, **k)

    def enc_forward(sample, t, text, **k):
        rec.setdefault("cloth_latents", sample.clone())
        return orig_enc_forward(sample, t, text, **k)

    def step(*a, **k):
        out = orig_step(*a, **k)
        rec["noises"].append(None if sch._last_noise is None else sch._last_noise.clone())
        return out

    unet.forward, unet_enc.forward, sch.step = unet_forward, enc_forward, step

    def on_step_end(p, i, t, k):
        rec["latents"].append(k["latents"].clone())
        return {}

    torch.manual_seed(1234)
    with torch.no_grad():
        images = pipe(**MG.call_kwargs(inp, torch.Generator().manual_seed(42)), output_type="pt",
                      callback_on_step_end=on_step_end)[0]
    x13 = rec["x13"]
    B = inp["image"].shape[0]
    loop_in = dict(latents=x13[B:, :4], mask=x13[:, 4:5], masked_image_latents=x13[:, 5:9], pose_latents=x13[:, 9:13],
                   cloth_latents=rec["cloth_latents"], prompt_embeds=rec["prompt_embeds"],
                   add_text_embeds=rec["added"]["text_embeds"], add_time_ids=rec["added"]["time_ids"],
                   image_embeds=rec["added"]["image_embeds"], text_embeds_cloth=inp["text_embeds_cloth"])
    return dict(freeu=kw, timesteps=sch.timesteps.clone(), images=images.half(),
                latents_per_step=[t.clone() for t in rec["latents"]],
                loop_inputs={k: v.clone() for k, v in loop_in.items()},
                noises=[None if n is None else n.clone() for n in rec["noises"]])


def signatures():
    from oracle.make_signature_golden import extract
    ref = os.environ.get("IDM_VTON_REFERENCE", "")
    methods = ("enable_freeu", "disable_freeu")
    return {"pipeline": extract(os.path.join(ref, "src", "tryon_pipeline.py"), "StableDiffusionXLInpaintPipeline",
                                methods),
            "unet": extract(os.path.join(ref, "src", "unet_hacked_tryon.py"), "UNet2DConditionModel", methods)}


def main():
    sys.path.insert(0, ROOT)
    install_apply_freeu()
    from oracle.make_golden import import_reference
    ut, ug = import_reference()
    import src.tryon_pipeline as tp
    import src.unet_block_hacked_tryon as ubt
    from oracle import freeu_ref as FR
    assert ubt.apply_freeu is FR.apply_freeu
    unet = unet_cases(ut)
    pipe = pipeline_case(tp, ut, ug, CASES["sdxl"])
    sig = signatures()
    print("signatures", sig)
    torch.save({
        "note": "REFERENCE modules with enable_freeu (src/unet_hacked_tryon.py, src/tryon_pipeline.py on the diffusers "
                "shim with oracle/freeu_ref.apply_freeu), CPU fp32. unet: tiny config, weights seed 11 / 22, inputs "
                f"oracle.make_golden.synth_inputs(B=1, h={UNET_SIZE[0]}, w={UNET_SIZE[1]}, seed=1234); pipeline: config "
                "1 as oracle/make_golden_pipeline.py, FreeU at the SDXL values",
        "cases": CASES, "unet": unet, "pipeline": pipe, "signatures": sig,
    }, os.path.join(GOLDEN, "freeu_ref.pt"))
    print("wrote", os.path.join(GOLDEN, "freeu_ref.pt"))


if __name__ == "__main__":
    main()
