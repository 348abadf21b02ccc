"""The denoising-schedule arguments on the GPU: the fused CFG + guidance-rescale + DDPM kernel against its float64
restatement (tests/test_schedule_cpu.py, which also proves every mutant below lies at least 4x the tolerance away), its
exact invariants, and the engine pipeline against the reference pipeline for every case of
tests/golden/pipeline_schedule_ref.pt (oracle/make_golden_schedule.py)."""
import os

import pytest
import torch

from test_schedule_cpu import (COEF, KERNEL_CASES, MUTANTS, TOL_RESCALE, cfg_rescale_ddpm_ref, kernel_inputs,
                               mutant_visible, rel_err)

pytestmark = pytest.mark.gpu

G = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def lib():
    from idm_vton_b200 import lib as L
    L.load()
    return L


def _coef(phi):
    return torch.tensor([*COEF, phi], dtype=torch.float32, device="cuda")


@pytest.mark.parametrize("B,H,W,phi,with_noise,ldc", KERNEL_CASES)
def test_cfg_rescale_ddpm_kernel_vs_float64(lib, B, H, W, phi, with_noise, ldc):
    eps, lat, noise = kernel_inputs(B, H, W, ldc, with_noise, seed=B * 1000 + H)
    out = lib.cfg_rescale_ddpm_step(eps.cuda(), lat.cuda(), None if noise is None else noise.cuda(), _coef(phi)).cpu()
    ref = cfg_rescale_ddpm_ref(eps, lat, noise, COEF, phi)
    e = rel_err(out, ref)
    for m in MUTANTS:
        if mutant_visible(m, H, W, phi):
            assert e <= 0.25 * rel_err(cfg_rescale_ddpm_ref(eps, lat, noise, COEF, phi, mutant=m), ref), m
    assert e <= TOL_RESCALE, e


def test_cfg_rescale_ddpm_exact_invariants(lib):
    B, H, W = 2, 16, 12
    eps, lat, noise = (x.cuda() for x in kernel_inputs(B, H, W, 16, True, seed=5))
    plain = lib.cfg_ddpm_step(eps, lat, noise, _coef(0.0))
    # phi = 0: fp16(0 * x) + fp16(1 * g) = g, so the plain kernel's bits
    assert torch.equal(lib.cfg_rescale_ddpm_step(eps, lat, noise, _coef(0.0)), plain)
    # phi = 1 with a zero uncond half: g = fp16(0 + fp16(gs * cond)); at gs = 1 that is cond, so r = std(cond) / std(g) = 1
    # and the (1 - phi) term is zero: the plain step's bits
    e0 = eps.clone()
    e0[:B] = 0
    c1 = _coef(1.0)
    c1[0] = 1.0
    assert torch.equal(lib.cfg_rescale_ddpm_step(e0, lat, noise, c1), lib.cfg_ddpm_step(e0, lat, noise, c1))
    # without CFG phi is ignored, as in the reference
    e1 = eps[:B].contiguous()
    assert torch.equal(lib.cfg_rescale_ddpm_step(e1, lat, noise, _coef(0.7), do_cfg=False),
                       lib.cfg_ddpm_step(e1, lat, noise, _coef(0.7), do_cfg=False))
    # deterministic, and a graph replay equals the eager launch
    c = _coef(0.7)
    eager = lib.cfg_rescale_ddpm_step(eps, lat, noise, c)
    assert torch.equal(eager, lib.cfg_rescale_ddpm_step(eps, lat, noise, c))
    out = torch.empty_like(lat)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        lib.cfg_rescale_ddpm_step(eps, lat, noise, c, out=out)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        lib.cfg_rescale_ddpm_step(eps, lat, noise, c, out=out)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)


# ------------------------------------------------------------------------------------------------------------------
# the pipeline vs the reference pipeline, per schedule case
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tiny_modules():
    from oracle import unet_ref as R
    from idm_vton_b200 import unet as U
    cfg_t, cfg_g = R.tiny_config("tryon"), R.tiny_config("garment")
    sd_t, sd_g = R.make_state_dict(cfg_t, seed=11), R.make_state_dict(cfg_g, seed=22)
    net_t = U.UNet2DConditionModel(cfg_t, sd_t).to("cuda", torch.float16)
    net_g = U.UNet2DConditionModelGarment(cfg_g, sd_g).to("cuda", torch.float16)
    return dict(cfg_t=cfg_t, cfg_g=cfg_g, sd_t=sd_t, sd_g=sd_g, net_t=net_t, net_g=net_g)


def _err(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return (a - b).abs().max().item() / max(1.0, b.abs().max().item())


def _make_pipe(tiny):
    from oracle import make_golden_pipeline as MG
    from idm_vton_b200.pipeline import StableDiffusionXLInpaintPipeline
    from idm_vton_b200.scheduler import DDPMScheduler
    dev, f16 = "cuda", torch.float16
    return StableDiffusionXLInpaintPipeline(
        vae=MG.make_vae().to(dev, f16), text_encoder=None, text_encoder_2=None, tokenizer=None, tokenizer_2=None,
        unet=tiny["net_t"], unet_encoder=tiny["net_g"], scheduler=DDPMScheduler(),
        image_encoder=MG.make_image_encoder(tiny["cfg_t"]["resampler"]["embedding_dim"]).to(dev, f16))


def _run_recorded(pipe, kwargs, gen):
    """__call__ recording the denoiser's inputs, the step noises and the latents after every step. The golden run drew
    every random tensor in fp32 on the CPU generator; the fp16 pipeline's draws from that generator are taken in fp32 and
    rounded (as tests/test_seams_gpu.py does), so order, shapes and count of the draws stay the pipeline's own."""
    from idm_vton_b200.denoise import TryOnDenoiser
    if pipe._denoiser is None:
        pipe._denoiser = TryOnDenoiser(pipe.unet.engine(), pipe.unet_encoder.engine())
    den = pipe._denoiser
    rec = {"noises": [], "latents": []}
    names = ("latents", "mask", "masked_image_latents", "pose_latents", "cloth_latents", "prompt_embeds", "add_text_embeds",
             "add_time_ids", "image_embeds", "text_embeds_cloth")
    real_prepare, real_step = TryOnDenoiser.prepare, TryOnDenoiser.step

    def prepare(*a, **kw):
        rec["inputs"] = {n: v.detach().float().cpu().clone() for n, v in zip(names, a)}
        return real_prepare(den, *a, **kw)

    def step(i, noise=None, use_graph=True):
        rec["noises"].append(None if noise is None else noise.detach().float().clone())
        return real_step(den, i, noise, use_graph=use_graph)

    def on_step_end(p, i, t, kw):
        rec["latents"].append((int(t), kw["latents"].float().cpu().clone()))
        return {}

    real_randn = torch.randn

    def randn_fp32_draws(*size, generator=None, dtype=None, **kw):
        if generator is gen and dtype == torch.float16:
            return real_randn(*size, generator=generator, dtype=torch.float32, **kw).to(torch.float16)
        return real_randn(*size, generator=generator, dtype=dtype, **kw)

    den.prepare, den.step = prepare, step
    torch.manual_seed(1234)
    torch.randn = randn_fp32_draws
    try:
        pipe(**kwargs, output_type="pt", callback_on_step_end=on_step_end)
    finally:
        torch.randn = real_randn
        del den.prepare, den.step
    return rec


@pytest.mark.parametrize("case", ["default", "strength_rescale", "custom_timesteps", "denoising_end", "start_end",
                                  "start_only"])
def test_pipeline_schedule_vs_reference_golden(tiny_modules, case):
    """Per case of the golden, the three checks of test_seams_gpu.test_pipeline_call_vs_reference_golden:
    (i) the tensors handed to the loop equal the reference's (pins the RNG order: with strength < 1 the image-latents
    sample, then the noise, then the masked-image, pose and garment samples; and add_noise / the image latents as start);
    (ii) the engine loop equals the oracle loop on the same tensors and noises, per step (timesteps, custom steps,
    guidance rescale on the device); (iii) a loose end-to-end gate: the engine's result against the oracle loop run on
    the reference's own loop inputs with the engine's step noises."""
    from oracle import schedule_ref as SR
    from oracle import make_golden_pipeline as MG
    from oracle import make_golden_schedule as MS
    g = torch.load(os.path.join(G, "pipeline_schedule_ref.pt"))
    c = g["cases"][case]
    dev, f16 = "cuda", torch.float16
    cfg_t, cfg_g = tiny_modules["cfg_t"], tiny_modules["cfg_g"]
    inp = {k: (v.to(dev, f16) if k not in ("image", "mask_image") else v.to(dev)) for k, v in MG.make_call_inputs(cfg_t).items()}
    pipe = _make_pipe(tiny_modules)
    gen = torch.Generator().manual_seed(42)
    rec = _run_recorded(pipe, MS.case_kwargs(MG, inp, gen, case), gen)
    assert [t for t, _ in rec["latents"]] == c["timesteps"].tolist()
    # ---- (i)
    ref_in = MS.loop_inputs(g, case, MG.make_call_inputs(cfg_t))
    e_in = {n: _err(rec["inputs"][n], ref_in[n]) for n in ref_in}
    print(f"{case} (i) loop inputs: " + ", ".join(f"{n} {e:.1e}" for n, e in e_in.items()))
    for n in ("mask", "prompt_embeds", "add_text_embeds", "add_time_ids", "text_embeds_cloth"):
        assert e_in[n] == 0.0, n
    from_image = c["kwargs"].get("strength", 0.9999) < 1.0
    # pure noise: the fp32 draw rounded to fp16; from the image: the fp32 VAE (TF32 convolutions) result rounded to fp16,
    # noised by add_noise in fp16 (coefficients and products rounded)
    assert e_in["latents"] < (4e-3 if from_image else 1e-3)
    for n in ("masked_image_latents", "pose_latents", "cloth_latents"):
        assert e_in[n] < 3e-3, n
    assert e_in["image_embeds"] < 5e-3
    # ---- (ii)
    sd_t32 = {k: v.half().float().to(dev) for k, v in tiny_modules["sd_t"].items()}
    sd_g32 = {k: v.half().float().to(dev) for k, v in tiny_modules["sd_g"].items()}
    li = {n: v.to(dev) for n, v in rec["inputs"].items()}
    num_steps, ts = MS.oracle_schedule(case, c["timesteps"].tolist())
    phi = c["kwargs"].get("guidance_rescale", 0.0)
    e_loop = []
    with torch.no_grad():
        for n in range(1, len(rec["latents"]) + 1):
            ref = SR.denoise_loop(sd_t32, cfg_t, sd_g32, cfg_g, li, num_steps, guidance_scale=MG.GUIDANCE,
                                  noises=rec["noises"], max_steps=n, timesteps=ts, guidance_rescale=phi)
            e_loop.append(_err(rec["latents"][n - 1][1], ref))
    # ---- (iii) end to end given the step noises: the engine's last latents against the oracle loop on the REFERENCE's own
    # loop inputs (golden). The engine's variance-noise draws are not the reference's (they differ completely at step 0,
    # for strength 1.0 as well), so the reference's own latents and images cannot be compared at these sigmas; the
    # oracle takes the engine's noises instead.
    gold_in = {n: v.to(dev) for n, v in ref_in.items()}
    with torch.no_grad():
        ref_e2e = SR.denoise_loop(sd_t32, cfg_t, sd_g32, cfg_g, gold_in, num_steps, guidance_scale=MG.GUIDANCE,
                                  noises=rec["noises"], timesteps=ts, guidance_rescale=phi)
    e_e2e = _err(rec["latents"][-1][1], ref_e2e)
    print(f"{case} (ii) engine vs oracle loop per step {[f'{e:.2e}' for e in e_loop]}; (iii) vs oracle on the reference's "
          f"inputs {e_e2e:.2e}")
    assert max(e_loop) < 4e-3
    assert e_e2e < 2e-2


def test_rescale_toggle_does_not_replay_stale_graph(tiny_modules):
    """Same-shaped calls with guidance_rescale switched on, off and on again: each takes the step kernel it asks for (the
    graph is re-captured), and results repeat exactly."""
    from oracle import make_golden_pipeline as MG
    dev, f16 = "cuda", torch.float16
    inp = {k: (v.to(dev, f16) if k not in ("image", "mask_image") else v.to(dev))
           for k, v in MG.make_call_inputs(tiny_modules["cfg_t"]).items()}
    pipe = _make_pipe(tiny_modules)

    def run(phi):
        torch.manual_seed(1234)
        kw = dict(MG.call_kwargs(inp, torch.Generator().manual_seed(42)), guidance_rescale=phi)
        pipe(**kw, output_type="latent")
        return pipe._last_latents.float().cpu()

    out, graphs = [], []
    for phi in (0.7, 0.0, 0.7, 0.0):
        out.append(run(phi))
        graphs.append(pipe._denoiser._graph)
    assert torch.equal(out[0], out[2]) and torch.equal(out[1], out[3])
    assert _err(out[0], out[1]) > 1e-3
    assert all(a is not b for a, b in zip(graphs, graphs[1:]))      # re-captured at every switch
