"""Denoising-schedule arguments without a GPU: the restated DDPMScheduler's custom timesteps and add_noise, the denoiser's
step coefficients on a custom schedule, the pipeline's timestep selection against the reference's own (golden
tests/golden/pipeline_schedule_ref.pt, made by oracle/make_golden_schedule.py), the oracle loop with guidance rescale, and
the float64 restatement of the fused CFG + guidance-rescale + DDPM kernel that tests/test_schedule_gpu.py gates against,
with proof that every mutant of it lies at least 4x the tolerance away at the shapes the GPU tests use."""
import math
import os
import types

import pytest
import torch

G = os.path.join(os.path.dirname(__file__), "golden")
U16 = 2.0 ** -11          # fp16 unit roundoff

# Kernel vs the float64 restatement, max|a - b| / max|b|. The restatement rounds to fp16 at the same points; the kernel
# forms each product in fp32 first, which rounds to the other side of an fp16 tie than the exact product about once in
# 2^13 operations: one fp16 ulp (2 U16) of that intermediate, carried to the output with a weight below 1 at the test
# coefficients. A few such flips and the output rounding itself stay within 8 U16 of the output scale.
TOL_RESCALE = 8 * U16

# (B, H, W, phi, with_noise, ldc) of the GPU kernel cases
KERNEL_CASES = [(b, h, w, phi, nz, ldc) for b in (1, 2, 8) for (h, w) in ((2, 2), (16, 12), (128, 96))
                for phi in (0.3, 0.7, 1.0) for nz, ldc in ((True, 16), (False, 13))]
MUTANTS = ("std_uncond", "per_channel", "inverted", "swap_phi", "population_one")
COEF = (2.0, 0.83, 1.0 / 0.55, 0.31, 0.68, 0.12)          # gs, sqrt(1-abar), 1/sqrt(abar), c0, c1, sigma


def r16(x):
    return x.half().to(x.dtype)


def rel_err(a, b):
    a, b = a.double(), b.double()
    den = b.abs().max().item()
    err = (a - b).abs().max().item()
    return err / den if den > 0 else (0.0 if err == 0 else math.inf)


def mutant_visible(m, H, W, phi):
    """Where a mutant is a plausible, detectable bug: swapping phi and 1 - phi changes nothing near phi = 0.5 (and the
    test's phi = 0.3 / 0.7 pair only exchanges the weights); a population std in one of the two statistics shifts the
    ratio by sqrt(N / (N - 1)), which only small samples (2x2: N = 16) make larger than the tolerance. (The same estimator
    in both statistics cancels in the ratio, so only the one-sided mistake is a mutant.)"""
    if m == "swap_phi":
        return phi != 0.5
    if m == "population_one":
        return H * W <= 4 and phi == 1.0
    return True


def kernel_inputs(B, H, W, ldc, with_noise, seed=0, device="cpu"):
    """eps [2B, H, W, ldc] NHWC fp16 whose cond half has a per-channel correlation with the uncond half and a per-channel
    spread of its own (so the per-channel std ratios differ from the per-sample one, and std(cond) from std(uncond));
    latents / noise [B, 4, H, W] fp16. The latents are small against the guided eps, so the rescaled eps dominates the
    step's output."""
    g = torch.Generator().manual_seed(seed)
    ch = torch.tensor([1.0, 1.0, 0.7, 0.5], dtype=torch.float64)
    u = torch.randn(B, H, W, 4, generator=g, dtype=torch.float64) * ch
    k = torch.tensor([1.0, 0.8, 0.2, -0.5], dtype=torch.float64)         # cond vs uncond correlation per channel
    n = torch.tensor([0.2, 1.0, 2.0, 3.0], dtype=torch.float64)          # and spread of the cond-only part
    t = u * k + torch.randn(B, H, W, 4, generator=g, dtype=torch.float64) * ch * n
    eps = torch.randn(2 * B, H, W, ldc, generator=g, dtype=torch.float64)        # padding columns stay random
    eps[:B, ..., :4], eps[B:, ..., :4] = u, t
    lat = torch.randn(B, 4, H, W, generator=g, dtype=torch.float64) * 0.1
    noise = torch.randn(B, 4, H, W, generator=g, dtype=torch.float64) if with_noise else None
    f = lambda x: None if x is None else x.half().to(device)  # noqa: E731
    return f(eps), f(lat), f(noise)


def cfg_rescale_ddpm_ref(eps, lat, noise, coef, phi, mutant=None):
    """float64 restatement of b200vton_cfg_rescale_ddpm_step with the reference's fp16 rounding points:
    g = u + fp16(gs fp16(t - u)); s = fp16(std) (unbiased, per sample over C*H*W); r = fp16(s_t / s_g);
    g' = fp16(fp16(phi fp16(g r)) + fp16((1 - phi) g)); then the DDPM step of cfg_ddpm_step on g'.
    mutant: 'std_uncond' | 'per_channel' | 'inverted' | 'swap_phi' | 'population_one' (std_cfg population)."""
    B, C = lat.shape[0], lat.shape[1]
    e = eps[..., :C].permute(0, 3, 1, 2).double()
    u, t = e[:B], e[B:]
    gs, sb, inv_sa, c0, c1, sigma = (float(torch.tensor(c, dtype=torch.float32)) for c in coef)
    phi32 = torch.tensor(phi, dtype=torch.float32)
    a, b = float(phi32), float(1.0 - phi32)                  # the kernel forms 1 - phi in fp32
    if mutant == "swap_phi":
        a, b = b, a
    g = r16(u + r16(gs * r16(t - u)))
    dims = (2, 3) if mutant == "per_channel" else (1, 2, 3)
    s_t = r16((u if mutant == "std_uncond" else t).std(dim=dims, keepdim=True))
    s_g = r16(g.std(dim=dims, keepdim=True, correction=0 if mutant == "population_one" else 1))
    r = r16(s_g / s_t) if mutant == "inverted" else r16(s_t / s_g)
    gr = r16(r16(a * r16(g * r)) + r16(b * g))
    x = lat.double()
    x0 = r16(r16(x - r16(sb * gr)) * inv_sa)
    prev = r16(r16(c0 * x0) + r16(c1 * x))
    if noise is not None:
        prev = r16(prev + r16(sigma * noise.double()))
    return prev


# ------------------------------------------------------------------------------------------------------------------
# restated scheduler
# ------------------------------------------------------------------------------------------------------------------
def test_custom_timesteps_and_previous_timestep():
    from idm_vton_b200.scheduler import DDPMScheduler
    s = DDPMScheduler()
    s.set_timesteps(timesteps=[901, 601, 301, 1])
    assert s.custom_timesteps and s.timesteps.tolist() == [901, 601, 301, 1] and s.timesteps.dtype == torch.int64
    assert [s.previous_timestep(t) for t in (901, 601, 301, 1)] == [601, 301, 1, -1]
    s.set_timesteps(4)                                       # a step count switches back to the spaced schedule
    assert not s.custom_timesteps and s.timesteps.tolist() == [751, 501, 251, 1] and s.previous_timestep(501) == 251
    for bad in ([601, 901, 1], [901, 901, 1], [1000, 500, 1]):
        with pytest.raises(ValueError):
            s.set_timesteps(timesteps=bad)
    with pytest.raises(ValueError, match="only pass one"):
        s.set_timesteps(4, timesteps=[901, 1])


def test_add_noise_formula():
    from idm_vton_b200.scheduler import DDPMScheduler
    s = DDPMScheduler(rescale_betas_zero_snr=True)
    g = torch.Generator().manual_seed(0)
    x0, eps = torch.randn(3, 4, 8, 8, generator=g), torch.randn(3, 4, 8, 8, generator=g)
    ts = torch.tensor([999, 500, 0])
    out = s.add_noise(x0, eps, ts)
    ac = s.alphas_cumprod.double()
    ref = ac[ts].sqrt().view(-1, 1, 1, 1) * x0.double() + (1 - ac[ts]).sqrt().view(-1, 1, 1, 1) * eps.double()
    assert rel_err(out, ref) < 1e-6
    assert torch.equal(out[0], eps[0] * (1 - s.alphas_cumprod[999]) ** 0.5)     # zero terminal SNR: pure noise at T-1
    # fp16 samples: alphas_cumprod cast to fp16 first, the arithmetic in fp16 (diffusers)
    out16 = s.add_noise(x0.half(), eps.half(), ts)
    ac16 = s.alphas_cumprod.half()
    assert out16.dtype == torch.float16
    assert torch.equal(out16, ac16[ts].pow(0.5).view(-1, 1, 1, 1) * x0.half() + (1 - ac16[ts]).pow(0.5).view(-1, 1, 1, 1) * eps.half())


def test_step_coefficients_on_custom_schedule():
    """The coefficients the engine uploads reproduce the scheduler's own step() on a custom schedule (uneven gaps, the
    last timestep stepping to -1)."""
    from idm_vton_b200.denoise import ddpm_step_coefficients
    from idm_vton_b200.scheduler import DDPMScheduler
    s = DDPMScheduler()
    s.set_timesteps(timesteps=[950, 700, 333, 90, 3])
    g = torch.Generator().manual_seed(1)
    x, eps, noise = (torch.randn(1, 4, 8, 8, generator=g) for _ in range(3))
    for t in s.timesteps.tolist():
        sb, inv_sa, c0, c1, sigma = ddpm_step_coefficients(s, t)
        assert (sb, inv_sa, c0, c1, sigma) == s.step_coefficients(t)
        gen = torch.Generator().manual_seed(7)
        want = s.step(eps, t, x, generator=gen, return_dict=False)[0]
        drawn = torch.randn(x.shape, generator=torch.Generator().manual_seed(7))
        mine = c0 * ((x - sb * eps) * inv_sa) + c1 * x + sigma * drawn
        assert rel_err(mine, want) < 1e-5, t


def test_custom_schedule_without_previous_timestep_raises():
    """A scheduler with a custom list and no previous_timestep(): t - T_train // steps would step to the wrong timestep."""
    from idm_vton_b200.denoise import ddpm_step_coefficients
    from idm_vton_b200.scheduler import DDPMScheduler
    foreign = types.SimpleNamespace(alphas_cumprod=DDPMScheduler().alphas_cumprod, num_inference_steps=None,
                                    custom_timesteps=True, config=dict(num_train_timesteps=1000))
    with pytest.raises(TypeError, match="previous_timestep"):
        ddpm_step_coefficients(foreign, 901)
    foreign.custom_timesteps = False
    foreign.num_inference_steps = 4
    assert ddpm_step_coefficients(foreign, 751) == ddpm_step_coefficients(
        types.SimpleNamespace(**{**vars(foreign), "previous_timestep": lambda t: t - 250}), 751)


# ------------------------------------------------------------------------------------------------------------------
# the pipeline's timestep selection and the oracle loop vs the reference (golden)
# ------------------------------------------------------------------------------------------------------------------
def _golden():
    return torch.load(os.path.join(G, "pipeline_schedule_ref.pt"))


def _pipe_on_cpu():
    from idm_vton_b200.pipeline import StableDiffusionXLInpaintPipeline as P
    from idm_vton_b200.scheduler import DDPMScheduler
    from idm_vton_b200.vae import AutoencoderKL
    unet = types.SimpleNamespace(config=types.SimpleNamespace(time_cond_proj_dim=None, sample_size=32, in_channels=13),
                                 device=torch.device("cpu"))
    return P(AutoencoderKL(block_out_channels=(32, 32), layers_per_block=1), None, None, None, None, unet, None,
             DDPMScheduler())


def select_timesteps(p, steps, timesteps=None, strength=0.9999, denoising_start=None, denoising_end=None, **_):
    """The pipeline's own steps 4 and 11 of __call__: retrieve_timesteps, get_timesteps, the denoising_end cut."""
    from idm_vton_b200.pipeline import retrieve_timesteps
    p._denoising_start, p._denoising_end = denoising_start, denoising_end
    ts, n = retrieve_timesteps(p.scheduler, steps if timesteps is None else None, None, timesteps)
    ts, n = p.get_timesteps(n, strength, None, denoising_start=denoising_start)
    first = ts[:1]
    ts, n = p._apply_denoising_end(ts, n)
    return ts.tolist(), n, first.tolist()


def test_pipeline_timestep_selection_matches_reference():
    g = _golden()
    p = _pipe_on_cpu()
    assert len(g["cases"]) == 6
    for name, c in g["cases"].items():
        ts, n, first = select_timesteps(p, g["steps"], **c["kwargs"])
        assert ts == c["timesteps"].tolist() and n == len(ts), name
    # the default call (strength 0.9999) runs 29 of 30 steps from the second timestep
    ts, n, first = select_timesteps(p, 30)
    assert n == 29 and first == [925] and ts[-1] == 1
    with pytest.raises(ValueError, match="cannot be larger"):
        select_timesteps(p, 4, denoising_start=0.6, denoising_end=0.4)
    # the quirk: with denoising_end not a float, denoising_start is never checked against it and still cuts the start
    ts, _, _ = select_timesteps(p, 4, denoising_start=0.6)
    assert ts == [251, 1]


def test_oracle_loop_with_rescale_and_custom_schedule_vs_reference_golden():
    """schedule_ref.denoise_loop reproduces the reference loop on the golden's inputs and noises (rescale, custom list),
    and with no schedule arguments it is loop_ref.denoise_loop."""
    from oracle import loop_ref as LR
    from oracle import make_golden_pipeline as MG
    from oracle import make_golden_schedule as MS
    from oracle import schedule_ref as SR
    from oracle import unet_ref as R
    g = _golden()
    cfg_t, cfg_g = R.tiny_config("tryon"), R.tiny_config("garment")
    sd_t = {k: v.half().float() for k, v in R.make_state_dict(cfg_t, seed=11).items()}
    sd_g = {k: v.half().float() for k, v in R.make_state_dict(cfg_g, seed=22).items()}
    call_inputs = MG.make_call_inputs(cfg_t)
    assert set(MS.REPLAY_CASES) == {n for n, c in g["cases"].items() if c["noises"] is not None}
    for name in MS.REPLAY_CASES:
        c = g["cases"][name]
        num_steps, ts = MS.oracle_schedule(name, c["timesteps"].tolist())
        with torch.no_grad():
            out = SR.denoise_loop(sd_t, cfg_t, sd_g, cfg_g, MS.loop_inputs(g, name, call_inputs), num_steps,
                                  guidance_scale=2.0, noises=c["noises"], timesteps=ts,
                                  guidance_rescale=c["kwargs"].get("guidance_rescale", 0.0))
        ref = c["final_latents"]
        assert (out - ref).abs().max().item() < 1e-4 * max(1.0, ref.abs().max().item()), name
    inp = MS.loop_inputs(g, "denoising_end", call_inputs)
    noises = [torch.randn(1, 4, 32, 32, generator=torch.Generator().manual_seed(i)) for i in range(2)]
    with torch.no_grad():
        a = SR.denoise_loop(sd_t, cfg_t, sd_g, cfg_g, inp, 30, noises=noises, max_steps=2)
        b = LR.denoise_loop(sd_t, cfg_t, sd_g, cfg_g, inp, 30, noises=noises, max_steps=2)
    assert torch.equal(a, b)


def test_rescale_noise_cfg_oracle_formula():
    from oracle.schedule_ref import rescale_noise_cfg
    g = torch.Generator().manual_seed(2)
    cfg, text = torch.randn(2, 4, 6, 5, generator=g, dtype=torch.float64), torch.randn(2, 4, 6, 5, generator=g, dtype=torch.float64) * 3
    out = rescale_noise_cfg(cfg, text, 0.7)
    for b in range(2):
        n = cfg[b].numel()
        sd = lambda x: ((x - x.mean()) ** 2).sum().div(n - 1).sqrt()  # noqa: E731
        want = 0.7 * cfg[b] * sd(text[b]) / sd(cfg[b]) + 0.3 * cfg[b]
        assert torch.allclose(out[b], want, rtol=1e-12, atol=0)


# ------------------------------------------------------------------------------------------------------------------
# the kernel's restatement and its mutants
# ------------------------------------------------------------------------------------------------------------------
def test_rescale_reference_phi_zero_is_plain_step():
    """At phi = 0 the restatement is the plain CFG + DDPM step (the rounding points of test_kernels_gpu's cfg_ddpm)."""
    eps, lat, noise = kernel_inputs(2, 16, 12, 16, True, seed=3)
    ref = cfg_rescale_ddpm_ref(eps, lat, noise, COEF, 0.0)
    e = eps[..., :4].permute(0, 3, 1, 2).double()
    u, t = e[:2], e[2:]
    gs, sb, inv_sa, c0, c1, sigma = (float(torch.tensor(c, dtype=torch.float32)) for c in COEF)
    gg = r16(u + r16(gs * r16(t - u)))
    x = lat.double()
    plain = r16(r16(r16(c0 * r16(r16(x - r16(sb * gg)) * inv_sa)) + r16(c1 * x)) + r16(sigma * noise.double()))
    assert torch.equal(ref, plain)


@pytest.mark.parametrize("B,H,W,phi,with_noise,ldc", KERNEL_CASES)
def test_rescale_mutants_are_far_from_truth(B, H, W, phi, with_noise, ldc):
    eps, lat, noise = kernel_inputs(B, H, W, ldc, with_noise, seed=B * 1000 + H)
    ref = cfg_rescale_ddpm_ref(eps, lat, noise, COEF, phi)
    checked = 0
    for m in MUTANTS:
        if not mutant_visible(m, H, W, phi):
            continue
        d = rel_err(cfg_rescale_ddpm_ref(eps, lat, noise, COEF, phi, mutant=m), ref)
        assert d >= 4 * TOL_RESCALE, (m, d)
        checked += 1
    assert checked >= 3
