"""DDIM, Euler and DPM-Solver++ without a GPU: the restated scheduler classes, the coefficients the engine derives from
a scheduler object, closed-form identities of the float64 update rules (oracle/solver_ref.py), the float64 restatement
of b200vton_cfg_solver_step that tests/test_solvers_gpu.py gates against, proof that every mutant of it lies at least 4x
the tolerance away, and the refusal of every scheduler the engine does not implement."""
import math
import types

import numpy as np
import pytest
import torch

from test_schedule_cpu import U16, kernel_inputs, r16, rel_err

# Kernel vs restatement, max|a - b| / max|b| (as tests/test_schedule_cpu.py): the kernel forms each product in fp32
# before rounding it to fp16, which lands on the other side of an fp16 tie than the exact product about once in 2^13
# operations; a few such one-ulp flips, carried with weights below 1, stay within 8 U16 of the output scale.
TOL = 8 * U16
KINDS = ("ddim", "euler", "dpmpp")
# {gs, s, inv_a, p, q, r, sigma_n, k} per kind at a mid-schedule step (sigma_n only used with noise)
COEF = {
    "ddim": (2.0, 0.83, 1.0 / 0.557, 0.0, 0.62, 0.70, 0.21, 0.0),
    "euler": (2.0, 1.6, 1.0 / 1.6, 1.0, 0.0, -0.55, 0.0, 0.0),
    "dpmpp": (2.0, 0.83, 1.0 / 0.557, 0.78, 0.21, 0.0, 0.0, 1.0 / 0.62),
}
KERNEL_CASES = [(kind, b, h, w, cfg, nz, ldc) for kind in KINDS for b in (1, 2) for (h, w) in ((16, 12), (7, 9))
                for cfg in (True, False) for nz, ldc in ((True, 16), (False, 13)) if nz is False or kind == "ddim"]
MUTANTS = {"dpmpp": ("r0_one", "x0_prev_not_updated", "lower_order_final_ignored"), "ddim": ("sigma_sq_swap",),
           "euler": ("no_scale_model_input",)}


def _c32(c):
    return [float(torch.tensor(v, dtype=torch.float32)) for v in c]


def f32(x):
    return x.float().double() if torch.is_tensor(x) else float(torch.tensor(x, dtype=torch.float32))


def cfg_solver_ref(eps, lat, noise, x0_prev, coef, kind, do_cfg=True):
    """float64 restatement of b200vton_cfg_solver_step with each kind's rounding points (elementwise.cu). Returns
    (out, x0) — x0 is the new x0_prev of kind dpmpp."""
    B, C = lat.shape[0], lat.shape[1]
    e = eps[..., :C].permute(0, 3, 1, 2).double()
    gs, s, inv_a, p, q, r, sigma_n, k = _c32(coef)
    g = r16(e[:B] + r16(gs * r16(e[B:] - e[:B]))) if do_cfg else e[:B]
    x = lat.double()
    x0 = None
    if kind == "ddim":
        x0 = r16(r16(x - r16(s * g)) * inv_a)
        out = r16(r16(q * x0) + r16(r * g))
    elif kind == "euler":
        x0 = f32(x - r16(s * g))
        d = f32(f32(x - x0) * inv_a)
        out = r16(f32(x + f32(d * r)))
    else:
        x0 = r16(r16(x - r16(s * g)) * inv_a)
        d1 = r16(k * r16(x0 - x0_prev.double()))
        out = r16(f32(f32(f32(p * x) + r16(q * x0)) + r16(f32(0.5 * q) * d1)))
    if noise is not None:
        out = r16(out + r16(sigma_n * noise.double()))
    return out, x0


def mutant_ref(eps, lat, noise, x0_prev, coef, kind, mutant, do_cfg=True):
    """The restatement with a plausible bug in the step kernel or its coefficients."""
    c = list(coef)
    if mutant == "r0_one":                      # DPM++ second order with r0 = 1
        c[7] = 1.0
    elif mutant == "lower_order_final_ignored":  # a first-order step (k = 0) taken at second order
        c[7] = 1.0 / 0.62
        if coef[7] != 0.0:
            return None
    elif mutant == "sigma_sq_swap":             # DDIM: sqrt(1 - a_prev - sigma) and sigma^2 noise
        a_prev = c[4] ** 2
        sig = c[6]
        if noise is None:
            return None
        c[5] = math.sqrt(max(1 - a_prev - sig, 0.0))
        c[6] = sig * sig
    elif mutant == "x0_prev_not_updated":       # second step reads the state from before the first
        return None
    elif mutant == "no_scale_model_input":      # checked on the input scatter, not here
        return None
    return cfg_solver_ref(eps, lat, noise, x0_prev, c, kind, do_cfg)[0]


def x0_prev_input(B, H, W, seed):
    g = torch.Generator().manual_seed(seed + 7)
    return (torch.randn(B, 4, H, W, generator=g, dtype=torch.float64) * 0.5).half()


# ------------------------------------------------------------------------------------------------------------------
# restated scheduler classes
# ------------------------------------------------------------------------------------------------------------------
def _ddpm_config():
    from idm_vton_b200.scheduler import DDPMScheduler
    return DDPMScheduler().config


@pytest.mark.parametrize("n", [4, 10, 15, 20, 30])
@pytest.mark.parametrize("spacing", ["leading", "trailing", "linspace"])
def test_restated_timesteps_and_sigmas(n, spacing):
    from idm_vton_b200.scheduler import DDIMScheduler, DPMSolverMultistepScheduler, EulerDiscreteScheduler
    T = 1000
    ddim = DDIMScheduler.from_config(_ddpm_config(), timestep_spacing=spacing)
    ddim.set_timesteps(n)
    want = {"leading": np.arange(n)[::-1] * (T // n) + 1, "trailing": np.round(np.arange(T, 0, -T / n)) - 1,
            "linspace": np.linspace(0, T - 1, n).round()[::-1]}[spacing]
    assert ddim.timesteps.tolist() == want.astype(np.int64).tolist() and ddim.timesteps.dtype == torch.int64
    ac = ddim.alphas_cumprod.double()
    sig_train = ((1 - ac) / ac).sqrt()

    eu = EulerDiscreteScheduler.from_config(_ddpm_config(), timestep_spacing=spacing)
    eu.set_timesteps(n)
    ts = eu.timesteps.double()
    assert len(ts) == n and eu.timesteps.dtype == torch.float32 and len(eu.sigmas) == n + 1 and eu.sigmas[-1] == 0
    assert torch.all(ts[1:] < ts[:-1])
    if spacing == "linspace":
        assert torch.allclose(ts, torch.linspace(T - 1, 0, n, dtype=torch.float64), atol=1e-3)
        assert (T - 1) % (n - 1) == 0 or any(t != round(t) for t in ts.tolist())   # fractional timesteps survive
    # linear interpolation of the training sigmas at the (possibly fractional) timesteps
    lo = ts.floor().long().clamp(max=T - 2)
    w = ts - lo
    interp = (1 - w) * sig_train[lo] + w * sig_train[lo + 1]
    assert torch.allclose(eu.sigmas[:-1].double(), interp, rtol=1e-6)
    smax = eu.sigmas.max().double().item()
    want_init = smax if spacing in ("linspace", "trailing") else math.sqrt(smax ** 2 + 1)
    assert abs(float(eu.init_noise_sigma) - want_init) < 1e-5 * want_init

    for karras in (False, True):
        dpm = DPMSolverMultistepScheduler.from_config(_ddpm_config(), timestep_spacing=spacing, use_karras_sigmas=karras)
        dpm.set_timesteps(n)
        ts = dpm.timesteps
        assert len(ts) == n and len(dpm.sigmas) == n + 1 and ts.dtype == torch.int64
        assert torch.all(ts[1:] <= ts[:-1]) and dpm.init_noise_sigma == 1.0 and dpm.order == 1
        s = dpm.sigmas.double()
        if karras:
            rho = 7.0
            lo_, hi_ = sig_train[0].item(), sig_train[-1].item()
            ramp = torch.linspace(0, 1, n, dtype=torch.float64)
            want_s = (hi_ ** (1 / rho) + ramp * (lo_ ** (1 / rho) - hi_ ** (1 / rho))) ** rho
            assert torch.allclose(s[:-1], want_s, rtol=1e-6) and s[-1] == s[-2]
        else:
            assert torch.allclose(s[:-1], sig_train[ts], rtol=1e-6)
            assert abs(s[-1].item() - sig_train[0].item()) < 1e-6


def test_dpm_known_timesteps():
    from idm_vton_b200.scheduler import DPMSolverMultistepScheduler, EulerDiscreteScheduler
    d = DPMSolverMultistepScheduler()
    d.set_timesteps(4)
    assert d.timesteps.tolist() == [999, 749, 500, 250]
    d = DPMSolverMultistepScheduler(timestep_spacing="leading", steps_offset=1)
    d.set_timesteps(4)
    assert d.timesteps.tolist() == [801, 601, 401, 201]
    e = EulerDiscreteScheduler.from_config(_ddpm_config())         # the IDM-VTON config: leading, steps_offset 1
    e.set_timesteps(4)
    assert e.timesteps.tolist() == [751.0, 501.0, 251.0, 1.0]


def test_from_config_of_the_ddpm_config():
    from idm_vton_b200.scheduler import DDIMScheduler, DPMSolverMultistepScheduler, EulerDiscreteScheduler
    for cls in (DDIMScheduler, EulerDiscreteScheduler, DPMSolverMultistepScheduler):
        s = cls.from_config(_ddpm_config())
        assert s.config.timestep_spacing == "leading" and s.config.steps_offset == 1
        assert torch.equal(s.alphas_cumprod, DDIMScheduler().alphas_cumprod)
        assert cls.from_config(dict(s.config)).config == s.config            # a plain dict config, as diffusers'
    assert DDIMScheduler.from_config(_ddpm_config()).config.clip_sample is False


# ------------------------------------------------------------------------------------------------------------------
# coefficients from scheduler objects
# ------------------------------------------------------------------------------------------------------------------
def _schedulers(n=6):
    from idm_vton_b200.scheduler import DDIMScheduler, DPMSolverMultistepScheduler, EulerDiscreteScheduler
    out = {}
    for name, s in (("ddim", DDIMScheduler.from_config(_ddpm_config())),
                    ("euler", EulerDiscreteScheduler.from_config(_ddpm_config())),
                    ("euler_linspace", EulerDiscreteScheduler.from_config(_ddpm_config(), timestep_spacing="linspace")),
                    ("dpmpp", DPMSolverMultistepScheduler.from_config(_ddpm_config())),
                    ("dpmpp_karras", DPMSolverMultistepScheduler.from_config(_ddpm_config(), use_karras_sigmas=True))):
        s.set_timesteps(n)
        out[name] = s
    return out


def _make_foreign(cls_name, attrs):
    cls = type(cls_name, (), {"step": lambda self, model_output, timestep, sample, eta=0.0, generator=None: None})
    obj = cls()
    for k, v in attrs.items():
        setattr(obj, k, v)
    return obj


def test_foreign_scheduler_objects_give_the_same_coefficients():
    from idm_vton_b200.denoise import solver_step_tables
    for name, s in _schedulers().items():
        f = _make_foreign(type(s).__name__, {**{k: getattr(s, k) for k in (
            "alphas_cumprod", "final_alpha_cumprod", "sigmas", "timesteps", "num_inference_steps") if hasattr(s, k)},
            "config": dict(s.config)})
        for eta in (0.0, 1.0):
            ts = s.timesteps[1:]                                    # a strength < 1 run starts past the first step
            assert solver_step_tables(f, ts, eta) == solver_step_tables(s, ts, eta), name


def _host_step_with_coefficients(kind, row, x, eps, x0_prev):
    """The kernel's formula in float64 on one coefficient row (no CFG, no rounding)."""
    s, inv_a, p, q, r, sn, k = row
    x0 = (x - s * eps) * inv_a
    if kind == "ddim":
        return q * x0 + r * eps, x0
    if kind == "euler":
        return x + r * eps, x0
    return p * x + q * ((1 + k / 2) * x0 - k / 2 * x0_prev), x0


@pytest.mark.parametrize("name", ["ddim", "euler", "euler_linspace", "dpmpp", "dpmpp_karras"])
def test_coefficients_reproduce_the_restated_step(name):
    """Every row the engine uploads, applied in float64, equals the restated class's own step() over a whole run."""
    from idm_vton_b200.denoise import solver_step_tables
    s = _schedulers(8)[name]
    kind, rows, scales, draws, applied = solver_step_tables(s, s.timesteps, 0.0)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(1, 4, 6, 5, generator=g, dtype=torch.float64) * float(s.init_noise_sigma)
    xr, x0p = x.clone(), torch.zeros_like(x)
    for i, t in enumerate(s.timesteps):
        eps = torch.randn(1, 4, 6, 5, generator=g, dtype=torch.float64)
        if scales is not None:
            assert abs(scales[i] - float(s.scale_model_input(torch.ones(1), t))) < 1e-7
        x = s.step(eps, t, x, return_dict=False)[0]
        xr, x0p = _host_step_with_coefficients(kind, rows[i], xr, eps, x0p)
        assert rel_err(xr, x) < 1e-5, (name, i)
    assert draws == ([True] * 8 if kind == "euler" else [False] * 8) and applied == (kind == "ddim")


def test_dpm_orders_and_lower_order_final():
    from idm_vton_b200.denoise import solver_step_tables
    s = _schedulers(6)["dpmpp"]
    ks = [r[6] for r in solver_step_tables(s, s.timesteps)[1]]
    assert ks[0] == 0 and ks[-1] == 0 and all(k > 0 for k in ks[1:-1])
    s.config["lower_order_final"] = False
    assert all(r[6] > 0 for r in solver_step_tables(s, s.timesteps)[1][1:])
    from idm_vton_b200.scheduler import DPMSolverMultistepScheduler
    s = DPMSolverMultistepScheduler.from_config(_ddpm_config())
    s.set_timesteps(20)                                   # >= 15 steps: the last step stays second order
    assert solver_step_tables(s, s.timesteps)[1][-1][6] > 0
    part = solver_step_tables(s, s.timesteps[10:])[1]    # a run that starts mid-schedule starts at first order
    assert part[0][6] == 0 and part[1][6] > 0


# ------------------------------------------------------------------------------------------------------------------
# closed-form identities of the float64 update rules (oracle/solver_ref.py)
# ------------------------------------------------------------------------------------------------------------------
def _ac():
    from idm_vton_b200.scheduler import DDIMScheduler
    return DDIMScheduler().alphas_cumprod.double()


def test_first_order_dpmpp_equals_ddim_eta0():
    from oracle.solver_ref import ddim_update, dpmpp_update
    ac = _ac()
    g = torch.Generator().manual_seed(0)
    x, eps = (torch.randn(2, 4, 5, 5, generator=g, dtype=torch.float64) for _ in range(2))
    for t, tp in ((999, 749), (500, 250), (250, 1)):
        a, ap = ac[t].item(), ac[tp].item()
        x0 = (x - math.sqrt(1 - a) * eps) / math.sqrt(a)
        d = dpmpp_update(x, x0, math.sqrt(a), math.sqrt(1 - a), math.sqrt(ap), math.sqrt(1 - ap))
        assert rel_err(d, ddim_update(x, eps, a, ap)) < 1e-12


def test_euler_in_scaled_coordinates_equals_ddim_eta0():
    from oracle.solver_ref import ddim_update, euler_update
    ac = _ac()
    g = torch.Generator().manual_seed(1)
    x, eps = (torch.randn(2, 4, 5, 5, generator=g, dtype=torch.float64) for _ in range(2))
    for t, tp in ((999, 749), (500, 250), (251, 1)):
        a, ap = ac[t].item(), ac[tp].item()
        s, sp = math.sqrt((1 - a) / a), math.sqrt((1 - ap) / ap)
        e = euler_update(x / math.sqrt(a), eps, s, sp)                  # x_bar = x / alpha
        assert rel_err(e * math.sqrt(ap), ddim_update(x, eps, a, ap)) < 1e-12


@pytest.mark.parametrize("name", ["ddim", "euler", "euler_linspace", "dpmpp", "dpmpp_karras"])
def test_point_mass_stays_on_its_path(name):
    """With the exact denoiser of a point mass, eps(x, t) = (x - alpha x0*) / sigma, x stays on alpha x0* + sigma n and
    reaches x0* where the schedule ends at sigma = 0 (DDIM with alpha_prev = 1, Euler)."""
    from oracle.solver_ref import SolverRef
    s = _schedulers(10)[name]
    kind = {"euler_linspace": "euler", "dpmpp_karras": "dpmpp"}.get(name, name)
    g = torch.Generator().manual_seed(2)
    x0s, n = (torch.randn(1, 4, 5, 5, generator=g, dtype=torch.float64) for _ in range(2))
    ref = SolverRef(s, kind)
    ac = s.alphas_cumprod.double()

    def alpha_sigma(i, t):                       # the scheduler's own parametrisation at step i
        if kind == "ddim":
            return math.sqrt(ac[int(t)]), math.sqrt(1 - ac[int(t)])
        sg = s.sigmas[i].double().item()
        return (1.0, sg) if kind == "euler" else (1 / math.sqrt(sg * sg + 1), sg / math.sqrt(sg * sg + 1))

    a, sg = alpha_sigma(0, s.timesteps[0])
    x = a * x0s + sg * n
    for i, t in enumerate(s.timesteps):
        a, sg = alpha_sigma(i, t)
        assert rel_err(x, a * x0s + sg * n) < 1e-9, (name, i)
        x = ref.step((x - a * x0s) / sg, t, x)
    if kind == "euler":
        assert rel_err(x, x0s) < 1e-12
    elif kind == "ddim":
        assert rel_err(x, x0s) < 1e-12                   # set_alpha_to_one: the last step lands at alpha = 1
    else:
        a_end, s_end = alpha_sigma(len(s.timesteps), None)
        assert rel_err(x, a_end * x0s + s_end * n) < 1e-9


# ------------------------------------------------------------------------------------------------------------------
# the kernel's restatement and its mutants
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,B,H,W,cfg,with_noise,ldc", KERNEL_CASES)
def test_solver_mutants_are_far_from_truth(kind, B, H, W, cfg, with_noise, ldc):
    eps, lat, noise = kernel_inputs(B, H, W, ldc, with_noise, seed=B * 100 + H)
    x0p = x0_prev_input(B, H, W, B)
    ref, _ = cfg_solver_ref(eps, lat, noise, x0p, COEF[kind], kind, cfg)
    for m in MUTANTS[kind]:
        mut = mutant_ref(eps, lat, noise, x0p, COEF[kind], kind, m, cfg)
        if mut is not None:
            assert rel_err(mut, ref) >= 4 * TOL, (m, rel_err(mut, ref))
    if kind == "dpmpp":
        first = list(COEF[kind])
        first[7] = 0.0
        ref1, _ = cfg_solver_ref(eps, lat, noise, x0p, first, kind, cfg)
        assert rel_err(mutant_ref(eps, lat, noise, x0p, first, kind, "lower_order_final_ignored", cfg), ref1) >= 4 * TOL
        # two steps with the state carried, against the second step reading the state from before the first
        out1, x0 = cfg_solver_ref(eps, lat, None, x0p, COEF[kind], kind, cfg)
        out2, _ = cfg_solver_ref(eps, out1, None, x0.half(), COEF[kind], kind, cfg)
        stale, _ = cfg_solver_ref(eps, out1, None, x0p, COEF[kind], kind, cfg)
        assert rel_err(stale, out2) >= 4 * TOL


# ------------------------------------------------------------------------------------------------------------------
# the reference pipeline's own runs (tests/golden/pipeline_solvers_ref.pt, oracle/make_golden_solvers.py)
# ------------------------------------------------------------------------------------------------------------------
def _solvers_golden():
    import os
    return torch.load(os.path.join(os.path.dirname(__file__), "golden", "pipeline_solvers_ref.pt"))


def test_oracle_loop_replays_the_reference_golden():
    """oracle/solver_ref.denoise_loop reproduces the reference loop of every golden case from its loop inputs."""
    from oracle import make_golden_pipeline as MG
    from oracle import make_golden_schedule as MS
    from oracle import make_golden_solvers as MGS
    from oracle import solver_ref as SV
    from oracle import unet_ref as R
    g = _solvers_golden()
    assert set(g["cases"]) == set(MGS.CASES) and g["steps"] == MGS.STEPS
    cfg_t, cfg_g = R.tiny_config("tryon"), R.tiny_config("garment")
    sd_t = {k: v.half().float() for k, v in R.make_state_dict(cfg_t, seed=11).items()}
    sd_g = {k: v.half().float() for k, v in R.make_state_dict(cfg_g, seed=22).items()}
    call_inputs = MG.make_call_inputs(cfg_t)
    for name, c in g["cases"].items():
        s = MGS.make_scheduler(name)
        s.set_timesteps(MGS.STEPS)
        with torch.no_grad():
            out = SV.denoise_loop(sd_t, cfg_t, sd_g, cfg_g, MS.loop_inputs(g, name, call_inputs), s,
                                  MGS.KIND[c["scheduler"]], c["timesteps"], guidance_scale=MG.GUIDANCE,
                                  eta=c["kwargs"].get("eta", 0.0), noises=c["noises"])
        ref = c["final_latents"]
        assert (out - ref).abs().max().item() < 1e-4 * max(1.0, ref.abs().max().item()), name


def test_pipeline_timestep_selection_matches_reference_golden():
    """The engine pipeline's own timestep selection (retrieve_timesteps, get_timesteps with strength) on each restated
    scheduler gives the timesteps the reference ran; Euler's linspace ones stay fractional."""
    from oracle import make_golden_solvers as MGS
    from test_schedule_cpu import _pipe_on_cpu, select_timesteps
    g = _solvers_golden()
    p = _pipe_on_cpu()
    for name, c in g["cases"].items():
        p.scheduler = MGS.make_scheduler(name)
        ts, n, _ = select_timesteps(p, MGS.STEPS, strength=c["kwargs"].get("strength", 1.0))
        assert [float(t) for t in ts] == c["timesteps"].tolist() and n == len(ts), name
    assert any(t != int(t) for t in g["cases"]["euler_linspace"]["timesteps"].tolist())
    # the initial latents of a strength-1 call are the noise times init_noise_sigma (about 14.6 for Euler leading)
    assert g["cases"]["euler_leading"]["latents"].abs().max() > 20 and g["cases"]["dpmpp_2m"]["latents"].abs().max() < 6


# ------------------------------------------------------------------------------------------------------------------
# refusals
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["EulerAncestralDiscreteScheduler", "HeunDiscreteScheduler", "PNDMScheduler",
                                  "LMSDiscreteScheduler", "UniPCMultistepScheduler", "DEISMultistepScheduler",
                                  "KDPM2DiscreteScheduler", "LCMScheduler", "DPMSolverSinglestepScheduler",
                                  "DPMSolverSDEScheduler"])
def test_unsupported_scheduler_classes_raise(name):
    from idm_vton_b200.denoise import ddpm_step_coefficients, scheduler_kind, solver_step_tables
    from idm_vton_b200.scheduler import DDPMScheduler
    d = DDPMScheduler()
    d.set_timesteps(4)
    f = _make_foreign(name, {"alphas_cumprod": d.alphas_cumprod, "timesteps": d.timesteps, "num_inference_steps": 4,
                             "config": dict(num_train_timesteps=1000, prediction_type="epsilon")})
    with pytest.raises(NotImplementedError, match=name):
        scheduler_kind(f)
    with pytest.raises(NotImplementedError, match=name):
        solver_step_tables(f, d.timesteps)
    # ddpm_step_coefficients itself is unchanged: it only reads the DDPM attributes
    assert ddpm_step_coefficients(f, 751) == ddpm_step_coefficients(d, 751)


def test_unsupported_configs_raise():
    from idm_vton_b200.denoise import solver_step_tables
    from idm_vton_b200.scheduler import DDIMScheduler, DPMSolverMultistepScheduler, EulerDiscreteScheduler
    bad = [(DDIMScheduler, dict(clip_sample=True)), (DDIMScheduler, dict(thresholding=True)),
           (DDIMScheduler, dict(prediction_type="v_prediction")),
           (EulerDiscreteScheduler, dict(prediction_type="v_prediction")),
           (EulerDiscreteScheduler, dict(interpolation_type="log_linear")),
           (DPMSolverMultistepScheduler, dict(solver_order=3)),
           (DPMSolverMultistepScheduler, dict(algorithm_type="dpmsolver")),
           (DPMSolverMultistepScheduler, dict(algorithm_type="sde-dpmsolver++")),
           (DPMSolverMultistepScheduler, dict(solver_type="heun")),
           (DPMSolverMultistepScheduler, dict(thresholding=True)),
           (DPMSolverMultistepScheduler, dict(prediction_type="v_prediction")),
           (DPMSolverMultistepScheduler, dict(use_lu_lambdas=True))]
    ok = {DDIMScheduler: DDIMScheduler.from_config(_ddpm_config()),
          EulerDiscreteScheduler: EulerDiscreteScheduler.from_config(_ddpm_config()),
          DPMSolverMultistepScheduler: DPMSolverMultistepScheduler.from_config(_ddpm_config())}
    for cls, over in bad:
        s = ok[cls]
        s.set_timesteps(4)
        f = _make_foreign(cls.__name__, {**{k: getattr(s, k) for k in (
            "alphas_cumprod", "final_alpha_cumprod", "sigmas", "timesteps", "num_inference_steps") if hasattr(s, k)},
            "config": {**dict(s.config), **over}})
        with pytest.raises(NotImplementedError):
            solver_step_tables(f, s.timesteps)
    # no supported scheduler is stepped as DDPM
    for name, s in _schedulers().items():
        assert solver_step_tables(s, s.timesteps)[0] != "ddpm", name


def test_pipeline_refuses_unsupported_scheduler_and_rescale():
    from idm_vton_b200.pipeline import StableDiffusionXLInpaintPipeline as P
    from idm_vton_b200.scheduler import DPMSolverMultistepScheduler
    from idm_vton_b200.vae import AutoencoderKL
    unet = types.SimpleNamespace(config=types.SimpleNamespace(time_cond_proj_dim=None, sample_size=32, in_channels=13),
                                 device=torch.device("cpu"))
    p = P(AutoencoderKL(block_out_channels=(32, 32), layers_per_block=1), None, None, None, None, unet, None,
          DPMSolverMultistepScheduler())
    kw = dict(prompt_embeds=torch.zeros(1, 77, 8), image=torch.zeros(1, 3, 64, 64), mask_image=torch.zeros(1, 1, 64, 64))
    with pytest.raises(NotImplementedError, match="guidance_rescale"):
        p(guidance_rescale=0.5, **kw)
    p.scheduler = _make_foreign("HeunDiscreteScheduler", {})
    with pytest.raises(NotImplementedError, match="HeunDiscreteScheduler"):
        p(**kw)
    from idm_vton_b200.scheduler import DDIMScheduler, DDPMScheduler
    p.scheduler = DDIMScheduler()
    assert p.prepare_extra_step_kwargs(None, 0.3) == {"eta": 0.3, "generator": None}
    p.scheduler = DDPMScheduler()
    assert p.prepare_extra_step_kwargs(None, 0.3) == {"generator": None}
