"""DDIM, Euler and DPM-Solver++ on the GPU: b200vton_cfg_solver_step per kind against its float64 restatement
(tests/test_solvers_cpu.py, which also proves every mutant lies at least 4x the tolerance away), the scaled input
scatter, the DPM-Solver++ state inside a CUDA graph, and the engine pipeline against the float64-rule oracle loop
(oracle/solver_ref.py) per scheduler, with scheduler switches and garment-cache hits."""
import pytest
import torch

from test_schedule_cpu import kernel_inputs, r16, rel_err
from test_solvers_cpu import COEF, KERNEL_CASES, MUTANTS, TOL, cfg_solver_ref, mutant_ref, x0_prev_input

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    from idm_vton_b200 import lib as L
    L.load()
    return L


def _coef(c):
    return torch.tensor(c, dtype=torch.float32, device="cuda")


@pytest.mark.parametrize("kind,B,H,W,cfg,with_noise,ldc", KERNEL_CASES)
def test_cfg_solver_kernel_vs_float64(lib, kind, B, H, W, cfg, with_noise, ldc):
    eps, lat, noise = kernel_inputs(B, H, W, ldc, with_noise, seed=B * 100 + H)
    if not cfg:
        eps = eps[:B].contiguous()
    x0p = x0_prev_input(B, H, W, B)
    coefs = [COEF[kind]]
    if kind == "dpmpp":
        first = list(COEF[kind])
        first[7] = 0.0
        coefs.append(tuple(first))
    for c in coefs:
        state = x0p.cuda().clone() if kind == "dpmpp" else None
        out = lib.cfg_solver_step(eps.cuda(), lat.cuda(), None if noise is None else noise.cuda(), _coef(c), kind,
                                  x0_prev=state, do_cfg=cfg).cpu()
        ref, x0 = cfg_solver_ref(eps, lat, noise, x0p, c, kind, cfg)
        e = rel_err(out, ref)
        for m in MUTANTS[kind] + (("lower_order_final_ignored",) if kind == "dpmpp" else ()):
            mut = mutant_ref(eps, lat, noise, x0p, c, kind, m, cfg)
            if mut is not None:
                assert e <= 0.25 * rel_err(mut, ref), m
        assert e <= TOL, (kind, e)
        if kind == "dpmpp":
            assert rel_err(state.cpu(), x0) <= TOL               # the state now holds this step's x0


def test_dpmpp_state_carried_over_two_steps(lib):
    B, H, W = 2, 16, 12
    eps, lat, _ = kernel_inputs(B, H, W, 16, False, seed=11)
    x0p = x0_prev_input(B, H, W, 3)
    state = x0p.cuda().clone()
    c = _coef(COEF["dpmpp"])
    out1 = lib.cfg_solver_step(eps.cuda(), lat.cuda(), None, c, "dpmpp", x0_prev=state)
    out2 = lib.cfg_solver_step(eps.cuda(), out1, None, c, "dpmpp", x0_prev=state).cpu()
    r1, x0 = cfg_solver_ref(eps, lat, None, x0p, COEF["dpmpp"], "dpmpp")
    r2, _ = cfg_solver_ref(eps, r1.half(), None, x0.half(), COEF["dpmpp"], "dpmpp")
    stale, _ = cfg_solver_ref(eps, r1.half(), None, x0p, COEF["dpmpp"], "dpmpp")
    e = rel_err(out2, r2)
    assert e <= TOL and e <= 0.25 * rel_err(stale, r2)


def test_scaled_scatter(lib):
    """fp16(x * scale) into the latent channels only; the unscaled entry point is still a copy."""
    B, H, W, ldc = 2, 7, 9, 16
    x = (torch.randn(B, 4, H, W, generator=torch.Generator().manual_seed(4)) * 14).half()
    dst = torch.full((2 * B, H, W, ldc), 7.0, dtype=torch.float16, device="cuda")
    scale = 1.0 / (14.6 ** 2 + 1) ** 0.5
    lib.nchw_to_nhwc_scaled(x.cuda(), dst, torch.tensor([scale], dtype=torch.float32, device="cuda"))
    want = r16(x.double() * float(torch.tensor(scale, dtype=torch.float32))).permute(0, 2, 3, 1)
    got = dst.cpu().double()
    assert torch.equal(got[:B, ..., :4], want) and torch.equal(got[B:, ..., :4], want)
    assert torch.all(got[..., 4:] == 7.0)
    assert rel_err(x.double().permute(0, 2, 3, 1), want) >= 4 * TOL          # the unscaled mutant is visible
    lib.nchw_to_nhwc(x.cuda(), dst)
    assert torch.equal(dst[:B, ..., :4].cpu(), x.permute(0, 2, 3, 1))


def test_rejects_bad_arguments(lib):
    """Error code 1 before any launch: DPM++ without its state, an unknown kind, misaligned operands."""
    import types
    eps, lat = (t.cuda() for t in kernel_inputs(1, 4, 4, 16, False)[:2])
    c = _coef(COEF["dpmpp"])
    n0 = lib.launch_count()
    with pytest.raises(RuntimeError, match="code 1"):
        lib.cfg_solver_step(eps, lat, None, c, "dpmpp", x0_prev=None)
    raw = lib.load()
    rc = raw.b200vton_cfg_solver_step(eps.data_ptr(), 16, 1, 4, 4, 4, lat.data_ptr(), None, None, c.data_ptr(), 3, 1,
                                      lat.data_ptr(), None)
    assert rc == 1
    odd = lambda t, k: types.SimpleNamespace(data_ptr=lambda: t.data_ptr() + k, shape=t.shape)  # noqa: E731
    with pytest.raises(RuntimeError, match="code 1"):
        lib.cfg_solver_step(eps, lat, None, odd(c, 2), "ddim")
    with pytest.raises(RuntimeError, match="code 1"):
        lib.cfg_solver_step(eps, odd(lat, 1), None, c, "euler", out=torch.empty_like(lat))
    with pytest.raises(RuntimeError, match="code 1"):
        lib.nchw_to_nhwc_scaled(lat, torch.empty(1, 4, 4, 16, dtype=torch.float16, device="cuda"),
                                types.SimpleNamespace(dtype=torch.float32, is_cuda=True, numel=lambda: 1,
                                                      data_ptr=lambda: c.data_ptr() + 2))
    assert lib.launch_count() == n0


def test_graph_replay_equals_eager_over_a_dpmpp_run(lib):
    """A DPM++ 2M run through one captured kernel launch (coefficients and x0_prev on the device) is bit-identical to
    eager launches."""
    from idm_vton_b200.denoise import solver_step_tables
    from idm_vton_b200.scheduler import DDPMScheduler, DPMSolverMultistepScheduler
    s = DPMSolverMultistepScheduler.from_config(DDPMScheduler().config)
    s.set_timesteps(8)
    _, rows, _, _, _ = solver_step_tables(s, s.timesteps)
    table = torch.tensor([[2.0, *r] for r in rows], dtype=torch.float32, device="cuda")
    B, H, W = 2, 16, 12
    eps, lat, _ = (t.cuda() if t is not None else None for t in kernel_inputs(B, H, W, 16, False, seed=21))
    # eager
    x, st = lat.clone(), torch.zeros_like(lat)
    for i in range(len(rows)):
        x = lib.cfg_solver_step(eps, x, None, table[i].contiguous(), "dpmpp", x0_prev=st)
    eager = x.clone()
    # graph
    coef = torch.zeros(8, dtype=torch.float32, device="cuda")
    xs, nxt, st2 = lat.clone(), torch.empty_like(lat), torch.zeros_like(lat)
    keep = (xs.clone(), st2.clone())
    s_ = torch.cuda.Stream()
    s_.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s_):
        lib.cfg_solver_step(eps, xs, None, coef, "dpmpp", x0_prev=st2, out=nxt)
    torch.cuda.current_stream().wait_stream(s_)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        lib.cfg_solver_step(eps, xs, None, coef, "dpmpp", x0_prev=st2, out=nxt)
        xs.copy_(nxt)
    xs.copy_(keep[0])
    st2.copy_(keep[1])
    for i in range(len(rows)):
        coef.copy_(table[i])
        g.replay()
    torch.cuda.synchronize()
    assert torch.equal(xs, eager)


def test_point_mass_invariant_on_the_kernel(lib):
    """With the exact denoiser of a point mass, eps = (x - alpha x0*) / sigma, a whole run of the kernel keeps x on
    alpha x0* + sigma n at every step and ends at x0* where the schedule ends at alpha = 1 / sigma = 0 (DDIM, Euler), up to
    the fp16 rounding of x and eps."""
    from idm_vton_b200.denoise import solver_step_tables
    from oracle.make_golden_solvers import make_scheduler
    B, H, W = 2, 16, 12
    g = torch.Generator().manual_seed(8)
    x0s = torch.randn(B, 4, H, W, generator=g, dtype=torch.float64)
    n = torch.randn(B, 4, H, W, generator=g, dtype=torch.float64)
    for case, kind in (("ddim_eta0", "ddim"), ("euler_leading", "euler"), ("dpmpp_2m", "dpmpp")):
        s = make_scheduler(case)
        s.set_timesteps(10)
        _, rows, scales, _, _ = solver_step_tables(s, s.timesteps)
        ac = s.alphas_cumprod.double()

        def alpha_sigma(i):
            if kind == "ddim":
                a = 1.0 if i == len(rows) else ac[int(s.timesteps[i])].item()
                return a ** 0.5, (1 - a) ** 0.5
            sg = s.sigmas[i].double().item()
            return (1.0, sg) if kind == "euler" else (1 / (sg * sg + 1) ** 0.5, sg / (sg * sg + 1) ** 0.5)

        a, sg = alpha_sigma(0)
        x = (a * x0s + sg * n).half().cuda()
        state = torch.zeros_like(x)
        for i, row in enumerate(rows):
            a, sg = alpha_sigma(i)
            xd = x.double().cpu()
            assert rel_err(xd, a * x0s + sg * n) < 5e-3, (case, i)
            eps = ((xd - a * x0s) / sg).half().permute(0, 2, 3, 1).contiguous().cuda()
            x = lib.cfg_solver_step(eps, x, None, _coef([1.0, *row]), kind, x0_prev=state, do_cfg=False)
        a, sg = alpha_sigma(len(rows))
        assert rel_err(x.double().cpu(), a * x0s + sg * n) < 5e-3, case
        if kind != "dpmpp":
            assert sg == 0.0


# ------------------------------------------------------------------------------------------------------------------
# the pipeline per scheduler against the reference pipeline (tests/golden/pipeline_solvers_ref.pt)
# ------------------------------------------------------------------------------------------------------------------
from test_schedule_gpu import tiny_modules  # noqa: E402,F401  (module-scoped fixture)


def _call_kwargs(tiny, case, steps=None, gen=None):
    from oracle import make_golden_pipeline as MG
    from oracle import make_golden_solvers as MGS
    dev, f16 = "cuda", torch.float16
    inp = {k: (v.to(dev, f16) if k not in ("image", "mask_image") else v.to(dev))
           for k, v in MG.make_call_inputs(tiny["cfg_t"]).items()}
    kw = MGS.case_kwargs(MG, inp, gen if gen is not None else torch.Generator().manual_seed(42), case)
    if steps is not None:
        kw["num_inference_steps"] = steps
    return kw


@pytest.mark.parametrize("case", ["ddim_eta0", "ddim_eta1", "euler_leading", "euler_linspace", "dpmpp_2m",
                                  "dpmpp_2m_karras", "dpmpp_2m_strength"])
def test_pipeline_vs_reference_golden(tiny_modules, case):
    """The three checks of test_schedule_gpu.test_pipeline_schedule_vs_reference_golden, per scheduler case:
    (i) the tensors handed to the loop equal the reference's (init_noise_sigma, add_noise at strength < 1, the RNG order);
    (ii) the engine's latents after every step equal the float64-rule oracle loop run on the engine's own loop inputs and
    step noises; (iii) the deterministic samplers draw no step noise, so the engine's final latents are compared with the
    REFERENCE's own final latents; DDIM at eta = 1 against the oracle on the reference's inputs with the engine's noises."""
    from oracle import make_golden_pipeline as MG
    from oracle import make_golden_schedule as MS
    from oracle import make_golden_solvers as MGS
    from oracle import solver_ref as SV
    from test_schedule_gpu import _err, _make_pipe, _run_recorded
    import os
    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", "pipeline_solvers_ref.pt"))
    c = g["cases"][case]
    pipe = _make_pipe(tiny_modules)
    pipe.scheduler = MGS.make_scheduler(case)
    gen = torch.Generator().manual_seed(42)
    rec = _run_recorded(pipe, _call_kwargs(tiny_modules, case, gen=gen), gen)
    assert [t for t, _ in rec["latents"]] == [int(t) for t in c["timesteps"].tolist()]
    assert torch.equal(pipe.scheduler.timesteps[-len(c["timesteps"]):].double().cpu(), c["timesteps"])
    kind = MGS.KIND[MGS.CASES[case][0]]
    assert pipe._denoiser.kind == kind
    # ---- (i)
    ref_in = MS.loop_inputs(g, case, MG.make_call_inputs(tiny_modules["cfg_t"]))
    e_in = {n: _err(rec["inputs"][n], ref_in[n]) for n in ref_in}
    print(f"{case} (i) loop inputs: " + ", ".join(f"{n} {e:.1e}" for n, e in e_in.items()))
    for n in ("mask", "prompt_embeds", "add_text_embeds", "add_time_ids", "text_embeds_cloth"):
        assert e_in[n] == 0.0, n
    assert e_in["latents"] < (4e-3 if c["kwargs"].get("strength", 1.0) < 1.0 else 1e-3)
    for n in ("masked_image_latents", "pose_latents", "cloth_latents"):
        assert e_in[n] < 3e-3, n
    assert e_in["image_embeds"] < 5e-3
    # ---- (ii)
    dev = "cuda"
    sd_t32 = {k: v.half().float().to(dev) for k, v in tiny_modules["sd_t"].items()}
    sd_g32 = {k: v.half().float().to(dev) for k, v in tiny_modules["sd_g"].items()}
    li = {n: v.to(dev) for n, v in rec["inputs"].items()}
    ts = c["timesteps"]
    eta = c["kwargs"].get("eta", 0.0)

    def oracle(inputs, n=None):
        s = MGS.make_scheduler(case)
        s.set_timesteps(MGS.STEPS)
        with torch.no_grad():
            return SV.denoise_loop(sd_t32, tiny_modules["cfg_t"], sd_g32, tiny_modules["cfg_g"], inputs, s, kind, ts,
                                   guidance_scale=MG.GUIDANCE, eta=eta, noises=rec["noises"], max_steps=n)

    e_loop = [_err(rec["latents"][n - 1][1], oracle(li, n)) for n in range(1, len(rec["latents"]) + 1)]
    # ---- (iii)
    if case in MGS.DETERMINISTIC:
        assert all(x is None for x in rec["noises"])
        e_e2e = _err(rec["latents"][-1][1], c["final_latents"])
    else:
        assert all(x is not None for x in rec["noises"])
        e_e2e = _err(rec["latents"][-1][1], oracle({n: v.to(dev) for n, v in ref_in.items()}))
    print(f"{case}: timesteps {ts.tolist()} (ii) engine vs oracle per step {[f'{e:.2e}' for e in e_loop]}; (iii) "
          f"{'vs the reference' if case in MGS.DETERMINISTIC else 'vs oracle on the reference inputs'} {e_e2e:.2e}")
    assert max(e_loop) < 4e-3
    assert e_e2e < 2e-2


def test_switching_schedulers_recaptures(tiny_modules):
    """Same-shaped calls with DPM++, Euler, DDPM and DPM++ again: each re-captures and equals a fresh pipeline's result."""
    from test_schedule_gpu import _make_pipe
    from oracle.make_golden_solvers import make_scheduler as _scheduler
    from idm_vton_b200.scheduler import DDPMScheduler

    def run(pipe, sch):
        pipe.scheduler = sch
        torch.manual_seed(1234)
        pipe(**_call_kwargs(tiny_modules, "dpmpp_2m", steps=4), output_type="latent")
        return pipe._last_latents.float().cpu()

    pipe = _make_pipe(tiny_modules)
    seq = [lambda: _scheduler("dpmpp_2m"), lambda: _scheduler("euler_leading"), DDPMScheduler, lambda: _scheduler("dpmpp_2m")]
    outs, graphs = [], []
    for make in seq:
        outs.append(run(pipe, make()))
        graphs.append(pipe._denoiser._graph)
    assert all(a is not b for a, b in zip(graphs, graphs[1:]))
    assert torch.equal(outs[0], outs[3])
    assert not torch.equal(outs[0], outs[1]) and not torch.equal(outs[1], outs[2])
    for make, out in zip(seq[:3], outs[:3]):
        assert torch.equal(run(_make_pipe(tiny_modules), make()), out)


@pytest.mark.parametrize("case", ["dpmpp_2m", "euler_linspace"])
def test_serving_garment_cache_hit_equals_miss(tiny_modules, case):
    """serving.TryOnServer under DPM-Solver++ and under Euler's fractional linspace timesteps: a garment seen before takes
    its K/V of all steps from the cache (keyed on the exact timesteps) and gives the bits of the uncached run."""
    from oracle import make_golden_pipeline as MG
    from oracle.make_golden_solvers import make_scheduler
    from test_schedule_gpu import _make_pipe
    from idm_vton_b200.serving import TryOnRequest, TryOnServer
    cfg_t = tiny_modules["cfg_t"]

    def make_pipe():
        p = _make_pipe(tiny_modules)
        p.scheduler = make_scheduler(case)
        return p

    def req(seed):
        i = MG.make_call_inputs(cfg_t, B=1, seed=seed)
        gi = MG.make_call_inputs(cfg_t, B=1, seed=1001)
        return TryOnRequest(garment_id="A", image=i["image"][0], mask_image=i["mask_image"][0], pose_img=i["pose_img"][0],
                            prompt_embeds=i["prompt_embeds"][0], negative_prompt_embeds=i["negative_prompt_embeds"][0],
                            pooled_prompt_embeds=i["pooled_prompt_embeds"][0],
                            negative_pooled_prompt_embeds=i["negative_pooled_prompt_embeds"][0], cloth=gi["cloth"][0],
                            ip_adapter_image=gi["ip_adapter_image"][0], text_embeds_cloth=gi["text_embeds_cloth"][0])

    kw = dict(height=MG.H, width=MG.W, num_inference_steps=4, guidance_scale=2.0, max_batch=4, seed=7)
    srv = TryOnServer(make_pipe(), **kw)
    t1 = srv.submit(req(1))
    out1 = srv.run()
    assert srv.pipe.garment_cache.hits == 0
    t2 = srv.submit(req(1))
    out2 = srv.run()
    assert srv.pipe.garment_cache.hits == 1
    assert torch.equal(out2[t2], out1[t1])
    srv_nc = TryOnServer(make_pipe(), garment_cache_bytes=0, **kw)
    t3 = srv_nc.submit(req(1))
    assert torch.equal(srv_nc.run()[t3], out1[t1])
