"""Sampling presets on the GPU:
  * b200vton_cfg_step_mixed_rows: each row bit-identical to the per-kind kernel launched on that sample alone (the
    rescale kernel for a DDPM row with phi > 0), x0_prev of the other kinds untouched, noise ignored on Euler and
    DPM-Solver++ rows, and mutants (one kind for every row, phi zeroed) that must differ;
  * the scaled scatter at scale 1 against the plain scatter;
  * ContinuousTryOnServer with presets (tiny config): each request the same bits as in a one-preset server of its
    preset whatever its neighbours, slots and arrival order; graph replay against eager launches; each preset against
    TryOnServer(max_batch=1) (gated by batch mode's batch-size spread, bit-identical in pool mode at slots = 1); page
    sharing by timesteps, and results across page hits and evictions;
  * SDXL width: a DDPM and a DPM-Solver++ request in 2 slots against the batch-mode denoiser.
"""
import pytest
import torch

from test_continuous_gpu import _bound, _drive, _err, _pair_inputs, _report, _request, _scheduler

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------
# kernel
# ------------------------------------------------------------------------------------------------
# rows: DDIM (eta > 0), Euler, DPM-Solver++ first order, DPM-Solver++ second order, DDPM, DDPM with rescale 0.7
KINDS6 = ["ddim", "euler", "dpmpp", "dpmpp", "ddpm", "ddpm"]
CODES = {"ddim": 0, "euler": 1, "dpmpp": 2, "ddpm": 3}


def _mixed_inputs(seed=7, B=6, H=24, W=20, ldc=16):
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s, k=1.0: (torch.randn(*s, generator=g, device="cuda") * k).half()  # noqa: E731
    coef = torch.tensor([
        [2.5, 0.6, 1.7, 0.0, 0.55, 0.3, 0.12, 0.0],            # DDIM {gs, s, inv_a, p, q, r, sigma_n, k}
        [3.0, 4.0, 0.25, 1.0, 0.0, -1.3, 0.0, 0.0],            # Euler
        [2.0, 0.9, 2.2, 0.7, 0.45, 0.0, 0.0, 0.0],             # DPM-Solver++, first order (k = 0)
        [4.5, 0.8, 1.9, 0.6, 0.5, 0.0, 0.0, 1.4],              # DPM-Solver++, second order
        [2.0, 0.7, 1.4, 0.2, 0.8, 0.1, 0.0, 0.0],              # DDPM {gs, sb, inv_sa, c0, c1, sigma, phi, 0}
        [3.5, 0.5, 1.2, 0.25, 0.85, 0.15, 0.7, 0.0],           # DDPM with guidance rescale 0.7
    ], dtype=torch.float32, device="cuda")
    return (r(2 * B, H, W, ldc, k=1.5), r(B, 4, H, W, k=3.0), r(B, 4, H, W), r(B, 4, H, W), coef,
            torch.tensor([CODES[k] for k in KINDS6], dtype=torch.int32, device="cuda"))


def _per_kind(L, kind, eps, lat, noise, coef, x0p, cfg):
    """The per-kind kernel on one sample, with the noise its scheduler applies (DDPM, DDIM)."""
    if kind == "ddpm":
        step = L.cfg_rescale_ddpm_step if float(coef[6]) > 0 else L.cfg_ddpm_step
        return step(eps, lat, noise, coef, do_cfg=cfg)
    return L.cfg_solver_step(eps, lat, noise if kind == "ddim" else None, coef, kind, x0_prev=x0p, do_cfg=cfg)


@pytest.mark.parametrize("cfg", [True, False])
def test_mixed_kernel_rows_equal_per_kind_kernels(cfg):
    from idm_vton_b200 import lib as L
    eps, lat, noise, x0p, coef, kinds = _mixed_inputs()
    B = lat.shape[0]
    if not cfg:
        eps = eps[:B].contiguous()
    state = x0p.clone()
    out = L.cfg_step_mixed_rows(eps, lat, noise, coef, kinds, state, do_cfg=cfg)
    refs = []
    for b, kind in enumerate(KINDS6):
        rows = [b, B + b] if cfg else [b]
        st = x0p[b:b + 1].clone()
        ref = _per_kind(L, kind, eps[rows].contiguous(), lat[b:b + 1].contiguous(), noise[b:b + 1].contiguous(),
                        coef[b].contiguous(), st, cfg)
        refs.append(ref)
        assert torch.equal(out[b:b + 1], ref), (kind, b)
        assert torch.equal(state[b:b + 1], st if kind == "dpmpp" else x0p[b:b + 1]), (kind, b)
    assert not torch.equal(state[2:4], x0p[2:4])                        # the DPM-Solver++ rows did advance
    # noise on the Euler and DPM-Solver++ rows changes nothing
    quiet = noise.clone()
    quiet[1:4] = 0
    assert torch.equal(L.cfg_step_mixed_rows(eps, lat, quiet, coef, kinds, x0p.clone(), do_cfg=cfg), out)
    # mutants: one kind for every row; no rescale on the rescale row
    for wrong in ("ddim", "ddpm"):
        one = torch.full_like(kinds, CODES[wrong])
        mut = L.cfg_step_mixed_rows(eps, lat, noise, coef, one, x0p.clone(), do_cfg=cfg)
        for b, kind in enumerate(KINDS6):
            if kind != wrong:
                assert not torch.equal(mut[b:b + 1], refs[b]), (wrong, kind, b)
    if cfg:
        no_phi = coef.clone()
        no_phi[5, 6] = 0.0
        mut = L.cfg_step_mixed_rows(eps, lat, noise, no_phi, kinds, x0p.clone(), do_cfg=cfg)
        assert not torch.equal(mut[5:6], refs[5]) and torch.equal(mut[:5], out[:5])


def test_mixed_kernel_checks_arguments():
    from idm_vton_b200 import lib as L
    eps, lat, noise, x0p, coef, kinds = _mixed_inputs()
    n0 = L.launch_count()
    with pytest.raises(RuntimeError, match="code 1"):
        L.cfg_step_mixed_rows(eps, lat, noise, coef[:, :7].contiguous(), kinds, x0p)
    with pytest.raises(RuntimeError, match="code 1"):
        L.cfg_step_mixed_rows(eps, lat, noise, coef, kinds, None)
    with pytest.raises(ValueError, match="kinds"):
        L.cfg_step_mixed_rows(eps, lat, noise, coef, kinds.long(), x0p)
    with pytest.raises(ValueError, match="kinds"):
        L.cfg_step_mixed_rows(eps, lat, noise, coef, kinds[:5], x0p)
    assert L.launch_count() == n0


def test_scaled_scatter_at_scale_one_equals_the_plain_scatter():
    from idm_vton_b200 import lib as L
    B, H, W, ldc = 3, 7, 9, 64
    x = (torch.randn(B, 4, H, W, device="cuda") * 14).half()
    a = torch.full((2 * B, H, W, ldc), 7.0, dtype=torch.float16, device="cuda")
    b = a.clone()
    L.nchw_to_nhwc_scaled_rows(x, a, torch.ones(B, dtype=torch.float32, device="cuda"))
    L.nchw_to_nhwc(x, b)
    assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------
# the servers (tiny config)
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tiny_modules():
    from oracle import unet_ref as R
    from idm_vton_b200 import unet as U
    cfg_t, cfg_g = R.tiny_config("tryon"), R.tiny_config("garment")
    sd_t, sd_g = R.make_state_dict(cfg_t, seed=11), R.make_state_dict(cfg_g, seed=22)
    net_t = U.UNet2DConditionModel(cfg_t, sd_t).to("cuda", torch.float16)
    net_g = U.UNet2DConditionModelGarment(cfg_g, sd_g).to("cuda", torch.float16)
    return dict(cfg_t=cfg_t, cfg_g=cfg_g, net_t=net_t, net_g=net_g)


PRESETS = ["ddpm", "ddim", "euler", "dpmpp", "rescale", "strength"]


def _preset(name):
    from idm_vton_b200.serving import SamplingPreset
    return {"ddpm": lambda: SamplingPreset(_scheduler("ddpm"), 4),
            "ddim": lambda: SamplingPreset(_scheduler("ddim"), 4, eta=1.0),
            "euler": lambda: SamplingPreset(_scheduler("euler"), 4),
            "dpmpp": lambda: SamplingPreset(_scheduler("dpmpp"), 3),
            "rescale": lambda: SamplingPreset(_scheduler("ddpm"), 4, guidance_rescale=0.7),
            "strength": lambda: SamplingPreset(_scheduler("ddpm"), 4, strength=0.5)}[name]()


def _make_pipe(tiny):
    from test_schedule_gpu import _make_pipe as make
    return make(tiny)


def _server(tiny, names, slots=3, pages=None):
    from oracle import make_golden_pipeline as MG
    from idm_vton_b200.serving import ContinuousTryOnServer
    srv = ContinuousTryOnServer(_make_pipe(tiny), height=MG.H, width=MG.W, slots=slots, seed=7, output_type="pt",
                                presets={n: _preset(n) for n in names}, default_preset=names[0],
                                garment_kv_bytes=None if pages is None else 0)
    if pages is not None:
        srv.garment_kv_bytes = pages * srv.page_bytes()
    return srv


def _req(tiny, k, name, garment=None):
    r = _request(tiny, 60 + k, garment or "ABC"[k % 3])
    r.sampling = name
    return r


def test_presets_server_takes_the_mixed_path_only_when_needed(tiny_modules):
    one = _server(tiny_modules, ["dpmpp"])
    one.submit(_req(tiny_modules, 0, "dpmpp"))
    one.step()
    assert not one.mixed and one.den.kind == "dpmpp" and one.den.kinds is None
    two = _server(tiny_modules, ["ddpm", "dpmpp"])
    two.submit(_req(tiny_modules, 0, "dpmpp"))
    two.step()
    assert two.mixed and two.den.kind == "mixed" and two.den.kinds is not None
    assert _server(tiny_modules, ["rescale"]).mixed


def test_mixed_server_requests_equal_one_preset_servers(tiny_modules):
    """At S = 3 each request's final latents in a server with all six presets are the bits of the same request in a
    server of its preset alone, beside neighbours on other presets, in other slots and at two arrival orders."""
    alone = {}
    for k, n in enumerate(PRESETS):
        _, lat, _ = _drive(_server(tiny_modules, [n]), [([_req(tiny_modules, k, n)], 0)])
        alone[n] = lat[0]
    reqs = lambda: [_req(tiny_modules, k, n) for k, n in enumerate(PRESETS)]  # noqa: E731
    r = reqs()
    _, lat_a, _ = _drive(_server(tiny_modules, PRESETS), [([r[0], r[3]], 1), ([r[2]], 2), ([r[1], r[4], r[5]], 0)])
    order_a = [0, 3, 2, 1, 4, 5]                                      # tickets in submit order
    r = reqs()
    _, lat_b, _ = _drive(_server(tiny_modules, PRESETS[::-1]), [([r[5], r[4], r[3]], 2), ([r[2], r[1], r[0]], 0)])
    order_b = [5, 4, 3, 2, 1, 0]
    for order, lat in ((order_a, lat_a), (order_b, lat_b)):
        for ticket, k in enumerate(order):
            assert torch.equal(lat[ticket], alone[PRESETS[k]]), (PRESETS[k], ticket)
    assert not torch.equal(alone["ddpm"], alone["rescale"]) and not torch.equal(alone["ddpm"], alone["strength"])


def test_mixed_graph_replay_equals_eager(tiny_modules):
    script = lambda: [([_req(tiny_modules, 0, "dpmpp"), _req(tiny_modules, 1, "rescale")], 1),  # noqa: E731
                      ([_req(tiny_modules, 2, "euler")], 2),
                      ([_req(tiny_modules, 3, "ddim"), _req(tiny_modules, 4, "strength"), _req(tiny_modules, 5, "ddpm")], 0)]
    img_g, lat_g, _ = _drive(_server(tiny_modules, PRESETS), script(), use_graph=True)
    img_e, lat_e, _ = _drive(_server(tiny_modules, PRESETS), script(), use_graph=False)
    assert sorted(lat_g) == sorted(lat_e) == list(range(6))
    assert all(torch.equal(lat_g[k], lat_e[k]) and torch.equal(img_g[k], img_e[k]) for k in lat_g)


def _batch_mode(tiny, name, r, monkeypatch, rec):
    """TryOnServer(max_batch=1) on one request with preset `name`, recording the denoiser's inputs and step noises."""
    from oracle import make_golden_pipeline as MG
    from idm_vton_b200.denoise import TryOnDenoiser
    from idm_vton_b200.serving import TryOnServer
    names = ("latents", "mask", "masked_image_latents", "pose_latents", "cloth_latents", "prompt_embeds",
             "add_text_embeds", "add_time_ids", "image_embeds", "text_embeds_cloth")
    real_prepare, real_tables, real_step = TryOnDenoiser.prepare, TryOnDenoiser.set_step_tables, TryOnDenoiser.step

    def prepare(self, *a, **kw):
        rec.append(dict(inp={n: v.clone() for n, v in zip(names, a)}, kw=kw, noises=[]))
        return real_prepare(self, *a, **kw)

    def set_step_tables(self, scheduler, timesteps, **kw):
        rec[-1].update(scheduler=scheduler, timesteps=timesteps, eta=kw.get("eta", 0.0))
        return real_tables(self, scheduler, timesteps, **kw)

    def step(self, i, noise=None, use_graph=True):
        rec[-1]["noises"].append(None if noise is None else noise.clone())
        return real_step(self, i, noise, use_graph=use_graph)
    with monkeypatch.context() as m:
        m.setattr(TryOnDenoiser, "prepare", prepare)
        m.setattr(TryOnDenoiser, "set_step_tables", set_step_tables)
        m.setattr(TryOnDenoiser, "step", step)
        pipe = _make_pipe(tiny)
        srv = TryOnServer(pipe, height=MG.H, width=MG.W, max_batch=1, seed=r.seed, garment_cache_bytes=0,
                          output_type="latent", presets={name: _preset(name)})
        srv.submit(r)
        srv.run()
    return pipe._last_latents.clone()


@pytest.mark.parametrize("name", PRESETS)
def test_each_preset_against_batch_mode(tiny_modules, name, monkeypatch):
    """A request of each preset in a mixed server against TryOnServer(max_batch=1) with that preset, gated by batch
    mode's own spread between batch 1 and batch 2 on the same loop inputs and noises (test_continuous_gpu.py)."""
    from idm_vton_b200.denoise import TryOnDenoiser
    other = "ddpm" if name != "ddpm" else "dpmpp"
    k = PRESETS.index(name)
    _, lat, _ = _drive(_server(tiny_modules, [name, other], slots=2),
                       [([_req(tiny_modules, 10, other)], 1), ([_req(tiny_modules, k, name)], 0)])
    rec = []
    ref = _batch_mode(tiny_modules, name, _req(tiny_modules, k, name), monkeypatch, rec)
    ref2 = _batch_mode(tiny_modules, name, _req(tiny_modules, k + 1, name), monkeypatch, rec)
    a, b = rec
    den = TryOnDenoiser(tiny_modules["net_t"].engine(), tiny_modules["net_g"].engine())
    den.prepare(*_pair_inputs(a["inp"], b["inp"]).values(), **a["kw"])
    den.set_step_tables(a["scheduler"], a["timesteps"], eta=a["eta"])
    for i, (na, nb) in enumerate(zip(a["noises"], b["noises"])):
        den.step(i, None if na is None else torch.cat([na, nb]))
    spread = max(_err(den.latents[0:1], ref), _err(den.latents[1:2], ref2))
    bound = _bound(spread)
    err, mutant = _err(lat[1], ref), _err(lat[1], ref2)
    _report(case=f"preset {name} vs batch mode", err=err, bit_identical=bool(torch.equal(lat[1], ref)),
            batch2_vs_batch1=spread, bound=bound, other_request=mutant)
    assert err <= bound and mutant >= 10 * bound, (name, err, bound, mutant)


def test_pool_single_slot_equals_batch_mode_per_preset(tiny_modules, monkeypatch):
    """Pool mode at slots = 1 with all presets: every request the bits of TryOnServer(max_batch=1) with its preset."""
    reqs = lambda: [_req(tiny_modules, k, n) for k, n in enumerate(PRESETS)]  # noqa: E731
    _, lat, _ = _drive(_server(tiny_modules, PRESETS, slots=1, pages=1), [(reqs(), 0)])
    exact = {}
    for k, r in enumerate(reqs()):
        ref = _batch_mode(tiny_modules, r.sampling, r, monkeypatch, [])
        exact[r.sampling] = bool(torch.equal(lat[k], ref[0]))              # ref: the batch of one [1,4,h,w]
    _report(case="pool presets slots=1 vs TryOnServer(max_batch=1)", bit_identical=exact)
    assert all(exact.values()), exact


def test_pool_pages_are_shared_by_timesteps(tiny_modules):
    """DDPM 4 and DDPM 4 with rescale have the same timesteps: one page for garment A (one fill, one hit). DPM-Solver++
    3 has others: a page of its own. Results are the same bits on a miss, a hit and after an eviction."""
    srv = _server(tiny_modules, ["ddpm", "rescale"], slots=2, pages=2)
    _drive(srv, [([_req(tiny_modules, 0, "ddpm", "A"), _req(tiny_modules, 1, "rescale", "A")], 0)])
    assert srv.stats["garment_page_fills"] == 1 and srv.stats["garment_page_hits"] == 1
    srv = _server(tiny_modules, ["ddpm", "dpmpp"], slots=2, pages=2)
    _drive(srv, [([_req(tiny_modules, 0, "ddpm", "A"), _req(tiny_modules, 1, "dpmpp", "A")], 0)])
    assert srv.stats["garment_page_fills"] == 2 and srv.stats["garment_page_hits"] == 0 and len(srv.page_of) == 2
    # miss, then hit, then a miss after the page was evicted: the same bits for the same request
    t = lambda: _req(tiny_modules, 3, "dpmpp", "A")  # noqa: E731
    _, alone, _ = _drive(_server(tiny_modules, ["ddpm", "dpmpp"], slots=2, pages=2), [([t()], 0)])
    srv = _server(tiny_modules, ["ddpm", "dpmpp"], slots=2, pages=2)
    _, lat, _ = _drive(srv, [([_req(tiny_modules, 4, "dpmpp", "A")], 0), ([t()], 0),            # hit
                             ([_req(tiny_modules, 5, "ddpm", "B"), _req(tiny_modules, 6, "dpmpp", "C")], 0),
                             ([t()], 0)])                                                       # evicted: refilled
    assert srv.stats["garment_page_hits"] >= 1 and srv.stats["garment_page_evictions"] >= 1, srv.stats
    assert torch.equal(lat[1], alone[0]) and torch.equal(lat[4], alone[0])


# ------------------------------------------------------------------------------------------------
# SDXL width
# ------------------------------------------------------------------------------------------------
def test_fullsize_mixed_slots_against_batch_mode():
    """SDXL-width UNets (random weights), 2 slots: a DDPM request (3 steps) and a DPM-Solver++ request (2 steps) in one
    mixed-kind step, each against the batch-mode denoiser on that request alone, gated by batch mode's own spread
    between batch 1 and batch 2 under each scheduler."""
    from test_fullsize_gpu import _forward_inputs
    from oracle.make_golden_solvers import make_scheduler
    from idm_vton_b200 import unet as U
    from idm_vton_b200.denoise import SlotDenoiser, TryOnDenoiser, step_plan
    from idm_vton_b200.engine import SDXL_GARMENT, SDXL_TRYON, UNetEngine
    from idm_vton_b200.scheduler import DDPMScheduler
    eng_t = UNetEngine(SDXL_TRYON, U.random_state_dict(SDXL_TRYON, seed=11, device="cuda"), "tryon")
    eng_g = UNetEngine(SDXL_GARMENT, U.random_state_dict(SDXL_GARMENT, seed=22, device="cuda"), "garment")
    h, w = 128, 96
    ddpm, dpm = DDPMScheduler(), make_scheduler("dpmpp_2m")
    ddpm.set_timesteps(30)
    dpm.set_timesteps(30)
    runs = [(ddpm, ddpm.timesteps[:3]), (dpm, dpm.timesteps[:2])]
    inps = [_forward_inputs(SDXL_TRYON, SDXL_GARMENT, 1, h, w, seed=s) for s in (3, 4)]
    g = torch.Generator(device="cuda").manual_seed(5)
    noises = [[torch.randn(1, 4, h, w, generator=g, device="cuda").half() for _ in range(3)] for _ in inps]
    noises[1] = [None, None]                                        # DPM-Solver++ applies no noise

    def batch_mode(inp, nz, sch, ts):
        den = TryOnDenoiser(eng_t, eng_g)
        den.prepare(**inp, guidance_scale=2.0)
        den.set_step_tables(sch, ts)
        for i in range(len(ts)):
            den.step(i, nz[i])
        return den.latents.clone()

    refs = [batch_mode(inp, nz, *run) for inp, nz, run in zip(inps, noises, runs)]
    spread = 0.0
    for j, (sch, ts) in enumerate(runs):                            # both requests as one batch, each scheduler
        nz = [None if n is None else torch.cat([n, n]) for n in noises[j]]
        pair = batch_mode(_pair_inputs(inps[j], inps[1 - j]), nz, sch, ts)
        spread = max(spread, _err(pair[0:1], refs[j]))
    den = SlotDenoiser(eng_t, eng_g, 2)
    den.configure_presets([step_plan(sch, ts, 2.0) for sch, ts in runs], h, w)

    def admit(s, inp):
        den.admit(s, latents=inp["latents"], mask=inp["mask"], masked_image_latents=inp["masked_image_latents"],
                  pose_latents=inp["pose_latents"], cloth_latents=inp["cloth_latents"], prompt_embeds=inp["prompt_embeds"],
                  add_text_embeds=inp["add_text_embeds"], add_time_ids=inp["add_time_ids"],
                  image_embeds=inp["image_embeds"], text_embeds_cloth=inp["text_embeds_cloth"])
    admit(0, inps[0])
    den.step([(0, 0), None], {0: noises[0][0]})
    admit(1, inps[1])
    den.step([(0, 1), (1, 0)], {0: noises[0][1]})
    den.step([(0, 2), (1, 1)], {0: noises[0][2]})
    out0, out1 = den.latents[0:1].clone(), den.latents[1:2].clone()
    errs = [_err(out0, refs[0]), _err(out1, refs[1])]
    mutant = min(_err(out0, refs[1]), _err(out1, refs[0]))
    bound = _bound(spread)
    _report(case="fullsize mixed S=2", errs=errs, batch2_vs_batch1=spread, bound=bound, other_request=mutant)
    assert max(errs) <= bound and mutant >= 10 * bound, (errs, bound, mutant)
