"""Continuous batching on the GPU:
  * the per-sample step kernels (b200vton_cfg_*_step_rows, b200vton_nchw_to_nhwc_scaled_rows) bit-identical to the
    single-row kernels launched per sample with that sample's coefficients, and to the single-row kernel on the whole
    batch when every row is equal;
  * serving.ContinuousTryOnServer (tiny config, as the other serving tests): a request's result does not depend on its
    neighbours, its slot or the arrival order; graph replay equals eager launches; each request against
    TryOnServer(max_batch=1) with its seed for DDPM, DDIM at eta 1, Euler and DPM-Solver++;
  * a short run at SDXL width (2 slots, 3 steps) against the batch-mode denoiser.
"""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

KINDS = ["ddpm", "ddim", "euler", "dpmpp"]
# Continuous vs batch mode runs the same arithmetic at other batch sizes (garment UNet at batch `slots` instead of 1 or
# the hoisted timestep chunk, try-on UNet at 2 * slots instead of 2), so fp16 results may differ by reordering
# (GroupNorm picks its split from the batch size): on an H100 0.9-2.3e-3 of the scale. Batch mode itself differs the
# same way between two batch sizes (1.3-2.3e-3 on the same inputs and noises), so
# each comparison measures that spread on the same requests and gates on it: continuous vs batch mode
# <= max(1e-3, 2 * spread) — two UNets change batch size here, and each contributes its own reordering. The spread itself
# must stay within SPREAD_CAP (4 fp16 ulps of the scale), so the bound cannot drift; a request compared with another
# request's batch-mode result lies at least 10x above the bound, as would any wrong coefficient row, timestep or garment.
SPREAD_CAP = 4 * 2.0 ** -10


def _bound(spread):
    assert spread <= SPREAD_CAP, f"batch mode's own batch-size spread {spread} exceeds {SPREAD_CAP}"
    return max(1e-3, 2 * spread)


def _err(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return (a - b).abs().max().item() / max(1.0, b.abs().max().item())


def _report(**kw):
    """Observed values, appended to $CONTINUOUS_REPORT when set (the PR quotes them)."""
    path = os.environ.get("CONTINUOUS_REPORT")
    if path:
        import json
        with open(path, "a") as f:
            f.write(json.dumps(kw) + "\n")


# ------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------
def _kernel_inputs(B, H, W, ldc, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    eps = (torch.randn(2 * B, H, W, ldc, generator=g, device="cuda") * 1.5).half()
    lat = (torch.randn(B, 4, H, W, generator=g, device="cuda") * 3).half()
    noise = torch.randn(B, 4, H, W, generator=g, device="cuda").half()
    x0p = torch.randn(B, 4, H, W, generator=g, device="cuda").half()
    return eps, lat, noise, x0p


def _rows(kind, B, seed):
    """B distinct coefficient rows in the ranges of real schedules (8 floats: the DDPM kernel reads the first 6)."""
    g = torch.Generator().manual_seed(seed)
    u = lambda lo, hi: float(lo + (hi - lo) * torch.rand(1, generator=g))  # noqa: E731
    rows = []
    for _ in range(B):
        if kind == "ddpm":
            rows.append([u(1, 7.5), u(0.1, 1), u(1, 14), u(0.01, 0.3), u(0.7, 1), u(0, 0.2), 0.0, 0.0])
        elif kind == "ddim":
            rows.append([u(1, 7.5), u(0.1, 1), u(1, 14), 0.0, u(0.1, 1), u(0, 0.9), u(0, 0.2), 0.0])
        elif kind == "euler":
            s = u(0.1, 14)
            rows.append([u(1, 7.5), s, 1 / s, 1.0, 0.0, -u(0.01, s), 0.0, 0.0])
        else:
            rows.append([u(1, 7.5), u(0.1, 14), u(1, 14), u(0.1, 1), u(0.1, 1), 0.0, 0.0, u(0, 2)])
    return torch.tensor(rows, dtype=torch.float32, device="cuda")


def _single(L, kind, eps, lat, noise, coef, x0p, cfg):
    if kind == "ddpm":
        return L.cfg_ddpm_step(eps, lat, noise, coef, do_cfg=cfg)
    return L.cfg_solver_step(eps, lat, noise if kind == "ddim" else None, coef, kind, x0_prev=x0p, do_cfg=cfg)


def _multi(L, kind, eps, lat, noise, coef, x0p, cfg):
    if kind == "ddpm":
        return L.cfg_ddpm_step_rows(eps, lat, noise, coef, do_cfg=cfg)
    return L.cfg_solver_step_rows(eps, lat, noise if kind == "ddim" else None, coef, kind, x0_prev=x0p, do_cfg=cfg)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("cfg", [True, False])
def test_rows_kernel_equals_per_sample_launches(kind, cfg):
    from idm_vton_b200 import lib as L
    B, H, W, ldc = 3, 12, 10, 16
    eps, lat, noise, x0p = _kernel_inputs(B, H, W, ldc, seed=7 + KINDS.index(kind))
    if not cfg:
        eps = eps[:B].contiguous()
    coef = _rows(kind, B, seed=3)
    state = x0p.clone()
    out = _multi(L, kind, eps, lat, noise, coef, state if kind == "dpmpp" else None, cfg)
    for b in range(B):
        rows = [b, B + b] if cfg else [b]
        st = x0p[b:b + 1].clone()
        ref = _single(L, kind, eps[rows].contiguous(), lat[b:b + 1].contiguous(), noise[b:b + 1].contiguous(),
                      coef[b].contiguous(), st if kind == "dpmpp" else None, cfg)
        assert torch.equal(out[b:b + 1], ref), (kind, b)
        if kind == "dpmpp":
            assert torch.equal(state[b:b + 1], st)
    # every row equal (and the stride-0 broadcast): the single-row kernel on the whole batch
    same = coef[1:2].repeat(B, 1).contiguous()
    st1, st2, st3 = x0p.clone(), x0p.clone(), x0p.clone()
    whole = _single(L, kind, eps, lat, noise, coef[1].contiguous(), st1 if kind == "dpmpp" else None, cfg)
    assert torch.equal(_multi(L, kind, eps, lat, noise, same, st2 if kind == "dpmpp" else None, cfg), whole)
    assert torch.equal(_multi(L, kind, eps, lat, noise, coef[1].contiguous(), st3 if kind == "dpmpp" else None, cfg), whole)
    if kind == "dpmpp":
        assert torch.equal(st1, st2) and torch.equal(st1, st3)


def test_scaled_scatter_rows_equals_per_sample_launches():
    from idm_vton_b200 import lib as L
    B, H, W, ldc = 3, 7, 9, 64
    x = (torch.randn(B, 4, H, W, device="cuda") * 14).half()
    scale = torch.tensor([0.07, 0.5, 0.9], dtype=torch.float32, device="cuda")
    dst = torch.full((2 * B, H, W, ldc), 7.0, dtype=torch.float16, device="cuda")
    L.nchw_to_nhwc_scaled_rows(x, dst, scale)
    for b in range(B):
        ref = torch.full((2, H, W, ldc), 7.0, dtype=torch.float16, device="cuda")
        L.nchw_to_nhwc_scaled(x[b:b + 1].contiguous(), ref, scale[b:b + 1])
        assert torch.equal(dst[b], ref[0]) and torch.equal(dst[B + b], ref[1])
    same = torch.full_like(dst, 7.0)
    L.nchw_to_nhwc_scaled_rows(x, same, scale[1:2].repeat(B).contiguous())
    whole = torch.full_like(dst, 7.0)
    L.nchw_to_nhwc_scaled(x, whole, scale[1:2])
    assert torch.equal(same, whole)


def test_rows_kernels_reject_bad_arguments():
    from idm_vton_b200 import lib as L
    eps, lat, noise, x0p = _kernel_inputs(2, 4, 4, 16, seed=1)
    n0 = L.launch_count()
    with pytest.raises(RuntimeError, match="code 1"):
        L.cfg_ddpm_step_rows(eps, lat, noise, torch.zeros(2, 5, device="cuda"))
    with pytest.raises(RuntimeError, match="code 1"):
        L.cfg_solver_step_rows(eps, lat, None, torch.zeros(2, 7, device="cuda"), "euler")
    with pytest.raises(RuntimeError, match="code 1"):
        L.cfg_solver_step_rows(eps, lat, None, torch.zeros(2, 8, device="cuda"), "dpmpp", x0_prev=None)
    assert L.launch_count() == n0


# ------------------------------------------------------------------------------------------------
# the server (tiny config)
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


def _scheduler(kind):
    from oracle.make_golden_solvers import make_scheduler
    from idm_vton_b200.scheduler import DDPMScheduler
    return {"ddpm": DDPMScheduler, "ddim": lambda: make_scheduler("ddim_eta1"),
            "euler": lambda: make_scheduler("euler_leading"), "dpmpp": lambda: make_scheduler("dpmpp_2m")}[kind]()


def _pipe(tiny, kind="ddpm"):
    from test_schedule_gpu import _make_pipe
    p = _make_pipe(tiny)
    p.scheduler = _scheduler(kind)
    return p


def _request(tiny, person_seed, garment, seed=7):
    from oracle import make_golden_pipeline as MG
    from idm_vton_b200.serving import TryOnRequest
    i = MG.make_call_inputs(tiny["cfg_t"], B=1, seed=person_seed)
    gi = MG.make_call_inputs(tiny["cfg_t"], B=1, seed={"A": 1001, "B": 1002, "C": 1003}[garment])
    return TryOnRequest(garment_id=garment, image=i["image"][0].cuda(), mask_image=i["mask_image"][0].cuda(),
                        pose_img=i["pose_img"][0], prompt_embeds=i["prompt_embeds"][0],
                        negative_prompt_embeds=i["negative_prompt_embeds"][0],
                        pooled_prompt_embeds=i["pooled_prompt_embeds"][0],
                        negative_pooled_prompt_embeds=i["negative_pooled_prompt_embeds"][0], cloth=gi["cloth"][0],
                        ip_adapter_image=gi["ip_adapter_image"][0], text_embeds_cloth=gi["text_embeds_cloth"][0],
                        seed=seed)


def _server(tiny, kind="ddpm", slots=3, steps=4, eta=0.0):
    from oracle import make_golden_pipeline as MG
    from idm_vton_b200.serving import ContinuousTryOnServer
    return ContinuousTryOnServer(_pipe(tiny, kind), height=MG.H, width=MG.W, slots=slots, num_inference_steps=steps,
                                 guidance_scale=2.0, seed=7, output_type="pt", eta=eta)


def _drive(srv, script, use_graph=True):
    """script: a list of (requests to submit, steps to run after submitting them); then runs to the end. Returns
    ({ticket: image}, {ticket: final latents}, {ticket: slot})."""
    out, lat, slot = {}, {}, {}
    for reqs, n in script:
        for r in reqs:
            srv.submit(r)
        for _ in range(n):
            out.update(srv.step(use_graph=use_graph))
            lat.update(srv.last_latents)
            slot.update({e["req"].ticket: s for s, e in enumerate(srv.slots) if e is not None})
    while srv.pending():
        out.update(srv.step(use_graph=use_graph))
        lat.update(srv.last_latents)
        slot.update({e["req"].ticket: s for s, e in enumerate(srv.slots) if e is not None})
    return out, lat, slot


def test_request_result_is_independent_of_neighbours_slot_and_order(tiny_modules):
    """At a fixed number of slots a request's image is the same bits alone, beside requests at other phases with other
    garments in another slot, and at another arrival order; its final latents also when it finishes beside others."""
    t = lambda: _request(tiny_modules, 40, "A")  # noqa: E731
    x = lambda: _request(tiny_modules, 41, "B")  # noqa: E731
    y = lambda: _request(tiny_modules, 42, "C")  # noqa: E731
    img_a, lat_a, slot_a = _drive(_server(tiny_modules), [([t()], 0)])
    # beside two requests at steps 2 and 1, with other garments, in slot 2
    img_b, lat_b, slot_b = _drive(_server(tiny_modules), [([x()], 2), ([y()], 1), ([t()], 0)])
    # another arrival order: admitted second, in slot 1, before a later request
    img_c, lat_c, slot_c = _drive(_server(tiny_modules), [([y()], 1), ([t()], 1), ([x()], 0)])
    # admitted with two others at once, finishing with them
    img_d, lat_d, _ = _drive(_server(tiny_modules), [([y(), t(), x()], 0)])
    assert slot_a[0] == 0 and slot_b[2] == 2 and slot_c[1] == 1
    assert torch.equal(lat_b[2], lat_a[0]) and torch.equal(lat_c[1], lat_a[0]) and torch.equal(lat_d[1], lat_a[0])
    assert torch.equal(img_b[2], img_a[0]) and torch.equal(img_c[1], img_a[0])
    assert not torch.equal(lat_b[0], lat_a[0])                      # the neighbours are different requests
    _report(case="composition", image_batch3_vs_alone_maxabs=(img_d[1] - img_a[0]).abs().max().item())


def test_graph_replay_equals_eager_over_admissions_and_retirements(tiny_modules):
    script = lambda: [([_request(tiny_modules, 41, "B")], 2), ([_request(tiny_modules, 42, "C")], 1),  # noqa: E731
                      ([_request(tiny_modules, 40, "A"), _request(tiny_modules, 43, "A")], 0)]
    for kind in ("ddpm", "dpmpp"):
        img_g, lat_g, _ = _drive(_server(tiny_modules, kind), script(), use_graph=True)
        img_e, lat_e, _ = _drive(_server(tiny_modules, kind), script(), use_graph=False)
        assert sorted(lat_g) == sorted(lat_e) == [0, 1, 2, 3]
        assert all(torch.equal(lat_g[k], lat_e[k]) and torch.equal(img_g[k], img_e[k]) for k in lat_g), kind


class _EtaPipe:
    """The pipeline with a fixed `eta` added to every call (TryOnServer passes none)."""

    def __init__(self, pipe, eta):
        self.__dict__["_p"], self.__dict__["_eta"] = pipe, eta

    def __getattr__(self, k):
        return getattr(self._p, k)

    def __setattr__(self, k, v):
        setattr(self._p, k, v)

    def __call__(self, **kw):
        return self._p(eta=self._eta, **kw)


PER_GARMENT = ("latents", "cloth_latents", "text_embeds_cloth")     # [B] rows; every other loop input has [2B]


def _pair_inputs(a, b):
    """Two batch-1 loop inputs as one batch of 2 ([uncond a, uncond b, cond a, cond b] rows)."""
    return {k: torch.cat([a[k], b[k]]) if k in PER_GARMENT else
            torch.cat([a[k][0:1], b[k][0:1], a[k][1:2], b[k][1:2]]) for k in a}


@pytest.mark.parametrize("kind", KINDS)
def test_each_request_against_batch_mode(tiny_modules, kind, monkeypatch):
    """Each request's final latents against TryOnServer(max_batch=1) with the request's seed. Not bit-identical in
    general: the UNets run at other batch sizes. Gated by batch mode's own difference between batch 1 and batch 2 on
    the same loop inputs and noises (_bound): the batch-1 runs' denoiser inputs are recorded and replayed as one batch
    of 2 (TryOnServer itself draws one noise tensor per batch, so its requests' noises depend on the batch)."""
    from oracle import make_golden_pipeline as MG
    from idm_vton_b200.denoise import TryOnDenoiser
    from idm_vton_b200.serving import TryOnServer
    eta = 1.0 if kind == "ddim" else 0.0
    steps = 4
    names = ("latents", "mask", "masked_image_latents", "pose_latents", "cloth_latents", "prompt_embeds",
             "add_text_embeds", "add_time_ids", "image_embeds", "text_embeds_cloth")
    reqs = lambda: [_request(tiny_modules, 50, "A"), _request(tiny_modules, 51, "B"),  # noqa: E731
                    _request(tiny_modules, 52, "A")]
    _, lat, _ = _drive(_server(tiny_modules, kind, slots=2, steps=steps, eta=eta), [(reqs()[:1], 1), (reqs()[1:], 0)])
    rec = []
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
    monkeypatch.setattr(TryOnDenoiser, "prepare", prepare)
    monkeypatch.setattr(TryOnDenoiser, "set_step_tables", set_step_tables)
    monkeypatch.setattr(TryOnDenoiser, "step", step)
    errs, exact, refs = [], [], []
    for k, r in enumerate(reqs()):
        pipe = _pipe(tiny_modules, kind)
        srv = TryOnServer(_EtaPipe(pipe, eta), height=MG.H, width=MG.W, num_inference_steps=steps, guidance_scale=2.0,
                          max_batch=1, seed=r.seed, garment_cache_bytes=0, output_type="latent")
        srv.submit(r)
        srv.run()
        refs.append(pipe._last_latents.clone())
        errs.append(_err(lat[k], refs[-1]))
        exact.append(bool(torch.equal(lat[k], refs[-1])))
    monkeypatch.undo()
    # batch mode's own spread across batch sizes: the recorded inputs of requests 0 and 1 as one batch of 2
    a, b = rec[0], rec[1]
    den = TryOnDenoiser(tiny_modules["net_t"].engine(), tiny_modules["net_g"].engine())
    den.prepare(*_pair_inputs(a["inp"], b["inp"]).values(), **a["kw"])
    den.set_step_tables(a["scheduler"], a["timesteps"], eta=a["eta"])
    for i, (na, nb) in enumerate(zip(a["noises"], b["noises"])):
        den.step(i, None if na is None else torch.cat([na, nb]))
    spread = max(_err(den.latents[0:1], refs[0]), _err(den.latents[1:2], refs[1]))
    mutant = _err(lat[0], refs[1])
    bound = _bound(spread)
    _report(case=f"vs batch mode {kind}", errs=errs, bit_identical=exact, batch2_vs_batch1=spread, bound=bound,
            other_request=mutant)
    assert max(errs) <= bound, (kind, errs, bound)
    assert mutant >= 10 * bound, (kind, mutant)


def test_refusals_on_the_engine(tiny_modules):
    srv = _server(tiny_modules)
    srv.guidance_rescale = 0.5
    srv.submit(_request(tiny_modules, 40, "A"))
    with pytest.raises(NotImplementedError, match="guidance_rescale"):
        srv.step()


# ------------------------------------------------------------------------------------------------
# SDXL width
# ------------------------------------------------------------------------------------------------
def test_fullsize_slots_against_batch_mode():
    """SDXL-width UNets (random weights), 2 slots, 3 DDPM steps: request 0 alone for one step, request 1 joins at its
    step 0; each request's latents against the batch-mode denoiser run on that request alone, gated by the batch-mode
    denoiser's own difference between running the two requests alone and together."""
    from test_fullsize_gpu import _forward_inputs
    from idm_vton_b200 import unet as U
    from idm_vton_b200.denoise import SlotDenoiser, TryOnDenoiser
    from idm_vton_b200.engine import SDXL_GARMENT, SDXL_TRYON, UNetEngine
    from idm_vton_b200.scheduler import DDPMScheduler
    eng_t = UNetEngine(SDXL_TRYON, U.random_state_dict(SDXL_TRYON, seed=11, device="cuda"), "tryon")
    eng_g = UNetEngine(SDXL_GARMENT, U.random_state_dict(SDXL_GARMENT, seed=22, device="cuda"), "garment")
    h, w, steps = 128, 96, 3
    sch = DDPMScheduler()
    sch.set_timesteps(30)
    ts = sch.timesteps[:steps]
    inps = [_forward_inputs(SDXL_TRYON, SDXL_GARMENT, 1, h, w, seed=s) for s in (3, 4)]
    g = torch.Generator(device="cuda").manual_seed(5)
    noises = [[torch.randn(1, 4, h, w, generator=g, device="cuda").half() for _ in range(steps)] for _ in inps]
    def batch_mode(inp, nz):
        den = TryOnDenoiser(eng_t, eng_g)
        den.prepare(**inp, guidance_scale=2.0)
        den.set_step_tables(sch, ts)
        for i in range(steps):
            den.step(i, nz[i])
        return den.latents.clone()

    refs = [batch_mode(inp, nz) for inp, nz in zip(inps, noises)]
    # batch mode's own spread: both requests as one batch of 2 ([uncond 0, uncond 1, cond 0, cond 1] rows)
    pair = batch_mode(_pair_inputs(inps[0], inps[1]), [torch.cat([noises[0][i], noises[1][i]]) for i in range(steps)])
    spread = max(_err(pair[0:1], refs[0]), _err(pair[1:2], refs[1]))
    den = SlotDenoiser(eng_t, eng_g, 2)
    den.configure(sch, ts, h, w, guidance_scale=2.0)

    def admit(s, inp):
        den.admit(s, latents=inp["latents"], mask=inp["mask"], masked_image_latents=inp["masked_image_latents"],
                  pose_latents=inp["pose_latents"], cloth_latents=inp["cloth_latents"], prompt_embeds=inp["prompt_embeds"],
                  add_text_embeds=inp["add_text_embeds"], add_time_ids=inp["add_time_ids"],
                  image_embeds=inp["image_embeds"], text_embeds_cloth=inp["text_embeds_cloth"])
    admit(0, inps[0])
    den.step([0, None], {0: noises[0][0]})
    admit(1, inps[1])
    den.step([1, 0], {0: noises[0][1], 1: noises[1][0]})
    den.step([2, 1], {0: noises[0][2], 1: noises[1][1]})
    out0 = den.latents[0:1].clone()
    den.step([None, 2], {1: noises[1][2]})
    out1 = den.latents[1:2].clone()
    errs = [_err(out0, refs[0]), _err(out1, refs[1])]
    mutant = _err(out0, refs[1])
    bound = _bound(spread)
    _report(case="fullsize S=2 3 steps", errs=errs, bit_identical=[bool(torch.equal(out0, refs[0])),
                                                                   bool(torch.equal(out1, refs[1]))],
            batch2_vs_batch1=spread, bound=bound, other_request=mutant)
    assert max(errs) <= bound and mutant >= 10 * bound, (errs, bound, mutant)
