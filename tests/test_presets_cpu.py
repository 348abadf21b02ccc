"""Sampling presets without a GPU: the mixed tables of SlotDenoiser.configure_presets (rows, timesteps, scales, kinds,
base offsets, pool rows), the servers' preset handling (page keys, legacy construction, refusals before any launch),
a strength < 1 request's RNG draws against the pipeline's own __call__ at batch 1, and the new C-ABI entry point."""
import ctypes
import os
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.abspath(__file__)).rsplit(os.sep, 1)[0]
MIXED = "b200vton_cfg_step_mixed_rows"
ROWS_SYMBOLS = ("b200vton_cfg_ddpm_step_rows", "b200vton_cfg_solver_step_rows", "b200vton_nchw_to_nhwc_scaled_rows",
                "b200vton_attention_rows", MIXED)


class _Blk:
    def __init__(self, c):
        self.c = c


def _engine(symbols=ROWS_SYMBOLS):
    L = types.SimpleNamespace(has_symbol=lambda n: n in symbols)
    return types.SimpleNamespace(L=L, device=torch.device("cpu"), ch=(8, 16),
                                 blocks=lambda: [_Blk(16), _Blk(16), _Blk(8)])


def _schedulers():
    from oracle.make_golden_solvers import make_scheduler
    from idm_vton_b200.scheduler import DDPMScheduler
    return {"ddpm": (DDPMScheduler(), 0.0), "ddim": (make_scheduler("ddim_eta1"), 1.0),
            "euler": (make_scheduler("euler_leading"), 0.0), "dpmpp": (make_scheduler("dpmpp_2m"), 0.0)}


def _plans():
    """DDPM 5 with rescale, Euler 3, DPM-Solver++ 4, DDIM eta 1 at 2: four kinds, four step counts."""
    from idm_vton_b200.denoise import step_plan
    out = []
    for kind, n, phi in (("ddpm", 5, 0.7), ("euler", 3, 0.0), ("dpmpp", 4, 0.0), ("ddim", 2, 0.0)):
        sch, eta = _schedulers()[kind]
        sch.set_timesteps(n)
        out.append(step_plan(sch, sch.timesteps, 2.0 + n, phi, eta))
    return out


def test_gathered_rows_are_each_plans_rows_and_idle_is_identity():
    from idm_vton_b200.denoise import MIXED_KIND_CODES, SlotDenoiser, identity_step_row
    plans = _plans()
    den = SlotDenoiser(_engine(), _engine(), 4)
    den.configure_presets(plans, 4, 4)
    assert den.kind == "mixed" and den.base == [0, 5, 8, 12] and den.idle == 14 and den.T_page == 5
    assert den.x0_prev.shape == (4, 4, 4, 4) and den.kinds.dtype == torch.int32
    steps = [(0, 4), (2, 3), None, (3, 1)]
    den.gather(steps)
    for s, e in enumerate(steps):
        if e is None:
            row, t, scale, kind = torch.tensor(identity_step_row("ddpm")), 0.0, 1.0, "ddpm"
        else:
            p = plans[e[0]]
            row, t, kind = p.coef_table[e[1]], p.t_table[e[1]].item(), p.kind
            scale = 1.0 if p.scale_table is None else p.scale_table[e[1]].item()
        assert den.coef[s].tolist() == row.tolist(), s
        assert den.t_g[s].item() == t and den.t_t[s].item() == t and den.t_t[4 + s].item() == t
        assert den.scale[s].item() == scale and den.kinds[s].item() == MIXED_KIND_CODES[kind]
    assert den.coef[0, 6].item() == pytest.approx(0.7)                     # the rescale phi of the DDPM plan
    den.gather([(1, 2), (1, 0), (0, 0), (2, 0)])                           # Euler: its own input scales
    assert den.scale[0].item() == plans[1].scale_table[2].item() != 1.0
    for bad in ([(1, 3), None, None, None], [(4, 0), None, None, None], [(0, -1), None, None, None]):
        with pytest.raises(ValueError, match="outside the configured plans"):
            den.gather(bad)


def test_pool_rows_are_page_times_t_max_plus_step():
    from idm_vton_b200.denoise import SlotDenoiser
    den = SlotDenoiser(_engine(), _engine(), 3, pages=4)
    den.configure_presets(_plans(), 4, 4)
    assert [tuple(p.shape) for p in den.pool] == [(20, 4, 32), (20, 4, 32), (20, 16, 16)]    # 4 pages of T_max = 5
    den.page = [3, None, 1]
    den.gather([(2, 3), None, (3, 1)])
    assert den.rows.tolist() == [3 * 5 + 3, -1, 5 + 1]
    with pytest.raises(ValueError, match="needs the timesteps"):
        den.fill_page(0, torch.zeros(1, 4, 4, 4), torch.zeros(1, 77, 8))
    with pytest.raises(ValueError, match="do not fit"):
        den.fill_page(0, torch.zeros(1, 4, 4, 4), torch.zeros(1, 77, 8), torch.zeros(6))


def test_configure_is_unchanged_after_presets():
    """configure() after configure_presets() is the per-kind denoiser again, refusals included."""
    from idm_vton_b200.denoise import SlotDenoiser
    sch = _schedulers()["ddpm"][0]
    sch.set_timesteps(4)
    den = SlotDenoiser(_engine(), _engine(), 2)
    den.configure_presets(_plans(), 4, 4)
    den.configure(sch, sch.timesteps, 4, 4)
    assert den.kind == "ddpm" and den.kinds is None and den.plans is None and den.x0_prev is None and den.T == 4
    with pytest.raises(NotImplementedError, match="guidance_rescale"):
        den.configure(sch, sch.timesteps, 4, 4, guidance_rescale=0.7)


# ------------------------------------------------------------------------------------------------------------------
# the servers
# ------------------------------------------------------------------------------------------------------------------
def _req(gid, sampling=None, seed=None, size=32):
    from idm_vton_b200.serving import TryOnRequest
    z = torch.zeros
    return TryOnRequest(garment_id=gid, image=z(3, size, size), mask_image=z(1, size, size), pose_img=z(3, size, size),
                        prompt_embeds=z(77, 8), negative_prompt_embeds=z(77, 8), pooled_prompt_embeds=z(4),
                        negative_pooled_prompt_embeds=z(4), cloth=z(3, size, size), ip_adapter_image=z(3, 224, 224),
                        text_embeds_cloth=z(77, 8), seed=seed, sampling=sampling)


class _ImageEncoder(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.ones(1))

    def forward(self, x, output_hidden_states=True):
        h = x.flatten(1)[:, :64].reshape(x.shape[0], 4, 16) * self.w
        return types.SimpleNamespace(hidden_states=[h, h])


def _cpu_pipe(scheduler):
    from idm_vton_b200.pipeline import StableDiffusionXLInpaintPipeline as P
    from idm_vton_b200.vae import AutoencoderKL
    torch.manual_seed(0)
    vae = AutoencoderKL(block_out_channels=(32, 32), layers_per_block=1)
    eng_t, eng_g = object(), object()
    unet = types.SimpleNamespace(
        config=types.SimpleNamespace(time_cond_proj_dim=None, sample_size=16, in_channels=13, addition_time_embed_dim=2),
        device=torch.device("cpu"), dtype=torch.float32, engine=lambda: eng_t, encoder_hid_proj=lambda x: x * 2,
        add_embedding=types.SimpleNamespace(linear_1=types.SimpleNamespace(in_features=2 * 6 + 4)))
    enc = types.SimpleNamespace(engine=lambda: eng_g)
    return P(vae, None, None, None, None, unet, enc, scheduler, image_encoder=_ImageEncoder()), eng_t, eng_g


class _FakeDen:
    """Stand-in SlotDenoiser (as test_continuous_cpu.py's): latents[s] = the admitted request's ticket, +1 per step."""

    def __init__(self, S, T):
        self.S, self.T = S, T
        self.latents = torch.zeros(S, 4, 2, 2)
        self.step_draws, self.noise_applied = [False] * T, True
        self.log = []

    def admit(self, s, **kw):
        self.log.append(("admit", s, int(kw["latents"])))
        self.latents[s] = float(kw["latents"])

    def step(self, steps, noises=None, use_graph=True):
        self.log.append(("step", list(steps)))
        for s, i in enumerate(steps):
            if i is not None:
                self.latents[s] += 1
        return self.latents

    def release(self, s):
        self.log.append(("release", s))
        self.latents[s] = 0


def _server(presets, default=None, scheduler=None, slots=2, **kw):
    """A ContinuousTryOnServer on the CPU pipeline whose SlotDenoiser runs on a stand-in engine (no launch can happen)."""
    from idm_vton_b200.denoise import SlotDenoiser
    from idm_vton_b200.serving import ContinuousTryOnServer
    pipe, _, _ = _cpu_pipe(scheduler or _schedulers()["ddpm"][0])
    symbols = kw.pop("symbols", ROWS_SYMBOLS)
    pipe.unet.engine = lambda: _engine(symbols)                       # page sizes from the stand-in's blocks

    class Srv(ContinuousTryOnServer):
        def _make_denoiser(self, pages=None):
            return SlotDenoiser(_engine(symbols), _engine(symbols), self.S, pages=pages)
    return Srv(pipe, height=32, width=32, slots=slots, seed=1, presets=presets, default_preset=default, **kw)


def _p(kind="ddpm", n=3, **kw):
    from idm_vton_b200.serving import SamplingPreset
    return SamplingPreset(_schedulers()[kind][0], n, **kw)


def test_refusals_fire_before_any_launch():
    from idm_vton_b200 import lib
    lib.load()
    n0 = lib.launch_count()
    # rescale with a non-DDPM scheduler
    srv = _server({"a": _p("ddpm"), "b": _p("euler", guidance_rescale=0.5)}, "a")
    srv.submit(_req("A", "b"))
    with pytest.raises(NotImplementedError, match="guidance_rescale"):
        srv.step()
    # no-CFG beside CFG
    srv = _server({"a": _p("ddpm"), "b": _p("ddim", guidance_scale=1.0)}, "a")
    srv.submit(_req("A"))
    with pytest.raises(ValueError, match="guidance_scale <= 1"):
        srv.step()
    # a library without the mixed-kind step
    srv = _server({"a": _p("ddpm"), "b": _p("dpmpp", 4)}, "a", symbols=ROWS_SYMBOLS[:4])
    srv.submit(_req("A"))
    with pytest.raises(NotImplementedError, match=MIXED):
        srv.step()
    srv = _server({"a": _p("ddpm", guidance_rescale=0.3)}, symbols=ROWS_SYMBOLS[:4])
    srv.submit(_req("A"))
    with pytest.raises(NotImplementedError, match=MIXED):
        srv.step()
    # an unknown preset at submit; a default that is not a preset
    srv = _server({"a": _p("ddpm"), "b": _p("dpmpp", 4)}, "a")
    with pytest.raises(ValueError, match="sampling preset 'c'"):
        srv.submit(_req("A", "c"))
    with pytest.raises(ValueError, match="default_preset"):
        _server({"a": _p("ddpm"), "b": _p("dpmpp", 4)})
    assert lib.launch_count() == n0


def test_refusals_with_the_stand_in_denoiser():
    """The refusals of the mixed path need no denoiser: with the stand-in they fire before it is used."""
    from idm_vton_b200.serving import ContinuousTryOnServer
    pipe, _, _ = _cpu_pipe(_schedulers()["ddpm"][0])
    made = []

    class Srv(ContinuousTryOnServer):
        def _make_denoiser(self, pages=None):
            made.append(_FakeDen(self.S, 3))
            return made[-1]
    srv = Srv(pipe, height=32, width=32, slots=2, presets={"a": _p("ddpm"), "b": _p("dpmpp", guidance_rescale=0.2)},
              default_preset="a")
    srv.submit(_req("A"))
    with pytest.raises(NotImplementedError, match="guidance_rescale"):
        srv.step()
    assert made == []
    with pytest.raises(ValueError, match="unknown|sampling preset"):
        srv.submit(_req("A", "zzz"))


def test_mixed_server_tables_and_page_keys():
    """Two presets: one plan per preset from the pipeline's own timesteps (strength applied), a private scheduler per
    preset (pipe.scheduler untouched), T_max pages, and page keys (garment, the plan's timesteps)."""
    srv = _server({"q": _p("ddpm", 5), "f": _p("dpmpp", 4, strength=0.5)}, "q", garment_kv_bytes=0)
    srv.garment_kv_bytes = 3 * srv.page_bytes()
    before = srv.pipe.scheduler.timesteps
    srv._configure()
    assert srv.mixed and srv.den.kind == "mixed" and [p.T for p in srv.plans] == [5, 2] and srv.T == 5
    assert srv.pipe.scheduler.timesteps is before                                   # the pipeline's scheduler untouched
    assert srv._schedulers["q"] is not srv.presets["q"].scheduler
    assert srv.plans[1].t_table[:2].tolist() == srv._timesteps["f"].float().tolist()
    assert srv.page_bytes() == srv.page_bytes(5) and srv.den.T_page == 5
    filled = []
    srv.den.fill_page = lambda p, lat, txt, t_table=None: filled.append((p, t_table.tolist()))
    g = dict(latents=None, text_embeds_cloth=None)
    t_f = srv.plans[1].t_table[:2]
    p1 = srv._pin_page(("A", tuple(float(t) for t in t_f)), g, t_f)
    p2 = srv._pin_page(("A", tuple(float(t) for t in t_f)), g, t_f)
    assert p1 == p2 and filled == [(p1, t_f.tolist())] and srv.stats["garment_page_hits"] == 1
    assert list(srv.page_of) == [("A", tuple(t_f.tolist()))]


def test_legacy_construction_selects_the_per_kind_path():
    """presets=None: the same single plan as today's configure, the per-kind kernels, pages keyed by garment; one
    preset without rescale takes the same path."""
    from idm_vton_b200.denoise import step_plan
    from idm_vton_b200.serving import ContinuousTryOnServer, SamplingPreset
    for kind in ("ddpm", "euler"):
        pipe, _, _ = _cpu_pipe(_schedulers()[kind][0])

        class Srv(ContinuousTryOnServer):
            def _make_denoiser(self, pages=None):
                from idm_vton_b200.denoise import SlotDenoiser
                return SlotDenoiser(_engine(), _engine(), self.S, pages=pages)
        legacy = Srv(pipe, height=32, width=32, slots=2, num_inference_steps=4, guidance_scale=3.0)
        legacy._configure()
        want = step_plan(pipe.scheduler, pipe.scheduler.timesteps, 3.0)
        assert not legacy.mixed and legacy.den.kind == kind and legacy.den.plans is None and legacy.den.kinds is None
        assert torch.equal(legacy.den.coef_table, want.coef_table) and legacy.T == 4
        assert MIXED not in legacy.den._needs(legacy.den.kind)
        pipe2, _, _ = _cpu_pipe(_schedulers()[kind][0])
        one = Srv(pipe2, height=32, width=32, slots=2,
                  presets={"x": SamplingPreset(_schedulers()[kind][0], 4, guidance_scale=3.0)})
        one._configure()
        assert not one.mixed and one.den.kind == kind and torch.equal(one.den.coef_table, want.coef_table)


def test_tryon_server_batches_by_garment_and_preset():
    from idm_vton_b200.serving import TryOnServer
    calls = []

    class Pipe:
        scheduler = "pipe's"

        def __call__(self, **kw):
            calls.append((self.scheduler, kw["num_inference_steps"], kw["strength"], kw.get("eta"),
                          kw.get("guidance_rescale"), kw["prompt_embeds"].shape[0]))
            return (torch.zeros(kw["prompt_embeds"].shape[0], 3, 4, 4),)
    pipe = Pipe()
    pipe._execution_device, pipe.unet = torch.device("cpu"), types.SimpleNamespace(dtype=torch.float32)
    srv = TryOnServer(pipe, garment_cache_bytes=0, presets={"q": _p("ddpm", 5), "f": _p("ddim", 2, strength=0.5, eta=1.0,
                                                                                         guidance_rescale=0.0)},
                      default_preset="q")
    srv.garments["A"] = dict(latents=None, ip_adapter_image=None, text_embeds_cloth=None)
    for s in ("q", "f", None, "f"):
        srv.submit(_req("A", s))
    srv.run()
    assert [c[1:] for c in calls] == [(5, 1.0, None, None, 2), (2, 0.5, 1.0, None, 2)]
    assert type(calls[0][0]).__name__ == "DDPMScheduler" and type(calls[1][0]).__name__ == "DDIMScheduler"
    assert pipe.scheduler == "pipe's"                                   # restored after each call


def _record_randn(log, gens):
    real = torch.randn

    def randn(*a, generator=None, **kw):
        shape = tuple(a[0]) if a and isinstance(a[0], (tuple, list, torch.Size)) else tuple(a)
        log.append((shape, gens.get(id(generator), "global" if generator is None else "other")))
        return real(*a, generator=generator, **kw)
    return randn


def test_strength_request_draws_equal_the_pipelines_at_batch_one(monkeypatch):
    """A strength-0.6 request through the pipeline's __call__ at batch 1 and through a ContinuousTryOnServer preset:
    the same draws (the image's VAE sample, then the noise, ...) in the same order, and the same loop inputs."""
    from idm_vton_b200 import serving
    from idm_vton_b200.denoise import solver_step_tables
    from idm_vton_b200.serving import SamplingPreset
    steps, seed, strength = 5, 7, 0.6
    req = _req("A", "s", seed=seed)
    g = torch.Generator().manual_seed(3)
    for name in ("image", "pose_img", "cloth"):
        setattr(req, name, torch.rand(3, 32, 32, generator=g))
    req.mask_image = (torch.rand(1, 32, 32, generator=g) > 0.5).float()
    req.prompt_embeds, req.negative_prompt_embeds = torch.randn(77, 8, generator=g), torch.randn(77, 8, generator=g)
    req.pooled_prompt_embeds, req.negative_pooled_prompt_embeds = torch.randn(4, generator=g), torch.randn(4, generator=g)
    req.ip_adapter_image = torch.rand(3, 8, 8, generator=g)

    pipe, eng_t, eng_g = _cpu_pipe(_schedulers()["ddpm"][0])
    seen = {}

    class PipeDen:
        tryon, garment = eng_t, eng_g

        def prepare(self, latents, mask, masked, pose, cloth, pe, ate, ati, ie, tec, **kw):
            seen.update(latents=latents.clone(), masked=masked[:1], pose=pose[:1])
            self.latents = latents

        def set_step_tables(self, scheduler, timesteps, garment_keys=None, cache=None, eta=0.0):
            seen["timesteps"] = timesteps
            _, _, _, self.step_draws, self.noise_applied = solver_step_tables(scheduler, timesteps, eta)

        def step(self, i, noise=None, use_graph=True):
            return self.latents

    pipe._denoiser = PipeDen()
    garment = serving._encode_garment(pipe, req, seed, "cpu", torch.float32)
    gen = torch.Generator().manual_seed(seed)
    log_p = []
    monkeypatch.setattr(torch, "randn", _record_randn(log_p, {id(gen): "request"}))
    with serving._seeded_global_rng("cpu", seed):
        pipe(prompt_embeds=req.prompt_embeds[None], negative_prompt_embeds=req.negative_prompt_embeds[None],
             pooled_prompt_embeds=req.pooled_prompt_embeds[None],
             negative_pooled_prompt_embeds=req.negative_pooled_prompt_embeds[None], num_inference_steps=steps,
             generator=gen, strength=strength, pose_img=req.pose_img[None],
             text_embeds_cloth=garment["text_embeds_cloth"], cloth=garment["latents"], mask_image=req.mask_image[None],
             image=req.image[None], height=32, width=32, ip_adapter_image=garment["ip_adapter_image"],
             guidance_scale=2.0, output_type="latent")
    monkeypatch.undo()

    pipe2, _, _ = _cpu_pipe(_schedulers()["euler"][0])          # the preset's scheduler, not the pipeline's, is used
    admitted = {}

    class SrvDen:
        def configure(self, scheduler, timesteps, h, w, **kw):
            _, _, _, self.step_draws, self.noise_applied = solver_step_tables(scheduler, timesteps, kw["eta"])
            self.T = len(timesteps)
            self.latents = torch.zeros(1, 4, h, w)

        def admit(self, s, **kw):
            admitted.update(kw)

        def step(self, steps, noises=None, use_graph=True):
            return self.latents

        def release(self, s):
            pass

    labels = {}

    class Srv(serving.ContinuousTryOnServer):
        def _make_denoiser(self):
            return SrvDen()

        def _admit(self):
            real = torch.Generator

            def make(device):
                gg = real(device)
                labels[id(gg)] = "request"
                return gg
            with monkeypatch.context() as m:
                m.setattr(torch, "Generator", make)
                super()._admit()

    srv = Srv(pipe2, height=32, width=32, slots=1, seed=seed, output_type="latent",
              presets={"s": SamplingPreset(_schedulers()["ddpm"][0], steps, strength=strength)})
    srv.submit(req)
    srv._garment(req, "cpu", torch.float32)
    log_s = []
    monkeypatch.setattr(torch, "randn", _record_randn(log_s, labels))
    out = srv.run()
    monkeypatch.undo()
    assert srv.T == 3 and srv._timesteps["s"].tolist() == seen["timesteps"].tolist()
    assert log_p == log_s and len(log_p) == 4 + 3                       # image sample, noise, masked, pose; 3 steps
    assert log_p[:2] == [((1, 4, 16, 16), "request")] * 2 and log_p[3] == ((1, 4, 16, 16), "global")
    assert list(out) == [0]
    for k_p, k_s in (("latents", "latents"), ("masked", "masked_image_latents"), ("pose", "pose_latents")):
        assert torch.equal(seen[k_p], admitted[k_s]), k_p


# ------------------------------------------------------------------------------------------------------------------
# the C ABI
# ------------------------------------------------------------------------------------------------------------------
def test_mixed_symbol_declared_exported_and_validated():
    from test_fp8_cpu import _declared_args
    from idm_vton_b200 import build, lib
    header = open(os.path.join(ROOT, "include", "b200vton.h")).read()
    so = ctypes.CDLL(build.build())
    assert f"int {MIXED}(" in header and hasattr(so, MIXED)
    assert lib.OPTIONAL_SIGNATURES[MIXED] == _declared_args(header, MIXED)
    raw = lib.load()
    assert raw.b200vton_version() == lib.ABI_VERSION == 109 and lib.has_symbol(MIXED)
    fn = getattr(raw, MIXED)
    n0 = lib.launch_count()

    def call(eps=64, lat=64, x0p=64, coef=256, stride=8, kinds=512, out=64):
        return fn(eps, 16, 1, 4, 4, 4, lat, None, x0p, coef, stride, kinds, 1, out, None)
    for kw in (dict(eps=None), dict(lat=None), dict(x0p=None), dict(coef=None), dict(kinds=None), dict(out=None)):
        assert call(**kw) == 1, kw
    for stride in (1, 7, -8):
        assert call(stride=stride) == 1 and b"coef_stride" in raw.b200vton_last_error(), stride
    for kw in (dict(kinds=514), dict(coef=258), dict(x0p=65)):
        assert call(**kw) == 1 and b"aligned" in raw.b200vton_last_error(), kw
    assert lib.launch_count() == n0


def test_library_without_the_mixed_symbol_refuses_in_the_binding():
    from idm_vton_b200 import lib
    lib.load()
    present = set(lib._present)
    try:
        lib._present.discard(MIXED)
        with pytest.raises(NotImplementedError, match=MIXED):
            lib.cfg_step_mixed_rows(None, None, None, None, None, None)
    finally:
        lib._present.update(present)
