"""Continuous batching without a GPU: the slot manager of serving.ContinuousTryOnServer on a stand-in denoiser, the
per-slot table gather of denoise.SlotDenoiser, the per-request RNG draw order against the pipeline's own __call__ for a
batch of one, the new C-ABI entry points (declared, exported, argument checks) and every refusal."""
import ctypes
import os
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROWS_SYMBOLS = ("b200vton_cfg_ddpm_step_rows", "b200vton_cfg_solver_step_rows", "b200vton_nchw_to_nhwc_scaled_rows")


def _req(gid, ticket_value=0.0, cloth=True, size=32, seed=None):
    from idm_vton_b200.serving import TryOnRequest
    z = torch.zeros
    return TryOnRequest(garment_id=gid, image=z(3, size, size) + ticket_value, mask_image=z(1, size, size),
                        pose_img=z(3, size, size), prompt_embeds=z(77, 8), negative_prompt_embeds=z(77, 8),
                        pooled_prompt_embeds=z(4), negative_pooled_prompt_embeds=z(4),
                        cloth=z(3, size, size) if cloth else None, ip_adapter_image=z(3, 224, 224) if cloth else None,
                        text_embeds_cloth=z(77, 8) if cloth else None, seed=seed)


# ------------------------------------------------------------------------------------------------------------------
# the slot manager
# ------------------------------------------------------------------------------------------------------------------
class _FakeDen:
    """Stand-in SlotDenoiser: latents[s] = the admitted request's ticket, +1 per step for occupied slots."""

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


def _fake_server(S=2, T=3):
    from idm_vton_b200.serving import ContinuousTryOnServer

    class Srv(ContinuousTryOnServer):
        def _configure(self):
            self.den, self.T, self._configured = _FakeDen(S, T), T, True

        def _garment(self, req, device, dtype):
            self.stats["garments_encoded"] += req.garment_id not in self.garments
            self.garments[req.garment_id] = dict(latents=None, image_embeds=None, text_embeds_cloth=None)
            return self.garments[req.garment_id]

        def _prepare_request(self, req, gen):
            return dict(latents=torch.tensor(float(req.ticket)))

        def _decode(self, latents):
            return latents * 10

    pipe = types.SimpleNamespace(vae_scale_factor=8, _execution_device=torch.device("cpu"),
                                 unet=types.SimpleNamespace(dtype=torch.float32))
    return Srv(pipe, height=32, width=32, slots=S, num_inference_steps=T, seed=1)


def test_slot_manager_admits_steps_retires_and_refills():
    srv = _fake_server(S=2, T=3)
    t = [srv.submit(_req("A")), srv.submit(_req("B")), srv.submit(_req("A", cloth=False)), srv.submit(_req("C"))]
    assert t == [0, 1, 2, 3] and srv.pending() == 4
    out1 = srv.step()                                  # tickets 0, 1 into slots 0, 1
    assert out1 == {} and srv.den.log[:3] == [("admit", 0, 0), ("admit", 1, 1), ("step", [0, 0])]
    assert [e["req"].ticket for e in srv.slots] == [0, 1]
    srv.step()
    out3 = srv.step()                                  # both finish after T = 3 steps, decoded together
    assert sorted(out3) == [0, 1]
    assert all(torch.equal(out3[k], torch.full((4, 2, 2), (k + 3) * 10.0)) for k in out3)
    assert srv.slots == [None, None] and ("release", 0) in srv.den.log and ("release", 1) in srv.den.log
    srv.den.log.clear()
    srv.step()                                         # refilled before the next step, lowest slot first, ticket order
    assert srv.den.log == [("admit", 0, 2), ("admit", 1, 3), ("step", [0, 0])]


def test_per_slot_step_indices_and_results_by_ticket():
    srv = _fake_server(S=3, T=3)
    out = {}
    srv.submit(_req("A"))
    out.update(srv.step())
    srv.submit(_req("B"))
    srv.submit(_req("C"))
    out.update(srv.step())                             # joins beside a request at step 1
    steps = [e for e in srv.den.log if e[0] == "step"]
    assert steps == [("step", [0, None, None]), ("step", [1, 0, 0])]
    srv.submit(_req("D"))
    out.update(srv.step())                             # ticket 0 finishes here; ticket 3 waits for a free slot
    assert sorted(out) == [0] and srv.den.log[-2:] == [("step", [2, 1, 1]), ("release", 0)]
    out.update(srv.step())                             # ticket 3 takes slot 0; tickets 1 and 2 finish
    assert srv.den.log[-4:] == [("admit", 0, 3), ("step", [0, 2, 2]), ("release", 1), ("release", 2)]
    assert sorted(out) == [0, 1, 2]
    out.update(srv.run())
    assert sorted(out) == [0, 1, 2, 3]
    assert all(torch.equal(v, torch.full((4, 2, 2), (k + 3) * 10.0)) for k, v in out.items())
    assert srv.stats["images"] == 4 and srv.stats["garments_encoded"] == 4


def test_submit_refusals():
    from idm_vton_b200.serving import ContinuousTryOnServer
    srv = ContinuousTryOnServer(types.SimpleNamespace(vae_scale_factor=8), height=32, width=32, slots=2)
    with pytest.raises(ValueError, match="is new"):
        srv.submit(_req("A", cloth=False))
    with pytest.raises(ValueError, match="latent size"):
        srv.submit(_req("A", size=40))                 # a 40x40 cloth is 5x5 latents, the server's persons 4x4
    srv.submit(_req("A"))
    srv.submit(_req("A", cloth=False))                 # known garment now
    assert srv.pending() == 2


# ------------------------------------------------------------------------------------------------------------------
# the per-slot gather and the idle rows
# ------------------------------------------------------------------------------------------------------------------
def _schedulers():
    from oracle.make_golden_solvers import make_scheduler
    from idm_vton_b200.scheduler import DDPMScheduler
    return {"ddpm": (DDPMScheduler(), 0.0), "ddim": (make_scheduler("ddim_eta1"), 1.0),
            "euler": (make_scheduler("euler_leading"), 0.0), "dpmpp": (make_scheduler("dpmpp_2m"), 0.0)}


def _slot_denoiser(S, symbols=ROWS_SYMBOLS):
    from idm_vton_b200.denoise import SlotDenoiser
    L = types.SimpleNamespace(has_symbol=lambda n: n in symbols)
    eng = types.SimpleNamespace(L=L, device=torch.device("cpu"))
    return SlotDenoiser(eng, eng, S)


def _r16(x):
    return x.to(torch.float16).to(torch.float32)


def _step_restated(kind, row, x, g):
    """The rows kernels' update on one sample (rounding points of elementwise.cu), noise and x0_prev zero."""
    gs, a, b, c, d, e, f, k = (float(v) for v in row)
    if kind == "ddpm":
        x0 = _r16(_r16(x - _r16(a * g)) * b)
        return _r16(_r16(c * x0) + _r16(d * x))
    if kind == "ddim":
        x0 = _r16(_r16(x - _r16(a * g)) * b)
        return _r16(_r16(d * x0) + _r16(e * g))
    if kind == "euler":
        x0 = x - _r16(a * g)
        return _r16(x + (x - x0) * b * e)
    x0 = _r16(_r16(x - _r16(a * g)) * b)
    return _r16((c * x + _r16(d * x0)) + _r16(0.5 * d * _r16(k * x0)))


@pytest.mark.parametrize("kind", ["ddpm", "ddim", "euler", "dpmpp"])
def test_gathered_rows_equal_the_tables_and_idle_rows_are_identity(kind):
    from idm_vton_b200.denoise import identity_step_row, solver_step_tables
    sch, eta = _schedulers()[kind]
    sch.set_timesteps(5)
    den = _slot_denoiser(3)
    den.configure(sch, sch.timesteps, 4, 4, guidance_scale=2.0, do_cfg=True, eta=eta)
    _, coefs, scales, draws, _ = solver_step_tables(sch, sch.timesteps, eta)
    assert den.T == 5 and den.step_draws == draws
    assert den.latents.shape == (3, 4, 4, 4) and den.x_t.shape == (6, 4, 4, 64) and den.x_g.shape == (3, 4, 4, 64)
    steps = [3, None, 0]
    den.gather(steps)
    ts = [float(t) for t in sch.timesteps]
    for s, i in enumerate(steps):
        want = identity_step_row(kind) if i is None else [2.0, *coefs[i]] + [0.0] * (8 - 1 - len(coefs[i]))
        assert den.coef[s].tolist() == torch.tensor(want, dtype=torch.float32).tolist()
        want_t = 0.0 if i is None else float(torch.tensor(ts[i], dtype=torch.float32))
        assert den.t_g[s].item() == want_t and den.t_t[s].item() == want_t and den.t_t[3 + s].item() == want_t
        if kind == "euler":
            assert den.scale[s].item() == (1.0 if i is None else float(torch.tensor(scales[i], dtype=torch.float32)))
    # the idle row leaves any finite fp16 latents unchanged, whatever the finite eps
    g = torch.Generator().manual_seed(0)
    x, eps = _r16(torch.randn(4, 8, 8, generator=g) * 3), _r16(torch.randn(4, 8, 8, generator=g) * 2)
    assert torch.equal(_step_restated(kind, den.coef[1], x, eps), x)
    assert torch.equal(_step_restated(kind, den.coef[1], torch.zeros_like(x), eps), torch.zeros_like(x))


def test_slot_denoiser_refusals():
    from idm_vton_b200.scheduler import DDPMScheduler
    sch = DDPMScheduler()
    sch.set_timesteps(4)
    with pytest.raises(NotImplementedError, match="guidance_rescale"):
        _slot_denoiser(2).configure(sch, sch.timesteps, 4, 4, guidance_rescale=0.7)
    with pytest.raises(NotImplementedError, match="b200vton_cfg_ddpm_step_rows"):
        _slot_denoiser(2, symbols=()).configure(sch, sch.timesteps, 4, 4)
    eu = _schedulers()["euler"][0]
    eu.set_timesteps(4)
    with pytest.raises(NotImplementedError, match="b200vton_nchw_to_nhwc_scaled_rows"):
        _slot_denoiser(2, symbols=ROWS_SYMBOLS[:2]).configure(eu, eu.timesteps, 4, 4)
    with pytest.raises(RuntimeError, match="before any admission"):
        den = _slot_denoiser(2)
        den.configure(sch, sch.timesteps, 4, 4)
        den.step([None, None])


def test_library_without_the_symbols_refuses_in_the_bindings():
    """lib.py binds the per-slot kernels only when the library exports them; the wrappers name the missing symbol."""
    from idm_vton_b200 import lib
    lib.load()
    present = set(lib._present)
    try:
        lib._present.clear()
        for fn, args in ((lib.cfg_ddpm_step_rows, (None, None, None, None)),
                         (lib.cfg_solver_step_rows, (None, None, None, None, "ddim"))):
            with pytest.raises(NotImplementedError, match="_step_rows"):
                fn(*args)
        with pytest.raises(NotImplementedError, match="b200vton_nchw_to_nhwc_scaled_rows"):
            lib.nchw_to_nhwc_scaled_rows(torch.zeros(1, 4, 2, 2, dtype=torch.float16),
                                         torch.zeros(2, 2, 2, 8, dtype=torch.float16), torch.ones(1))
    finally:
        lib._present.update(present)


# ------------------------------------------------------------------------------------------------------------------
# the C ABI
# ------------------------------------------------------------------------------------------------------------------
def test_rows_symbols_declared_exported_and_validated():
    from idm_vton_b200 import build, lib
    header = open(os.path.join(ROOT, "include", "b200vton.h")).read()
    so = ctypes.CDLL(build.build())
    for name in ROWS_SYMBOLS:
        assert f"int {name}(" in header and hasattr(so, name) and name in lib.OPTIONAL_SIGNATURES
    raw = lib.load()
    assert raw.b200vton_version() == lib.ABI_VERSION == 109
    assert all(lib.has_symbol(n) for n in ROWS_SYMBOLS)
    n0 = lib.launch_count()
    ddpm, solver, scat = (getattr(raw, n) for n in ROWS_SYMBOLS)
    # null pointers
    assert ddpm(None, 16, 1, 4, 4, 4, 64, None, 256, 8, 1, 64, None) == 1
    assert solver(64, 16, 1, 4, 4, 4, 64, None, None, None, 8, 0, 1, 64, None) == 1
    assert scat(None, 1, 4, 4, 4, 64, 2, 64, 0, 256, None) == 1
    assert scat(64, 1, 4, 4, 4, 64, 2, 64, 0, None, None) == 1
    # a stride shorter than the kind's coefficients (0 is allowed: one row for every sample)
    assert ddpm(64, 16, 1, 4, 4, 4, 64, None, 256, 5, 1, 64, None) == 1
    assert b"coef_stride" in raw.b200vton_last_error()
    assert solver(64, 16, 1, 4, 4, 4, 64, None, None, 256, 7, 0, 1, 64, None) == 1
    assert solver(64, 16, 1, 4, 4, 4, 64, None, None, 256, -8, 1, 1, 64, None) == 1
    # misalignment
    assert ddpm(64, 16, 1, 4, 4, 4, 65, None, 256, 8, 1, 64, None) == 1
    assert ddpm(64, 16, 1, 4, 4, 4, 64, None, 258, 8, 1, 64, None) == 1
    assert b"aligned" in raw.b200vton_last_error()
    assert solver(64, 16, 1, 4, 4, 4, 64, None, None, 254, 8, 1, 1, 64, None) == 1
    assert scat(64, 1, 4, 4, 4, 64, 2, 64, 0, 258, None) == 1
    assert scat(65, 1, 4, 4, 4, 64, 2, 64, 0, 256, None) == 1
    # the solver's own checks still apply: DPM-Solver++ without its state, an unknown kind
    assert solver(64, 16, 1, 4, 4, 4, 64, None, None, 256, 8, 2, 1, 64, None) == 1
    assert solver(64, 16, 1, 4, 4, 4, 64, None, None, 256, 8, 3, 1, 64, None) == 1
    assert lib.launch_count() == n0


# ------------------------------------------------------------------------------------------------------------------
# the per-request RNG draws against the pipeline's own __call__ at batch 1
# ------------------------------------------------------------------------------------------------------------------
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


def _record_randn(log, gens):
    real = torch.randn

    def randn(*a, generator=None, **kw):
        shape = tuple(a[0]) if a and isinstance(a[0], (tuple, list, torch.Size)) else tuple(a)
        log.append((shape, gens.get(id(generator), "global" if generator is None else "other")))
        return real(*a, generator=generator, **kw)
    return randn


@pytest.mark.parametrize("kind", ["ddpm", "euler"])
def test_request_draws_equal_the_pipelines_at_batch_one(monkeypatch, kind):
    """The same request through the pipeline's __call__ at batch 1 (as TryOnServer runs it, with its seed) and through
    ContinuousTryOnServer: the same random draws in the same order from the same generators, and the same loop inputs."""
    from idm_vton_b200 import serving
    from idm_vton_b200.denoise import solver_step_tables
    sch = _schedulers()[kind][0]
    steps, seed = 3, 7
    req = _req("A", seed=seed)
    g = torch.Generator().manual_seed(3)
    for name in ("image", "pose_img", "cloth"):
        setattr(req, name, torch.rand(3, 32, 32, generator=g))
    req.mask_image = (torch.rand(1, 32, 32, generator=g) > 0.5).float()
    req.prompt_embeds, req.negative_prompt_embeds = torch.randn(77, 8, generator=g), torch.randn(77, 8, generator=g)
    req.pooled_prompt_embeds, req.negative_pooled_prompt_embeds = torch.randn(4, generator=g), torch.randn(4, generator=g)
    req.ip_adapter_image = torch.rand(3, 8, 8, generator=g)

    # -- the pipeline, as TryOnServer.step calls it for one request
    pipe, eng_t, eng_g = _cpu_pipe(sch)
    seen = {}

    class PipeDen:
        tryon, garment = eng_t, eng_g

        def prepare(self, latents, mask, masked, pose, cloth, pe, ate, ati, ie, tec, **kw):
            seen.update(latents=latents.clone(), mask=mask[:1], masked=masked[:1], pose=pose[:1], pe=pe, ate=ate, ati=ati,
                        ie=ie)
            self.latents = latents

        def set_step_tables(self, scheduler, timesteps, garment_keys=None, cache=None, eta=0.0):
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
             generator=gen, strength=1.0, pose_img=req.pose_img[None], text_embeds_cloth=garment["text_embeds_cloth"],
             cloth=garment["latents"], mask_image=req.mask_image[None], image=req.image[None], height=32, width=32,
             ip_adapter_image=garment["ip_adapter_image"], guidance_scale=2.0, output_type="latent")
    monkeypatch.undo()

    # -- the continuous server
    pipe2, _, _ = _cpu_pipe(_schedulers()[kind][0])
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

    class Srv(serving.ContinuousTryOnServer):
        def _make_denoiser(self):
            return SrvDen()

        def _admit(self):
            real = torch.Generator

            def make(device):                  # label the request's generator for the record
                gg = real(device)
                labels[id(gg)] = "request"
                return gg
            with monkeypatch.context() as m:
                m.setattr(torch, "Generator", make)
                super()._admit()

    labels = {}
    srv = Srv(pipe2, height=32, width=32, slots=1, num_inference_steps=steps, guidance_scale=2.0, seed=seed,
              output_type="latent")
    srv.submit(req)
    srv._garment(req, "cpu", torch.float32)          # the garment's own sample: its own generator, once per garment
    log_s = []
    monkeypatch.setattr(torch, "randn", _record_randn(log_s, labels))
    out = srv.run()
    monkeypatch.undo()
    n_step = sum(solver_step_tables(pipe2.scheduler, srv.timesteps)[3])
    assert log_p == log_s
    assert log_p[:3] == [((1, 4, 16, 16), "request"), ((1, 4, 16, 16), "request"), ((1, 4, 16, 16), "global")]
    assert log_p[3:] == [((1, 4, 16, 16), "request")] * n_step and n_step == steps
    assert list(out) == [0]
    for k_p, k_s in (("latents", "latents"), ("mask", "mask"), ("masked", "masked_image_latents"),
                     ("pose", "pose_latents"), ("pe", "prompt_embeds"), ("ate", "add_text_embeds"),
                     ("ati", "add_time_ids"), ("ie", "image_embeds")):
        assert torch.equal(seen[k_p], admitted[k_s]), k_p
