"""FreeU on the engine (b200vton_freeu_nhwc, UNetEngine.freeu, enable_freeu on the try-on UNet and the pipeline, both
servers), against float64 and against the reference's own modules (tests/golden/freeu_ref.pt).

  * kernel: the filtered skip against fourier_filter in float64 on the fp16 input, max|d| / max|ref| <= 2^-10, at least
    4x closer than each mutant (tests/helpers/freeu_cases.py); the scaled half of hidden bit-identical to
    fp16(float(h) * b), the other half untouched; repeated launches, graph replay and the batch do not change a bit;
  * B2: the tiny try-on module with enable_freeu against the reference UNet with enable_freeu;
  * full size: SDXL width, B = 2, 128x96, t = 967, under DESIGN.md section 3's gate against ref16 / ref32 with FreeU;
  * B1: pipe.enable_freeu at config 1 against the reference pipeline, and the switches' bits;
  * servers: TryOnServer honours pipe.enable_freeu; ContinuousTryOnServer keeps a request's bits alone and beside
    others with FreeU on, refuses a change in flight and takes one while idle.
"""
import importlib.util
import json
import os

import pytest
import torch

from test_continuous_gpu import _drive, _request, _server
from test_continuous_pool_gpu import _pool_server
from test_fullsize_gpu import _cast, _engine_step, _forward_inputs, _gate, _oracle_step, full  # noqa: F401
from test_schedule_gpu import _make_pipe, _run_recorded

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "freeu_ref.pt")
SDXL = (0.9, 0.2, 1.3, 1.4)          # (s1, s2, b1, b2)


def load_cases():
    spec = importlib.util.spec_from_file_location("freeu_cases", os.path.join(ROOT, "tests", "helpers", "freeu_cases.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


FC = load_cases()


def _err(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return (a - b).abs().max().item() / max(1.0, b.abs().max().item())


def _report(**kw):
    print("FREEU " + json.dumps(kw))


def _values(case):
    return tuple(case[k] for k in ("s1", "s2", "b1", "b2"))


# ------------------------------------------------------------------------------------------------------------------
# the kernel
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", range(len(FC.SHAPES)), ids=[c[0] for c in FC.SHAPES])
def test_kernel_vs_float64(k):
    from idm_vton_b200 import lib as L
    name, B, H, W, Ch, Cs = FC.SHAPES[k]
    hidden, skip = FC.make_inputs(B, H, W, Ch, Cs, seed=k)
    ref = FC.truth(skip, FC.S_VALUE)
    h_dev, s_dev = hidden.cuda(), skip.cuda()
    out = torch.empty_like(s_dev)
    L.freeu(h_dev, s_dev, FC.B_VALUE, FC.S_VALUE, out=out)
    torch.cuda.synchronize()
    assert torch.equal(s_dev.cpu(), skip)                                     # out of place: skip is only read
    e = FC.rel(out.cpu(), ref)
    c = Ch // 2
    assert torch.equal(h_dev[..., :c].cpu(), FC.hidden_truth(hidden, FC.B_VALUE)[..., :c])
    assert torch.equal(h_dev[..., c:].cpu(), hidden[..., c:])
    mut = {m: FC.rel(fn(skip, FC.S_VALUE), ref) for m, fn in FC.SKIP_MUTANTS.items() if FC.distinct(m, H, W)}
    _report(case=name, shape=[B, H, W, Ch, Cs], err=e, gate=FC.TOL, mutants=mut)
    assert e <= FC.TOL, (name, e)
    for m, d in mut.items():
        assert d >= FC.MUTANT_FACTOR * max(e, 2.0 ** -24), (name, m, d, e)
    # in place gives the same bits
    h2, s2 = hidden.cuda(), skip.cuda()
    L.freeu(h2, s2, FC.B_VALUE, FC.S_VALUE)
    assert torch.equal(s2, out) and torch.equal(h2, h_dev)


def test_kernel_is_deterministic_graph_capturable_and_batch_independent():
    from idm_vton_b200 import lib as L
    hidden, skip = FC.make_inputs(4, 32, 24, 1280, 640, seed=77)
    h0, s0 = hidden.cuda(), skip.cuda()
    outs = []
    for _ in range(3):
        h = h0.clone()
        o = torch.empty_like(s0)
        L.freeu(h, s0, 1.3, 0.2, out=o)
        outs.append((h, o))
    assert all(torch.equal(outs[0][0], h) and torch.equal(outs[0][1], o) for h, o in outs[1:])
    # graph replay == eager
    hg, og = h0.clone(), torch.empty_like(s0)
    L.freeu(hg.clone(), s0, 1.3, 0.2, out=og)               # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        L.freeu(hg, s0, 1.3, 0.2, out=og)
    hg.copy_(h0)
    og.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(hg, outs[0][0]) and torch.equal(og, outs[0][1])
    # a sample's bits do not depend on the batch around it
    h1, o1 = h0[2:3].clone(), torch.empty_like(s0[2:3])
    L.freeu(h1, s0[2:3].contiguous(), 1.3, 0.2, out=o1)
    assert torch.equal(h1, outs[0][0][2:3]) and torch.equal(o1, outs[0][1][2:3])


def test_kernel_rejects_bad_arguments():
    from idm_vton_b200 import lib as L
    h = torch.zeros(1, 4, 4, 16, dtype=torch.float16, device="cuda")
    with pytest.raises(ValueError, match="same B, H, W"):
        L.freeu(h, torch.zeros(1, 4, 5, 16, dtype=torch.float16, device="cuda"), 1.3, 0.2)
    with pytest.raises(RuntimeError, match="multiples of 8"):
        L.freeu(h, torch.zeros(1, 4, 4, 12, dtype=torch.float16, device="cuda"), 1.3, 0.2)
    with pytest.raises(TypeError):
        L.freeu(h.float(), torch.zeros(1, 4, 4, 16, dtype=torch.float16, device="cuda"), 1.3, 0.2)
    with pytest.raises(ValueError, match="contiguous"):
        L.freeu(h, torch.zeros(1, 4, 4, 32, dtype=torch.float16, device="cuda")[..., :16], 1.3, 0.2)


# ------------------------------------------------------------------------------------------------------------------
# B2: the try-on module
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tiny():
    from oracle import unet_ref as R
    from idm_vton_b200 import unet as U
    cfg_t, cfg_g = R.tiny_config("tryon"), R.tiny_config("garment")
    sd_t, sd_g = R.make_state_dict(cfg_t, seed=11), R.make_state_dict(cfg_g, seed=22)
    net_t = U.UNet2DConditionModel(cfg_t, sd_t).to("cuda", torch.float16)
    net_g = U.UNet2DConditionModelGarment(cfg_g, sd_g).to("cuda", torch.float16)
    return dict(R=R, cfg_t=cfg_t, cfg_g=cfg_g, sd_t=sd_t, sd_g=sd_g, net_t=net_t, net_g=net_g)


def test_unet_module_with_freeu_vs_reference_golden(tiny):
    """The module seam called as the reference pipeline calls it, with enable_freeu, against the reference UNet with
    enable_freeu (fp32), at the B2 gate of tests/test_seams_gpu.py; s1 = 0 and disable_freeu give the plain bits."""
    from oracle.make_golden import synth_inputs
    g = torch.load(GOLDEN)
    u = g["unet"]
    x = synth_inputs(tiny["cfg_t"], tiny["cfg_g"], u["B"], u["h"], u["w"])
    net_t, net_g = tiny["net_t"], tiny["net_g"]
    dev, f16 = "cuda", torch.float16
    _, feats = net_g(x["cloth"].to(dev, f16), x["timestep"], x["text_embeds_cloth"].to(dev, f16), return_dict=False)
    fc = [torch.cat([torch.zeros_like(d), d]) for d in feats]
    img = net_t.encoder_hid_proj(x["clip_tokens"].to(dev, f16))
    added = {"text_embeds": x["text_embeds"].to(dev, f16), "time_ids": x["time_ids"].to(dev), "image_embeds": img}

    def run():
        return net_t(x["sample"].to(dev, f16), x["timestep"], encoder_hidden_states=x["prompt_embeds"].to(dev, f16),
                     added_cond_kwargs=added, return_dict=False, garment_features=fc)[0]
    off = run()
    errs = {"off": _err(off, u["noise_pred"]["off"])}
    try:
        for name, case in g["cases"].items():
            net_t.enable_freeu(**case)
            out = run()
            errs[name] = _err(out, u["noise_pred"][name])
            if name == "s1_zero":
                assert torch.equal(out, off)
            else:
                assert _err(u["noise_pred"][name], u["noise_pred"]["off"]) > 10 * 8e-3
    finally:
        net_t.disable_freeu()
    assert torch.equal(run(), off)
    _report(case="B2 module vs reference golden", errs=errs)
    assert max(errs.values()) < 8e-3, errs


def test_garment_module_refuses_freeu(tiny):
    with pytest.raises(NotImplementedError, match="garment"):
        tiny["net_g"].enable_freeu(*SDXL)


# ------------------------------------------------------------------------------------------------------------------
# full size
# ------------------------------------------------------------------------------------------------------------------
def test_fullsize_freeu_vs_oracle(full):  # noqa: F811
    """SDXL width, B = 2, 128x96, t = 967, SDXL FreeU values: engine vs ref32 <= ref16 vs ref32 + 2.5e-4 (and vs ref16
    where ref16 is within 1e-3 of ref32). The FreeU effect on noise_pred is at least 10x that bound, and a stage-swap
    mutant (stage 0 run with b2 / s2, stage 1 with b1 / s1) lies outside it."""
    from oracle import freeu_ref as FR
    R = full["R"]
    B, h, w, t = 2, 128, 96, 967
    inp = _forward_inputs(full["cfg_t"], full["cfg_g"], B, h, w, seed=9)
    eng = full["eng_t"]
    _, eps_off = _engine_step(full, inp, t, B, h, w)
    eng.freeu = SDXL
    try:
        _, eps = _engine_step(full, inp, t, B, h, w)
    finally:
        eng.freeu = None
    torch.cuda.synchronize()
    with torch.no_grad():
        with FR.enabled(full["sd_t32"], full["cfg_t"], SDXL):
            _, e32 = _oracle_step(R, full["sd_t32"], full["sd_g32"], full["cfg_t"], full["cfg_g"], inp, t)
        with FR.enabled(full["sd_t"], full["cfg_t"], SDXL), torch.autocast("cuda", dtype=torch.float16):
            _, e16 = _oracle_step(R, full["sd_t"], full["sd_g"], full["cfg_t"], full["cfg_g"], _cast(inp, torch.float16), t)
        _, off32 = _oracle_step(R, full["sd_t32"], full["sd_g32"], full["cfg_t"], full["cfg_g"], inp, t)
        with FR.enabled(full["sd_t32"], full["cfg_t"], SDXL, stage_of={0: 1, 1: 0}):
            _, swap32 = _oracle_step(R, full["sd_t32"], full["sd_g32"], full["cfg_t"], full["cfg_g"], inp, t)
    d_eng32, d_ref32, d_eng16 = _err(eps, e32), _err(e16, e32), _err(eps, e16)
    bound = d_ref32 + 2.5e-4
    effect, swap, eng_effect = _err(e32, off32), _err(swap32, e32), _err(eps, eps_off)
    _report(case=f"fullsize B={B} {h}x{w} t={t} FreeU {SDXL}", eng_vs_32=d_eng32, ref16_vs_32=d_ref32,
            eng_vs_ref16=d_eng16, bound=bound, effect_ref32=effect, effect_engine=eng_effect, stage_swap=swap)
    _gate("noise_pred with FreeU", d_eng32, d_ref32, d_eng16)
    assert effect >= 10 * bound, (effect, bound)
    assert swap > bound and _err(eps, swap32) > bound, (swap, bound)


# ------------------------------------------------------------------------------------------------------------------
# B1: the pipeline
# ------------------------------------------------------------------------------------------------------------------
def _call_kwargs(tiny):
    from oracle import make_golden_pipeline as MG
    dev, f16 = "cuda", torch.float16
    inp = {k: (v.to(dev, f16) if k not in ("image", "mask_image") else v.to(dev))
           for k, v in MG.make_call_inputs(tiny["cfg_t"]).items()}
    gen = torch.Generator().manual_seed(42)
    return MG.call_kwargs(inp, gen), gen


def _latents(pipe, tiny):
    kw, gen = _call_kwargs(tiny)
    return torch.stack([l for _, l in _run_recorded(pipe, kw, gen)["latents"]])


def test_pipeline_enable_freeu_vs_reference_golden(tiny):
    """pipe.enable_freeu at the SDXL values, __call__ at config 1: (ii) the engine's loop equals the oracle loop with
    FreeU on the pipeline's own loop inputs and noises, per step, at the gate of the plain B1 test; (iii) end to end
    against the reference pipeline's latents with enable_freeu, at that test's loose gate."""
    from oracle import freeu_ref as FR
    from oracle import loop_ref as LR
    from oracle import make_golden_pipeline as MG
    p = torch.load(GOLDEN)["pipeline"]
    freeu = _values(p["freeu"])
    pipe = _make_pipe(tiny)
    try:
        pipe.enable_freeu(*freeu)
        kw, gen = _call_kwargs(tiny)
        rec = _run_recorded(pipe, kw, gen)
    finally:
        pipe.disable_freeu()
    assert [t for t, _ in rec["latents"]] == p["timesteps"].tolist()
    dev = "cuda"
    sd_t32 = {k: v.half().float().to(dev) for k, v in tiny["sd_t"].items()}
    sd_g32 = {k: v.half().float().to(dev) for k, v in tiny["sd_g"].items()}
    li = {n: v.to(dev) for n, v in rec["inputs"].items()}
    steps = len(rec["latents"])
    e_loop = []
    with torch.no_grad(), FR.enabled(sd_t32, tiny["cfg_t"], freeu):
        for n in range(1, steps + 1):
            ref = LR.denoise_loop(sd_t32, tiny["cfg_t"], sd_g32, tiny["cfg_g"], li, steps, guidance_scale=MG.GUIDANCE,
                                  noises=rec["noises"], max_steps=n)
            e_loop.append(_err(rec["latents"][n - 1][1], ref))
    e_e2e = [_err(l, r) for (_, l), r in zip(rec["latents"], p["latents_per_step"])]
    _report(case="B1 pipeline with FreeU", loop_vs_oracle=e_loop, e2e_vs_reference=e_e2e)
    assert max(e_loop) < 4e-3
    assert max(e_e2e) < 5e-2


def test_pipeline_freeu_switches_give_the_right_bits(tiny):
    """disable_freeu gives the bits of a pipeline that never enabled it; enable, change the values, call gives the bits
    of a fresh pipeline with those values (no stale captured step); s1 = 0 gives the bits of FreeU off."""
    fresh = _make_pipe(tiny)
    plain = _latents(fresh, tiny)
    pipe = _make_pipe(tiny)
    try:
        pipe.enable_freeu(*SDXL)
        on = _latents(pipe, tiny)
        pipe.enable_freeu(s1=0.6, s2=0.5, b1=1.1, b2=1.2)
        changed = _latents(pipe, tiny)
        pipe.disable_freeu()
        off = _latents(pipe, tiny)
        pipe.enable_freeu(s1=0.0, s2=0.2, b1=1.3, b2=1.4)
        zero = _latents(pipe, tiny)
        other = _make_pipe(tiny)
        other.enable_freeu(s1=0.6, s2=0.5, b1=1.1, b2=1.2)
        changed_fresh = _latents(other, tiny)
        other.disable_freeu()
    finally:
        pipe.disable_freeu()
    assert not torch.equal(on, plain) and not torch.equal(changed, on)
    assert torch.equal(off, plain) and torch.equal(zero, plain) and torch.equal(changed, changed_fresh)


# ------------------------------------------------------------------------------------------------------------------
# servers
# ------------------------------------------------------------------------------------------------------------------
def test_tryon_server_honours_pipe_enable_freeu(tiny, monkeypatch):
    """TryOnServer goes through pipe(...): with pipe.enable_freeu its latents change, and they are the bits of a fresh
    denoiser with FreeU on the loop inputs and noises the server's run handed to its denoiser."""
    from oracle import make_golden_pipeline as MG
    from idm_vton_b200.denoise import TryOnDenoiser
    from idm_vton_b200.serving import TryOnServer
    names = ("latents", "mask", "masked_image_latents", "pose_latents", "cloth_latents", "prompt_embeds",
             "add_text_embeds", "add_time_ids", "image_embeds", "text_embeds_cloth")
    rec = {}
    real_prepare, real_tables, real_step = TryOnDenoiser.prepare, TryOnDenoiser.set_step_tables, TryOnDenoiser.step

    def prepare(self, *a, **kw):
        rec.update(inp=[v.clone() for v in a], kw=kw, noises=[])
        return real_prepare(self, *a, **kw)

    def set_step_tables(self, scheduler, timesteps, **kw):
        rec.update(scheduler=scheduler, timesteps=timesteps, tkw=kw)
        return real_tables(self, scheduler, timesteps, **kw)

    def step(self, i, noise=None, use_graph=True):
        rec["noises"].append(None if noise is None else noise.clone())
        return real_step(self, i, noise, use_graph=use_graph)

    def serve(freeu):
        pipe = _make_pipe(tiny)
        if freeu:
            pipe.enable_freeu(*freeu)
        try:
            srv = TryOnServer(pipe, height=MG.H, width=MG.W, num_inference_steps=4, guidance_scale=2.0, max_batch=1,
                              seed=7, garment_cache_bytes=0, output_type="latent")
            srv.submit(_request(tiny, 40, "A"))
            srv.run()
            return pipe._last_latents.clone()
        finally:
            pipe.disable_freeu()
    plain = serve(None)
    monkeypatch.setattr(TryOnDenoiser, "prepare", prepare)
    monkeypatch.setattr(TryOnDenoiser, "set_step_tables", set_step_tables)
    monkeypatch.setattr(TryOnDenoiser, "step", step)
    on = serve(SDXL)
    monkeypatch.undo()
    tiny["net_t"].enable_freeu(*SDXL)
    try:
        den = TryOnDenoiser(tiny["net_t"].engine(), tiny["net_g"].engine())
        den.prepare(*rec["inp"], **rec["kw"])
        den.set_step_tables(rec["scheduler"], rec["timesteps"], **rec["tkw"])
        for i, n in enumerate(rec["noises"]):
            den.step(i, n)
        replay = den.latents.clone()
    finally:
        tiny["net_t"].disable_freeu()
    assert not torch.equal(on, plain)
    assert torch.equal(on, replay)


@pytest.mark.parametrize("mode", ["default", "pool"])
def test_continuous_server_freeu_request_bits_alone_and_beside_others(tiny, mode):
    """With FreeU on, a request's final latents are the same bits alone and beside requests at other phases with other
    garments, in default and pool mode; FreeU changes them."""
    def make():
        return _server(tiny) if mode == "default" else _pool_server(tiny, 3)
    t = lambda: _request(tiny, 40, "A")  # noqa: E731
    x = lambda: _request(tiny, 41, "B")  # noqa: E731
    y = lambda: _request(tiny, 42, "C")  # noqa: E731
    _, lat_off, _ = _drive(make(), [([t()], 0)])
    tiny["net_t"].enable_freeu(*SDXL)
    try:
        _, lat_a, _ = _drive(make(), [([t()], 0)])
        _, lat_b, _ = _drive(make(), [([x()], 2), ([y()], 1), ([t()], 0)])
    finally:
        tiny["net_t"].disable_freeu()
    assert torch.equal(lat_b[2], lat_a[0]) and not torch.equal(lat_a[0], lat_off[0])


def test_continuous_server_freeu_change_in_flight_raises_and_idle_change_applies(tiny):
    srv = _server(tiny)
    try:
        srv.submit(_request(tiny, 40, "A"))
        srv.step()
        srv.pipe.enable_freeu(*SDXL)
        with pytest.raises(RuntimeError, match="FreeU"):
            srv.step()
        srv.pipe.disable_freeu()
        while srv.pending():
            srv.step()
        # idle: the change takes effect at the next admission
        srv.pipe.enable_freeu(*SDXL)
        _, lat, _ = _drive(srv, [([_request(tiny, 40, "A")], 0)])
        fresh = _server(tiny)
        _, lat_fresh, _ = _drive(fresh, [([_request(tiny, 40, "A")], 0)])
    finally:
        srv.pipe.disable_freeu()
    assert torch.equal(lat[1], lat_fresh[0])
