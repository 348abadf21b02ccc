"""Parity of the engine (both UNets + the denoise loop) against the oracle (oracle/unet_ref.py, loop_ref.py).

Three yard-sticks, same seeded inputs / weights (fp16-rounded so every path sees identical values):
  * `ref32`  : oracle in fp32 on the GPU (TF32 off)            — the high-precision answer
  * `ref16`  : oracle under torch.autocast(fp16), fp16 weights — the reference's own rounding points (inference.py:339)
  * `golden` : outputs of the REFERENCE modules themselves (tests/golden/unet_tiny_ref.pt, made by oracle/make_golden.py)
Gate (north star: "fp16 outputs within 1e-3 of the reference diffusers path"): max|engine - ref16| <= 1e-3 * max(1,|ref|max)
per UNet forward where stated; and the engine must not be further from fp32 truth than 2x the reference's own fp16 path.
"""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "unet_tiny_ref.pt")


def _h(sd):
    return {k: v.half() for k, v in sd.items()}


def _to(d, device, dtype):
    return {k: (v.to(device=device, dtype=dtype) if torch.is_floating_point(v) else v.to(device)) for k, v in d.items()}


def _err(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return (a - b).abs().max().item() / max(1.0, b.abs().max().item())


@pytest.fixture(scope="module")
def tiny():
    from oracle import unet_ref as R
    from idm_vton_b200.engine import UNetEngine
    prev_tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)   # restored at teardown
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cfg_t, cfg_g = R.tiny_config("tryon"), R.tiny_config("garment")
    sd_t, sd_g = _h(R.make_state_dict(cfg_t, seed=11)), _h(R.make_state_dict(cfg_g, seed=22))
    eng_t = UNetEngine(cfg_t, sd_t, "tryon")
    eng_g = UNetEngine(cfg_g, sd_g, "garment")
    yield dict(R=R, cfg_t=cfg_t, cfg_g=cfg_g, sd_t=sd_t, sd_g=sd_g, eng_t=eng_t, eng_g=eng_g)
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev_tf32


def _engine_unets(env, x, B, h, w):
    """Runs garment + try-on engines on make_golden-style inputs; returns (features, eps NCHW)."""
    from idm_vton_b200 import lib as L
    from idm_vton_b200.engine import CIN_PAD
    eng_t, eng_g = env["eng_t"], env["eng_g"]
    dev = "cuda"
    t_dev = torch.tensor([float(x["timestep"])], device=dev)
    xg = torch.zeros(B, h, w, CIN_PAD, dtype=torch.float16, device=dev)
    L.nchw_to_nhwc(x["cloth"].half().to(dev).contiguous(), xg)
    ctx_g = eng_g.encode_context(x["text_embeds_cloth"].half().to(dev))
    feats = []
    eng_g.forward(xg, eng_g.time_embedding(t_dev, B), ctx_g, collect=feats)
    xt = torch.zeros(2 * B, h, w, CIN_PAD, dtype=torch.float16, device=dev)
    L.nchw_to_nhwc(x["sample"].half().to(dev).contiguous(), xt)
    ctx_t = eng_t.encode_context(x["prompt_embeds"].half().to(dev), x["image_embeds"].half().to(dev))
    aug = eng_t.aug_embedding(x["text_embeds"].half().to(dev), x["time_ids"].to(dev))
    eps = eng_t.forward(xt, eng_t.time_embedding(t_dev, 2 * B, aug), ctx_t, gfeats=feats, n_persons=B)
    return feats, L.nhwc_to_nchw(eps, 4)


def test_tiny_unets_vs_reference_golden(tiny):
    """Engine vs the outputs of the reference's own modules (golden fixture; CPU fp32)."""
    from oracle.make_golden import synth_inputs
    g = torch.load(GOLDEN)
    B, h, w = g["B"], g["h"], g["w"]
    x = synth_inputs(tiny["cfg_t"], tiny["cfg_g"], B, h, w)
    x["image_embeds"] = g["image_embeds"]
    feats, eps = _engine_unets(tiny, x, B, h, w)
    assert len(feats) == len(g["garment_feature_norms"])
    e0 = _err(feats[0], g["garment_feature_0"])
    e1 = _err(feats[-1], g["garment_feature_last"])
    ee = _err(eps, g["noise_pred"])
    print(f"golden: feat0 {e0:.2e} feat_last {e1:.2e} eps {ee:.2e}")
    # golden was produced with fp32 weights/inputs; the engine sees fp16-rounded weights -> allow fp16-level slack
    assert e0 < 4e-3 and e1 < 8e-3 and ee < 8e-3


@pytest.mark.parametrize("B,h,w", [(1, 16, 16), (2, 16, 24), (1, 8, 8)])
def test_tiny_unets_vs_oracle(tiny, B, h, w):
    from oracle.make_golden import synth_inputs
    R = tiny["R"]
    x = synth_inputs(tiny["cfg_t"], tiny["cfg_g"], B, h, w, seed=7)
    x = {k: (v.half().float() if torch.is_floating_point(v) else v) for k, v in x.items()}
    dev = "cuda"
    sd_t32, sd_g32 = _to(tiny["sd_t"], dev, torch.float32), _to(tiny["sd_g"], dev, torch.float32)
    sd_t16, sd_g16 = _to(tiny["sd_t"], dev, torch.float16), _to(tiny["sd_g"], dev, torch.float16)
    with torch.no_grad():
        x32 = _to(x, dev, torch.float32)
        img32 = R.resampler_forward(sd_t32, "encoder_hid_proj", tiny["cfg_t"]["resampler"], x32["clip_tokens"])
        img = img32.half().float()
        x["image_embeds"] = img.cpu()

        def run(sd_t, sd_g, xin):
            feats = R.unet_garment_forward(sd_g, tiny["cfg_g"], xin["cloth"], xin["timestep"], xin["text_embeds_cloth"])
            fc = [torch.cat([torch.zeros_like(d), d]) for d in feats]
            added = {"text_embeds": xin["text_embeds"], "time_ids": xin["time_ids"], "image_embeds": img.to(xin["sample"].dtype)}
            return feats, R.unet_tryon_forward(sd_t, tiny["cfg_t"], xin["sample"], xin["timestep"], xin["prompt_embeds"], added, fc)

        f32, e32 = run(sd_t32, sd_g32, x32)
        with torch.autocast("cuda", dtype=torch.float16):
            x16 = _to(x, dev, torch.float16)
            x16["time_ids"] = x32["time_ids"]
            f16, e16 = run(sd_t16, sd_g16, x16)
    feats, eps = _engine_unets(tiny, x, B, h, w)
    fe = max(_err(a, b) for a, b in zip(feats, f32))
    fe16 = max(_err(a, b) for a, b in zip(f16, f32))
    d_eng32, d_ref32, d_eng16 = _err(eps, e32), _err(e16, e32), _err(eps, e16)
    print(f"B={B} {h}x{w}: feats eng-32 {fe:.2e} (ref16-32 {fe16:.2e}); eps eng-32 {d_eng32:.2e} ref16-32 {d_ref32:.2e} eng-ref16 {d_eng16:.2e}")
    assert fe <= 2 * fe16 + 1e-3
    assert d_eng32 <= 2 * d_ref32 + 1e-3
    assert d_eng16 <= 2e-3


def test_tiny_loop_and_graph(tiny):
    """3-step denoise loop: CUDA-graph replay == eager launches (bit-exact), and both track the oracle loop."""
    from oracle import loop_ref as LR
    from idm_vton_b200.denoise import TryOnDenoiser
    from idm_vton_b200.scheduler import DDPMScheduler
    R = tiny["R"]
    B, h, w, steps = 2, 16, 16, 30
    inp = LR.synth_loop_inputs(tiny["cfg_t"], tiny["cfg_g"], B, h, w, seed=3)
    inp = {k: (v.half().float() if k != "add_time_ids" else v) for k, v in inp.items()}
    g = torch.Generator().manual_seed(5)
    noises = [torch.randn(B, 4, h, w, generator=g).half().float() for _ in range(3)]
    dev = "cuda"
    den = TryOnDenoiser(tiny["eng_t"], tiny["eng_g"])
    sch = DDPMScheduler()
    sch.set_timesteps(steps)

    def run_engine(use_graph):
        cuda_in = {k: v.to(dev) for k, v in inp.items()}
        den.prepare(**cuda_in, guidance_scale=2.0)
        den.set_step_tables(sch, sch.timesteps)
        for i in range(3):
            den.step(i, noises[i].half().to(dev), use_graph=use_graph)
        torch.cuda.synchronize()
        return den.latents.clone()

    lat_eager = run_engine(False)
    lat_graph = run_engine(True)
    assert torch.equal(lat_eager, lat_graph), "graph replay must be bit-identical to eager launches"
    sd_t32, sd_g32 = _to(tiny["sd_t"], dev, torch.float32), _to(tiny["sd_g"], dev, torch.float32)
    with torch.no_grad():
        ref = LR.denoise_loop(sd_t32, tiny["cfg_t"], sd_g32, tiny["cfg_g"], _to(inp, dev, torch.float32), steps,
                              noises=[n.to(dev) for n in noises], max_steps=3)
        with torch.autocast("cuda", dtype=torch.float16):
            i16 = _to(inp, dev, torch.float16)
            i16["add_time_ids"] = inp["add_time_ids"].to(dev)
            ref16 = LR.denoise_loop(_to(tiny["sd_t"], dev, torch.float16), tiny["cfg_t"],
                                    _to(tiny["sd_g"], dev, torch.float16), tiny["cfg_g"], i16, steps,
                                    noises=[n.half().to(dev) for n in noises], max_steps=3)
    d_eng, d_ref = _err(lat_graph, ref), _err(ref16, ref)
    print(f"loop 3 steps: engine-32 {d_eng:.2e}, ref16-32 {d_ref:.2e}, engine-ref16 {_err(lat_graph, ref16):.2e}")
    assert d_eng <= 2 * d_ref + 2e-3


def test_shared_garment_batch(tiny):
    """Config 3 shape: several persons share ONE garment (garment batch 1, K/V broadcast by index)."""
    from oracle import loop_ref as LR
    from idm_vton_b200.denoise import TryOnDenoiser
    from idm_vton_b200.scheduler import DDPMScheduler
    B, h, w = 3, 8, 8
    inp = LR.synth_loop_inputs(tiny["cfg_t"], tiny["cfg_g"], B, h, w, Bg=1, seed=9)
    inp = {k: (v.half().float() if k != "add_time_ids" else v) for k, v in inp.items()}
    dev = "cuda"
    den = TryOnDenoiser(tiny["eng_t"], tiny["eng_g"])
    sch = DDPMScheduler()
    sch.set_timesteps(30)
    den.prepare(**{k: v.to(dev) for k, v in inp.items()})
    den.set_step_tables(sch, sch.timesteps)
    noise = torch.zeros(B, 4, h, w)
    den.step(0, noise.half().to(dev), use_graph=False)
    with torch.no_grad():
        ref = LR.denoise_loop(_to(tiny["sd_t"], dev, torch.float32), tiny["cfg_t"], _to(tiny["sd_g"], dev, torch.float32),
                              tiny["cfg_g"], _to(inp, dev, torch.float32), 30, noises=[noise.to(dev)], max_steps=1)
    e = _err(den.latents, ref)
    print(f"shared garment: {e:.2e}")
    assert e < 4e-3


def test_hoisted_garment_pass_matches_stepwise(tiny):
    """Running all garment-UNet passes before the loop (batched over timesteps) gives the same latents as the
    reference's step-by-step order (same arithmetic per (step, garment); only GEMM tiling / GN chunking differ)."""
    from oracle import loop_ref as LR
    from idm_vton_b200.denoise import TryOnDenoiser
    from idm_vton_b200.scheduler import DDPMScheduler
    B, h, w = 2, 16, 16
    inp = LR.synth_loop_inputs(tiny["cfg_t"], tiny["cfg_g"], B, h, w, seed=21)
    inp = {k: (v.half().float() if k != "add_time_ids" else v) for k, v in inp.items()}
    dev = "cuda"
    sch = DDPMScheduler()
    sch.set_timesteps(30)
    outs = []
    for hoist in (False, True):
        den = TryOnDenoiser(tiny["eng_t"], tiny["eng_g"], hoist_garment=hoist, garment_chunk=7)
        den.prepare(**{k: v.to(dev) for k, v in inp.items()})
        den.set_step_tables(sch, sch.timesteps)
        for i in range(4):
            den.step(i, None, use_graph=hoist)
        torch.cuda.synchronize()
        outs.append(den.latents.clone())
    e = _err(outs[1], outs[0])
    print(f"hoisted vs stepwise after 4 steps: {e:.2e}")
    assert e < 3e-3


def test_windowed_hoisting_is_bit_identical(tiny):
    """K/V budget smaller than the whole loop (config 4: 84 GB at 1024^2 / 50 steps / batch 4): the garment passes are
    hoisted window by window. Same launches per (step, garment), so the latents must be bit-identical to the fully
    resident schedule, and the captured graph must survive the window switches."""
    from oracle import loop_ref as LR
    from idm_vton_b200.denoise import TryOnDenoiser
    from idm_vton_b200.scheduler import DDPMScheduler
    B, h, w, steps, run = 2, 16, 16, 30, 7
    inp = LR.synth_loop_inputs(tiny["cfg_t"], tiny["cfg_g"], B, h, w, seed=31)
    inp = {k: (v.half().float() if k != "add_time_ids" else v).cuda() for k, v in inp.items()}
    sch = DDPMScheduler()
    sch.set_timesteps(steps)
    outs, windows = [], []
    for steps_resident in (None, 3):
        den = TryOnDenoiser(tiny["eng_t"], tiny["eng_g"], garment_chunk=2)
        den.prepare(**inp)
        if steps_resident:
            den.max_kv_bytes = steps_resident * den.kv_bytes_per_step()
        den.set_step_tables(sch, sch.timesteps)
        windows.append(den.window)
        for i in range(run):
            den.step(i, None, use_graph=True)
        torch.cuda.synchronize()
        outs.append(den.latents.clone())
    assert windows == [steps, 2]          # 3 steps fit -> rounded down to a multiple of the garment chunk (2)
    assert torch.equal(outs[0], outs[1])
