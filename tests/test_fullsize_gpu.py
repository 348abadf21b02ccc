"""Full-size integrated parity: the SDXL-width engine (70 transformer blocks, the production wgmma GEMM / two-segment
flash-attention / fused cross-attention kernels) against the oracle on the SAME GPU, same fp16-rounded weights and inputs.

Three evaluations of every case:
  * ref32 : oracle (oracle/unet_ref.py, loop_ref.py) in fp32, TF32 off       — the high-precision answer
  * ref16 : oracle under torch.autocast(fp16) with fp16 weights              — the reference's own rounding points
            (inference.py:223,339: fp16 modules under torch.cuda.amp.autocast())
  * eng   : the engine (libb200vton.so)
Contract (north star: "fp16 outputs within 1e-3 of the reference diffusers path"; metric max|a-b| / max(1, max|b|)):
  (i)  eng-vs-ref16 <= 1e-3 wherever two independent fp16 evaluations of the network can agree that closely, i.e.
       wherever ref16 itself is within 1e-3 of ref32;
  (ii) always: eng-vs-ref32 <= ref16-vs-ref32 + 2.5e-4 (the engine is never further from the truth than the reference's own
       fp16 path, up to a quarter of the contract) and eng-vs-ref16 <= eng-vs-ref32 + ref16-vs-ref32 (triangle, sanity).
The measured triples are printed (`PARITY {...}` lines, visible with `pytest -s`).

Shapes: 128x96 latents, B=2 (BASELINE config 2: 3072 / 768 tokens, try-on batch 4) and 128x128 latents, B=1
(config 4 token counts 4096 / 1024).
"""
import json

import pytest
import torch

pytestmark = pytest.mark.gpu

def _record(**kw):
    print("PARITY " + json.dumps(kw))


def _err(a, b):
    a, b = a.float(), b.float()
    return (a - b).abs().max().item() / max(1.0, b.abs().max().item())


def _rel_l2(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def _cast(d, dtype):
    return {k: (v.to(dtype) if torch.is_floating_point(v) and k not in ("add_time_ids", "time_ids") else v) for k, v in d.items()}


@pytest.fixture(scope="module")
def full():
    from oracle import unet_ref as R
    from idm_vton_b200 import unet as U
    from idm_vton_b200.engine import SDXL_GARMENT, SDXL_TRYON, UNetEngine
    prev_tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)   # restored at teardown
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = "cuda"
    sd_t = U.random_state_dict(SDXL_TRYON, seed=11, device=dev)          # fp16: every path sees identical values
    sd_g = U.random_state_dict(SDXL_GARMENT, seed=22, device=dev)
    assert set(sd_t) == set(R.unet_param_shapes(R.SDXL_TRYON)) and set(sd_g) == set(R.unet_param_shapes(R.SDXL_GARMENT))
    env = dict(R=R, cfg_t=SDXL_TRYON, cfg_g=SDXL_GARMENT, sd_t=sd_t, sd_g=sd_g,
               eng_t=UNetEngine(SDXL_TRYON, sd_t, "tryon"), eng_g=UNetEngine(SDXL_GARMENT, sd_g, "garment"))
    env["sd_t32"] = {k: v.float() for k, v in sd_t.items()}
    env["sd_g32"] = {k: v.float() for k, v in sd_g.items()}
    yield env
    env.clear()
    torch.cuda.empty_cache()
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev_tf32


def _forward_inputs(cfg_t, cfg_g, B, h, w, seed):
    from oracle import loop_ref as LR
    inp = LR.synth_loop_inputs(cfg_t, cfg_g, B, h, w, seed=seed)
    inp = {k: (v.half().float() if k != "add_time_ids" else v) for k, v in inp.items()}
    return {k: v.cuda() for k, v in inp.items()}


def _oracle_step(R, sd_t, sd_g, cfg_t, cfg_g, inp, t):
    """One reference step body (src/tryon_pipeline.py:1769-1808): returns (garment features, noise_pred)."""
    lat = torch.cat([inp["latents"]] * 2)
    x = torch.cat([lat, inp["mask"], inp["masked_image_latents"], inp["pose_latents"]], dim=1)
    tt = torch.as_tensor(t, device=x.device)
    feats = R.unet_garment_forward(sd_g, cfg_g, inp["cloth_latents"], tt, inp["text_embeds_cloth"])
    fc = [torch.cat([torch.zeros_like(d), d]) for d in feats]
    added = {"text_embeds": inp["add_text_embeds"], "time_ids": inp["add_time_ids"], "image_embeds": inp["image_embeds"]}
    return feats, R.unet_tryon_forward(sd_t, cfg_t, x, tt, inp["prompt_embeds"], added, fc)


def _engine_step(env, inp, t, B, h, w):
    from idm_vton_b200 import lib as L
    from idm_vton_b200.engine import CIN_PAD
    eng_t, eng_g = env["eng_t"], env["eng_g"]
    f16 = torch.float16
    t_dev = torch.tensor([float(t)], device="cuda")
    xg = torch.zeros(B, h, w, CIN_PAD, dtype=f16, device="cuda")
    L.nchw_to_nhwc(inp["cloth_latents"].half().contiguous(), xg)
    feats = []
    eng_g.forward(xg, eng_g.time_embedding(t_dev, B), eng_g.encode_context(inp["text_embeds_cloth"].half()), collect=feats)
    xt = torch.zeros(2 * B, h, w, CIN_PAD, dtype=f16, device="cuda")
    L.nchw_to_nhwc(inp["latents"].half().contiguous(), xt, c_off=0)          # CFG duplication by the modulo scatter
    L.nchw_to_nhwc(inp["mask"].half().contiguous(), xt, c_off=4)
    L.nchw_to_nhwc(inp["masked_image_latents"].half().contiguous(), xt, c_off=5)
    L.nchw_to_nhwc(inp["pose_latents"].half().contiguous(), xt, c_off=9)
    ctx = eng_t.encode_context(inp["prompt_embeds"].half(), inp["image_embeds"].half())
    aug = eng_t.aug_embedding(inp["add_text_embeds"].half(), inp["add_time_ids"])
    eps = eng_t.forward(xt, eng_t.time_embedding(t_dev, 2 * B, aug), ctx, gfeats=feats, n_persons=B)
    return feats, L.nhwc_to_nchw(eps, 4)


def _gate(tag, d_eng32, d_ref32, d_eng16):
    assert d_eng32 <= d_ref32 + 2.5e-4, f"{tag}: engine further from fp32 truth ({d_eng32:.2e}) than the reference's fp16 path ({d_ref32:.2e})"
    assert d_eng16 <= d_eng32 + d_ref32 + 1e-6, f"{tag}: triangle inequality violated?"
    if d_ref32 <= 1e-3:
        assert d_eng16 <= 1e-3 + d_ref32, f"{tag}: engine vs fp16 reference {d_eng16:.2e}"


@pytest.mark.parametrize("B,h,w,t", [(2, 128, 96, 967), (1, 128, 128, 301)])
def test_fullsize_unets_vs_oracle(full, B, h, w, t):
    """Garment UNet (70 exported features) + try-on UNet forward at SDXL width on the production kernels."""
    from idm_vton_b200 import lib as L
    R = full["R"]
    inp = _forward_inputs(full["cfg_t"], full["cfg_g"], B, h, w, seed=7 + B)
    n0 = L.launch_count()
    feats, eps = _engine_step(full, inp, t, B, h, w)
    torch.cuda.synchronize()
    launches = L.launch_count() - n0
    assert len(feats) == 70
    with torch.no_grad():
        f32, e32 = _oracle_step(R, full["sd_t32"], full["sd_g32"], full["cfg_t"], full["cfg_g"], inp, t)
        with torch.autocast("cuda", dtype=torch.float16):
            f16, e16 = _oracle_step(R, full["sd_t"], full["sd_g"], full["cfg_t"], full["cfg_g"], _cast(inp, torch.float16), t)
    assert torch.isfinite(e32).all() and torch.isfinite(e16.float()).all() and torch.isfinite(eps.float()).all()
    fe = [(_err(a, b), _err(c, b)) for a, b, c in zip(feats, f32, f16)]
    f_eng32, f_ref32 = max(x[0] for x in fe), max(x[1] for x in fe)
    f_eng16 = max(_err(a, c) for a, c in zip(feats, f16))
    d_eng32, d_ref32, d_eng16 = _err(eps, e32), _err(e16, e32), _err(eps, e16)
    _record(case=f"unets B={B} {h}x{w} t={t}", launches=launches, eps_absmax=e32.abs().max().item(),
            feats=dict(eng_vs_32=f_eng32, ref16_vs_32=f_ref32, eng_vs_ref16=f_eng16),
            eps=dict(eng_vs_32=d_eng32, ref16_vs_32=d_ref32, eng_vs_ref16=d_eng16,
                     rel_l2_eng_vs_32=_rel_l2(eps, e32), rel_l2_ref16_vs_32=_rel_l2(e16, e32)))
    _gate("garment features", f_eng32, f_ref32, f_eng16)
    _gate("noise_pred", d_eng32, d_ref32, d_eng16)


def test_fullsize_hoisted_loop_vs_oracle(full):
    """3 denoise steps of the production loop (hoisted + batched garment passes, K/V of all steps resident, one CUDA graph
    per step) at config-2 shapes vs the oracle loop (src/tryon_pipeline.py:1765-1823)."""
    from oracle import loop_ref as LR
    from idm_vton_b200.denoise import TryOnDenoiser
    from idm_vton_b200.scheduler import DDPMScheduler
    B, h, w, steps, run = 2, 128, 96, 30, 3
    inp = _forward_inputs(full["cfg_t"], full["cfg_g"], B, h, w, seed=3)
    g = torch.Generator().manual_seed(5)
    noises = [torch.randn(B, 4, h, w, generator=g).half().float().cuda() for _ in range(run)]
    den = TryOnDenoiser(full["eng_t"], full["eng_g"])
    sch = DDPMScheduler()
    sch.set_timesteps(steps)
    den.prepare(**inp, guidance_scale=2.0)
    den.set_step_tables(sch, sch.timesteps)
    for i in range(run):
        den.step(i, noises[i].half(), use_graph=True)
    torch.cuda.synchronize()
    lat = den.latents.clone()
    del den
    with torch.no_grad():
        ref = LR.denoise_loop(full["sd_t32"], full["cfg_t"], full["sd_g32"], full["cfg_g"], inp, steps, noises=noises,
                              max_steps=run)
        with torch.autocast("cuda", dtype=torch.float16):
            ref16 = LR.denoise_loop(full["sd_t"], full["cfg_t"], full["sd_g"], full["cfg_g"], _cast(inp, torch.float16),
                                    steps, noises=[n.half() for n in noises], max_steps=run)
    d_eng32, d_ref32, d_eng16 = _err(lat, ref), _err(ref16, ref), _err(lat, ref16)
    _record(case=f"hoisted loop {run} of {steps} steps B={B} {h}x{w}", latents_absmax=ref.abs().max().item(),
            latents=dict(eng_vs_32=d_eng32, ref16_vs_32=d_ref32, eng_vs_ref16=d_eng16))
    _gate("latents", d_eng32, d_ref32, d_eng16)


def test_fullsize_shared_garment_step_vs_oracle(full):
    """BASELINE config 3 semantics at full size: three persons share ONE garment (garment UNet at batch 1, its K/V indexed
    by every person through the modulo / base scalars of the attention kernel); one hoisted denoise step vs the oracle loop,
    which expands the garment features to the batch like the reference would (src/tryon_pipeline.py:1787-1796)."""
    from oracle import loop_ref as LR
    from idm_vton_b200.denoise import TryOnDenoiser
    from idm_vton_b200.scheduler import DDPMScheduler
    B, h, w, steps = 3, 128, 96, 30
    inp = LR.synth_loop_inputs(full["cfg_t"], full["cfg_g"], B, h, w, Bg=1, seed=13)
    inp = {k: (v.half().float() if k != "add_time_ids" else v).cuda() for k, v in inp.items()}
    noise = torch.randn(B, 4, h, w, generator=torch.Generator().manual_seed(6)).half().float().cuda()
    den = TryOnDenoiser(full["eng_t"], full["eng_g"])
    sch = DDPMScheduler()
    sch.set_timesteps(steps)
    den.prepare(**inp, guidance_scale=2.0)
    den.set_step_tables(sch, sch.timesteps)
    assert den.Bg == 1 and den.gkv_all[0].shape[0] == steps
    den.step(0, noise.half(), use_graph=True)
    torch.cuda.synchronize()
    lat = den.latents.clone()
    del den
    with torch.no_grad():
        ref = LR.denoise_loop(full["sd_t32"], full["cfg_t"], full["sd_g32"], full["cfg_g"], inp, steps, noises=[noise], max_steps=1)
        with torch.autocast("cuda", dtype=torch.float16):
            ref16 = LR.denoise_loop(full["sd_t"], full["cfg_t"], full["sd_g"], full["cfg_g"], _cast(inp, torch.float16), steps,
                                    noises=[noise.half()], max_steps=1)
    d_eng32, d_ref32, d_eng16 = _err(lat, ref), _err(ref16, ref), _err(lat, ref16)
    _record(case=f"shared garment, 1 step, B={B} persons / 1 garment {h}x{w}", latents_absmax=ref.abs().max().item(),
            latents=dict(eng_vs_32=d_eng32, ref16_vs_32=d_ref32, eng_vs_ref16=d_eng16))
    _gate("latents (shared garment)", d_eng32, d_ref32, d_eng16)
