"""Image sizes that are multiples of 8 but not of 32, and the garment at a size of its own, on the engine:
  * b200vton_upsample_nearest_nhwc bit-identical to F.interpolate(size=..., mode="nearest") on CUDA, and its 2x case to
    the scale-2 gather of b200vton_upsample2x_nhwc;
  * `StableDiffusionXLInpaintPipeline.__call__` against the REFERENCE pipeline's own run at four geometries (golden
    tests/golden/pipeline_resolution_ref.pt, oracle/make_golden_resolution.py) with the three checks of
    test_seams_gpu.py::test_pipeline_call_vs_reference_golden, and through a TryOnServer;
  * the SDXL-width engine at odd sizes against the oracle (the full-size policy of DESIGN.md section 3);
  * determinism: graph replay vs eager launches, garment-cache hits, and a cache miss when only the cloth size changes.
"""
import json
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

G = os.path.join(os.path.dirname(__file__), "golden")
CASES = ["odd_both", "even_not_x4", "cloth_larger", "cloth_smaller"]
NAMES = ("latents", "mask", "masked_image_latents", "pose_latents", "cloth_latents", "prompt_embeds", "add_text_embeds",
         "add_time_ids", "image_embeds", "text_embeds_cloth")


def _err(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return (a - b).abs().max().item() / max(1.0, b.abs().max().item())


# ------------------------------------------------------------------------------------------------
# the resize kernel
# ------------------------------------------------------------------------------------------------
RESIZES = [(9, 7, 17, 13), (8, 6, 15, 11), (17, 13, 33, 25), (6, 5, 12, 9), (12, 9, 24, 18), (33, 25, 17, 13),
           (5, 7, 5, 7), (3, 4, 10, 9), (7, 7, 3, 16), (64, 48, 128, 96)]


@pytest.mark.parametrize("C", [64, 320, 1280])
def test_upsample_nearest_bit_identical_to_interpolate(C):
    from idm_vton_b200 import lib as L
    g = torch.Generator(device="cuda").manual_seed(C)
    for B in (1, 2, 3):
        for H, W, Ho, Wo in RESIZES:
            x = torch.randn(B, H, W, C, generator=g, device="cuda").half()
            y = L.upsample_nearest(x, (Ho, Wo))
            ref = F.interpolate(x.permute(0, 3, 1, 2).contiguous(), size=(Ho, Wo), mode="nearest").permute(0, 2, 3, 1)
            assert torch.equal(y, ref), (B, H, W, C, Ho, Wo)
            if (Ho, Wo) == (2 * H, 2 * W):
                # the scale-2 entry point is the same kernel and keeps the parent's gather: dst[y, x] = src[y >> 1, x >> 1]
                gather = x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
                assert torch.equal(L.upsample2x(x), gather) and torch.equal(y, gather)


def test_upsample_nearest_rejects_bad_arguments():
    from idm_vton_b200 import lib as L
    n0 = L.launch_count()
    with pytest.raises(RuntimeError, match="code 1"):
        L.upsample_nearest(torch.zeros(1, 4, 4, 12, dtype=torch.float16, device="cuda"), (8, 8))
    with pytest.raises(RuntimeError, match="code 1"):
        L.upsample_nearest(torch.zeros(1, 4, 4, 64, dtype=torch.float16, device="cuda"), (0, 8))
    assert L.launch_count() == n0


# ------------------------------------------------------------------------------------------------
# the pipeline against the reference pipeline's own run
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tiny_modules():
    from oracle import unet_ref as R
    from idm_vton_b200 import unet as U
    cfg_t, cfg_g = R.tiny_config("tryon"), R.tiny_config("garment")
    sd_t, sd_g = R.make_state_dict(cfg_t, seed=11), R.make_state_dict(cfg_g, seed=22)
    net_t = U.UNet2DConditionModel(cfg_t, sd_t).to("cuda", torch.float16)
    net_g = U.UNet2DConditionModelGarment(cfg_g, sd_g).to("cuda", torch.float16)
    sd_t32 = {k: v.half().float().cuda() for k, v in sd_t.items()}
    sd_g32 = {k: v.half().float().cuda() for k, v in sd_g.items()}
    return dict(cfg_t=cfg_t, cfg_g=cfg_g, sd_t32=sd_t32, sd_g32=sd_g32, net_t=net_t, net_g=net_g)


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(G, "pipeline_resolution_ref.pt"))


def _make_pipe(tiny_modules):
    from oracle import make_golden_pipeline as MG
    from idm_vton_b200.denoise import TryOnDenoiser
    from idm_vton_b200.pipeline import StableDiffusionXLInpaintPipeline
    from idm_vton_b200.scheduler import DDPMScheduler
    dev, f16 = "cuda", torch.float16
    cfg_t = tiny_modules["cfg_t"]
    pipe = StableDiffusionXLInpaintPipeline(
        vae=MG.make_vae().to(dev, f16), text_encoder=None, text_encoder_2=None, tokenizer=None, tokenizer_2=None,
        unet=tiny_modules["net_t"], unet_encoder=tiny_modules["net_g"], scheduler=DDPMScheduler(),
        image_encoder=MG.make_image_encoder(cfg_t["resampler"]["embedding_dim"]).to(dev, f16))
    den = TryOnDenoiser(pipe.unet.engine(), pipe.unet_encoder.engine())
    pipe._denoiser = den
    rec = {"runs": []}
    real_prepare, real_step = den.prepare, den.step

    def prepare(*a, **kw):
        rec["runs"].append({"inputs": {n: v.detach().float().clone() for n, v in zip(NAMES, a)}, "noises": [],
                            "latents": []})
        return real_prepare(*a, **kw)

    def step(i, noise=None, use_graph=True):
        rec["runs"][-1]["noises"].append(None if noise is None else noise.detach().float().clone())
        out = real_step(i, noise, use_graph=use_graph)
        rec["runs"][-1]["latents"].append(out.detach().float().clone())
        return out

    den.prepare, den.step = prepare, step
    return pipe, rec


def _oracle_loop_errors(tiny_modules, run, steps):
    """(ii): the engine's latents after each step against resolution_ref.denoise_loop on the same inputs and noises."""
    from oracle import make_golden_pipeline as MG
    from oracle import resolution_ref as RR
    li = {n: v.cuda() for n, v in run["inputs"].items()}
    errs = []
    with torch.no_grad():
        for n in range(1, len(run["latents"]) + 1):
            ref = RR.denoise_loop(tiny_modules["sd_t32"], tiny_modules["cfg_t"], tiny_modules["sd_g32"], tiny_modules["cfg_g"],
                                  li, steps, guidance_scale=MG.GUIDANCE, noises=run["noises"], max_steps=n)
            errs.append(_err(run["latents"][n - 1], ref))
    return errs


@pytest.mark.parametrize("name", CASES)
def test_pipeline_call_vs_reference_golden(tiny_modules, golden, name):
    """__call__ at the case's person / cloth sizes, CUDA graph on, against the reference pipeline: (i) the loop's inputs,
    (ii) the engine loop vs the oracle loop on those inputs, (iii) end to end; the gates of
    test_seams_gpu.py::test_pipeline_call_vs_reference_golden."""
    from oracle import make_golden_pipeline as MG
    from oracle import make_golden_resolution as MR
    c = golden["cases"][name]
    dev, f16 = "cuda", torch.float16
    cfg_t = tiny_modules["cfg_t"]
    call_inputs = MR.make_case_inputs(cfg_t, name)
    ref_in = MR.loop_inputs(c, call_inputs)
    inp = {k: (v.to(dev, f16) if k not in ("image", "mask_image") else v.to(dev)) for k, v in call_inputs.items()}
    pipe, rec = _make_pipe(tiny_modules)
    assert pipe.use_cuda_graph
    seen = []

    def on_step_end(p, i, t, kw):
        seen.append(int(t))
        return {}

    # fp32 CPU draws rounded to fp16, as in test_seams_gpu.py: the order, shapes and count of the draws stay the pipeline's
    gen = torch.Generator().manual_seed(42)
    real_randn = torch.randn

    def randn_fp32_draws(*size, generator=None, dtype=None, **kw):
        if generator is gen and dtype == torch.float16:
            return real_randn(*size, generator=generator, dtype=torch.float32, **kw).to(torch.float16)
        return real_randn(*size, generator=generator, dtype=dtype, **kw)

    torch.manual_seed(1234)
    torch.randn = randn_fp32_draws
    try:
        images = pipe(**MR.call_kwargs(MG, inp, gen, name), output_type="pt", callback_on_step_end=on_step_end)[0]
    finally:
        torch.randn = real_randn
    (H, W), _ = MR.CASES[name]
    run = rec["runs"][-1]
    assert seen == c["timesteps"].tolist() and images.shape == (1, 3, H, W)
    assert pipe._denoiser.x_g.shape[1:3] == c["stored"]["cloth_latents"].shape[-2:]
    # (i)
    e_in = {n: _err(run["inputs"][n], ref_in[n]) for n in NAMES}
    for n in ("mask", "prompt_embeds", "add_text_embeds", "add_time_ids", "text_embeds_cloth"):
        assert e_in[n] == 0.0, n
    assert e_in["latents"] < 1e-3
    for n in ("masked_image_latents", "pose_latents", "cloth_latents"):
        assert e_in[n] < 3e-3, n
    assert e_in["image_embeds"] < 5e-3
    # (ii)
    e_loop = _oracle_loop_errors(tiny_modules, run, golden["steps"])
    # (iii)
    e_e2e = [_err(l, r) for l, r in zip(run["latents"], c["latents_per_step"])]
    ref_images = MR.decode_images(MG.make_vae(), c["latents_per_step"][-1])
    d_img = (images.float().cpu() - ref_images).abs()
    print("RESOLUTION " + json.dumps(dict(case=name, inputs=e_in, loop=e_loop, e2e=e_e2e, image_max=d_img.max().item(),
                                          image_mean=d_img.mean().item())))
    assert max(e_loop) < 4e-3
    assert max(e_e2e) < 5e-2 and d_img.mean().item() < 2e-2


def test_server_garments_at_their_own_size(tiny_modules):
    """A TryOnServer for 256x192 persons gets a 264x200 garment and a 192x144 garment: each batch's loop equals the oracle
    loop on its own inputs, the images have the person's size, and a garment seen before is a cache hit with bit-identical
    images."""
    from oracle import make_golden_resolution as MR
    from idm_vton_b200.serving import TryOnRequest, TryOnServer
    cfg_t = tiny_modules["cfg_t"]
    pipe, rec = _make_pipe(tiny_modules)
    person = MR.make_case_inputs(cfg_t, "cloth_larger", seed=5)               # 256x192 person, 264x200 cloth
    garments = {"L": MR.make_case_inputs(cfg_t, "cloth_larger", seed=1001),
                "S": MR.make_case_inputs(cfg_t, "cloth_smaller", seed=1002)}  # cloth 192x144

    def req(gid):
        i, gi = person, garments[gid]
        return TryOnRequest(garment_id=gid, image=i["image"][0], mask_image=i["mask_image"][0], pose_img=i["pose_img"][0],
                            prompt_embeds=i["prompt_embeds"][0], negative_prompt_embeds=i["negative_prompt_embeds"][0],
                            pooled_prompt_embeds=i["pooled_prompt_embeds"][0],
                            negative_pooled_prompt_embeds=i["negative_pooled_prompt_embeds"][0], cloth=gi["cloth"][0],
                            ip_adapter_image=gi["ip_adapter_image"][0], text_embeds_cloth=gi["text_embeds_cloth"][0])

    steps = 2
    srv = TryOnServer(pipe, height=256, width=192, num_inference_steps=steps, guidance_scale=2.0, max_batch=4, seed=7)
    t = [srv.submit(req("L")), srv.submit(req("S"))]
    out1 = srv.run()
    assert srv.pipe.garment_cache.hits == 0 and srv.pipe.garment_cache.misses == 2
    for ticket, run, (hg, wg) in zip(t, rec["runs"], ((33, 25), (24, 18))):
        assert out1[ticket].shape == (3, 256, 192) and run["inputs"]["cloth_latents"].shape[-2:] == (hg, wg)
        e_loop = _oracle_loop_errors(tiny_modules, run, steps)
        print(f"server: cloth latents {hg}x{wg}, engine loop vs oracle loop per step {e_loop}")
        assert max(e_loop) < 4e-3
    t2 = srv.submit(req("L"))
    out2 = srv.run()
    assert srv.pipe.garment_cache.hits == 1
    assert torch.equal(out2[t2], out1[t[0]])


# ------------------------------------------------------------------------------------------------
# determinism at odd sizes
# ------------------------------------------------------------------------------------------------
def _odd_inputs(cfg_t, cfg_g, h, w, hg, wg, seed):
    from oracle import loop_ref as LR
    inp = LR.synth_loop_inputs(cfg_t, cfg_g, 1, h, w, seed=seed)
    inp["cloth_latents"] = torch.randn(1, 4, hg, wg, generator=torch.Generator().manual_seed(seed + 1)) * 0.5
    return {k: (v.half().float() if k != "add_time_ids" else v).cuda() for k, v in inp.items()}


def test_graph_replay_and_garment_cache_at_odd_sizes(tiny_modules):
    from idm_vton_b200.denoise import GarmentKVCache, TryOnDenoiser
    from idm_vton_b200.scheduler import DDPMScheduler
    net_t, net_g = tiny_modules["net_t"], tiny_modules["net_g"]
    inp = _odd_inputs(tiny_modules["cfg_t"], tiny_modules["cfg_g"], 33, 25, 24, 18, seed=21)
    g = torch.Generator().manual_seed(8)
    noises = [torch.randn(1, 4, 33, 25, generator=g).half().cuda() for _ in range(3)]
    sch = DDPMScheduler()
    sch.set_timesteps(3)

    def run(den, use_graph, inputs=inp, keys=None, cache=None):
        den.prepare(**inputs, guidance_scale=2.0)
        den.set_step_tables(sch, sch.timesteps, garment_keys=keys, cache=cache)
        for i in range(3):
            den.step(i, noises[i], use_graph=use_graph)
        torch.cuda.synchronize()
        return den.latents.clone()

    eager = run(TryOnDenoiser(net_t.engine(), net_g.engine()), False)
    den = TryOnDenoiser(net_t.engine(), net_g.engine())
    graph = run(den, True)
    assert den._graph is not None and den.x_g.shape[1:3] == (24, 18)
    assert torch.equal(graph, eager)
    # garment K/V cache: a hit at cloth != person size reproduces the computed run bit for bit
    cache = GarmentKVCache()
    first = run(den, True, keys=["g"], cache=cache)
    hit = run(den, True, keys=["g"], cache=cache)
    assert (cache.misses, cache.hits) == (1, 1) and torch.equal(first, eager) and torch.equal(hit, eager)
    # the same key with only the cloth size changed is a miss; the buffers and the graph follow the new size
    inp2 = dict(inp, cloth_latents=torch.nn.functional.interpolate(inp["cloth_latents"], size=(32, 24)))
    other = run(den, True, inputs=inp2, keys=["g"], cache=cache)
    assert (cache.misses, cache.hits) == (2, 1) and den.x_g.shape[1:3] == (32, 24)
    assert den.gkv_all[0].shape[1] == 16 * 12 and not torch.equal(other, eager)


# ------------------------------------------------------------------------------------------------
# SDXL width at odd sizes
# ------------------------------------------------------------------------------------------------
def _cast(d, dtype):
    return {k: (v.to(dtype) if torch.is_floating_point(v) and k != "add_time_ids" else v) for k, v in d.items()}


def test_sdxl_width_odd_sizes_vs_oracle():
    """One hoisted denoise step at SDXL width and depth, person latents 33x25 (both UNets' up paths resize to the skips)
    with a 32x24 garment, B = 2: engine vs ref32 <= ref16 vs ref32 + 2.5e-4 (DESIGN.md section 3)."""
    from oracle import resolution_ref as RR
    from oracle import unet_ref as R
    from idm_vton_b200 import unet as U
    from idm_vton_b200.denoise import TryOnDenoiser
    from idm_vton_b200.engine import SDXL_GARMENT, SDXL_TRYON, UNetEngine
    from idm_vton_b200.scheduler import DDPMScheduler
    prev_tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    try:
        sd_t = U.random_state_dict(SDXL_TRYON, seed=11, device="cuda")
        sd_g = U.random_state_dict(SDXL_GARMENT, seed=22, device="cuda")
        B, h, w, hg, wg, steps = 2, 33, 25, 32, 24, 30
        from oracle import loop_ref as LR
        inp = LR.synth_loop_inputs(SDXL_TRYON, SDXL_GARMENT, B, h, w, seed=17)
        inp["cloth_latents"] = torch.randn(B, 4, hg, wg, generator=torch.Generator().manual_seed(18)) * 0.5
        inp = {k: (v.half().float() if k != "add_time_ids" else v).cuda() for k, v in inp.items()}
        noise = torch.randn(B, 4, h, w, generator=torch.Generator().manual_seed(6)).half().float().cuda()
        den = TryOnDenoiser(UNetEngine(SDXL_TRYON, sd_t, "tryon"), UNetEngine(SDXL_GARMENT, sd_g, "garment"))
        sch = DDPMScheduler()
        sch.set_timesteps(steps)
        den.prepare(**inp, guidance_scale=2.0)
        den.set_step_tables(sch, sch.timesteps)
        assert den.gkv_all[-1].shape[1] == (hg // 2) * (wg // 2)
        den.step(0, noise.half(), use_graph=True)
        torch.cuda.synchronize()
        lat = den.latents.clone()
        del den
        with torch.no_grad():
            ref = RR.denoise_loop({k: v.float() for k, v in sd_t.items()}, SDXL_TRYON,
                                  {k: v.float() for k, v in sd_g.items()}, SDXL_GARMENT, inp, steps, noises=[noise],
                                  max_steps=1)
            with torch.autocast("cuda", dtype=torch.float16):
                ref16 = RR.denoise_loop(sd_t, SDXL_TRYON, sd_g, SDXL_GARMENT, _cast(inp, torch.float16), steps,
                                        noises=[noise.half()], max_steps=1)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev_tf32
    d_eng32, d_ref32, d_eng16 = _err(lat, ref), _err(ref16, ref), _err(lat, ref16)
    print("PARITY " + json.dumps(dict(case=f"odd sizes, person {h}x{w}, cloth {hg}x{wg}, B={B}, 1 step",
                                      latents=dict(eng_vs_32=d_eng32, ref16_vs_32=d_ref32, eng_vs_ref16=d_eng16))))
    assert d_eng32 <= d_ref32 + 2.5e-4
    assert d_eng16 <= d_eng32 + d_ref32 + 1e-6
    if d_ref32 <= 1e-3:
        assert d_eng16 <= 1e-3 + d_ref32
    assert set(sd_t) == set(R.unet_param_shapes(R.SDXL_TRYON))
