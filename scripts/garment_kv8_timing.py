"""FP8 garment K/V against fp16 on one GPU, with the card's name and power limit read in the same run:
  * kernels: the self + garment attention of the try-on blocks (b200vton_attention_kv8 against b200vton_attention /
    _rows) at the config-2 try-on shapes, level 1 (B = 4 under CFG, H = 10, 3072 self + 3072 garment keys) and level 2
    (H = 20, 768 + 768), both addressing modes; ms per launch from CUDA events around a replayed graph of `reps`
    launches, TFLOP/s from the shapes (4 * Nq * (N0 + N1) * 64 per head and sample, the CFG-uncond half counted with N0
    keys only, as the kernel runs it); and the quantizer's bandwidth on 30 rows of one level-1 block;
  * with --pool: ContinuousTryOnServer pool mode at config-2 geometry (768x1024, DDPM 30 steps, S = 4, random SDXL
    weights as bench.py builds them, a budget of --kv-gb): pages, the full-occupancy step and one page fill;
  * with --config4: the config-4 loop (1024x1024, 50 steps, B = 4, one garment per request): hoisted garment passes
    plus the 50 steps, and the number of K/V windows, with TryOnDenoiser's default budget.
The two formats are alternated over --rounds rounds in the same process.

    python scripts/garment_kv8_timing.py [--reps 50] [--pool] [--config4] [--rounds 2] [--kv-gb 40]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _time(fn, reps):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    g.replay()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(5):
        g.replay()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / (5 * reps)


def _events(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def pool_mode(pipe, fmt, kv_bytes):
    """Pages, the full-occupancy step (S = 4, 10 replays) and one page fill of a pool-mode server in format fmt."""
    import gc
    from idm_vton_b200.serving import ContinuousTryOnServer
    from scripts.continuous_timing import H, T, W, make_requests
    pipe.set_garment_kv_precision(fmt)
    pipe.garment_cache, pipe._denoiser = None, None
    gc.collect()
    torch.cuda.empty_cache()
    S = 4
    srv = ContinuousTryOnServer(pipe, height=H, width=W, slots=S, num_inference_steps=T, guidance_scale=2.0, seed=7,
                                garment_kv_bytes=kv_bytes)
    reqs = make_requests(S, S, "cuda", seed=1)
    for r in reqs:
        srv.submit(r)
    srv.step()                                                 # admits all (4 fills), captures the graph
    srv.den.step([5] * S)
    step = _events(lambda: [srv.den.step([5] * S) for _ in range(10)]) / 10
    g = srv.garments[reqs[0].garment_id]
    fill = _events(lambda: srv.den.fill_page(srv.den.P - 1, g["latents"], g["text_embeds_cloth"]))
    res = dict(pages=srv.den.P, page_bytes=srv.page_bytes(), step_ms=round(step, 2), fill_ms=round(fill, 1))
    del srv, g
    return res


def config4(unet, unet_enc, fmt):
    """The config-4 loop in format fmt: set_step_tables (the hoisted garment passes of the first window) plus 50 steps,
    the later windows' passes included."""
    import gc
    from idm_vton_b200.denoise import TryOnDenoiser
    from idm_vton_b200.engine import SDXL_GARMENT, SDXL_TRYON
    from idm_vton_b200.scheduler import DDPMScheduler
    import bench
    unet.set_garment_kv_precision(fmt)
    gc.collect()
    torch.cuda.empty_cache()
    T, B = 50, 4
    req = bench.synth_request(SDXL_TRYON, SDXL_GARMENT, B, 128, 128, seed=42, device="cuda")
    den = TryOnDenoiser(unet.engine(), unet_enc.engine())
    sch = DDPMScheduler()
    sch.set_timesteps(T)
    den.prepare(**req, guidance_scale=2.0)

    def loop():
        den.set_step_tables(sch, sch.timesteps)
        for i in range(T):
            den.step(i, None)
    loop()                                                     # captures the graph
    ms = _events(loop)
    res = dict(loop_s=round(ms / 1e3, 2), windows=-(-T // den.window), window_steps=den.window,
               kv_bytes_per_step=den.kv_bytes_per_step())
    del den
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--pool", action="store_true")
    ap.add_argument("--config4", action="store_true")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--kv-gb", type=float, default=40, help="pool budget (GB, 1e9 bytes)")
    args = ap.parse_args()
    from idm_vton_b200 import lib as L
    from scripts.schedule_timing import card
    L.load()
    dev = "cuda"
    out = dict(card=card())
    for name, H, N in (("level1", 10, 3072), ("level2", 20, 768)):
        C, B, T = H * 64, 4, 30
        g = torch.Generator(device=dev).manual_seed(0)
        q, k0, v0 = (torch.randn(B, N, C, device=dev, generator=g).half() for _ in range(3))
        kv16 = torch.randn(T, N, 2 * C, device=dev, generator=g).half()
        kv8 = L.quantize_kv_e4m3(kv16, L.GarmentKV8.empty(T, N, C, dev))
        base = torch.tensor([5], dtype=torch.int32, device=dev)
        rows = torch.tensor([3, 17], dtype=torch.int32, device=dev)
        flops = 4 * N * 64 * H * (B * (N + N) - (B // 2) * N)
        res = {}
        res["fp16_step_base"] = _time(lambda: L.attention(q, k0, v0, kv16[..., :C], kv16[..., C:], kv1_off=B // 2,
                                                          heads=H, kv1_mod=1, kv1_base=base), args.reps)
        res["kv8_step_base"] = _time(lambda: L.attention_kv8(q, k0, v0, kv8, kv1_off=B // 2, heads=H, kv1_mod=1,
                                                             kv1_base=base), args.reps)
        res["fp16_rows"] = _time(lambda: L.attention_rows(q, k0, v0, kv16[..., :C], kv16[..., C:], rows,
                                                          kv1_off=B // 2, heads=H), args.reps)
        res["kv8_rows"] = _time(lambda: L.attention_kv8(q, k0, v0, kv8, kv1_off=B // 2, heads=H, kv1_rows=rows),
                                args.reps)
        out[name] = {k: dict(ms=round(v, 4), tflops=round(flops / v / 1e9, 1)) for k, v in res.items()}
        if name == "level1":
            ms = _time(lambda: L.quantize_kv_e4m3(kv16, kv8), 5)
            moved = kv16.numel() * 2 + kv8.q.numel() + kv8.e.numel()
            out["quantize_level1_30rows"] = dict(ms=round(ms, 4), MB_moved=round(moved / 1e6, 1),
                                                 GBps=round(moved / ms / 1e6, 1))
        del q, k0, v0, kv16, kv8
    if args.pool or args.config4:
        import bench
        unet, unet_enc, _ = bench.build_components(torch.device(dev, 0), 0, 1, lambda m: None)
        pipe = bench.make_pipeline(unet, unet_enc, torch.device(dev, 0)) if args.pool else None
        for key in (("pool",) if args.pool else ()) + (("config4",) if args.config4 else ()):
            out[key] = {"fp16": [], "fp8": []}
            for _ in range(args.rounds):
                for fmt in ("fp16", "fp8"):
                    r = pool_mode(pipe, fmt, int(args.kv_gb * 1e9)) if key == "pool" else config4(unet, unet_enc, fmt)
                    out[key][fmt].append(r)
                    print(key, fmt, r, flush=True)
        unet.set_garment_kv_precision("fp16")
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
