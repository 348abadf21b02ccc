"""Continuous batching against batch mode on one GPU, at config-2 geometry (768x1024, DDPM 30 steps, guidance 2.0) with
random SDXL-shaped weights as bench.py builds them.

A seeded Poisson arrival trace of `--requests` requests over `--garments` garments goes through three modes, alternated
in one process (`--rounds` rounds after a warm-up of each):
  batch:            serving.TryOnServer(max_batch=S) with a garment K/V cache of `--kv-gb`;
  continuous:       serving.ContinuousTryOnServer(slots=S), the garment UNet inside every step;
  continuous_pool:  serving.ContinuousTryOnServer(slots=S, garment_kv_bytes=--kv-gb), hoisted garment K/V pages.
Batch mode's cache and the pool get the same budget (one garment's K/V of all 30 steps is 9.44 GB, so the default 40 GB
holds 4 garments). Every round starts each mode afresh: a new server, a new denoiser, an empty cache or pool. So each
round's numbers include the capture of its CUDA graphs (a continuous denoiser captures one graph, at its first step;
batch mode's denoiser captures one per batch shape and again whenever a batch of another size follows, as it does in
service) and, in pool mode, every page fill. The rate is `--load` times the capacity of a default continuous server at
full occupancy, measured first. Prints one JSON line with, per mode:
  images_per_s:   requests / (last image - first arrival);
  latency_s:      p50 / p95 from arrival to image;
  (pool mode) garment_page_fills / garment_page_hits and the hit rate;
and the step time at full occupancy (the default continuous step graph and the pool step graph at S slots) against the
batch-mode step at batch S with one garment plus its hoisted garment passes per step; the time of one page fill (a
miss); the card's name and power limit, read in the same run.
--garment-kv fp8 runs batch mode and pool mode with the pipeline's FP8 garment K/V (pipe.set_garment_kv_precision):
batch mode's cache entries and the pool's pages are then about half the size. The default continuous mode holds no
garment K/V and refuses the format, so it only sets the arrival rate, as in fp16.
Usage: python scripts/continuous_timing.py [--slots 4] [--requests 32] [--garments 8] [--rounds 2] [--kv-gb 40]
       [--garment-kv fp16|fp8]"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import idm_vton_b200  # noqa: F401,E402
import bench  # noqa: E402
from scripts.schedule_timing import card  # noqa: E402

H, W, T = 1024, 768, 30


def make_requests(n, n_garments, device, seed):
    from idm_vton_b200.serving import TryOnRequest
    g = torch.Generator(device="cpu").manual_seed(seed)
    garments = {}
    for k in range(n_garments):
        garments[k] = dict(cloth=(torch.rand(3, H, W, generator=g) * 2 - 1).to(device, torch.float16),
                           ip_adapter_image=torch.randn(3, 224, 224, generator=g).to(device, torch.float16),
                           text_embeds_cloth=torch.randn(77, 2048, generator=g).to(device, torch.float16))
    reqs = []
    for i in range(n):
        mask = torch.zeros(1, H, W)
        mask[:, H // 4:3 * H // 4, W // 4:3 * W // 4] = 1.0
        gid = int(torch.randint(n_garments, (1,), generator=g))
        r = lambda *s: torch.randn(*s, generator=g).to(device, torch.float16)  # noqa: E731
        reqs.append(dict(garment_id=gid, image=torch.rand(3, H, W, generator=g).to(device), mask_image=mask.to(device),
                         pose_img=(torch.rand(3, H, W, generator=g) * 2 - 1).to(device, torch.float16),
                         prompt_embeds=r(77, 2048), negative_prompt_embeds=r(77, 2048), pooled_prompt_embeds=r(1280),
                         negative_pooled_prompt_embeds=r(1280), seed=i, **garments[gid]))
    return [TryOnRequest(**d) for d in reqs]


def serve(server, reqs, arrivals):
    """Submits each request at its arrival time (seconds from the start), steps while there is work, and returns
    (images/s, latencies in s)."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    done, sub, nxt = {}, {}, 0
    while len(done) < len(reqs):
        now = time.perf_counter() - t0
        while nxt < len(reqs) and arrivals[nxt] <= now:
            sub[server.submit(reqs[nxt])] = arrivals[nxt]
            nxt += 1
        if server.pending():
            out = server.step()
            if out:
                torch.cuda.synchronize()
                t = time.perf_counter() - t0
                done.update({k: t for k in out})
        elif nxt < len(reqs):
            time.sleep(max(0.0, arrivals[nxt] - (time.perf_counter() - t0)))
    lat = sorted(done[k] - sub[k] for k in done)
    return len(reqs) / (max(done.values()) - arrivals[0]), lat


def pct(v, p):
    return v[min(len(v) - 1, int(round(p / 100 * (len(v) - 1))))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, default=4)
    ap.add_argument("--requests", type=int, default=32)
    ap.add_argument("--garments", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--load", type=float, default=0.9)
    ap.add_argument("--kv-gb", type=float, default=40,
                    help="garment K/V budget of batch mode's cache and of the pool (GB, 1e9 bytes)")
    ap.add_argument("--garment-kv", default="fp16", choices=("fp16", "fp8"), dest="garment_kv",
                    help="precision of the hoisted garment K/V (cache entries and pool pages)")
    args = ap.parse_args()
    kv_bytes = int(args.kv_gb * 1e9)
    from idm_vton_b200 import lib as L
    from idm_vton_b200.denoise import TryOnDenoiser
    from idm_vton_b200.engine import SDXL_GARMENT, SDXL_TRYON
    from idm_vton_b200.scheduler import DDPMScheduler
    from idm_vton_b200.serving import ContinuousTryOnServer, TryOnServer
    assert torch.cuda.is_available(), "continuous_timing needs a GPU"
    L.load()
    dev = torch.device("cuda", 0)
    S = args.slots
    unet, unet_enc, _ = bench.build_components(dev, 0, 1, lambda m: None)
    pipe = bench.make_pipeline(unet, unet_enc, dev)
    out = {"card": card(), "config": f"768x1024, DDPM {T} steps, guidance 2.0, random SDXL weights, S = {S}, "
                                      f"{args.requests} requests over {args.garments} garments, "
                                      f"garment K/V {args.garment_kv}"}
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731

    # the step at full occupancy: continuous (S slots, per-slot garment passes) vs batch (S persons, one garment,
    # its hoisted garment passes spread over the steps)
    cont = ContinuousTryOnServer(pipe, height=H, width=W, slots=S, num_inference_steps=T, guidance_scale=2.0, seed=7)
    for r in make_requests(S, S, dev, seed=1):
        cont.submit(r)
    cont.step()                                                # admits all, captures the graph
    e0, e1 = ev(), ev()
    e0.record()
    for _ in range(10):
        cont.den.step([5] * S)
    e1.record()
    torch.cuda.synchronize()
    cont_step = e0.elapsed_time(e1) / 10
    del cont
    torch.cuda.empty_cache()
    # the garment K/V format from here on (the default continuous server above, which holds no garment K/V, sets the
    # arrival rate in either format; with fp8 it is not a mode of the trace: it refuses FP8 garment K/V)
    pipe.set_garment_kv_precision(args.garment_kv)
    # the same for pool mode (S garments filled at admission), then the time of one page fill
    pool = ContinuousTryOnServer(pipe, height=H, width=W, slots=S, num_inference_steps=T, guidance_scale=2.0, seed=7,
                                 garment_kv_bytes=kv_bytes)
    reqs = make_requests(S, S, dev, seed=1)
    for r in reqs:
        pool.submit(r)
    pool.step()
    e0, e1 = ev(), ev()
    e0.record()
    for _ in range(10):
        pool.den.step([5] * S)
    e1.record()
    torch.cuda.synchronize()
    pool_step = e0.elapsed_time(e1) / 10
    g = pool.garments[reqs[0].garment_id]
    fills = []
    for _ in range(3):
        e0, e1 = ev(), ev()
        e0.record()
        pool.den.fill_page(pool.den.P - 1, g["latents"], g["text_embeds_cloth"])
        e1.record()
        torch.cuda.synchronize()
        fills.append(e0.elapsed_time(e1))
    out["pool"] = dict(pages=pool.den.P, page_bytes=pool.page_bytes(), fill_ms=[round(f, 1) for f in fills])
    del pool, g
    torch.cuda.empty_cache()
    req = bench.synth_request(SDXL_TRYON, SDXL_GARMENT, S, H // 8, W // 8, seed=42, device=dev, garments=1)
    den = TryOnDenoiser(unet.engine(), unet_enc.engine())
    sch = DDPMScheduler()
    sch.set_timesteps(T)
    den.prepare(**req, guidance_scale=2.0)
    den.set_step_tables(sch, sch.timesteps)
    den.step(0, None)
    e0, e1, e2 = ev(), ev(), ev()
    e0.record()
    den.set_step_tables(sch, sch.timesteps)
    e1.record()
    for i in range(10):
        den.step(i, None)
    e2.record()
    torch.cuda.synchronize()
    batch_garment, batch_step = e0.elapsed_time(e1), e1.elapsed_time(e2) / 10
    del den
    out["step_ms"] = dict(continuous_full=round(cont_step, 2), continuous_pool_full=round(pool_step, 2),
                          batch=round(batch_step, 2),
                          batch_garment_passes_per_step=round(batch_garment / T, 2),
                          batch_total=round(batch_step + batch_garment / T, 2))

    # the arrival trace
    capacity = S / (T * cont_step / 1e3)                        # images/s of a full continuous server's loop
    rate = args.load * capacity
    g = torch.Generator().manual_seed(2024)
    gaps = -torch.log(1 - torch.rand(args.requests, generator=g)) / rate
    arrivals = torch.cumsum(gaps, 0).tolist()
    arrivals = [a - arrivals[0] for a in arrivals]
    out["arrival_rate_per_s"] = round(rate, 3)
    modes = {
        "batch": lambda: TryOnServer(pipe, height=H, width=W, num_inference_steps=T, guidance_scale=2.0, max_batch=S,
                                     seed=7, garment_cache_bytes=kv_bytes),
        "continuous": lambda: ContinuousTryOnServer(pipe, height=H, width=W, slots=S, num_inference_steps=T,
                                                    guidance_scale=2.0, seed=7),
        "continuous_pool": lambda: ContinuousTryOnServer(pipe, height=H, width=W, slots=S, num_inference_steps=T,
                                                         guidance_scale=2.0, seed=7, garment_kv_bytes=kv_bytes),
    }
    if args.garment_kv == "fp8":
        del modes["continuous"]
    import gc

    def fresh(name):
        """A new server of mode `name`, after the previous servers' denoisers, graphs and garment cache are released."""
        pipe.garment_cache = None
        pipe._denoiser = None
        gc.collect()
        torch.cuda.empty_cache()
        return modes[name]()

    warm = make_requests(S, 2, dev, seed=3)
    for name in modes:                                         # warm-up: kernels, VAE / CLIP twins
        srv = fresh(name)
        for r in warm:
            srv.submit(r)
        srv.run()
        del srv
    res = {n: [] for n in modes}
    pages = []
    for _ in range(args.rounds):
        for name in modes:
            srv = fresh(name)
            res[name].append(serve(srv, make_requests(args.requests, args.garments, dev, seed=5), arrivals))
            if name == "continuous_pool":
                pages.append((srv.stats["garment_page_fills"], srv.stats["garment_page_hits"]))
            del srv
    for name, runs in res.items():
        out[name] = dict(images_per_s=[round(r[0], 3) for r in runs],
                         latency_p50_s=[round(pct(r[1], 50), 2) for r in runs],
                         latency_p95_s=[round(pct(r[1], 95), 2) for r in runs])
    out["continuous_pool"].update(garment_page_fills=[f for f, _ in pages], garment_page_hits=[h for _, h in pages],
                                  hit_rate=[round(h / max(1, f + h), 3) for f, h in pages])
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
