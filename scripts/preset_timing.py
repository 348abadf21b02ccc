"""Sampling presets on one GPU, at config-2 geometry (768x1024, guidance 2.0) with random SDXL-shaped weights as bench.py
builds them.

A seeded Poisson arrival trace of `--requests` requests over `--garments` garments, each request picking "quality"
(DDPM 30 steps) or "fast" (DPM-Solver++ 15 steps) at 50/50, goes through two modes, alternated in one process
(`--rounds` rounds after a warm-up of each):
  mixed:   ContinuousTryOnServer(slots=S, presets={quality, fast}): both presets in one batch (mixed-kind step kernel);
  single:  ContinuousTryOnServer(slots=S) without presets: every request at DDPM 30, what one server can offer
           without presets.
`--kv-gb` runs both in pool mode with that garment K/V budget. The arrival rate is `--load` times the capacity of a
full single server. Prints one JSON line with, per mode, images/s and p50 / p95 latency per preset (in single mode the
preset the request asked for); the step time at full occupancy of the mixed path against the per-kind path at the same
S; the time of cfg_step_mixed_rows against cfg_ddpm_step_rows / cfg_solver_step_rows over 200 launches at S samples;
the card's name and power limit, read in the same run.
Usage: python scripts/preset_timing.py [--slots 4] [--requests 16] [--garments 4] [--rounds 2] [--kv-gb 40]"""
import argparse
import gc
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import idm_vton_b200  # noqa: F401,E402
import bench  # noqa: E402
from scripts.continuous_timing import H, W, make_requests, pct  # noqa: E402
from scripts.schedule_timing import card  # noqa: E402


def presets():
    from idm_vton_b200.scheduler import DDPMScheduler, DPMSolverMultistepScheduler
    from idm_vton_b200.serving import SamplingPreset
    return {"quality": SamplingPreset(DDPMScheduler(), 30),
            "fast": SamplingPreset(DPMSolverMultistepScheduler.from_config(DDPMScheduler().config), 15)}


def serve(server, reqs, arrivals, asked):
    """Submits each request at its arrival time, steps while there is work; returns (images/s, {preset: latencies})."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    done, sub, nxt = {}, {}, 0
    while len(done) < len(reqs):
        now = time.perf_counter() - t0
        while nxt < len(reqs) and arrivals[nxt] <= now:
            sub[server.submit(reqs[nxt])] = (arrivals[nxt], asked[nxt])
            nxt += 1
        if server.pending():
            out = server.step()
            if out:
                torch.cuda.synchronize()
                t = time.perf_counter() - t0
                done.update({k: t for k in out})
        elif nxt < len(reqs):
            time.sleep(max(0.0, arrivals[nxt] - (time.perf_counter() - t0)))
    lat = {}
    for k, t in done.items():
        lat.setdefault(sub[k][1], []).append(t - sub[k][0])
    return len(reqs) / (max(done.values()) - arrivals[0]), {p: sorted(v) for p, v in lat.items()}


def kernel_ms(S, ev):
    """cfg_step_mixed_rows (half DDPM, half DPM-Solver++ rows) against the per-kind rows kernels at S samples of
    config-2 latents, 200 launches each after a warm-up."""
    from idm_vton_b200 import lib as L
    h, w = H // 8, W // 8
    g = torch.Generator(device="cuda").manual_seed(0)
    eps = torch.randn(2 * S, h, w, 4, generator=g, device="cuda").half()
    lat = torch.randn(S, 4, h, w, generator=g, device="cuda").half()
    noise, x0p, out = torch.randn_like(lat), torch.zeros_like(lat), torch.empty_like(lat)
    coef = torch.rand(S, 8, generator=g, device="cuda")
    coef[:, 6] = 0.0
    kinds = torch.tensor([3 if s % 2 == 0 else 2 for s in range(S)], dtype=torch.int32, device="cuda")
    runs = {"mixed": lambda: L.cfg_step_mixed_rows(eps, lat, noise, coef, kinds, x0p, out=out),
            "ddpm_rows": lambda: L.cfg_ddpm_step_rows(eps, lat, noise, coef, out=out),
            "dpmpp_rows": lambda: L.cfg_solver_step_rows(eps, lat, None, coef, "dpmpp", x0_prev=x0p, out=out)}
    res = {}
    for name, fn in runs.items():
        for _ in range(20):
            fn()
        e0, e1 = ev(), ev()
        e0.record()
        for _ in range(200):
            fn()
        e1.record()
        torch.cuda.synchronize()
        res[name] = round(e0.elapsed_time(e1) / 200 * 1e3, 2)      # us per launch
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, default=4)
    ap.add_argument("--requests", type=int, default=16)
    ap.add_argument("--garments", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--load", type=float, default=0.9)
    ap.add_argument("--kv-gb", type=float, default=None, help="pool mode with this garment K/V budget (GB, 1e9 bytes)")
    args = ap.parse_args()
    kv = None if args.kv_gb is None else int(args.kv_gb * 1e9)
    from idm_vton_b200 import lib as L
    from idm_vton_b200.serving import ContinuousTryOnServer
    assert torch.cuda.is_available(), "preset_timing needs a GPU"
    L.load()
    dev = torch.device("cuda", 0)
    S = args.slots
    unet, unet_enc, _ = bench.build_components(dev, 0, 1, lambda m: None)
    pipe = bench.make_pipeline(unet, unet_enc, dev)
    out = {"card": card(), "config": f"768x1024, guidance 2.0, random SDXL weights, S = {S}, {args.requests} requests "
                                      f"over {args.garments} garments, quality = DDPM 30, fast = DPM-Solver++ 15, "
                                      f"{'pool ' + str(args.kv_gb) + ' GB' if kv else 'default mode'}"}
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    modes = {"mixed": lambda: ContinuousTryOnServer(pipe, height=H, width=W, slots=S, seed=7, garment_kv_bytes=kv,
                                                    presets=presets(), default_preset="quality"),
             "single": lambda: ContinuousTryOnServer(pipe, height=H, width=W, slots=S, num_inference_steps=30,
                                                     guidance_scale=2.0, seed=7, garment_kv_bytes=kv)}

    def fresh(name):
        pipe._denoiser = None
        gc.collect()
        torch.cuda.empty_cache()
        return modes[name]()

    # full-occupancy step: mixed path (half the slots on each preset) against the per-kind path, same S
    step_ms = {}
    for name in modes:
        srv = fresh(name)
        reqs = make_requests(S, S, dev, seed=1)
        for k, r in enumerate(reqs):
            r.sampling = ("quality", "fast")[k % 2] if name == "mixed" else None
        for r in reqs:
            srv.submit(r)
        srv.step()                                                 # admits all, captures the graph
        steps = [(k % 2, 5) for k in range(S)] if name == "mixed" else [5] * S
        e0, e1 = ev(), ev()
        e0.record()
        for _ in range(10):
            srv.den.step(steps)
        e1.record()
        torch.cuda.synchronize()
        step_ms[name] = round(e0.elapsed_time(e1) / 10, 2)
        del srv
    out["step_ms_full"] = step_ms
    out["step_kernel_us"] = kernel_ms(S, ev)

    capacity = S / (30 * step_ms["single"] / 1e3)
    rate = args.load * capacity
    g = torch.Generator().manual_seed(2024)
    gaps = -torch.log(1 - torch.rand(args.requests, generator=g)) / rate
    arrivals = torch.cumsum(gaps, 0).tolist()
    arrivals = [a - arrivals[0] for a in arrivals]
    asked = ["quality" if x < 0.5 else "fast" for x in torch.rand(args.requests, generator=g).tolist()]
    out["arrival_rate_per_s"] = round(rate, 3)
    out["asked"] = {p: asked.count(p) for p in ("quality", "fast")}

    def trace(name, seed):
        reqs = make_requests(args.requests, args.garments, dev, seed=seed)
        for r, p in zip(reqs, asked):
            r.sampling = p if name == "mixed" else None
        return reqs
    for name in modes:                                             # warm-up
        srv = fresh(name)
        for r in trace(name, 3)[:S]:
            srv.submit(r)
        srv.run()
        del srv
    res = {n: [] for n in modes}
    for _ in range(args.rounds):
        for name in modes:
            srv = fresh(name)
            res[name].append(serve(srv, trace(name, 5), arrivals, asked))
            if kv:
                res[name][-1] += (dict(fills=srv.stats["garment_page_fills"], hits=srv.stats["garment_page_hits"]),)
            del srv
    for name, runs in res.items():
        out[name] = dict(images_per_s=[round(r[0], 3) for r in runs],
                         **{f"{p}_latency_p50_s": [round(pct(r[1][p], 50), 2) for r in runs] for p in ("quality", "fast")},
                         **{f"{p}_latency_p95_s": [round(pct(r[1][p], 95), 2) for r in runs] for p in ("quality", "fast")})
        if kv:
            out[name]["pages"] = [r[2] for r in runs]
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
