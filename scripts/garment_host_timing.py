"""The host tier of the garment K/V pool on one GPU, at config-2 geometry (768x1024, DDPM 30 steps, guidance 2.0) with
random SDXL-shaped weights as bench.py builds them. Prints one JSON line with, beside the card's name and power limit
(read in the same run):
  1. rows: the host-to-device and device-to-host rates of one row's block copies (one cudaMemcpyAsync per block, and
     one more per block for the fp8 exponents) between page-locked host memory and the pool, timed with device events
     over `--row-reps` rows, and the host time to issue one row's copies;
  2. step_ms: the full-occupancy step (S = `--slots`) with 0..S of its slots streaming from the host tier and the rest
     reading device pages, every streaming slot's next row copied beside the step as the server does; the counts are
     alternated over `--rounds` rounds of `--steps` steps;
  3. trace: a catalog trace in scripts/continuous_timing.py's style, `--requests` requests over `--garments` garments
     (more than the device budget `--kv-gb` holds), served with and without a host tier of `--host-gb` GB (capped at
     half of MemAvailable in /proc/meminfo), alternated over `--trace-rounds` rounds: fills and hits per tier,
     images/s and p50 / p95 latency.
Every page-locked byte is released before exit.
Usage: python scripts/garment_host_timing.py [--garment-kv fp16|fp8] [--slots 4] [--kv-gb 40] [--host-gb 120]
       [--garments 24] [--requests 48] [--trace-rounds 1] [--skip-trace]"""
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
from scripts.continuous_timing import make_requests, pct, serve  # noqa: E402
from scripts.schedule_timing import card  # noqa: E402

H, W, T = 1024, 768, 30


def mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    raise RuntimeError("no MemAvailable in /proc/meminfo")


def row_rates(den, reps):
    """(H2D GB/s, D2H GB/s, host us to issue one row's H2D copies, bytes per row) over `reps` rows."""
    from idm_vton_b200.denoise import copy_kv_rows
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    stream = torch.cuda.Stream()
    Tp, ring, Q = den.T_page, den.ring, den.Q
    nbytes, issue = 0, []
    with torch.cuda.stream(stream):
        for host_kv, kv in zip(den.host.blocks, den.pool):   # warm-up
            copy_kv_rows(kv, ring, host_kv, 0)
        stream.synchronize()
        e0, e1 = ev(), ev()
        e0.record(stream)
        for r in range(reps):
            t0 = time.perf_counter()
            n = 0
            for host_kv, kv in zip(den.host.blocks, den.pool):
                n += copy_kv_rows(kv, ring + (r & 1), host_kv, r % (Q * Tp))
            issue.append(time.perf_counter() - t0)
            nbytes = n
        e1.record(stream)
        stream.synchronize()
        h2d = reps * nbytes / (e0.elapsed_time(e1) / 1e3) / 1e9
        e0.record(stream)
        for r in range(reps):
            for host_kv, kv in zip(den.host.blocks, den.pool):
                copy_kv_rows(host_kv, r % (Q * Tp), kv, ring + (r & 1))
        e1.record(stream)
        stream.synchronize()
        d2h = reps * nbytes / (e0.elapsed_time(e1) / 1e3) / 1e9
    issue.sort()
    return h2d, d2h, 1e6 * issue[len(issue) // 2], nbytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--garment-kv", default="fp8", choices=("fp16", "fp8"), dest="garment_kv")
    ap.add_argument("--slots", type=int, default=4)
    ap.add_argument("--kv-gb", type=float, default=40, help="device pool budget (GB, 1e9 bytes)")
    ap.add_argument("--host-gb", type=float, default=120, help="host tier budget (GB), capped at MemAvailable / 2")
    ap.add_argument("--row-reps", type=int, default=60)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--garments", type=int, default=24)
    ap.add_argument("--requests", type=int, default=48)
    ap.add_argument("--trace-rounds", type=int, default=1)
    ap.add_argument("--load", type=float, default=0.9)
    ap.add_argument("--skip-trace", action="store_true")
    args = ap.parse_args()
    from idm_vton_b200 import lib as L
    from idm_vton_b200.serving import ContinuousTryOnServer
    assert torch.cuda.is_available(), "garment_host_timing needs a GPU"
    L.load()
    dev = torch.device("cuda", 0)
    S = args.slots
    unet, unet_enc, _ = bench.build_components(dev, 0, 1, lambda m: None)
    pipe = bench.make_pipeline(unet, unet_enc, dev)
    pipe.set_garment_kv_precision(args.garment_kv)
    avail = mem_available()
    host_bytes = int(min(args.host_gb * 1e9, avail // 2))
    kv_bytes = int(args.kv_gb * 1e9)
    out = {"card": card(), "config": f"768x1024, DDPM {T} steps, guidance 2.0, random SDXL weights, S = {S}, garment "
                                     f"K/V {args.garment_kv}", "mem_available_bytes": avail}
    mk = lambda host: ContinuousTryOnServer(pipe, height=H, width=W, slots=S, num_inference_steps=T,  # noqa: E731
                                            guidance_scale=2.0, seed=7, garment_kv_bytes=kv_bytes,
                                            garment_kv_host_bytes=host)

    # 1-2: S device pages filled and written through; slots then read either their page or its host copy
    srv = mk(host_bytes)
    reqs = make_requests(S, S, dev, seed=1)
    for r in reqs:
        srv.submit(r)
    srv.step()
    den = srv.den
    torch.cuda.synchronize()
    out["pages"] = dict(device=den.P, host=den.Q, page_bytes=srv.page_bytes(), host_bytes=den.host.bytes,
                        ring_rows=2 * S)
    h2d, d2h, issue_us, row_bytes = row_rates(den, args.row_reps)
    out["rows"] = dict(row_bytes=row_bytes, h2d_GBps=round(h2d, 2), d2h_GBps=round(d2h, 2),
                       issue_us_median=round(issue_us, 1), copies_per_row=sum(len(x) if isinstance(x, tuple) else 1
                                                                              for x in den.pool))
    pages = [srv.slots[s]["page"] for s in range(S)]
    host_of = [srv.host_page_of[srv.slots[s]["req"].garment_id] for s in range(S)]
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    times = {k: [] for k in range(S + 1)}
    for _ in range(args.rounds):
        for k in range(S + 1):                                # slots 0..k-1 stream, the others read device pages
            for s in range(S):
                den.page[s], den.host_page[s] = (None, host_of[s]) if s < k else (pages[s], None)
            if k:
                den._stream_rows([(s, 0) for s in range(k)], after_last_step=True)
            den.step([0] * S)                                 # warm
            e0, e1 = ev(), ev()
            e0.record()
            for i in range(1, args.steps + 1):
                den.step([i] * S)
            e1.record()
            torch.cuda.synchronize()
            times[k].append(round(e0.elapsed_time(e1) / args.steps, 2))
            den.take_streamed()
    out["step_ms"] = {f"{k}_streaming": v for k, v in times.items()}
    for s in range(S):
        den.page[s], den.host_page[s] = pages[s], None
    srv.run()
    srv.close()
    del srv, den

    # 3: the catalog trace, with and without the host tier
    if not args.skip_trace:
        step_full = min(times[0]) / 1e3
        rate = args.load * S / (T * step_full)
        g = torch.Generator().manual_seed(2024)
        gaps = -torch.log(1 - torch.rand(args.requests, generator=g)) / rate
        arrivals = torch.cumsum(gaps, 0).tolist()
        arrivals = [a - arrivals[0] for a in arrivals]
        out["arrival_rate_per_s"] = round(rate, 3)
        res = {"device_only": [], "host_tier": []}
        for _ in range(args.trace_rounds):
            for name in res:
                pipe._denoiser = None
                torch.cuda.empty_cache()
                srv = mk(host_bytes if name == "host_tier" else None)
                try:
                    # configure outside the trace: page-locking the host tier is set-up, timed on its own
                    warm = make_requests(1, 1, dev, seed=9)[0]
                    warm.garment_id = "warm-up"
                    t0 = time.perf_counter()
                    srv.submit(warm)
                    srv.run()
                    torch.cuda.synchronize()
                    setup_s = time.perf_counter() - t0
                    srv.stats.clear()
                    ips, lat = serve(srv, make_requests(args.requests, args.garments, dev, seed=5), arrivals)
                    st = srv.stats
                    res[name].append(dict(setup_and_first_request_s=round(setup_s, 2), images_per_s=round(ips, 3), latency_p50_s=round(pct(lat, 50), 2),
                                          latency_p95_s=round(pct(lat, 95), 2),
                                          **{k: v for k, v in st.items() if k.startswith("garment")}))
                finally:
                    srv.close()
                del srv
        out["trace"] = dict(requests=args.requests, garments=args.garments, **res)
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
