"""FreeU on one GPU, with the card's name and power limit read in the same run:
  * kernel: the 6 b200vton_freeu_nhwc launches of one config-2 try-on step (768x1024, try-on batch 4: up stage 0 at
    32x24 with skips of 1280, 1280, 640 channels, stage 1 at 64x48 with 640, 640, 320), ms per launch from CUDA events
    around a replayed graph of `reps` launches, and GB/s against the bytes the shapes require (skip read and written
    once, the scaled half of hidden read and written once);
  * the reference's route on the same tensors (NCHW): diffusers' apply_freeu (oracle/freeu_ref.py), i.e. the fp32
    FFT round trip of the skip (24 and 48 are not powers of two) plus the in-place scaling, eager, CUDA events;
  * the config-2 denoise step (TryOnDenoiser with hoisted garment K/V, random SDXL weights as bench.py builds them)
    with FreeU off and on (SDXL values), alternated over --rounds rounds, --steps replays each.

    python scripts/freeu_timing.py [--reps 200] [--rounds 3] [--steps 20] [--out results/freeu_timing.json]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SDXL_FREEU = (0.9, 0.2, 1.3, 1.4)
# (stage, H, W, hidden channels, skip channels) of the 6 launches at config 2
LAUNCHES = [(0, 32, 24, 1280, 1280), (0, 32, 24, 1280, 1280), (0, 32, 24, 1280, 640),
            (1, 64, 48, 1280, 640), (1, 64, 48, 640, 640), (1, 64, 48, 640, 320)]
BATCH = 4


def _graph_ms(fn, reps):
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


def _eager_ms(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / reps


def kernels(reps):
    from idm_vton_b200 import lib as L
    from oracle import freeu_ref as FR
    s1, s2, b1, b2 = SDXL_FREEU
    rows, tot_k, tot_r, tot_bytes = [], 0.0, 0.0, 0
    g = torch.Generator(device="cuda").manual_seed(0)
    for stage, H, W, Ch, Cs in LAUNCHES:
        b, s = (b1, s1) if stage == 0 else (b2, s2)
        hidden = torch.randn(BATCH, H, W, Ch, device="cuda", generator=g).half()
        skip = torch.randn(BATCH, H, W, Cs, device="cuda", generator=g).half()
        out = torch.empty_like(skip)
        # b = 1 keeps hidden's values over the repeated launches (the work is the same for any b)
        ms = _graph_ms(lambda: L.freeu(hidden, skip, 1.0, s, out=out), reps)
        need = 2 * skip.numel() * 2 + 2 * (hidden.numel() // 2) * 2
        h_nchw = hidden.permute(0, 3, 1, 2).contiguous()
        s_nchw = skip.permute(0, 3, 1, 2).contiguous()
        ref_ms = _eager_ms(lambda: FR.apply_freeu(stage, h_nchw, s_nchw, s1=s1, s2=s2, b1=1.0, b2=1.0), reps)
        rows.append(dict(stage=stage, H=H, W=W, Ch=Ch, Cs=Cs, ms=round(ms, 5), MB=round(need / 1e6, 2),
                         GBps=round(need / ms / 1e6, 1), reference_ms=round(ref_ms, 4)))
        tot_k, tot_r, tot_bytes = tot_k + ms, tot_r + ref_ms, tot_bytes + need
        print(rows[-1], flush=True)
    return dict(launches=rows, kernel_ms_per_step=round(tot_k, 4), reference_ms_per_step=round(tot_r, 3),
                MB_per_step=round(tot_bytes / 1e6, 1), GBps_per_step=round(tot_bytes / tot_k / 1e6, 1))


def denoise_step(rounds, steps):
    import bench
    from idm_vton_b200.denoise import TryOnDenoiser
    from idm_vton_b200.engine import SDXL_GARMENT, SDXL_TRYON
    from idm_vton_b200.scheduler import DDPMScheduler
    unet, unet_enc, _ = bench.build_components(torch.device("cuda", 0), 0, 1, lambda m: None)
    req = bench.synth_request(SDXL_TRYON, SDXL_GARMENT, 2, 128, 96, seed=42, device="cuda")
    den = TryOnDenoiser(unet.engine(), unet_enc.engine())
    sch = DDPMScheduler()
    sch.set_timesteps(30)
    den.prepare(**req, guidance_scale=2.0)
    den.set_step_tables(sch, sch.timesteps)
    res = {"off": [], "on": []}
    for _ in range(rounds):
        for mode in ("off", "on"):
            if mode == "on":
                unet.enable_freeu(*SDXL_FREEU)
            else:
                unet.disable_freeu()
            den.step(5, None)                                  # re-captures the step for this setting
            torch.cuda.synchronize()
            res[mode].append(round(_eager_ms(lambda: den.step(5, None), steps), 3))
            print(mode, res[mode][-1], flush=True)
    unet.disable_freeu()
    return dict(step_ms=res, median_off=sorted(res["off"])[len(res["off"]) // 2],
                median_on=sorted(res["on"])[len(res["on"]) // 2])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("freeu_timing needs a CUDA device")
    from idm_vton_b200 import lib as L
    from scripts.schedule_timing import card
    L.load()
    out = dict(card=card(), kernels=kernels(args.reps))
    out["denoise_step_config2"] = denoise_step(args.rounds, args.steps)
    out["card_after"] = card()
    print(json.dumps(out))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
