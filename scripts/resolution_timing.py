"""Denoise-loop time per megapixel at image sizes that are not multiples of 32 and with the garment at its own size
(random SDXL-shaped weights as in bench.py, batch 1, guidance 2.0, DDPM 30 steps), on one GPU, with device events.
Prints one JSON line with the card's name and power limit, read in the same run:
  loop_ms:         set_step_tables (the hoisted garment passes) + every step replayed from the captured graph, the
                   geometries alternated in `--rounds` rounds after a warm-up loop of each;
  ms_per_mpix:     median loop_ms / person megapixels;
  garment_ms:      the hoisted garment passes alone (set_step_tables), median;
  step_ms:         one replayed step graph (try-on UNet + the fused step), median over the loop's steps.
Geometries: person 768x1024 against 720x960 (latents 96x128 vs 90x120: the up path resizes to the skips, and the 45x60 /
23x30 levels run convolution boxes of odd width), and person 576x768 with the cloth at 768x1024 against the cloth at 576x768.
Usage: python scripts/resolution_timing.py [--rounds 3]"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import idm_vton_b200  # noqa: F401,E402
import bench  # noqa: E402
from scripts.schedule_timing import card  # noqa: E402

# name -> ((person H, W), (cloth H, W)) in pixels
GEOMETRIES = {
    "person_768x1024": ((1024, 768), (1024, 768)),
    "person_720x960": ((960, 720), (960, 720)),
    "person_576x768_cloth_768x1024": ((768, 576), (1024, 768)),
    "person_576x768_cloth_576x768": ((768, 576), (768, 576)),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    from idm_vton_b200 import lib as L
    from idm_vton_b200.denoise import TryOnDenoiser
    from idm_vton_b200.engine import SDXL_GARMENT, SDXL_TRYON
    from idm_vton_b200.scheduler import DDPMScheduler
    assert torch.cuda.is_available(), "resolution_timing needs a GPU"
    L.load()
    dev = torch.device("cuda", 0)
    B = 1
    unet, unet_enc, _ = bench.build_components(dev, 0, 1, lambda m: None)
    out = {"card": card(), "config": "batch 1, guidance 2.0, DDPM 30 steps, random SDXL weights"}
    reqs, dens = {}, {}
    for name, ((H, W), (Hc, Wc)) in GEOMETRIES.items():
        req = bench.synth_request(SDXL_TRYON, SDXL_GARMENT, B, H // 8, W // 8, seed=42, device=dev)
        if (Hc, Wc) != (H, W):
            g = torch.Generator(device=dev).manual_seed(43)
            req["cloth_latents"] = torch.randn(B, 4, Hc // 8, Wc // 8, generator=g, device=dev,
                                               dtype=req["cloth_latents"].dtype)
        reqs[name] = req
        dens[name] = TryOnDenoiser(unet.engine(), unet_enc.engine())     # one captured graph per geometry
    sch = DDPMScheduler()
    sch.set_timesteps(30)

    def loop(name):
        d = dens[name]
        d.prepare(**reqs[name], guidance_scale=bench.GUIDANCE)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(sch.timesteps) + 2)]
        torch.cuda.synchronize()
        ev[0].record()
        d.set_step_tables(sch, sch.timesteps)
        ev[1].record()
        for i in range(len(sch.timesteps)):
            d.step(i, None)
            ev[i + 2].record()
        torch.cuda.synchronize()
        steps = sorted(ev[i + 1].elapsed_time(ev[i + 2]) for i in range(1, len(sch.timesteps)))
        return ev[0].elapsed_time(ev[-1]), ev[0].elapsed_time(ev[1]), steps[len(steps) // 2]

    for n in GEOMETRIES:
        loop(n)                                   # capture + warm-up of each geometry
    res = {n: [] for n in GEOMETRIES}
    for _ in range(args.rounds):
        for n in GEOMETRIES:
            res[n].append(loop(n))
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    out["loop_ms"] = {n: [round(r[0], 1) for r in v] for n, v in res.items()}
    out["ms_per_mpix"] = {n: round(med([r[0] for r in v]) / (GEOMETRIES[n][0][0] * GEOMETRIES[n][0][1] / 1e6), 1)
                          for n, v in res.items()}
    out["garment_ms"] = {n: round(med([r[1] for r in v]), 1) for n, v in res.items()}
    out["step_ms"] = {n: round(med([r[2] for r in v]), 2) for n, v in res.items()}
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
