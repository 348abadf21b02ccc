"""Images/s of the denoise loop at config 2 (768x1024, batch 2, guidance 2.0; random SDXL-shaped weights as in bench.py)
for DDPM at 30 steps against DPM-Solver++(2M) at 15 and 20 steps, on one GPU, with device events. Prints one JSON line
with the card's name and power limit, read in the same run:
  loop_ms:    set_step_tables (the hoisted garment passes) + every step replayed from the captured graph, the three
              schedules alternated in `--rounds` rounds after a warm-up loop of each; images_per_s = batch / loop time;
  kernel_us:  the step's last kernel alone over 200 launches: b200vton_cfg_ddpm_step and b200vton_cfg_solver_step per kind.
Image quality at fewer steps is not measured here (random weights).
Usage: python scripts/solver_timing.py [--rounds 3]"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import idm_vton_b200  # noqa: F401,E402
import bench  # noqa: E402
from scripts.schedule_timing import card, events_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    from idm_vton_b200 import lib as L
    from idm_vton_b200.denoise import TryOnDenoiser
    from idm_vton_b200.engine import SDXL_GARMENT, SDXL_TRYON
    from idm_vton_b200.scheduler import DDPMScheduler, DPMSolverMultistepScheduler
    assert torch.cuda.is_available(), "solver_timing needs a GPU"
    L.load()
    dev = torch.device("cuda", 0)
    B, H, W = 2, 1024, 768
    h, w = H // 8, W // 8
    unet, unet_enc, _ = bench.build_components(dev, 0, 1, lambda m: None)
    req = bench.synth_request(SDXL_TRYON, SDXL_GARMENT, B, h, w, seed=42, device=dev)
    out = {"card": card(), "config": "768x1024, batch 2, guidance 2.0"}

    def schedule(name):
        if name == "ddpm_30":
            s = DDPMScheduler()
            s.set_timesteps(30)
        else:
            s = DPMSolverMultistepScheduler.from_config(DDPMScheduler().config)
            s.set_timesteps(int(name.split("_")[1]))
        return s

    names = ("ddpm_30", "dpmpp2m_15", "dpmpp2m_20")
    # one denoiser per schedule: switching the scheduler kind on one denoiser re-captures its graph
    dens = {n: TryOnDenoiser(unet.engine(), unet_enc.engine()) for n in names}
    noise = torch.randn(B, 4, h, w, generator=torch.Generator(device=dev).manual_seed(1), device=dev, dtype=torch.float16)

    def loop(name):
        s = schedule(name)
        d = dens[name]
        d.prepare(**req, guidance_scale=bench.GUIDANCE)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        d.set_step_tables(s, s.timesteps)
        for i, t in enumerate(s.timesteps):
            d.step(i, noise if d.step_draws[i] and d.noise_applied else None)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    for n in names:
        loop(n)                                  # capture + warm-up of each schedule
    ms = {n: [] for n in names}
    for _ in range(args.rounds):
        for n in names:
            ms[n].append(loop(n))
    med = {n: sorted(v)[len(v) // 2] for n, v in ms.items()}
    out["loop_ms"] = {n: [round(x, 1) for x in v] for n, v in ms.items()}
    out["images_per_s"] = {n: round(B / (m / 1e3), 4) for n, m in med.items()}

    d = dens["ddpm_30"]
    eps = d.eps
    coef = torch.zeros(8, dtype=torch.float32, device=dev)
    coef[:6] = torch.tensor([2.0, 0.8, 1.6, 0.3, 0.7, 0.1])
    st = torch.zeros_like(d.latents)
    kern = {"cfg_ddpm_step": lambda: L.cfg_ddpm_step(eps, d.latents, noise, coef, out=d.latents_next)}
    for kind in ("ddim", "euler", "dpmpp"):
        kern[f"cfg_solver_step[{kind}]"] = (lambda k=kind: L.cfg_solver_step(
            eps, d.latents, noise if k == "ddim" else None, coef, k, x0_prev=st, out=d.latents_next))
    for fn in kern.values():
        events_ms(fn, 20)
    ks = {k: [] for k in kern}
    for _ in range(args.rounds):
        for k, fn in kern.items():
            ks[k].append(events_ms(fn, 200) * 1e3)
    out["kernel_us"] = {k: round(sorted(v)[len(v) // 2], 2) for k, v in ks.items()}
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
