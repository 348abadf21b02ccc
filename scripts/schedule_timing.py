"""Cost of the denoising-schedule features at config 2 (768x1024, batch 2, guidance 2.0, 30 steps; random SDXL-shaped
weights as in bench.py) on one GPU, with device events. Prints one JSON line with the card's name and power limit:
  step_ms:    one denoise step replayed from its CUDA graph, guidance_rescale 0 (plain CFG + DDPM kernel) and 0.7 (the fused
              rescale kernel), two denoisers on the same weights timed in alternating blocks;
  kernel_us:  the last kernel of the step alone, b200vton_cfg_ddpm_step vs b200vton_cfg_rescale_ddpm_step;
  call_ms:    one pipeline __call__ at strength 1.0 and 0.5 (the latter runs 15 of 30 steps and their garment passes),
              alternated after a warm-up call of each.
Usage: python scripts/schedule_timing.py [--rounds 4]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import idm_vton_b200  # noqa: F401,E402
import bench  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def events_ms(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=4)
    args = ap.parse_args()
    from idm_vton_b200 import lib as L
    from idm_vton_b200.denoise import TryOnDenoiser
    from idm_vton_b200.engine import SDXL_GARMENT, SDXL_TRYON
    from idm_vton_b200.scheduler import DDPMScheduler
    assert torch.cuda.is_available(), "schedule_timing needs a GPU"
    L.load()
    dev = torch.device("cuda", 0)
    B, H, W, T = 2, 1024, 768, 30
    h, w = H // 8, W // 8
    unet, unet_enc, _ = bench.build_components(dev, 0, 1, lambda m: None)
    req = bench.synth_request(SDXL_TRYON, SDXL_GARMENT, B, h, w, seed=42, device=dev)
    sch = DDPMScheduler()
    sch.set_timesteps(T)
    out = {"card": card(), "config": "768x1024, batch 2, guidance 2.0, 30 steps"}

    # ---- per-step graph replay, phi = 0 vs 0.7
    dens = {}
    for phi in (0.0, 0.7):
        d = TryOnDenoiser(unet.engine(), unet_enc.engine())
        d.prepare(**req, guidance_scale=bench.GUIDANCE, guidance_rescale=phi)
        d.set_step_tables(sch, sch.timesteps)
        noise = torch.randn(d.latents.shape, generator=torch.Generator(device=dev).manual_seed(1), device=dev,
                            dtype=torch.float16)
        d.step(0, noise)                              # capture + warm-up
        dens[phi] = (d, noise)
    torch.cuda.synchronize()
    per = {0.0: [], 0.7: []}
    for _ in range(args.rounds):
        for phi, (d, noise) in dens.items():
            per[phi].append(events_ms(lambda: d.step(5, noise), 10))
    out["step_ms"] = {f"phi={phi}": [round(x, 3) for x in v] for phi, v in per.items()}
    out["step_ms_median"] = {f"phi={phi}": round(sorted(v)[len(v) // 2], 3) for phi, v in per.items()}

    # ---- the step's last kernel alone
    d, noise = dens[0.7]
    coef = torch.cat([d.coef_table[5, :6], torch.tensor([0.7], device=dev)]).contiguous()
    eps = d.eps
    kern = {"cfg_ddpm_step": lambda: L.cfg_ddpm_step(eps, d.latents, noise, coef, out=d.latents_next),
            "cfg_rescale_ddpm_step": lambda: L.cfg_rescale_ddpm_step(eps, d.latents, noise, coef, out=d.latents_next)}
    for fn in kern.values():
        events_ms(fn, 20)
    ks = {k: [] for k in kern}
    for _ in range(args.rounds):
        for k, fn in kern.items():
            ks[k].append(events_ms(fn, 200) * 1e3)
    out["kernel_us"] = {k: round(sorted(v)[len(v) // 2], 2) for k, v in ks.items()}
    del dens, d, eps
    torch.cuda.empty_cache()

    # ---- one __call__ at strength 1.0 and 0.5
    pipe = bench.make_pipeline(unet, unet_enc, dev)
    g = torch.Generator().manual_seed(7)
    host = dict(image=torch.rand(B, 3, H, W, generator=g), mask_image=(torch.rand(B, 1, H, W, generator=g) > 0.5).float(),
                pose_img=torch.rand(B, 3, H, W, generator=g) * 2 - 1, cloth=torch.rand(B, 3, H, W, generator=g) * 2 - 1,
                ip_adapter_image=torch.randn(B, 3, 224, 224, generator=g),
                prompt_embeds=torch.randn(B, 77, 2048, generator=g).half(),
                negative_prompt_embeds=torch.randn(B, 77, 2048, generator=g).half(),
                pooled_prompt_embeds=torch.randn(B, 1280, generator=g).half(),
                negative_pooled_prompt_embeds=torch.randn(B, 1280, generator=g).half(),
                text_embeds_cloth=torch.randn(B, 77, 2048, generator=g).half())
    dv = {k: v.to(dev) for k, v in host.items()}

    def call(strength):
        torch.cuda.synchronize()
        t0 = time.time()
        pipe(**dv, num_inference_steps=T, generator=torch.Generator(dev).manual_seed(42), strength=strength, height=H,
             width=W, guidance_scale=bench.GUIDANCE, output_type="pt")
        torch.cuda.synchronize()
        return (time.time() - t0) * 1e3

    calls = {1.0: [], 0.5: []}
    for s in calls:
        call(s)
    for _ in range(2):
        for s in calls:
            calls[s].append(call(s))
    out["call_ms"] = {f"strength={s}": [round(x, 1) for x in v] for s, v in calls.items()}
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
