"""Where the time of one config-2 denoise step goes (768x1024, batch 2, guidance 2.0, 30 steps; random SDXL-shaped
weights and `bench.synth_request` inputs, as in bench.py), measured with torch.profiler's CUDA activities around
  * one replay of the captured denoise step (garment K/V hoisted, as bench.py runs it), and
  * one `precompute_garment(0)`: the batched garment-UNet passes of all 30 steps plus their garment K/V.
Kernel time is grouped by family: flash_kernel<...> / gemm_conv_kernel<...> per template, GroupNorm, LayerNorm and the
rest ("elementwise"); `gaps_ms` is the time inside the region with no kernel running. Prints the card's name, power
limit and max SM clock read in the same run, and writes the full result as JSON to <out>/step_profile.json.
Usage: python scripts/step_profile.py --out DIR [--reps 3]"""
import argparse
import json
import os
import re
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import idm_vton_b200  # noqa: F401,E402
import bench  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def family(name):
    """Kernel family of a demangled kernel name: template kernels keep their template arguments."""
    for kern in ("flash_kernel", "gemm_conv_kernel"):
        m = re.search(kern + r"<[^(]*>", name)
        if m:
            return re.sub(r"\s+", "", m.group(0))
        if kern in name:
            return kern
    if "gn_fused_kernel" in name or "gn32_" in name:
        return "groupnorm"
    if "layernorm_kernel" in name:
        return "layernorm"
    return "elementwise"


def kernel_table(prof):
    """[(start_us, end_us, name)] of the device kernels the profiler recorded (memcpy / memset excluded)."""
    out = []
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        low = e.name.lower()
        if low.startswith("memcpy") or low.startswith("memset"):
            continue
        out.append((e.time_range.start, e.time_range.end, e.name))
    return sorted(out)


def summarise(kernels):
    fams = {}
    busy_end, gaps = None, 0.0
    for t0, t1, name in kernels:
        f = fams.setdefault(family(name), {"ms": 0.0, "launches": 0})
        f["ms"] += (t1 - t0) / 1e3
        f["launches"] += 1
        if busy_end is not None and t0 > busy_end:
            gaps += (t0 - busy_end) / 1e3
        busy_end = t1 if busy_end is None else max(busy_end, t1)
    span = (kernels[-1][1] - kernels[0][0]) / 1e3 if kernels else 0.0
    kern_ms = sum(f["ms"] for f in fams.values())
    for f in fams.values():
        f["ms"] = round(f["ms"], 3)
        f["share"] = round(f["ms"] / kern_ms, 4) if kern_ms else 0.0
    attn = sum(f["ms"] for k, f in fams.items() if k.startswith("flash_kernel"))
    return {"span_ms": round(span, 3), "kernel_ms": round(kern_ms, 3), "gaps_ms": round(gaps, 3),
            "attention_ms": round(attn, 3), "attention_share": round(attn / kern_ms, 4) if kern_ms else 0.0,
            "families": dict(sorted(fams.items(), key=lambda kv: -kv[1]["ms"]))}


def profile(fn, reps):
    """Profiles `reps` calls of fn (after one warm-up call) and keeps the call with the shortest kernel span."""
    from torch.profiler import ProfilerActivity
    fn()
    torch.cuda.synchronize()
    best = None
    for _ in range(reps):
        with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        s = summarise(kernel_table(prof))
        if best is None or s["span_ms"] < best["span_ms"]:
            best = s
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for step_profile.json")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    from idm_vton_b200 import lib as L
    from idm_vton_b200.denoise import TryOnDenoiser
    from idm_vton_b200.engine import SDXL_GARMENT, SDXL_TRYON
    from idm_vton_b200.scheduler import DDPMScheduler
    assert torch.cuda.is_available(), "step_profile needs a GPU"
    L.load()
    dev = torch.device("cuda", 0)
    B, H, W, T = 2, 1024, 768, 30
    h, w = H // 8, W // 8
    out = {"card": card(), "config": "768x1024, batch 2, guidance 2.0, 30 steps"}
    print(out["card"], flush=True)
    unet, unet_enc, _ = bench.build_components(dev, 0, 1, lambda m: None)
    den = TryOnDenoiser(unet.engine(), unet_enc.engine())
    req = bench.synth_request(SDXL_TRYON, SDXL_GARMENT, B, h, w, seed=42, device=dev)
    sch = DDPMScheduler()
    sch.set_timesteps(T)
    den.prepare(**req, guidance_scale=bench.GUIDANCE)
    den.set_step_tables(sch, sch.timesteps)
    den.capture()
    noise = torch.randn(den.latents.shape, generator=torch.Generator(device=dev).manual_seed(1), device=dev,
                        dtype=torch.float16)
    out["denoise_step"] = profile(lambda: den.step(5, noise, use_graph=True), args.reps)
    if den.hoist_garment:
        out["garment_pass"] = profile(lambda: den.precompute_garment(0), args.reps)
    out["card_after"] = card()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "step_profile.json"), "w") as f:
        json.dump(out, f, indent=1)
    for part in ("denoise_step", "garment_pass"):
        if part in out:
            s = out[part]
            top = {k: v["ms"] for k, v in list(s["families"].items())[:6]}
            print(json.dumps({part: {k: s[k] for k in ("span_ms", "kernel_ms", "gaps_ms", "attention_ms",
                                                        "attention_share")}, "top": top}), flush=True)
    print(out["card_after"], flush=True)


if __name__ == "__main__":
    main()
