"""FP8 linears against fp16 on one GPU. Prints the card's name and power limit (read in the same run), then JSON lines:
  gemm:  per linear of a BasicTransformerBlock at L1 (C = 640, 12288 tokens) and L2 (C = 1280, 3072 tokens) of config 2's
         try-on batch of 4: b200vton_gemm_f16 against b200vton_gemm_e4m3 on the same shape, alone with L2 flushed and back
         to back inside a replayed CUDA graph, as TFLOP/s. FF2 (input: the GEGLU output, no LayerNorm to quantize it)
         adds the least time any quantize pass over its input could take at the data-sheet HBM3 bandwidth (3.35 TB/s:
         read fp16, write e4m3 + a row scale) — a floor, not a kernel;
  norm:  b200vton_layernorm against b200vton_layernorm_e4m3 (what FP8 mode launches before QKV, q2 and FF1);
  loop:  config 2 (768x1024, batch 2, 30 DDPM steps, guidance 2.0, random SDXL weights as in bench.py): set_step_tables
         (the hoisted garment passes) + every step replayed from its graph, fp16 and FP8 denoisers alternated for
         `--rounds` rounds after a warm-up loop of each; images/s = batch / loop time; and how far the FP8 loop's final
         latents are from the fp16 loop's.
Usage: python scripts/fp8_timing.py [--rounds 3]"""
import argparse
import json
import os
import sys

import torch

if not torch.cuda.is_available():
    sys.exit("fp8_timing.py measures on the GPU and found none")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import idm_vton_b200  # noqa: F401,E402
import bench  # noqa: E402
from idm_vton_b200 import lib as L  # noqa: E402
from idm_vton_b200.engine import pack_geglu  # noqa: E402
from scripts.microbench import rnd, timeit, timeit_graph  # noqa: E402
from scripts.schedule_timing import card  # noqa: E402

HBM_BYTES_PER_MS = 3.35e9     # data-sheet HBM3 bandwidth of the H100 SXM, bytes per millisecond


def _times(fn):
    return timeit(fn), timeit_graph(fn)


def gemm_rows():
    for lvl, C, M in (("L1", 640, 12288), ("L2", 1280, 3072)):
        for name, N, K in (("qkv", 3 * C, C), ("q2", C, C), ("ff1_geglu", 8 * C, C), ("ff2", C, 4 * C)):
            a, w, b = rnd(M, K), rnd(N, K, scale=K ** -0.5), rnd(N)
            geglu = name == "ff1_geglu"
            res = rnd(M, C) if name == "ff2" else None
            if geglu:
                w, b = pack_geglu(w, b, 256)
            bias = b if name in ("ff1_geglu", "ff2") else None
            out = torch.empty(M, N // 2 if geglu else N, dtype=torch.float16, device="cuda")
            qa, sa = L.quantize_rows_e4m3(a)
            qw, sw = L.quantize_rows_e4m3(w)
            bn = 256 if geglu else 0
            f16 = lambda: L.gemm(a, w, bias=bias, residual=res, geglu=geglu, out=out, force_bn=bn)  # noqa: E731
            f8 = lambda: L.gemm_e4m3(qa, sa, qw, sw, bias=bias, residual=res, geglu=geglu, out=out, force_bn=bn)  # noqa: E731
            flops = 2.0 * M * N * K
            (t16, g16), (t8, g8) = _times(f16), _times(f8)
            row = dict(gemm=f"{lvl} {name}", shape=[M, N, K], ms_f16=round(t16, 4), ms_e4m3=round(t8, 4),
                       tflops_f16=round(flops / t16 / 1e9, 1), tflops_e4m3=round(flops / t8 / 1e9, 1),
                       ms_in_graph_f16=round(g16, 4), ms_in_graph_e4m3=round(g8, 4),
                       tflops_in_graph_f16=round(flops / g16 / 1e9, 1), tflops_in_graph_e4m3=round(flops / g8 / 1e9, 1))
            if name == "ff2":
                floor = (M * K * 3 + M * 4) / HBM_BYTES_PER_MS
                row.update(quantize_floor_ms=round(floor, 4), e4m3_plus_floor_ms=round(g8 + floor, 4),
                           fp8_ff2_can_win=bool(g8 + floor < g16))
            print(json.dumps(row), flush=True)


def norm_rows():
    for lvl, C, M in (("L1", 640, 12288), ("L2", 1280, 3072)):
        x, g, b = rnd(M, C), rnd(C), rnd(C)
        t16, t8 = _times(lambda: L.layernorm(x, g, b)), _times(lambda: L.layernorm_e4m3(x, g, b))
        print(json.dumps(dict(norm=f"{lvl} layernorm", shape=[M, C], ms_f16=round(t16[0], 4), ms_e4m3=round(t8[0], 4),
                              ms_in_graph_f16=round(t16[1], 4), ms_in_graph_e4m3=round(t8[1], 4))), flush=True)


def loop_rows(rounds):
    from idm_vton_b200.denoise import TryOnDenoiser
    from idm_vton_b200.engine import SDXL_GARMENT, SDXL_TRYON
    from idm_vton_b200.scheduler import DDPMScheduler
    dev = torch.device("cuda", 0)
    B, h, w = 2, 128, 96
    unet, unet_enc, _ = bench.build_components(dev, 0, 1, lambda m: None)
    req = bench.synth_request(SDXL_TRYON, SDXL_GARMENT, B, h, w, seed=42, device=dev)
    kv = 12 << 30      # both denoisers' hoisted garment K/V stay resident (9.4 GB each at this size)
    dens = {"fp16": TryOnDenoiser(unet.engine(), unet_enc.engine(), max_kv_bytes=kv)}
    for m in (unet, unet_enc):
        m.set_linear_precision("fp8")
    dens["fp8"] = TryOnDenoiser(unet.engine(), unet_enc.engine(), max_kv_bytes=kv)
    noise = torch.randn(B, 4, h, w, generator=torch.Generator(device=dev).manual_seed(1), device=dev, dtype=torch.float16)
    final = {}

    def loop(name):
        s = DDPMScheduler()
        s.set_timesteps(30)
        d = dens[name]
        d.prepare(**req, guidance_scale=bench.GUIDANCE)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        d.set_step_tables(s, s.timesteps)
        for i in range(len(s.timesteps)):
            d.step(i, noise if d.step_draws[i] and d.noise_applied else None)
        e1.record()
        torch.cuda.synchronize()
        final[name] = d.latents.float().clone()
        return e0.elapsed_time(e1)

    for n in dens:
        loop(n)                                          # capture + warm-up
    ms = {n: [] for n in dens}
    for _ in range(rounds):
        for n in dens:
            ms[n].append(loop(n))
    med = {n: sorted(v)[len(v) // 2] for n, v in ms.items()}
    d = (final["fp8"] - final["fp16"]).abs().max().item() / max(1.0, final["fp16"].abs().max().item())
    print(json.dumps(dict(loop="config 2, 30 DDPM steps", loop_ms={n: [round(x, 1) for x in v] for n, v in ms.items()},
                          images_per_s={n: round(B / (m / 1e3), 4) for n, m in med.items()},
                          speedup=round(med["fp16"] / med["fp8"], 4), final_latents_fp8_vs_fp16=d)), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--skip-loop", action="store_true")
    args = ap.parse_args()
    L.load()
    print(json.dumps(dict(card=card())), flush=True)
    gemm_rows()
    norm_rows()
    if not args.skip_loop:
        loop_rows(args.rounds)
    print(json.dumps(dict(card_after=card())), flush=True)


if __name__ == "__main__":
    main()
