"""Full-resolution photos: GPU prepare (crop + resample to the server size) and paste-back (resample to the crop size +
paste) against Pillow on the host, per request, at 3024 x 4032 (a phone photo) and 1080 x 1920.

GPU times: CUDA events around prepare_photos (photo staged from a host uint8 tensor through pinned memory, so the
H2D copy is included) and around paste_back (from a server-size uint8 output on the device); the median over --iters
runs after --warmup. Host times: Pillow's crop, resize, resize back and paste on one thread, the median over --iters.
Prints one JSON line per size, with the card's name and power limit read in the same run.

Then one short serving run (unless --no-serve): `--requests` requests with 3024 x 4032 photos through
ContinuousTryOnServer(slots=--slots) at config-2 geometry (768 x 1024, DDPM 30 steps, random SDXL weights as bench.py
builds them), all submitted at once, output_type "pil". Two modes, alternated over --rounds rounds after one warm-up
round each, a fresh server per run (graph capture included):
  host:  Pillow crops and resizes each photo on the host, the request carries `image`; Pillow resizes each output back
         and pastes it (the demo's flow);
  photo: the request carries `photo` (a host uint8 tensor); the server prepares and pastes back on the GPU.
Prints one JSON line: wall seconds and images/s per mode, and the host mode's Pillow seconds.

    python scripts/photo_timing.py [--iters 20] [--warmup 3] [--filter bicubic] [--requests 4] [--slots 4] [--rounds 2]
                                   [--no-serve]
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import idm_vton_b200  # noqa: E402,F401
from idm_vton_b200 import photo as P  # noqa: E402
from scripts.schedule_timing import card  # noqa: E402


def _events(fn, iters, warmup):
    out = []
    for i in range(warmup + iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        if i >= warmup:
            out.append(a.elapsed_time(b))
    return statistics.median(out)


def _wall(fn, iters, warmup):
    out = []
    for i in range(warmup + iters):
        t = time.perf_counter()
        fn()
        if i >= warmup:
            out.append((time.perf_counter() - t) * 1e3)
    return statistics.median(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--filter", default="bicubic")
    ap.add_argument("--requests", type=int, default=4)
    ap.add_argument("--slots", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--no-serve", action="store_true")
    args = ap.parse_args()
    the_card = card()
    import PIL.Image
    h, w = 1024, 768
    flt = P.PIL_FILTERS[args.filter]
    g = np.random.default_rng(0)
    for W, H in ((3024, 4032), (1080, 1920)):
        a = g.integers(0, 256, (H, W, 3), dtype=np.uint8)
        host = torch.from_numpy(a)
        out = torch.from_numpy(g.integers(0, 256, (1, h, w, 3), dtype=np.uint8)).cuda()
        prep = P.prepare_photos([host], h, w, filter=args.filter)
        gpu_prepare = _events(lambda: P.prepare_photos([host], h, w, filter=args.filter), args.iters, args.warmup)
        gpu_prepare_dev = _events(lambda: P.prepare_photos([prep[0].photo], h, w, filter=args.filter), args.iters,
                                  args.warmup)
        gpu_paste = _events(lambda: P.paste_back(prep, out), args.iters, args.warmup)
        img = PIL.Image.fromarray(a)
        box = P.crop_box((W, H), h, w)
        small = PIL.Image.fromarray(out[0].cpu().numpy())
        crop = img.crop(box)
        pil_crop = _wall(lambda: img.crop(box), args.iters, args.warmup)
        pil_down = _wall(lambda: crop.resize((w, h), flt), args.iters, args.warmup)
        pil_up = _wall(lambda: small.resize(crop.size, flt), args.iters, args.warmup)
        back = small.resize(crop.size, flt)
        pil_paste = _wall(lambda: img.copy().paste(back, P.paste_offset(box)), args.iters, args.warmup)
        print(json.dumps(dict(photo=f"{W}x{H}", server=f"{w}x{h}", filter=args.filter, card=the_card,
                              gpu_prepare_from_host_ms=round(gpu_prepare, 3),
                              gpu_prepare_on_device_ms=round(gpu_prepare_dev, 3), gpu_paste_back_ms=round(gpu_paste, 3),
                              pillow_crop_ms=round(pil_crop, 2), pillow_resize_down_ms=round(pil_down, 2),
                              pillow_resize_up_ms=round(pil_up, 2), pillow_paste_with_copy_ms=round(pil_paste, 2))),
              flush=True)
    if not args.no_serve:
        serve(args, the_card)


def serve(args, the_card):
    import PIL.Image
    import bench
    from scripts.continuous_timing import make_requests
    from idm_vton_b200.serving import ContinuousTryOnServer
    H, W, PH, PW = 1024, 768, 4032, 3024
    dev = torch.device("cuda", 0)
    unet, unet_enc, _ = bench.build_components(dev, 0, 1, lambda m: None)
    pipe = bench.make_pipeline(unet, unet_enc, dev)
    flt = P.PIL_FILTERS[args.filter]
    g = np.random.default_rng(1)
    photos = [g.integers(0, 256, (PH, PW, 3), dtype=np.uint8) for _ in range(args.requests)]

    def run(mode):
        reqs = make_requests(args.requests, args.requests, dev, seed=2)
        srv = ContinuousTryOnServer(pipe, height=H, width=W, slots=args.slots, num_inference_steps=30,
                                    guidance_scale=2.0, seed=7, output_type="pil", photo_filter=args.filter)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        host = 0.0
        boxes = []
        for r, a in zip(reqs, photos):
            if mode == "photo":
                r.image, r.photo = None, torch.from_numpy(a)
            else:
                t = time.perf_counter()
                img = PIL.Image.fromarray(a)
                box = P.crop_box((PW, PH), H, W)
                crop = img.crop(box)
                small = np.asarray(crop.resize((W, H), flt), np.float32) / 255
                r.image = torch.from_numpy(small).permute(2, 0, 1).contiguous().to(dev)
                boxes.append((img, box, crop.size))
                host += time.perf_counter() - t
            srv.submit(r)
        out = srv.run()
        if mode == "host":
            t = time.perf_counter()
            for k, (img, box, size) in enumerate(boxes):
                img.paste(out[k].resize(size, flt), P.paste_offset(box))
            host += time.perf_counter() - t
        torch.cuda.synchronize()
        return time.perf_counter() - t0, host

    res = {"host": [], "photo": []}
    for rnd in range(args.rounds + 1):
        for mode in ("host", "photo"):
            wall, host = run(mode)
            if rnd:
                res[mode].append((wall, host))
    print(json.dumps(dict(serving=f"ContinuousTryOnServer(slots={args.slots}), 768x1024, DDPM 30 steps, random SDXL "
                                  f"weights, {args.requests} photos of {PW}x{PH} submitted at once, output pil",
                          card=the_card,
                          **{f"{m}_wall_s": [round(w, 3) for w, _ in v] for m, v in res.items()},
                          **{f"{m}_images_per_s": [round(args.requests / w, 4) for w, _ in v] for m, v in res.items()},
                          host_pillow_s=[round(h, 3) for _, h in res["host"]])), flush=True)


if __name__ == "__main__":
    main()
