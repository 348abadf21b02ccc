"""TFLOP/s of the GEMM / convolution launches that carry the config-2 denoise step and the hoisted garment passes, one row
per launch: alone with L2 flushed (`timeit`) and back to back inside a replayed CUDA graph (`timeit_graph`). Prints the
card's name, power limit and max SM clock first (a rate means nothing without them), then one JSON line per launch.
Needs a GPU: there is no fallback."""
import json
import os
import subprocess
import sys

import torch

if not torch.cuda.is_available():
    sys.exit("gemm_tile_timing.py measures on the GPU and found none")

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from idm_vton_b200 import lib as L  # noqa: E402
from idm_vton_b200.engine import pack_conv3x3, pack_geglu  # noqa: E402
from scripts.microbench import rnd, timeit, timeit_graph  # noqa: E402

# (tag, M, N, K, kind): kind "geglu" = FF1 with the GEGLU epilogue (packed for 256-wide tiles), "res" = bias + residual
LINEARS = [
    ("L2 ff1 geglu", 3072, 10240, 1280, "geglu"),
    ("L2 qkv", 3072, 3840, 1280, "plain"),
    ("L2 out-proj + residual", 3072, 1280, 1280, "res"),
    ("L2 ff2", 3072, 1280, 5120, "res"),
    ("L1 ff1 geglu", 12288, 5120, 640, "geglu"),
    ("L1 qkv", 12288, 1920, 640, "plain"),
    ("garment pass L2 out-proj", 46080, 1280, 1280, "res"),
    ("garment pass L1 out-proj", 184320, 640, 640, "res"),
]
# (tag, B, H, W, Cin, Cout, shortcut source channels or 0)
CONVS = [
    ("L0 resnet conv 320->320", 4, 128, 96, 320, 320, 0),
    ("L1 resnet conv 640->640", 4, 64, 48, 640, 640, 0),
    ("L2 resnet conv 1280->1280", 4, 32, 24, 1280, 1280, 0),
    ("L1 up conv 640->640 + 1920->640 shortcut", 4, 64, 48, 640, 640, 1920),
]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip()
    name, power, clock = [f.strip() for f in q.split(",")]
    return dict(card=name, power_limit=power, max_sm_clock=clock, sms=torch.cuda.get_device_properties(0).multi_processor_count)


def row(tag, fn, flops, shape):
    ms, ms_graph = timeit(fn), timeit_graph(fn)
    print(json.dumps(dict(launch=tag, shape=shape, ms_l2_flushed=round(ms, 4), tflops_l2_flushed=round(flops / ms / 1e9, 1),
                          ms_in_graph=round(ms_graph, 4), tflops_in_graph=round(flops / ms_graph / 1e9, 1))), flush=True)


def main():
    L.load()
    print(json.dumps(card()), flush=True)
    for tag, M, N, K, kind in LINEARS:
        a, w, b = rnd(M, K), rnd(N, K, scale=K ** -0.5), rnd(N)
        out = torch.empty(M, N // 2 if kind == "geglu" else N, dtype=torch.float16, device="cuda")
        if kind == "geglu":
            wp, bp = pack_geglu(w, b, 256)
            fn = lambda: L.gemm(a, wp, bias=bp, geglu=True, out=out, force_bn=256)  # noqa: E731
        elif kind == "res":
            res = rnd(M, N)
            fn = lambda: L.gemm(a, w, bias=b, residual=res, out=out)  # noqa: E731
        else:
            fn = lambda: L.gemm(a, w, bias=b, out=out)  # noqa: E731
        row(tag, fn, 2.0 * M * N * K, [M, N, K])
    for tag, B, H, W, Cin, Cout, Csc in CONVS:
        x, b = rnd(B, H, W, Cin), rnd(Cout)
        w = pack_conv3x3(rnd(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5))
        out = torch.empty(B, H, W, Cout, dtype=torch.float16, device="cuda")
        kw = dict(temb=rnd(B, Cout))
        if Csc:   # conv2 of an up-path resnet: the 1x1 shortcut over the concatenated [hidden | skip] input rides along
            kw = dict(sc0=rnd(B, H, W, Csc - Cout), sc1=rnd(B, H, W, Cout), w_sc=rnd(Cout, Csc, scale=Csc ** -0.5), bias_sc=rnd(Cout))
        fn = lambda: L.conv3x3(x, w, bias=b, out=out, **kw)  # noqa: E731
        row(tag, fn, 2.0 * B * H * W * Cout * (9 * Cin + Csc), [B, H, W, Cin, Cout] + ([Csc] if Csc else []))


if __name__ == "__main__":
    main()
