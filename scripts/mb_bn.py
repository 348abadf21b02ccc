"""Tile-width (BN) sweep of the GEMM / conv kernel (forced widths vs the automatic choice of gemm.cu pick_bn) on the UNet's
shapes, with cuBLAS beside it. Tuning aid; prints JSON lines."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scripts.microbench import timeit, timeit_graph, rnd  # noqa: E402
from idm_vton_b200 import lib as L  # noqa: E402
from idm_vton_b200.engine import pack_conv3x3  # noqa: E402

L.load()
SHAPES = [(12288, 640, 640, "L1 out-proj"), (12288, 640, 2560, "L1 ff2"), (12288, 1920, 640, "L1 qkv"),
          (3072, 1280, 1280, "L2 out-proj"), (3072, 3840, 1280, "L2 qkv"), (49152, 640, 640, "garment-chunk L1 out (16 samples)"),
          (12288, 1280, 1280, "garment-chunk L2 out")]
for (M, N, K, tag) in SHAPES:
    a, w, b, r = rnd(M, K), rnd(N, K, scale=K ** -0.5), rnd(N), rnd(M, N)
    o = torch.empty(M, N, dtype=torch.float16, device="cuda")
    res = {}
    for bn in (0, 128, 160, 192, 256):
        try:
            fn = lambda: L.gemm(a, w, bias=b, residual=r, out=o, force_bn=(1000 + bn) if bn else 0)  # noqa: E731
            t, tg = timeit(fn), timeit_graph(fn)
            res["auto" if bn == 0 else bn] = dict(us_flush=round(1e3 * t, 1), us_graph=round(1e3 * tg, 1),
                                                  tflops_graph=round(2.0 * M * N * K / tg / 1e9))
        except Exception as ex:
            res[bn] = str(ex)[:80]
    wt = w.t().contiguous()
    tc = timeit_graph(lambda: torch.addmm(r, a, wt, out=o))
    res["cublas_addmm"] = dict(us_graph=round(1e3 * tc, 1), tflops_graph=round(2.0 * M * N * K / tc / 1e9))
    print(json.dumps({"op": "gemm bias+res", "tag": tag, "shape": [M, N, K], "bn": res}), flush=True)
# convs (B=4 try-on batch): Cout=640 at 64x48, Cout=320 at 128x96
for (B, H, W, Cin, Cout, tag) in [(4, 64, 48, 640, 640, "L1 conv 640->640"), (4, 64, 48, 1280, 640, "L1 conv 1280->640"),
                                  (4, 128, 96, 320, 320, "L0 conv 320->320"), (4, 32, 24, 1280, 1280, "L2 conv 1280->1280")]:
    x = rnd(B, H, W, Cin)
    wp = pack_conv3x3(rnd(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5))
    bias = rnd(Cout)
    o = torch.empty(B, H, W, Cout, dtype=torch.float16, device="cuda")
    res = {}
    fl = 2.0 * B * H * W * Cout * Cin * 9
    for bn in (0, 128, 160, 192, 256):
        try:
            fn = lambda: L.conv3x3(x, wp, bias=bias, out=o, force_bn=(1000 + bn) if bn else 0)  # noqa: E731
            tg = timeit_graph(fn, n=10)
            res["auto" if bn == 0 else bn] = dict(us_graph=round(1e3 * tg, 1), tflops_graph=round(fl / tg / 1e9))
        except Exception as ex:
            res[bn] = str(ex)[:80]
    print(json.dumps({"op": "conv3x3 bias", "tag": tag, "shape": [B, H, W, Cin, Cout], "bn": res}), flush=True)
