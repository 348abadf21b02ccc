"""Per-kernel timing of the hot ops at BASELINE config-2 shapes (device events, L2 flushed between launches).
Prints one line per (op, shape, variant) with achieved TFLOP/s or GB/s. Not a bench value; a tuning aid.
MB_ONLY=gemm stops after the GEMM / convolution rows, MB_ONLY=attention runs the attention rows only."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from idm_vton_b200 import lib as L  # noqa: E402
from idm_vton_b200.engine import pack_conv3x3, pack_geglu  # noqa: E402

V2 = os.environ.get("MB_V2", "1") == "1"
ONLY = os.environ.get("MB_ONLY", "")
dev = "cuda"
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)


def timeit(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2]


def timeit_graph(fn, n=20, reps=5):
    """Per-launch GPU time of fn inside a replayed CUDA graph of n back-to-back launches (no host time, L2-warm data —
    how the kernel runs inside the captured denoise step)."""
    fn()
    torch.cuda.synchronize()
    st = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(st):
        fn()
        with torch.cuda.graph(g, stream=st):
            for _ in range(n):
                fn()
    g.replay()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        s_, e_ = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s_.record()
        g.replay()
        e_.record()
        torch.cuda.synchronize()
        ts.append(s_.elapsed_time(e_) / n)
    ts.sort()
    return ts[len(ts) // 2]


def rnd(*s, scale=1.0):
    return (torch.randn(*s, device=dev) * scale).half()


out = []


def rec(name, ms, flops=None, bytes_=None, **kw):
    d = dict(op=name, ms=round(ms, 4), **kw)
    if flops:
        d["tflops"] = round(flops / ms / 1e9, 1)
    if bytes_:
        d["gbs"] = round(bytes_ / ms / 1e6, 1)
    out.append(d)
    print(json.dumps(d), flush=True)


def main():
    L.load()
    # ---- linears (M = 2B*N tokens with B=2: L1 M=12288 C=640, L2 M=3072 C=1280)
    skip = ONLY == "attention"
    for (M, N, K, tag) in [] if skip else [(12288, 1920, 640, "L1 qkv"), (12288, 640, 640, "L1 out"), (12288, 5120, 640, "L1 ff1"),
                           (12288, 640, 2560, "L1 ff2"), (3072, 3840, 1280, "L2 qkv"), (3072, 1280, 1280, "L2 out"),
                           (3072, 10240, 1280, "L2 ff1"), (3072, 1280, 5120, "L2 ff2"), (1536, 2560, 1280, "L2 garment kv"),
                           (8192, 8192, 8192, "square 8k")]:
        a, w = rnd(M, K), rnd(N, K, scale=K ** -0.5)
        for bn in (128, 256):
            if N % bn:
                continue
            ms = timeit(lambda: L.gemm(a, w, force_bn=bn))
            rec("gemm", ms, flops=2.0 * M * N * K, shape=[M, N, K], tag=tag, bn=bn)
        if V2:
            for bn in (128, 160, 192, 256):
                if N % bn:
                    continue
                ms = timeit(lambda: L.gemm(a, w, force_bn=1000 + bn))
                rec("gemm2", ms, flops=2.0 * M * N * K, shape=[M, N, K], tag=tag, bn=bn)
        if "ff1" in tag:
            wp, bp = pack_geglu(w, rnd(N), 256)
            ms = timeit(lambda: L.gemm(a, wp, bias=bp, geglu=True, force_bn=256))
            rec("gemm_geglu", ms, flops=2.0 * M * N * K, shape=[M, N, K], tag=tag, bn=256)
            if V2:
                ms = timeit(lambda: L.gemm(a, wp, bias=bp, geglu=True, force_bn=1256))
                rec("gemm2_geglu", ms, flops=2.0 * M * N * K, shape=[M, N, K], tag=tag, bn=256)
        ref = timeit(lambda: torch.matmul(a, w.t()))
        rec("cublas", ref, flops=2.0 * M * N * K, shape=[M, N, K], tag=tag)
    # ---- convs (NHWC, B=4)
    for (B, H, W, Cin, Cout, tag) in [] if skip else [(4, 128, 96, 320, 320, "L0 res"), (4, 64, 48, 640, 640, "L1 res"),
                                      (4, 32, 24, 1280, 1280, "L2 res"), (4, 32, 24, 2560, 1280, "L2 up res"),
                                      (4, 128, 96, 960, 320, "L0 up res"), (4, 128, 96, 64, 320, "conv_in")]:
        x = rnd(B, H, W, Cin)
        w = pack_conv3x3(rnd(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5))
        b = rnd(Cout)
        for bn in ((160,) if Cout == 320 else (128, 256)):
            ms = timeit(lambda: L.conv3x3(x, w, bias=b, force_bn=bn))
            rec("conv3x3", ms, flops=2.0 * B * H * W * 9 * Cin * Cout, shape=[B, H, W, Cin, Cout], tag=tag, bn=bn)
            if V2:
                ms = timeit(lambda: L.conv3x3(x, w, bias=b, force_bn=1000 + bn))
                rec("conv3x3_2cta", ms, flops=2.0 * B * H * W * 9 * Cin * Cout, shape=[B, H, W, Cin, Cout], tag=tag, bn=bn)
        xc = x.permute(0, 3, 1, 2).contiguous(memory_format=torch.channels_last)
        wc = rnd(Cout, Cin, 3, 3).contiguous(memory_format=torch.channels_last)
        ref = timeit(lambda: torch.nn.functional.conv2d(xc, wc, b, padding=1))
        rec("cudnn", ref, flops=2.0 * B * H * W * 9 * Cin * Cout, shape=[B, H, W, Cin, Cout], tag=tag)
    if ONLY == "gemm":
        return
    # ---- attention
    for (B, H, N, Ng, tag) in [(4, 10, 3072, 3072, "L1 self+garment"), (4, 20, 768, 768, "L2 self+garment"),
                               (2, 10, 3072, 0, "L1 garment-unet self"), (4, 10, 3072, -77, "L1 cross text"),
                               (4, 20, 768, -16, "L2 cross ip")]:
        C = H * 64
        q = rnd(B, N, C)
        if Ng >= 0:
            k, v = rnd(B, N, C), rnd(B, N, C)
            gk = rnd(B // 2, Ng, C) if Ng else None
            gv = rnd(B // 2, Ng, C) if Ng else None
            ms = timeit(lambda: L.attention(q, k, v, gk, gv, kv1_off=B // 2, heads=H))
            fl = 4.0 * B * H * N * N * 64 + (4.0 * (B // 2) * H * N * Ng * 64 if Ng else 0)
            ref = timeit(lambda: torch.nn.functional.scaled_dot_product_attention(
                q.view(B, N, H, 64).transpose(1, 2), k.view(B, N, H, 64).transpose(1, 2), v.view(B, N, H, 64).transpose(1, 2)))
            rec("sdpa_self_only", ref, flops=4.0 * B * H * N * N * 64, tag=tag)
        else:
            T = -Ng
            k, v = rnd(B, T, C), rnd(B, T, C)
            ms = timeit(lambda: L.attention(q, k, v, heads=H))
            fl = 4.0 * B * H * N * T * 64
        rec("attention", ms, flops=fl, shape=[B, H, N, Ng], tag=tag)
    # text (77 tokens) + IP (16 tokens) cross-attention of the try-on blocks, one call
    for (B, H, N, tag) in [(4, 10, 3072, "L1 cross text+ip"), (4, 20, 768, "L2 cross text+ip")]:
        C = H * 64
        q, kt, vt, ki, vi = rnd(B, N, C), rnd(B, 77, C), rnd(B, 77, C), rnd(B, 16, C), rnd(B, 16, C)
        ms = timeit(lambda: L.cross_attention(q, kt, vt, ki, vi, heads=H))
        rec("cross_attention", ms, flops=4.0 * B * H * N * (77 + 16) * 64, shape=[B, H, N, 77, 16], tag=tag)
    if ONLY == "attention":
        return
    # ---- HBM-bound side kernels
    for (B, HW, C, tag) in [(4, 12288, 320, "L0"), (4, 3072, 640, "L1"), (4, 768, 2560, "L2 cat")]:
        x = rnd(B, HW, C)
        g, b = rnd(C), rnd(C)
        ms = timeit(lambda: L.groupnorm(x, g, b, 1e-5, True))
        rec("groupnorm", ms, bytes_=3.0 * x.numel() * 2, shape=[B, HW, C], tag=tag)
    for (rows, C) in [(12288, 640), (3072, 1280)]:
        x = rnd(rows, C)
        g, b = rnd(C), rnd(C)
        ms = timeit(lambda: L.layernorm(x, g, b))
        rec("layernorm", ms, bytes_=2.0 * x.numel() * 2, shape=[rows, C])
    json.dump(out, sys.stdout, indent=1)


if __name__ == "__main__":
    main()
