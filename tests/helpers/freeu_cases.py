"""FreeU kernel cases shared by tests/test_freeu_cpu.py and tests/test_freeu_gpu.py: the shapes, seeded inputs with
low-frequency content, the float64 truth and the mutants the kernel must be told apart from.

Skip features of a UNet are spatially smooth; white noise has almost nothing at the frequencies FreeU scales, so every
mutant below would sit within rounding of the truth on it. The inputs are white noise plus, per channel, a constant
and waves at the frequencies (+-1, +-1) with random amplitudes and phases.
"""
import math

import torch

TOL = 2.0 ** -10          # max|kernel - truth| / max|truth| on the filtered skip
MUTANT_FACTOR = 4.0

# (name, B, H, W, Ch, Cs): config-2 stages (768x1024, try-on batch 4), 1024x1024 (powers of two), the odd deepest
# levels of a 33x25 latent (resolution suite) and size-1 / tiny planes, channel widths from 8 to 1280
SHAPES = [
    ("cfg2_L2_r0", 4, 32, 24, 1280, 1280),
    ("cfg2_L2_r2", 4, 32, 24, 1280, 640),
    ("cfg2_L1_r0", 4, 64, 48, 1280, 640),
    ("cfg2_L1_r2", 4, 64, 48, 640, 320),
    ("1024_L2", 2, 32, 32, 1280, 1280),
    ("1024_L1", 2, 64, 64, 640, 320),
    ("odd_L2", 2, 9, 7, 1280, 640),
    ("odd_L1", 2, 17, 13, 640, 320),
    ("plane_1x1", 3, 1, 1, 16, 8),
    ("plane_1x5", 2, 1, 5, 8, 24),
    ("plane_3x1", 2, 3, 1, 24, 40),
    ("plane_2x3", 1, 2, 3, 8, 8),
    ("plane_7x2", 2, 7, 2, 32, 72),
]
B_VALUE, S_VALUE = 1.3, 0.2


def make_inputs(B, H, W, Ch, Cs, seed):
    """hidden [B,H,W,Ch] and skip [B,H,W,Cs], fp16 NHWC on the CPU."""
    g = torch.Generator().manual_seed(seed)
    hidden = torch.randn(B, H, W, Ch, generator=g) * 2
    h = torch.arange(H, dtype=torch.float64)[:, None] * (2 * math.pi / H)
    w = torch.arange(W, dtype=torch.float64)[None, :] * (2 * math.pi / W)
    skip = torch.randn(B, Cs, H, W, generator=g, dtype=torch.float64) * 0.5
    skip += torch.randn(B, Cs, 1, 1, generator=g, dtype=torch.float64)
    for sh, sw in ((1, 1), (1, -1), (1, 0), (0, 1)):
        amp = torch.rand(B, Cs, 1, 1, generator=g, dtype=torch.float64) * 2
        ph = torch.rand(B, Cs, 1, 1, generator=g, dtype=torch.float64) * (2 * math.pi)
        skip += amp * torch.cos(sh * h + sw * w + ph)
    return hidden.half(), skip.permute(0, 2, 3, 1).contiguous().half()


def filter_freqs(skip_nhwc, scale, kh, kw):
    """float64: the plane plus (scale - 1) times its components at the frequencies kh x kw (taken modulo H and W, each
    distinct frequency once). skip_nhwc: [B,H,W,C]; returns [B,H,W,C] float64."""
    x = skip_nhwc.double().permute(0, 3, 1, 2)
    H, W = x.shape[-2:]
    X = torch.fft.fft2(x)
    keep = torch.zeros(H, W, dtype=torch.float64)
    for a in {k % H for k in kh}:
        for b in {k % W for k in kw}:
            keep[a, b] = 1.0
    low = torch.fft.ifft2(X * keep).real
    return (x + (scale - 1) * low).permute(0, 2, 3, 1)


def truth(skip, scale):
    """fourier_filter(skip, 1, scale) in float64 (frequencies {0, -1} along each axis)."""
    return filter_freqs(skip, scale, (0, -1), (0, -1))


SKIP_MUTANTS = {
    "mask off-centre along W": lambda x, s: filter_freqs(x, s, (0, -1), (0, 1)),
    "3x3 low-pass": lambda x, s: filter_freqs(x, s, (-1, 0, 1), (-1, 0, 1)),
    "DC only": lambda x, s: filter_freqs(x, s, (0,), (0,)),
}


def hidden_truth(hidden, b):
    """fp16(float(h) * b) on channels [0, Ch/2), the rest unchanged (PyTorch's half tensor times a Python float)."""
    out = hidden.clone()
    c = hidden.shape[-1] // 2
    out[..., :c] = hidden[..., :c] * b
    return out


def hidden_mutant(hidden, b):
    """Every channel scaled."""
    return hidden * b


def rel(a, ref):
    """max|a - ref| / max|ref|, in float64."""
    ref = ref.double()
    return ((a.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


def distinct(name, H, W):
    """Whether mutant `name` differs from the truth at plane size H x W: +1 and -1 coincide modulo 2 and 1, and for a
    real plane the components at (kh, kw) and (-kh, -kw) are conjugate, so {0, -1} x {0, +1} is the filter itself
    unless both sizes exceed 2."""
    if name == "mask off-centre along W":
        return H > 2 and W > 2
    if name == "3x3 low-pass":
        return H > 2 or W > 2
    return H > 1 or W > 1
