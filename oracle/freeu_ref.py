"""ORACLE (test infrastructure, not product): FreeU (https://arxiv.org/abs/2309.11497) as diffusers==0.25.0 applies it
in the reference's up blocks (src/unet_block_hacked_tryon.py:2322-2344,2458-2480), and its closed form.

Only tests/, scripts and oracle/make_golden_freeu.py may import this module.

  * `fourier_filter` / `apply_freeu`: diffusers.utils.torch_utils of diffusers 0.25.0 (third-party, pinned by
    environment.yaml:20, not vendored: restated from its published algorithm), in the FFT form. The test-only diffusers
    shim leaves `apply_freeu` unimplemented; oracle/make_golden_freeu.py installs this one before it imports the
    reference, so the golden fixture is the reference's own up blocks running this restatement.
  * `fourier_filter_closed`: the same filter as 7 sums per (sample, channel) plane, in float64 (the kernel's algorithm).
  * `enabled(sd_t, cfg_t, freeu)`: for the duration of a `with`, the oracle's try-on UNet (oracle/unet_ref.py, and
    everything built on it: loop_ref, resolution_ref) runs FreeU before every resnet of up stages 0 and 1. Only the
    resnets evaluated with the state dict `sd_t` are affected, so the garment UNet, which runs the same trunk with its
    own state dict, is not (src/tryon_pipeline.py's enable_freeu touches `self.unet` only).
"""
import contextlib
import math

import torch

from . import unet_ref as R


def is_on(freeu):
    """The reference's rule (src/unet_block_hacked_tryon.py:2322-2327): FreeU runs only if s1, s2, b1 and b2 are all
    truthy; any of them 0 (or None) switches it off."""
    return freeu is not None and bool(freeu[0] and freeu[1] and freeu[2] and freeu[3])


def fourier_filter(x_in, threshold, scale):
    """diffusers 0.25.0 `fourier_filter`: the shifted 2-D spectrum over (H, W) times `scale` on
    [crow - threshold : crow + threshold, ccol - threshold : ccol + threshold], then back, real part, input dtype. The
    input is cast to fp32 unless both H and W are powers of two."""
    x = x_in
    B, C, H, W = x.shape
    if (W & (W - 1)) != 0 or (H & (H - 1)) != 0:
        x = x.to(dtype=torch.float32)
    elif x.dtype == torch.float16 and x.device.type == "cpu":
        # CPU torch has no half-precision FFT (cuFFT has one for power-of-two sizes): a CPU fp16 evaluation upcasts
        x = x.to(dtype=torch.float32)
    return spectral_filter(x, threshold, scale).to(dtype=x_in.dtype)


def spectral_filter(x, threshold, scale):
    """The FFT round trip of `fourier_filter` in x's own precision (the mask is float32, as diffusers builds it)."""
    x_freq = torch.fft.fftn(x, dim=(-2, -1))
    x_freq = torch.fft.fftshift(x_freq, dim=(-2, -1))
    B, C, H, W = x_freq.shape
    mask = torch.ones((B, C, H, W), device=x.device)
    crow, ccol = H // 2, W // 2
    mask[..., crow - threshold:crow + threshold, ccol - threshold:ccol + threshold] = scale
    x_freq = x_freq * mask
    x_freq = torch.fft.ifftshift(x_freq, dim=(-2, -1))
    return torch.fft.ifftn(x_freq, dim=(-2, -1)).real


def apply_freeu(resolution_idx, hidden_states, res_hidden_states, **freeu_kwargs):
    """diffusers 0.25.0 `apply_freeu`: stage 0 scales the first half of the backbone channels by b1 (in place, in the
    activation dtype) and filters the skip with s1; stage 1 the same with b2 / s2; other stages are untouched."""
    if resolution_idx == 0:
        num_half_channels = hidden_states.shape[1] // 2
        hidden_states[:, :num_half_channels] = hidden_states[:, :num_half_channels] * freeu_kwargs["b1"]
        res_hidden_states = fourier_filter(res_hidden_states, threshold=1, scale=freeu_kwargs["s1"])
    if resolution_idx == 1:
        num_half_channels = hidden_states.shape[1] // 2
        hidden_states[:, :num_half_channels] = hidden_states[:, :num_half_channels] * freeu_kwargs["b2"]
        res_hidden_states = fourier_filter(res_hidden_states, threshold=1, scale=freeu_kwargs["s2"])
    return hidden_states, res_hidden_states


def fourier_filter_closed(x, scale):
    """fourier_filter(x, 1, scale) in float64 by the closed form: with theta = 2 pi h / H and phi = 2 pi w / W,
    x + (scale - 1) / HW * [A + Re(P e^-i phi) + Re(Q e^-i theta) + Re(R e^-i (theta + phi))], A = sum x,
    P = sum x e^i phi, Q = sum x e^i theta, R = sum x e^i (theta + phi); P and R drop when W = 1, Q and R when H = 1.
    x: [B, C, H, W] (any float dtype); returns float64."""
    x = x.double()
    H, W = x.shape[-2:]
    th = torch.arange(H, dtype=torch.float64, device=x.device) * (2 * math.pi / H)
    ph = torch.arange(W, dtype=torch.float64, device=x.device) * (2 * math.pi / W)
    e = torch.exp(1j * (th[:, None] + 0 * ph[None, :]))          # e^i theta  [H, W]
    f = torch.exp(1j * (0 * th[:, None] + ph[None, :]))          # e^i phi
    xc = x.to(torch.complex128)
    terms = [torch.ones_like(e)]
    if W > 1:
        terms.append(f)
    if H > 1:
        terms.append(e)
    if H > 1 and W > 1:
        terms.append(e * f)
    corr = torch.zeros_like(x)
    for t in terms:
        s = (xc * t).sum(dim=(-2, -1), keepdim=True)
        corr = corr + (s * t.conj()).real
    return x + (scale - 1) * corr / (H * W)


def _hidden_widths(cfg):
    """{"up_blocks.i.resnets.j": channels of the backbone input} for up stages 0 and 1 (the rest of the resnet's input
    is the skip, src/unet_hacked_tryon.py:700-740)."""
    rev = list(reversed(cfg["block_out_channels"]))
    out = {}
    for i in (0, 1):
        for j in range(cfg["layers_per_block"] + 1):
            out[f"up_blocks.{i}.resnets.{j}"] = rev[max(i - 1, 0)] if j == 0 else rev[i]
    return out


@contextlib.contextmanager
def enabled(sd_t, cfg_t, freeu, stage_of=None):
    """Runs the oracle's try-on UNet (state dict `sd_t`) with FreeU (s1, s2, b1, b2) inside the `with`. Nothing changes
    when FreeU is off by the reference's rule. stage_of: optional {up block index: resolution_idx} (default identity),
    which lets a test build a wiring mutant."""
    if not is_on(freeu):
        yield
        return
    s1, s2, b1, b2 = freeu
    widths = _hidden_widths(cfg_t)
    orig = R.resnet_block

    def resnet_block(sd, p, x, temb, eps=1e-5):
        if sd is sd_t and p in widths:
            i = int(p.split(".")[1])
            c = widths[p]
            hidden, skip = x[:, :c].clone(), x[:, c:]
            hidden, skip = apply_freeu(i if stage_of is None else stage_of[i], hidden, skip, s1=s1, s2=s2, b1=b1, b2=b2)
            x = torch.cat([hidden, skip], dim=1)
        return orig(sd, p, x, temb, eps)

    R.resnet_block = resnet_block
    try:
        yield
    finally:
        R.resnet_block = orig
