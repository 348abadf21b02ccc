"""AutoencoderKL (SDXL VAE) and VaeImageProcessor stand-ins — HOST-SIDE PLUMBING around the hot path.

The reference pipeline receives a diffusers `AutoencoderKL` as a component (src/tryon_pipeline.py:387-401) and calls
`vae.encode(x).latent_dist.sample(generator)`, `vae.decode(z, return_dict=False)[0]`, `vae.config.{scaling_factor,
force_upcast,latent_channels,block_out_channels}` (:911-932,1646,1868-1880). diffusers is not installable in this image, so
this module supplies an architecture-compatible VAE (same parameter names as diffusers 0.25.0's AutoencoderKL, restated
from its published structure) so that `__call__` runs end to end. The VAE is row (f)1 of SURVEY.md 8 ("next"): on a GPU
the fp32 VAE runs NHWC with its 3x3 / stride-1 convolutions on the wgmma kernels `b200vton_conv3x3_nhwc_f32` (TF32
operands) / `b200vton_conv3x3_nhwc_f16in_f32` (fp16 operands handed over by the norm: `_gn_silu_conv`) and every GroupNorm(+SiLU)
on `b200vton_groupnorm_nhwc_f32` (default ON, see `_ENGINE_NHWC`), the resnets' residual add rides in the convolution's epilogue, the mid-block attention is a split-TF32 formulation (cuBLAS GEMMs between this library's one-pass split /
softmax kernels); resampling and the stride-2 / 3-8-channel / 1x1 convolutions are PyTorch.
"""
import os
import types

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F


# Feeding the NHWC convolution from torch's NCHW GroupNorm adds two layout copies per convolution over tensors of up to
# 805 MB, while the convolutions are a minor part of the VAE's time; this NCHW switch therefore stays off
# (B200VTON_VAE_TF32_CONV=1 to enable) and the NHWC route below is the engine's path.
_ENGINE_CONV = os.environ.get("B200VTON_VAE_TF32_CONV", "0") == "1"
# The whole fp32 VAE in NHWC (channels_last): the engine convolution then needs no layout copies and GroupNorm(+SiLU) runs on
# `b200vton_groupnorm_nhwc_f32` (checked by tests -k "fp32_nhwc or vae_nhwc"). Default ON
# (B200VTON_VAE_NHWC=0 restores the cuDNN NCHW route); fp32 data, TF32 products — the arithmetic class the reference's
# fp32 VAE gets from cuDNN under torch's default `cudnn.allow_tf32`.
_ENGINE_NHWC = os.environ.get("B200VTON_VAE_NHWC", "1") == "1"


def _use_nhwc(x):
    return _ENGINE_NHWC and x.is_cuda and x.dtype == torch.float32 and x.dim() == 4


def _gn(norm, x, silu):
    """GroupNorm (+ SiLU). NHWC mode: fp32 channels_last tensors go to the engine's fp32 GroupNorm kernel."""
    if _use_nhwc(x) and norm.num_groups == 32 and x.shape[1] % 32 == 0 and x.shape[1] <= 2048:
        from . import lib as L
        x = x.contiguous(memory_format=torch.channels_last)
        return L.groupnorm_f32_nhwc(x, norm.weight, norm.bias, norm.eps, silu)
    y = norm(x)
    return F.silu(y) if silu else y


def _conv_device_ok(x):
    return x.is_cuda


# Round 2, last step: the resnets' residual add rides in the convolution's epilogue (bit-identical: fp32 (acc + bias) + x) and
# the mid-block attention's split operands / probabilities come from one-pass kernels (`b200vton_split_tf32`,
# `b200vton_softmax_split_tf32`) with the three score products folded into ONE GEMM over a 3x-long contraction; the ATen
# formulation measured at a fifth of the VAE's time (profiles/r2_vae_kernel_shares.json). B200VTON_VAE_FUSED=0 /
# B200VTON_VAE_ATTN_FUSED=0 restore the ATen formulations.
_ENGINE_FUSED = os.environ.get("B200VTON_VAE_FUSED", "1") == "1"                 # residual add in the convolution's epilogue
_ATTN_FUSED = os.environ.get("B200VTON_VAE_ATTN_FUSED", "1") == "1"           # one-pass split / softmax-split kernels


def _tf32_engine(conv, x, width=None):
    """True when `_conv(conv, x)` runs on the engine's TF32 convolution; width: its input's width when x is taken before
    the 2x upsampling that produces that input."""
    if (_conv_device_ok(x) and x.dtype == torch.float32 and conv.kernel_size == (3, 3) and conv.stride == (1, 1)
            and conv.padding == (1, 1) and conv.dilation == (1, 1) and conv.groups == 1
            and torch.backends.cudnn.allow_tf32 and (_ENGINE_CONV or _ENGINE_NHWC)):
        from . import lib as L
        if width is None:
            return L.conv3x3_f32_supported(x, conv.in_channels, conv.out_channels)
        return L.conv3x3_f32_supported(x, conv.in_channels, conv.out_channels, width=width)
    return False


def _conv(conv, x, residual=None):
    """3x3 / stride 1 / pad 1 fp32 convolutions with 32-aligned channel counts run on the engine's TF32 tensor-core
    kernel on CUDA (`b200vton_conv3x3_nhwc_f32`: TF32 products, fp32 accumulation — the arithmetic class cuDNN uses for
    fp32 convolutions under torch's default `allow_tf32`); every other case (CPU, fp16, conv_in / conv_out with 3-8
    channels, stride-2 downsamplers, 1x1 shortcuts, TF32 disabled by the caller) stays on `nn.Conv2d`.
    The tensor core truncates its fp32 operands (it ignores their 13 low mantissa bits) where cuDNN rounds them to
    nearest; truncation shrinks every product, a slope of 1 - 7e-4 against the exact convolution (measured on an H100,
    tests/test_vae_parity_gpu.py). So on the device the packed weights are rounded to nearest once, and `_Up` rounds the
    input (the only caller whose input is not already fp16 from the norm)."""
    if _tf32_engine(conv, x):
        from . import lib as L
        key = (conv.weight.data_ptr(), conv.weight._version)
        cache = getattr(conv, "_b200_packed", None)
        if cache is None or cache[0] != key:
            w = L.pack_conv3x3_f32(conv.weight)
            cache = (key, _tf32(w) if w.is_cuda else w)     # only the tensor core truncates: nothing to compensate on a CPU
            conv._b200_packed = cache
        if residual is not None and not _ENGINE_FUSED:
            return residual + L.conv3x3_f32(x, cache[1], conv.bias)
        return L.conv3x3_f32(x, cache[1], conv.bias, residual=residual)
    return conv(x) if residual is None else residual + conv(x)


# GroupNorm(+SiLU) -> convolution with an fp16 hand-off: the TF32 convolution reduces its fp32 operands to 10 mantissa bits
# anyway, so the norm stores fp16 (same mantissa, rounded to nearest as cuDNN's TF32 convolutions round; its outputs are
# O(1-10), far inside fp16's range) and the convolution runs
# with fp16 operands — half the norm's write and the convolution's read, twice the MMA rate, fp32 accumulation / bias /
# residual / output as before (`b200vton_conv3x3_nhwc_f16in_f32`). B200VTON_VAE_F16ACT=0 keeps the fp32 hand-off.
_F16_ACT = os.environ.get("B200VTON_VAE_F16ACT", "1") == "1"


def _gn_silu_conv(norm, conv, x, residual=None):
    """conv(silu(norm(x))) (+ residual): the fp16 hand-off when both kernels take the shapes, else `_conv(conv, _gn(...))`."""
    if (_F16_ACT and _ENGINE_FUSED and _use_nhwc(x) and norm.num_groups == 32 and x.shape[1] % 64 == 0 and x.shape[1] <= 2048
            and conv.kernel_size == (3, 3) and conv.stride == (1, 1) and conv.padding == (1, 1) and conv.dilation == (1, 1)
            and conv.groups == 1 and torch.backends.cudnn.allow_tf32):
        from . import lib as L
        if L.conv3x3_f32_supported(x, conv.in_channels, conv.out_channels):
            key = (conv.weight.data_ptr(), conv.weight._version)
            cache = getattr(conv, "_b200_packed16", None)
            if cache is None or cache[0] != key:
                cache = (key, L.pack_conv3x3_f32(conv.weight).to(torch.float16))
                conv._b200_packed16 = cache
            h16 = L.groupnorm_f32_nhwc(x.contiguous(memory_format=torch.channels_last), norm.weight, norm.bias, norm.eps, True,
                                       out_half=True)
            return L.conv3x3_f16in(h16, cache[1], conv.bias, residual=residual)
    return _conv(conv, _gn(norm, x, True), residual=residual)


class _Resnet(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.norm1 = nn.GroupNorm(32, cin, eps=1e-6)
        self.conv1 = nn.Conv2d(cin, cout, 3, padding=1)
        self.norm2 = nn.GroupNorm(32, cout, eps=1e-6)
        self.conv2 = nn.Conv2d(cout, cout, 3, padding=1)
        self.conv_shortcut = nn.Conv2d(cin, cout, 1) if cin != cout else None

    def forward(self, x):
        h = _gn_silu_conv(self.norm1, self.conv1, x)
        if self.conv_shortcut is not None:
            x = self.conv_shortcut(x)
        return _gn_silu_conv(self.norm2, self.conv2, h, residual=x)        # x + conv2(silu(norm2(h)))


def _tf32(t):
    """fp32 -> the nearest TF32 value (10 mantissa bits, ties away from zero), still fp32: round half up on the 13 low
    mantissa bits, then clear them."""
    return ((t.view(torch.int32) + 4096) & -8192).view(torch.float32)


def _tf32_(t):
    """`_tf32` in place (no temporaries: the decoder's largest upsampler input is 200 MB)."""
    t.view(torch.int32).add_(4096).bitwise_and_(-8192)
    return t


def _split_tf32(x):
    """x ~ hi + lo with BOTH parts exactly representable in TF32 (10 mantissa bits): hi = tf32(x), lo = tf32(x - hi), so the
    tensor core — which ignores the 13 low mantissa bits of its fp32 operands, i.e. truncates — sees them unchanged.
    What is dropped is 2^-22 |x|."""
    hi = _tf32(x)
    return hi, _tf32(x - hi)


def _attention_fp32_3xtf32(q, k, v, chunk=2048):
    """softmax(q k^T / sqrt(C)) v for the VAE mid block — ONE head of C = 512 channels over H*W tokens (12288 at
    768x1024), exact fp32 in the reference (SDPA on fp32 tensors with torch's default matmul precision). PyTorch's fp32
    memory-efficient kernel uses no tensor cores. Here every product runs on the TF32
    tensor cores three times with split operands — a·b ≈ a_hi·b_hi + a_hi·b_lo + a_lo·b_hi, fp32 accumulation — which
    removes the TF32 operand rounding (the dropped a_lo·b_lo term is 2^-22 relative); what remains is the tensor core's own
    fp32 accumulation over thousands of keys, which grows with their number: 5e-6 to 5e-5 of the output scale against
    fp64 at 1155 to 12 288 keys, where fp32 SDPA has 1-2e-6 and a single TF32 pass 5-8e-4 (H100,
    tests/test_vae_parity_gpu.py) — an order below the error of the TF32 convolutions around it. Queries are processed in chunks so the score block stays small. The products are cuBLAS TF32 GEMMs; the split operands and
    the softmax come from `b200vton_split_tf32` / `b200vton_softmax_split_tf32` (one pass each; the three score products are ONE
    GEMM over the concatenated contraction [q_lo | q_hi | q_hi] . [k_hi | k_lo | k_hi]^T, small terms first); `_ATTN_FUSED = False` is the ATen formulation
    of the same arithmetic (kept as the cross-check of tests/test_kernels_gpu.py). Host-side plumbing of a SURVEY 8f row."""
    B, N, C = q.shape
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        if _ATTN_FUSED and q.is_cuda and N % 4 == 0 and C % 4 == 0:
            from . import lib as L
            kh, kl = L.split_tf32(k)
            vh, vl = L.split_tf32(v)
            k3_t = torch.cat([kh, kl, kh], dim=2).transpose(1, 2)      # [B, 3C, N]: contraction order = small terms first
            del kh, kl
            out = torch.empty_like(q)
            for c0 in range(0, N, chunk):
                qh, ql = L.split_tf32(q[:, c0:c0 + chunk], scale=C ** -0.5)
                s = torch.bmm(torch.cat([ql, qh, qh], dim=2), k3_t)    # ql.kh + qh.kl + qh.kh in ONE pass over the scores
                ph, pl = L.softmax_split_tf32(s)
                del s
                out[:, c0:c0 + chunk] = torch.baddbmm(torch.baddbmm(torch.bmm(pl, vh), ph, vl), ph, vh)
            return out
        kh, kl = _split_tf32(k)
        vh, vl = _split_tf32(v)
        kh_t, kl_t = kh.transpose(1, 2), kl.transpose(1, 2)
        out = torch.empty_like(q)
        scale = C ** -0.5
        for c0 in range(0, N, chunk):
            qh, ql = _split_tf32(q[:, c0:c0 + chunk] * scale)
            s = torch.baddbmm(torch.baddbmm(torch.bmm(ql, kh_t), qh, kl_t), qh, kh_t)      # small terms first
            p = torch.softmax(s, dim=-1)
            ph, pl = _split_tf32(p)
            out[:, c0:c0 + chunk] = torch.baddbmm(torch.baddbmm(torch.bmm(pl, vh), ph, vl), ph, vh)
        return out
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


_ATTN_3XTF32 = os.environ.get("B200VTON_VAE_ATTN_3XTF32", "1") == "1"


class _Attn(nn.Module):
    """Single-head spatial self-attention of the VAE mid block (diffusers Attention with group_norm, bias=True)."""

    def __init__(self, c):
        super().__init__()
        self.group_norm = nn.GroupNorm(32, c, eps=1e-6)
        self.to_q, self.to_k, self.to_v = nn.Linear(c, c), nn.Linear(c, c), nn.Linear(c, c)
        self.to_out = nn.ModuleList([nn.Linear(c, c), nn.Dropout(0.0)])

    def forward(self, x):
        b, c, h, w = x.shape
        if _use_nhwc(x):                                   # tokens are a free view of the NHWC tensor
            t = _gn(self.group_norm, x, False).permute(0, 2, 3, 1).reshape(b, h * w, c)
        else:
            t = self.group_norm(x).view(b, c, h * w).transpose(1, 2)
        q, k, v = self.to_q(t), self.to_k(t), self.to_v(t)
        if _ATTN_3XTF32 and t.is_cuda and t.dtype == torch.float32 and t.shape[1] >= 1024:
            o = _attention_fp32_3xtf32(q, k, v)
        else:
            o = F.scaled_dot_product_attention(q[:, None], k[:, None], v[:, None])[:, 0]
        o = self.to_out[0](o)
        if _use_nhwc(x):
            return x + o.reshape(b, h, w, c).permute(0, 3, 1, 2)
        return x + o.transpose(1, 2).reshape(b, c, h, w)


class _Mid(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.attentions = nn.ModuleList([_Attn(c)])
        self.resnets = nn.ModuleList([_Resnet(c, c), _Resnet(c, c)])

    def forward(self, x):
        return self.resnets[1](self.attentions[0](self.resnets[0](x)))


class _Down(nn.Module):
    def __init__(self, cin, cout, layers, add_down):
        super().__init__()
        self.resnets = nn.ModuleList([_Resnet(cin if i == 0 else cout, cout) for i in range(layers)])
        self.downsamplers = None
        if add_down:
            d = nn.Module()
            d.conv = nn.Conv2d(cout, cout, 3, stride=2, padding=0)
            self.downsamplers = nn.ModuleList([d])

    def forward(self, x):
        for r in self.resnets:
            x = r(x)
        if self.downsamplers is not None:
            x = self.downsamplers[0].conv(F.pad(x, (0, 1, 0, 1)))
        return x


class _Up(nn.Module):
    def __init__(self, cin, cout, layers, add_up):
        super().__init__()
        self.resnets = nn.ModuleList([_Resnet(cin if i == 0 else cout, cout) for i in range(layers)])
        self.upsamplers = None
        if add_up:
            u = nn.Module()
            u.conv = nn.Conv2d(cout, cout, 3, padding=1)
            self.upsamplers = nn.ModuleList([u])

    def forward(self, x):
        for r in self.resnets:
            x = r(x)
        if self.upsamplers is not None:
            conv = self.upsamplers[0].conv
            # the engine's TF32 convolution truncates its input: round it to nearest first, before the upsampling, where
            # it is a quarter of the size (nearest upsampling copies values, so the rounding commutes with it)
            if x.is_cuda and _tf32_engine(conv, x, width=2 * x.shape[3]):
                x = _tf32_(x)                      # in place: x is the last resnet's fresh output, read by nothing else
            x = _conv(conv, F.interpolate(x, scale_factor=2.0, mode="nearest"))
        return x


class _Encoder(nn.Module):
    def __init__(self, cin, ch, layers, latent):
        super().__init__()
        self.conv_in = nn.Conv2d(cin, ch[0], 3, padding=1)
        self.down_blocks = nn.ModuleList(
            [_Down(ch[max(i - 1, 0)], c, layers, i < len(ch) - 1) for i, c in enumerate(ch)])
        self.mid_block = _Mid(ch[-1])
        self.conv_norm_out = nn.GroupNorm(32, ch[-1], eps=1e-6)
        self.conv_out = nn.Conv2d(ch[-1], 2 * latent, 3, padding=1)

    def forward(self, x):
        x = self.conv_in(x)
        for d in self.down_blocks:
            x = d(x)
        x = self.mid_block(x)
        return self.conv_out(_gn(self.conv_norm_out, x, True))


class _Decoder(nn.Module):
    def __init__(self, cout, ch, layers, latent):
        super().__init__()
        rch = list(reversed(ch))
        self.conv_in = nn.Conv2d(latent, rch[0], 3, padding=1)
        self.mid_block = _Mid(rch[0])
        self.up_blocks = nn.ModuleList(
            [_Up(rch[max(i - 1, 0)], c, layers + 1, i < len(ch) - 1) for i, c in enumerate(rch)])
        self.conv_norm_out = nn.GroupNorm(32, rch[-1], eps=1e-6)
        self.conv_out = nn.Conv2d(rch[-1], cout, 3, padding=1)

    def forward(self, z):
        x = self.mid_block(self.conv_in(z))
        for u in self.up_blocks:
            x = u(x)
        return self.conv_out(_gn(self.conv_norm_out, x, True))


class DiagonalGaussianDistribution:
    def __init__(self, parameters):
        self.mean, self.logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(self.logvar, -30.0, 20.0)
        self.std = torch.exp(0.5 * self.logvar)

    def sample(self, generator=None):
        # diffusers' randn_tensor: a CPU generator draws on the CPU and the sample is moved to the latents' device
        dev = self.mean.device
        rand_dev = "cpu" if (generator is not None and generator.device.type == "cpu" and dev.type != "cpu") else dev
        noise = torch.randn(self.mean.shape, generator=generator, device=rand_dev, dtype=self.mean.dtype).to(dev)
        return self.mean + self.std * noise

    def mode(self):
        return self.mean


class AutoencoderKL(nn.Module):
    """SDXL VAE geometry by default (block_out_channels 128/256/512/512, 4 latent channels, scaling 0.13025)."""

    def __init__(self, in_channels=3, out_channels=3, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                 latent_channels=4, scaling_factor=0.13025, force_upcast=True):
        super().__init__()
        ch = tuple(block_out_channels)
        self.encoder = _Encoder(in_channels, ch, layers_per_block, latent_channels)
        self.decoder = _Decoder(out_channels, ch, layers_per_block, latent_channels)
        self.quant_conv = nn.Conv2d(2 * latent_channels, 2 * latent_channels, 1)
        self.post_quant_conv = nn.Conv2d(latent_channels, latent_channels, 1)
        self.config = types.SimpleNamespace(in_channels=in_channels, out_channels=out_channels, block_out_channels=ch,
                                            layers_per_block=layers_per_block, latent_channels=latent_channels,
                                            scaling_factor=scaling_factor, force_upcast=force_upcast)

    @property
    def dtype(self):
        return next(self.parameters()).dtype

    @property
    def device(self):
        return next(self.parameters()).device

    def encode(self, x, return_dict=True):
        if _use_nhwc(x):
            x = x.contiguous(memory_format=torch.channels_last)
            dist = DiagonalGaussianDistribution(self.quant_conv(self.encoder(x)).contiguous())
            return types.SimpleNamespace(latent_dist=dist) if return_dict else (dist,)
        dist = DiagonalGaussianDistribution(self.quant_conv(self.encoder(x)))
        return types.SimpleNamespace(latent_dist=dist) if return_dict else (dist,)

    def decode(self, z, return_dict=True, generator=None):
        if _use_nhwc(z):
            img = self.decoder(self.post_quant_conv(z.contiguous(memory_format=torch.channels_last))).contiguous()
        else:
            img = self.decoder(self.post_quant_conv(z))
        return types.SimpleNamespace(sample=img) if return_dict else (img,)

    def enable_slicing(self):
        pass

    disable_slicing = enable_tiling = disable_tiling = enable_slicing


class VaeImageProcessor:
    """The subset of diffusers' VaeImageProcessor the pipeline uses (src/tryon_pipeline.py:418-421,1588-1602,1885):
    resize to (height, width), [0,1] -> [-1,1] normalisation, optional grayscale + binarisation for masks; tensors,
    numpy arrays and PIL images are accepted; postprocess to "pil" / "np" / "pt" / "latent"."""

    def __init__(self, vae_scale_factor=8, do_resize=True, do_normalize=True, do_binarize=False,
                 do_convert_grayscale=False):
        self.vae_scale_factor = vae_scale_factor
        self.do_resize, self.do_normalize = do_resize, do_normalize
        self.do_binarize, self.do_convert_grayscale = do_binarize, do_convert_grayscale

    def _to_tensor(self, image):
        import PIL.Image
        if isinstance(image, torch.Tensor):
            t = image
            if t.ndim == 3:
                t = t[None] if not self.do_convert_grayscale or t.shape[0] in (1, 3) else t[:, None]
            return t.float(), True
        if isinstance(image, PIL.Image.Image):
            image = [image]
        if isinstance(image, (list, tuple)) and isinstance(image[0], PIL.Image.Image):
            arrs = []
            for im in image:
                im = im.convert("L") if self.do_convert_grayscale else im.convert("RGB")
                a = np.asarray(im, dtype=np.float32) / 255.0
                arrs.append(a[..., None] if a.ndim == 2 else a)
            return torch.from_numpy(np.stack(arrs)).permute(0, 3, 1, 2), False
        if isinstance(image, np.ndarray):
            a = image[None] if image.ndim == 3 else image
            return torch.from_numpy(a.astype(np.float32)).permute(0, 3, 1, 2), False
        if isinstance(image, (list, tuple)) and isinstance(image[0], torch.Tensor):
            return torch.stack([i if i.ndim == 3 else i[0] for i in image]).float(), True
        raise ValueError(f"unsupported image input type {type(image)}")

    def preprocess(self, image, height=None, width=None, resize_mode="default", crops_coords=None):
        if crops_coords is not None or resize_mode != "default":
            raise NotImplementedError("padding_mask_crop is not on the IDM-VTON inference path")
        t, was_tensor = self._to_tensor(image)
        if t.shape[1] == 4 and not self.do_convert_grayscale:   # already latents
            return t
        if self.do_convert_grayscale and t.shape[1] == 3:
            t = (0.299 * t[:, 0:1] + 0.587 * t[:, 1:2] + 0.114 * t[:, 2:3])
        if self.do_resize and height is not None and (t.shape[-2] != height or t.shape[-1] != width):
            t = F.interpolate(t, size=(height, width))
        do_norm = self.do_normalize
        if was_tensor and do_norm and t.min() < 0:
            do_norm = False          # diffusers: tensors already in [-1, 1] are not normalised again
        if do_norm:
            t = 2.0 * t - 1.0
        if self.do_binarize:
            t = (t >= 0.5).to(t.dtype)
        return t

    def postprocess(self, image, output_type="pil", do_denormalize=None):
        if output_type == "latent":
            return image
        if not isinstance(image, torch.Tensor):
            return image
        img = (image.float() / 2 + 0.5).clamp(0, 1)
        if output_type == "pt":
            return img
        arr = img.cpu().permute(0, 2, 3, 1).numpy()
        if output_type == "np":
            return arr
        import PIL.Image
        arr = (arr * 255).round().astype("uint8")
        return [PIL.Image.fromarray(a.squeeze()) if a.shape[-1] == 1 else PIL.Image.fromarray(a) for a in arr]
