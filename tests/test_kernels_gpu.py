"""Per-kernel parity of the C-ABI ops (libb200vton.so) against plain PyTorch restatements of the same op with the
reference's fp16 rounding points. Tolerances: outputs are fp16; a result may differ from the restatement by fp32
accumulation order only, so we gate at 2 fp16 ulp of the output scale (rtol 2e-3 / atol scaled)."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    from idm_vton_b200 import lib as L
    L.load()
    return L


def rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).half()


def close(a, b, tol=2e-3):
    a, b = a.float(), b.float()
    denom = max(1.0, b.abs().max().item())
    err = (a - b).abs().max().item() / denom
    assert math.isfinite(err) and err <= tol, f"max scaled err {err:.3e} > {tol}"
    return err


def r16(x):
    return x.half().float()


@pytest.mark.parametrize("M,N,K,bn", [(128, 128, 64, 0), (256, 256, 128, 0), (3072, 1280, 1280, 0), (300, 320, 192, 0),
                                      (1000, 640, 640, 128), (512, 1920, 640, 128), (128, 64, 64, 64),
                                      (640, 2560, 1280, 256), (77 * 4, 1280, 2048, 0)])
def test_gemm_plain(lib, M, N, K, bn):
    a, w = rnd(M, K, seed=1), rnd(N, K, scale=K ** -0.5, seed=2)
    out = lib.gemm(a, w, force_bn=bn)
    ref = a.float() @ w.float().t()
    close(out, ref)


def test_gemm_bias_residual_rowvec(lib):
    M, N, K = 2 * 768, 1280, 1280
    a, w = rnd(M, K, seed=1), rnd(N, K, scale=K ** -0.5, seed=2)
    bias, res, rv = rnd(N, seed=3), rnd(M, N, seed=4), rnd(2, N, seed=5)
    out = lib.gemm(a, w, bias=bias, residual=res, rowvec=rv, rows_per_sample=768)
    acc = a.float() @ w.float().t()
    v = r16(acc + bias.float())
    v = r16(v + rv.float().repeat_interleave(768, 0))
    v = r16(v + res.float())
    close(out, v)


def test_gemm_strided_views(lib):
    M, K = 512, 640
    buf = rnd(M, 3 * K, seed=1)
    a = buf[:, K:2 * K]
    w = rnd(640, K, scale=K ** -0.5, seed=2)
    big = torch.zeros(M, 2 * 640, dtype=torch.float16, device="cuda")
    out = lib.gemm(a, w, out=big[:, 640:])
    close(out, a.float() @ w.float().t())
    assert big[:, :640].abs().max().item() == 0


@pytest.mark.parametrize("bn", [128, 256])
def test_gemm_geglu(lib, bn):
    from idm_vton_b200.engine import pack_geglu
    M, C = 640, 640
    a = rnd(M, C, seed=1)
    w = rnd(8 * C, C, scale=C ** -0.5, seed=2)
    b = rnd(8 * C, seed=3)
    wp, bp = pack_geglu(w, b, bn)
    out = lib.gemm(a, wp, bias=bp, geglu=True, force_bn=bn)
    proj = r16(a.float() @ w.float().t() + b.float())
    h, g = proj.chunk(2, dim=-1)
    ref = r16(h * r16(F.gelu(g)))
    close(out, ref)


def _conv_ref(x, w, bias):
    # x NHWC fp16, w [Cout,Cin,3,3] fp16 -> fp32 NHWC
    y = F.conv2d(x.permute(0, 3, 1, 2).float(), w.float(), None, padding=1)
    if bias is not None:
        y = y + bias.float()[None, :, None, None]
    return y.permute(0, 2, 3, 1)


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 32, 24, 64, 320), (1, 16, 16, 128, 64), (4, 8, 8, 320, 640),
                                            (2, 64, 48, 320, 320), (1, 128, 96, 64, 320), (3, 5, 6, 64, 128),
                                            (2, 32, 24, 1280, 1280)])
def test_conv3x3_plain(lib, B, H, W, Cin, Cout):
    from idm_vton_b200.engine import pack_conv3x3
    x = rnd(B, H, W, Cin, seed=1)
    w = rnd(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=2)
    bias = rnd(Cout, seed=3)
    out = lib.conv3x3(x, pack_conv3x3(w), bias=bias)
    close(out, _conv_ref(x, w, bias))


def test_conv3x3_temb_residual(lib):
    from idm_vton_b200.engine import pack_conv3x3
    B, H, W, C = 2, 32, 24, 640
    x = rnd(B, H, W, C, seed=1)
    w = rnd(C, C, 3, 3, scale=(9 * C) ** -0.5, seed=2)
    bias, temb, res = rnd(C, seed=3), rnd(B, C, seed=4), rnd(B, H, W, C, seed=5)
    o1 = lib.conv3x3(x, pack_conv3x3(w), bias=bias, temb=temb)
    ref1 = r16(r16(_conv_ref(x, w, bias)) + temb.float()[:, None, None, :])
    close(o1, ref1)
    o2 = lib.conv3x3(x, pack_conv3x3(w), bias=bias, residual=res)
    ref2 = r16(r16(_conv_ref(x, w, bias)) + res.float())
    close(o2, ref2)


def test_conv3x3_shortcut_two_sources(lib):
    from idm_vton_b200.engine import pack_conv3x3
    B, H, W = 2, 16, 24
    C0, C1, Cout = 640, 320, 640
    h = rnd(B, H, W, Cout, seed=1)          # normalised conv2 input
    s0, s1 = rnd(B, H, W, C0, seed=2), rnd(B, H, W, C1, seed=3)
    w = rnd(Cout, Cout, 3, 3, scale=(9 * Cout) ** -0.5, seed=4)
    wsc = rnd(Cout, C0 + C1, scale=(C0 + C1) ** -0.5, seed=5)
    b2, bsc = rnd(Cout, seed=6), rnd(Cout, seed=7)
    out = lib.conv3x3(h, pack_conv3x3(w), bias=b2, sc0=s0, sc1=s1, w_sc=wsc, bias_sc=bsc)
    main = r16(_conv_ref(h, w, b2))
    cat = torch.cat([s0, s1], -1).float()
    sc = r16(cat @ wsc.float().t() + bsc.float())
    close(out, r16(sc + main))


def _attn_ref(q, k, v, heads, scale, n_zero=0):
    B, Nq, C = q.shape
    qh = q.float().view(B, Nq, heads, 64).transpose(1, 2)
    kh = k.float().view(B, -1, heads, 64).transpose(1, 2)
    vh = v.float().view(B, -1, heads, 64).transpose(1, 2)
    if n_zero:
        kh = torch.cat([kh, torch.zeros(B, heads, n_zero, 64, device=q.device)], 2)
        vh = torch.cat([vh, torch.zeros(B, heads, n_zero, 64, device=q.device)], 2)
    p = torch.softmax(qh @ kh.transpose(-1, -2) * scale, -1)
    return (p @ vh).transpose(1, 2).reshape(B, Nq, C)


@pytest.mark.parametrize("B,H,Nq,N0", [(1, 1, 128, 128), (2, 5, 256, 384), (2, 10, 768, 768), (1, 2, 64, 64),
                                       (2, 3, 200, 77), (1, 20, 16, 273)])
def test_attention_single_segment(lib, B, H, Nq, N0):
    C = H * 64
    q, k, v = rnd(B, Nq, C, seed=1), rnd(B, N0, C, seed=2), rnd(B, N0, C, seed=3)
    out = lib.attention(q, k, v, heads=H)
    close(out, _attn_ref(q, k, v, H, 0.125), tol=3e-3)


def test_attention_peaky(lib):
    B, H, N = 1, 4, 384
    C = H * 64
    q, k, v = rnd(B, N, C, scale=4.0, seed=1), rnd(B, N, C, scale=2.0, seed=2), rnd(B, N, C, seed=3)
    out = lib.attention(q, k, v, heads=H)
    close(out, _attn_ref(q, k, v, H, 0.125), tol=4e-3)


def test_attention_two_segments_and_zero_kv(lib):
    # try-on attn1: samples [uncond(2) ; cond(2)], garment K/V for 2 garments; uncond half sees zero K/V
    Bp, H, N, Ng = 2, 5, 256, 384
    C = H * 64
    qkv = rnd(2 * Bp, N, 3 * C, seed=1)
    q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
    gkv = rnd(Bp, Ng, 2 * C, seed=2)
    gk, gv = gkv[..., :C], gkv[..., C:]
    out = lib.attention(q, k, v, gk, gv, kv1_off=Bp, heads=H)
    ref_u = _attn_ref(q[:Bp], k[:Bp], v[:Bp], H, 0.125, n_zero=Ng)
    ref_c = _attn_ref(q[Bp:], torch.cat([k[Bp:], gk], 1), torch.cat([v[Bp:], gv], 1), H, 0.125)
    close(out[:Bp], ref_u, tol=3e-3)
    close(out[Bp:], ref_c, tol=3e-3)
    # dropping the zero tokens instead of the closed form would be visibly wrong:
    wrong = _attn_ref(q[:Bp], k[:Bp], v[:Bp], H, 0.125)
    assert (wrong - ref_u).abs().max() > 10 * (out[:Bp].float() - ref_u).abs().max()


def test_attention_shared_garment_modulo(lib):
    Bp, H, N, Ng = 3, 2, 128, 128
    C = H * 64
    q, k, v = rnd(2 * Bp, N, C, seed=1), rnd(2 * Bp, N, C, seed=2), rnd(2 * Bp, N, C, seed=3)
    gk, gv = rnd(1, Ng, C, seed=4), rnd(1, Ng, C, seed=5)
    out = lib.attention(q, k, v, gk, gv, kv1_off=Bp, heads=H)
    ref_c = _attn_ref(q[Bp:], torch.cat([k[Bp:], gk.expand(Bp, -1, -1)], 1),
                      torch.cat([v[Bp:], gv.expand(Bp, -1, -1)], 1), H, 0.125)
    close(out[Bp:], ref_c, tol=3e-3)


def test_attention_accumulate_decoupled(lib):
    # attn2: text softmax + IP softmax, fp16 outputs summed in fp16
    B, H, N = 2, 10, 256
    C = H * 64
    q = rnd(B, N, C, seed=1)
    kt, vt = rnd(B, 77, C, seed=2), rnd(B, 77, C, seed=3)
    ki, vi = rnd(B, 16, C, seed=4), rnd(B, 16, C, seed=5)
    out = lib.attention(q, kt, vt, heads=H)
    out = lib.attention(q, ki, vi, heads=H, accumulate=True, out=out)
    ref = r16(r16(_attn_ref(q, kt, vt, H, 0.125)) + r16(_attn_ref(q, ki, vi, H, 0.125)))
    close(out, ref, tol=3e-3)


@pytest.mark.parametrize("B,HW,C0,C1,silu,eps", [(2, 768, 1280, 0, 1, 1e-5), (2, 3072, 320, 0, 0, 1e-6),
                                                 (3, 500, 640, 320, 1, 1e-5), (2, 768, 1280, 640, 1, 1e-5),
                                                 (1, 64, 2560, 0, 1, 1e-5), (4, 12288, 320, 0, 1, 1e-5)])
def test_groupnorm(lib, B, HW, C0, C1, silu, eps):
    x0 = rnd(B, HW, C0, seed=1) + 0.5
    x1 = rnd(B, HW, C1, seed=2) * 2 if C1 else None
    C = C0 + C1
    gamma, beta = rnd(C, seed=3), rnd(C, seed=4)
    out = lib.groupnorm(x0, gamma, beta, eps, silu, x1=x1)
    x = torch.cat([x0, x1], -1) if C1 else x0
    ref = F.group_norm(x.float().transpose(1, 2), 32, gamma.float(), beta.float(), eps).transpose(1, 2)
    if silu:
        ref = F.silu(ref)
    close(out, ref)


@pytest.mark.parametrize("B,HW,C0,C1", [(16, 12288, 320, 0),     # hoisted garment chunk: rows do not fit smem (streaming mode)
                                        (4, 12288, 640, 320),    # up-block skip concat at full resolution (streaming mode)
                                        (4, 3072, 640, 0),       # resident mode, 37 chunks per sample
                                        (200, 64, 256, 0),       # more samples than SMs: one CTA per sample, no barrier
                                        (37, 300, 128, 64)])
def test_groupnorm_single_launch_modes(lib, B, HW, C0, C1):
    """The one-launch GroupNorm in both modes (rows parked in shared memory / re-read), across the per-sample barrier:
    repeated launches on the same workspace (sense reversal) and CUDA-graph replay must be bit-identical."""
    x0 = rnd(B, HW, C0, seed=1) + 0.5
    x1 = rnd(B, HW, C1, seed=2) * 2 if C1 else None
    C = C0 + C1
    gamma, beta = rnd(C, seed=3), rnd(C, seed=4)
    n0 = lib.launch_count()
    out = lib.groupnorm(x0, gamma, beta, 1e-5, True, x1=x1)
    assert lib.launch_count() - n0 == 1
    x = torch.cat([x0, x1], -1) if C1 else x0
    ref = F.silu(F.group_norm(x.float().transpose(1, 2), 32, gamma.float(), beta.float(), 1e-5).transpose(1, 2))
    close(out, ref)
    for _ in range(3):
        assert torch.equal(lib.groupnorm(x0, gamma, beta, 1e-5, True, x1=x1), out)
    st = torch.cuda.Stream()
    o2 = torch.empty_like(out)
    with torch.cuda.stream(st):
        lib.groupnorm(x0, gamma, beta, 1e-5, True, x1=x1, out=o2)      # workspace of this stream allocated outside capture
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            lib.groupnorm(x0, gamma, beta, 1e-5, True, x1=x1, out=o2)
    o2.zero_()
    g.replay()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(o2, out)


@pytest.mark.parametrize("rows,C", [(768, 1280), (1000, 640), (33, 2048), (16, 1280)])
def test_layernorm(lib, rows, C):
    x = rnd(rows, C, seed=1) * 3 + 1
    g, b = rnd(C, seed=2), rnd(C, seed=3)
    out = lib.layernorm(x, g, b, 1e-5)
    close(out, F.layer_norm(x.float(), (C,), g.float(), b.float(), 1e-5))


def test_layout_and_samplers(lib):
    B, C, H, W = 2, 4, 16, 12
    lat = rnd(B, C, H, W, seed=1)
    dst = torch.zeros(2 * B, H, W, 64, dtype=torch.float16, device="cuda")
    lib.nchw_to_nhwc(lat, dst, c_off=0)
    extra = rnd(2 * B, 9, H, W, seed=2)
    lib.nchw_to_nhwc(extra, dst, c_off=4)
    ref = torch.cat([torch.cat([lat, lat]), extra], 1).permute(0, 2, 3, 1)
    assert torch.equal(dst[..., :13], ref) and dst[..., 13:].abs().max() == 0
    back = lib.nhwc_to_nchw(dst, 13)
    assert torch.equal(back, ref.permute(0, 3, 1, 2))
    x = rnd(2, 8, 6, 64, seed=3)
    up = lib.upsample2x(x)
    assert torch.equal(up, F.interpolate(x.permute(0, 3, 1, 2).float(), scale_factor=2, mode="nearest")
                       .permute(0, 2, 3, 1).half())


def test_downsample_conv_via_im2col(lib):
    B, H, W, C, Cout = 2, 16, 12, 128, 128
    x = rnd(B, H, W, C, seed=1)
    w = rnd(Cout, C, 3, 3, scale=(9 * C) ** -0.5, seed=2)
    bias = rnd(Cout, seed=3)
    cols = lib.im2col3x3_s2(x)
    wk = w.permute(0, 2, 3, 1).reshape(Cout, 9 * C).contiguous()
    out = lib.gemm(cols, wk, bias=bias).view(B, H // 2, W // 2, Cout)
    ref = F.conv2d(x.permute(0, 3, 1, 2).float(), w.float(), bias.float(), stride=2, padding=1).permute(0, 2, 3, 1)
    close(out, ref)


def test_timestep_embedding_and_skinny_linear(lib):
    t = torch.tensor([967.0], device="cuda")
    emb = lib.timestep_embedding(t, 320, rows_repeat=4)
    half = 160
    freqs = torch.exp(-math.log(10000) * torch.arange(half, device="cuda", dtype=torch.float32) / half)
    arg = t[:, None] * freqs[None]
    ref = torch.cat([torch.cos(arg), torch.sin(arg)], -1).expand(4, -1)
    close(emb, ref, tol=1e-3)
    x = rnd(4, 320, seed=1)
    w1, b1 = rnd(1280, 320, scale=320 ** -0.5, seed=2), rnd(1280, seed=3)
    add = rnd(4, 1280, seed=4)
    y = lib.skinny_linear(x, w1, b1, out_silu=True, addend=add)
    ref = r16(r16(F.silu(r16(x.float() @ w1.float().t() + b1.float()))) + add.float())
    close(y, ref)
    y2 = lib.skinny_linear(y, rnd(3000, 1280, scale=1280 ** -0.5, seed=5), None, in_silu=True)
    ref2 = r16(r16(F.silu(y.float())) @ rnd(3000, 1280, scale=1280 ** -0.5, seed=5).float().t())
    close(y2, ref2)


def test_cfg_ddpm_step(lib):
    B, C, H, W = 2, 4, 16, 12
    eps = rnd(2 * B, H, W, 16, seed=1)
    lat, noise = rnd(B, C, H, W, seed=2), rnd(B, C, H, W, seed=3)
    coef = torch.tensor([2.0, 0.83, 1.0 / 0.55, 0.31, 0.68, 0.12], device="cuda")
    out = lib.cfg_ddpm_step(eps, lat, noise, coef)
    e = eps[..., :C].permute(0, 3, 1, 2).float()
    u, t = e[:B], e[B:]
    g = r16(u + r16(2.0 * r16(t - u)))
    x = lat.float()
    x0 = r16(r16(x - r16(coef[1] * g)) * coef[2])
    prev = r16(r16(coef[3] * x0) + r16(coef[4] * x))
    ref = r16(prev + r16(coef[5] * noise.float()))
    close(out, ref, tol=1e-3)


# ------------------------------------------------------------------------------------------------
# force_bn = 1000 + tile width: the C ABI's encoding of a forced width (64/128/160/192/256 of the one GEMM kernel)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,N,K,bn", [(256, 256, 64, 256), (512, 512, 128, 256), (3072, 1280, 1280, 256),
                                      (12288, 1920, 640, 192), (12288, 640, 640, 160), (1000, 640, 192, 128),
                                      (300, 320, 256, 160), (3072, 3840, 1280, 256), (777, 1280, 2560, 256),
                                      (128, 256, 64, 256), (20000, 256, 64, 128)])
def test_gemm2_plain(lib, M, N, K, bn):
    a, w = rnd(M, K, seed=1), rnd(N, K, scale=K ** -0.5, seed=2)
    out = lib.gemm(a, w, force_bn=1000 + bn)
    close(out, a.float() @ w.float().t())


def test_gemm2_epilogues(lib):
    from idm_vton_b200.engine import pack_geglu
    M, N, K = 2 * 768, 1280, 1280
    a, w = rnd(M, K, seed=1), rnd(N, K, scale=K ** -0.5, seed=2)
    bias, res, rv = rnd(N, seed=3), rnd(M, N, seed=4), rnd(2, N, seed=5)
    out = lib.gemm(a, w, bias=bias, residual=res, rowvec=rv, rows_per_sample=768, force_bn=1256)
    v = r16(a.float() @ w.float().t() + bias.float())
    v = r16(v + rv.float().repeat_interleave(768, 0))
    close(out, r16(v + res.float()))
    for bn in (128, 256):
        C = 640
        a2 = rnd(1500, C, seed=6)
        wg, bg = rnd(8 * C, C, scale=C ** -0.5, seed=7), rnd(8 * C, seed=8)
        wp, bp = pack_geglu(wg, bg, bn)
        o2 = lib.gemm(a2, wp, bias=bp, geglu=True, force_bn=1000 + bn)
        proj = r16(a2.float() @ wg.float().t() + bg.float())
        h, g = proj.chunk(2, dim=-1)
        close(o2, r16(h * r16(F.gelu(g))))


@pytest.mark.parametrize("B,H,W,Cin,Cout,bn", [(2, 32, 24, 64, 320, 160), (4, 8, 8, 320, 640, 128),
                                               (2, 64, 48, 320, 320, 160), (3, 5, 6, 64, 128, 128),
                                               (2, 32, 24, 1280, 1280, 256), (1, 16, 16, 128, 256, 256)])
def test_conv3x3_2cta(lib, B, H, W, Cin, Cout, bn):
    from idm_vton_b200.engine import pack_conv3x3
    x = rnd(B, H, W, Cin, seed=1)
    w = rnd(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=2)
    bias, temb = rnd(Cout, seed=3), rnd(B, Cout, seed=4)
    out = lib.conv3x3(x, pack_conv3x3(w), bias=bias, temb=temb, force_bn=1000 + bn)
    close(out, r16(r16(_conv_ref(x, w, bias)) + temb.float()[:, None, None, :]))


def test_gemm_auto_matches_1cta(lib):
    """The automatic tile-width choice gives the same fp16 results as a forced 256-wide tile."""
    a, w = rnd(4096, 1280, seed=1), rnd(1280, 1280, scale=1280 ** -0.5, seed=2)
    o_auto = lib.gemm(a, w)
    o_v1 = lib.gemm(a, w, force_bn=256)
    assert (o_auto.float() - o_v1.float()).abs().max() <= 2e-3 * o_v1.float().abs().max()


# ------------------------------------------------------------------------------------------------
# attention at UNet sizes (Nq >= 256): two segments, ragged tails, the zero-K/V closed form
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,Nq,N0,Ng", [(1, 1, 256, 128, 0), (2, 5, 3072, 3072, 3072), (2, 3, 300, 500, 77),
                                          (2, 20, 768, 768, 768), (1, 2, 1024, 77, 0), (1, 2, 257, 16, 0)])
def test_attention_pingpong(lib, B, H, Nq, N0, Ng):
    C = H * 64
    q, k, v = rnd(B, Nq, C, seed=1), rnd(B, N0, C, seed=2), rnd(B, N0, C, seed=3)
    if Ng:
        gk, gv = rnd(B, Ng, C, seed=4), rnd(B, Ng, C, seed=5)
        out = lib.attention(q, k, v, gk, gv, kv1_off=0, heads=H)
        ref = _attn_ref(q, torch.cat([k, gk], 1), torch.cat([v, gv], 1), H, 0.125)
    else:
        out = lib.attention(q, k, v, heads=H)
        ref = _attn_ref(q, k, v, H, 0.125)
    close(out, ref, tol=3e-3)


def test_attention_pingpong_lazy_rescale(lib):
    """Row maxima that grow by far more than 2^8 between K/V tiles exercise the online-softmax rescale of O. The
    option attention_pingpong selects a kernel of another GPU generation; here it is accepted and changes nothing."""
    B, H, N = 1, 2, 512
    C = H * 64
    q = rnd(B, N, C, scale=3.0, seed=1)
    k = rnd(B, N, C, scale=1.0, seed=2)
    k[:, 256:] *= 6.0            # later tiles have much larger scores
    v = rnd(B, N, C, seed=3)
    out = lib.attention(q, k, v, heads=H)
    close(out, _attn_ref(q, k, v, H, 0.125), tol=4e-3)
    lib.set_option("attention_pingpong", 0)
    try:
        out1 = lib.attention(q, k, v, heads=H)
    finally:
        lib.set_option("attention_pingpong", 1)
    assert torch.equal(out, out1)


def test_attention_per_step_kv_base(lib):
    """Hoisted garment K/V: segment 1 lives in a [T*Bg, Ng, C] tensor and a device scalar selects the timestep slice."""
    Bp, H, N, Ng, T = 2, 4, 256, 256, 3
    C = H * 64
    q, k, v = rnd(2 * Bp, N, C, seed=1), rnd(2 * Bp, N, C, seed=2), rnd(2 * Bp, N, C, seed=3)
    gkv = rnd(T * Bp, Ng, 2 * C, seed=4)
    for step in range(T):
        base = torch.tensor([step * Bp], dtype=torch.int32, device="cuda")
        out = lib.attention(q, k, v, gkv[..., :C], gkv[..., C:], kv1_off=Bp, heads=H, kv1_mod=Bp, kv1_base=base)
        sl = gkv[step * Bp:(step + 1) * Bp]
        ref_c = _attn_ref(q[Bp:], torch.cat([k[Bp:], sl[..., :C]], 1), torch.cat([v[Bp:], sl[..., C:]], 1), H, 0.125)
        ref_u = _attn_ref(q[:Bp], k[:Bp], v[:Bp], H, 0.125, n_zero=Ng)
        close(out[Bp:], ref_c, tol=3e-3)
        close(out[:Bp], ref_u, tol=3e-3)


def test_attention_p_in_tmem_variant(lib):
    """The attention kernel vs the fp32 reference: two segments with ragged tails, the zero-KV half, the accumulate mode
    and a peaky distribution. The options attention_pingpong / attention_q_tiles select kernels of another GPU
    generation; they are accepted and must not change the result."""
    Bp, H, N, Ng = 2, 5, 640, 1000
    C = H * 64
    qkv = rnd(2 * Bp, N, 3 * C, seed=21)
    q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
    gkv = rnd(Bp, Ng, 2 * C, seed=22)
    o5 = lib.attention(q, k, v, gkv[..., :C], gkv[..., C:], kv1_off=Bp, heads=H)
    try:
        lib.set_option("attention_pingpong", 0)
        o3 = lib.attention(q, k, v, gkv[..., :C], gkv[..., C:], kv1_off=Bp, heads=H)
    finally:
        lib.set_option("attention_pingpong", 1)
    ref_c = _attn_ref(q[Bp:], torch.cat([k[Bp:], gkv[..., :C]], 1), torch.cat([v[Bp:], gkv[..., C:]], 1), H, 0.125)
    ref_u = _attn_ref(q[:Bp], k[:Bp], v[:Bp], H, 0.125, n_zero=Ng)
    close(o5[Bp:], ref_c, tol=3e-3)
    close(o5[:Bp], ref_u, tol=3e-3)
    assert torch.equal(o5, o3)
    for qt in (1, 2):
        lib.set_option("attention_q_tiles", qt)
        try:
            oq = lib.attention(q, k, v, gkv[..., :C], gkv[..., C:], kv1_off=Bp, heads=H)
            q9, k9, v9 = rnd(1, 2048, 128, scale=4.0, seed=33), rnd(1, 2048, 128, seed=34), rnd(1, 2048, 128, seed=35)
            o9 = lib.attention(q9, k9, v9, heads=2)
        finally:
            lib.set_option("attention_q_tiles", 0)
        assert torch.equal(oq, o5)
        close(o9, _attn_ref(q9, k9, v9, 2, 0.125), tol=4e-3)
    # peaky scores exercise the rescale of O; a long single segment exercises the K/V stage ring wrap
    q2, k2, v2 = rnd(1, 2048, 128, scale=4.0, seed=23), rnd(1, 2048, 128, seed=24), rnd(1, 2048, 128, seed=25)
    close(lib.attention(q2, k2, v2, heads=2), _attn_ref(q2, k2, v2, 2, 0.125), tol=4e-3)
    # accumulate mode (decoupled cross-attention adds the second attention onto the first)
    base = lib.attention(q2, k2, v2, heads=2)
    k3, v3 = rnd(1, 300, 128, seed=26), rnd(1, 300, 128, seed=27)
    acc = base.clone()
    lib.attention(q2, k3, v3, heads=2, out=acc, accumulate=True)
    close(acc, base.float() + _attn_ref(q2, k3, v3, 2, 0.125), tol=4e-3)


@pytest.mark.parametrize("B,H,N,Nt,Ni", [(2, 10, 256, 77, 16), (4, 20, 768, 77, 16), (2, 10, 3072, 77, 0),
                                         (1, 5, 200, 77, 16), (3, 2, 40, 33, 7), (2, 4, 128, 80, 16)])
def test_cross_attention_fused(lib, B, H, N, Nt, Ni):
    """cross_attention: text + IP-token cross-attention vs the fp32 reference with the reference's fp16 rounding points
    (two softmaxes, fp16 outputs summed in fp16) and vs the two-call accumulate path."""
    C = H * 64
    q = rnd(B, N, 3 * C, seed=1)[..., C:2 * C]              # strided view, like a slice of a fused projection
    kvt = rnd(B, Nt, 2 * C, seed=2)
    kt, vt = kvt[..., :C], kvt[..., C:]
    ref = r16(_attn_ref(q, kt, vt, H, 0.125))
    ki = vi = None
    if Ni:
        kvi = rnd(B, Ni, 2 * C, seed=3)
        ki, vi = kvi[..., :C], kvi[..., C:]
        ref = r16(ref + r16(_attn_ref(q, ki, vi, H, 0.125)))
    out = lib.cross_attention(q, kt, vt, ki, vi, heads=H)
    close(out, ref, tol=3e-3)
    two = lib.attention(q, kt, vt, heads=H)
    if Ni:
        two = lib.attention(q, ki, vi, heads=H, accumulate=True, out=two)
    close(out, two, tol=2e-3)


def test_cross_attention_ip_scale_and_peaky(lib):
    B, H, N = 2, 4, 384
    C = H * 64
    q = rnd(B, N, C, scale=4.0, seed=5)
    kt, vt, ki, vi = rnd(B, 77, C, seed=6), rnd(B, 77, C, seed=7), rnd(B, 16, C, seed=8), rnd(B, 16, C, seed=9)
    out = lib.cross_attention(q, kt, vt, ki, vi, heads=H, ip_scale=0.5)
    ref = r16(r16(_attn_ref(q, kt, vt, H, 0.125)) + r16(0.5 * r16(_attn_ref(q, ki, vi, H, 0.125))))
    close(out, ref, tol=3e-3)


@pytest.mark.parametrize("B,H,W,C0,C1,Cout,force_bn", [(2, 32, 24, 640, 320, 640, 1064), (2, 32, 24, 640, 320, 640, 1128),
                                                      (4, 32, 24, 1280, 1280, 1280, 64), (1, 32, 24, 320, 0, 640, 0),
                                                      (3, 16, 24, 1280, 640, 1280, 0), (2, 64, 48, 640, 320, 320, 0)])
def test_conv3x3_shortcut_2cta_variants(lib, B, H, W, C0, C1, Cout, force_bn):
    """Resnet conv2 with the fused 1x1 shortcut (second register accumulator) at the tile widths a shortcut can use
    (64 / 128, forced or automatic): against the fp32 reference with the reference's rounding (both conv outputs rounded
    to fp16, then added) and against the 128-wide tile. A wider forced tile is refused with an error."""
    from idm_vton_b200.engine import pack_conv3x3
    h = rnd(B, H, W, Cout, seed=1)
    s0 = rnd(B, H, W, C0, seed=2)
    s1 = rnd(B, H, W, C1, seed=3) if C1 else None
    w = rnd(Cout, Cout, 3, 3, scale=(9 * Cout) ** -0.5, seed=4)
    wsc = rnd(Cout, C0 + C1, scale=(C0 + C1) ** -0.5, seed=5)
    b2, bsc = rnd(Cout, seed=6), rnd(Cout, seed=7)
    wp = pack_conv3x3(w)
    out = lib.conv3x3(h, wp, bias=b2, sc0=s0, sc1=s1, w_sc=wsc, bias_sc=bsc, force_bn=force_bn)
    cat = (torch.cat([s0, s1], -1) if C1 else s0).float()
    ref = r16(r16(cat @ wsc.float().t() + bsc.float()) + r16(_conv_ref(h, w, b2)))
    close(out, ref)
    v1 = lib.conv3x3(h, wp, bias=b2, sc0=s0, sc1=s1, w_sc=wsc, bias_sc=bsc, force_bn=128)
    close(out, v1, tol=1e-3)
    with pytest.raises(RuntimeError, match="unsupported"):
        lib.conv3x3(h, wp, bias=b2, sc0=s0, sc1=s1, w_sc=wsc, bias_sc=bsc, force_bn=1256)


def test_gemm_four_cta_cluster_variant(lib):
    """force_bn = 2000 + width, the C ABI's encoding of a multicast-cluster variant, selects the same tile as 1000 + width:
    bit-identical results (odd N-tile counts, ragged M, GEGLU) and the fp32 reference."""
    from idm_vton_b200.engine import pack_geglu
    for (M, N, K) in [(1024, 1280, 256), (3000, 768, 192), (2048, 512, 1280)]:
        a, w, b, r = rnd(M, K, seed=1), rnd(N, K, scale=K ** -0.5, seed=2), rnd(N, seed=3), rnd(M, N, seed=4)
        o4 = lib.gemm(a, w, bias=b, residual=r, force_bn=2256)
        o2 = lib.gemm(a, w, bias=b, residual=r, force_bn=1256)
        assert torch.equal(o4, o2)
        close(o4, r16(r16(a.float() @ w.float().t() + b.float()) + r.float()))
    a, w, b = rnd(1024, 640, seed=5), rnd(5120, 640, scale=640 ** -0.5, seed=6), rnd(5120, seed=7)
    wp, bp = pack_geglu(w, b, 256)
    assert torch.equal(lib.gemm(a, wp, bias=bp, geglu=True, force_bn=2256), lib.gemm(a, wp, bias=bp, geglu=True, force_bn=1256))


def test_attention_polynomial_exp_fraction(lib):
    """The option attention_poly_exp (0, 1 or 2 polynomial exponentials of every 4 in a kernel of another GPU generation)
    is accepted and has no effect: every setting is bit-identical and within tolerance of the fp32 reference on a diffuse
    and on a peaky distribution with a ragged two-segment K/V stream."""
    Bp, H, N, Ng = 1, 3, 520, 700
    C = H * 64
    for qscale in (1.0, 5.0):
        q, k, v = rnd(2 * Bp, N, C, scale=qscale, seed=41), rnd(2 * Bp, N, C, seed=42), rnd(2 * Bp, N, C, seed=43)
        gk, gv = rnd(Bp, Ng, C, seed=44), rnd(Bp, Ng, C, seed=45)
        ref_c = _attn_ref(q[Bp:], torch.cat([k[Bp:], gk], 1), torch.cat([v[Bp:], gv], 1), H, 0.125)
        ref_u = _attn_ref(q[:Bp], k[:Bp], v[:Bp], H, 0.125, n_zero=Ng)
        errs = []
        try:
            for n in (0, 1, 2):
                lib.set_option("attention_poly_exp", n)
                o = lib.attention(q, k, v, gk, gv, kv1_off=Bp, heads=H)
                errs.append((close(o[Bp:], ref_c, tol=3e-3), close(o[:Bp], ref_u, tol=3e-3)))
                if n == 0:
                    o0 = o
                assert torch.equal(o, o0)
        finally:
            lib.set_option("attention_poly_exp", 0)
        print(f"qscale {qscale}: errors (cond, uncond) for poly 0/1/2: {errs}")


@pytest.mark.parametrize("B,Cin,Cout,H,W", [(1, 128, 128, 128, 96), (2, 256, 128, 64, 48), (1, 512, 512, 32, 24),
                                            (2, 512, 256, 37, 24), (1, 128, 256, 50, 40), (3, 64, 64, 16, 8)])
def test_conv3x3_fp32_tf32(lib, B, Cin, Cout, H, W):
    """b200vton_conv3x3_nhwc_f32 (the VAE's convolutions): against cuDNN's full-fp32 convolution (TF32 off) as the
    exact result, with cuDNN's own TF32 path beside it — same arithmetic class, so both must sit within TF32 rounding.
    Ragged H, several pixel-box shapes, both tile widths."""
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(B, Cin, H, W, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) * (9 * Cin) ** -0.5
    b = torch.randn(Cout, device="cuda", generator=g)
    assert lib.conv3x3_f32_supported(x, Cin, Cout)
    out = lib.conv3x3_f32(x, lib.pack_conv3x3_f32(w), b)
    assert out.shape == (B, Cout, H, W) and out.is_contiguous(memory_format=torch.channels_last)
    with torch.backends.cudnn.flags(enabled=True, benchmark=False, deterministic=False, allow_tf32=False):
        ref = torch.nn.functional.conv2d(x, w, b, padding=1)
    e_ours = close(out, ref, tol=2e-3)
    with torch.backends.cudnn.flags(enabled=True, benchmark=False, deterministic=False, allow_tf32=True):
        e_cudnn = close(torch.nn.functional.conv2d(x, w, b, padding=1), ref, tol=2e-3)
    print(f"tf32 conv err vs fp32: ours {e_ours:.2e}, cuDNN-TF32 {e_cudnn:.2e}")
    # the resnet's residual add in the epilogue: (acc + bias) + residual in fp32 = what `residual + conv(x)` computes, bit for bit
    res = torch.randn(B, Cout, H, W, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
    fused = lib.conv3x3_f32(x, lib.pack_conv3x3_f32(w), b, residual=res)
    assert torch.equal(fused, res + out)
    res_nchw = res.contiguous()                    # any strides are accepted (converted to channels_last)
    assert torch.equal(lib.conv3x3_f32(x, lib.pack_conv3x3_f32(w), b, residual=res_nchw), fused)


@pytest.mark.parametrize("B,Cin,Cout,H,W", [(1, 128, 128, 128, 96), (2, 256, 128, 64, 48), (1, 512, 512, 32, 24),
                                            (2, 512, 256, 37, 24), (1, 128, 256, 50, 40), (3, 64, 64, 16, 8)])
def test_conv3x3_f16_operands_fp32_out(lib, B, Cin, Cout, H, W):
    """b200vton_conv3x3_nhwc_f16in_f32 (the VAE's GroupNorm -> convolution hand-off in fp16): on fp16-representable operands
    the only difference from an exact fp32 convolution is the accumulation order; against the fp32 convolution of the
    UNROUNDED operands it sits in the TF32 kernel's error class (10-bit operand mantissa). Residual epilogue bit-exact."""
    g = torch.Generator(device="cuda").manual_seed(6)
    x = torch.randn(B, Cin, H, W, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) * (9 * Cin) ** -0.5
    b = torch.randn(Cout, device="cuda", generator=g)
    x16 = x.half().contiguous(memory_format=torch.channels_last)
    w16 = lib.pack_conv3x3_f32(w).half()
    out = lib.conv3x3_f16in(x16, w16, b)
    assert out.shape == (B, Cout, H, W) and out.dtype == torch.float32 and out.is_contiguous(memory_format=torch.channels_last)
    with torch.backends.cudnn.flags(enabled=True, benchmark=False, deterministic=False, allow_tf32=False):
        ref_rounded = torch.nn.functional.conv2d(x.half().float(), w.half().float(), b, padding=1)
        ref = torch.nn.functional.conv2d(x, w, b, padding=1)
    e_acc = close(out, ref_rounded, tol=2e-4)
    e_f16 = close(out, ref, tol=2e-3)
    e_tf32 = close(lib.conv3x3_f32(x, lib.pack_conv3x3_f32(w), b), ref, tol=2e-3)
    print(f"fp16-operand conv vs fp32: {e_f16:.2e} (TF32 kernel {e_tf32:.2e}); vs fp32 conv of the rounded operands {e_acc:.2e}")
    res = torch.randn(B, Cout, H, W, device="cuda", generator=g)
    assert torch.equal(lib.conv3x3_f16in(x16, w16, b, residual=res), res + out)


@pytest.mark.parametrize("B,C,H,W,silu", [(2, 128, 64, 48, True), (1, 256, 37, 24, True), (2, 512, 16, 12, False),
                                          (1, 128, 256, 192, True)])
def test_groupnorm_fp32_nhwc(lib, B, C, H, W, silu):
    """b200vton_groupnorm_nhwc_f32 (VAE norms) vs torch.nn.functional.group_norm (+SiLU) in fp32."""
    g = torch.Generator(device="cuda").manual_seed(3)
    x = (torch.randn(B, C, H, W, device="cuda", generator=g) * 2 + 0.5).contiguous(memory_format=torch.channels_last)
    gamma, beta = torch.randn(C, device="cuda", generator=g), torch.randn(C, device="cuda", generator=g)
    out = lib.groupnorm_f32_nhwc(x, gamma, beta, 1e-6, silu)
    ref = torch.nn.functional.group_norm(x.contiguous(), 32, gamma, beta, 1e-6)
    ref = torch.nn.functional.silu(ref) if silu else ref
    assert out.is_contiguous(memory_format=torch.channels_last)
    close(out, ref, tol=1e-5)
    out16 = lib.groupnorm_f32_nhwc(x, gamma, beta, 1e-6, silu, out_half=True)       # one rounding of the same fp32 values
    assert out16.dtype == torch.float16 and out16.is_contiguous(memory_format=torch.channels_last)
    assert torch.equal(out16, out.half())


def test_vae_nhwc_route_matches_default(lib, monkeypatch):
    """Whole VAE through the NHWC route (engine fp32 GroupNorm + TF32 convolution) vs the default PyTorch route."""
    import idm_vton_b200.vae as V
    torch.manual_seed(0)
    vae = V.AutoencoderKL().cuda().float().eval()
    x = torch.rand(1, 3, 256, 192, device="cuda") * 2 - 1
    z = torch.randn(1, 4, 32, 24, device="cuda")
    # the route under test needs cuDNN's TF32 switch at its default (on), whatever earlier test files left behind
    with torch.no_grad(), torch.backends.cudnn.flags(enabled=True, benchmark=False, deterministic=False, allow_tf32=True):
        monkeypatch.setattr(V, "_ENGINE_NHWC", False)
        m0, d0 = vae.encode(x).latent_dist.mean, vae.decode(z).sample
        monkeypatch.setattr(V, "_ENGINE_NHWC", True)
        monkeypatch.setattr(V, "_F16_ACT", False)
        m1, d1 = vae.encode(x).latent_dist.mean, vae.decode(z).sample
        monkeypatch.setattr(V, "_F16_ACT", True)                 # GroupNorm -> convolution hand-off in fp16 (the default)
        m2, d2 = vae.encode(x).latent_dist.mean, vae.decode(z).sample
    e1 = (close(m1, m0, tol=5e-3), close(d1, d0, tol=5e-3))
    e2 = (close(m2, m0, tol=5e-3), close(d2, d0, tol=5e-3))
    print(f"VAE vs the cuDNN route (encode mean, decode): TF32 hand-off {e1[0]:.2e} {e1[1]:.2e}, fp16 hand-off {e2[0]:.2e} {e2[1]:.2e}")



def test_fused_pre_and_postprocessing_match_vae_image_processor(lib):
    """b200vton_preprocess_inpaint / b200vton_postprocess_image vs the VaeImageProcessor arithmetic the pipeline used before
    (src/tryon_pipeline.py:1588-1602, 940-943, 1885): bit-exact, including the `min < 0 => already normalised` rule."""
    from idm_vton_b200.vae import VaeImageProcessor
    ip = VaeImageProcessor(vae_scale_factor=8)
    mp = VaeImageProcessor(vae_scale_factor=8, do_normalize=False, do_binarize=True, do_convert_grayscale=True)
    g = torch.Generator(device="cuda").manual_seed(5)
    B, H, W = 2, 64, 48
    for lo in (0.0, -1.0):                      # [0,1] images are normalised, [-1,1] images are not
        for cm in (1, 3):
            image = torch.rand(B, 3, H, W, device="cuda", generator=g) * (1 - lo) + lo
            mask = torch.rand(B, cm, H, W, device="cuda", generator=g)
            init, mbin, masked, mlat = lib.preprocess_inpaint(image, mask, 8)
            r_init = ip.preprocess(image, height=H, width=W).float()
            r_mask = mp.preprocess(mask, height=H, width=W)
            assert torch.equal(init, r_init) and torch.equal(mbin, r_mask)
            assert torch.equal(masked, r_init * (r_mask < 0.5))
            assert torch.equal(mlat.float(), F.interpolate(r_mask, size=(H // 8, W // 8)))
    x = torch.randn(B, 3, H, W, device="cuda", generator=g) * 0.8
    for t in (x, x.contiguous(memory_format=torch.channels_last)):
        pt, u8 = lib.postprocess_image(t, want_pt=True, want_u8=True)
        ref = ip.postprocess(x, output_type="pt")
        assert torch.equal(pt, ref)
        ref_pil = ip.postprocess(x, output_type="pil")
        import numpy as np
        assert all(np.array_equal(np.asarray(p), a) for p, a in zip(ref_pil, u8.cpu().numpy()))


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(4, 128, 96, 320, 320), (4, 64, 48, 640, 640), (1, 16, 16, 64, 64), (2, 24, 40, 128, 128)])
def test_conv3x3_stride2_downsample(lib, B, H, W, Cin, Cout):
    """Downsample2D's conv (3x3, stride 2, pad 1; src/unet_block_hacked_tryon.py:1113,1246) on the implicit-GEMM kernel with
    a stride-2 TMA traversal — no im2col buffer — vs F.conv2d and vs the round-1 im2col + GEMM formulation."""
    from idm_vton_b200.engine import pack_conv3x3, pack_conv3x3_s2
    x = rnd(B, H, W, Cin, seed=1)
    w = rnd(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=2)
    b = rnd(Cout, seed=3)
    out = lib.conv3x3(x, pack_conv3x3(w), bias=b, stride=2)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float(), b.float(), stride=2, padding=1).permute(0, 2, 3, 1)
    assert out.shape == ref.shape
    close(out, ref)
    old = lib.gemm(lib.im2col3x3_s2(x), pack_conv3x3_s2(w), bias=b).view_as(out)
    close(out, old, tol=1e-3)


def test_split_tf32_and_softmax_split_kernels(lib):
    """b200vton_split_tf32 == the ATen formulation of vae._split_tf32 bit for bit (dense and row-sliced inputs, with a scale);
    b200vton_softmax_split_tf32: both parts TF32-representable, hi + lo = softmax to 2^-22, softmax itself at fp32 accuracy."""
    from idm_vton_b200.vae import _split_tf32
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(3, 1000, 512, device="cuda", generator=g) * 7
    hi, lo = lib.split_tf32(x)
    rh, rl = _split_tf32(x)
    assert torch.equal(hi, rh) and torch.equal(lo, rl)
    sl = x[:, 100:356]                                  # what the attention passes per query chunk
    hi, lo = lib.split_tf32(sl, scale=512 ** -0.5)
    rh, rl = _split_tf32(sl * 512 ** -0.5)
    assert hi.is_contiguous() and torch.equal(hi, rh) and torch.equal(lo, rl)
    assert not (hi.view(torch.int32) & 8191).any() and not (lo.view(torch.int32) & 8191).any()
    for rows, N in ((64, 12288), (7, 3072), (5, 4)):
        s = torch.randn(2, rows, N, device="cuda", generator=g) * 4
        ph, pl = lib.softmax_split_tf32(s)
        p64 = torch.softmax(s.double(), -1)
        p32 = torch.softmax(s, -1)
        assert not (ph.view(torch.int32) & 8191).any() and not (pl.view(torch.int32) & 8191).any()
        e_kernel = ((ph.double() + pl.double()) - p64).abs().max().item()
        e_torch = (p32.double() - p64).abs().max().item()
        print(f"softmax_split rows {rows} N {N}: |hi+lo - fp64| {e_kernel:.2e}, torch fp32 softmax {e_torch:.2e}")
        assert e_kernel <= 4 * e_torch + 3e-7 * p64.max().item()
        assert ((ph.double() + pl.double()).sum(-1) - 1).abs().max().item() < 1e-5


def test_vae_attention_fused_equals_aten_formulation(monkeypatch):
    """The one-pass kernels + the 3x-long contraction against the ATen formulation of the same 3xTF32 attention."""
    import idm_vton_b200.vae as V
    g = torch.Generator(device="cuda").manual_seed(10)
    B, N, C = 2, 3072, 512
    q, k, v = (torch.randn(B, N, C, device="cuda", generator=g) * s for s in (1.5, 1.5, 1.0))
    ref = F.scaled_dot_product_attention(q[:, None].double(), k[:, None].double(), v[:, None].double())[:, 0]
    monkeypatch.setattr(V, "_ATTN_FUSED", True)
    o_f = V._attention_fp32_3xtf32(q, k, v, chunk=1024)
    monkeypatch.setattr(V, "_ATTN_FUSED", False)
    o_a = V._attention_fp32_3xtf32(q, k, v, chunk=1024)
    e_f, e_a = ((x.double() - ref).abs().max().item() for x in (o_f, o_a))
    print(f"VAE attention vs fp64: fused {e_f:.2e}, ATen formulation {e_a:.2e}, fused vs ATen {(o_f - o_a).abs().max().item():.2e}")
    assert e_f <= 2 * e_a + 1e-6


def test_vae_attention_3xtf32_matches_fp32_sdpa():
    """The VAE mid-block attention on split TF32 products (vae._attention_fp32_3xtf32) vs fp64 truth at 3072 keys,
    beside PyTorch's fp32 SDPA (the reference's arithmetic) and a single TF32 pass: the split removes the operand rounding (75x), what remains is the tensor core's fp32 accumulation
    over thousands of keys (not IEEE round-to-nearest) — an order of magnitude below the error of the TF32 convolutions
    around it (6e-4 of scale, same file), which the reference's cuDNN path has too."""
    from idm_vton_b200.vae import _attention_fp32_3xtf32
    g = torch.Generator(device="cuda").manual_seed(9)
    B, N, C = 2, 3072, 512
    q, k, v = (torch.randn(B, N, C, device="cuda", generator=g) * s for s in (1.5, 1.5, 1.0))
    ref = F.scaled_dot_product_attention(q[:, None].double(), k[:, None].double(), v[:, None].double())[:, 0]
    o = _attention_fp32_3xtf32(q, k, v, chunk=1024)
    o32 = F.scaled_dot_product_attention(q[:, None], k[:, None], v[:, None])[:, 0]
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        o_tf32 = torch.softmax((q * C ** -0.5) @ k.transpose(1, 2), -1) @ v
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    e, e32, e1 = ((x.double() - ref).abs().max().item() for x in (o, o32, o_tf32))
    print(f"VAE attention vs fp64: 3xTF32 {e:.2e}, fp32 SDPA {e32:.2e}, single TF32 pass {e1:.2e}")
    assert e <= 20 * e32 and e < 0.05 * e1
