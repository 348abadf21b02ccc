"""The fp32 VAE path against float64: its engine kernels one by one, and whole encode / decode at every size the pipeline
accepts.

Kernels: the TF32 convolution (`conv3x3_f32`) and its fp16-operand twin (`conv3x3_f16in`), the fp32 GroupNorm
(`groupnorm_f32_nhwc`), the split kernels of the mid-block attention (`split_tf32`, `softmax_split_tf32`) and the attention
itself. Conventions of test_kernel_edges_gpu.py: the metric is max|a - b| / max|b| per sample (no floor), each tolerance is
derived beside it, and every gate has a mutant the kernel must be at least 4x closer to the truth than; the CPU tests at
the end prove that separation without a GPU wherever it can be computed there.

Operand model of the TF32 convolution (measured here on an H100): the tensor core ignores the 13 low mantissa bits of an
fp32 operand, i.e. truncates it, which shrinks every product by ~3.4e-4 per operand on average (a slope of 1 - 7e-4 on
raw operands). cuDNN's TF32 convolutions, the reference's arithmetic under torch's default `cudnn.allow_tf32`, round to
nearest. So vae.py rounds the packed weights and the upsamplers' inputs (the one input of that kernel that is not already
an fp16 hand-off) to nearest before they reach the tensor core; the operand-model and L2 gates below fail without that.

Whole VAE: the truth is the float64 copy of the module (every engine switch of vae.py takes the torch route in float64),
the yardstick is the same fp32 module on the reference's route (cuDNN with TF32, fp32 SDPA). The engine route must be as
close to the truth as the yardstick (`PARITY {...}` lines, visible with `pytest -s`)."""
import copy
import json
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_kernel_edges_gpu import grid16, rel_err, report, tol_norm32


# ------------------------------------------------------------------------------------------------------------------
# operand models and metrics
# ------------------------------------------------------------------------------------------------------------------
def tf32_rn(x):
    """fp32 -> float64 values of the nearest TF32 value (ties away from zero): the formula of vae._tf32, as int32 bits."""
    return ((x.float().view(torch.int32) + 4096) & -8192).view(torch.float32).double()


def tf32_trunc(x):
    """fp32 -> float64 values of the fp32 operand with its 13 low mantissa bits cleared (what the tensor core reads)."""
    return (x.float().view(torch.int32) & -8192).view(torch.float32).double()


def slope(y, y64):
    """Least-squares slope of y against the truth: <y, y64> / <y64, y64>. Operands truncated to TF32 give ~1 - 7e-4."""
    y, y64 = y.double().flatten(), y64.double().flatten()
    return (torch.dot(y, y64) / torch.dot(y64, y64)).item()


def per_sample(a, b, fn=rel_err):
    return max(fn(a[i], b[i]) for i in range(a.shape[0]))


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm()).item()


def tol_acc(K, k_step):
    """fp32 accumulation of K exact products on the tensor core: each wgmma step adds k_step products to the accumulator
    and truncates the sum to fp32 (<= 1 ulp = 2^-23 of the running sum, whose magnitude stays below the output's max, with
    one sign: the errors add up linearly), so K / k_step * 2^-23 of the output scale. K = 9 * 512 with TF32's k8 steps:
    6.9e-5; measured up to 1.1e-5 (its truncation bias is ~0.7 ulp per step, not random)."""
    return K / k_step * 2.0 ** -23


# |slope - 1| of a TF32 convolution whose operands are rounded to nearest: the rounding errors have zero mean, so what is
# left is their random projection on y (~3e-4 / sqrt(#outputs) < 3e-6 here) and the accumulation bias (~1e-5 at
# K = 4608): 2^-13 = 1.2e-4 sits 10x above that and 6x below the truncation bias (7e-4).
SLOPE_TOL = 2.0 ** -13


# ------------------------------------------------------------------------------------------------------------------
# 1. TF32 convolution: operand model, accumulation, epilogue order
# ------------------------------------------------------------------------------------------------------------------
CONV_CASES = [(cin, cout) for cin in (32, 128, 512) for cout in (64, 128, 256, 512)]   # Cout 256/512: BN = 256;
CONV_BHW = (2, 8, 16)                    # Cin 32: 9 slabs of 32 channels, fewer per tap than STAGES; one box per sample
F16_CASES = [(128, 64), (128, 256), (512, 128), (512, 512)]


def conv_operands(Cin, Cout, seed=0):
    """Random, non-grid fp32 operands (every mantissa bit in play): x ~ N(0, 1), w ~ N(0, 1 / (9 Cin)), y ~ N(0, 1)."""
    g = torch.Generator().manual_seed(seed + 7 * Cin + Cout)
    B, H, W = CONV_BHW
    x = torch.randn(B, Cin, H, W, generator=g, dtype=torch.float64).float()
    w = (torch.randn(Cout, Cin, 3, 3, generator=g, dtype=torch.float64) * (9 * Cin) ** -0.5).float()
    b = torch.randn(Cout, generator=g, dtype=torch.float64).float()
    res = (0.5 * torch.randn(B, Cout, H, W, generator=g, dtype=torch.float64)).float()
    return x, w, b, res


def conv64(x, w):
    return F.conv2d(x.double(), w.double(), padding=1)


def f16in_ref(acc, b, res, mutant=None):
    """The fp32 epilogue of the fp16-operand convolution on the float64 accumulator: fp32(acc), + bias, + residual, each
    rounded to fp32. mutant 'acc_fp16': the accumulator rounded to fp16 first (the fp16 convolution's store)."""
    a = acc.half().float() if mutant == "acc_fp16" else acc.float()
    return (a + b.float()[None, :, None, None]) + res.float()


@pytest.fixture(scope="module")
def lib():
    from idm_vton_b200 import lib as L
    L.load()
    return L


@pytest.mark.gpu
@pytest.mark.parametrize("Cin,Cout", CONV_CASES)
def test_conv3x3_tf32_operand_model(lib, Cin, Cout):
    """conv3x3_f32 against conv(T(x), T(w)) in float64 for T = round-to-nearest and T = truncation. On raw operands the
    kernel follows one of the two (printed; it is the tensor core's own behaviour); as vae._conv calls it (weights
    rounded when packed, an input rounded as `_Up` rounds it) it must follow rounding, and its slope must be 1 within SLOPE_TOL.
    cuDNN's TF32 convolution is measured beside it (printed, not gated)."""
    x, w, _, _ = conv_operands(Cin, Cout)
    xc, wc = x.cuda(), w.cuda()
    models = {"tf32_rn": conv64(tf32_rn(xc), tf32_rn(wc)), "tf32_trunc": conv64(tf32_trunc(xc), tf32_trunc(wc))}
    y64 = conv64(xc, wc)
    tol = tol_acc(9 * Cin, 8)
    y_raw = lib.conv3x3_f32(xc, lib.pack_conv3x3_f32(wc))                 # raw operands
    e_raw = {m: per_sample(y_raw, r) for m, r in models.items()}
    k_model = min(e_raw, key=e_raw.get)
    other = "tf32_trunc" if k_model == "tf32_rn" else "tf32_rn"
    report(f"conv3x3_f32 raw operands Cin={Cin} Cout={Cout} follows {k_model}", e_raw[k_model], tol,
           {other: e_raw[other]})
    import idm_vton_b200.vae as V
    conv = torch.nn.Conv2d(Cin, Cout, 3, padding=1, bias=False).cuda()
    with torch.no_grad():
        conv.weight.copy_(wc)
    with torch.backends.cudnn.flags(enabled=True, benchmark=False, deterministic=False, allow_tf32=True):
        assert V._tf32_engine(conv, xc)
        y = V._conv(conv, V._tf32(xc))                  # vae.py's route: weights rounded there, the input as `_Up` does
    e = {m: per_sample(y, r) for m, r in models.items()}
    report(f"conv3x3_f32 as vae.py calls it Cin={Cin} Cout={Cout}", e["tf32_rn"], tol,
           {"tf32_trunc": e["tf32_trunc"]})
    with torch.backends.cudnn.flags(enabled=True, benchmark=False, deterministic=False, allow_tf32=True):
        y_cudnn = F.conv2d(xc, wc, padding=1)
    e_c = {m: per_sample(y_cudnn, r) for m, r in models.items()}
    c_model = min(e_c, key=e_c.get)
    s_raw, s, s_c = slope(y_raw, y64), slope(y, y64), slope(y_cudnn, y64)
    print(f"[vae] TF32 operand model Cin={Cin} Cout={Cout}: kernel (raw operands) follows {k_model} "
          f"(rn {e_raw['tf32_rn']:.2e}, trunc {e_raw['tf32_trunc']:.2e}) slope-1 {s_raw - 1:+.2e}; kernel as the VAE "
          f"calls it slope-1 {s - 1:+.2e}; cuDNN TF32 nearer {c_model} (rn {e_c['tf32_rn']:.2e}, trunc "
          f"{e_c['tf32_trunc']:.2e}) slope-1 {s_c - 1:+.2e}")
    assert abs(s - 1) <= SLOPE_TOL, f"slope {s:.7f}: the operands reach the tensor core biased"


@pytest.mark.gpu
@pytest.mark.parametrize("Cin,Cout", F16_CASES)
def test_conv3x3_f16in_accumulation(lib, Cin, Cout):
    """conv3x3_f16in on random fp16 operands (exact in the kernel): the float64 convolution of the fp16 values, then bias
    and residual added in fp32. What is left is the fp32 accumulation over K = 9 Cin (k16 steps)."""
    x, w, b, res = conv_operands(Cin, Cout, seed=1)
    x16, w16 = x.half().cuda(), w.half().cuda()
    bc, rc = b.cuda(), res.cuda()
    out = lib.conv3x3_f16in(x16.contiguous(memory_format=torch.channels_last), lib.pack_conv3x3_f32(w16).half(), bc,
                           residual=rc)
    acc = conv64(x16, w16)
    ref = f16in_ref(acc, bc, rc)
    mut = f16in_ref(acc, bc, rc, mutant="acc_fp16")
    report(f"conv3x3_f16in Cin={Cin} Cout={Cout}", per_sample(out, ref), tol_acc(9 * Cin, 16),
           {"acc_fp16": per_sample(mut, ref)})


# (B, H, W, Cout): box shapes the other convolution tests miss (gemm.cu pick_box)
EPI_BOXES = [
    (5, 4, 8, 64),        # bw 8, bh 4, bb 4: a box spans 4 samples, the second box holds sample 5 alone
    (2, 37, 16, 128),     # bw 16, bh 8: the last box row is partial (37 = 4 * 8 + 5)
    (2, 5, 360, 64),      # bw 8 (360 = 8 * 45), bh 4, bb 4: half-empty sample boxes, partial rows
    (2, 5, 600, 256),     # bw 8 (600 = 8 * 75), BN = 256
    (2, 5, 720, 64),      # bw 16 (720 = 16 * 45), bh 4, bb 2
]


def epi_operands(B, H, W, Cout, Cin=64):
    """Grid operands (products and fp32 sums exact), random fp32 bias and residual."""
    x = grid16(B, Cin, H, W, scale=1.0, seed=B + H + W).double()
    w = grid16(Cout, Cin, 3, 3, scale=0.25, seed=Cout).double()
    g = torch.Generator().manual_seed(H * W)
    b = torch.randn(Cout, generator=g, dtype=torch.float64).float()
    res = torch.randn(B, Cout, H, W, generator=g, dtype=torch.float64).float()
    return x, w, b, res


def epi_ref(acc, b, res, mutant=None):
    """fp32 (acc + bias) + residual; mutants: 'res_before_bias', 'res_wrong_sample' (the previous sample's residual)."""
    a, bb = acc.float(), b[None, :, None, None]
    if mutant == "res_before_bias":
        return (a + res) + bb
    return (a + bb) + (res.roll(1, 0) if mutant == "res_wrong_sample" else res)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["tf32", "f16"])
@pytest.mark.parametrize("B,H,W,Cout", EPI_BOXES)
def test_conv3x3_fp32_epilogue_boxes(lib, kind, B, H, W, Cout):
    """Bit-exact (acc + bias) + residual at odd box geometries, for the TF32 and the fp16-operand kernel."""
    x, w, b, res = epi_operands(B, H, W, Cout)
    acc = F.conv2d(x, w, padding=1)
    ref = epi_ref(acc, b, res)
    merr = {m: rel_err(epi_ref(acc, b, res, m), ref) for m in ("res_before_bias", "res_wrong_sample")}
    xc = x.float().cuda().contiguous(memory_format=torch.channels_last)
    wc, bc, rc = w.float().cuda(), b.cuda(), res.cuda()
    if kind == "tf32":
        out = lib.conv3x3_f32(xc, lib.pack_conv3x3_f32(wc), bc, residual=rc).cpu()
    else:
        out = lib.conv3x3_f16in(xc.half(), lib.pack_conv3x3_f32(wc).half(), bc, residual=rc).cpu()
    report(f"conv {kind} epilogue B={B} H={H} W={W} Cout={Cout}", rel_err(out, ref), 0.0, merr)
    assert torch.equal(out, ref)


# ------------------------------------------------------------------------------------------------------------------
# 2. fp32 GroupNorm
# ------------------------------------------------------------------------------------------------------------------
def gn_chunks(B, HW):
    """groupnorm_f32_impl's statistics chunks: (chunks, rows per chunk)."""
    chunks = min(max(1184 // B, 1), -(-HW // 16))
    rows = -(-HW // chunks)
    return -(-HW // rows), rows


# (name, B, H, W, C, silu, mutants)
GN32_CASES = [
    ("bench_level", 1, 1024, 768, 128, True, ("drop_last_chunk", "double_last_chunk")),   # 1183 chunks, last one ragged
    ("batch3", 3, 96, 128, 128, True, ("stats_of_sample_0",)),
    ("batch8", 8, 64, 48, 256, False, ("stats_of_sample_0",)),
    ("hw1", 2, 1, 1, 128, True, ("var_n_minus_1",)),
    ("hw15", 2, 3, 5, 128, False, ("var_n_minus_1",)),
    ("hw16", 2, 4, 4, 128, True, ("var_n_minus_1",)),
    ("hw17", 2, 1, 17, 128, False, ("var_n_minus_1",)),
    ("c96", 2, 12, 25, 96, True, ("var_n_minus_1",)),          # cpg 3; 21 row lanes of 24 threads, 8 threads idle
    ("c384", 2, 12, 25, 384, False, ("stats_of_sample_0",)),  # 5 row lanes of 96 threads, 32 idle
    ("c2048", 2, 8, 16, 2048, True, ("stats_of_sample_0",)),  # one row lane
]
LAST_CHUNK_OFFSET = 8.0
# fp32 GroupNorm vs float64: the statistics' fp32 partial sums and the fp32 apply, 2^-18 of the output scale (the
# shifted sums make the group mean irrelevant; tol_norm32 of test_kernel_edges_gpu.py at an offset of one std)
TOL_GN32 = tol_norm32(1)


def gn_input(name, B, H, W, C):
    """Per-sample mean and spread differ (sample b: 0.5 b + (1 + 0.25 b) N(0, 1)); in the bench-level case the rows of the
    last statistics chunk sit LAST_CHUNK_OFFSET higher, so losing or repeating that chunk moves every group's mean."""
    g = torch.Generator().manual_seed(B * 1000 + C + H * W)
    sb = torch.arange(B, dtype=torch.float64)[:, None, None, None]
    x = 0.5 * sb + (1 + 0.25 * sb) * torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    if name == "bench_level":
        chunks, rows = gn_chunks(B, H * W)
        x.view(B, C, H * W)[:, :, (chunks - 1) * rows:] += LAST_CHUNK_OFFSET
    gamma = torch.randn(C, generator=g, dtype=torch.float64).float()
    beta = torch.randn(C, generator=g, dtype=torch.float64).float()
    return x.float(), gamma, beta


def gn64(x, gamma, beta, silu, mutant=None):
    """Float64 GroupNorm(32, eps 1e-6) (+SiLU) with the statistics written out. Mutants: 'var_n_minus_1' (unbiased
    variance), 'drop_last_chunk' / 'double_last_chunk' (the last statistics chunk's rows weighted 0 / 2),
    'stats_of_sample_0' (every sample normalised with sample 0's statistics)."""
    B, C, H, W = x.shape
    xd = x.double().reshape(B, 32, C // 32, H * W)
    wr = torch.ones(H * W, dtype=torch.float64, device=x.device)
    if mutant in ("drop_last_chunk", "double_last_chunk"):
        chunks, rows = gn_chunks(B, H * W)
        wr[(chunks - 1) * rows:] = 0.0 if mutant == "drop_last_chunk" else 2.0
    n = wr.sum() * (C // 32)
    mu = (xd * wr).sum((2, 3), keepdim=True) / n
    var = ((xd - mu) ** 2 * wr).sum((2, 3), keepdim=True) / (n - 1 if mutant == "var_n_minus_1" else n)
    if mutant == "stats_of_sample_0":
        mu, var = mu[:1].expand_as(mu), var[:1].expand_as(var)
    y = ((xd - mu) / torch.sqrt(var + 1e-6)).reshape(B, C, H, W)
    if gamma is not None:
        y = y * gamma.double()[None, :, None, None]
    if beta is not None:
        y = y + beta.double()[None, :, None, None]
    return F.silu(y) if silu else y


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,H,W,C,silu,mutants", GN32_CASES, ids=[c[0] for c in GN32_CASES])
def test_groupnorm_f32_against_float64(lib, name, B, H, W, C, silu, mutants):
    x, gamma, beta = gn_input(name, B, H, W, C)
    xc = x.cuda().contiguous(memory_format=torch.channels_last)
    gc, bc = gamma.cuda(), beta.cuda()
    out = lib.groupnorm_f32_nhwc(xc, gc, bc, 1e-6, silu)
    ref = F.group_norm(xc.double(), 32, gc.double(), bc.double(), 1e-6)
    ref = F.silu(ref) if silu else ref
    merr = {m: per_sample(gn64(xc, gc, bc, silu, mutant=m), ref) for m in mutants}
    report(f"groupnorm fp32 {name} (chunks {gn_chunks(B, H * W)})", per_sample(out, ref), TOL_GN32, merr)
    out16 = lib.groupnorm_f32_nhwc(xc, gc, bc, 1e-6, silu, out_half=True)       # the hand-off: fp16 RN of the fp32 result
    assert out16.dtype == torch.float16 and torch.equal(out16, out.half())


@pytest.mark.gpu
def test_groupnorm_f32_constant_group_and_null_affine(lib):
    """A constant group has variance 0: the output is exactly beta (silu(beta) with SiLU, within its fp32 evaluation);
    null gamma / beta are accepted and mean 1 / 0."""
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 128, 6, 8, generator=g, dtype=torch.float64).float()
    x[0, :4] = 0.37                                        # group 0 of sample 0 (4 channels per group)
    beta = torch.randn(128, generator=g, dtype=torch.float64).float().cuda()
    gamma = torch.randn(128, generator=g, dtype=torch.float64).float().cuda()
    xc = x.cuda().contiguous(memory_format=torch.channels_last)
    out = lib.groupnorm_f32_nhwc(xc, gamma, beta, 1e-6, False)
    assert torch.equal(out[0, :4], beta[:4, None, None].expand(4, 6, 8))
    out_s = lib.groupnorm_f32_nhwc(xc, gamma, beta, 1e-6, True)
    report("groupnorm fp32 constant group + SiLU", rel_err(out_s[0, :4], F.silu(beta[:4].double())[:, None, None]
                                                           .expand(4, 6, 8)), 2.0 ** -20)
    report("groupnorm fp32 constant group, other groups", per_sample(out_s, F.silu(gn64(xc, gamma, beta, False))), TOL_GN32)
    for gm, bt in ((None, None), (gamma, None), (None, beta)):
        o = lib.groupnorm_f32_nhwc(xc, gm, bt, 1e-6, False)
        report(f"groupnorm fp32 gamma={'set' if gm is not None else 'null'} beta={'set' if bt is not None else 'null'}",
               per_sample(o, gn64(xc, gm, bt, False)), TOL_GN32)


# ------------------------------------------------------------------------------------------------------------------
# 3. split kernels and the mid-block attention
# ------------------------------------------------------------------------------------------------------------------
def special_values():
    """fp32 values where a TF32 split can go wrong, as bit patterns: ties (low 13 bits exactly 0x1000) and their
    neighbours, all-ones mantissas (the rounding carries into the exponent, FLT_MAX to inf), +-0, subnormals, random
    normals; both signs. The count is a multiple of 4."""
    rng = np.random.default_rng(11)
    upper = rng.integers(0x30000000 >> 13, 0x4F000000 >> 13, 256, dtype=np.uint64) << 13
    vals = [upper | 0x1000, upper | 0x0FFF, upper | 0x1001]
    exps = np.arange(1, 255, dtype=np.uint64)
    vals.append((exps << 23) | 0x7FFFFF)                                       # 1.11..1 x 2^e; e = 254 is FLT_MAX
    vals.append(np.array([0x0, 0x1, 0xFFF, 0x1000, 0x1001, 0x1FFF, 0x7FFFFF, 0x7FF000, 0x400000, 0x3000], dtype=np.uint64))
    vals.append(rng.integers(0x00800000, 0x7F000000, 256, dtype=np.uint64))
    v = np.concatenate(vals)
    v = np.concatenate([v, v | 0x80000000])
    v = v[: len(v) // 4 * 4].astype(np.uint32)
    return torch.from_numpy(v.view(np.float32).copy())


def split_ref(x, scale=1.0):
    """Int32 restatement of split_tf32 on fp32 x: xs = fp32(x * fp32(scale)) (one IEEE multiply), hi = tf32(xs),
    lo = tf32(xs - hi), where xs - hi is exact in fp32."""
    x = x.float()
    if scale != 1.0:
        s32 = torch.tensor(scale, dtype=torch.float32).double()
        x = (x.double() * s32).float()                                         # the product of two fp32 values is exact in float64
    hi = tf32_rn(x).float()
    return hi, tf32_rn((x.double() - hi.double()).float()).float()


def bits_equal(a, b):
    return torch.equal(a.cpu().view(torch.int32), b.cpu().view(torch.int32))


@pytest.mark.gpu
def test_split_tf32_bit_exact(lib):
    v = special_values()
    n = v.numel()
    for scale in (1.0, 512 ** -0.5, 0.7):
        vv = v if scale == 1.0 else v[v.abs() < 1e38][: (v.abs() < 1e38).sum() // 4 * 4]
        for B, per in ((1, vv.numel()), (vv.numel() // 12, 12), (3, 4 * 771)):
            x = vv.repeat(-(-B * per // vv.numel()))[: B * per].reshape(B, per)   # per: 3 float4 / a ragged last block
            hi, lo = lib.split_tf32(x.cuda(), scale=scale)
            rh, rl = split_ref(x, scale)
            assert bits_equal(hi, rh) and bits_equal(lo, rl), (scale, B, per)
    print(f"[vae] split_tf32: {n} special values bit-exact (ties, carries, +-0, subnormals, FLT_MAX)")
    g = torch.Generator().manual_seed(12)
    big = torch.randn(3, 1000, 512, generator=g, dtype=torch.float64).float() * 7
    big.view(-1)[: n] = v
    bc = big.cuda()
    sl = bc[:, 100:356]                                   # the attention's per-chunk row slice: batch stride != block size
    hi, lo = lib.split_tf32(sl, scale=512 ** -0.5)
    rh, rl = split_ref(big[:, 100:356].contiguous(), 512 ** -0.5)
    assert bits_equal(hi, rh) and bits_equal(lo, rl)
    h1, l1 = lib.split_tf32(bc[1:2, 100:356], scale=512 ** -0.5)       # B = 1 takes the block size as its stride
    assert bits_equal(h1[0], hi[1]) and bits_equal(l1[0], lo[1])
    for t in (hi, lo):
        assert not (t.view(torch.int32) & 8191).any()


SOFTMAX_SHAPES = [(2048, 12288), (560, 10800), (1356, 7500)]    # the VAE's query chunks: 768x1024, 720x960 tail, 600x800 tail
# hi + lo vs the float64 softmax, per row, relative to the row's largest probability: expf (<= 2 ulp), the fp32 row sum
# (<= 26 additions on the path of any term: 12 serial float4 steps, 2 in the float4, 5 shuffles, 7 warps, each <= 2^-24),
# the reciprocal and the product (1/2 ulp each) and lo's own TF32 rounding (2^-22): <= 2^-18.7; 2^-18
TOL_SOFTMAX = 2.0 ** -18


def softmax_scores(rows, N, seed):
    """Row 0: one score of 120 over N(0, 1) scores, every other exp(s - max) < e^-115 underflows to 0 in fp32; row 1: all
    scores equal (p = 1/N, not representable); rows 2..9: scores uniform in [-100, 100]; the rest N(0, 16)."""
    g = torch.Generator().manual_seed(seed)
    s = torch.randn(rows, N, generator=g) * 4
    s[0] = torch.randn(N, generator=g)
    s[0, N // 3] = 120.0
    s[1] = 0.5
    s[2:10] = torch.rand(8, N, generator=g) * 200 - 100
    return s


def softmax_no_max(s):
    """Mutant: the softmax without the max subtraction, in fp32 (exp overflows past 88.7)."""
    e = torch.exp(s.float())
    return e / e.sum(-1, keepdim=True)


def finite_or_inf(e):
    return e if math.isfinite(e) else math.inf


@pytest.mark.gpu
@pytest.mark.parametrize("rows,N", SOFTMAX_SHAPES)
def test_softmax_split_tf32_against_float64(lib, rows, N):
    s = softmax_scores(rows, N, seed=N).cuda()
    ph, pl = lib.softmax_split_tf32(s)
    assert not (ph.view(torch.int32) & 8191).any() and not (pl.view(torch.int32) & 8191).any()
    p64 = torch.softmax(s.double(), -1)
    err = ((ph.double() + pl.double() - p64).abs().amax(-1) / p64.amax(-1)).max().item()
    merr = finite_or_inf(per_sample(softmax_no_max(s[:10]), p64[:10]))
    report(f"softmax_split_tf32 rows={rows} N={N}", err, TOL_SOFTMAX, {"no_max_subtraction": merr})
    assert (ph[0] + pl[0]).max().item() == 1.0 and (ph[0] + pl[0]).sum().item() == 1.0    # the dominant row


ATTN_NS = [1155, 1156, 7500, 10800, 12288]     # 1155 = 33 x 35 (N % 4 != 0: the ATen split path), the rest the kernels


@pytest.mark.gpu
@pytest.mark.parametrize("N", ATTN_NS)
@pytest.mark.parametrize("B", [1, 3])
def test_vae_attention_3xtf32_against_float64(N, B):
    """The mid-block attention (one head, C = 512) per sample against float64: within 20x fp32 SDPA's error (the
    reference's arithmetic) or the accumulation bound over N keys, whichever is larger, and under 0.1x the error of a
    single TF32 pass (what the split removes)."""
    from idm_vton_b200.vae import _attention_fp32_3xtf32
    g = torch.Generator(device="cuda").manual_seed(N + B)
    C = 512
    q, k, v = (torch.randn(B, N, C, device="cuda", generator=g) * s for s in (1.5, 1.5, 1.0))
    o = _attention_fp32_3xtf32(q, k, v)
    ref = F.scaled_dot_product_attention(q[:, None].double(), k[:, None].double(), v[:, None].double())[:, 0]
    o32 = F.scaled_dot_product_attention(q[:, None], k[:, None], v[:, None])[:, 0]
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = True
    try:
        o1 = torch.cat([torch.softmax((q[:, c:c + 2048] * C ** -0.5) @ k.transpose(1, 2), -1) @ v
                        for c in range(0, N, 2048)], 1)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    for b in range(B):
        e, e32, e1 = rel_err(o[b], ref[b]), rel_err(o32[b], ref[b]), rel_err(o1[b], ref[b])
        print(f"[vae] attention N={N} B={B} sample {b}: 3xTF32 {e:.2e}, fp32 SDPA {e32:.2e}, one TF32 pass {e1:.2e}")
        # the split removes the operand rounding; left is the tensor core's truncating fp32 accumulation of P V over N keys,
        # which grows with N (tol_acc(N, 8): 1.6e-4 at 10 800 keys, measured up to 4.8e-5) past 20x fp32 SDPA's error and
        # to 1/15 of a single TF32 pass at 10^4 keys (H100): a tenth of that pass, 2.5x stricter than a 4x mutant margin
        assert e <= max(20 * e32, tol_acc(N, 8)) and e < 0.1 * e1


# ------------------------------------------------------------------------------------------------------------------
# 4. whole VAE against float64
# ------------------------------------------------------------------------------------------------------------------
DECODE_LATENTS = [(128, 96), (120, 90), (100, 75), (33, 35), (33, 25)]
ENCODE_IMAGES = [(1024, 768, 1), (800, 600, 1), (960, 720, 3)]
MUTANT_CASES = {"decode 128x96", "encode 800x600"}
# (case, mutant) -> the gates it must fail. A hand-off truncated instead of rounded passes every gate at both cases
# (measured: its slope moves by < 1.5e-5), so the truncation mutant is the parent's TF32 convolution operands (raw
# weights, an unrounded upsampler input), which the relative-L2 gate rejects.
MUTANT_GATES = {
    ("decode 128x96", "bf16_handoff"): ("max_ok", "l2_ok"),
    ("decode 128x96", "parent_tf32_truncation"): ("l2_ok",),
    ("encode 800x600", "bf16_handoff"): ("max_ok", "l2_ok", "slope_ok"),
}


@pytest.fixture(scope="module")
def vaes():
    """Seeded default initialisation, weights rounded to fp16 and held in fp32 (what pipeline._vae32 makes from the fp16
    VAE), and its float64 copy."""
    import idm_vton_b200.vae as V
    torch.manual_seed(0)
    vae16 = V.AutoencoderKL().half().eval()
    vae = copy.deepcopy(vae16).float().cuda()
    vae64 = copy.deepcopy(vae).double()
    return V, vae, vae64


def smooth_images(B, H, W, seed):
    """Sums of six random low-frequency plane waves, scaled into [-1, 1] per image."""
    g = torch.Generator().manual_seed(seed)
    yy = torch.linspace(0, 1, H, dtype=torch.float64)[:, None]
    xx = torch.linspace(0, 1, W, dtype=torch.float64)[None, :]
    img = torch.zeros(B, 3, H, W, dtype=torch.float64)
    for _ in range(6):
        f = torch.rand(B, 3, 2, generator=g, dtype=torch.float64) * 6 + 0.5
        ph = torch.rand(B, 3, 1, 1, generator=g, dtype=torch.float64) * 2 * math.pi
        img += torch.sin(2 * math.pi * (f[..., 0, None, None] * xx + f[..., 1, None, None] * yy) + ph)
    return (img / img.abs().amax((1, 2, 3), keepdim=True)).float()


def _run(vae, kind, inp):
    with torch.no_grad():
        if kind == "decode":
            return vae.decode(inp).sample
        d = vae.encode(inp).latent_dist
        return torch.cat([d.mean, d.logvar], 1)


def _route(V, monkeypatch, engine):
    monkeypatch.setattr(V, "_ENGINE_NHWC", engine)
    monkeypatch.setattr(V, "_ATTN_3XTF32", engine)


def _gates(y, y_ref, y64):
    """Per sample: (max-error ratio, rel-L2 ratio, slope gate value) and the raw numbers."""
    out = []
    for b in range(y64.shape[0]):
        e, er = rel_err(y[b], y64[b]), rel_err(y_ref[b], y64[b])
        l2, l2r = rel_l2(y[b], y64[b]), rel_l2(y_ref[b], y64[b])
        s, sr = slope(y[b], y64[b]), slope(y_ref[b], y64[b])
        out.append(dict(err=e, err_ref=er, l2=l2, l2_ref=l2r, slope_m1=s - 1, slope_ref_m1=sr - 1,
                        max_ok=e <= 1.5 * er, l2_ok=l2 <= 1.25 * l2r,
                        slope_ok=abs(s - 1) <= max(2 * abs(sr - 1), 2.0 ** -16)))
    return out


def _mutants(V, lib_mod, monkeypatch, vae, kind, inp, y_ref, y64):
    """The gates applied to mutated engine routes: the fp16 hand-off rounded through bf16, and (decode) the parent's TF32
    operands: raw weights and an unrounded upsampler input, which the tensor core truncates."""
    orig_gn = lib_mod.groupnorm_f32_nhwc

    def bf16(x, gamma, beta, eps, silu, out_half=False):
        y = orig_gn(x, gamma, beta, eps, silu)
        return y.bfloat16().half() if out_half else y

    res = {}
    muts = [("bf16_handoff", lib_mod, "groupnorm_f32_nhwc", bf16)]
    if kind == "decode":
        muts.append(("parent_tf32_truncation", V, ("_tf32", "_tf32_"), lambda t: t))
    for name, owner, attrs, fn in muts:
        with monkeypatch.context() as m:
            for attr in (attrs if isinstance(attrs, tuple) else (attrs,)):
                m.setattr(owner, attr, fn)
            for mod in vae.modules():                      # packed weights are cached per module
                for a in ("_b200_packed", "_b200_packed16"):
                    if hasattr(mod, a):
                        delattr(mod, a)
            res[name] = _gates(_run(vae, kind, inp), y_ref, y64)
    for mod in vae.modules():
        for a in ("_b200_packed", "_b200_packed16"):
            if hasattr(mod, a):
                delattr(mod, a)
    return res


VAE_CASES = [("decode", f"{h}x{w}", (h, w, 1)) for h, w in DECODE_LATENTS] + \
            [("encode", f"{h}x{w}" + (f" B={b}" if b > 1 else ""), (h, w, b)) for h, w, b in ENCODE_IMAGES]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,label,shape", VAE_CASES, ids=[f"{k}_{l.replace(' ', '_')}" for k, l, _ in VAE_CASES])
def test_vae_against_float64(vaes, monkeypatch, kind, label, shape):
    V, vae, vae64 = vaes
    from idm_vton_b200 import lib as lib_mod
    h, w, B = shape
    if kind == "decode":
        g = torch.Generator().manual_seed(h * w)
        inp = (torch.randn(B, 4, h, w, generator=g) / vae.config.scaling_factor).cuda()
    else:
        inp = smooth_images(B, h, w, seed=h + w + B).cuda()
    case = f"{kind} {label}"
    with torch.backends.cudnn.flags(enabled=True, benchmark=False, deterministic=False, allow_tf32=True):
        prev = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = False            # torch's default: fp32 SDPA / matmuls in full fp32
        try:
            y64 = _run(vae64, kind, inp.double())
            _route(V, monkeypatch, False)
            y_ref = _run(vae, kind, inp)
            _route(V, monkeypatch, True)
            y = _run(vae, kind, inp)
            singles = torch.cat([_run(vae, kind, inp[i:i + 1]) for i in range(B)]) if B > 1 else None
            muts = _mutants(V, lib_mod, monkeypatch, vae, kind, inp, y_ref, y64) if case in MUTANT_CASES else {}
        finally:
            torch.backends.cuda.matmul.allow_tf32 = prev
    for t in (y, y_ref, y64):
        assert torch.isfinite(t).all()
    gates = _gates(y, y_ref, y64)
    for b, gt in enumerate(gates):
        std64 = y64[b].std().item()
        rec = dict(case=case, sample=b, std64=std64, **{k: v for k, v in gt.items() if not k.endswith("_ok")},
                   peak_gb=torch.cuda.max_memory_allocated() / 1e9)
        if singles is not None:
            rec["batched_vs_single"] = rel_err(y[b], singles[b])
        for mn, mg in muts.items():
            rec[f"mutant_{mn}"] = {k: v for k, v in mg[b].items() if k in ("err", "l2", "slope_m1", "max_ok", "l2_ok",
                                                                             "slope_ok")}
        print("PARITY " + json.dumps(rec))
        assert 1e-3 < std64 < 1e3, f"{case}: float64 output std {std64:.3e} out of range: a vacuous comparison"
        assert gt["max_ok"], f"{case} sample {b}: max error {gt['err']:.3e} > 1.5x the yardstick's {gt['err_ref']:.3e}"
        assert gt["l2_ok"], f"{case} sample {b}: rel L2 {gt['l2']:.3e} > 1.25x the yardstick's {gt['l2_ref']:.3e}"
        assert gt["slope_ok"], f"{case} sample {b}: slope-1 {gt['slope_m1']:+.3e} (yardstick {gt['slope_ref_m1']:+.3e})"
    if singles is not None:
        # the batched encode and the per-sample encodes differ by more than fp32 reordering (cuDNN picks other TF32
        # algorithms per batch size; measured 2e-3 of scale, the size of the TF32 error itself): each must be as close to
        # the truth as the yardstick
        for b, gt in enumerate(_gates(singles, y_ref, y64)):
            assert gt["max_ok"] and gt["l2_ok"] and gt["slope_ok"], (case, "per-sample encode", b, gt)
    for (c, mn), gate in MUTANT_GATES.items():
        if c == case:
            for k in gate:
                assert not any(m[k] for m in muts[mn]), f"{case}: mutant {mn} passes the {k} gate"


# ------------------------------------------------------------------------------------------------------------------
# CPU: the models are what they say, and every mutant is at least 4x the tolerance away at the shapes above
# ------------------------------------------------------------------------------------------------------------------
def test_tf32_models_match_their_definition():
    """Against an independent float64 statement: |x| = m 2^e, m in [1, 2); TF32 keeps 10 fraction bits of m."""
    v = special_values()
    v = v[torch.isfinite(v) & (v.abs() >= 2.0 ** -126) & (v.abs() < 2.0 ** 127)]   # normal, no carry past FLT_MAX
    d = v.double()
    m, e = torch.frexp(d.abs())                            # m in [0.5, 1)
    q = m * 2.0 ** 11                                      # [1024, 2048): 11 significant bits
    assert torch.equal(tf32_trunc(v), d.sign() * torch.floor(q) * 2.0 ** (e - 11).double())
    assert torch.equal(tf32_rn(v), d.sign() * torch.floor(q + 0.5) * 2.0 ** (e - 11).double())   # ties away from zero
    ties = (v.view(torch.int32) & 8191) == 0x1000
    assert ties.sum() >= 256 and (tf32_rn(v[ties]).abs() > d[ties].abs()).all()
    import idm_vton_b200.vae as V
    assert bits_equal(V._tf32(v), tf32_rn(v).float()) and bits_equal(V._tf32_(v.clone()), tf32_rn(v).float())
    assert bits_equal(V._split_tf32(v)[1], split_ref(v)[1])


@pytest.mark.parametrize("Cin,Cout", CONV_CASES)
def test_conv_operand_models_separate(Cin, Cout):
    """At every conv shape: the two models are > 4x the accumulation tolerance apart, rounding has |slope - 1| under
    SLOPE_TOL / 4 and truncation a slope below 1 - 4 SLOPE_TOL."""
    x, w, _, _ = conv_operands(Cin, Cout)
    y64 = conv64(x, w)
    rn, tr = conv64(tf32_rn(x), tf32_rn(w)), conv64(tf32_trunc(x), tf32_trunc(w))
    assert per_sample(tr, rn) >= 4 * tol_acc(9 * Cin, 8) and per_sample(rn, tr) >= 4 * tol_acc(9 * Cin, 8)
    assert abs(slope(rn, y64) - 1) <= SLOPE_TOL / 4
    assert slope(tr, y64) - 1 <= -4 * SLOPE_TOL


@pytest.mark.parametrize("Cin,Cout", F16_CASES)
def test_f16in_mutant_separates(Cin, Cout):
    x, w, b, res = conv_operands(Cin, Cout, seed=1)
    acc = conv64(x.half(), w.half())
    ref = f16in_ref(acc, b, res)
    assert per_sample(f16in_ref(acc, b, res, mutant="acc_fp16"), ref) >= 4 * tol_acc(9 * Cin, 16)


@pytest.mark.parametrize("B,H,W,Cout", EPI_BOXES)
def test_epilogue_mutants_differ(B, H, W, Cout):
    x, w, b, res = epi_operands(B, H, W, Cout)
    acc = F.conv2d(x, w, padding=1)
    assert torch.equal(acc.float().double(), acc)                               # exact accumulation: bit-exact gates hold
    ref = epi_ref(acc, b, res)
    assert rel_err(epi_ref(acc, b, res, "res_before_bias"), ref) > 0
    assert rel_err(epi_ref(acc, b, res, "res_wrong_sample"), ref) > 0.1


@pytest.mark.parametrize("name,B,H,W,C,silu,mutants", GN32_CASES, ids=[c[0] for c in GN32_CASES])
def test_groupnorm_references_and_mutants(name, B, H, W, C, silu, mutants):
    """gn64 is F.group_norm in float64, and each case's mutants are >= 4x TOL_GN32 from it."""
    x, gamma, beta = gn_input(name, B, H, W, C)
    ref = gn64(x, gamma, beta, silu)
    direct = F.group_norm(x.double(), 32, gamma.double(), beta.double(), 1e-6)
    assert torch.allclose(ref, F.silu(direct) if silu else direct, rtol=1e-10, atol=1e-10)
    for m in mutants:
        assert per_sample(gn64(x, gamma, beta, silu, mutant=m), ref) >= 4 * TOL_GN32, m
    if name == "bench_level":
        assert gn_chunks(B, H * W) == (1183, 665) and H * W - 1182 * 665 == 402     # a ragged last chunk


def test_softmax_cases_and_mutant():
    for rows, N in SOFTMAX_SHAPES:
        s = softmax_scores(rows, N, seed=N)[:10]
        e = torch.exp(s - s.amax(-1, keepdim=True))
        assert (e[0] > 0).sum().item() == 1                                    # row 0: every other weight underflows
        assert not torch.isfinite(softmax_no_max(s)[2:]).all()                 # the mutant overflows on the +-100 rows
        assert s[2:].abs().max().item() > 88.8


def test_float64_vae_takes_the_torch_route(monkeypatch):
    """In float64 no vae.py switch reaches the engine: with lib.load raising, and the device conditions lifted so that
    only the dtype conditions decide, the float64 VAE runs, while its float32 twin reaches the engine (and raises)."""
    import idm_vton_b200.vae as V
    from idm_vton_b200 import lib as L

    def no_engine(*a, **k):
        raise RuntimeError("engine called")

    monkeypatch.setattr(L, "load", no_engine)
    monkeypatch.setattr(V, "_use_nhwc", lambda t: V._ENGINE_NHWC and t.dtype == torch.float32 and t.dim() == 4)
    monkeypatch.setattr(V, "_conv_device_ok", lambda t: True)
    monkeypatch.setattr(L, "conv3x3_f32_supported", lambda t, cin, cout: cin % 32 == 0 and cout % 32 == 0 and cout >= 64)
    torch.manual_seed(0)
    vae = V.AutoencoderKL(block_out_channels=(64, 64), layers_per_block=1).eval()
    x = torch.rand(1, 3, 32, 24, dtype=torch.float64) * 2 - 1
    z = torch.randn(1, 4, 16, 12, dtype=torch.float64)
    vae64 = copy.deepcopy(vae).double()
    y = _run(vae64, "encode", x)
    img = _run(vae64, "decode", z)
    assert y.dtype == img.dtype == torch.float64 and torch.isfinite(img).all()
    for kind, inp in (("encode", x.float()), ("decode", z.float())):
        with pytest.raises(RuntimeError, match="engine called"):
            _run(vae, kind, inp)
