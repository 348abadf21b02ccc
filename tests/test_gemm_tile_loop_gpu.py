"""The GEMM / convolution kernel's tile loop and its epilogue on the accumulator fragments.

A CTA of gemm_conv_kernel walks tiles b, b + grid, ... with one operand ring and one slab counter that run on across
tiles, and stores from the wgmma fragment after a transposition across each quad. The cases here are the ones that depend
on that: many tiles per CTA with a slab count the ring depth does not divide, fewer tiles than SMs, ragged edges in both
directions at once with guard bands around the output, conv boxes that reach past the batch, and the fp32-output kinds.

Two kinds of reference, both exact:
  * the same call split along M into pieces of at most one wave of tiles: a row's arithmetic does not depend on which tile
    or which CTA carries it, so the outputs are bit-identical;
  * operands on a coarse grid (products and their fp32 sums are exact), against the epilogue's rounding points written
    out in float64: bit-identical as well.
Every test runs its launches once."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _lib():
    from idm_vton_b200 import lib as L
    L.load()
    return L


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def rnd16(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).half().to(DEV)


def grid(*shape, seed, dtype=torch.float16, levels=8):
    """Values k / levels, |k| <= levels: exact in fp16 and TF32, and so are sums of a few hundred of their products."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    k = torch.randint(-levels, levels + 1, shape, generator=g).double()
    return (k / levels).to(dtype).to(DEV)


def r16(x):
    return x.half().double()


# ------------------------------------------------------------------------------------------------------------------
# many tiles per CTA: the whole call against the same call in pieces of at most one wave
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [64, 192, 320])          # 1, 3, 5 slabs: no ring depth (4, 5, 6, 8) divides all of them
@pytest.mark.parametrize("bn", [64, 128, 160, 192, 256])
def test_gemm_many_tiles_matches_single_wave_pieces(bn, K):
    L = _lib()
    sms = _sms()
    N = 2 * bn
    m_tiles = (5 * sms + 1) // 2 + 1                     # x 2 n tiles: more than 5 tiles per CTA, not a multiple of the grid
    M = m_tiles * 128 - 37
    a, w = rnd16(M, K, seed=1), rnd16(N, K, scale=K ** -0.5, seed=2)
    bias, res = rnd16(N, seed=3), rnd16(M, N, seed=4)
    rowvec = rnd16(m_tiles, N, seed=5)                   # one "sample" per 128 rows
    whole = L.gemm(a, w, bias=bias, residual=res, rowvec=rowvec, rows_per_sample=128, force_bn=bn)
    pieces = torch.empty_like(whole)
    step = (sms // 2) * 128
    for r in range(0, M, step):
        e = min(M, r + step)
        L.gemm(a[r:e], w, bias=bias, residual=res[r:e], rowvec=rowvec[r // 128:], rows_per_sample=128, out=pieces[r:e],
               force_bn=bn)
    torch.cuda.synchronize()
    assert torch.equal(whole, pieces)


@pytest.mark.parametrize("K", [64, 192, 320])
@pytest.mark.parametrize("bn", [128, 256])
def test_geglu_many_tiles_matches_single_wave_pieces(bn, K):
    from idm_vton_b200.engine import pack_geglu
    L = _lib()
    sms = _sms()
    N = 2 * bn
    m_tiles = (5 * sms + 1) // 2 + 1
    M = m_tiles * 128 - 37
    a = rnd16(M, K, seed=6)
    wp, bp = pack_geglu(rnd16(N, K, scale=K ** -0.5, seed=7), rnd16(N, seed=8), bn)
    whole = L.gemm(a, wp, bias=bp, geglu=True, force_bn=bn)
    pieces = torch.empty_like(whole)
    step = (sms // 2) * 128
    for r in range(0, M, step):
        e = min(M, r + step)
        L.gemm(a[r:e], wp, bias=bp, geglu=True, out=pieces[r:e], force_bn=bn)
    torch.cuda.synchronize()
    assert torch.equal(whole, pieces)


@pytest.mark.parametrize("shortcut", [False, True])
@pytest.mark.parametrize("bn", [64, 128])
def test_conv_many_tiles_matches_single_wave_pieces(bn, shortcut):
    """Cin = 64: 9 slabs (+ 2 shortcut slabs from two sources) per tile against rings of 8 and 6 stages."""
    from idm_vton_b200.engine import pack_conv3x3
    L = _lib()
    sms = _sms()
    H = W = 16                                           # two 16 x 8 boxes per image, x 2 n tiles
    Cin, Cout = 64, 2 * bn
    B = (5 * sms) // 4 + 2
    x = rnd16(B, H, W, Cin, seed=9)
    w = pack_conv3x3(rnd16(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=10))
    bias, temb = rnd16(Cout, seed=11), rnd16(B, Cout, seed=12)
    kw = {}
    if shortcut:
        sc0, sc1 = rnd16(B, H, W, 64, seed=13), rnd16(B, H, W, 64, seed=14)
        kw = dict(w_sc=rnd16(Cout, 128, scale=128 ** -0.5, seed=15), bias_sc=rnd16(Cout, seed=16))
    else:
        res = rnd16(B, H, W, Cout, seed=17)
    whole = L.conv3x3(x, w, bias=bias, temb=temb, force_bn=bn,
                      **(dict(sc0=sc0, sc1=sc1, **kw) if shortcut else dict(residual=res)))
    pieces = torch.empty_like(whole)
    step = sms // 4
    for b in range(0, B, step):
        e = min(B, b + step)
        extra = dict(sc0=sc0[b:e], sc1=sc1[b:e], **kw) if shortcut else dict(residual=res[b:e])
        L.conv3x3(x[b:e], w, bias=bias, temb=temb[b:e], out=pieces[b:e], force_bn=bn, **extra)
    torch.cuda.synchronize()
    assert torch.equal(whole, pieces)


# ------------------------------------------------------------------------------------------------------------------
# exact references on grid operands
# ------------------------------------------------------------------------------------------------------------------
def gemm_ref(a, w, bias, rowvec, rows_per_sample, res):
    """fp16(acc + bias); fp16(v + rowvec[m // rows_per_sample]); fp16(v + res) on the exact accumulator."""
    v = r16(a.double() @ w.double().t() + bias.double())
    if rowvec is not None:
        idx = torch.arange(a.shape[0], device=a.device) // rows_per_sample
        v = r16(v + rowvec.double()[idx])
    if res is not None:
        v = r16(v + res.double())
    return v.half()


@pytest.mark.parametrize("M,N,bn", [(100, 64, 64), (128, 256, 256), (128 * 7, 384, 192), (128 * 3 + 5, 320, 160)])
def test_gemm_fewer_tiles_than_sms(M, N, bn):
    """One tile ((100, 64) and (128, 256)) and a handful: the grid is the tile count and each CTA's loop runs once."""
    L = _lib()
    K = 192
    a, w = grid(M, K, seed=20), grid(N, K, seed=21)
    bias, res = grid(N, seed=22), grid(M, N, seed=23)
    out = L.gemm(a, w, bias=bias, residual=res, force_bn=bn)
    assert torch.equal(out, gemm_ref(a, w, bias, None, 0, res))


def test_gemm_ragged_m_and_n_leaves_guard_bands_alone():
    """Last M tile and last N tile ragged at once, output a strided view inside a sentinel-filled buffer: nothing past
    row M or past column N is written, and every element inside is exact."""
    L = _lib()
    M, N, K, G = 128 * 3 + 40, 200, 320, 8               # N = 128 + 72: the second n tile stops inside an 8-group run
    a, w = grid(M, K, seed=30), grid(N, K, seed=31)
    bias, res, rowvec = grid(N, seed=32), grid(M, N, seed=33), grid(4, N, seed=34)
    sentinel = -7.0
    buf = torch.full((M + 2 * G, N + 2 * G), sentinel, dtype=torch.float16, device=DEV)
    out = buf[G:G + M, G:G + N]
    L.gemm(a, w, bias=bias, residual=res, rowvec=rowvec, rows_per_sample=128, out=out)
    torch.cuda.synchronize()
    assert torch.equal(out, gemm_ref(a, w, bias, rowvec, 128, res))
    guard = buf.clone()
    guard[G:G + M, G:G + N] = sentinel
    assert torch.equal(guard, torch.full_like(buf, sentinel))


def test_conv_box_past_batch_with_time_embedding():
    """8 x 8 images: a box is two images, so with B = 3 the last box reaches one image past the batch. Its rows have no
    time-embedding row and no output row; the three real images are exact."""
    from idm_vton_b200.engine import pack_conv3x3
    L = _lib()
    B, H, W, Cin, Cout = 3, 8, 8, 64, 192
    x = grid(B, H, W, Cin, seed=40)
    wt = grid(Cout, Cin, 3, 3, seed=41)
    bias, temb, res = grid(Cout, seed=42), grid(B, Cout, seed=43), grid(B, H, W, Cout, seed=44)
    out = L.conv3x3(x, pack_conv3x3(wt), bias=bias, temb=temb, residual=res)
    acc = F.conv2d(x.double().permute(0, 3, 1, 2), wt.double(), padding=1).permute(0, 2, 3, 1)
    v = r16(acc + bias.double())
    v = r16(v + temb.double()[:, None, None, :])
    v = r16(v + res.double())
    assert torch.equal(out, v.half())


@pytest.mark.parametrize("in_fp16", [False, True])
@pytest.mark.parametrize("Cout", [96, 160, 288])         # tile widths 128 / 128 / 128: one ragged tile, 1 + ragged, 2 + ragged
def test_conv_f32_out_ragged_cout(Cout, in_fp16):
    L = _lib()
    B, H, W, Cin = 2, 16, 16, 64
    dt = torch.float16 if in_fp16 else torch.float32
    x = grid(B, Cin, H, W, seed=50, dtype=dt).contiguous(memory_format=torch.channels_last)
    wt = grid(Cout, Cin, 3, 3, seed=51, dtype=dt)
    bias = grid(Cout, seed=52, dtype=torch.float32)
    res = grid(B, Cout, H, W, seed=53, dtype=torch.float32)
    wp = L.pack_conv3x3_f32(wt)
    out = L.conv3x3_f16in(x, wp, bias=bias, residual=res) if in_fp16 else L.conv3x3_f32(x, wp, bias=bias, residual=res)
    ref = F.conv2d(x.double(), wt.double(), padding=1) + bias.double()[None, :, None, None] + res.double()
    assert torch.equal(out, ref.float())                 # every partial sum is a small multiple of 1/64: exact in fp32
