"""Schedule independence of the split fp16 epilogue of gemm_conv_kernel.

The consumer warpgroups write each finished tile, residual added, to a shared-memory staging tile and go on to the next
tile's K loop; the store warps (warps 9..11) store it while that loop runs and then bulk-copy the next tile's residual
into the staging tile, one staging tile per CTA guarded by a staged / ready mbarrier pair. A tile's arithmetic does not
depend on which CTA carries it or on what came before it in the CTA's schedule, so one launch with many tiles per CTA
must be bit-identical to the same problem computed as separate launches over slices of one 128-row tile (conv: a few
samples) each. A staging or handshake error (a tile read before it is staged, overwritten before it is stored, a
residual of the wrong tile, a row-table mismatch) shows up as a bit difference.

Every epilogue variant is covered, with ragged M and N where the variant allows it; the conv cases have a batch extent past
B in their last box."""
import pytest
import torch

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


def _m_rows():
    return (3 * _sms() + 5) * 128 - 45     # > 3 tiles per CTA along M alone, ragged last tile


def _slices(M, step=128):
    return [(r, min(M, r + step)) for r in range(0, M, step)]


# (variant, bn, N): N not a multiple of bn where the tile width allows a ragged last column tile
LINEAR_CASES = [
    ("bias", 64, 200),
    ("bias", 160, 480),
    ("residual", 128, 392),
    ("residual", 192, 384),
    ("residual", 256, 512),
    ("rowvec", 128, 264),
    ("rowvec", 256, 512),
    ("gelu", 128, 392),
    ("quick_gelu", 160, 320),
]


@pytest.mark.parametrize("variant,bn,N", LINEAR_CASES)
def test_linear_one_launch_matches_128_row_slices(variant, bn, N):
    L = _lib()
    M, K = _m_rows(), 192
    a, w = rnd16(M, K, seed=1), rnd16(N, K, scale=K ** -0.5, seed=2)
    kw = dict(bias=rnd16(N, seed=3))
    res = rnd16(M, N, seed=4) if variant == "residual" else None
    rowvec = rnd16(-(-M // 64), N, seed=5) if variant == "rowvec" else None   # two samples per 128-row tile
    kw.update(gelu=variant == "gelu", quick_gelu=variant == "quick_gelu", rows_per_sample=64 if rowvec is not None else 0)
    whole = L.gemm(a, w, residual=res, rowvec=rowvec, force_bn=bn, **kw)
    pieces = torch.full_like(whole, float("nan"))
    for r, e in _slices(M):
        L.gemm(a[r:e], w, residual=res[r:e] if res is not None else None,
               rowvec=rowvec[r // 64:] if rowvec is not None else None, out=pieces[r:e], force_bn=bn, **kw)
    torch.cuda.synchronize()
    assert torch.equal(whole, pieces)


@pytest.mark.parametrize("bn", [128, 256])
def test_geglu_one_launch_matches_128_row_slices(bn):
    from idm_vton_b200.engine import pack_geglu
    L = _lib()
    M, K, N = _m_rows(), 128, 4 * bn
    a, w, b = rnd16(M, K, seed=6), rnd16(N, K, scale=K ** -0.5, seed=7), rnd16(N, seed=8)
    wp, bp = pack_geglu(w, b, bn)
    whole = L.gemm(a, wp, bias=bp, geglu=True, force_bn=bn)
    pieces = torch.full_like(whole, float("nan"))
    for r, e in _slices(M):
        L.gemm(a[r:e], wp, bias=bp, geglu=True, out=pieces[r:e], force_bn=bn)
    torch.cuda.synchronize()
    assert torch.equal(whole, pieces)


@pytest.mark.parametrize("geglu,bn,N", [(False, 160, 480), (False, 256, 768), (True, 256, 1024)])
def test_e4m3_one_launch_matches_128_row_slices(geglu, bn, N):
    from idm_vton_b200.engine import pack_geglu
    L = _lib()
    M, K = _m_rows(), 256
    a, w, b = rnd16(M, K, seed=9), rnd16(N, K, scale=K ** -0.5, seed=10), rnd16(N, seed=11)
    if geglu:
        w, b = pack_geglu(w, b, bn)
    a_q, a_s = L.quantize_rows_e4m3(a)
    w_q, w_s = L.quantize_rows_e4m3(w)
    res = None if geglu else rnd16(M, N, seed=12)
    whole = L.gemm_e4m3(a_q, a_s, w_q, w_s, bias=b, residual=res, geglu=geglu, force_bn=bn)
    pieces = torch.full_like(whole, float("nan"))
    for r, e in _slices(M):
        L.gemm_e4m3(a_q[r:e], a_s[r:e], w_q, w_s, bias=b, residual=res[r:e] if res is not None else None, geglu=geglu,
                    out=pieces[r:e], force_bn=bn)
    torch.cuda.synchronize()
    assert torch.equal(whole, pieces)


# (variant, bn): 8x8 images tile as 2-sample boxes, so an odd B puts the last box's second sample past B
CONV_CASES = [("temb_residual", 64), ("temb_residual", 128), ("temb_residual", 160), ("temb_residual", 256),
              ("shortcut", 64), ("shortcut", 128)]


@pytest.mark.parametrize("variant,bn", CONV_CASES)
def test_conv_one_launch_matches_per_sample_launches(variant, bn):
    from idm_vton_b200.engine import pack_conv3x3
    L = _lib()
    Cout = 2 * bn if bn != 160 else 320
    B, H, W, Cin = 2 * (3 * _sms() // 2) + 1, 8, 8, 64   # > 3 tiles per CTA, odd B
    x = rnd16(B, H, W, Cin, seed=13)
    w = pack_conv3x3(rnd16(Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5, seed=14))
    b = rnd16(Cout, seed=15)
    if variant == "shortcut":
        C0, C1 = 64, 128
        sc0, sc1 = rnd16(B, H, W, C0, seed=16), rnd16(B, H, W, C1, seed=17)
        w_sc, b_sc = rnd16(Cout, C0 + C1, scale=(C0 + C1) ** -0.5, seed=18), rnd16(Cout, seed=19)

        def kw(s, e):
            return dict(sc0=sc0[s:e].contiguous(), sc1=sc1[s:e].contiguous(), w_sc=w_sc, bias_sc=b_sc)
    else:
        temb, res = rnd16(B, Cout, seed=20), rnd16(B, H, W, Cout, seed=21)

        def kw(s, e):
            return dict(temb=temb[s:e].contiguous(), residual=res[s:e].contiguous())
    whole = L.conv3x3(x, w, bias=b, force_bn=bn, **kw(0, B))
    pieces = torch.full_like(whole, float("nan"))
    for s in range(0, B, 3):
        e = min(B, s + 3)
        pieces[s:e] = L.conv3x3(x[s:e].contiguous(), w, bias=b, force_bn=bn, **kw(s, e))
    torch.cuda.synchronize()
    assert torch.equal(whole, pieces)
