"""Edge cases of the hot-path kernels against float64 restatements of the same op.

Every reference below is the op in float64 with the fp16 rounding points of the reference pipeline written out (the ones
of test_kernels_gpu.py, gemm_common.cuh and attn.cu). The metric is max|a - b| / max|b| (no floor), per (sample, head)
for attention, and each tolerance is derived from the op's rounding model in a comment beside it.

A gate is only worth something if it can fail. Where a plausible bug is small, the test builds the *mutant* reference as
well and asserts err(kernel, ref) <= 0.25 * err(mutant, ref); the CPU tests at the end of this file prove, without a
GPU, that every mutant is at least 4x the tolerance away from the true reference at every shape the GPU tests use.
The GPU tests are marked one by one (the CPU tests of the references run everywhere)."""
import math

import pytest
import torch
import torch.nn.functional as F

U16 = 2.0 ** -11          # fp16 unit roundoff: half an ulp, relative to the value

# fp16 GEMM / convolution on random operands vs the unrounded float64 product: the fp16 output rounding (<= U16 of the
# largest output) plus fp32 accumulation on the tensor cores (<= 2^-22 per addition; over K <= 2880 terms of random sign
# the accumulated error stays below 2^-13 of the output scale).
TOL_GEMM = U16 + 2.0 ** -13
# attention vs the exact float64 softmax, per (sample, head): the output rounding (U16) and P rounded to fp16 before P V
# (each term carries <= U16 relative error; the errors are independent, so the sum's error stays within ~3 U16 of the
# output scale at the tails of ~10^4 outputs), plus ex2.approx (2^-22): 4 U16, with one more U16 for the fp16 rounding of
# O_t and O_i that the decoupled cross-attention adds (ip cases) and that the restatement keeps exact.
TOL_ATTN = 4 * U16
TOL_ATTN_IP = 6 * U16
# GroupNorm / LayerNorm (fp16 out) vs float64 statistics: output rounding U16 plus the fp32 statistics and apply (2^-13)
TOL_NORM16 = U16 + 2.0 ** -13
# fp32 GroupNorm: fp32 partial sums of shifted values over short lanes (relative error of the variance well below 2^-20)
# and fp32 output: 2^-18 of the output scale; plus the fp32 rounding of the mean itself (2^-24 |mean|), which the
# normalised output carries in units of the group's std: offset * 2^-24 for a mean of offset x std
def tol_norm32(offset):
    return 2.0 ** -18 + offset * 2.0 ** -24
# epilogue cases on exactly-representable operands (the fp32 accumulator is exact): every fp16 rounding point of the
# kernel sees the same value as the restatement, so the result is bit-identical, except that the erf-GELU / quick-GELU of
# the kernel are approximations (< 2e-7 absolute) that may flip one intermediate rounding by an ulp: 2^-9 of the scale.
TOL_EPI_ACT = 2.0 ** -9


def r16(x):
    """Round to fp16 (round to nearest even), keep the dtype."""
    return x.half().to(x.dtype)


def rel_err(a, b):
    a, b = a.double(), b.double()
    den = b.abs().max().item()
    err = (a - b).abs().max().item()
    return err / den if den > 0 else (0.0 if err == 0 else math.inf)


def grid16(*shape, scale, seed, device="cpu", levels=8):
    """fp16 values on the grid k * scale / levels, |k| <= levels: products and their fp32 sums are exact."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    k = torch.randint(-levels, levels + 1, shape, generator=g).double()
    return (k * (scale / levels)).half().to(device)


def rnd16(*shape, scale=1.0, seed=0, device="cpu"):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g, dtype=torch.float64) * scale).half().to(device)


# ------------------------------------------------------------------------------------------------------------------
# float64 references
# ------------------------------------------------------------------------------------------------------------------
def gelu64(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def quick_gelu64(x):
    return x * torch.sigmoid(1.702 * x)


def gemm_epilogue_ref(acc, bias=None, act=None, rowvec=None, rows_per_sample=0, residual=None, mutant=None):
    """The fused fp16 epilogue of gemm_common.cuh on an exact accumulator acc [M, N] (float64):
    v = fp16(acc + bias); v = fp16(act(v)); v = fp16(v + rowvec[m // rows_per_sample]); v = fp16(v + residual).
    mutant: 'gelu_before_bias' | 'rowvec_tile_sample' (sample of the 128-row tile's first row) | 'res_before_round'
    (residual added before the rowvec sum is rounded)."""
    v = acc.double()
    if act is not None and mutant == "gelu_before_bias":
        v = r16(act(r16(v)))
        v = v + bias.double() if bias is not None else v
        v = r16(v)
    else:
        v = r16(v + bias.double()) if bias is not None else r16(v)
        if act is not None:
            v = r16(act(v))
    if rowvec is not None:
        m = torch.arange(v.shape[0], device=v.device)
        if mutant == "rowvec_tile_sample":
            m = m // 128 * 128
        idx = m // rows_per_sample if rows_per_sample > 0 else torch.zeros_like(m)
        v = v + rowvec.double()[idx]
        if residual is None or mutant != "res_before_round":
            v = r16(v)
    if residual is not None:
        v = r16(v + residual.double())
    return v


def conv3x3_acc(x, w, stride=1):
    """x [B,H,W,Cin] NHWC, w [Cout,Cin,3,3] -> exact float64 accumulator [B,Ho,Wo,Cout]."""
    y = F.conv2d(x.double().permute(0, 3, 1, 2), w.double(), None, stride=stride, padding=1)
    return y.permute(0, 2, 3, 1)


def attn_head_ref(q, k, v, scale, n_zero=0, causal=False, mutant=None):
    """softmax(q k^T * scale) v for one (sample, head) in float64: q [Nq, D], k / v [Nk, D]; n_zero all-zero key/value
    tokens appended (the CFG-uncond closed form); causal: key j visible to query i iff j <= i.
    mutant 'no_alpha_rescale': the zero tokens weighted exp(-max(m, 0)) while the real weights exp(s - m) (and so o
    and l) are not rescaled by alpha = exp(m - max(m, 0)): wrong whenever every real score is negative."""
    q, k, v = q.double(), k.double(), v.double()
    s = q @ k.t() * scale
    if causal:
        s = s.masked_fill(torch.ones_like(s, dtype=torch.bool).triu(1), -math.inf)
    if mutant == "no_alpha_rescale":
        m = s.max(-1, keepdim=True).values
        e = torch.exp(s - m)
        return (e @ v) / (e.sum(-1, keepdim=True) + n_zero * torch.exp(-m.clamp(min=0)))
    if n_zero:
        s = torch.cat([s, s.new_zeros(s.shape[0], n_zero)], 1)
        v = torch.cat([v, v.new_zeros(n_zero, v.shape[1])], 0)
    return torch.softmax(s, -1) @ v


def attn_errs(out, q, k, v, heads, D, scale, **kw):
    """Per-(sample, head) errors of out [B, Nq, >= heads*D] against attn_head_ref; q/k/v are [B, N, >= heads*D]."""
    errs = []
    for b in range(q.shape[0]):
        for h in range(heads):
            c = slice(h * D, (h + 1) * D)
            ref = attn_head_ref(q[b, :, c], k[b, :, c], v[b, :, c], scale, **kw)
            errs.append(rel_err(out[b, :, c], ref))
    return errs


def group_norm64(x, groups, gamma, beta, eps):
    """x [B, HW, C] -> float64 GroupNorm (two-pass statistics)."""
    xd = x.double().transpose(1, 2)
    y = F.group_norm(xd, groups, gamma.double() if gamma is not None else None,
                     beta.double() if beta is not None else None, eps)
    return y.transpose(1, 2)


def report(name, err, tol, mutant_errs=None):
    m = min(mutant_errs.values()) if mutant_errs else None
    margin = f"{m / err:.1f}x" if mutant_errs and err > 0 else "inf"
    extra = f"  smallest mutant err {m:.3e} ({min(mutant_errs, key=mutant_errs.get)}) margin {margin}" \
        if mutant_errs else ""
    print(f"[edge] {name}: err {err:.3e} (tol {tol:.2e}){extra}")
    assert math.isfinite(err) and err <= tol, f"{name}: err {err:.3e} > tol {tol:.2e}"
    for mn, me in (mutant_errs or {}).items():
        assert err <= 0.25 * me, f"{name}: err {err:.3e} not below a quarter of mutant {mn} ({me:.3e})"


# ------------------------------------------------------------------------------------------------------------------
# case tables shared by the GPU tests and the CPU checks of the mutants
# ------------------------------------------------------------------------------------------------------------------
# GEMM: every forced width with K-slab counts 1, STAGES-1, STAGES, STAGES+1, 2*STAGES+1 (gemm.cu dispatch)
STAGES = {64: 8, 128: 6, 160: 5, 192: 4, 256: 4}
GEMM_SLAB_CASES = [(bn, s) for bn in (64, 128, 160, 192, 256)
                   for s in sorted({1, STAGES[bn] - 1, STAGES[bn], STAGES[bn] + 1, 2 * STAGES[bn] + 1})]
# (M, N, K, force_bn): M tails 1 / 65 / 127, N of 8 / 16 / 24, N % BN of 8 and 40
GEMM_EDGE_SHAPES = [(1, 64, 64, 0), (65, 128, 128, 0), (127, 192, 64, 0), (129, 8, 64, 0), (200, 16, 128, 64),
                    (77, 24, 64, 0), (300, 264, 128, 128), (256, 296, 192, 256), (131, 168, 64, 160),
                    (64, 200, 128, 192), (127, 8, 64, 256)]
# epilogue combinations: (name, M, N, K, rows_per_sample, act, mutants)
EPI_CASES = [
    ("bias_gelu_rowvec_res", 300, 192, 128, 150, "gelu", ("gelu_before_bias", "rowvec_tile_sample")),
    ("quickgelu_res", 200, 128, 64, 0, "quick", ("gelu_before_bias",)),
    ("rows_per_sample_77", 4 * 77, 320, 128, 77, None, ("rowvec_tile_sample", "res_before_round")),
    ("rows_per_sample_300", 3 * 300, 256, 64, 300, None, ("rowvec_tile_sample", "res_before_round")),
    ("strided", 2 * 77, 128, 64, 77, None, ("rowvec_tile_sample", "res_before_round")),
]
# attention: (name, B, H, Nq, N0, N1, segment-1 kind, kernel options)
ATTN_CASES = [
    ("one_tile_n1", 1, 2, 129, 1, 0, None),
    ("n0_127", 1, 2, 127, 127, 0, None),
    ("n0_128", 1, 2, 128, 128, 0, None),
    ("n0_129", 1, 2, 1, 129, 0, None),
    ("n0_257", 2, 2, 257, 257, 0, None),
    ("seg_127_1", 2, 2, 130, 127, 1, "kv"),
    ("seg_1_129", 1, 3, 128, 1, 129, "kv"),
    ("seg_128_257", 2, 2, 129, 128, 257, "kv"),          # 1 + 3 tiles
    ("seg_129_257", 1, 2, 127, 129, 257, "kv"),          # 2 + 3 = 5 tiles
    ("seg_257_129_base_last", 2, 2, 128, 257, 129, "base"),   # kv1_base + kv1_mod reaching the last slice
]
# zero-K/V closed form: (name, H, Nq, N0, N1, q kind, mutants)
ZERO_KV_CASES = [
    ("negative_scores", 2, 128, 128, 16, "negative", ("n1_minus", "n1_plus", "no_alpha_rescale")),
    ("negative_scores_129", 2, 129, 129, 17, "negative", ("n1_minus", "n1_plus", "no_alpha_rescale")),
    ("n0_1_n1_1", 2, 127, 1, 1, "random", ("n1_minus", "n1_plus")),
    ("n0_127_n1_1", 2, 128, 127, 1, "deep", ("n1_minus", "n1_plus", "no_alpha_rescale")),
    ("n0_129_n1_127", 1, 130, 129, 127, "small", ()),
    ("underflow", 2, 128, 257, 128, "large", ()),
]
ENC_DIMS = (16, 32, 48, 64, 80, 96)
ENC_NS = (1, 127, 128, 129, 257)


def zero_kv_inputs(kind, H, Nq, N0, seed):
    """q/k/v [1, N, H*64] fp16 for the zero-K/V cases. 'negative': every real score in [-1.5, -1] with N1 ~ N0/8, so real
    and zero tokens carry comparable mass ('deep': the same for N1 = 1); 'small': scores of a few tenths (the zero tokens matter); 'large': scores in
    the hundreds, so exp(-m) of the zero tokens underflows."""
    C = H * 64
    g = torch.Generator().manual_seed(seed)
    if kind == "negative":
        q = torch.rand(1, Nq, C, generator=g, dtype=torch.float64) * 0.25 + 0.5
        k = -(torch.rand(1, N0, C, generator=g, dtype=torch.float64) * 0.25 + 0.25)
        # score = 0.125 * sum_64(q * k): q*k in [-0.1875, -0.125] * 64 * 0.125 = [-1.5, -1]
    elif kind == "deep":          # scores in [-5.3, -4]: 127 real tokens weigh about as much as one zero token
        q = torch.rand(1, Nq, C, generator=g, dtype=torch.float64) * 0.1 + 0.8
        k = -(torch.rand(1, N0, C, generator=g, dtype=torch.float64) * 0.07 + 0.625)
    elif kind == "large":
        q = torch.randn(1, Nq, C, generator=g, dtype=torch.float64) * 8
        k = torch.randn(1, N0, C, generator=g, dtype=torch.float64) * 8
    elif kind == "small":
        q = torch.randn(1, Nq, C, generator=g, dtype=torch.float64) * 0.4
        k = torch.randn(1, N0, C, generator=g, dtype=torch.float64) * 0.4
    else:
        q = torch.randn(1, Nq, C, generator=g, dtype=torch.float64)
        k = torch.randn(1, N0, C, generator=g, dtype=torch.float64)
    v = torch.randn(1, N0, C, generator=g, dtype=torch.float64)
    return q.half(), k.half(), v.half()


def zero_kv_ref(q, k, v, H, n1, mutant=None):
    outs = []
    for h in range(H):
        c = slice(64 * h, 64 * h + 64)
        if mutant in ("n1_minus", "n1_plus"):
            outs.append(attn_head_ref(q[0, :, c], k[0, :, c], v[0, :, c], 0.125, n_zero=n1 + (1 if mutant == "n1_plus" else -1)))
        else:
            outs.append(attn_head_ref(q[0, :, c], k[0, :, c], v[0, :, c], 0.125, n_zero=n1, mutant=mutant))
    return outs


def ip_exact_inputs(H, Nq, Nt, Ni, device="cpu"):
    """Decoupled cross-attention with q = 0: every score is 0, the softmax is a plain mean the kernel computes exactly
    (P = 1, l = N, grid-valued V sums exactly in fp32), so only the fp16 rounding points decide the result. Vi is Vt plus
    a small grid perturbation and ip_scale = -1: the output nearly cancels, which magnifies the rounding of O_t (N = 12 is
    not a power of two, so the mean is not an fp16 value)."""
    C = H * 64
    q = torch.zeros(1, Nq, C, dtype=torch.float16, device=device)
    kt = rnd16(1, Nt, C, seed=61, device=device)
    ki = rnd16(1, Ni, C, seed=62, device=device)
    vt = grid16(1, Nt, C, scale=2.0, seed=63, device=device, levels=64)
    vi = (vt.double() + grid16(1, Ni, C, scale=1 / 256, seed=64, device=device, levels=1).double()).half()
    return q, kt, vt, ki, vi


def ip_ref(ot, oi, ip_scale, mutant=None):
    """out = fp16(fp16(O_t) + fp16(ip_scale * fp16(O_i))); mutant 'ot_unrounded': O_t enters the sum unrounded."""
    t = ot if mutant == "ot_unrounded" else r16(ot)
    return r16(t + r16(ip_scale * r16(oi)))


def mean_attn(v):
    return v.double().mean(1)            # [1, N, C] -> [1, C]: the softmax of all-zero scores


# ------------------------------------------------------------------------------------------------------------------
# GPU tests
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from idm_vton_b200 import lib as L
    L.load()
    return L


@pytest.mark.gpu
@pytest.mark.parametrize("bn,slabs", GEMM_SLAB_CASES)
def test_gemm_tile_width_and_pipeline_depth(lib, bn, slabs):
    """Each forced width at K-slab counts around its ring depth (the mbarrier phase flips at STAGES), M with a ragged
    last tile, N with a partial last tile; every width agrees with the forced 128-wide tile within the gate."""
    M, N, K = 257, 2 * bn + 40, 64 * slabs
    a, w = rnd16(M, K, seed=1, device="cuda"), rnd16(N, K, scale=K ** -0.5, seed=2, device="cuda")
    out = lib.gemm(a, w, force_bn=bn)
    ref = a.double() @ w.double().t()
    report(f"gemm bn={bn} slabs={slabs}", rel_err(out, ref), TOL_GEMM)
    o128 = lib.gemm(a, w, force_bn=128)
    assert rel_err(out, o128) <= 2 * TOL_GEMM


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K,bn", GEMM_EDGE_SHAPES)
def test_gemm_ragged_shapes(lib, M, N, K, bn):
    a, w = rnd16(M, K, seed=3, device="cuda"), rnd16(N, K, scale=K ** -0.5, seed=4, device="cuda")
    out = lib.gemm(a, w, force_bn=bn)
    report(f"gemm M={M} N={N} K={K} bn={bn}", rel_err(out, a.double() @ w.double().t()), TOL_GEMM)


def _epi_operands(name, M, N, K, rps, device):
    a = grid16(M, K, scale=1.0, seed=11, device=device)
    w = grid16(N, K, scale=0.25, seed=12, device=device)
    bias = rnd16(N, seed=13, device=device)
    S = (M + rps - 1) // rps if rps else 1
    if name == "strided":
        rv_buf = rnd16(S, N + 24, seed=14, device=device)
        res_buf = rnd16(M, N + 40, seed=15, device=device)
        return a, w, bias, rv_buf[:, 16:16 + N], res_buf[:, 8:8 + N]
    rv = rnd16(S, N, seed=14, device=device) if rps else None
    return a, w, bias, rv, rnd16(M, N, seed=15, device=device)


@pytest.mark.gpu
@pytest.mark.parametrize("name,M,N,K,rps,act,mutants", EPI_CASES, ids=[c[0] for c in EPI_CASES])
def test_gemm_epilogue_rounding_points(lib, name, M, N, K, rps, act, mutants):
    """bias / GELU / rowvec / residual with the reference's rounding points, on operands whose fp32 accumulation is exact
    (the result is then bit-identical without an activation). rows_per_sample 77 / 150 / 300 put sample boundaries
    inside 128-row tiles; 'strided' passes row-strided rowvec / residual / out views."""
    a, w, bias, rv, res = _epi_operands(name, M, N, K, rps, "cuda")
    actf = {"gelu": gelu64, "quick": quick_gelu64, None: None}[act]
    out = None
    if name == "strided":
        big = torch.zeros(M, N + 64, dtype=torch.float16, device="cuda")
        out = big[:, 32:32 + N]
    out = lib.gemm(a, w, bias=bias, residual=res, rowvec=rv, rows_per_sample=rps, gelu=act == "gelu",
                   quick_gelu=act == "quick", out=out)
    if name == "strided":
        assert big[:, :32].abs().max().item() == 0 and big[:, 32 + N:].abs().max().item() == 0
    acc = a.double() @ w.double().t()
    ref = gemm_epilogue_ref(acc, bias, actf, rv, rps, res)
    tol = TOL_EPI_ACT if act else 0.0
    errs = {m: rel_err(gemm_epilogue_ref(acc, bias, actf, rv, rps, res, mutant=m), ref) for m in mutants}
    report(f"gemm epilogue {name}", rel_err(out, ref), tol, errs)
    if not act:
        assert torch.equal(out.double(), ref)


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W,Cin,Cout,temb_off", [
    (2, 12, 8, 320, 16, 0),        # conv_out: Cout padded to 16, N < 64
    (3, 2, 1, 64, 64, 64),         # W = 1: one-pixel boxes, H below the box height, B not a multiple of the batch extent
    (5, 3, 3, 128, 128, 128),      # W = 3
    (3, 5, 6, 64, 192, 320),       # W = 6
    (2, 4, 24, 64, 320, 640),      # W = 24
])
def test_conv3x3_boxes_and_temb_slice(lib, B, H, W, Cin, Cout, temb_off):
    """Implicit-GEMM convolution at box shapes where the pixel box spans several samples, with temb a column slice at a
    non-zero offset of a wider tensor (what _resnet passes: temb_all[:, off:off+cout]). Exact accumulation: bit-identical
    to the restatement; a temb taken from the wrong sample is caught."""
    from idm_vton_b200.engine import pack_conv3x3
    x = grid16(B, H, W, Cin, scale=1.0, seed=21, device="cuda")
    w = grid16(Cout, Cin, 3, 3, scale=0.25, seed=22, device="cuda")
    bias = rnd16(Cout, seed=23, device="cuda")
    temb_all = rnd16(B, temb_off + Cout + 64, seed=24, device="cuda")
    temb = temb_all[:, temb_off:temb_off + Cout]
    out = lib.conv3x3(x, pack_conv3x3(w), bias=bias, temb=temb)
    acc = conv3x3_acc(x, w)
    ref = r16(r16(acc + bias.double()) + temb.double()[:, None, None, :])
    wrong = r16(r16(acc + bias.double()) + temb.double().roll(1, 0)[:, None, None, :])
    report(f"conv B={B} H={H} W={W} Cout={Cout}", rel_err(out, ref), 0.0, {"temb_wrong_sample": rel_err(wrong, ref)})
    assert torch.equal(out.double(), ref)


@pytest.mark.gpu
@pytest.mark.parametrize("C0,C1,Cout,bn", [(192, 0, 128, 64), (320, 0, 64, 128), (128, 192, 128, 64)])
def test_conv3x3_shortcut_slab_counts(lib, C0, C1, Cout, bn):
    """Fused 1x1 shortcut with main + shortcut slab totals that are not multiples of STAGES (9 * Cin/64 + Csc/64)."""
    from idm_vton_b200.engine import pack_conv3x3
    B, H, W = 2, 8, 16
    h = grid16(B, H, W, Cout, scale=1.0, seed=31, device="cuda")
    s0 = grid16(B, H, W, C0, scale=1.0, seed=32, device="cuda")
    s1 = grid16(B, H, W, C1, scale=1.0, seed=33, device="cuda") if C1 else None
    w = grid16(Cout, Cout, 3, 3, scale=0.25, seed=34, device="cuda")
    wsc = grid16(Cout, C0 + C1, scale=0.25, seed=35, device="cuda")
    b2, bsc = rnd16(Cout, seed=36, device="cuda"), rnd16(Cout, seed=37, device="cuda")
    out = lib.conv3x3(h, pack_conv3x3(w), bias=b2, sc0=s0, sc1=s1, w_sc=wsc, bias_sc=bsc, force_bn=bn)
    cat = torch.cat([s0, s1], -1) if C1 else s0
    ref = r16(r16(cat.double() @ wsc.double().t() + bsc.double()) + r16(conv3x3_acc(h, w) + b2.double()))
    report(f"conv shortcut C0={C0} C1={C1} bn={bn}", rel_err(out, ref), 0.0)
    assert torch.equal(out.double(), ref)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,Cin,Cout", [("tf32", 32, 96), ("tf32", 64, 160), ("f16", 64, 96), ("f16", 128, 160)])
def test_conv3x3_fp32_out_cout_not_tile_multiple(lib, kind, Cin, Cout):
    """The VAE's fp32-output convolutions at Cout = 96 / 160 (a partial last 128-wide tile), TF32 also at Cin = 32.
    Grid operands: products and sums are exact in TF32 / fp16 operands with fp32 accumulation, so the result equals the
    float64 convolution up to the fp32 rounding of the output (2^-24) and of the bias / residual adds."""
    B, H, W = 2, 6, 8
    x = grid16(B, H, W, Cin, scale=1.0, seed=41).double()
    w = grid16(Cout, Cin, 3, 3, scale=0.25, seed=42).double()
    b = torch.randn(Cout, generator=torch.Generator().manual_seed(43), dtype=torch.float64).float()
    res = torch.randn(B, Cout, H, W, generator=torch.Generator().manual_seed(44), dtype=torch.float64).float()
    xc = x.permute(0, 3, 1, 2).float().cuda().contiguous(memory_format=torch.channels_last)
    wp = lib.pack_conv3x3_f32(w.float().cuda())
    if kind == "tf32":
        out = lib.conv3x3_f32(xc, wp, b.cuda(), residual=res.cuda())
    else:
        out = lib.conv3x3_f16in(xc.half(), wp.half(), b.cuda(), residual=res.cuda())
    ref = (F.conv2d(x.permute(0, 3, 1, 2), w, None, padding=1) + b.double()[None, :, None, None]).float().double() \
        + res.double()
    report(f"conv fp32-out {kind} Cin={Cin} Cout={Cout}", rel_err(out.cpu(), ref), 2.0 ** -22)


def _attn_inputs(B, H, Nq, N0, N1, kind, seed):
    C = H * 64
    q = rnd16(B, Nq, C, seed=seed, device="cuda")
    k0, v0 = rnd16(B, N0, C, seed=seed + 1, device="cuda"), rnd16(B, N0, C, seed=seed + 2, device="cuda")
    if kind is None:
        return q, k0, v0, None, None, 0, None
    T = 3 if kind == "base" else 1
    kv1 = rnd16(T * B, N1, 2 * C, seed=seed + 3, device="cuda")
    base = torch.tensor([(T - 1) * B], dtype=torch.int32, device="cuda") if kind == "base" else None
    return q, k0, v0, kv1[..., :C], kv1[..., C:], (T - 1) * B, base


@pytest.mark.gpu
@pytest.mark.parametrize("name,B,H,Nq,N0,N1,kind", ATTN_CASES, ids=[c[0] for c in ATTN_CASES])
def test_attention_tile_edges(lib, name, B, H, Nq, N0, N1, kind):
    """Two-segment flash attention with N0 / N1 / Nq one off a 128-key tile, 1..5 K/V tiles in total, and a per-step K/V
    base that selects the last slice of a [T*B, N1, .] tensor."""
    q, k0, v0, k1, v1, sl, base = _attn_inputs(B, H, Nq, N0, N1, kind, seed=50 + N0 + N1)
    if k1 is None:
        out = lib.attention(q, k0, v0, heads=H)
        kk, vv = k0, v0
    else:
        out = lib.attention(q, k0, v0, k1, v1, kv1_off=0, heads=H, kv1_mod=B if base is not None else 0, kv1_base=base)
        kk = torch.cat([k0, k1[sl:sl + B]], 1)
        vv = torch.cat([v0, v1[sl:sl + B]], 1)
    errs = attn_errs(out, q, kk, vv, H, 64, 0.125)
    report(f"attention {name}", max(errs), TOL_ATTN)


@pytest.mark.gpu
@pytest.mark.parametrize("name,H,Nq,N0,N1,qkind,mutants", ZERO_KV_CASES, ids=[c[0] for c in ZERO_KV_CASES])
def test_attention_zero_kv_closed_form(lib, name, H, Nq, N0, N1, qkind, mutants):
    """CFG-uncond rows: N1 all-zero garment tokens in closed form. Cases with all-negative real scores (the max(m, 0)
    branch), N1 = 1, and scores so large that the zero tokens' weight underflows. The uncond sample sits beside a cond
    sample with real garment K/V (kv1_off = 1)."""
    q, k, v = (t.cuda() for t in zero_kv_inputs(qkind, H, Nq, N0, seed=70 + N0))
    C = H * 64
    gkv = rnd16(1, N1, 2 * C, seed=71, device="cuda")
    q2, k2, v2 = torch.cat([q, q]), torch.cat([k, k]), torch.cat([v, v])
    out = lib.attention(q2, k2, v2, gkv[..., :C], gkv[..., C:], kv1_off=1, heads=H)
    refs = zero_kv_ref(q, k, v, H, N1)
    errs = [rel_err(out[0, :, 64 * h:64 * h + 64], refs[h]) for h in range(H)]
    merrs = {}
    for m in mutants:
        mref = zero_kv_ref(q, k, v, H, N1, mutant=m)
        merrs[m] = min(rel_err(mref[h], refs[h]) for h in range(H))
    report(f"zero-K/V {name}", max(errs), TOL_ATTN, merrs)
    cond = attn_errs(out[1:], q, torch.cat([k, gkv[..., :C]], 1), torch.cat([v, gkv[..., C:]], 1), H, 64, 0.125)
    report(f"zero-K/V {name} (cond sample)", max(cond), TOL_ATTN)


@pytest.mark.gpu
def test_attention_exact_invariants(lib):
    """N0 = 1 without segment 1: softmax of one key is exactly 1, out == v bit for bit. Causal query row 0 sees key 0 only:
    out[:, 0] == v[:, 0]. Accumulate mode into a row-strided out (row stride > H*64) leaves the padding untouched."""
    H = 3
    C = H * 64
    q, k, v = rnd16(2, 300, C, seed=81, device="cuda"), rnd16(2, 1, C, seed=82, device="cuda"), rnd16(2, 1, C, seed=83,
                                                                                                       device="cuda")
    out = lib.attention(q, k, v, heads=H)
    assert torch.equal(out, v.expand(-1, 300, -1))
    for D in (64, 80):
        qq, kk, vv = (rnd16(2, 129, 2 * D, seed=84 + i, device="cuda") for i in range(3))
        oc = lib.encoder_attention(qq, kk, vv, 2, D, causal=True)
        assert torch.equal(oc[:, 0], vv[:, 0])
    k2, v2 = rnd16(2, 129, C, seed=87, device="cuda"), rnd16(2, 129, C, seed=88, device="cuda")
    big = rnd16(2, 300, C + 64, seed=89, device="cuda")
    before = big.clone()
    dst = big[..., :C]
    lib.attention(q, k2, v2, heads=H, accumulate=True, out=dst)
    assert torch.equal(big[..., C:], before[..., C:])
    errs = []
    for b in range(2):
        for h in range(H):
            c = slice(64 * h, 64 * h + 64)
            o = attn_head_ref(q[b, :, c], k2[b, :, c], v2[b, :, c], 0.125)
            ref = r16(before[b, :, c].double() + r16(o))
            errs.append(rel_err(big[b, :, c], ref))
    report("attention accumulate, strided out", max(errs), TOL_ATTN_IP)


@pytest.mark.gpu
@pytest.mark.parametrize("ip_scale", [0.0, 0.5, -1.0])
def test_cross_attention_ip_scale(lib, ip_scale):
    """Decoupled text + IP cross-attention at ip_scale 0 (bit-identical to the text-only result), 0.5 and -1."""
    B, H, N, Nt, Ni = 2, 3, 129, 77, 16
    C = H * 64
    q = rnd16(B, N, C, seed=91, device="cuda")
    kvt, kvi = rnd16(B, Nt, 2 * C, seed=92, device="cuda"), rnd16(B, Ni, 2 * C, seed=93, device="cuda")
    kt, vt, ki, vi = kvt[..., :C], kvt[..., C:], kvi[..., :C], kvi[..., C:]
    out = lib.cross_attention(q, kt, vt, ki, vi, heads=H, ip_scale=ip_scale)
    if ip_scale == 0.0:
        assert torch.equal(out, lib.cross_attention(q, kt, vt, heads=H))
    errs = []
    for b in range(B):
        for h in range(H):
            c = slice(64 * h, 64 * h + 64)
            ot = attn_head_ref(q[b, :, c], kt[b, :, c], vt[b, :, c], 0.125)
            oi = attn_head_ref(q[b, :, c], ki[b, :, c], vi[b, :, c], 0.125)
            errs.append(rel_err(out[b, :, c], ip_ref(ot, oi, ip_scale)))
    report(f"cross-attention ip_scale={ip_scale}", max(errs), TOL_ATTN_IP)


@pytest.mark.gpu
def test_cross_attention_rounding_of_text_output(lib):
    """Exact softmax (all scores 0) so that the rounding points alone decide: O_t must be rounded to fp16 before the IP
    term is added. Bit-identical to the restatement."""
    H, Nq, Nt, Ni = 2, 130, 12, 12
    q, kt, vt, ki, vi = (t.cuda() for t in ip_exact_inputs(H, Nq, Nt, Ni))
    out = lib.cross_attention(q, kt, vt, ki, vi, heads=H, ip_scale=-1.0)
    ot, oi = mean_attn(vt)[:, None], mean_attn(vi)[:, None]
    ref = ip_ref(ot, oi, -1.0).expand(1, Nq, -1)
    merr = rel_err(ip_ref(ot, oi, -1.0, mutant="ot_unrounded"), ref[:, :1])
    report("cross-attention O_t rounding", rel_err(out, ref), TOL_ATTN_IP, {"ot_unrounded": merr})


@pytest.mark.gpu
@pytest.mark.parametrize("D", ENC_DIMS)
@pytest.mark.parametrize("causal", [False, True])
def test_encoder_attention_head_dims(lib, D, causal):
    """CLIP-tower self-attention at every head width the ABI accepts, causal or not, N one off a 128-row tile; q/k/v are
    column blocks of a fused QKV buffer."""
    H = 2
    C = H * D
    errs = []
    for N in ENC_NS:
        qkv = rnd16(2, N, 3 * C, seed=100 + N + D, device="cuda")
        q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
        out = lib.encoder_attention(q, k, v, H, D, causal=causal)
        errs.append(max(attn_errs(out, q, k, v, H, D, D ** -0.5, causal=causal)))
    report(f"encoder attention D={D} causal={causal} (N {ENC_NS})", max(errs), TOL_ATTN)


GN_CASES = [  # (B, HW, C, offset in std units); (1, 3072, 320) parks its rows in shared memory, (4, 12288, 320) streams
    (1, 3072, 320, 50), (1, 3072, 320, 200), (1, 3072, 320, 1000),
    (4, 12288, 320, 50), (4, 12288, 320, 200), (4, 12288, 320, 1000),
]


def gn_offset_input(B, HW, C, offset):
    """fp16 [B, HW, C] with unit noise around a mean of `offset`: every channel's mean is offset + 0.01 * N(0, 1), so the
    spread between the channels of a group adds only ~1e-4 to the group's variance and mean / std stays ~offset."""
    g = torch.Generator().manual_seed(offset + HW)
    means = offset + 0.01 * torch.randn(C, generator=g, dtype=torch.float64)
    return (means + torch.randn(B, HW, C, generator=g, dtype=torch.float64)).half()


@pytest.mark.gpu
@pytest.mark.parametrize("B,HW,C,offset", GN_CASES)
def test_groupnorm_mean_offset(lib, B, HW, C, offset):
    """GroupNorm of fp16 activations whose group mean is far from zero relative to their spread (offset x std): the
    statistics must not lose the variance to cancellation."""
    x = gn_offset_input(B, HW, C, offset).cuda()
    gamma, beta = rnd16(C, seed=5, device="cuda"), rnd16(C, seed=6, device="cuda")
    out = lib.groupnorm(x, gamma, beta, 1e-5, False)
    report(f"groupnorm fp16 B={B} HW={HW} offset={offset}", rel_err(out, group_norm64(x, 32, gamma, beta, 1e-5)),
           TOL_NORM16)


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [50, 200, 1000])
def test_groupnorm_fp32_mean_offset(lib, offset):
    B, H, W, C = 2, 32, 24, 128
    g = torch.Generator().manual_seed(offset)
    x = (offset + torch.randn(B, C, H, W, generator=g, dtype=torch.float64)).float()
    gamma = torch.randn(C, generator=g, dtype=torch.float64).float()
    beta = torch.randn(C, generator=g, dtype=torch.float64).float()
    xc = x.cuda().contiguous(memory_format=torch.channels_last)
    out = lib.groupnorm_f32_nhwc(xc, gamma.cuda(), beta.cuda(), 1e-6, False)
    ref = F.group_norm(x.double(), 32, gamma.double(), beta.double(), 1e-6)
    report(f"groupnorm fp32 offset={offset}", rel_err(out.cpu(), ref), tol_norm32(offset))


@pytest.mark.gpu
def test_groupnorm_constant_group_and_single_pixel(lib):
    """A group whose values are all equal (variance 0, eps 1e-6: out = beta) and HW = 1 (one pixel per group)."""
    B, HW, C = 2, 64, 320
    x = rnd16(B, HW, C, seed=7, device="cuda")
    x[:, :, :10] = x[0, 0, 0]                              # group 0 of both samples constant
    gamma, beta = rnd16(C, seed=8, device="cuda"), rnd16(C, seed=9, device="cuda")
    out = lib.groupnorm(x, gamma, beta, 1e-6, True)
    ref = F.silu(group_norm64(x, 32, gamma, beta, 1e-6))
    report("groupnorm constant group", rel_err(out, ref), TOL_NORM16)
    assert torch.equal(out[:, :, :10], r16(F.silu(beta[:10].double())).half().expand(B, HW, -1))
    x1 = rnd16(3, 1, 640, seed=10, device="cuda") * 4
    g1, b1 = rnd16(640, seed=11, device="cuda"), rnd16(640, seed=12, device="cuda")
    report("groupnorm HW=1", rel_err(lib.groupnorm(x1, g1, b1, 1e-5, False), group_norm64(x1, 32, g1, b1, 1e-5)),
           TOL_NORM16)


@pytest.mark.gpu
@pytest.mark.parametrize("rows,C", [(33, 8), (17, 2048)])
def test_layernorm_narrow_wide_strided(lib, rows, C):
    """LayerNorm at C = 8 (one vector per row) and C = 2048 (the register limit), reading and writing row-strided views."""
    xb = rnd16(rows, C + 64, scale=3.0, seed=13, device="cuda") + 1
    x = xb[:, 32:32 + C]
    g, b = rnd16(C, seed=14, device="cuda"), rnd16(C, seed=15, device="cuda")
    ob = torch.zeros(rows, C + 16, dtype=torch.float16, device="cuda")
    lib.layernorm(x, g, b, 1e-5, out=ob[:, 8:8 + C])
    ref = F.layer_norm(x.double(), (C,), g.double(), b.double(), 1e-5)
    report(f"layernorm C={C}", rel_err(ob[:, 8:8 + C], ref), TOL_NORM16)
    assert ob[:, :8].abs().max().item() == 0 and ob[:, 8 + C:].abs().max().item() == 0


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 16])
def test_skinny_linear_add_embedding(lib, M):
    """skinny_linear at M = 1 / 16 with K = 2816 (add_embedding's input width), strided x / addend / out.
    fp32 dot products of 2816 terms: output rounding U16 plus accumulation (2^-13), as TOL_GEMM."""
    K, N = 2816, 1280
    xb = rnd16(M, K + 64, seed=16, device="cuda")
    x = xb[:, 64:]
    w, bias = rnd16(N, K, scale=K ** -0.5, seed=17, device="cuda"), rnd16(N, seed=18, device="cuda")
    ab = rnd16(M, N + 8, seed=19, device="cuda")
    add = ab[:, 8:]
    ob = torch.zeros(M, N + 16, dtype=torch.float16, device="cuda")
    lib.skinny_linear(x, w, bias, in_silu=True, out_silu=True, addend=add, out=ob[:, 16:])
    xs = r16(F.silu(x.double()))
    y = r16(F.silu(r16(xs @ w.double().t() + bias.double())))
    ref = r16(y + add.double())
    report(f"skinny_linear M={M}", rel_err(ob[:, 16:], ref), TOL_GEMM)
    assert ob[:, :16].abs().max().item() == 0


# ------------------------------------------------------------------------------------------------------------------
# CPU: the references are the ops they restate, and every mutant is at least 4x the tolerance away from them
# ------------------------------------------------------------------------------------------------------------------
def test_references_match_torch_float64():
    g = torch.Generator().manual_seed(0)
    q, k, v = (torch.randn(2, 3, 33, 48, generator=g, dtype=torch.float64) for _ in range(3))
    for causal in (False, True):
        ref = F.scaled_dot_product_attention(q, k, v, is_causal=causal, scale=0.3)
        mine = torch.stack([torch.stack([attn_head_ref(q[b, h], k[b, h], v[b, h], 0.3, causal=causal) for h in range(3)])
                            for b in range(2)])
        assert torch.allclose(mine, ref, rtol=1e-12, atol=1e-12)
    kz = torch.cat([k, torch.zeros(2, 3, 7, 48, dtype=torch.float64)], 2)
    vz = torch.cat([v, torch.zeros(2, 3, 7, 48, dtype=torch.float64)], 2)
    ref = F.scaled_dot_product_attention(q, kz, vz, scale=0.3)
    assert torch.allclose(attn_head_ref(q[1, 2], k[1, 2], v[1, 2], 0.3, n_zero=7), ref[1, 2], rtol=1e-12, atol=1e-12)
    x = torch.randn(2, 5, 7, 64, generator=g, dtype=torch.float64)
    w = torch.randn(32, 64, 3, 3, generator=g, dtype=torch.float64)
    assert torch.allclose(conv3x3_acc(x, w), F.conv2d(x.permute(0, 3, 1, 2), w, padding=1).permute(0, 2, 3, 1),
                          rtol=1e-12, atol=1e-12)
    xg = torch.randn(3, 40, 320, generator=g, dtype=torch.float64)
    gm, bt = torch.randn(320, generator=g, dtype=torch.float64), torch.randn(320, generator=g, dtype=torch.float64)
    ref = F.group_norm(xg.transpose(1, 2), 32, gm, bt, 1e-5).transpose(1, 2)
    assert torch.allclose(group_norm64(xg, 32, gm, bt, 1e-5), ref, rtol=1e-12, atol=1e-12)
    # two-pass float64 statistics directly
    xs = xg.view(3, 40, 32, 10)
    mu = xs.mean((1, 3), keepdim=True)
    var = ((xs - mu) ** 2).mean((1, 3), keepdim=True)
    direct = ((xs - mu) / torch.sqrt(var + 1e-5)).view(3, 40, 320) * gm + bt
    assert torch.allclose(direct, ref, rtol=1e-10, atol=1e-10)
    xl = torch.randn(5, 2048, generator=g, dtype=torch.float64)
    mu, var = xl.mean(-1, keepdim=True), xl.var(-1, unbiased=False, keepdim=True)
    assert torch.allclose(F.layer_norm(xl, (2048,), None, None, 1e-5), (xl - mu) / torch.sqrt(var + 1e-5), atol=1e-10)
    assert torch.allclose(gelu64(xl), F.gelu(xl), atol=1e-14) and torch.allclose(quick_gelu64(xl), xl * torch.sigmoid(1.702 * xl))


def grid_sums_exact(K):
    """Grid operands (a: scale 1, w: scale 1/4) accumulate exactly in fp32 at depth K: every product is a multiple of
    2^-8 of magnitude <= 1/4, so every partial sum, in any order, is a multiple of 2^-8 below K / 4, exact while
    K / 4 < 2^16 (fewer than 2^24 steps of 2^-8). One row reaches the largest sum the grid allows."""
    a = grid16(300, K, scale=1.0, seed=11)
    w = grid16(64, K, scale=0.25, seed=12)
    a[0], w[0] = 1.0, 0.25
    acc64 = a.double() @ w.double().t()
    assert torch.equal(acc64.float().double(), acc64)
    assert acc64.abs().max().item() == K / 4 < 2 ** 16
    assert torch.equal((acc64 * 256).round(), acc64 * 256)


def test_gemm_operands_on_the_grid_accumulate_exactly():
    """The premise of the bit-exact epilogue / convolution cases: grid operands' products and sums are exact in fp32."""
    grid_sums_exact(1152)


def test_grid_operands_exact_at_the_largest_full_size_k():
    """The same premise at 9 * 2560, the largest K a full-size step launches (conv1 of the first up-block resnets, after
    the 1280 + 1280 skip concat; tests/test_launch_inventory_gpu.py checks its inventory against it)."""
    grid_sums_exact(9 * 2560)


@pytest.mark.parametrize("name,M,N,K,rps,act,mutants", EPI_CASES, ids=[c[0] for c in EPI_CASES])
def test_gemm_epilogue_mutants_are_caught(name, M, N, K, rps, act, mutants):
    a, w, bias, rv, res = _epi_operands(name, M, N, K, rps, "cpu")
    actf = {"gelu": gelu64, "quick": quick_gelu64, None: None}[act]
    acc = a.double() @ w.double().t()
    ref = gemm_epilogue_ref(acc, bias, actf, rv, rps, res)
    # the restatement follows the header's formula literally
    v = r16(acc + bias.double())
    if actf is not None:
        v = r16(actf(v))
    if rv is not None:
        v = r16(v + rv.double()[torch.arange(M) // rps])
    assert torch.equal(ref, r16(v + res.double()))
    tol = TOL_EPI_ACT if act else 0.0
    for m in mutants:
        e = rel_err(gemm_epilogue_ref(acc, bias, actf, rv, rps, res, mutant=m), ref)
        assert e >= 4 * tol and e >= 4 * U16 / 8, (m, e)      # exact cases: at least an fp16 rounding step of the scale


@pytest.mark.parametrize("B,H,W,Cin,Cout,temb_off", [(2, 12, 8, 320, 16, 0), (3, 2, 1, 64, 64, 64)])
def test_conv_temb_mutant_is_caught(B, H, W, Cin, Cout, temb_off):
    x = grid16(B, H, W, Cin, scale=1.0, seed=21)
    w = grid16(Cout, Cin, 3, 3, scale=0.25, seed=22)
    bias = rnd16(Cout, seed=23)
    temb = rnd16(B, temb_off + Cout + 64, seed=24)[:, temb_off:temb_off + Cout]
    acc = conv3x3_acc(x, w)
    assert torch.equal(acc.float().double(), acc)
    ref = r16(r16(acc + bias.double()) + temb.double()[:, None, None, :])
    wrong = r16(r16(acc + bias.double()) + temb.double().roll(1, 0)[:, None, None, :])
    assert rel_err(wrong, ref) > 0.1


@pytest.mark.parametrize("name,H,Nq,N0,N1,qkind,mutants", ZERO_KV_CASES, ids=[c[0] for c in ZERO_KV_CASES])
def test_zero_kv_mutants_are_caught(name, H, Nq, N0, N1, qkind, mutants):
    q, k, v = zero_kv_inputs(qkind, H, Nq, N0, seed=70 + N0)
    s = torch.stack([q[0, :, 64 * h:64 * h + 64].double() @ k[0, :, 64 * h:64 * h + 64].double().t() * 0.125
                     for h in range(H)])
    if qkind in ("negative", "deep"):
        assert s.max().item() < -0.5 and s.min().item() > -6
        mass_real = torch.exp(s).sum(-1).mean().item()
        assert 0.2 < mass_real / N1 < 5                      # real and zero tokens carry comparable mass
    if qkind == "large":
        assert (s.max(-1).values > 88).all()                 # exp(-m) < 2^-126: the zero tokens' weight flushes to 0
    refs = zero_kv_ref(q, k, v, H, N1)
    for m in mutants:
        mrefs = zero_kv_ref(q, k, v, H, N1, mutant=m)
        e = min(rel_err(mrefs[h], refs[h]) for h in range(H))
        assert e >= 4 * TOL_ATTN, (m, e)


def test_ip_rounding_mutant_is_caught():
    q, kt, vt, ki, vi = ip_exact_inputs(2, 130, 12, 12)
    ot, oi = mean_attn(vt)[:, None], mean_attn(vi)[:, None]
    # the kernel's sums are exact: grid values, 12 terms
    assert torch.equal(vt.float().sum(1).double(), vt.double().sum(1))
    assert torch.equal(vi.float().sum(1).double(), vi.double().sum(1))
    ref = ip_ref(ot, oi, -1.0)
    e = rel_err(ip_ref(ot, oi, -1.0, mutant="ot_unrounded"), ref)
    assert e >= 4 * TOL_ATTN_IP, e


@pytest.mark.parametrize("B,HW,C,offset", GN_CASES)
def test_groupnorm_offset_inputs_reach_their_ratio(B, HW, C, offset):
    """The GroupNorm offset cases test what they are named after: every group's mean / std is within 5% of the offset
    (the fp16 rounding of values near 1000, ulp 0.5, adds ~1% to the std)."""
    x = gn_offset_input(B, HW, C, offset).double().view(B, HW, 32, C // 32)
    ratio = x.mean((1, 3)) / x.std((1, 3), unbiased=False)
    assert ((ratio / offset - 1).abs() < 0.05).all(), (ratio.min().item(), ratio.max().item())
