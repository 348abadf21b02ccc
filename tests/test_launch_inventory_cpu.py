"""The launch inventory (tests/test_launch_inventory_gpu.py) without a GPU: signatures and aliasing are captured as the
calls ran, the replay's operands reproduce the recorded strides, offsets and shared storage, and every mutant the GPU
replay gates against lies at least 4x the tolerance from the truth at representative recorded shapes."""
import importlib.util
import os
import types

import torch
import torch.nn.functional as F

from test_kernel_edges_gpu import TOL_ATTN, TOL_ATTN_IP, TOL_NORM16, attn_head_ref, group_norm64, ip_ref, rel_err
from test_schedule_cpu import COEF, cfg_rescale_ddpm_ref, kernel_inputs
from test_solvers_cpu import TOL

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("launch_inventory", os.path.join(ROOT, "tests", "helpers",
                                                                                  "launch_inventory.py"))
LI = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(LI)

# representative recorded shapes (SDXL width, 128x96 latents, B = 2 under CFG, hoisted K/V of 30 steps x 2 garments):
# (B, H, Nq, N0, N1, B1, kv1_off, kv1_mod, base)
ATTN_SHAPES = [(4, 2, 3072, 3072, 3072, 60, 2, 2, 0), (4, 2, 768, 768, 768, 60, 2, 2, 58), (2, 2, 3072, 3072, 3072, 1, 1,
                                                                                              0, 0)]
# (B, HW, C0, C1, eps): the up-block concats (straddling and not) and a transformer's GroupNorm
GN_SHAPES = [(1, 768, 1280, 640, 1e-5), (1, 3072, 640, 320, 1e-5), (1, 768, 1280, 1280, 1e-5), (1, 3072, 640, 0, 1e-6)]


def _fake_lib():
    """Wrappers with the parameter names and defaults of idm_vton_b200.lib that do nothing (the recorder only binds)."""
    def gemm(a, w, bias=None, residual=None, rowvec=None, rows_per_sample=0, geglu=False, gelu=False, out=None,
             force_bn=0, quick_gelu=False):
        return out

    def attention(q, k0, v0, k1=None, v1=None, n1=0, kv1_off=0, heads=None, scale=None, accumulate=False, out=None,
                  kv1_mod=0, kv1_base=None):
        return out
    return types.SimpleNamespace(gemm=gemm, attention=attention)


def test_signature_captures_views_aliasing_scalars_and_tables():
    mp = __import__("pytest").MonkeyPatch()
    L = _fake_lib()
    rec = LI.Recorder(L, mp)
    try:
        assert "gemm" not in rec.missing and "conv3x3" in rec.missing
        kv = torch.zeros(6, 10, 2 * 128, dtype=torch.float16)          # fused [K | V]: one storage
        q = torch.zeros(4, 7, 128, dtype=torch.float16)
        base = torch.tensor([4], dtype=torch.int32)
        L.attention(q, q, q, kv[..., :128], kv[..., 128:], kv1_off=2, heads=2, kv1_mod=2, kv1_base=base)
        L.attention(q, q, q, kv[..., :128], kv[..., 128:], kv1_off=2, heads=2, kv1_mod=2, kv1_base=base)
        big = torch.zeros(3000, 64 + 40, dtype=torch.float16)
        a = torch.zeros(3000, 64, dtype=torch.float16)
        w = torch.zeros(64, 64, dtype=torch.float16)
        L.gemm(a, w, residual=big[:, 8:72], out=big[:, 40:104], force_bn=128)
        base.fill_(2)
        L.attention(q, q, q, kv[..., :128], kv[..., 128:], kv1_off=2, heads=2, kv1_mod=2, kv1_base=base)
    finally:
        mp.undo()
    sigs = list(rec.sigs)
    assert len(sigs) == 3 and rec.sigs[sigs[0]] == 2                  # deduplicated; a new table value is a new one
    at = LI.args_of(sigs[0])
    assert at["q"][4] == at["k0"][4] == at["v0"][4] != at["k1"][4]     # q, k0, v0 one storage; k1 / v1 another
    assert at["k1"][4] == at["v1"][4] and at["v1"][5] - at["k1"][5] == 128
    assert at["k1"][2] == (10 * 256, 256, 1) and at["kv1_mod"] == 2 and at["kv1_off"] == 2 and at["heads"] == 2
    assert at["kv1_base"][6] == (4,) and LI.args_of(sigs[2])["kv1_base"][6] == (2,)
    g = LI.args_of(sigs[1])
    assert g["residual"][4] == g["out"][4] != g["a"][4]
    assert (g["residual"][5], g["out"][5]) == (8, 40) and g["out"][2] == (104, 1) and g["force_bn"] == 128


def test_offsets_rebase_to_an_aligned_base():
    mp = __import__("pytest").MonkeyPatch()
    L = _fake_lib()
    rec = LI.Recorder(L, mp)
    try:
        buf = torch.zeros(5000, 64, dtype=torch.float16)
        w = torch.zeros(64, 64, dtype=torch.float16)
        L.gemm(buf[40:80], w, out=buf[3000:3040])
        L.gemm(buf[40 + 16:80 + 16], w, out=buf[3000 + 16:3040 + 16])   # both moved by 16 rows (1024 elements)
        L.gemm(buf[41:81], w, out=buf[3001:3041])                         # moved by one row: another alignment
    finally:
        mp.undo()
    s1, s2 = list(rec.sigs)
    assert rec.sigs[s1] == 2
    a1, a2 = LI.args_of(s1), LI.args_of(s2)
    assert (a1["a"][5], a1["out"][5]) == (40 * 64 % 1024, 3000 * 64 - 40 * 64 // 1024 * 1024)
    assert a2["out"][5] - a2["a"][5] == a1["out"][5] - a1["a"][5]
    assert all(d[5] % 1024 == o % 1024 for d, o in ((a2["a"], 41 * 64), (a2["out"], 3001 * 64)))


def test_operands_reproduce_strides_offsets_and_sharing():
    mp = __import__("pytest").MonkeyPatch()
    L = _fake_lib()
    rec = LI.Recorder(L, mp)
    try:
        kv = torch.zeros(6, 10, 256, dtype=torch.float16)
        q = torch.zeros(2, 4, 7, 384, dtype=torch.float16)[1, :, :, 128:256]     # a view at an offset
        L.attention(q, q, q, kv[..., :128], kv[..., 128:], kv1_off=2, heads=2, kv1_mod=2,
                    kv1_base=torch.tensor([4], dtype=torch.int32))
    finally:
        mp.undo()
    sig = next(iter(rec.sigs))
    o = LI.build_operands(sig, "cpu")
    assert o["q"].shape == q.shape and o["q"].stride() == q.stride()
    assert o["q"].storage_offset() % 1024 == q.storage_offset() % 1024
    assert o["k1"].stride() == (2560, 256, 1) and o["v1"].storage_offset() - o["k1"].storage_offset() == 128
    assert o["q"].untyped_storage().data_ptr() == o["k0"].untyped_storage().data_ptr()
    o["v1"].fill_(3)
    assert o["k1"].abs().max() == 0                                     # disjoint columns of one buffer
    assert torch.equal(torch.as_strided(o["k1"], (6, 10, 256), (2560, 256, 1))[..., 128:], o["v1"])
    assert o["kv1_base"].tolist() == [4] and o["kv1_mod"] == 2 and o["heads"] == 2
    assert LI.seed_of(sig) == LI.seed_of(sig) and 0 <= LI.seed_of(sig) < 2 ** 31


def test_row_sample_covers_every_tile_and_both_warpgroups():
    M = 60 * 3072 + 5
    rows = LI.sample_rows(M)
    assert rows[-1] == M - 1 and len({r // 128 for r in rows}) == -(-M // 128)
    assert {r % 128 for r in rows[:-1]} == {0, 63, 64, 127}
    assert LI.sample_rows(300) == list(range(300))


def test_pick_bn_restatement():
    assert LI.pick_bn(1920, 3072, False, 0) in (64, 128, 160, 192, 256)
    assert LI.pick_bn(10240, 768, True, 256) == 256 and LI.pick_bn(640, 1, False, 1128) == 128
    assert LI.pick_bn(16, 3072, False, 0) == 64                          # conv_out's N = 16: one 64-wide tile


def _attn_inputs(B, H, Nq, N0, N1, B1, seed):
    g = torch.Generator().manual_seed(seed)
    C = 64 * H
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64).half()   # noqa: E731
    return r(B, Nq, C), r(B, N0, C), r(B, N0, C), r(B1, N1, C), r(B1, N1, C)


def test_attention_mutants_are_far_from_truth_at_recorded_shapes():
    for B, H, Nq, N0, N1, B1, off, mod, base in ATTN_SHAPES:
        q, k0, v0, k1, v1 = _attn_inputs(B, H, Nq, N0, N1, B1, seed=Nq + B1)
        truth = LI.seg1_rows(B, off, B1, mod, base)
        nb = LI.neighbour_rows(B, off, B1, truth, mod, base)
        assert truth[:off] == [None] * off and all(t is not None for t in truth[off:])
        qr = torch.tensor(LI.sample_rows(Nq))[:: max(1, len(LI.sample_rows(Nq)) // 64)]
        m_nb, m_drop, m_n1 = [], [], []
        for b in range(B):
            for h in range(H):
                c = slice(64 * h, 64 * h + 64)

                def ref(row, nz):
                    kk, vv = k0[b, :, c], v0[b, :, c]
                    if row is not None:
                        kk, vv = torch.cat([kk, k1[row, :, c]]), torch.cat([vv, v1[row, :, c]])
                    return attn_head_ref(q[b, qr, c], kk, vv, 0.125, n_zero=nz)
                t = ref(truth[b], N1 if truth[b] is None else 0)
                if nb[b] is not None:
                    m_nb.append(rel_err(ref(nb[b], 0), t))
                if truth[b] is None:
                    m_drop.append(rel_err(ref(None, 0), t))
                    m_n1.append(rel_err(ref(None, N1 - 1), t))
        assert min(m_drop) >= 4 * TOL_ATTN, min(m_drop)
        if B1 > 1:
            assert min(m_nb) >= 4 * TOL_ATTN, min(m_nb)
            assert all(r != t for r, t in zip(nb, truth) if r is not None)
        # one zero token among N1 >= 768 is below the gate: the GPU replay prints it and gates the mutants above
        assert max(m_n1) < TOL_ATTN


def test_seg1_rows_follow_the_header():
    assert LI.seg1_rows(4, 2, 60, 2, 58) == [None, None, 58, 59]
    assert LI.seg1_rows(4, 2, 6, 0, 0) == [None, None, 0, 1]
    assert LI.seg1_rows(5, 2, 90, rows=[33, -1, 10]) == [None, None, 33, None, 10]
    assert LI.neighbour_rows(4, 2, 60, [None, None, 58, 59], 2, 58) == [None, None, 0, 1]
    assert LI.neighbour_rows(3, 1, 90, [None, 33, 10], rows=[33, 10]) == [None, 34, 11]


def test_groupnorm_mutants_are_far_from_truth_at_recorded_shapes():
    for B, HW, C0, C1, eps in GN_SHAPES:
        x0 = LI.gn_offset_dev((B, HW, C0), 1, "cpu")
        x1 = LI.gn_offset_dev((B, HW, C1), 2, "cpu") if C1 else None
        g = torch.Generator().manual_seed(3)
        gamma = torch.randn(C0 + C1, generator=g, dtype=torch.float64).half()
        beta = torch.randn(C0 + C1, generator=g, dtype=torch.float64).half()
        x = torch.cat([x0, x1], -1) if C1 else x0
        xs = x.double().view(B, HW, 32, -1)
        ratio = xs.mean((1, 3)) / xs.std((1, 3), unbiased=False)
        assert (ratio > 50).all()                                         # the group mean is far from zero
        truth = F.silu(group_norm64(x, 32, gamma, beta, eps))
        e_eps = rel_err(F.silu(group_norm64(x, 32, gamma, beta, 0.0)), truth)
        assert e_eps >= 4 * TOL_NORM16, (C0, C1, e_eps)
        gs, straddle = LI.gn_groups(C0, C1)
        if C1:
            assert (straddle is not None) == (C0 % gs != 0)
        if C1 and C1 != C0:                                               # equal widths: the same layout
            xm = torch.cat([x0, LI.gn_x1_in_x0_layout(x1, C0)], -1)
            e_lay = rel_err(F.silu(group_norm64(xm, 32, gamma, beta, eps)), truth)
            assert e_lay >= 4 * TOL_NORM16, (C0, C1, e_lay)
    assert LI.gn_groups(1280, 640) == (60, 21) and LI.gn_groups(640, 320) == (30, 21)
    assert LI.gn_groups(1280, 1280)[1] is None and LI.gn_groups(320, 320)[1] is None


def test_ip_rounding_mutant_is_far_from_truth_at_recorded_shapes():
    for B, Nt, Ni, C in ((4, 77, 16, 640), (4, 77, 16, 1280)):
        vt, vi = LI.ip_cancel_values((B, Nt, C), (B, Ni, C), 11, "cpu")
        assert torch.equal(vt.float().sum(1).double(), vt.double().sum(1))
        assert torch.equal(vi.float().sum(1).double(), vi.double().sum(1))
        ot, oi = vt.double().mean(1, keepdim=True), vi.double().mean(1, keepdim=True)
        truth = ip_ref(ot, oi, 1.0)
        e = rel_err(ip_ref(ot, oi, 1.0, mutant="ot_unrounded"), truth)
        assert e >= 4 * TOL_ATTN_IP, e


def test_cfg_step_mutant_is_far_from_truth_at_recorded_shapes():
    for B, H, W, ldc in ((2, 128, 96, 16), (3, 128, 96, 16), (2, 33, 25, 16)):
        eps, lat, noise = kernel_inputs(B, H, W, ldc, True, seed=1)
        for b in range(B):
            u, t = eps[b:b + 1], eps[B + b:B + b + 1]
            truth = cfg_rescale_ddpm_ref(torch.cat([u, t]), lat[b:b + 1], noise[b:b + 1], COEF, 0.0)
            swapped = cfg_rescale_ddpm_ref(torch.cat([t, u]), lat[b:b + 1], noise[b:b + 1], COEF, 0.0)
            assert rel_err(swapped, truth) >= 4 * TOL


def test_timestep_arguments_are_formed_in_fp32():
    t = torch.tensor([999.0, 1024.0, 768.0])
    arg = LI.timestep_args(t, 320)
    assert arg.dtype == torch.float32 and arg.shape == (3, 160)
    freq = torch.exp(-torch.log(torch.tensor(10000.0, dtype=torch.float64)) * torch.arange(160) / 160)
    assert torch.allclose(arg.double(), t.double()[:, None] * freq[None], rtol=2 ** -19)                 # the fp32 exponent of up to 9.2: 2^-20
    assert torch.equal(LI.ulp16(torch.tensor([1.0, 0.75, 1e-6])), torch.tensor([2.0 ** -10, 2.0 ** -11, 2.0 ** -24],
                                                                             dtype=torch.float64))
