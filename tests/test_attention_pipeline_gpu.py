"""The structure of the warp-specialised flash-attention kernel (attn.cu) against float64 restatements.

The kernel streams K/V tiles of 128 keys through a 3-stage ring (D = 64), overlaps each consumer warpgroup's softmax with
its own P V and with the other warpgroup's MMAs, takes an unmasked softmax on full key tiles, schedules the samples that
read a segment 1 first, and runs the text + IP-token cross-attention in one launch. The cases put each of those at its
edges: K/V tile counts around the ring depth in each segment and across the segment boundary, Nq that leaves the second
consumer warpgroup a partial or empty half-tile, N0 / N1 on and one off a tile multiple, heavy-first ordering with a
shared garment (kv1_mod) and a per-step K/V base, and the one-launch cross-attention at Nt in {1, 77, 80} and
Ni in {0, 1, 16}.

Same conventions as test_kernel_edges_gpu.py: max|a - b| / max|b| per (sample, head), the tolerances derived there, and
where a plausible bug is small the mutant reference is built too and the kernel must be at least 4x closer to the truth.
The CPU tests at the end check, without a GPU, that every mutant lies at least 4x the tolerance from the truth."""
import math

import pytest
import torch

U16 = 2.0 ** -11
TOL_ATTN = 4 * U16        # output rounding + P rounded to fp16 + ex2.approx (derivation in test_kernel_edges_gpu.py)
TOL_ATTN_IP = 6 * U16     # one more U16 for the fp16 rounding of O_t and O_i of the decoupled cross-attention
SCALE = 0.125


def r16(x):
    return x.half().to(x.dtype)


def rel_err(a, b):
    a, b = a.double(), b.double()
    den = b.abs().max().item()
    err = (a - b).abs().max().item()
    return err / den if den > 0 else (0.0 if err == 0 else math.inf)


def rnd16(*shape, scale=1.0, seed=0, device="cpu"):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g, dtype=torch.float64) * scale).half().to(device)


def grid16(*shape, scale, seed, device="cpu", levels=8):
    g = torch.Generator(device="cpu").manual_seed(seed)
    k = torch.randint(-levels, levels + 1, shape, generator=g).double()
    return (k * (scale / levels)).half().to(device)


def head_ref(q, k, v, n_zero=0):
    """softmax(q k^T / 8) v of one (sample, head) in float64, with n_zero all-zero key/value tokens appended. The
    unmasked-last-tile mutant is this with the padding keys of the partial tiles as zero tokens: the TMA fills keys past
    the end of a segment with zeros, so a kernel that skipped the mask would weigh them exp(0 - m)."""
    q, k, v = q.double(), k.double(), v.double()
    s = q @ k.t() * SCALE
    if n_zero:
        s = torch.cat([s, s.new_zeros(s.shape[0], n_zero)], 1)
        v = torch.cat([v, v.new_zeros(n_zero, v.shape[1])], 0)
    return torch.softmax(s, -1) @ v


def pad(n):
    return (-n) % 128


def report(name, err, tol, mutant_errs=None):
    print(f"[pipeline] {name}: err {err:.3e} (tol {tol:.2e}) mutants {mutant_errs}")
    assert math.isfinite(err) and err <= tol, f"{name}: err {err:.3e} > tol {tol:.2e}"
    for mn, me in (mutant_errs or {}).items():
        assert err <= 0.25 * me, f"{name}: err {err:.3e} not below a quarter of mutant {mn} ({me:.3e})"


# (name, B, H, Nq, N0, N1): K/V tiles 1..6 in total around the 3-stage ring, split across the two segments
RING_CASES = [
    ("t2_full", 1, 2, 256, 256, 0),
    ("t3_full", 1, 2, 128, 384, 0),
    ("t4_full", 1, 2, 128, 512, 0),
    ("t4_off", 1, 2, 129, 385, 0),
    ("t3_seg_2_1", 2, 2, 128, 256, 128),
    ("t4_seg_1_3", 1, 2, 130, 128, 384),
    ("t4_seg_3_1_off", 1, 2, 128, 384, 129),
    ("t6_seg_3_3_off", 1, 2, 127, 257, 257),
    ("t5_seg_4_1_off", 1, 1, 128, 511, 1),
]
# (name, Nq): the second consumer warpgroup (rows 64..127 of a query tile) partial or empty
NQ_CASES = [("nq_64", 64), ("nq_65", 65), ("nq_100", 100), ("nq_192", 192), ("nq_200", 200)]
# N0 / N1 on and one off a tile multiple: the fast path vs the masked path of the last tile
MASK_CASES = [("n0_128", 128, 0), ("n0_129", 129, 0), ("n0_257_n1_128", 257, 128), ("n0_256_n1_129", 256, 129),
              ("n0_129_n1_129", 129, 129)]
CROSS_CASES = [(nt, ni) for nt in (1, 77, 80) for ni in (0, 1, 16)]


def seg_inputs(B, H, Nq, N0, N1, seed, device="cpu"):
    C = H * 64
    q = rnd16(B, Nq, C, seed=seed, device=device)
    k0, v0 = rnd16(B, N0, C, seed=seed + 1, device=device), rnd16(B, N0, C, seed=seed + 2, device=device)
    kv1 = rnd16(B, N1, 2 * C, seed=seed + 3, device=device) if N1 else None
    return q, k0, v0, kv1


def seg_refs(q, k0, v0, kv1, H, n_zero=0):
    """[(b, h, ref)] for q attending to [k0 ; kv1 of the same sample]."""
    C = H * 64
    out = []
    for b in range(q.shape[0]):
        kk, vv = k0[b], v0[b]
        if kv1 is not None:
            kk, vv = torch.cat([kk, kv1[b, :, :C]]), torch.cat([vv, kv1[b, :, C:]])
        for h in range(H):
            c = slice(64 * h, 64 * h + 64)
            out.append((b, h, head_ref(q[b, :, c], kk[:, c], vv[:, c], n_zero)))
    return out


def mask_mutant_errs(q, k0, v0, kv1, H, N0, N1):
    n = pad(N0) + (pad(N1) if N1 else 0)
    if n < 64:          # a few zero tokens among hundreds move the output less than 4 tolerances
        return {}
    truth = seg_refs(q, k0, v0, kv1, H)
    mut = seg_refs(q, k0, v0, kv1, H, n_zero=n)
    return {"unmasked_last_tile": min(rel_err(m[2], t[2]) for m, t in zip(mut, truth))}


def cross_inputs(B, H, Nq, Nt, Ni, seed, device="cpu"):
    C = H * 64
    q = rnd16(B, Nq, C, seed=seed, device=device)
    kvt = rnd16(B, Nt, 2 * C, seed=seed + 1, device=device)
    kvi = rnd16(B, Ni, 2 * C, seed=seed + 2, device=device) if Ni else None
    return q, kvt, kvi


def ip_exact_inputs(H, Nq, Nt, Ni, device="cpu"):
    """q = 0: every score is 0, the softmax is a plain mean that the kernel computes exactly (grid-valued V, fp32 sums),
    so only the fp16 rounding points decide. Each IP value row is fp16(mean of the text values) plus a small grid step and
    ip_scale = -1: the output nearly cancels, which magnifies the rounding of O_t (77 and 80 are not powers of two)."""
    C = H * 64
    q = torch.zeros(1, Nq, C, dtype=torch.float16, device=device)
    kt = rnd16(1, Nt, C, seed=161, device=device)
    ki = rnd16(1, Ni, C, seed=162, device=device)
    vt = grid16(1, Nt, C, scale=2.0, seed=163, device=device, levels=64)
    base = r16(vt.double().mean(1, keepdim=True))
    vi = (base + grid16(1, Ni, C, scale=1 / 256, seed=164, device=device, levels=1).double()).half()
    return q, kt, vt, ki, vi


def ip_ref(ot, oi, ip_scale, mutant=None):
    t = ot if mutant == "ot_unrounded" else r16(ot)
    return r16(t + r16(ip_scale * r16(oi)))


@pytest.fixture(scope="module")
def lib():
    from idm_vton_b200 import lib as L
    L.load()
    return L


def _run_seg(lib, q, k0, v0, kv1, H):
    C = H * 64
    if kv1 is None:
        return lib.attention(q, k0, v0, heads=H)
    return lib.attention(q, k0, v0, kv1[..., :C], kv1[..., C:], kv1_off=0, heads=H)


# ------------------------------------------------------------------------------------------------------------------
# GPU tests
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name,B,H,Nq,N0,N1", RING_CASES, ids=[c[0] for c in RING_CASES])
def test_kv_tiles_around_ring_depth(lib, name, B, H, Nq, N0, N1):
    q, k0, v0, kv1 = seg_inputs(B, H, Nq, N0, N1, seed=200 + N0 + N1, device="cuda")
    out = _run_seg(lib, q, k0, v0, kv1, H)
    errs = [rel_err(out[b, :, 64 * h:64 * h + 64], r) for b, h, r in seg_refs(q, k0, v0, kv1, H)]
    report(f"ring {name}", max(errs), TOL_ATTN, mask_mutant_errs(q, k0, v0, kv1, H, N0, N1))


@pytest.mark.gpu
@pytest.mark.parametrize("name,Nq", NQ_CASES, ids=[c[0] for c in NQ_CASES])
def test_partial_or_empty_consumer_half_tile(lib, name, Nq):
    B, H, N0, N1 = 2, 2, 256, 129
    q, k0, v0, kv1 = seg_inputs(B, H, Nq, N0, N1, seed=300 + Nq, device="cuda")
    C = H * 64
    out = torch.full((B, Nq, C + 64), 7.0, dtype=torch.float16, device="cuda")
    dst = out[..., :C]
    lib.attention(q, k0, v0, kv1[..., :C], kv1[..., C:], kv1_off=0, heads=H, out=dst)
    assert (out[..., C:] == 7.0).all()        # nothing stored past the head columns or the last query row
    errs = [rel_err(dst[b, :, 64 * h:64 * h + 64], r) for b, h, r in seg_refs(q, k0, v0, kv1, H)]
    report(f"half-tile {name}", max(errs), TOL_ATTN)


@pytest.mark.gpu
@pytest.mark.parametrize("name,N0,N1", MASK_CASES, ids=[c[0] for c in MASK_CASES])
def test_fast_and_masked_last_tile(lib, name, N0, N1):
    B, H, Nq = 1, 2, 130
    q, k0, v0, kv1 = seg_inputs(B, H, Nq, N0, N1, seed=400 + N0 + N1, device="cuda")
    out = _run_seg(lib, q, k0, v0, kv1, H)
    errs = [rel_err(out[b, :, 64 * h:64 * h + 64], r) for b, h, r in seg_refs(q, k0, v0, kv1, H)]
    report(f"mask {name}", max(errs), TOL_ATTN, mask_mutant_errs(q, k0, v0, kv1, H, N0, N1))


@pytest.mark.gpu
@pytest.mark.parametrize("kv1_mod,T", [(1, 3), (2, 3), (0, 1)])
def test_heavy_first_order_with_shared_garment_and_step_base(lib, kv1_mod, T):
    """B = 4 with kv1_off = 2: samples 0, 1 take the zero-K/V closed form, samples 2, 3 read segment 1 and run first.
    kv1_mod = 1 shares one garment, 2 gives each its own; the device base selects the last of T per-step slices."""
    B, H, Nq, N0, N1 = 4, 2, 200, 257, 256
    C = H * 64
    q, k0, v0, _ = seg_inputs(B, H, Nq, N0, 0, seed=500 + kv1_mod, device="cuda")
    G = kv1_mod if kv1_mod else B - 2
    kv1 = rnd16(T * G, N1, 2 * C, seed=510 + kv1_mod, device="cuda")
    base = torch.tensor([(T - 1) * G], dtype=torch.int32, device="cuda") if T > 1 else None
    out = lib.attention(q, k0, v0, kv1[..., :C], kv1[..., C:], kv1_off=2, heads=H, kv1_mod=kv1_mod, kv1_base=base)
    errs = []
    for b in range(B):
        for h in range(H):
            c = slice(64 * h, 64 * h + 64)
            if b < 2:
                ref = head_ref(q[b, :, c], k0[b, :, c], v0[b, :, c], n_zero=N1)
            else:
                g = (T - 1) * G + (b - 2) % G
                ref = head_ref(q[b, :, c], torch.cat([k0[b, :, c], kv1[g, :, c]]),
                               torch.cat([v0[b, :, c], kv1[g, :, C + 64 * h:C + 64 * h + 64]]))
            errs.append(rel_err(out[b, :, c], ref))
    report(f"heavy-first kv1_mod={kv1_mod} T={T}", max(errs), TOL_ATTN)


@pytest.mark.gpu
@pytest.mark.parametrize("Nt,Ni", CROSS_CASES)
def test_one_launch_cross_attention(lib, Nt, Ni):
    B, H, Nq = 2, 2, 193
    C = H * 64
    q, kvt, kvi = cross_inputs(B, H, Nq, Nt, Ni, seed=600 + Nt + Ni, device="cuda")
    kt, vt = kvt[..., :C], kvt[..., C:]
    ki, vi = (kvi[..., :C], kvi[..., C:]) if Ni else (None, None)
    n0 = lib.launch_count()
    out = lib.cross_attention(q, kt, vt, ki, vi, heads=H, ip_scale=0.5)
    assert lib.launch_count() - n0 == 1
    text = lib.cross_attention(q, kt, vt, heads=H)
    if Ni:
        assert torch.equal(lib.cross_attention(q, kt, vt, ki, vi, heads=H, ip_scale=0.0), text)
    errs = []
    for b in range(B):
        for h in range(H):
            c = slice(64 * h, 64 * h + 64)
            ot = head_ref(q[b, :, c], kt[b, :, c], vt[b, :, c])
            ref = ip_ref(ot, head_ref(q[b, :, c], ki[b, :, c], vi[b, :, c]), 0.5) if Ni else ot
            errs.append(rel_err(out[b, :, c], ref))
    report(f"cross Nt={Nt} Ni={Ni}", max(errs), TOL_ATTN_IP)


@pytest.mark.gpu
@pytest.mark.parametrize("Nt,Ni", [(77, 16), (80, 16), (80, 1)])
def test_one_launch_cross_attention_rounds_text_output(lib, Nt, Ni):
    """Exact softmax (all scores 0): O_t must be rounded to fp16 before the IP term is added."""
    H, Nq = 2, 130
    q, kt, vt, ki, vi = (t.cuda() for t in ip_exact_inputs(H, Nq, Nt, Ni))
    out = lib.cross_attention(q, kt, vt, ki, vi, heads=H, ip_scale=-1.0)
    ot, oi = vt.double().mean(1)[:, None], vi.double().mean(1)[:, None]
    ref = ip_ref(ot, oi, -1.0)
    merr = rel_err(ip_ref(ot, oi, -1.0, mutant="ot_unrounded"), ref)
    report(f"cross O_t rounding Nt={Nt} Ni={Ni}", rel_err(out, ref.expand(1, Nq, -1)), TOL_ATTN_IP,
           {"ot_unrounded": merr})


# ------------------------------------------------------------------------------------------------------------------
# CPU checks: every mutant the GPU tests use lies at least 4x the tolerance from the truth
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,B,H,Nq,N0,N1", RING_CASES, ids=[c[0] for c in RING_CASES])
def test_ring_mask_mutants_are_caught(name, B, H, Nq, N0, N1):
    q, k0, v0, kv1 = seg_inputs(B, H, Nq, N0, N1, seed=200 + N0 + N1)
    for m, e in mask_mutant_errs(q, k0, v0, kv1, H, N0, N1).items():
        assert e >= 4 * TOL_ATTN, (m, e)


@pytest.mark.parametrize("name,N0,N1", MASK_CASES, ids=[c[0] for c in MASK_CASES])
def test_mask_mutants_are_caught(name, N0, N1):
    q, k0, v0, kv1 = seg_inputs(1, 2, 130, N0, N1, seed=400 + N0 + N1)
    merrs = mask_mutant_errs(q, k0, v0, kv1, 2, N0, N1)
    if pad(N0) + (pad(N1) if N1 else 0) >= 64:
        assert merrs, name
    for m, e in merrs.items():
        assert e >= 4 * TOL_ATTN, (m, e)


@pytest.mark.parametrize("Nt,Ni", [(77, 16), (80, 16), (80, 1)])
def test_cross_rounding_mutant_is_caught(Nt, Ni):
    q, kt, vt, ki, vi = ip_exact_inputs(2, 130, Nt, Ni)
    # the kernel's sums are exact: grid values of at most 80 terms
    assert torch.equal(vt.float().sum(1).double(), vt.double().sum(1))
    assert torch.equal(vi.float().sum(1).double(), vi.double().sum(1))
    ot, oi = vt.double().mean(1)[:, None], vi.double().mean(1)[:, None]
    e = rel_err(ip_ref(ot, oi, -1.0, mutant="ot_unrounded"), ip_ref(ot, oi, -1.0))
    assert e >= 4 * TOL_ATTN_IP, e
