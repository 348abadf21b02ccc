"""Image sizes that are multiples of 8 but not of 32, and a garment at a size of its own, without a GPU: the oracle loop
against the reference pipeline's own loop (golden tests/golden/pipeline_resolution_ref.pt, made by
oracle/make_golden_resolution.py), the nearest-resize index rule of b200vton_upsample_nearest_nhwc against
F.interpolate, the garment K/V budget, and the checks that run before any launch."""
import ctypes
import os
import types

import pytest
import torch
import torch.nn.functional as F

G = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(G, "pipeline_resolution_ref.pt"))


@pytest.fixture(scope="module")
def tiny():
    from oracle import unet_ref as R
    cfg_t, cfg_g = R.tiny_config("tryon"), R.tiny_config("garment")
    sd_t = {k: v.half().float() for k, v in R.make_state_dict(cfg_t, seed=11).items()}
    sd_g = {k: v.half().float() for k, v in R.make_state_dict(cfg_g, seed=22).items()}
    return dict(cfg_t=cfg_t, cfg_g=cfg_g, sd_t=sd_t, sd_g=sd_g)


def test_golden_cases(golden):
    from oracle import make_golden_resolution as MR
    assert set(golden["cases"]) == set(MR.CASES)
    for name, c in golden["cases"].items():
        (H, W), (Hc, Wc) = MR.CASES[name]
        assert tuple(c["person"]) == (H, W) and tuple(c["cloth"]) == (Hc, Wc)
        assert c["stored"]["latents"].shape[-2:] == (H // 8, W // 8)
        assert c["stored"]["cloth_latents"].shape[-2:] == (Hc // 8, Wc // 8)
        assert c["timesteps"].tolist() == [501, 1] and len(c["latents_per_step"]) == 2
    assert os.path.getsize(os.path.join(G, "pipeline_resolution_ref.pt")) < 1 << 20


@pytest.mark.parametrize("name", ["odd_both", "even_not_x4", "cloth_larger", "cloth_smaller"])
def test_oracle_loop_reproduces_reference_golden(golden, tiny, name):
    """resolution_ref.denoise_loop on the tensors the reference handed to its loop, with the reference's step noises,
    equals the reference's latents after every step."""
    from oracle import make_golden_resolution as MR
    from oracle import resolution_ref as RR
    c = golden["cases"][name]
    inp = MR.loop_inputs(c, MR.make_case_inputs(tiny["cfg_t"], name))
    with torch.no_grad():
        for n, ref in enumerate(c["latents_per_step"], start=1):
            lat = RR.denoise_loop(tiny["sd_t"], tiny["cfg_t"], tiny["sd_g"], tiny["cfg_g"], inp, golden["steps"],
                                  noises=c["noises"], max_steps=n)
            d = (lat - ref).abs().max().item()
            assert d <= 1e-4 * max(1.0, ref.abs().max().item()), (name, n, d)


def test_scale_two_upsampling_cannot_run_the_golden_sizes(golden, tiny):
    """The size rule is what the golden pins: the scale-2 oracle (unet_ref / loop_ref) cannot even concatenate its skips
    at these sizes, and at a size that is a multiple of 4 the resolution oracle equals it exactly."""
    from oracle import loop_ref as LR
    from oracle import make_golden_resolution as MR
    from oracle import resolution_ref as RR
    inp = MR.loop_inputs(golden["cases"]["even_not_x4"], MR.make_case_inputs(tiny["cfg_t"], "even_not_x4"))
    with torch.no_grad(), pytest.raises(RuntimeError, match="[Ss]izes of tensors must match"):
        LR.denoise_loop(tiny["sd_t"], tiny["cfg_t"], tiny["sd_g"], tiny["cfg_g"], inp, 2, noises=[None, None], max_steps=1)
    inp8 = LR.synth_loop_inputs(tiny["cfg_t"], tiny["cfg_g"], 1, 8, 12, seed=4)
    with torch.no_grad():
        a = LR.denoise_loop(tiny["sd_t"], tiny["cfg_t"], tiny["sd_g"], tiny["cfg_g"], inp8, 2, max_steps=1,
                            noises=[torch.zeros(1, 4, 8, 12)])
        b = RR.denoise_loop(tiny["sd_t"], tiny["cfg_t"], tiny["sd_g"], tiny["cfg_g"], inp8, 2, max_steps=1,
                            noises=[torch.zeros(1, 4, 8, 12)])
    assert torch.equal(a, b)


def test_nearest_index_rule_equals_interpolate():
    """The kernel's index rule, restated in Python, against F.interpolate(size=..., mode="nearest") for every
    (in, out) with in in 1..40 and out in 1..90."""
    from oracle.resolution_ref import nearest_index
    bad = []
    for n_in in range(1, 41):
        src = torch.arange(n_in, dtype=torch.float32).view(1, 1, n_in)
        for n_out in range(1, 91):
            want = F.interpolate(src, size=n_out, mode="nearest").view(-1).long().tolist()
            got = [nearest_index(d, n_in, n_out) for d in range(n_out)]
            if got != want:
                bad.append((n_in, n_out))
    assert not bad, bad[:10]
    # the 2-D resize is the same rule per axis
    x = torch.arange(7 * 5, dtype=torch.float32).view(1, 1, 7, 5)
    y = F.interpolate(x, size=(13, 11), mode="nearest")
    ref = torch.tensor([[x[0, 0, nearest_index(i, 7, 13), nearest_index(j, 5, 11)].item() for j in range(11)]
                        for i in range(13)])
    assert torch.equal(y[0, 0], ref)


def _denoiser(ch=(320, 640, 1280), layers=(1, 2, 10)):
    from idm_vton_b200.denoise import TryOnDenoiser
    blocks = [types.SimpleNamespace(c=c) for lvl, c in enumerate(ch) for _ in range(2 * layers[lvl] if lvl else 0)]
    blocks += [types.SimpleNamespace(c=ch[-1])] * layers[-1]
    blocks += [types.SimpleNamespace(c=c) for lvl, c in enumerate(ch) for _ in range(3 * layers[lvl] if lvl else 0)]
    den = TryOnDenoiser.__new__(TryOnDenoiser)
    den.tryon = types.SimpleNamespace(ch=ch, blocks=lambda: blocks)
    return den, blocks


def test_kv_bytes_per_step_follows_garment_size():
    den, blocks = _denoiser()
    assert len(blocks) == 70
    den.Bg, den.h, den.w = 2, 128, 96
    den.hg, den.wg = 128, 96
    same = den.kv_bytes_per_step()
    tokens = {640: 64 * 48, 1280: 32 * 24}
    assert same == sum(2 * tokens[b.c] * 2 * b.c * 2 for b in blocks)
    den.hg, den.wg = 33, 25                                # 17x13 and 9x7 tokens at the two attention levels
    tokens = {640: 17 * 13, 1280: 9 * 7}
    assert den.kv_bytes_per_step() == sum(2 * tokens[b.c] * 2 * b.c * 2 for b in blocks)
    den.h, den.w = 40, 30                                   # the person's size does not enter the garment K/V
    assert den.kv_bytes_per_step() == sum(2 * tokens[b.c] * 2 * b.c * 2 for b in blocks)


def test_prepare_rejects_person_inputs_of_another_size():
    """pose / mask / masked-image latents must have the latents' size (the reference's channel concat fails otherwise);
    the denoiser raises before it allocates or writes anything."""
    den, _ = _denoiser()
    den.L = None                      # any launch would fail on this
    den.device = torch.device("cpu")
    lat = torch.zeros(1, 4, 33, 25)
    ok = dict(mask=torch.zeros(2, 1, 33, 25), masked_image_latents=torch.zeros(2, 4, 33, 25),
              pose_latents=torch.zeros(2, 4, 33, 25))
    for name, bad in (("pose_latents", torch.zeros(2, 4, 32, 24)), ("mask", torch.zeros(2, 1, 33, 24)),
                      ("masked_image_latents", torch.zeros(2, 4, 34, 25))):
        kw = dict(ok, **{name: bad})
        with pytest.raises(ValueError, match=name):
            den._prepare(lat, kw["mask"], kw["masked_image_latents"], kw["pose_latents"], torch.zeros(1, 4, 32, 24),
                         torch.zeros(2, 77, 8), torch.zeros(2, 8), torch.zeros(2, 6), torch.zeros(2, 16, 8),
                         torch.zeros(1, 77, 8), 2.0, True, 0.0)
    assert not hasattr(den, "x_t") and not hasattr(den, "_key")


def test_scatter_bindings_refuse_a_destination_of_another_size():
    """The C ABI takes H and W from the source; the bindings compare them with dst before any launch."""
    from idm_vton_b200 import lib
    dst = torch.zeros(2, 33, 25, 64, dtype=torch.float16)
    scale = torch.ones(1)
    for src in (torch.zeros(1, 4, 32, 24, dtype=torch.float16), torch.zeros(1, 4, 33, 26, dtype=torch.float16),
                torch.zeros(1, 4, 34, 25, dtype=torch.float16)):
        with pytest.raises(ValueError, match="spatial size"):
            lib.nchw_to_nhwc(src, dst)
        with pytest.raises(ValueError, match="spatial size"):
            lib.nchw_to_nhwc_scaled(src, dst, scale)
    with pytest.raises(ValueError, match="do not fit"):
        lib.nchw_to_nhwc(torch.zeros(1, 4, 33, 25, dtype=torch.float16), dst, c_off=61)
    with pytest.raises(ValueError, match="contiguous"):
        lib.nchw_to_nhwc(torch.zeros(1, 25, 33, 4, dtype=torch.float16).permute(0, 3, 2, 1), dst)


class _ShapeBinding:
    """Stand-in for idm_vton_b200.lib that only propagates NHWC shapes and records the up path's resize calls."""

    def __init__(self, with_resize=True):
        self.calls = []
        if with_resize:
            self.upsample_nearest = lambda x, size: self._up("nearest", x, tuple(int(s) for s in size))

    def _up(self, kind, x, size):
        self.calls.append((kind, tuple(x.shape[1:3]), size))
        return torch.zeros(x.shape[0], size[0], size[1], x.shape[3])

    def upsample2x(self, x):
        return self._up("2x", x, (2 * x.shape[1], 2 * x.shape[2]))

    def conv3x3(self, x, w, bias=None, stride=1, **kw):
        B, H, W, _ = x.shape
        return torch.zeros(B, (H - 1) // stride + 1, (W - 1) // stride + 1, w.shape[1])

    def groupnorm(self, x0, gamma, beta, eps, silu, x1=None):
        assert x1 is None or x1.shape[1:3] == x0.shape[1:3], "skip and up-path sizes differ"
        return torch.zeros(*x0.shape[:-1], x0.shape[-1] + (0 if x1 is None else x1.shape[-1]))


def _shape_engine(L, ch=(64, 128, 256)):
    """A try-on UNetEngine with the SDXL block layout at tiny widths and no transformer stages."""
    from idm_vton_b200.engine import UNetEngine, _Resnet

    def res(cin, cout):
        r = _Resnet()
        r.cin, r.cout, r.temb_off = cin, cout, 0
        r.n1w = r.n1b = r.b1 = r.n2w = r.n2b = r.b2 = r.bsc = None
        r.w1, r.w2 = torch.zeros(9, cout, cin), torch.zeros(9, cout, cout)
        r.wsc = torch.zeros(cout, cin) if cin != cout else None
        return r

    eng = object.__new__(UNetEngine)
    eng.L, eng.cfg, eng.ch, eng.kind = L, {}, ch, "tryon"
    eng.w_in, eng.b_in = torch.zeros(9, ch[0], 64), None
    eng.down, prev = [], ch[0]
    for i, c in enumerate(ch):
        eng.down.append(dict(res=[res(prev, c), res(c, c)], attn=[],
                             down=(torch.zeros(9, c, c), None) if i < len(ch) - 1 else None))
        prev = c
    eng.mid_res, eng.mid_attn = [res(ch[-1], ch[-1])] * 2, None
    eng._t2d = lambda t, x, state: x
    rch, eng.up = list(reversed(ch)), []
    skip_c = [ch[0]] + [c for i, c in enumerate(ch) for _ in range(3 if i < len(ch) - 1 else 2)]
    for i, c in enumerate(rch):
        lvl = dict(res=[], attn=[], up=(torch.zeros(9, c, c), None) if i < len(ch) - 1 else None)
        for j in range(3):
            lvl["res"].append(res(prev + skip_c.pop(), c))
            prev = c
        eng.up.append(lvl)
    eng.no_w = eng.no_b = eng.b_out = None
    eng.w_out = torch.zeros(9, 16, ch[0])
    return eng


@pytest.mark.parametrize("h,w,want", [
    (18, 16, [("nearest", (5, 4), (9, 8)), ("nearest", (9, 8), (18, 16))]),
    (33, 25, [("nearest", (9, 7), (17, 13)), ("nearest", (17, 13), (33, 25))]),
    (30, 22, [("nearest", (8, 6), (15, 11)), ("nearest", (15, 11), (30, 22))]),
    (16, 12, [("2x", (4, 3), (8, 6)), ("2x", (8, 6), (16, 12))]),
])
def test_engine_up_path_resizes_to_the_skips(h, w, want):
    """The engine's launch sequence: at latent sizes that are not a multiple of 4 every upsampler resizes to the next
    skip's size with the nearest-resize kernel; at multiples of 4 it launches the scale-2 kernel, as before."""
    L = _ShapeBinding()
    eps = _shape_engine(L)._forward(torch.zeros(1, h, w, 64), torch.zeros(1, 4096), None, None, 0, None)
    assert L.calls == want and tuple(eps.shape) == (1, h, w, 16)


def test_engine_without_the_resize_kernel_refuses_before_any_launch():
    """A binding without the nearest-resize kernel still runs multiples of 4 and refuses other sizes up front."""
    L = _ShapeBinding(with_resize=False)
    eng = _shape_engine(L)
    eng._forward(torch.zeros(1, 16, 12, 64), torch.zeros(1, 4096), None, None, 0, None)
    assert [c[0] for c in L.calls] == ["2x", "2x"]
    L.calls.clear()
    L.conv3x3 = None                                   # any launch would fail
    with pytest.raises(NotImplementedError, match="b200vton_upsample_nearest_nhwc"):
        eng._forward(torch.zeros(1, 33, 25, 64), torch.zeros(1, 4096), None, None, 0, None)
    assert L.calls == []


def test_upsample_nearest_symbol_exported_and_validated():
    from idm_vton_b200 import build, lib
    so = ctypes.CDLL(build.build())
    assert hasattr(so, "b200vton_upsample_nearest_nhwc") and hasattr(so, "b200vton_upsample2x_nhwc")
    assert "b200vton_upsample_nearest_nhwc" in lib.SIGNATURES
    raw = lib.load()
    assert raw.b200vton_version() == lib.ABI_VERSION == 109
    n0 = lib.launch_count()
    # argument validation returns error 1 before any CUDA work
    assert raw.b200vton_upsample_nearest_nhwc(None, 1, 4, 4, 12, 8, 8, None, None) == 1
    assert b"bad shape" in raw.b200vton_last_error()
    assert raw.b200vton_upsample_nearest_nhwc(None, 1, 4, 4, 64, 0, 8, None, None) == 1
    assert raw.b200vton_upsample_nearest_nhwc(8, 1, 4, 4, 64, 8, 8, 16, None) == 1
    assert b"aligned" in raw.b200vton_last_error()
    assert raw.b200vton_upsample2x_nhwc(None, 1, 4, 4, 12, None, None) == 1
    assert lib.launch_count() == n0
