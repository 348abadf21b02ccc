"""FreeU without a GPU: the oracle against the reference's own modules with enable_freeu (tests/golden/freeu_ref.pt,
made by oracle/make_golden_freeu.py), the FFT filter against its closed form in float64, the distance of each kernel
mutant from the truth, the C-ABI declaration and argument checks, and the FreeU switches of the UNet modules, the
pipeline and ContinuousTryOnServer."""
import ast
import ctypes
import importlib.util
import os
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "freeu_ref.pt")


def load_cases():
    spec = importlib.util.spec_from_file_location("freeu_cases", os.path.join(ROOT, "tests", "helpers", "freeu_cases.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


FC = load_cases()


# ------------------------------------------------------------------------------------------------------------------
# the oracle, pinned to the reference
# ------------------------------------------------------------------------------------------------------------------
def test_oracle_freeu_matches_reference_unet_golden():
    """oracle/unet_ref.py with oracle/freeu_ref.enabled reproduces the reference try-on UNet with enable_freeu, for
    every case, at the tolerance of the tiny UNet golden (tests/test_cpu_host.py)."""
    from oracle import freeu_ref as FR
    from oracle import unet_ref as R
    from oracle.make_golden import synth_inputs
    g = torch.load(GOLDEN)
    u = g["unet"]
    cfg_t, cfg_g = R.tiny_config("tryon"), R.tiny_config("garment")
    sd_t, sd_g = R.make_state_dict(cfg_t, seed=11), R.make_state_dict(cfg_g, seed=22)
    x = synth_inputs(cfg_t, cfg_g, u["B"], u["h"], u["w"])
    with torch.no_grad():
        img = R.resampler_forward(sd_t, "encoder_hid_proj", cfg_t["resampler"], x["clip_tokens"])
        feats = R.unet_garment_forward(sd_g, cfg_g, x["cloth"], x["timestep"], x["text_embeds_cloth"])
        fc = [torch.cat([torch.zeros_like(d), d]) for d in feats]
        added = {"text_embeds": x["text_embeds"], "time_ids": x["time_ids"], "image_embeds": img}
        for name, ref in u["noise_pred"].items():
            freeu = None if name == "off" else tuple(g["cases"][name][k] for k in ("s1", "s2", "b1", "b2"))
            with FR.enabled(sd_t, cfg_t, freeu):
                eps = R.unet_tryon_forward(sd_t, cfg_t, x["sample"], x["timestep"], x["prompt_embeds"], added, fc)
            assert torch.allclose(eps, ref, atol=2e-3, rtol=2e-3), name
            if name not in ("off", "s1_zero"):
                # the case discriminates: FreeU moves the output far beyond the tolerance
                assert (ref - u["noise_pred"]["off"]).abs().max() > 50 * 2e-3, name
    assert R.resnet_block.__module__ == R.__name__          # the patch is gone after the `with`


def test_s1_zero_is_freeu_off():
    """The reference's truthiness rule: s1 = 0 switches FreeU off entirely (the golden's s1 = 0 output is the plain one)."""
    from idm_vton_b200.engine import active_freeu
    from oracle import freeu_ref as FR
    g = torch.load(GOLDEN)
    assert torch.equal(g["unet"]["noise_pred"]["s1_zero"], g["unet"]["noise_pred"]["off"])
    for f in ((0.0, 0.2, 1.3, 1.4), (0.9, 0.0, 1.3, 1.4), (0.9, 0.2, 0, 1.4), (0.9, 0.2, 1.3, 0.0), None,
              (None, 0.2, 1.3, 1.4)):
        assert not FR.is_on(f) and active_freeu(f) is None
    assert FR.is_on((0.9, 0.2, 1.3, 1.4)) and active_freeu((0.9, 0.2, 1.3, 1.4)) == (0.9, 0.2, 1.3, 1.4)
    assert active_freeu((-1.0, 0.5, 2.0, 1.0)) == (-1.0, 0.5, 2.0, 1.0)      # negative values are truthy


def test_oracle_loop_with_freeu_pinned_by_reference_pipeline():
    """oracle/loop_ref.denoise_loop with FreeU on the tensors and step noises the REFERENCE pipeline (enable_freeu at
    the SDXL values, config 1) handed to its loop reproduces that pipeline's latents at every step; without FreeU it
    does not."""
    from oracle import freeu_ref as FR
    from oracle import loop_ref as LR
    from oracle import unet_ref as R
    p = torch.load(GOLDEN)["pipeline"]
    cfg_t, cfg_g = R.tiny_config("tryon"), R.tiny_config("garment")
    sd_t = {k: v.half().float() for k, v in R.make_state_dict(cfg_t, seed=11).items()}
    sd_g = {k: v.half().float() for k, v in R.make_state_dict(cfg_g, seed=22).items()}
    steps = len(p["latents_per_step"])
    freeu = tuple(p["freeu"][k] for k in ("s1", "s2", "b1", "b2"))
    with torch.no_grad():
        for n in range(1, steps + 1):
            with FR.enabled(sd_t, cfg_t, freeu):
                lat = LR.denoise_loop(sd_t, cfg_t, sd_g, cfg_g, p["loop_inputs"], steps, guidance_scale=2.0,
                                      noises=p["noises"], max_steps=n)
            ref = p["latents_per_step"][n - 1]
            assert (lat - ref).abs().max().item() <= 1e-4 * max(1.0, ref.abs().max().item())
        off = LR.denoise_loop(sd_t, cfg_t, sd_g, cfg_g, p["loop_inputs"], steps, guidance_scale=2.0,
                              noises=p["noises"])
    assert (off - p["latents_per_step"][-1]).abs().max().item() > 100 * 1e-4


def test_reference_freeu_signatures_recorded_and_matched():
    """enable_freeu / disable_freeu have the reference's parameter lists, on the pipeline and on the try-on UNet."""
    from idm_vton_b200.unet import UNet2DConditionModel
    import inspect
    sig = torch.load(GOLDEN)["signatures"]
    tree = ast.parse(open(os.path.join(ROOT, "idm-vton_b200", "pipeline.py")).read())
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "StableDiffusionXLInpaintPipeline")
    mine = {f.name: [a.arg for a in f.args.args] for f in cls.body if isinstance(f, ast.FunctionDef)}
    for name, s in sig["pipeline"].items():
        assert mine[name] == s["args"] and not any(s["has_default"]), name
    for name, s in sig["unet"].items():
        assert list(inspect.signature(getattr(UNet2DConditionModel, name)).parameters) == s["args"], name


# ------------------------------------------------------------------------------------------------------------------
# the filter and the kernel's mutants
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,W", [(32, 24), (64, 48), (16, 16), (8, 4), (1, 1), (1, 5), (2, 3), (3, 5), (7, 2), (5, 1),
                                 (9, 7), (2, 1)])
def test_fft_filter_equals_closed_form_float64(H, W):
    """diffusers' FFT filter (oracle/freeu_ref, in float64) equals the closed form of 7 sums per plane; with its dtype
    rule (fp32 unless both sizes are powers of two) to fp32 round-off."""
    from oracle import freeu_ref as FR
    x = torch.randn(2, 3, H, W, generator=torch.Generator().manual_seed(H * 100 + W), dtype=torch.float64) + 1.0
    for s in (0.375, 0.0, 1.5):
        ref = FR.fourier_filter_closed(x, s)
        assert (FR.spectral_filter(x, 1, s) - ref).abs().max().item() < 1e-12
        ref_t = FC.truth(x.permute(0, 2, 3, 1), s).permute(0, 3, 1, 2)      # the tests' FFT statement of the truth
        assert (ref_t - ref).abs().max().item() < 1e-12
        y = FR.fourier_filter(x.float(), 1, s)
        assert y.dtype == torch.float32 and (y.double() - ref).abs().max().item() < 1e-5
    assert torch.equal(FR.fourier_filter_closed(x, 1.0), x)


@pytest.mark.parametrize("k", range(len(FC.SHAPES)), ids=[c[0] for c in FC.SHAPES])
def test_kernel_mutants_lie_outside_the_gate(k):
    """Each mutant of the GPU test lies at least 4x the kernel tolerance from the float64 truth on its inputs (where
    the mutant differs from the filter at all: +1 and -1 coincide on a plane of size 2 or 1)."""
    name, B, H, W, Ch, Cs = FC.SHAPES[k]
    hidden, skip = FC.make_inputs(B, H, W, Ch, Cs, seed=k)
    ref = FC.truth(skip, FC.S_VALUE)
    # the fp16 rounding of the output alone stays well inside the gate
    assert FC.rel(ref.half(), ref) < FC.TOL / 2
    for mname, fn in FC.SKIP_MUTANTS.items():
        d = FC.rel(fn(skip, FC.S_VALUE), ref)
        if FC.distinct(mname, H, W):
            assert d >= FC.MUTANT_FACTOR * FC.TOL, (mname, d)
        else:
            assert d < 1e-12, (mname, d)
    assert FC.rel(FC.hidden_mutant(hidden, FC.B_VALUE), FC.hidden_truth(hidden, FC.B_VALUE)) >= FC.MUTANT_FACTOR * FC.TOL


def test_hidden_rule_is_torch_half_times_float():
    """fp16(float(h) * b): what PyTorch computes for a half tensor times a Python float."""
    h = torch.randn(4096, generator=torch.Generator().manual_seed(0)).half() * 7
    for b in (1.3, 1.4, 0.7, 1.1):
        ref = (h.float() * torch.tensor(b, dtype=torch.float32)).half()
        assert torch.equal(h * b, ref)


# ------------------------------------------------------------------------------------------------------------------
# the C ABI
# ------------------------------------------------------------------------------------------------------------------
def test_freeu_entry_point_declared_exported_and_validated():
    from idm_vton_b200 import build, lib
    name = "b200vton_freeu_nhwc"
    header = open(os.path.join(ROOT, "include", "b200vton.h")).read()
    so = ctypes.CDLL(build.build())
    assert f"int {name}(" in header and hasattr(so, name) and name in lib.OPTIONAL_SIGNATURES
    raw = lib.load()
    assert lib.has_symbol(name)
    n0 = lib.launch_count()
    base = 1 << 20

    def call(hidden=base, Ch=64, skip=base + (1 << 16), out=base + (1 << 16), Cs=64, B=1, H=4, W=4):
        return raw.b200vton_freeu_nhwc(hidden, Ch, skip, out, Cs, B, H, W, 1.3, 0.2, None)
    for kw, msg in ((dict(hidden=None), b"required"), (dict(out=None), b"required"), (dict(Cs=12), b"multiples of 8"),
                    (dict(Ch=4), b"multiples of 8"), (dict(B=0), b"bad shape"), (dict(H=0), b"bad shape"),
                    (dict(W=-1), b"bad shape"), (dict(skip=base + 8, out=base + 8), b"aligned"),
                    (dict(hidden=base + (1 << 16) - 256), b"overlap"), (dict(out=base + (1 << 16) + 64), b"skip_out"),
                    (dict(H=1 << 16, W=1 << 16), b"too large")):
        assert call(**kw) == 1 and msg in raw.b200vton_last_error(), kw
    assert lib.launch_count() == n0


def test_library_without_the_freeu_entry_point_refuses_in_the_binding():
    from idm_vton_b200 import lib
    lib.load()
    present = set(lib._present)
    try:
        lib._present.discard("b200vton_freeu_nhwc")
        with pytest.raises(NotImplementedError, match="b200vton_freeu_nhwc"):
            lib.freeu(None, None, 1.3, 0.2)
    finally:
        lib._present.update(present)


# ------------------------------------------------------------------------------------------------------------------
# module, pipeline and server switches
# ------------------------------------------------------------------------------------------------------------------
def test_unet_and_pipeline_switches():
    from oracle import unet_ref as R
    from idm_vton_b200.pipeline import StableDiffusionXLInpaintPipeline as P
    from idm_vton_b200.unet import UNet2DConditionModel, UNet2DConditionModelGarment
    net = UNet2DConditionModel(R.tiny_config("tryon"), dtype=torch.float32)
    assert net.freeu is None
    net.enable_freeu(0.9, 0.2, 1.3, 1.4)
    assert net.freeu == (0.9, 0.2, 1.3, 1.4)
    eng = types.SimpleNamespace(freeu=None)
    net._engine = eng                                  # a packed engine follows the module without a re-pack
    net.enable_freeu(s1=0.5, s2=0.6, b1=1.1, b2=1.2)
    assert eng.freeu == (0.5, 0.6, 1.1, 1.2) and net._engine is eng
    net.disable_freeu()
    assert net.freeu is None and eng.freeu is None
    garment = UNet2DConditionModelGarment(R.tiny_config("garment"), dtype=torch.float32)
    with pytest.raises(NotImplementedError, match="garment"):
        garment.enable_freeu(0.9, 0.2, 1.3, 1.4)
    pipe = P.__new__(P)
    with pytest.raises(ValueError, match="must have `unet`"):
        pipe.enable_freeu(0.9, 0.2, 1.3, 1.4)
    pipe.unet = net
    pipe.enable_freeu(0.9, 0.2, 1.3, 1.4)
    assert net.freeu == (0.9, 0.2, 1.3, 1.4)
    pipe.disable_freeu()
    assert net.freeu is None


def test_denoiser_signature_carries_the_freeu_setting():
    """A captured step is re-captured when the try-on engine's FreeU setting changes (and only when it changes by
    the reference's rule: s1 = 0 is the same step as FreeU off)."""
    from idm_vton_b200.denoise import freeu_setting
    from idm_vton_b200.engine import UNetEngine
    eng = UNetEngine.__new__(UNetEngine)
    eng.kind, eng.freeu = "tryon", None
    assert freeu_setting(eng) is None
    eng.freeu = (0.0, 0.2, 1.3, 1.4)
    assert freeu_setting(eng) is None
    eng.freeu = (0.9, 0.2, 1.3, 1.4)
    assert freeu_setting(eng) == (0.9, 0.2, 1.3, 1.4)
    eng.kind = "garment"
    assert freeu_setting(eng) is None
    assert freeu_setting(types.SimpleNamespace()) is None
    import inspect
    from idm_vton_b200.denoise import _CapturedStep
    assert "freeu_setting(self.tryon)" in inspect.getsource(_CapturedStep._signature)


def test_continuous_server_refuses_a_freeu_change_in_flight():
    """ContinuousTryOnServer reads the FreeU setting at configure: a change with requests in slots raises, a change
    while idle re-configures at the next admission."""
    from idm_vton_b200.serving import ContinuousTryOnServer
    net = types.SimpleNamespace(freeu=None)
    srv = ContinuousTryOnServer.__new__(ContinuousTryOnServer)
    srv.pipe = types.SimpleNamespace(unet=net)
    srv.slots = [None, None]
    srv._configured, srv._freeu = True, None
    srv._check_freeu()
    assert srv._configured
    net.freeu = (0.0, 0.2, 1.3, 1.4)                  # off by the reference's rule: no change
    srv._check_freeu()
    assert srv._configured
    net.freeu = (0.9, 0.2, 1.3, 1.4)
    srv.slots[1] = dict(step=3)
    with pytest.raises(RuntimeError, match="FreeU"):
        srv._check_freeu()
    srv.slots[1] = None
    srv._check_freeu()
    assert not srv._configured
