"""FP8 garment K/V without a GPU: the rule's exponent at its boundaries, the proof that the kernel's dequantization route
gives the rule's bits, the byte counts that size the pools and caches, the cache key, the precision switch, the refusals,
and the two C-ABI entry points (declared, exported, argument checks, refused by the binding when missing)."""
import ctypes
import importlib.util
import os
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ("b200vton_quantize_kv_e4m3", "b200vton_attention_kv8")


def _load_ref():
    spec = importlib.util.spec_from_file_location("kv8_ref", os.path.join(ROOT, "tests", "helpers", "kv8_ref.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


R = _load_ref()


# ------------------------------------------------------------------------------------------------------------------
# the rule
# ------------------------------------------------------------------------------------------------------------------
def test_exponent_at_its_boundaries():
    k = torch.arange(-24, 9)
    at = 448.0 * torch.exp2(k.to(torch.float32))
    assert torch.equal(R.exponents(at), k.to(torch.int32))                       # amax = 448 * 2^k: e = k
    above = torch.nextafter(at, torch.full_like(at, float("inf")))
    assert torch.equal(R.exponents(above[:-1]), (k[:-1] + 1).to(torch.int32))    # the next float up: e = k + 1
    assert R.exponents(torch.tensor([65504.0])).item() == 8                      # the largest fp16
    tiny = torch.tensor([2.0 ** -24, 2.0 ** -20, 448.0 * 2.0 ** -25])            # below 448 * 2^-24: clamped
    assert R.exponents(tiny).tolist() == [-24, -24, -24]
    assert R.exponents(torch.zeros(1)).item() == 0


def test_quantize_zero_groups_and_no_saturation():
    g = torch.Generator().manual_seed(0)
    H = 2
    scale = torch.exp2(torch.randint(-20, 15, (3, 5, 4, 1), generator=g).to(torch.float32))
    kv = (torch.randn(3, 5, 4, 64, generator=g) * scale).reshape(3, 5, 256).clamp(-65504, 65504).to(torch.float16)
    kv[1, 2, 64:128] = 0                                                         # one all-zero group
    kv[2, 0, :64] = 65504
    kv[2, 0, 5] = -65504
    kv[0, 1, 128:192] = torch.tensor(2.0 ** -24, dtype=torch.float16)           # fp16 subnormals
    q, e = R.quantize(kv, H)
    assert e.shape == (3, 2 * H, 5)
    assert e[1, 1, 2].item() == 0 and (q[1, 2, 64:128].to(torch.float32) == 0).all()
    assert e[2, 0, 0].item() == 8 and e[0, 2, 1].item() == -24
    qf = q.to(torch.float32)
    assert torch.isfinite(qf).all() and qf.abs().max().item() <= 448
    # every nonzero group's largest code lies in (224, 448] unless the exponent was clamped
    amax = qf.reshape(3, 5, 2 * H, 64).abs().amax(-1).permute(0, 2, 1)
    live = (amax > 0) & (e > -24)
    assert (amax[live] > 224).all()
    # error: at most half an e4m3 step of the top binade (16) in units of 2^e, plus the final fp16 rounding
    x = kv.to(torch.float32)
    back = R.dequantize(q, e).to(torch.float32)
    err = (back - x).abs()
    unit = torch.exp2(e.permute(0, 2, 1).to(torch.float32)).repeat_interleave(64, -1)
    ok = x.abs() < 63488
    assert (err[ok] <= 16 * unit[ok] + x[ok].abs() * 2.0 ** -11).all()
    # the format's one overflow: |x| >= 63488 = 248 * 2^8 rounds to the code 256 at e = 8, and 256 * 2^8 is above fp16
    assert torch.isinf(back[2, 0, :64]).all() and back[2, 0, 5].item() == float("-inf")


def test_dequantization_in_fp16_gives_the_rules_bits():
    """fp16_rn(float(q) * 2^e) == fp16(q) * fp16(2^e) rounded once (the kernel's cvt + mul.rn.f16x2), for all 256
    codes and every exponent: both factors are exact fp16 numbers and their product is exact in fp32."""
    codes = torch.arange(256, dtype=torch.uint8).view(torch.float8_e4m3fn)
    nan = torch.isnan(codes.to(torch.float32))
    assert nan.sum().item() == 2                                                 # 0x7f, 0xff: never produced
    for e in range(-24, 9):
        rule = (codes.to(torch.float32) * 2.0 ** e).to(torch.float16)
        route = codes.to(torch.float16) * torch.tensor(2.0 ** e, dtype=torch.float16)
        assert torch.tensor(2.0 ** e, dtype=torch.float16).item() == 2.0 ** e
        assert torch.equal(rule[~nan].view(torch.int16), route[~nan].view(torch.int16)), e


# ------------------------------------------------------------------------------------------------------------------
# bytes
# ------------------------------------------------------------------------------------------------------------------
class _Blk:
    def __init__(self, c):
        self.c, self.heads = c, c // 64


def _sdxl(fmt):
    return types.SimpleNamespace(ch=(320, 640, 1280), blocks=lambda: [_Blk(640)] * 10 + [_Blk(1280)] * 60,
                                 garment_kv_format=fmt)


def test_bytes_from_the_shapes():
    from idm_vton_b200.denoise import garment_kv_bytes_per_step
    page16 = 30 * garment_kv_bytes_per_step(_sdxl("fp16"), 128, 96)
    page8 = 30 * garment_kv_bytes_per_step(_sdxl("fp8"), 128, 96)
    assert page16 == 9_437_184_000 and page8 == 4_792_320_000
    assert garment_kv_bytes_per_step(_sdxl("fp16"), 128, 96, "fp8") * 30 == page8
    assert int(40e9) // page16 == 4 and int(40e9) // page8 == 8
    # config 4: 1024 x 1024 (latents 128 x 128), 50 steps, four garments
    assert 4 * 50 * garment_kv_bytes_per_step(_sdxl("fp16"), 128, 128) == 83_886_080_000
    assert 4 * 50 * garment_kv_bytes_per_step(_sdxl("fp8"), 128, 128) == 42_598_400_000
    # a ragged garment: the exponent rows are padded to 16 tokens
    blk = types.SimpleNamespace(ch=(64,), blocks=lambda: [_Blk(64)], garment_kv_format="fp8")
    assert garment_kv_bytes_per_step(blk, 3, 7) == 21 * 128 + 2 * 32


def test_storage_layout():
    from idm_vton_b200.lib import GarmentKV8
    kv = GarmentKV8.empty(6, 21, 128, "cpu")
    assert kv.q.dtype == torch.float8_e4m3fn and tuple(kv.q.shape) == (6, 21, 256)
    assert kv.e.dtype == torch.int8 and tuple(kv.e.shape) == (6, 4, 32) and kv.e.is_contiguous()
    part = kv.map(lambda t: t[2:4])
    assert isinstance(part, GarmentKV8) and part.q.shape[0] == 2 and part.e.shape[0] == 2


# ------------------------------------------------------------------------------------------------------------------
# the denoisers: cache key, refusals
# ------------------------------------------------------------------------------------------------------------------
def _engine(fmt, symbols=SYMBOLS + ("b200vton_cfg_ddpm_step_rows", "b200vton_attention_rows")):
    L = types.SimpleNamespace(has_symbol=lambda n: n in symbols)
    return types.SimpleNamespace(L=L, device=torch.device("cpu"), ch=(64, 128), garment_kv_format=fmt,
                                 blocks=lambda: [_Blk(128), _Blk(64)])


def test_cache_keys_differ_between_formats():
    from idm_vton_b200.denoise import GarmentKVCache, TryOnDenoiser, new_garment_kv
    from idm_vton_b200.scheduler import DDPMScheduler
    sch = DDPMScheduler()
    sch.set_timesteps(3)
    cache = GarmentKVCache(1 << 30)
    eng = _engine("fp16")
    den = TryOnDenoiser(eng, None, max_kv_bytes=1 << 30)
    den.Bg, den.hg, den.wg, den.guidance_scale, den.guidance_rescale = 1, 4, 4, 2.0, 0.0
    den.latents = den.x0_prev = None
    fills = []

    def precompute(win_start=0):
        fills.append(eng.garment_kv_format)
        den.gkv_all = [new_garment_kv(eng, 3, ng, b) for b, ng in zip(eng.blocks(), (4, 16))]
        den.win_start = 0
    den.precompute_garment = precompute
    den.set_step_tables(sch, sch.timesteps, garment_keys=["g"], cache=cache)
    den.set_step_tables(sch, sch.timesteps, garment_keys=["g"], cache=cache)      # hit
    eng.garment_kv_format = "fp8"
    den.gkv_all = None
    den.set_step_tables(sch, sch.timesteps, garment_keys=["g"], cache=cache)      # a miss: the format is in the key
    assert fills == ["fp16", "fp8"] and cache.hits == 1 and len(cache.entries) == 2
    (k16, e16), (k8, e8) = cache.entries.items()
    assert k16[0] == k8[0] == "g" and k16[1][-1] == "fp16" and k8[1][-1] == "fp8"
    assert e16[0][0].dtype == torch.float16 and e8[0][0].q.dtype == torch.float8_e4m3fn
    assert e8[1] == 3 * (4 * 256 + 4 * 16 + 16 * 128 + 2 * 16)   # q and e bytes of one garment, 3 steps
    den.gkv_all = None
    den.set_step_tables(sch, sch.timesteps, garment_keys=["g"], cache=cache)      # fp8 hit: copied into (q, e)
    assert fills == ["fp16", "fp8"] and cache.hits == 2
    assert den.gkv_all[0].q.dtype == torch.float8_e4m3fn and den.gkv_all[0].e.shape == (3, 4, 16)


def _prepare_args(B=1):
    z = torch.zeros
    return (z(B, 4, 8, 8), z(2 * B, 1, 8, 8), z(2 * B, 4, 8, 8), z(2 * B, 4, 8, 8), z(1, 4, 8, 8), z(2 * B, 77, 8),
            z(2 * B, 6), z(2 * B, 6), z(2 * B, 16, 8), z(1, 77, 8))


def test_fp8_refused_where_no_garment_kv_is_held():
    from idm_vton_b200.denoise import SlotDenoiser, TryOnDenoiser
    from idm_vton_b200.scheduler import DDPMScheduler
    sch = DDPMScheduler()
    sch.set_timesteps(3)
    with pytest.raises(NotImplementedError, match=r"'fp8' with TryOnDenoiser\(hoist_garment=False\)"):
        TryOnDenoiser(_engine("fp8"), None, hoist_garment=False).prepare(*_prepare_args())
    den = SlotDenoiser(_engine("fp8"), None, 2)
    with pytest.raises(NotImplementedError, match="'fp8' with continuous batching without a garment K/V pool"):
        den.configure(sch, sch.timesteps, 4, 4)
    for name in SYMBOLS:                                   # a library without the kernels: refused, naming the symbol
        eng = _engine("fp8", symbols=tuple(n for n in SYMBOLS if n != name) + ("b200vton_cfg_ddpm_step_rows",
                                                                                "b200vton_attention_rows"))
        with pytest.raises(NotImplementedError, match=name):
            SlotDenoiser(eng, None, 2, pages=2).configure(sch, sch.timesteps, 4, 4)
    pool = SlotDenoiser(_engine("fp8"), None, 2, pages=3)   # pool mode holds the pages as (q, e)
    pool.configure(sch, sch.timesteps, 4, 4)
    assert pool.pool[0].q.shape == (9, 4, 256) and pool.pool[0].e.shape == (9, 4, 16)
    assert pool.pool[1].q.shape == (9, 16, 128) and pool.pool[1].e.shape == (9, 2, 16)
    fp16 = SlotDenoiser(_engine("fp16"), None, 2, pages=3)
    fp16.configure(sch, sch.timesteps, 4, 4)
    assert fp16.pool[0].dtype == torch.float16


def _tryon_cfg():
    from idm_vton_b200 import unet as U
    return dict(U.SDXL_TRYON, block_out_channels=(64, 128, 256), num_heads=(1, 2, 4), transformer_layers_per_block=(1, 1, 1),
                cross_attention_dim=64, projection_class_embeddings_input_dim=64 + 6 * 256,
                resampler=dict(U.SDXL_TRYON["resampler"], dim=64, depth=1, heads=1, embedding_dim=64, output_dim=64))


def test_precision_switch_and_the_module_seam_refusal():
    from idm_vton_b200 import unet as U
    from idm_vton_b200.denoise import GarmentKVCache
    from idm_vton_b200.pipeline import StableDiffusionXLInpaintPipeline as P
    cfg = _tryon_cfg()
    ut = U.UNet2DConditionModel(cfg, U.random_state_dict(cfg, device="cpu"))
    assert ut.garment_kv_precision == "fp16"
    with pytest.raises(ValueError, match="garment K/V precision"):
        ut.set_garment_kv_precision("int8")
    eng = types.SimpleNamespace(garment_kv_format="fp16")
    ut._engine = eng
    vae = types.SimpleNamespace(config=types.SimpleNamespace(block_out_channels=(1, 2, 3, 4)))
    pipe = P(vae, None, None, None, None, ut, None, None)
    pipe.garment_cache = GarmentKVCache()
    pipe.garment_cache.put("g", [torch.zeros(4)])
    held = object()
    pipe._denoiser = held
    pipe.set_garment_kv_precision("fp16")                  # unchanged: the denoiser and the cache stay
    assert pipe._denoiser is held and pipe.garment_cache.bytes == 16
    pipe.set_garment_kv_precision("fp8")                   # the weights stay packed; held K/V and cache go
    assert ut._engine is eng and eng.garment_kv_format == "fp8" and ut.garment_kv_precision == "fp8"
    assert pipe._denoiser is None and pipe.garment_cache.bytes == 0 and not pipe.garment_cache.entries
    with pytest.raises(ValueError, match="garment K/V precision"):
        pipe.set_garment_kv_precision("bf16")
    z = torch.zeros
    with pytest.raises(NotImplementedError, match="'fp8' with the module forward's reference-format"):
        ut(z(2, 13, 8, 8), 1, z(2, 77, 64), added_cond_kwargs=dict(text_embeds=z(2, 64), time_ids=z(2, 6),
                                                                   image_embeds=z(2, 16, 64)),
           garment_features=[z(2, 64, 64)])


# ------------------------------------------------------------------------------------------------------------------
# the C ABI
# ------------------------------------------------------------------------------------------------------------------
def test_kv8_entry_points_declared_exported_and_validated():
    from test_fp8_cpu import _declared_args
    from idm_vton_b200 import build, lib
    header = open(os.path.join(ROOT, "include", "b200vton.h")).read()
    so = ctypes.CDLL(build.build())
    for name in SYMBOLS:
        assert hasattr(so, name) and lib.OPTIONAL_SIGNATURES[name] == _declared_args(header, name), name
    raw = lib.load()
    assert all(lib.has_symbol(n) for n in SYMBOLS)
    n0 = lib.launch_count()
    quant = raw.b200vton_quantize_kv_e4m3
    assert quant(16, 256, 40, 4, 12, 16, 256, 16, 16, None) == 1 and b"multiple of Ng" in raw.b200vton_last_error()
    assert quant(16, 250, 40, 4, 10, 16, 256, 16, 16, None) == 1 and b"ldx" in raw.b200vton_last_error()
    assert quant(16, 256, 40, 4, 10, 16, 256, 16, 8, None) == 1 and b"lde" in raw.b200vton_last_error()
    assert quant(16, 256, 40, 4, 10, None, 256, 16, 16, None) == 1 and b"null" in raw.b200vton_last_error()
    attn = raw.b200vton_attention_kv8

    def call(ldkv1=256, lde1=16, n1=4, b1=2, e1=64, off=1, rows=None, B=2):
        return attn(64, 128, 64, 64, 128, 64, 64, ldkv1, e1, lde1, 64, 128, B, 2, 4, 4, n1, b1, off, 0, None, rows,
                    0.125, 0, None)
    assert call(ldkv1=136) == 1 and b"ldkv1" in raw.b200vton_last_error()
    assert call(lde1=8) == 1 and b"lde1" in raw.b200vton_last_error()
    assert call(n1=20) == 1 and b"lde1" in raw.b200vton_last_error()
    assert call(e1=None) == 1 and b"null" in raw.b200vton_last_error()
    for kw in (dict(n1=0), dict(b1=0)):
        assert call(**kw) == 1 and b"bad sizes" in raw.b200vton_last_error(), kw
    for off in (-1, 2):
        assert call(off=off) == 1 and b"kv1_off" in raw.b200vton_last_error()
    assert call(rows=258) == 1 and b"aligned" in raw.b200vton_last_error()
    assert lib.launch_count() == n0


def test_library_without_the_kv8_entry_points_refuses_in_the_binding():
    from idm_vton_b200 import lib
    lib.load()
    present = set(lib._present)
    try:
        for name, call in (("b200vton_quantize_kv_e4m3", lambda: lib.quantize_kv_e4m3(None, None)),
                           ("b200vton_attention_kv8", lambda: lib.attention_kv8(None, None, None, None))):
            lib._present.discard(name)
            with pytest.raises(NotImplementedError, match=name):
                call()
    finally:
        lib._present.update(present)


def test_continuous_server_follows_a_precision_change_only_when_idle():
    from test_continuous_cpu import _req
    from test_continuous_pool_cpu import _pool_fake_server
    srv = _pool_fake_server(S=2, T=3, P=2)
    srv.pipe.unet.garment_kv_precision = "fp16"
    srv.submit(_req("A"))
    srv.step()
    first = srv.den
    srv.pipe.unet.garment_kv_precision = "fp8"
    srv.submit(_req("B"))
    with pytest.raises(RuntimeError, match="changed to 'fp8' while requests run in 'fp16'"):
        srv.run()
    srv.pipe.unet.garment_kv_precision = "fp16"
    srv.run()                                              # back to the configured format: B runs on the same pool
    assert srv.den is first and srv.stats["images"] == 2
    srv.pipe.unet.garment_kv_precision = "fp8"
    srv.submit(_req("C"))
    srv.step()                                             # idle at the change: a new denoiser and page table
    assert srv.den is not first and srv._kv_format == "fp8" and srv.page_of == {"C": 0}
