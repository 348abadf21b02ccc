"""FP8 linears without a GPU: the quantization rule on hand-built rows, the distance of each plausible mistake from the
rule, the engine's pack-time quantizer against the rule, the C-ABI declarations and argument checks, and the precision
switch of the UNets and the pipeline."""
import ctypes
import importlib.util
import os
import re
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def load_fp8_ref():
    spec = importlib.util.spec_from_file_location("fp8_ref", os.path.join(ROOT, "tests", "helpers", "fp8_ref.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


Q = load_fp8_ref()
KERNEL_TOL = 2.0 ** -10          # the GPU gate of gemm_e4m3 against the float64 product (tests/test_fp8_gpu.py)


def _row(values, amax=448.0):
    """An fp16 row whose largest magnitude is `amax` (so inv = 448 / amax), followed by `values`."""
    return torch.tensor([[amax] + list(values)], dtype=torch.float16)


def test_rule_rounds_to_nearest_even_at_ties():
    # amax = 448: inv = 1, so q is the e4m3 rounding of the value itself; the e4m3 step on [1, 2) is 1/8
    q, s = Q.quantize_rows(_row([1.0625, 1.1875, -1.0625, 1.07, 3.0]))
    assert s.item() == 1.0
    assert q[0].tolist() == [448.0, 1.0, 1.25, -1.0, 1.125, 3.0]


def test_rule_saturates_at_448_and_scales_rows_to_it():
    # every row's largest magnitude lands on +-448, including rows where amax * (448 / amax) rounds above 448 in fp32
    hits = 0
    for a in torch.arange(1.0, 64.0, 0.0625, dtype=torch.float16):
        y = torch.tensor([[-a.item(), 0.5]], dtype=torch.float16)
        inv = torch.tensor(448.0, dtype=torch.float32) / y.float().abs().max()
        hits += int((y.float().abs().max() * inv).item() > 448.0)
        q, s = Q.quantize_rows(y)
        assert q[0, 0].item() == -448.0 and torch.isfinite(q).all()
        assert s.item() == pytest.approx(a.item() / 448.0, rel=1e-7)
    assert hits > 0, "no row exercised the product above 448"


def test_rule_zero_rows_and_subnormals():
    q, s = Q.quantize_rows(torch.zeros(2, 8, dtype=torch.float16))
    assert (q == 0).all() and (s == 1).all()
    # e4m3 subnormals: multiples of 2^-9 below 2^-6; ties round to even
    q, _ = Q.quantize_rows(_row([3 * 2.0 ** -10, 2.0 ** -10, 5 * 2.0 ** -10, 2.0 ** -9, 2.0 ** -11, 7 * 2.0 ** -9]))
    assert q[0, 1:].tolist() == [2.0 ** -8, 0.0, 2.0 ** -8, 2.0 ** -9, 0.0, 7 * 2.0 ** -9]
    # a row is scaled to its own amax: the same values at 1/1000 of the magnitude quantize to the same codes
    y = torch.randn(1, 64).half()
    q1, s1 = Q.quantize_rows(y)
    q2, s2 = Q.quantize_rows((y.float() / 1024).half())
    assert torch.equal(q1, q2) and s2.item() == pytest.approx(s1.item() / 1024, rel=1e-6)


def test_truncation_mutant_is_round_toward_zero():
    q, _ = Q.quantize_rows(_row([1.0625, 1.1875, -1.24, 1.126]), rounding="rz")
    assert q[0].tolist() == [448.0, 1.0, 1.125, -1.125, 1.125]


def _synthetic(M=96, K=640, N=256, seed=0):
    """Rows of very different magnitudes (tokens) and weight rows of different magnitudes (channels)."""
    g = torch.Generator().manual_seed(seed)
    a = (torch.randn(M, K, generator=g) * 2.0 ** torch.randint(-6, 3, (M, 1), generator=g)).half()
    w = (torch.randn(N, K, generator=g) * 2.0 ** torch.randint(-3, 3, (N, 1), generator=g) / K ** 0.5).half()
    bias = (torch.randn(N, generator=g) * 0.5).half()
    return a, w, bias


def row_err(out, ref):
    """max over rows of max|out - ref| / max|ref| of the row: every token is checked at its own scale."""
    out, ref = out.double(), ref.double()
    return ((out - ref).abs().amax(dim=1) / ref.abs().amax(dim=1).clamp_min(1e-30)).max().item()


def test_each_mutant_lies_well_outside_the_kernel_tolerance():
    a, w, bias = _synthetic()
    q_a, s_a = Q.quantize_rows(a)
    q_w, s_w = Q.quantize_rows(w)
    truth = Q.epilogue(Q.scaled_acc(q_a, s_a, q_w, s_w), bias)
    errs = {}
    qa_t, sa_t = Q.quantize_rows(a, per_tensor=True)
    errs["per-tensor scale"] = row_err(Q.epilogue(Q.scaled_acc(qa_t, sa_t, q_w, s_w), bias), truth)
    qa_z, sa_z = Q.quantize_rows(a, rounding="rz")
    qw_z, sw_z = Q.quantize_rows(w, rounding="rz")
    errs["truncation"] = row_err(Q.epilogue(Q.scaled_acc(qa_z, sa_z, qw_z, sw_z), bias), truth)
    errs["scale after bias"] = row_err(Q.epilogue(Q.scaled_acc(q_a, s_a, q_w, s_w, scale_after_bias=bias)), truth)
    # GEGLU: rows packed [value bn/2 | gate bn/2] per tile; the mutant keeps the scales in the unpacked row order
    from idm_vton_b200.engine import pack_geglu
    bn = 128
    wp, bp = pack_geglu(w, bias, bn)
    qp, sp = Q.quantize_rows(wp)
    truth_g = Q.epilogue(Q.scaled_acc(q_a, s_a, qp, sp), bp, geglu_bn=bn)
    _, s_unpacked = Q.quantize_rows(w)
    errs["GEGLU scales not interleaved"] = row_err(Q.epilogue(Q.scaled_acc(q_a, s_a, qp, s_unpacked), bp, geglu_bn=bn),
                                                   truth_g)
    print("FP8 mutants (row-relative error from the rule):", {k: f"{v:.3e}" for k, v in errs.items()})
    for name, e in errs.items():
        assert e >= 4 * KERNEL_TOL, f"mutant '{name}' is only {e:.2e} from the rule"


def test_pack_time_quantizer_is_the_rule():
    from idm_vton_b200 import lib
    a, w, _ = _synthetic(M=8, K=256, N=64, seed=3)
    w[5] = 0
    q, s = lib.quantize_rows_e4m3(w)
    q_ref, s_ref = Q.quantize_rows(w)
    assert q.dtype == torch.float8_e4m3fn and torch.equal(q.float(), q_ref) and torch.equal(s, s_ref)


def test_geglu_weights_carry_their_own_scale_after_packing():
    """Packing permutes rows, so quantizing after pack_geglu gives the packed rows of the unpacked quantization."""
    from idm_vton_b200 import lib
    from idm_vton_b200.engine import pack_geglu
    _, w, bias = _synthetic(M=8, K=256, N=512, seed=4)
    wp, _ = pack_geglu(w, bias, 256)
    q, s = lib.quantize_rows_e4m3(wp)
    q0, s0 = lib.quantize_rows_e4m3(w)
    qp, _ = pack_geglu(q0.float(), None, 256)
    sp, _ = pack_geglu(s0[:, None], None, 256)
    assert torch.equal(q.float(), qp) and torch.equal(s, sp[:, 0])


_CTYPES = {"const void*": ctypes.c_void_p, "void*": ctypes.c_void_p, "int64_t": ctypes.c_int64, "int": ctypes.c_int,
           "float": ctypes.c_float}


def _declared_args(header, name):
    m = re.search(rf"int {name}\((.*?)\);", header, re.S)
    assert m, f"{name} not declared"
    out = []
    for arg in m.group(1).split(","):
        t = " ".join(arg.split()[:-1]).replace(" *", "*")
        out.append(_CTYPES[t])
    return out


def test_fp8_entry_points_match_the_header_and_check_arguments():
    from idm_vton_b200 import build, lib
    path = build.build()
    header = open(os.path.join(ROOT, "include", "b200vton.h")).read()
    for name in ("b200vton_gemm_e4m3", "b200vton_layernorm_e4m3"):
        assert lib.OPTIONAL_SIGNATURES[name] == _declared_args(header, name), name
        assert hasattr(ctypes.CDLL(path), name)
    l = lib.load()
    assert lib.has_symbol("b200vton_gemm_e4m3") and lib.has_symbol("b200vton_layernorm_e4m3")
    # argument checks run before any launch: an error code and a message, no CUDA work
    g = l.b200vton_gemm_e4m3
    assert g(None, 64, None, None, 64, None, None, 8, 16, 16, 64, None, None, 0, 0, 0, None) == 1
    assert b"multiple of 128" in l.b200vton_last_error()
    assert g(16, 136, 16, 16, 128, 16, 16, 8, 16, 16, 128, None, None, 0, 0, 0, None) == 1
    assert b"multiples of 16 bytes" in l.b200vton_last_error()
    assert g(16, 128, 16, 24, 128, 16, 16, 8, 16, 16, 128, None, None, 0, 0, 0, None) == 1
    assert b"aligned" in l.b200vton_last_error()
    assert g(16, 128, 16, 16, 128, 16, 16, 8, 16, 16, 128, None, None, 0, 2, 0, None) == 1
    assert b"flags" in l.b200vton_last_error()
    ln = l.b200vton_layernorm_e4m3
    assert ln(16, 640, 4, 640, None, None, 1e-5, None, 0, 16, 648, 16, None) == 1
    assert b"ldq" in l.b200vton_last_error()
    assert ln(16, 640, 4, 640, None, None, 1e-5, None, 0, None, 640, 16, None) == 1
    assert b"must not be null" in l.b200vton_last_error()


def test_fp8_mode_raises_at_pack_time_for_widths_that_are_not_multiples_of_128():
    from idm_vton_b200 import unet as U
    from idm_vton_b200.engine import SDXL_GARMENT, UNetEngine
    cfg = dict(SDXL_GARMENT, block_out_channels=(64, 192, 256), num_heads=(1, 3, 4), transformer_layers_per_block=(1, 1, 1),
               cross_attention_dim=64)
    sd = U.random_state_dict(cfg, seed=0, device="cpu")
    UNetEngine(cfg, sd, "garment", device="cpu")                      # fp16: any width the kernels take
    with pytest.raises(ValueError, match="multiple of 128"):
        UNetEngine(cfg, sd, "garment", device="cpu", fp8=True)
    cfg2 = dict(cfg, block_out_channels=(64, 128, 256), num_heads=(1, 2, 4))
    eng = UNetEngine(cfg2, U.random_state_dict(cfg2, seed=0, device="cpu"), "garment", device="cpu", fp8=True)
    blk = eng.blocks()[0]
    assert set(blk.fp8) == {"qkv", "q2", "ff1"}
    assert blk.fp8["ff1"][0].shape == blk.wff1.shape and blk.fp8["ff1"][0].dtype == torch.float8_e4m3fn


def test_precision_switch_repacks_and_empties_the_garment_cache():
    from idm_vton_b200 import unet as U
    from idm_vton_b200.denoise import GarmentKVCache
    from idm_vton_b200.pipeline import StableDiffusionXLInpaintPipeline as P
    cfg = dict(U.SDXL_GARMENT, block_out_channels=(64, 128, 256), num_heads=(1, 2, 4), transformer_layers_per_block=(1, 1, 1),
               cross_attention_dim=64)
    ug = U.UNet2DConditionModelGarment(cfg, U.random_state_dict(cfg, device="cpu"))
    ut = types.SimpleNamespace(calls=[], set_linear_precision=lambda p: ut.calls.append(p))
    vae = types.SimpleNamespace(config=types.SimpleNamespace(block_out_channels=(1, 2, 3, 4)))
    pipe = P(vae, None, None, None, None, ut, ug, None)
    assert ug.linear_precision == "fp16"
    pipe.garment_cache = GarmentKVCache()
    pipe.garment_cache.put("g", [torch.zeros(4)])
    sentinel = object()
    ug._engine = sentinel
    pipe.set_linear_precision("fp16")                 # unchanged precision keeps the packed engine
    assert ug._engine is sentinel
    pipe.set_linear_precision("fp8")
    assert ug.linear_precision == "fp8" and ug._engine is None and ut.calls == ["fp16", "fp8"]
    assert pipe.garment_cache.get("g") is None and pipe.garment_cache.bytes == 0
    with pytest.raises(ValueError, match="linear precision"):
        pipe.set_linear_precision("int8")
