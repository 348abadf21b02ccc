"""FP8 linears on the H100: the quantizing LayerNorm and the e4m3 GEMM against their restatement (tests/helpers/fp8_ref.py),
the SDXL-width engine in FP8 mode against the oracle, and the pipeline / server in FP8 mode.

Metrics: the GEMM gate is max|out - ref| / max|ref|; the row-relative error max_r max|out_r - ref_r| / max|ref_r| (each
token at its own scale) is recorded beside it and separates the mutants; the network uses the metric of
tests/test_fullsize_gpu.py, max|a - b| / max(1, max|b|). Measured values are printed (`FP8 {...}` lines, visible with
`pytest -s`)."""
import importlib.util
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("fp8_ref", os.path.join(ROOT, "tests", "helpers", "fp8_ref.py"))
Q = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(Q)

# One fp16 ulp of the output's scale per rounding point of the epilogue that an accumulation difference can carry a value
# across (fp16(v + bias); then fp16(. + residual), or GEGLU's fp16(h) * fp16(gelu(.)) product). Measured on an H100:
# <= 4.5e-4 with one rounding, <= 1.0e-3 with two, at every K from 640 to 5120 once each slab's partial sum is promoted to
# the fp32 accumulator; without the promotion the error grew with K to 4.5e-3 at K = 5120.
GEMM_TOL = 2.0 ** -10


def _record(**kw):
    print("FP8 " + json.dumps(kw))


def _row_err(out, ref):
    out, ref = out.double(), ref.double()
    return ((out - ref).abs().amax(dim=1) / ref.abs().amax(dim=1).clamp_min(1e-30)).max().item()


def _err(a, b):
    a, b = a.float(), b.float()
    return (a - b).abs().max().item() / max(1.0, b.abs().max().item())


# ------------------------------------------------------------------------------------------------
# quantizing LayerNorm
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [640, 1280])
@pytest.mark.parametrize("rows", [1, 37, 3072 + 5])
def test_layernorm_e4m3_is_layernorm_then_the_rule(C, rows):
    from idm_vton_b200 import lib as L
    g = torch.Generator(device="cuda").manual_seed(C + rows)
    ldx = C + 64                                                       # rows of a wider buffer: ldx != C
    buf = torch.randn(rows, ldx, generator=g, device="cuda") * 3
    buf *= 2.0 ** torch.randint(-8, 6, (rows, 1), generator=g, device="cuda")   # tokens of very different magnitudes
    x = buf.half()[:, :C]
    gamma = (1 + 0.1 * torch.randn(C, generator=g, device="cuda")).half()
    beta = (0.1 * torch.randn(C, generator=g, device="cuda")).half()
    ref16 = L.layernorm(x, gamma, beta)
    q, s, y16 = L.layernorm_e4m3(x, gamma, beta, fp16_out=True)
    assert torch.equal(y16, ref16)
    q_ref, s_ref = Q.quantize_rows(y16)
    assert torch.equal(q.float(), q_ref) and torch.equal(s, s_ref)
    q2, s2, none = L.layernorm_e4m3(x, gamma, beta)                    # without the fp16 output
    assert none is None and torch.equal(q2.view(torch.uint8), q.view(torch.uint8)) and torch.equal(s2, s)
    # a constant row without beta normalises to zeros: scale 1, q 0
    xc = torch.full((3, C), 0.75, dtype=torch.float16, device="cuda")
    qc, sc, yc = L.layernorm_e4m3(xc, gamma, None, fp16_out=True)
    assert (yc == 0).all() and (qc.float() == 0).all() and (sc == 1).all()


# ------------------------------------------------------------------------------------------------
# e4m3 GEMM
# ------------------------------------------------------------------------------------------------
def _operands(M, N, K, seed, geglu_bn=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = (torch.randn(M, K, generator=g, device="cuda") * 2.0 ** torch.randint(-6, 3, (M, 1), generator=g, device="cuda"))
    w = torch.randn(N, K, generator=g, device="cuda") * 2.0 ** torch.randint(-3, 3, (N, 1), generator=g, device="cuda")
    a, w = a.half(), (w / K ** 0.5).half()
    bias = (0.5 * torch.randn(N, generator=g, device="cuda")).half()
    if geglu_bn:
        from idm_vton_b200.engine import pack_geglu
        w, bias = pack_geglu(w, bias, geglu_bn)
    return a, w, bias


def _run(L, a, w, bias=None, residual=None, geglu=False, force_bn=0):
    q_a, s_a = Q.quantize_rows(a)
    q_w, s_w = Q.quantize_rows(w)
    out = L.gemm_e4m3(q_a.to(torch.float8_e4m3fn), s_a, q_w.to(torch.float8_e4m3fn), s_w, bias=bias, residual=residual,
                      geglu=geglu, force_bn=force_bn)
    ref = Q.epilogue(Q.scaled_acc(q_a, s_a, q_w, s_w), bias, residual, geglu_bn=force_bn if geglu else 0)
    return out, ref, (q_a, s_a, q_w, s_w)


GEMM_CASES = [  # (M, N, K, force_bn, geglu, residual)
    (300, 1920, 640, 64, False, True), (300, 1920, 640, 128, False, False), (1000, 1920, 1280, 160, False, True),
    (1000, 1920, 1280, 192, False, False), (777, 1920, 1280, 256, False, True), (129, 1920, 5120, 128, False, True),
    (4101, 3840, 5120, 256, False, False), (3072, 1280, 640, 0, False, True),
    (500, 2560, 640, 128, True, False), (3077, 10240, 1280, 256, True, False), (65, 5120, 640, 256, True, False),
]


@pytest.mark.parametrize("M,N,K,bn,geglu,res", GEMM_CASES)
def test_gemm_e4m3_against_float64_product(M, N, K, bn, geglu, res):
    from idm_vton_b200 import lib as L
    a, w, bias = _operands(M, N, K, seed=M + N + K + bn, geglu_bn=bn if geglu else 0)
    residual = None
    if res:
        residual = torch.randn(M, N, device="cuda").half()
    out, ref, _ = _run(L, a, w, bias, residual, geglu, bn)
    e_row = _row_err(out, ref)
    e = (out.double() - ref.double()).abs().max().item() / ref.double().abs().max().item()
    _record(case=f"gemm_e4m3 M={M} N={N} K={K} bn={bn} geglu={geglu} residual={res}", err=e, row_err=e_row)
    assert torch.isfinite(out.float()).all()
    roundings = 2 if (res or geglu) else 1
    assert e <= roundings * GEMM_TOL, f"error {e:.3e} > {roundings} x 2^-10"


def test_gemm_e4m3_is_4x_closer_to_the_rule_than_each_mutant():
    from idm_vton_b200 import lib as L
    from idm_vton_b200.engine import pack_geglu
    M, N, K = 1000, 1280, 1280
    a, w, bias = _operands(M, N, K, seed=5)
    out, truth, (q_a, s_a, q_w, s_w) = _run(L, a, w, bias)
    e_kernel = _row_err(out, truth)
    mut = {}
    qa_t, sa_t = Q.quantize_rows(a, per_tensor=True)
    mut["per-tensor scale"] = Q.epilogue(Q.scaled_acc(qa_t, sa_t, q_w, s_w), bias)
    qa_z, sa_z = Q.quantize_rows(a, rounding="rz")
    qw_z, sw_z = Q.quantize_rows(w, rounding="rz")
    mut["truncation"] = Q.epilogue(Q.scaled_acc(qa_z, sa_z, qw_z, sw_z), bias)
    mut["scale after bias"] = Q.epilogue(Q.scaled_acc(q_a, s_a, q_w, s_w, scale_after_bias=bias))
    errs = {k: _row_err(v, truth) for k, v in mut.items()}
    # GEGLU: the kernel on the packed weights against the mutant whose scales kept the unpacked row order
    wg, bg = _operands(M, 2 * N, K, seed=6)[1:]
    wp, bp = pack_geglu(wg, bg, 256)
    out_g, truth_g, (q_a, s_a, qp, sp) = _run(L, a, wp, bp, geglu=True, force_bn=256)
    e_kernel_g = _row_err(out_g, truth_g)
    _, s_unpacked = Q.quantize_rows(wg)
    errs["GEGLU scales not interleaved"] = _row_err(Q.epilogue(Q.scaled_acc(q_a, s_a, qp, s_unpacked), bp, geglu_bn=256),
                                                    truth_g)
    _record(case="mutants", kernel=e_kernel, kernel_geglu=e_kernel_g, **errs)
    for name, e in errs.items():
        k = e_kernel_g if name.startswith("GEGLU") else e_kernel
        assert e >= 4 * max(k, GEMM_TOL), f"mutant '{name}' {e:.2e} not 4x further than the kernel {k:.2e}"


# ------------------------------------------------------------------------------------------------
# SDXL width, full depth: the engine in FP8 mode against the oracle
# ------------------------------------------------------------------------------------------------
def test_fullsize_fp8_engine_vs_oracle():
    """B=2, 128x96 latents (config 2), t=967. Four evaluations: ref32 (oracle, fp32), ref16 (oracle under fp16 autocast),
    ref8_16 (ref16 with the quantized linears of tests/helpers/fp8_ref.py) and the engine in FP8 mode."""
    from oracle import unet_ref as R
    from idm_vton_b200 import unet as U
    from idm_vton_b200.engine import SDXL_GARMENT, SDXL_TRYON, UNetEngine
    from test_fullsize_gpu import _cast, _engine_step, _forward_inputs, _oracle_step
    prev = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        sd_t = U.random_state_dict(SDXL_TRYON, seed=11, device="cuda")
        sd_g = U.random_state_dict(SDXL_GARMENT, seed=22, device="cuda")
        B, h, w, t = 2, 128, 96, 967
        inp = _forward_inputs(SDXL_TRYON, SDXL_GARMENT, B, h, w, seed=9)
        env16 = dict(eng_t=UNetEngine(SDXL_TRYON, sd_t, "tryon"), eng_g=UNetEngine(SDXL_GARMENT, sd_g, "garment"))
        feats16, eps16_before = _engine_step(env16, inp, t, B, h, w)
        env8 = dict(eng_t=UNetEngine(SDXL_TRYON, sd_t, "tryon", fp8=True),
                    eng_g=UNetEngine(SDXL_GARMENT, sd_g, "garment", fp8=True))
        feats8, eps8 = _engine_step(env8, inp, t, B, h, w)
        _, eps16_after = _engine_step(env16, inp, t, B, h, w)
        torch.cuda.synchronize()
        assert torch.equal(eps16_before, eps16_after), "the fp16 engine changed beside an FP8 one"
        del env8, env16
        torch.cuda.empty_cache()
        with torch.no_grad():
            sd_t32 = {k: v.float() for k, v in sd_t.items()}
            sd_g32 = {k: v.float() for k, v in sd_g.items()}
            f32, e32 = _oracle_step(R, sd_t32, sd_g32, SDXL_TRYON, SDXL_GARMENT, inp, t)
            del sd_t32, sd_g32
            inp16 = _cast(inp, torch.float16)
            with torch.autocast("cuda", dtype=torch.float16):
                f16, e16 = _oracle_step(R, sd_t, sd_g, SDXL_TRYON, SDXL_GARMENT, inp16, t)
                with Q.quantized_linears(R):
                    f8, e8 = _oracle_step(R, sd_t, sd_g, SDXL_TRYON, SDXL_GARMENT, inp16, t)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev
    assert len(feats8) == 70 and torch.isfinite(eps8.float()).all() and torch.isfinite(e8.float()).all()
    eps = dict(eng8_vs_32=_err(eps8, e32), ref8_16_vs_32=_err(e8, e32), eng8_vs_ref8_16=_err(eps8, e8),
               ref16_vs_ref8_16=_err(e16, e8), ref16_vs_32=_err(e16, e32), eng16_vs_32=_err(eps16_before, e32))
    feats = dict(eng8_vs_32=max(_err(a, b) for a, b in zip(feats8, f32)),
                 ref8_16_vs_32=max(_err(a, b) for a, b in zip(f8, f32)),
                 eng8_vs_ref8_16=max(_err(a, b) for a, b in zip(feats8, f8)),
                 ref16_vs_ref8_16=max(_err(a, b) for a, b in zip(f16, f8)))
    _record(case=f"fullsize fp8 B={B} {h}x{w} t={t}", eps_absmax=e32.abs().max().item(), eps=eps, feats=feats)
    # An fp16-level difference between two evaluations re-rounds the e4m3 values it carries across a rounding boundary (a
    # step of 1/16 of the value), and 70 blocks compound it: on an H100 the engine and ref8_16 landed 6.51e-3 / 6.20e-3
    # from ref32 (6.66e-3 / 6.77e-3 with a quantizer one ulp off in its division), while ref16 is 1.0e-3 away. So
    # (i) takes a tenth of the FP8 effect as slack beside the 2.5e-4 of the fp16 gate, and (ii) a factor 3/4: measured
    # 0.67 (noise_pred) and 0.73 (garment features).
    # (i) the engine adds no error beyond the specified FP8 arithmetic
    for tag, d in (("noise_pred", eps), ("garment features", feats)):
        assert d["eng8_vs_32"] <= d["ref8_16_vs_32"] * 1.1 + 2.5e-4, f"{tag}: {d}"
    # (ii) the engine tracks the specified quantization, not merely some error of that size
    assert eps["eng8_vs_ref8_16"] <= 0.75 * eps["ref16_vs_ref8_16"], f"noise_pred: {eps}"


# ------------------------------------------------------------------------------------------------
# pipeline and server in FP8 mode (tiny config: transformer widths 128 and 256)
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tiny8():
    from oracle import unet_ref as R
    from idm_vton_b200 import unet as U
    cfg_t, cfg_g = R.tiny_config("tryon"), R.tiny_config("garment")
    sd_t, sd_g = R.make_state_dict(cfg_t, seed=11), R.make_state_dict(cfg_g, seed=22)
    net_t = U.UNet2DConditionModel(cfg_t, sd_t).to("cuda", torch.float16)
    net_g = U.UNet2DConditionModelGarment(cfg_g, sd_g).to("cuda", torch.float16)
    return dict(cfg_t=cfg_t, cfg_g=cfg_g, net_t=net_t, net_g=net_g)


def _call(pipe, inp, seed=42, use_graph=True):
    from oracle import make_golden_pipeline as MG
    pipe.use_cuda_graph = use_graph
    torch.manual_seed(1234)              # the VAE encode's sample draws from the global generator
    pipe(**MG.call_kwargs(inp, torch.Generator().manual_seed(seed)), output_type="latent")
    return pipe._last_latents.clone()


def test_pipeline_fp8_graph_eager_repeat_and_switch(tiny8):
    from oracle import make_golden_pipeline as MG
    from idm_vton_b200.denoise import GarmentKVCache
    from test_schedule_gpu import _make_pipe
    dev, f16 = "cuda", torch.float16
    inp = {k: (v.to(dev, f16) if k not in ("image", "mask_image") else v.to(dev))
           for k, v in MG.make_call_inputs(tiny8["cfg_t"]).items()}
    pipe = _make_pipe(tiny8)
    lat16 = _call(pipe, inp)
    eng16 = pipe.unet.engine()
    pipe.garment_cache = GarmentKVCache()
    pipe.garment_cache.put("g", [torch.zeros(8, device=dev)])
    pipe.set_linear_precision("fp8")
    assert pipe.garment_cache.bytes == 0 and pipe.garment_cache.get("g") is None
    pipe.garment_cache = None
    lat8 = _call(pipe, inp)
    eng8 = pipe.unet.engine()
    assert eng8 is not eng16 and eng8.fp8 and pipe.unet_encoder.engine().fp8
    assert pipe._denoiser.tryon is eng8 and all(b.fp8 is not None for b in eng8.blocks())
    assert torch.equal(_call(pipe, inp), lat8)                                   # same seed, same bits
    assert torch.equal(_call(pipe, inp, use_graph=False), lat8)                  # eager launches = graph replay
    d = _err(lat8, lat16)
    _record(case="tiny pipeline fp8 vs fp16 final latents", err=d)
    assert 0 < d < 5e-2
    pipe.set_linear_precision("fp16")
    assert not pipe.unet.engine().fp8
    assert torch.equal(_call(pipe, inp), lat16)                                  # back to the fp16 bits


def test_continuous_server_fp8_request_is_batch_invariant(tiny8):
    """Per-row scales: a request's final latents are the same bits alone and beside other requests."""
    from test_continuous_gpu import _drive, _request
    from oracle import make_golden_pipeline as MG
    from idm_vton_b200.serving import ContinuousTryOnServer
    from test_schedule_gpu import _make_pipe

    def server():
        p = _make_pipe(tiny8)
        p.set_linear_precision("fp8")
        return ContinuousTryOnServer(p, height=MG.H, width=MG.W, slots=3, num_inference_steps=4, guidance_scale=2.0,
                                     seed=7, output_type="pt")

    t = lambda: _request(tiny8, 40, "A")  # noqa: E731
    _, lat_a, _ = _drive(server(), [([t()], 0)])
    _, lat_b, _ = _drive(server(), [([_request(tiny8, 41, "B")], 2), ([_request(tiny8, 42, "C")], 1), ([t()], 0)])
    _, lat_d, _ = _drive(server(), [([_request(tiny8, 42, "C"), t(), _request(tiny8, 41, "B")], 0)])
    assert server().pipe.unet.engine().fp8
    assert torch.equal(lat_b[2], lat_a[0]) and torch.equal(lat_d[1], lat_a[0])
    assert not torch.equal(lat_b[0], lat_a[0])
    tiny8["net_t"].set_linear_precision("fp16")
    tiny8["net_g"].set_linear_precision("fp16")
