"""ctypes binding of libb200vton.so (include/b200vton.h) plus thin torch-tensor wrappers.

PyTorch is used for device memory and streams only: every wrapper passes `tensor.data_ptr()` and the current CUDA
stream to the C ABI. There is no fallback: if the library is missing or an op fails, a RuntimeError is raised.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200vton.so")

_c = ctypes
_vp, _i, _i64, _f = _c.c_void_p, _c.c_int, _c.c_int64, _c.c_float

# name -> argtypes; restype is int for every op. Mirrors include/b200vton.h one to one.
SIGNATURES = {
    "b200vton_gemm_f16": [_vp, _i64, _vp, _i64, _vp, _i64, _i, _i, _i, _vp, _vp, _i64, _vp, _i64, _i, _i, _i, _vp],
    "b200vton_conv3x3_nhwc": [_vp, _i64, _i, _i, _i, _i, _vp, _i, _vp, _vp, _i64, _vp, _i, _vp, _i, _vp, _vp, _vp, _i64,
                              _vp, _i64, _i, _i, _vp],
    "b200vton_attention": [_vp, _i64, _vp, _vp, _i64, _vp, _vp, _i64, _vp, _i64, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _f, _i,
                           _vp],
    "b200vton_cross_attention": [_vp, _i64, _vp, _vp, _i64, _i, _vp, _vp, _i64, _i, _vp, _i64, _i, _i, _i, _f, _f, _vp],
    "b200vton_encoder_attention": [_vp, _i64, _vp, _vp, _i64, _vp, _i64, _i, _i, _i, _i, _f, _i, _vp],
    "b200vton_patchify": [_vp, _i, _i, _i, _i, _i, _vp, _i, _vp],
    "b200vton_token_embedding": [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp],
    "b200vton_conv3x3_nhwc_f32": [_vp, _i, _i, _i, _i, _vp, _i, _vp, _vp, _vp, _vp],
    "b200vton_split_tf32": [_vp, _i64, _i, _i64, _f, _vp, _vp, _vp],
    "b200vton_softmax_split_tf32": [_vp, _i64, _i, _vp, _vp, _vp],
    "b200vton_groupnorm_nhwc_f32": [_vp, _i, _i, _i, _vp, _vp, _f, _i, _vp, _i64, _vp, _i, _vp],
    "b200vton_conv3x3_nhwc_f16in_f32": [_vp, _i, _i, _i, _i, _vp, _i, _vp, _vp, _vp, _vp],
    "b200vton_groupnorm": [_vp, _i, _vp, _i, _i, _i, _vp, _vp, _f, _i, _vp, _vp, _vp],
    "b200vton_layernorm": [_vp, _i64, _i, _i, _vp, _vp, _f, _vp, _i64, _vp],
    "b200vton_nchw_to_nhwc": [_vp, _i, _i, _i, _i, _vp, _i, _i, _i, _vp],
    "b200vton_nchw_to_nhwc_scaled": [_vp, _i, _i, _i, _i, _vp, _i, _i, _i, _vp, _vp],
    "b200vton_nhwc_to_nchw": [_vp, _i, _i, _i, _i, _i, _vp, _vp],
    "b200vton_upsample2x_nhwc": [_vp, _i, _i, _i, _i, _vp, _vp],
    "b200vton_upsample_nearest_nhwc": [_vp, _i, _i, _i, _i, _i, _i, _vp, _vp],
    "b200vton_im2col3x3_s2_nhwc": [_vp, _i, _i, _i, _i, _vp, _vp],
    "b200vton_timestep_embedding": [_vp, _i, _i, _i, _vp, _vp],
    "b200vton_skinny_linear": [_vp, _i, _i, _i, _vp, _i64, _i, _vp, _i, _i, _vp, _i, _vp, _i, _vp],
    "b200vton_cfg_ddpm_step": [_vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _i, _vp, _vp],
    "b200vton_cfg_rescale_ddpm_step": [_vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _i, _vp, _vp],
    "b200vton_cfg_solver_step": [_vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp],
    "b200vton_preprocess_inpaint": [_vp, _vp, _i, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp],
    "b200vton_postprocess_image": [_vp, _i, _i, _i, _i, _vp, _vp, _vp],
}

# Entry points bound only when the loaded library exports them (added without an ABI version change): the per-sample
# step kernels of the continuous-batching denoiser (per kind, and mixed-kind for sampling presets), the FP8 linears,
# the per-sample-row attention of its pool mode, the FP8 garment K/V (quantizer and attention) and the full-resolution
# photo kernels (resampler, paste-back and the garment's CLIP pixels) and FreeU.
# `has_symbol` tells whether a binding can use them.
OPTIONAL_SIGNATURES = {
    "b200vton_cfg_ddpm_step_rows": [_vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _i, _i, _vp, _vp],
    "b200vton_cfg_solver_step_rows": [_vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp],
    "b200vton_nchw_to_nhwc_scaled_rows": [_vp, _i, _i, _i, _i, _vp, _i, _i, _i, _vp, _vp],
    "b200vton_gemm_e4m3": [_vp, _i64, _vp, _vp, _i64, _vp, _vp, _i64, _i, _i, _i, _vp, _vp, _i64, _i, _i, _vp],
    "b200vton_layernorm_e4m3": [_vp, _i64, _i, _i, _vp, _vp, _f, _vp, _i64, _vp, _i64, _vp, _vp],
    "b200vton_attention_rows": [_vp, _i64, _vp, _vp, _i64, _vp, _vp, _i64, _vp, _i64, _i, _i, _i, _i, _i, _i, _i, _vp,
                                _f, _i, _vp],
    "b200vton_cfg_step_mixed_rows": [_vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _i, _vp, _i, _vp, _vp],
    "b200vton_quantize_kv_e4m3": [_vp, _i64, _i, _i, _i, _vp, _i64, _vp, _i64, _vp],
    "b200vton_attention_kv8": [_vp, _i64, _vp, _vp, _i64, _vp, _vp, _i64, _vp, _i64, _vp, _i64, _i, _i, _i, _i, _i, _i,
                               _i, _i, _vp, _vp, _f, _i, _vp],
    "b200vton_resample_u8": [_vp, _vp, _i, _vp, _i64, _vp, _i64, _vp],
    "b200vton_paste_u8": [_vp, _vp, _i, _vp],
    "b200vton_clip_pixels_u8": [_vp, _vp, _i, _vp, _vp, _vp],
    "b200vton_freeu_nhwc": [_vp, _i, _vp, _vp, _i, _i, _i, _i, _f, _f, _vp],
}
_present = set()

_lib = None
ABI_VERSION = 109      # must equal b200vton_version() of the loaded library (bumped with every SIGNATURES change)


def load(build_if_missing=True):
    """Load (building first if needed) libb200vton.so and declare every exported symbol. The build runs under an
    exclusive file lock (several ranks may import at once); a library whose sources changed and that cannot be rebuilt,
    or whose ABI version differs from this binding, raises instead of being called with a stale argument layout."""
    global _lib
    if _lib is not None:
        return _lib
    if build_if_missing:
        from . import build as _build
        if _build.needs_build():
            import fcntl
            os.makedirs(os.path.join(_HERE, "build"), exist_ok=True)
            with open(os.path.join(_HERE, "build", ".lock"), "w") as lock:
                fcntl.flock(lock, fcntl.LOCK_EX)
                try:
                    _build.build()          # re-checks the source hash under the lock
                finally:
                    fcntl.flock(lock, fcntl.LOCK_UN)
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: the CUDA extension must be built (python idm-vton_b200/build.py); "
                           "there is no CPU fallback")
    lib = ctypes.CDLL(LIB_PATH)
    lib.b200vton_version.restype = _i
    got = lib.b200vton_version()
    if got != ABI_VERSION:
        raise RuntimeError(f"{LIB_PATH} reports ABI version {got}, this binding expects {ABI_VERSION}: rebuild it "
                           "(python idm-vton_b200/build.py --force)")
    lib.b200vton_last_error.restype = _c.c_char_p
    lib.b200vton_launch_count.restype = _c.c_longlong
    lib.b200vton_set_option.argtypes = [_c.c_char_p, _i]
    lib.b200vton_set_option.restype = _i
    if os.environ.get("B200VTON_GEMM2", "1") == "0":
        lib.b200vton_set_option(b"gemm_2cta_auto", 0)
    if os.environ.get("B200VTON_CLUSTER4", "1") == "0":
        lib.b200vton_set_option(b"gemm_cluster4", 0)
    if os.environ.get("B200VTON_PDL", "0") == "1":
        lib.b200vton_set_option(b"programmatic_launch", 1)
        _options["programmatic_launch"] = 1
    if os.environ.get("B200VTON_ATTN2", "1") == "0":
        lib.b200vton_set_option(b"attention_pingpong", 0)
    for name, args in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.argtypes = args
        fn.restype = _i
    for name, args in OPTIONAL_SIGNATURES.items():
        fn = getattr(lib, name, None)
        if fn is not None:
            fn.argtypes = args
            fn.restype = _i
            _present.add(name)
    _lib = lib
    return lib


_options = {}


def set_option(name, value):
    _check(load().b200vton_set_option(name.encode(), int(value)), "b200vton_set_option")
    _options[name] = int(value)


def get_option(name, default=0):
    """Last value set through set_option / the B200VTON_* environment switches (the C library has no getter)."""
    return _options.get(name, default)


def launch_count():
    """Kernels launched (or captured) by libb200vton.so since load."""
    return int(load().b200vton_launch_count())


def has_symbol(name):
    """Whether the loaded library exports the optional entry point `name` (OPTIONAL_SIGNATURES)."""
    load()
    return name in _present


def _optional(name):
    if not has_symbol(name):
        raise NotImplementedError(f"{LIB_PATH} does not export {name}: rebuild it (python idm-vton_b200/build.py --force)")
    return getattr(_lib, name)


def _check(rc, name):
    if rc != 0:
        msg = _lib.b200vton_last_error().decode()
        raise RuntimeError(f"{name} failed (code {rc}): {msg}")


def _p(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _f16(t, name):
    if t is not None:
        if t.dtype != torch.float16 or not t.is_cuda:
            raise TypeError(f"{name} must be a CUDA fp16 tensor, got {t.dtype} on {t.device}")
    return t


# ------------------------------------------------------------------------------------------------
# op wrappers
# ------------------------------------------------------------------------------------------------
def gemm(a, w, bias=None, residual=None, rowvec=None, rows_per_sample=0, geglu=False, gelu=False, out=None, force_bn=0,
         quick_gelu=False):
    """out[M,N] = epi(a[M,K] @ w[N,K]^T). a / residual / out may be row-strided 2-D views (last dim contiguous)."""
    lib = load()
    _f16(a, "a"); _f16(w, "w")
    M, K = a.shape
    N = w.shape[0]
    assert w.shape[1] == K and a.stride(1) == 1 and w.stride(1) == 1
    n_out = N // 2 if geglu else N
    if out is None:
        out = torch.empty((M, n_out), dtype=torch.float16, device=a.device)
    assert out.shape == (M, n_out) and out.stride(1) == 1
    if residual is not None:
        assert residual.shape == (M, n_out) and residual.stride(1) == 1
    rc = lib.b200vton_gemm_f16(_p(a), a.stride(0), _p(w), w.stride(0), _p(out), out.stride(0), M, N, K, _p(bias),
                               _p(residual), residual.stride(0) if residual is not None else 0, _p(rowvec),
                               rowvec.stride(0) if rowvec is not None else 0, rows_per_sample,
                               int(geglu) | (2 if gelu else 0) | (4 if quick_gelu else 0), force_bn,
                               _stream())
    _check(rc, "b200vton_gemm_f16")
    return out


def conv3x3(x, w_packed, bias=None, temb=None, sc0=None, sc1=None, w_sc=None, bias_sc=None, residual=None, out=None,
            force_bn=0, stride=1):
    """x: [B,H,W,Cin] NHWC fp16 (contiguous); w_packed: [9,Cout,Cin]; returns [B,Ho,Wo,Cout] (stride 1 or 2, pad 1)."""
    lib = load()
    _f16(x, "x"); _f16(w_packed, "w_packed")
    B, H, W, Cin = x.shape
    assert x.is_contiguous() and w_packed.is_contiguous() and w_packed.shape[0] == 9 and w_packed.shape[2] == Cin
    Cout = w_packed.shape[1]
    if out is None:
        out = torch.empty((B, (H - 1) // stride + 1, (W - 1) // stride + 1, Cout), dtype=torch.float16, device=x.device)
    C0 = sc0.shape[-1] if sc0 is not None else 0
    C1 = sc1.shape[-1] if sc1 is not None else 0
    rc = lib.b200vton_conv3x3_nhwc(_p(x), Cin, B, H, W, Cin, _p(w_packed), Cout, _p(bias), _p(temb),
                                   temb.stride(0) if temb is not None else 0, _p(sc0), C0, _p(sc1), C1, _p(w_sc),
                                   _p(bias_sc), _p(residual), residual.shape[-1] if residual is not None else 0,
                                   _p(out), out.shape[-1], force_bn, stride, _stream())
    _check(rc, "b200vton_conv3x3_nhwc")
    return out


def attention(q, k0, v0, k1=None, v1=None, n1=0, kv1_off=0, heads=None, scale=None, accumulate=False, out=None,
              kv1_mod=0, kv1_base=None):
    """q: [B,Nq,*], k0/v0: [B,N0,*], k1/v1: [B1,N1,*] 3-D views with contiguous last dim (row strides may exceed
    heads*64, e.g. slices of a fused QKV buffer). n1 > 0 with k1 None => all-zero segment-1 tokens for every sample."""
    lib = load()
    B, Nq = q.shape[0], q.shape[1]
    N0 = k0.shape[1]
    H = heads
    assert q.stride(2) == 1 and k0.stride(2) == 1 and v0.stride(2) == 1
    assert q.stride(0) == Nq * q.stride(1) and k0.stride(0) == N0 * k0.stride(1) and v0.stride() == k0.stride()
    if scale is None:
        scale = 64 ** -0.5
    if out is None:
        out = torch.empty((B, Nq, H * 64), dtype=torch.float16, device=q.device)
    B1 = 0
    ld1 = 0
    if k1 is not None:
        B1, n1 = k1.shape[0], k1.shape[1]
        ld1 = k1.stride(1)
        assert k1.stride(2) == 1 and k1.stride(0) == n1 * ld1 and v1.stride() == k1.stride()
    rc = lib.b200vton_attention(_p(q), q.stride(1), _p(k0), _p(v0), k0.stride(1), _p(k1), _p(v1), ld1, _p(out),
                                out.stride(1), B, H, Nq, N0, n1, B1, kv1_off, kv1_mod, _p(kv1_base), float(scale),
                                int(accumulate), _stream())
    _check(rc, "b200vton_attention")
    return out


def attention_rows(q, k0, v0, k1, v1, kv1_rows, kv1_off=0, heads=None, scale=None, accumulate=False, out=None):
    """attention with one segment-1 row per sample: sample b >= kv1_off reads row kv1_rows[b - kv1_off] of k1/v1
    [B1,N1,*]; a negative row takes the zero-K/V closed form. kv1_rows: int32 CUDA tensor of B - kv1_off entries."""
    fn = _optional("b200vton_attention_rows")
    B, Nq = q.shape[0], q.shape[1]
    N0 = k0.shape[1]
    assert q.stride(2) == 1 and k0.stride(2) == 1 and v0.stride(2) == 1
    assert q.stride(0) == Nq * q.stride(1) and k0.stride(0) == N0 * k0.stride(1) and v0.stride() == k0.stride()
    B1, n1, ld1 = k1.shape[0], k1.shape[1], k1.stride(1)
    assert k1.stride(2) == 1 and k1.stride(0) == n1 * ld1 and v1.stride() == k1.stride()
    if kv1_rows.dtype != torch.int32 or not kv1_rows.is_cuda or not kv1_rows.is_contiguous() or \
            kv1_rows.numel() != B - kv1_off:
        raise ValueError(f"attention_rows: kv1_rows must be a contiguous CUDA int32 tensor of B - kv1_off = "
                         f"{B - kv1_off} entries, got {kv1_rows.dtype} {tuple(kv1_rows.shape)} on {kv1_rows.device}")
    if scale is None:
        scale = 64 ** -0.5
    if out is None:
        out = torch.empty((B, Nq, heads * 64), dtype=torch.float16, device=q.device)
    rc = fn(_p(q), q.stride(1), _p(k0), _p(v0), k0.stride(1), _p(k1), _p(v1), ld1, _p(out), out.stride(1), B, heads, Nq,
            N0, n1, B1, kv1_off, _p(kv1_rows), float(scale), int(accumulate), _stream())
    _check(rc, "b200vton_attention_rows")
    return out


KV8_GROUP = 64     # columns per exponent of the FP8 garment K/V (one head of K or of V)


class GarmentKV8(tuple):
    """Hoisted garment K/V in the FP8 format (include/b200vton.h, b200vton_quantize_kv_e4m3): (q, e) with q e4m3
    [rows, Ng, 2C] and e int8 [rows, 2H, Ng_pad] (Ng_pad = Ng rounded up to 16). Both have `rows` first, so a row range,
    a view or a copy of the pair applies to both (map)."""

    def __new__(cls, q, e):
        return super().__new__(cls, (q, e))

    q = property(lambda self: self[0])
    e = property(lambda self: self[1])

    @staticmethod
    def empty(rows, ng, c, device):
        """Storage for `rows` rows of Ng tokens and C channels (2C / 64 exponent groups per token)."""
        return GarmentKV8(torch.empty((rows, ng, 2 * c), dtype=E4M3, device=device),
                          torch.empty((rows, 2 * c // KV8_GROUP, -(-ng // 16) * 16), dtype=torch.int8, device=device))

    def map(self, fn):
        return GarmentKV8(fn(self[0]), fn(self[1]))


def quantize_kv_e4m3(x, out):
    """x: fp16 [rows, Ng, 2C] (contiguous last dim, rows and tokens may be strided as one [rows*Ng, 2C] matrix) ->
    out = GarmentKV8 of the same rows, by the rule of include/b200vton.h (bit-identical)."""
    fn = _optional("b200vton_quantize_kv_e4m3")
    _f16(x, "x")
    rows, ng, c2 = x.shape
    q, e = out
    if q.dtype != E4M3 or e.dtype != torch.int8 or tuple(q.shape) != (rows, ng, c2) or \
            tuple(e.shape[:2]) != (rows, c2 // KV8_GROUP) or e.shape[2] < ng or not e.is_contiguous():
        raise ValueError(f"quantize_kv_e4m3: out must be (e4m3 {(rows, ng, c2)}, contiguous int8 "
                         f"{(rows, c2 // KV8_GROUP)} x >= {ng}), got {q.dtype} {tuple(q.shape)}, {e.dtype} "
                         f"{tuple(e.shape)}")
    x2, q2 = x.reshape(rows * ng, c2), q.view(rows * ng, c2)     # a view: the kernel must write the caller's storage
    assert x2.stride(1) == 1 and q2.stride(1) == 1
    rc = fn(_p(x2), x2.stride(0), rows * ng, c2 // KV8_GROUP, ng, _p(q2), q2.stride(0), _p(e), e.shape[2], _stream())
    _check(rc, "b200vton_quantize_kv_e4m3")
    return out


def attention_kv8(q, k0, v0, kv1, kv1_off=0, heads=None, scale=None, accumulate=False, out=None, kv1_mod=0,
                  kv1_base=None, kv1_rows=None):
    """attention (or, with kv1_rows, attention_rows) with segment 1 = kv1, a GarmentKV8 of [B1, N1, 2C] garment K/V
    (K = columns [0, C), V = [C, 2C), C = heads * 64): the result of those calls on kv1 dequantized, bit for bit."""
    fn = _optional("b200vton_attention_kv8")
    B, Nq = q.shape[0], q.shape[1]
    N0 = k0.shape[1]
    H = heads
    C = H * 64
    assert q.stride(2) == 1 and k0.stride(2) == 1 and v0.stride(2) == 1
    assert q.stride(0) == Nq * q.stride(1) and k0.stride(0) == N0 * k0.stride(1) and v0.stride() == k0.stride()
    kq, e = kv1
    B1, n1 = kq.shape[0], kq.shape[1]
    if kq.dtype != E4M3 or kq.shape[2] != 2 * C or kq.stride(2) != 1 or kq.stride(0) != n1 * kq.stride(1):
        raise ValueError(f"attention_kv8: kv1.q must be e4m3 [B1, N1, {2 * C}] rows, got {kq.dtype} {tuple(kq.shape)}")
    if e.dtype != torch.int8 or tuple(e.shape[:2]) != (B1, 2 * H) or not e.is_contiguous():
        raise ValueError(f"attention_kv8: kv1.e must be contiguous int8 [{B1}, {2 * H}, Ng_pad], got {e.dtype} "
                         f"{tuple(e.shape)}")
    if kv1_rows is not None and (kv1_rows.dtype != torch.int32 or not kv1_rows.is_cuda or
                                 not kv1_rows.is_contiguous() or kv1_rows.numel() != B - kv1_off):
        raise ValueError(f"attention_kv8: kv1_rows must be a contiguous CUDA int32 tensor of B - kv1_off = "
                         f"{B - kv1_off} entries, got {kv1_rows.dtype} {tuple(kv1_rows.shape)} on {kv1_rows.device}")
    if scale is None:
        scale = 64 ** -0.5
    if out is None:
        out = torch.empty((B, Nq, C), dtype=torch.float16, device=q.device)
    rc = fn(_p(q), q.stride(1), _p(k0), _p(v0), k0.stride(1), _p(kq), _p(kq[..., C:]), kq.stride(1), _p(e), e.shape[2],
            _p(out), out.stride(1), B, H, Nq, N0, n1, B1, kv1_off, kv1_mod, _p(kv1_base), _p(kv1_rows), float(scale),
            int(accumulate), _stream())
    _check(rc, "b200vton_attention_kv8")
    return out


def encoder_attention(q, k, v, heads, head_dim, scale=None, causal=False, out=None):
    """CLIP-tower self-attention. q / k / v: [B,N,heads*head_dim] views with contiguous last dim (e.g. the three column
    blocks of a fused QKV buffer); head_dim 16..96, multiple of 16."""
    lib = load()
    _f16(q, "q"); _f16(k, "k"); _f16(v, "v")
    B, N = q.shape[0], q.shape[1]
    assert q.stride(2) == 1 and k.stride(2) == 1 and v.stride() == k.stride() and k.shape[:2] == (B, N)
    assert q.stride(0) == N * q.stride(1) and k.stride(0) == N * k.stride(1)
    if scale is None:
        scale = head_dim ** -0.5
    if out is None:
        out = torch.empty((B, N, heads * head_dim), dtype=torch.float16, device=q.device)
    rc = lib.b200vton_encoder_attention(_p(q), q.stride(1), _p(k), _p(v), k.stride(1), _p(out), out.stride(1), B, heads, N,
                                        head_dim, float(scale), int(causal), _stream())
    _check(rc, "b200vton_encoder_attention")
    return out


def patchify(x, patch, ldk):
    """x: [B,C,H,W] fp16 -> [B*(H/P)*(W/P), ldk] rows of (c, ky, kx), zero-padded to ldk columns."""
    lib = load()
    _f16(x, "x")
    B, C, H, W = x.shape
    assert x.is_contiguous()
    out = torch.empty((B * (H // patch) * (W // patch), ldk), dtype=torch.float16, device=x.device)
    _check(lib.b200vton_patchify(_p(x), B, C, H, W, patch, _p(out), ldk, _stream()), "b200vton_patchify")
    return out


def token_embedding(ids, tok, pos, T):
    """ids: int64 [rows] (rows = B*T); out[r] = fp16(tok[ids[r]] + pos[r % T])."""
    lib = load()
    _f16(tok, "tok"); _f16(pos, "pos")
    assert ids.dtype == torch.int64 and ids.is_cuda and ids.is_contiguous() and tok.is_contiguous() and pos.is_contiguous()
    rows, C = ids.numel(), tok.shape[1]
    out = torch.empty((rows, C), dtype=torch.float16, device=tok.device)
    _check(lib.b200vton_token_embedding(_p(ids), rows, T, C, tok.shape[0], _p(tok), _p(pos), _p(out), _stream()),
           "b200vton_token_embedding")
    return out


def conv3x3_f32_supported(x, cin, cout, width=None):
    """Shapes the TF32 convolution kernel covers (everything else stays on the caller's fallback). width: the width of
    the convolution's input when it is not x's own (x taken before a 2x upsampling)."""
    w = x.shape[3] if width is None else width
    return (x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and cin % 32 == 0 and cout % 32 == 0 and cout >= 64
            and w % 8 == 0)


def pack_conv3x3_f32(weight):
    """[Cout,Cin,3,3] fp32 -> [9,Cout,Cin] (tap-major rows for the kernel's weight map)."""
    return weight.detach().permute(2, 3, 0, 1).reshape(9, weight.shape[0], weight.shape[1]).contiguous()


def conv3x3_f32(x, w_packed, bias=None, residual=None):
    """x: logical [B,Cin,H,W] fp32 (any strides; converted to channels_last = NHWC memory); residual: logical [B,Cout,H,W]
    fp32 or None, added after the bias in the epilogue; returns a channels_last [B,Cout,H,W] fp32 tensor."""
    lib = load()
    B, Cin, H, W = x.shape
    Cout = w_packed.shape[1]
    assert w_packed.dtype == torch.float32 and w_packed.is_contiguous() and w_packed.shape == (9, Cout, Cin)
    x = x.contiguous(memory_format=torch.channels_last)
    if residual is not None:
        assert residual.shape == (B, Cout, H, W) and residual.dtype == torch.float32
        residual = residual.contiguous(memory_format=torch.channels_last)
    out = torch.empty((B, Cout, H, W), dtype=torch.float32, device=x.device, memory_format=torch.channels_last)
    rc = lib.b200vton_conv3x3_nhwc_f32(_p(x), B, H, W, Cin, _p(w_packed), Cout, _p(bias), _p(residual), _p(out), _stream())
    _check(rc, "b200vton_conv3x3_nhwc_f32")
    return out


def split_tf32(x, scale=1.0):
    """x: fp32 [B, ...] whose per-batch block is contiguous (a dense tensor or a row slice x[:, a:b] of a dense [B,N,C] one).
    Returns dense (hi, lo) with hi = tf32(x*scale), lo = tf32(x*scale - hi)."""
    lib = load()
    assert x.is_cuda and x.dtype == torch.float32 and x.dim() >= 2
    B = x.shape[0]
    per = x[0].numel()
    if not x[0].is_contiguous():
        x = x.contiguous()
    hi = torch.empty(x.shape, dtype=torch.float32, device=x.device)
    lo = torch.empty_like(hi)
    rc = lib.b200vton_split_tf32(_p(x), x.stride(0) if B > 1 else per, B, per, float(scale), _p(hi), _p(lo), _stream())
    _check(rc, "b200vton_split_tf32")
    return hi, lo


def softmax_split_tf32(scores):
    """scores: dense fp32 [..., N]; returns (p_hi, p_lo), the TF32 parts of softmax(scores, -1)."""
    lib = load()
    assert scores.is_cuda and scores.dtype == torch.float32 and scores.is_contiguous()
    N = scores.shape[-1]
    hi = torch.empty_like(scores)
    lo = torch.empty_like(scores)
    rc = lib.b200vton_softmax_split_tf32(_p(scores), scores.numel() // N, N, _p(hi), _p(lo), _stream())
    _check(rc, "b200vton_softmax_split_tf32")
    return hi, lo


_gn32_ws = {}


def conv3x3_f16in(x16, w_packed16, bias=None, residual=None):
    """x16: logical [B,Cin,H,W] fp16 in channels_last memory (the fp16 output of groupnorm_f32_nhwc); w_packed16: [9,Cout,Cin]
    fp16; bias [Cout] fp32; residual logical [B,Cout,H,W] fp32 or None. Returns a channels_last [B,Cout,H,W] fp32 tensor."""
    lib = load()
    B, Cin, H, W = x16.shape
    Cout = w_packed16.shape[1]
    assert x16.dtype == torch.float16 and x16.is_contiguous(memory_format=torch.channels_last)
    assert w_packed16.dtype == torch.float16 and w_packed16.is_contiguous() and w_packed16.shape == (9, Cout, Cin)
    if residual is not None:
        assert residual.shape == (B, Cout, H, W) and residual.dtype == torch.float32
        residual = residual.contiguous(memory_format=torch.channels_last)
    out = torch.empty((B, Cout, H, W), dtype=torch.float32, device=x16.device, memory_format=torch.channels_last)
    rc = lib.b200vton_conv3x3_nhwc_f16in_f32(_p(x16), B, H, W, Cin, _p(w_packed16), Cout, _p(bias), _p(residual), _p(out),
                                             _stream())
    _check(rc, "b200vton_conv3x3_nhwc_f16in_f32")
    return out


def groupnorm_f32_nhwc(x, gamma, beta, eps, silu, out_half=False):
    """x: logical [B,C,H,W] fp32 in channels_last memory (= dense NHWC); returns the same layout, fp32 or (out_half) fp16."""
    lib = load()
    B, C, H, W = x.shape
    assert x.dtype == torch.float32 and x.is_contiguous(memory_format=torch.channels_last)
    key = (x.device, torch.cuda.current_stream().cuda_stream)
    ws = _gn32_ws.get(key)
    need = 64 * max(B, 1184)
    if ws is None or ws.numel() < need:
        ws = torch.empty(need, dtype=torch.float64, device=x.device)
        _gn32_ws[key] = ws
    out = torch.empty(x.shape, dtype=torch.float16 if out_half else torch.float32, device=x.device,
                      memory_format=torch.channels_last)
    rc = lib.b200vton_groupnorm_nhwc_f32(_p(x), B, H * W, C, _p(gamma), _p(beta), float(eps), int(silu), _p(ws),
                                         ws.numel(), _p(out), int(out_half), _stream())
    _check(rc, "b200vton_groupnorm_nhwc_f32")
    return out


def cross_attention(q, kt, vt, ki=None, vi=None, heads=None, scale=None, ip_scale=1.0, out=None):
    """Text (+ IP-Adapter image token) cross-attention in one launch. q: [B,Nq,*]; kt/vt: [B,Nt<=80,*]; ki/vi:
    [B,Ni<=16,*] or None. 3-D views with contiguous last dim (slices of fused [K|V] buffers are fine)."""
    lib = load()
    B, Nq = q.shape[0], q.shape[1]
    H = heads
    Nt = kt.shape[1]
    assert q.stride(2) == 1 and kt.stride(2) == 1 and vt.stride() == kt.stride() and kt.shape[0] == B
    assert q.stride(0) == Nq * q.stride(1) and kt.stride(0) == Nt * kt.stride(1)
    if scale is None:
        scale = 64 ** -0.5
    if out is None:
        out = torch.empty(B, Nq, H * 64, dtype=torch.float16, device=q.device)
    assert out.stride(2) == 1 and out.stride(0) == Nq * out.stride(1)
    Ni, ldi = 0, 0
    if ki is not None:
        Ni, ldi = ki.shape[1], ki.stride(1)
        assert ki.stride(2) == 1 and vi.stride() == ki.stride() and ki.shape[0] == B and ki.stride(0) == Ni * ldi
    rc = lib.b200vton_cross_attention(_p(q), q.stride(1), _p(kt), _p(vt), kt.stride(1), Nt, _p(ki), _p(vi), ldi, Ni,
                                      _p(out), out.stride(1), B, H, Nq, float(scale), float(ip_scale), _stream())
    _check(rc, "b200vton_cross_attention")
    return out


_gn_ws = {}


GN_BARRIER_DOUBLES = 4096      # 8 bytes of barrier state per sample, up to 4096 samples (include/b200vton.h)


def _stats_ws(device, B):
    """GroupNorm workspace: max(B,296)*64 doubles of partial sums followed by the per-sample barrier state, which must be
    ZERO before first use (the kernel leaves it reusable), hence torch.zeros."""
    key = (device, torch.cuda.current_stream().cuda_stream)
    ws = _gn_ws.get(key)
    if ws is None or ws.numel() < max(B, 296) * 64 + GN_BARRIER_DOUBLES:
        ws = torch.zeros(max(B, 296) * 64 + GN_BARRIER_DOUBLES, dtype=torch.float64, device=device)
        _gn_ws[key] = ws
    return ws


def groupnorm(x0, gamma, beta, eps, silu, x1=None, out=None, ws=None):
    """x0: [B,HW,C0] (or [B,H,W,C0]) contiguous, optional x1 [B,HW,C1]: GroupNorm(32) over the channel concat."""
    lib = load()
    B = x0.shape[0]
    C0 = x0.shape[-1]
    HW = x0.numel() // (B * C0)
    C1 = x1.shape[-1] if x1 is not None else 0
    assert x0.is_contiguous() and (x1 is None or x1.is_contiguous())
    if out is None:
        out = torch.empty(x0.shape[:-1] + (C0 + C1,), dtype=torch.float16, device=x0.device)
    if ws is None:
        ws = _stats_ws(x0.device, B)
    rc = lib.b200vton_groupnorm(_p(x0), C0, _p(x1), C1, B, HW, _p(gamma), _p(beta), float(eps), int(silu), _p(ws),
                                _p(out), _stream())
    _check(rc, "b200vton_groupnorm")
    return out


def layernorm(x, gamma, beta, eps=1e-5, out=None):
    lib = load()
    C = x.shape[-1]
    x2 = x.reshape(-1, C)
    assert x2.stride(1) == 1
    if out is None:
        out = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    o2 = out.reshape(-1, C)
    rc = lib.b200vton_layernorm(_p(x2), x2.stride(0), x2.shape[0], C, _p(gamma), _p(beta), float(eps), _p(o2),
                                o2.stride(0), _stream())
    _check(rc, "b200vton_layernorm")
    return out


E4M3 = torch.float8_e4m3fn
E4M3_MAX = 448.0


def layernorm_e4m3(x, gamma, beta, eps=1e-5, fp16_out=False):
    """LayerNorm whose output feeds an FP8 linear: returns (q [rows, C] e4m3, scale [rows] fp32, y16 or None), with y16
    the fp16 LayerNorm row (bit-identical to `layernorm`, written only when fp16_out), scale = max|y16| / 448 and
    q = e4m3(y16 * 448 / max|y16|) (include/b200vton.h)."""
    fn = _optional("b200vton_layernorm_e4m3")
    _f16(x, "x")
    C = x.shape[-1]
    x2 = x.reshape(-1, C)
    assert x2.stride(1) == 1
    rows = x2.shape[0]
    q = torch.empty((rows, C), dtype=E4M3, device=x.device)
    scale = torch.empty(rows, dtype=torch.float32, device=x.device)
    out = torch.empty((rows, C), dtype=torch.float16, device=x.device) if fp16_out else None
    rc = fn(_p(x2), x2.stride(0), rows, C, _p(gamma), _p(beta), float(eps), _p(out), C if fp16_out else 0, _p(q),
            q.stride(0), _p(scale), _stream())
    _check(rc, "b200vton_layernorm_e4m3")
    return q, scale, out


def quantize_rows_e4m3(w):
    """Per-row e4m3 quantization of an fp16 matrix with torch (the FP8 linears' weights, once at pack time): the rule of
    layernorm_e4m3 applied to every row. Returns (q [N, K] e4m3, scale [N] fp32)."""
    w32 = w.to(torch.float32)
    amax = w32.abs().amax(dim=1)
    nz = amax > 0
    # tensor / tensor keeps IEEE division (torch divides by a Python scalar as a product with its reciprocal)
    lim = torch.full_like(amax, E4M3_MAX)
    inv = torch.where(nz, lim / torch.where(nz, amax, torch.ones_like(amax)), torch.zeros_like(amax))
    q = (w32 * inv[:, None]).clamp(-E4M3_MAX, E4M3_MAX).to(E4M3).contiguous()
    scale = torch.where(nz, amax / lim, torch.ones_like(amax)).contiguous()
    return q, scale


def gemm_e4m3(a_q, a_scale, w_q, w_scale, bias=None, residual=None, geglu=False, out=None, force_bn=0):
    """out[M,N] = epi((a_q[M,K] @ w_q[N,K]^T) * a_scale[m] * w_scale[n]) with gemm's fp16 epilogue (bias, GEGLU,
    residual). a_q / w_q: e4m3 (row-strided 2-D views with contiguous last dim); a_scale [M], w_scale [N] fp32."""
    fn = _optional("b200vton_gemm_e4m3")
    if a_q.dtype != E4M3 or w_q.dtype != E4M3:
        raise TypeError(f"gemm_e4m3: operands must be {E4M3}, got {a_q.dtype} and {w_q.dtype}")
    M, K = a_q.shape
    N = w_q.shape[0]
    assert w_q.shape[1] == K and a_q.stride(1) == 1 and w_q.stride(1) == 1
    assert a_scale.dtype == torch.float32 and w_scale.dtype == torch.float32
    assert a_scale.numel() == M and w_scale.numel() == N
    n_out = N // 2 if geglu else N
    if out is None:
        out = torch.empty((M, n_out), dtype=torch.float16, device=a_q.device)
    assert out.shape == (M, n_out) and out.stride(1) == 1
    if residual is not None:
        assert residual.shape == (M, n_out) and residual.stride(1) == 1
    rc = fn(_p(a_q), a_q.stride(0), _p(a_scale), _p(w_q), w_q.stride(0), _p(w_scale), _p(out), out.stride(0), M, N, K,
            _p(bias), _p(residual), residual.stride(0) if residual is not None else 0, int(geglu), force_bn, _stream())
    _check(rc, "b200vton_gemm_e4m3")
    return out


def _check_scatter_shapes(src, dst, c_off):
    """The C ABI takes H, W from the source only: a dst of another size would be written out of bounds (larger src) or
    left partly unwritten (smaller src), so the sizes are compared here, before any launch."""
    if src.dim() != 4 or dst.dim() != 4:
        raise ValueError(f"nchw_to_nhwc: src must be [B,C,H,W] and dst [B,H,W,ldc], got {tuple(src.shape)} and "
                         f"{tuple(dst.shape)}")
    if tuple(src.shape[2:]) != tuple(dst.shape[1:3]):
        raise ValueError(f"nchw_to_nhwc: src spatial size {tuple(src.shape[2:])} differs from dst's "
                         f"{tuple(dst.shape[1:3])}")
    if c_off < 0 or c_off + src.shape[1] > dst.shape[3]:
        raise ValueError(f"nchw_to_nhwc: channels [{c_off}, {c_off + src.shape[1]}) do not fit dst's {dst.shape[3]}")
    if not (src.is_contiguous() and dst.is_contiguous()):
        raise ValueError("nchw_to_nhwc: src and dst must be contiguous")


def nchw_to_nhwc(src, dst, c_off=0):
    """dst[s,y,x,c_off+c] = src[s % Bs, c, y, x]; dst: [Bd,H,W,ldc] contiguous, the same H, W as src."""
    _check_scatter_shapes(src, dst, c_off)
    lib = load()
    Bs, Cs, H, W = src.shape
    rc = lib.b200vton_nchw_to_nhwc(_p(src), Bs, Cs, H, W, _p(dst), dst.shape[0], dst.shape[-1], c_off, _stream())
    _check(rc, "b200vton_nchw_to_nhwc")
    return dst


def nchw_to_nhwc_scaled(src, dst, scale, c_off=0):
    """nchw_to_nhwc with dst = fp16(src * scale[0]); scale: one fp32 on the device (a graph replays it per step)."""
    _check_scatter_shapes(src, dst, c_off)
    lib = load()
    Bs, Cs, H, W = src.shape
    assert scale.dtype == torch.float32 and scale.is_cuda and scale.numel() >= 1
    rc = lib.b200vton_nchw_to_nhwc_scaled(_p(src), Bs, Cs, H, W, _p(dst), dst.shape[0], dst.shape[-1], c_off, _p(scale),
                                          _stream())
    _check(rc, "b200vton_nchw_to_nhwc_scaled")
    return dst


def nhwc_to_nchw(src, C, out=None):
    lib = load()
    B, H, W, ldc = src.shape
    if out is None:
        out = torch.empty((B, C, H, W), dtype=torch.float16, device=src.device)
    rc = lib.b200vton_nhwc_to_nchw(_p(src), B, C, H, W, ldc, _p(out), _stream())
    _check(rc, "b200vton_nhwc_to_nchw")
    return out


def upsample2x(x, out=None):
    lib = load()
    B, H, W, C = x.shape
    if out is None:
        out = torch.empty((B, 2 * H, 2 * W, C), dtype=torch.float16, device=x.device)
    rc = lib.b200vton_upsample2x_nhwc(_p(x), B, H, W, C, _p(out), _stream())
    _check(rc, "b200vton_upsample2x_nhwc")
    return out


def upsample_nearest(x, size, out=None):
    """x: [B,H,W,C] NHWC fp16 (contiguous) -> [B,Hout,Wout,C], F.interpolate(size=(Hout, Wout), mode="nearest")."""
    lib = load()
    _f16(x, "x")
    B, H, W, C = x.shape
    Hout, Wout = int(size[0]), int(size[1])
    assert x.is_contiguous()
    if out is None:
        out = torch.empty((B, Hout, Wout, C), dtype=torch.float16, device=x.device)
    assert out.shape == (B, Hout, Wout, C) and out.is_contiguous()
    rc = lib.b200vton_upsample_nearest_nhwc(_p(x), B, H, W, C, Hout, Wout, _p(out), _stream())
    _check(rc, "b200vton_upsample_nearest_nhwc")
    return out


def im2col3x3_s2(x, out=None):
    lib = load()
    B, H, W, C = x.shape
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    if out is None:
        out = torch.empty((B * Ho * Wo, 9 * C), dtype=torch.float16, device=x.device)
    rc = lib.b200vton_im2col3x3_s2_nhwc(_p(x), B, H, W, C, _p(out), _stream())
    _check(rc, "b200vton_im2col3x3_s2_nhwc")
    return out


def timestep_embedding(values, dim, rows_repeat=1, out=None):
    """values: fp32 CUDA tensor [n]; returns [n*rows_repeat, dim] fp16 ([cos|sin])."""
    lib = load()
    assert values.dtype == torch.float32 and values.is_cuda
    n = values.numel()
    if out is None:
        out = torch.empty((n * rows_repeat, dim), dtype=torch.float16, device=values.device)
    rc = lib.b200vton_timestep_embedding(_p(values), n, dim, rows_repeat, _p(out), _stream())
    _check(rc, "b200vton_timestep_embedding")
    return out


def skinny_linear(x, w, bias=None, in_silu=False, out_silu=False, addend=None, out=None):
    lib = load()
    M, K = x.shape
    N = w.shape[0]
    if out is None:
        out = torch.empty((M, N), dtype=torch.float16, device=x.device)
    rc = lib.b200vton_skinny_linear(_p(x), x.stride(0), M, K, _p(w), w.stride(0), N, _p(bias), int(in_silu),
                                    int(out_silu), _p(addend), addend.stride(0) if addend is not None else 0, _p(out),
                                    out.stride(0), _stream())
    _check(rc, "b200vton_skinny_linear")
    return out


def cfg_ddpm_step(eps, latents, noise, coef, do_cfg=True, out=None):
    """eps: [2B,H,W,ldc] NHWC (or [B,...] without CFG); latents/noise: [B,C,H,W]; coef: 6 fp32 on device."""
    lib = load()
    B, C, H, W = latents.shape
    if out is None:
        out = torch.empty_like(latents)
    rc = lib.b200vton_cfg_ddpm_step(_p(eps), eps.shape[-1], B, C, H, W, _p(latents), _p(noise), _p(coef), int(do_cfg),
                                    _p(out), _stream())
    _check(rc, "b200vton_cfg_ddpm_step")
    return out


def cfg_rescale_ddpm_step(eps, latents, noise, coef, do_cfg=True, out=None):
    """cfg_ddpm_step with guidance rescale; coef: 7 fp32 on device (the 6 of cfg_ddpm_step, then guidance_rescale)."""
    lib = load()
    B, C, H, W = latents.shape
    if out is None:
        out = torch.empty_like(latents)
    rc = lib.b200vton_cfg_rescale_ddpm_step(_p(eps), eps.shape[-1], B, C, H, W, _p(latents), _p(noise), _p(coef),
                                            int(do_cfg), _p(out), _stream())
    _check(rc, "b200vton_cfg_rescale_ddpm_step")
    return out


def preprocess_inpaint(image, mask, vae_scale=8):
    """image [B,3,H,W] fp32 CUDA in [0,1] (or already [-1,1]), mask [B,1|3,H,W] fp32 -> (init_image, mask_bin, masked_image,
    mask_latent fp16 [B,1,H/s,W/s]); one launch, no host sync."""
    lib = load()
    B, _, H, W = image.shape
    assert image.is_cuda and image.dtype == torch.float32 and mask.dtype == torch.float32 and mask.shape[0] == B
    assert mask.shape[-2:] == image.shape[-2:] and image.is_contiguous() and mask.is_contiguous()
    img_min = image.amin().reshape(1)
    init = torch.empty_like(image)
    masked = torch.empty_like(image)
    mbin = torch.empty((B, 1, H, W), dtype=torch.float32, device=image.device)
    mlat = torch.empty((B, 1, H // vae_scale, W // vae_scale), dtype=torch.float16, device=image.device)
    rc = lib.b200vton_preprocess_inpaint(_p(image), _p(mask), mask.shape[1], _p(img_min), B, H, W, vae_scale, _p(init),
                                         _p(mbin), _p(masked), _p(mlat), _stream())
    _check(rc, "b200vton_preprocess_inpaint")
    return init, mbin, masked, mlat


def postprocess_image(x, want_pt=True, want_u8=False):
    """x: logical [B,3,H,W] fp32 CUDA, contiguous either as NCHW or as channels_last (NHWC memory). Returns
    (fp32 NCHW in [0,1] or None, uint8 NHWC or None)."""
    lib = load()
    B, C, H, W = x.shape
    assert C == 3 and x.is_cuda and x.dtype == torch.float32
    nhwc = 0
    if not x.is_contiguous():
        if x.is_contiguous(memory_format=torch.channels_last):
            nhwc = 1
        else:
            x = x.contiguous()
    pt = torch.empty((B, 3, H, W), dtype=torch.float32, device=x.device) if want_pt else None
    u8 = torch.empty((B, H, W, 3), dtype=torch.uint8, device=x.device) if want_u8 else None
    rc = lib.b200vton_postprocess_image(_p(x), nhwc, B, H, W, _p(pt), _p(u8), _stream())
    _check(rc, "b200vton_postprocess_image")
    return pt, u8


SOLVER_KINDS = {"ddim": 0, "euler": 1, "dpmpp": 2}


def cfg_solver_step(eps, latents, noise, coef, kind, x0_prev=None, do_cfg=True, out=None):
    """CFG + one DDIM / Euler / DPM-Solver++ step. eps, latents, noise as cfg_ddpm_step; coef: 8 fp32 on device
    {gs, s, inv_a, p, q, r, sigma_n, k}; kind: "ddim" | "euler" | "dpmpp"; x0_prev: [B,C,H,W] fp16 state of
    DPM-Solver++ (read, then overwritten with this step's data prediction)."""
    lib = load()
    B, C, H, W = latents.shape
    if out is None:
        out = torch.empty_like(latents)
    rc = lib.b200vton_cfg_solver_step(_p(eps), eps.shape[-1], B, C, H, W, _p(latents), _p(noise), _p(x0_prev), _p(coef),
                                      SOLVER_KINDS[kind], int(do_cfg), _p(out), _stream())
    _check(rc, "b200vton_cfg_solver_step")
    return out


def _coef_rows(coef, B, name):
    """coef: [B, stride] fp32 CUDA rows (contiguous) or one row [n] shared by all samples (stride 0)."""
    if coef.dtype != torch.float32 or not coef.is_cuda or not coef.is_contiguous():
        raise TypeError(f"{name}: coef must be a contiguous CUDA fp32 tensor")
    if coef.dim() == 1:
        return 0
    if coef.dim() != 2 or coef.shape[0] != B:
        raise ValueError(f"{name}: coef must be [B={B}, stride] or one row, got {tuple(coef.shape)}")
    return coef.shape[1]


def cfg_ddpm_step_rows(eps, latents, noise, coef, do_cfg=True, out=None):
    """cfg_ddpm_step with one coefficient row per sample: coef [B, stride >= 6] fp32 on device, sample b reads row b."""
    fn = _optional("b200vton_cfg_ddpm_step_rows")
    B, C, H, W = latents.shape
    stride = _coef_rows(coef, B, "cfg_ddpm_step_rows")
    if out is None:
        out = torch.empty_like(latents)
    rc = fn(_p(eps), eps.shape[-1], B, C, H, W, _p(latents), _p(noise), _p(coef), stride, int(do_cfg), _p(out), _stream())
    _check(rc, "b200vton_cfg_ddpm_step_rows")
    return out


def cfg_solver_step_rows(eps, latents, noise, coef, kind, x0_prev=None, do_cfg=True, out=None):
    """cfg_solver_step with one coefficient row per sample: coef [B, stride >= 8] fp32 on device, sample b reads row b."""
    fn = _optional("b200vton_cfg_solver_step_rows")
    B, C, H, W = latents.shape
    stride = _coef_rows(coef, B, "cfg_solver_step_rows")
    if out is None:
        out = torch.empty_like(latents)
    rc = fn(_p(eps), eps.shape[-1], B, C, H, W, _p(latents), _p(noise), _p(x0_prev), _p(coef), stride,
            SOLVER_KINDS[kind], int(do_cfg), _p(out), _stream())
    _check(rc, "b200vton_cfg_solver_step_rows")
    return out


def nchw_to_nhwc_scaled_rows(src, dst, scale, c_off=0):
    """nchw_to_nhwc with dst row s = fp16(src[s % Bs] * scale[s % Bs]); scale: Bs fp32 on the device."""
    _check_scatter_shapes(src, dst, c_off)
    fn = _optional("b200vton_nchw_to_nhwc_scaled_rows")
    Bs, Cs, H, W = src.shape
    assert scale.dtype == torch.float32 and scale.is_cuda and scale.numel() >= Bs
    rc = fn(_p(src), Bs, Cs, H, W, _p(dst), dst.shape[0], dst.shape[-1], c_off, _p(scale), _stream())
    _check(rc, "b200vton_nchw_to_nhwc_scaled_rows")
    return dst



def cfg_step_mixed_rows(eps, latents, noise, coef, kinds, x0_prev, do_cfg=True, out=None):
    """One step of a batch whose samples follow different schedulers: sample b takes kind kinds[b] (0 DDIM, 1 Euler, 2 DPM-Solver++, 3 DDPM) with
    coefficient row b of coef [B, 8] fp32 (DDPM rows {gs, sb, inv_sa, c0, c1, sigma, phi, 0}, the others as
    cfg_solver_step). noise enters DDPM and DDIM rows only; x0_prev [B,C,H,W] fp16 is required and only DPM-Solver++
    rows read and rewrite it. kinds: contiguous CUDA int32 tensor of B entries."""
    fn = _optional("b200vton_cfg_step_mixed_rows")
    B, C, H, W = latents.shape
    stride = _coef_rows(coef, B, "cfg_step_mixed_rows")
    if kinds.dtype != torch.int32 or not kinds.is_cuda or not kinds.is_contiguous() or kinds.numel() != B:
        raise ValueError(f"cfg_step_mixed_rows: kinds must be a contiguous CUDA int32 tensor of B = {B} entries, got "
                         f"{kinds.dtype} {tuple(kinds.shape)} on {kinds.device}")
    if out is None:
        out = torch.empty_like(latents)
    rc = fn(_p(eps), eps.shape[-1], B, C, H, W, _p(latents), _p(noise), _p(x0_prev), _p(coef), stride, _p(kinds),
            int(do_cfg), _p(out), _stream())
    _check(rc, "b200vton_cfg_step_mixed_rows")
    return out


class ResampleDesc(ctypes.Structure):
    """b200vton_resample_desc (include/b200vton.h): one crop to resample."""
    _fields_ = [("src", _vp), ("src_pitch", _i64), ("src_w", _c.c_int32), ("src_h", _c.c_int32),
                ("crop_x", _c.c_int32), ("crop_y", _c.c_int32), ("crop_w", _c.c_int32), ("crop_h", _c.c_int32),
                ("dst", _vp), ("dst_pitch", _i64), ("out_f32", _vp), ("out_w", _c.c_int32), ("out_h", _c.c_int32),
                ("channels", _c.c_int32), ("f32_mode", _c.c_int32),
                ("bounds_x", _c.c_int32), ("coefs_x", _c.c_int32), ("ksize_x", _c.c_int32), ("need_x", _c.c_int32),
                ("bounds_y", _c.c_int32), ("coefs_y", _c.c_int32), ("ksize_y", _c.c_int32), ("need_y", _c.c_int32),
                ("tmp_offset", _i64), ("tmp_first", _c.c_int32), ("tmp_rows", _c.c_int32)]


class PasteDesc(ctypes.Structure):
    """b200vton_paste_desc (include/b200vton.h): one photo's paste-back."""
    _fields_ = [("photo", _vp), ("photo_pitch", _i64), ("dst", _vp), ("dst_pitch", _i64), ("image", _vp),
                ("image_pitch", _i64), ("mask", _vp), ("mask_pitch", _i64),
                ("width", _c.c_int32), ("height", _c.c_int32), ("box_x", _c.c_int32), ("box_y", _c.c_int32),
                ("box_w", _c.c_int32), ("box_h", _c.c_int32), ("mask_x", _c.c_int32), ("mask_y", _c.c_int32),
                ("mask_w", _c.c_int32), ("mask_h", _c.c_int32)]


def _descs_to_device(descs, device):
    """A ctypes array of descriptors -> (the array, its device copy) through pinned memory (no host sync; the caching
    host allocator keeps the staging block until the copy has run)."""
    host = torch.frombuffer(bytearray(descs), dtype=torch.uint8).pin_memory()
    return host.to(device, non_blocking=True)


def resample_u8(descs, tables, workspace):
    """b200vton_resample_u8 on a list of ResampleDesc: tables, an int32 CUDA tensor holding every descriptor's bounds
    and fixed-point coefficients (the descriptors' offsets index it); workspace, a uint8 CUDA tensor for the
    intermediate rows (the descriptors' tmp_offset index it)."""
    fn = _optional("b200vton_resample_u8")
    if tables.dtype != torch.int32 or not tables.is_cuda or not tables.is_contiguous():
        raise ValueError("resample_u8: tables must be a contiguous CUDA int32 tensor")
    if workspace.dtype != torch.uint8 or not workspace.is_cuda or not workspace.is_contiguous():
        raise ValueError("resample_u8: workspace must be a contiguous CUDA uint8 tensor")
    arr = (ResampleDesc * len(descs))(*descs)
    dev = _descs_to_device(arr, tables.device)
    _check(fn(arr, _p(dev), len(descs), _p(tables), tables.numel(), _p(workspace), workspace.numel(), _stream()),
           "b200vton_resample_u8")


def paste_u8(descs, device):
    """b200vton_paste_u8 on a list of PasteDesc."""
    fn = _optional("b200vton_paste_u8")
    arr = (PasteDesc * len(descs))(*descs)
    dev = _descs_to_device(arr, device)
    _check(fn(arr, _p(dev), len(descs), _stream()), "b200vton_paste_u8")


CLIP_SIZE = 224        # B200VTON_CLIP_SIZE


class ClipDesc(ctypes.Structure):
    """b200vton_clip_desc (include/b200vton.h): one CLIP-size image and the origin of its 224 x 224 crop."""
    _fields_ = [("src", _vp), ("src_pitch", _i64), ("src_w", _c.c_int32), ("src_h", _c.c_int32),
                ("crop_x", _c.c_int32), ("crop_y", _c.c_int32)]


def clip_pixels_u8(descs, table, out):
    """b200vton_clip_pixels_u8 on a list of ClipDesc: table, a contiguous fp32 CUDA tensor of 3 x 256 entries; out, a
    contiguous fp32 CUDA tensor [len(descs), 3, 224, 224]."""
    fn = _optional("b200vton_clip_pixels_u8")
    if table.dtype != torch.float32 or not table.is_cuda or not table.is_contiguous() or table.numel() != 3 * 256:
        raise ValueError("clip_pixels_u8: table must be a contiguous CUDA fp32 tensor of 3 x 256 entries")
    if out.dtype != torch.float32 or not out.is_cuda or not out.is_contiguous() or \
            tuple(out.shape) != (len(descs), 3, CLIP_SIZE, CLIP_SIZE):
        raise ValueError(f"clip_pixels_u8: out must be a contiguous CUDA fp32 tensor [{len(descs)}, 3, {CLIP_SIZE}, "
                         f"{CLIP_SIZE}], got {out.dtype} {tuple(out.shape)} on {out.device}")
    arr = (ClipDesc * len(descs))(*descs)
    dev = _descs_to_device(arr, out.device)
    _check(fn(arr, _p(dev), len(descs), _p(table), _p(out), _stream()), "b200vton_clip_pixels_u8")


def freeu(hidden, skip, b, s, out=None):
    """FreeU before one up-stage resnet (diffusers `apply_freeu`): scales the first half of hidden's channels by b in
    place (fp16(float(h) * b)) and writes fourier_filter(skip, threshold=1, scale=s) to `out`, or in place into skip
    when out is None. hidden [B,H,W,Ch] and skip [B,H,W,Cs]: contiguous NHWC fp16 CUDA tensors at the same B, H, W.
    Returns the filtered skip."""
    fn = _optional("b200vton_freeu_nhwc")
    _f16(hidden, "hidden"); _f16(skip, "skip"); _f16(out, "out")
    if hidden.ndim != 4 or skip.ndim != 4 or hidden.shape[:3] != skip.shape[:3]:
        raise ValueError(f"freeu: hidden {tuple(hidden.shape)} and skip {tuple(skip.shape)} must be [B,H,W,C] at the "
                         "same B, H, W")
    if not hidden.is_contiguous() or not skip.is_contiguous():
        raise ValueError("freeu: hidden and skip must be contiguous")
    if out is None:
        out = skip
    elif out.shape != skip.shape or not out.is_contiguous():
        raise ValueError(f"freeu: out must be a contiguous tensor of skip's shape {tuple(skip.shape)}")
    B, H, W, Ch = hidden.shape
    rc = fn(_p(hidden), Ch, _p(skip), _p(out), skip.shape[3], B, H, W, float(b), float(s), _stream())
    _check(rc, "b200vton_freeu_nhwc")
    return out
