"""Launch inventory: record every call the engine makes to the op wrappers of idm_vton_b200.lib, and replay each distinct
call in isolation against the float64 restatements of tests/test_kernel_edges_gpu.py (and the solver / schedule / FP8 /
FP8-K/V references).

A recorded call is a *signature*: the wrapper name, then per argument either a tensor descriptor (shape, strides, dtype,
storage group, element offset within the group, and the values of small int32 / fp32 device tables), a pair of them (a
lib.GarmentKV8) or the scalar itself. Arguments that share storage get the same group, so `out=` views of larger
buffers, residuals and K/V column slices of one fused buffer replay as they ran. Offsets are rebased per group to a
multiple of 1024 elements below the smallest one, which keeps every alignment the kernels check.

Nothing here needs a GPU: the recorder and the operand builder work on CPU tensors, which is what the CPU tests use."""
import inspect
import math

import torch

# the op wrappers of idm_vton_b200.lib the engine, the denoisers and the servers call as L.<name>(...)
WRAPPED = ("gemm", "gemm_e4m3", "conv3x3", "attention", "attention_rows", "attention_kv8", "cross_attention",
           "groupnorm", "layernorm", "layernorm_e4m3", "quantize_kv_e4m3", "skinny_linear", "timestep_embedding",
           "upsample2x", "upsample_nearest", "nchw_to_nhwc", "nchw_to_nhwc_scaled", "nchw_to_nhwc_scaled_rows",
           "nhwc_to_nchw", "cfg_ddpm_step", "cfg_rescale_ddpm_step", "cfg_solver_step", "cfg_ddpm_step_rows",
           "cfg_solver_step_rows", "cfg_step_mixed_rows")
# int32 / fp32 device tensors up to this many entries are steering tables (kv1_base, kv1_rows, coefficient rows, kinds,
# timesteps, time ids, the input scale): their values are part of the signature
TABLE_MAX = 64
ALIGN = 1024


def _table(t):
    return t.dtype in (torch.int32, torch.float32) and t.numel() <= TABLE_MAX


def _tensors(v):
    if isinstance(v, torch.Tensor):
        return [v]
    if isinstance(v, tuple) and v and all(isinstance(x, torch.Tensor) for x in v):
        return list(v)
    return []


def signature(name, fn, args, kwargs, extra=None):
    """The signature of one call of wrapper `name` (fn: the wrapper, for its parameter names and defaults). extra: more
    (key, value) scalars (the GEGLU packing width of a weight)."""
    bound = inspect.signature(fn).bind(*args, **kwargs)
    bound.apply_defaults()
    groups, order = {}, []
    for v in bound.arguments.values():
        for t in _tensors(v):
            key = t.untyped_storage().data_ptr()
            if key not in groups:
                groups[key] = []
                order.append(key)
            groups[key].append(t)
    index = {k: i for i, k in enumerate(order)}
    base = {k: min(t.storage_offset() for t in ts) // ALIGN * ALIGN for k, ts in groups.items()}

    def desc(t):
        k = t.untyped_storage().data_ptr()
        vals = tuple(t.flatten().tolist()) if _table(t) else None
        return ("T", tuple(t.shape), tuple(t.stride()), str(t.dtype).replace("torch.", ""), index[k],
                t.storage_offset() - base[k], vals)

    items = []
    for n, v in bound.arguments.items():
        if isinstance(v, torch.Tensor):
            items.append((n, desc(v)))
        elif _tensors(v):
            items.append((n, ("K8",) + tuple(desc(t) for t in v)))
        elif isinstance(v, (torch.Size, list)):
            items.append((n, ("S", tuple(int(x) for x in v))))
        else:
            items.append((n, ("S", v)))
    return (name, tuple(items) + tuple(sorted((extra or {}).items())))


def args_of(sig):
    """{argument name: descriptor} of a signature; scalars unwrapped."""
    out = {}
    for n, d in sig[1]:
        if isinstance(d, tuple) and d and d[0] == "S":
            out[n] = d[1]
        else:
            out[n] = d
    return out


def is_tensor_desc(d):
    return isinstance(d, tuple) and len(d) == 7 and d[0] == "T"


def seed_of(sig):
    """A seed derived from the signature (stable across runs and processes: not Python's salted hash)."""
    h = 1469598103934665603
    for ch in repr(sig).encode():
        h = ((h ^ ch) * 1099511628211) % (1 << 61)
    return h % (1 << 31)


class Recorder:
    """Wraps the op wrappers of module L (idm_vton_b200.lib) through `monkeypatch`; every call passes through unchanged
    and its signature is recorded in first-seen order, deduplicated. pack_bn: {weight data_ptr: GEGLU packing width}."""

    def __init__(self, L, monkeypatch, pack_bn=None):
        self.L = L
        self.sigs = {}                 # signature -> number of calls
        self.pack_bn = pack_bn if pack_bn is not None else {}
        self.missing = []
        for name in WRAPPED:
            fn = getattr(L, name, None)
            if fn is None:
                self.missing.append(name)
                continue
            monkeypatch.setattr(L, name, self._wrap(name, fn))

    def _wrap(self, name, fn):
        def call(*args, **kwargs):
            extra = None
            if name in ("gemm", "gemm_e4m3"):
                b = inspect.signature(fn).bind(*args, **kwargs)
                w = b.arguments.get("w", b.arguments.get("w_q"))
                if b.arguments.get("geglu", False):
                    extra = {"pack_bn": self.pack_bn.get(w.data_ptr())}
            sig = signature(name, fn, args, kwargs, extra)
            self.sigs[sig] = self.sigs.get(sig, 0) + 1
            return fn(*args, **kwargs)
        return call


# ------------------------------------------------------------------------------------------------------------------
# operands
# ------------------------------------------------------------------------------------------------------------------
def _numel_extent(shape, stride):
    if any(s == 0 for s in shape):
        return 0
    return 1 + sum((n - 1) * st for n, st in zip(shape, stride))


def build_operands(sig, device):
    """Fresh storage for every group of the signature and the argument views into it, with the recorded shapes, strides
    and offsets; small tables hold their recorded values, everything else zeros (the replay fills the inputs).
    Returns {name: tensor | (tensor, tensor) | scalar}."""
    a = args_of(sig)
    descs = []
    for d in a.values():
        if is_tensor_desc(d):
            descs.append(d)
        elif isinstance(d, tuple) and d and d[0] == "K8":
            descs += list(d[1:])
    extent, dtype = {}, {}
    for d in descs:
        _, shape, stride, dt, g, off, _ = d
        extent[g] = max(extent.get(g, 0), off + _numel_extent(shape, stride))
        if dtype.setdefault(g, dt) != dt:
            raise ValueError(f"{sig[0]}: storage group {g} holds {dtype[g]} and {dt}")
    bufs = {}
    for g, n in extent.items():
        dt = getattr(torch, dtype[g])
        bufs[g] = torch.zeros(max(n, 1), dtype=torch.uint8 if dt.itemsize == 1 else dt, device=device)
        if dt.itemsize == 1:
            bufs[g] = bufs[g].view(dt)

    def view(d):
        _, shape, stride, _, g, off, vals = d
        t = torch.as_strided(bufs[g], shape, stride, off)
        if vals is not None:
            t.copy_(torch.tensor(vals, dtype=t.dtype).view(shape))
        return t

    out = {}
    for n, d in a.items():
        if is_tensor_desc(d):
            out[n] = view(d)
        elif isinstance(d, tuple) and d and d[0] == "K8":
            out[n] = tuple(view(x) for x in d[1:])
        else:
            out[n] = d
    return out


def sample_rows(M, full_below=512):
    """Rows {0, 63, 64, 127} of every 128-row tile plus the last row (every tile of the schedule, both consumer
    warpgroups); all rows up to full_below."""
    if M <= full_below:
        return list(range(M))
    return sorted({t + o for t in range(0, M, 128) for o in (0, 63, 64, 127) if t + o < M} | {M - 1})


def pick_bn(N, M, geglu, force_bn, sms=132):
    """The tile width gemm.cu's pick_bn takes for an (M, N) GEMM on an H100 SXM (132 SMs), for the report."""
    if force_bn:
        return force_bn % 1000
    best, best_bn = 1e300, 0
    for bn in (256, 192, 160, 128, 64):
        if geglu and (bn not in (256, 128) or N % bn):
            continue
        if bn != 128 and N % bn and not (bn == 64 and N < 64):
            continue
        cost = -(-(-(-M // 128) * -(-N // bn)) // sms) * (bn + 64)
        if cost < best * 0.999:
            best, best_bn = cost, bn
    return best_bn


# ------------------------------------------------------------------------------------------------------------------
# truths and mutants that are checked without a GPU as well
# ------------------------------------------------------------------------------------------------------------------
def seg1_rows(B, kv1_off, B1, kv1_mod=0, base=0, rows=None):
    """Per sample: the segment-1 row it reads, or None (the all-zero K/V closed form) (include/b200vton.h)."""
    out = []
    for b in range(B):
        if b < kv1_off:
            out.append(None)
        elif rows is not None:
            r = int(rows[b - kv1_off])
            out.append(None if r < 0 else r)
        else:
            out.append(base + (b - kv1_off) % (kv1_mod or B1))
    return out


def neighbour_rows(B, kv1_off, B1, truth_rows, kv1_mod=0, base=0, rows=None):
    """The mutant 'segment 1 from the neighbouring row': the row with kv1_mod / kv1_base ignored ((b - kv1_off) % B1),
    or, where that is the true row (or rows were given per sample), the next row; None where no other row exists."""
    out = []
    for b, r in enumerate(truth_rows):
        if r is None or B1 < 2:
            out.append(None)
            continue
        m = (b - kv1_off) % B1 if rows is None else (r + 1) % B1
        out.append(m if m != r else (r + 1) % B1)
    return out


def gn_x1_in_x0_layout(x1, C0):
    """GroupNorm mutant: the channels past C0 read with source 0's pixel stride (x1 flat index p * C0 + j)."""
    B, C1 = x1.shape[0], x1.shape[-1]
    flat = x1.reshape(B, -1)
    HW = flat.shape[1] // C1
    idx = (torch.arange(HW, device=x1.device)[:, None] * C0 + torch.arange(C1, device=x1.device)[None, :]) % flat.shape[1]
    return flat[:, idx.flatten()].view(x1.shape)


def gn_groups(C0, C1, groups=32):
    """(channels per group, index of the group that spans both sources or None)."""
    gs = (C0 + C1) // groups
    return gs, (C0 // gs if C1 and C0 % gs else None)


def gn_offset_dev(shape, seed, device, std=0.01, offset=100):
    """GroupNorm input as gn_offset_input builds it (every channel's mean = offset std + 0.01 std noise, unit-std spread
    around it), at std 0.01 so that eps (1e-5 / 1e-6) moves the output by eps / (2 var) >= 4x TOL_NORM16: the eps
    mutant is visible. Drawn on `device` (production sizes)."""
    g = torch.Generator(device=device).manual_seed(seed)
    C = shape[-1]
    means = offset * std + 0.01 * std * torch.randn(C, generator=g, device=device, dtype=torch.float64)
    return (means + std * torch.randn(*shape, generator=g, device=device, dtype=torch.float64)).half()


def grid_dev(shape, scale, seed, device, levels=8):
    """grid16's values (k * scale / levels, |k| <= levels) drawn on `device` (the operands of production-size launches)."""
    g = torch.Generator(device=device).manual_seed(seed)
    k = torch.randint(-levels, levels + 1, tuple(shape), generator=g, device=device, dtype=torch.int32)
    return (k.double() * (scale / levels)).half()


def randn_dev(shape, seed, device, scale=1.0, shift=0.0):
    g = torch.Generator(device=device).manual_seed(seed)
    return (torch.randn(tuple(shape), generator=g, device=device, dtype=torch.float32) * scale + shift).half()


def ip_cancel_values(vt_shape, vi_shape, seed, device):
    """V of text and IP tokens for the IP rounding check at a recorded shape (with q = 0, so every score is 0 and the
    softmax is a plain mean): vt on a 2^-5 grid, vi = -(the text mean rounded to 2^-10) plus a +-2^-8 grid, so that
    O_t + O_i nearly cancels and the fp16 rounding of O_t decides the result. Every sum is exact in fp32, and a mean
    of Nt = 77 such values lies at least 2^-15 / 77 from any fp16 tie, far beyond the fp32 error of the division."""
    vt = grid_dev(vt_shape, 2.0, seed, device, levels=64)
    m = torch.round(vt.double().mean(1, keepdim=True) * 1024) / 1024
    vi = (-m + grid_dev(vi_shape, 1 / 256, seed + 1, device, levels=1).double()).half()
    assert torch.equal(vi.double(), -m + grid_dev(vi_shape, 1 / 256, seed + 1, device, levels=1).double())
    return vt, vi


def ulp16(x):
    """One fp16 ulp at |x| (subnormal spacing below 2^-14)."""
    e = torch.floor(torch.log2(x.double().abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e - 10)


def timestep_args(values, dim):
    """t * freq formed in fp32 as diffusers' Timesteps does (exponent in fp32, exp in fp32, fp32 product)."""
    half = dim // 2
    exponent = -math.log(10000) * torch.arange(half, dtype=torch.float32, device=values.device) / half
    return values.float()[:, None] * torch.exp(exponent)[None, :]
