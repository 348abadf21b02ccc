"""Restatement of the FP8 linears (UNetEngine(fp8=True)) for the tests: the quantization rule, the quantized linear in
float arithmetic, the mistakes the tests must tell apart from the rule, and a BasicTransformerBlock for
oracle/unet_ref.py whose per-token linears (attn1 QKV, attn2.to_q, the GEGLU projection) are quantized.

The rule (one definition for activations and weights):
  y16 = the fp16 row the fp16 engine feeds the GEMM; amax = max|y16|; scale = amax / 448 (fp32);
  inv = 448 / amax (fp32, IEEE division); q = e4m3_rn_satfinite(y16 * inv); a row with amax == 0: scale 1, q 0.
  GEMM: v = (acc * scale_a[m]) * scale_w[n] in fp32, acc = sum_k q_a[m, k] q_w[n, k]; then the fp16 epilogue on v.
Nothing here imports the engine.
"""
import contextlib

import torch
import torch.nn.functional as F

E4M3_MAX = 448.0


def quantize_rows(y16, rounding="rn", per_tensor=False):
    """y16: [..., K] fp16. Returns (q as fp32 values of e4m3 numbers, scale fp32 [...]).
    rounding="rz" (truncation) and per_tensor=True are mutants, not the rule."""
    y = y16.to(torch.float32)
    if per_tensor:
        amax = y.abs().amax().expand(y.shape[:-1])
    else:
        amax = y.abs().amax(dim=-1)
    nz = amax > 0
    safe = torch.where(nz, amax, torch.ones_like(amax))
    # tensor / tensor: torch divides by a Python scalar as a product with its reciprocal, which is not IEEE division
    lim = torch.full_like(amax, E4M3_MAX)
    inv = torch.where(nz, lim / safe, torch.zeros_like(amax))
    x = (y * inv[..., None]).clamp(-E4M3_MAX, E4M3_MAX)            # satfinite
    if rounding == "rn":
        q = x.to(torch.float8_e4m3fn).to(torch.float32)
    else:                                                           # toward zero: the e4m3 neighbour of smaller magnitude
        q = x.to(torch.float8_e4m3fn).to(torch.float32)
        over = q.abs() > x.abs()
        q = torch.where(over, _next_toward_zero(q), q)
    return q, torch.where(nz, amax / lim, torch.ones_like(amax))


def _next_toward_zero(q):
    """The e4m3 value one step closer to zero than q (q != 0, an e4m3 value held in fp32)."""
    bits = q.to(torch.float8_e4m3fn).view(torch.uint8).to(torch.int16)
    mag = (bits & 0x7F) - 1
    return ((bits & 0x80) | mag).to(torch.uint8).view(torch.float8_e4m3fn).to(torch.float32)


def scaled_acc(q_a, s_a, q_w, s_w, scale_after_bias=None):
    """(q_a @ q_w^T) in float64 (exact for e4m3 operands at these K), then (acc * s_a[m]) * s_w[n] in fp32.
    scale_after_bias: a bias [N] to add BEFORE the scales (mutant); the result then already holds it."""
    acc = q_a.double() @ q_w.double().T
    if scale_after_bias is not None:
        return ((acc.float() + scale_after_bias.float()) * s_a[:, None]) * s_w[None, :]
    return (acc.float() * s_a[:, None]) * s_w[None, :]


def epilogue(v, bias=None, residual=None, geglu_bn=0):
    """The fp16 epilogue of the GEMM on v [M, N] fp32: fp16(v + bias); GEGLU over bn-wide interleaved tiles
    [value bn/2 | gate bn/2] -> fp16(h) * fp16(gelu(fp16(g))); fp16(out + residual)."""
    if bias is not None:
        v = v + bias.float()[None, :]
    v = v.half()
    if geglu_bn:
        M, N = v.shape
        t = v.view(M, N // geglu_bn, 2, geglu_bn // 2)
        h, g = t[:, :, 0].reshape(M, -1), t[:, :, 1].reshape(M, -1)
        v = (h.float() * F.gelu(g.float()).half().float()).half()
    if residual is not None:
        v = (v.float() + residual.float()).half()
    return v


def linear16(x, w, b=None):
    """The quantized nn.Linear at the reference's fp16 rounding point: fp16 input rows and weight rows quantized by the
    rule, the product of the exact e4m3 values in fp32 (TF32 off, autocast off), the scales, then fp16(v + b)."""
    lead = x.shape[:-1]
    q_a, s_a = quantize_rows(x.reshape(-1, x.shape[-1]).half())
    q_w, s_w = quantize_rows(w.half())
    with torch.autocast("cuda", enabled=False), torch.autocast("cpu", enabled=False):
        acc = q_a @ q_w.T
        v = (acc * s_a[:, None]) * s_w[None, :]
        if b is not None:
            v = v + b.float()[None, :]
    return v.half().reshape(*lead, -1)


def transformer_block(R, sd, p, x, enc, heads, ip_tokens, garment_features, idx, collect, ip_scale=1.0):
    """R.transformer_block (oracle/unet_ref.py) with attn1's Q/K/V of the block's own tokens, attn2.to_q and the GEGLU
    projection quantized; the garment tokens' K/V (fp16 in the engine), the text / image K/V, the out-projections and FF2
    stay as the oracle computes them."""
    n_tok = x.shape[-2]
    n1 = F.layer_norm(x, (x.shape[-1],), sd[f"{p}.norm1.weight"], sd[f"{p}.norm1.bias"], 1e-5)
    a1 = f"{p}.attn1"
    if collect is not None:
        collect.append(n1)
        mod = n1
    else:
        mod = torch.cat([n1, garment_features[idx].to(n1.dtype)], dim=1)
        idx += 1

    def qkv(name):
        own = linear16(n1, sd[f"{a1}.{name}.weight"])
        if mod.shape[1] == n_tok:
            return own
        rest = F.linear(mod[:, n_tok:], sd[f"{a1}.{name}.weight"])
        return torch.cat([own, rest.to(own.dtype)], dim=1)

    q, k, v = qkv("to_q"), qkv("to_k"), qkv("to_v")
    o = R._sdpa(q, k, v, heads)
    a = F.linear(o, sd[f"{a1}.to_out.0.weight"], sd[f"{a1}.to_out.0.bias"])
    x = a[:, :n_tok, :] + x
    n2 = F.layer_norm(x, (x.shape[-1],), sd[f"{p}.norm2.weight"], sd[f"{p}.norm2.bias"], 1e-5)
    a2 = f"{p}.attn2"
    q2 = linear16(n2, sd[f"{a2}.to_q.weight"])
    e = enc
    if ip_tokens:
        end = enc.shape[1] - ip_tokens
        e, ip = enc[:, :end], enc[:, end:]
    o = R._sdpa(q2, F.linear(e, sd[f"{a2}.to_k.weight"]), F.linear(e, sd[f"{a2}.to_v.weight"]), heads)
    if ip_tokens:
        o_ip = R._sdpa(q2, F.linear(ip, sd[f"{a2}.processor.to_k_ip.weight"]),
                       F.linear(ip, sd[f"{a2}.processor.to_v_ip.weight"]), heads)
        o = o + ip_scale * o_ip
    x = F.linear(o, sd[f"{a2}.to_out.0.weight"], sd[f"{a2}.to_out.0.bias"]) + x
    n3 = F.layer_norm(x, (x.shape[-1],), sd[f"{p}.norm3.weight"], sd[f"{p}.norm3.bias"], 1e-5)
    h = linear16(n3, sd[f"{p}.ff.net.0.proj.weight"], sd[f"{p}.ff.net.0.proj.bias"])
    h, gate = h.chunk(2, dim=-1)
    h = h * F.gelu(gate)
    x = F.linear(h, sd[f"{p}.ff.net.2.weight"], sd[f"{p}.ff.net.2.bias"]) + x
    return x, idx


@contextlib.contextmanager
def quantized_linears(R):
    """Within the block, oracle/unet_ref.py evaluates its transformer blocks with the quantized linears (ref8_16 when run
    under fp16 autocast). The module is restored on exit."""
    orig = R.transformer_block
    R.transformer_block = lambda *a, **k: transformer_block(R, *a, **k)
    try:
        yield
    finally:
        R.transformer_block = orig
