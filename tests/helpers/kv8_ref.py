"""The FP8 garment K/V rule (include/b200vton.h, b200vton_quantize_kv_e4m3), restated in torch for the tests.

K/V [rows, Ng, 2C] fp16 are split into groups of 64 columns (group g < H: head g of K, group H + g: head g of V). Per
token and group: amax = max |x| in fp32; e = 0 when amax == 0, else the smallest integer with amax <= 448 * 2^e,
clamped to e >= -24; q = e4m3_rn(x * 2^-e); the dequantized value is fp16_rn(float(q) * 2^e).
"""
import torch

GROUP = 64
E_MIN = -24


def exponents(amax):
    """e of each fp32 amax, from frexp: amax = m * 2^k with m in [0.5, 1), i.e. 1.f * 2^(k - 1) with 1.f = 2m."""
    m, k = torch.frexp(amax.to(torch.float32))
    E = k.to(torch.int32) - 1
    e = torch.where(2 * m <= 1.75, E - 8, E - 7).clamp(min=E_MIN)
    return torch.where(amax == 0, torch.zeros_like(e), e)


def quantize(kv, heads):
    """kv [rows, Ng, 2C] fp16 -> (q [rows, Ng, 2C] e4m3, e [rows, 2H, Ng] int32)."""
    rows, ng, c2 = kv.shape
    assert c2 == 2 * heads * GROUP
    x = kv.to(torch.float32).reshape(rows, ng, 2 * heads, GROUP)
    e = exponents(x.abs().amax(dim=-1))                                   # [rows, Ng, 2H]
    q = (x * torch.exp2(-e.to(torch.float32))[..., None]).to(torch.float8_e4m3fn).reshape(rows, ng, c2)
    return q, e.permute(0, 2, 1).contiguous()


def dequantize(q, e):
    """(q [rows, Ng, 2C] e4m3, e [rows, 2H, >= Ng]) -> fp16 [rows, Ng, 2C] by the rule."""
    rows, ng, c2 = q.shape
    g = c2 // GROUP
    s = torch.exp2(e[:, :, :ng].to(torch.float32)).permute(0, 2, 1)     # [rows, Ng, 2H]
    return (q.to(torch.float32).reshape(rows, ng, g, GROUP) * s[..., None]).reshape(rows, ng, c2).to(torch.float16)


def roundtrip(kv, heads):
    """The fp16 K/V the kernels see in place of kv."""
    return dequantize(*quantize(kv, heads))


def transformer_block(R, sd, p, x, enc, heads, ip_tokens, garment_features, idx, collect, ip_scale=1.0):
    """oracle/unet_ref.py's transformer_block with the garment tokens' K/V of attn1 passed through the rule (the try-on
    variant; the garment variant is unchanged). Under fp16 autocast the K/V are the fp16 projections the engine
    quantizes."""
    if collect is not None:
        return _ORIG[id(R)](sd, p, x, enc, heads, ip_tokens, garment_features, idx, collect, ip_scale)
    F = torch.nn.functional
    n1 = F.layer_norm(x, (x.shape[-1],), sd[f"{p}.norm1.weight"], sd[f"{p}.norm1.bias"], 1e-5)
    mod = torch.cat([n1, garment_features[idx].to(n1.dtype)], dim=1)
    idx += 1
    a1 = f"{p}.attn1"
    n = x.shape[-2]
    q = F.linear(mod, sd[f"{a1}.to_q.weight"])
    k = F.linear(mod, sd[f"{a1}.to_k.weight"])
    v = F.linear(mod, sd[f"{a1}.to_v.weight"])
    C = k.shape[-1]
    kv = roundtrip(torch.cat([k[:, n:], v[:, n:]], dim=-1).to(torch.float16), heads).to(k.dtype)
    k = torch.cat([k[:, :n], kv[..., :C]], dim=1)
    v = torch.cat([v[:, :n], kv[..., C:]], dim=1)
    a = F.linear(R._sdpa(q, k, v, heads), sd[f"{a1}.to_out.0.weight"], sd[f"{a1}.to_out.0.bias"])
    x = a[:, :n, :] + x
    n2 = F.layer_norm(x, (x.shape[-1],), sd[f"{p}.norm2.weight"], sd[f"{p}.norm2.bias"], 1e-5)
    x = R.attn_cross(sd, f"{p}.attn2", n2, enc, heads, ip_tokens, ip_scale) + x
    n3 = F.layer_norm(x, (x.shape[-1],), sd[f"{p}.norm3.weight"], sd[f"{p}.norm3.bias"], 1e-5)
    x = R.feed_forward(sd, f"{p}.ff", n3) + x
    return x, idx


_ORIG = {}


class quantized_garment_kv:
    """Within the block, oracle/unet_ref.py evaluates its try-on transformer blocks with the garment K/V quantized and
    dequantized by the rule (refkv8_16 when run under fp16 autocast). The module is restored on exit."""

    def __init__(self, R):
        self.R = R

    def __enter__(self):
        _ORIG[id(self.R)] = self.R.transformer_block
        self.R.transformer_block = lambda *a, **k: transformer_block(self.R, *a, **k)

    def __exit__(self, *exc):
        self.R.transformer_block = _ORIG.pop(id(self.R))
