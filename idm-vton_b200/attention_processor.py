"""Seam B3 (SURVEY.md 8b): the diffusers attention-processor protocol on the engine's kernels.

Mirrors, name for name, the two processor classes the IDM-VTON inference path installs and the `Attention` container
they are called with:

  * `AttnProcessor2_0`    — ip_adapter/attention_processor.py:189-278 (self-attention of every block, and the garment
                            UNet's cross-attention)
  * `IPAttnProcessor2_0`  — ip_adapter/attention_processor.py:1879-2010 (try-on cross-attention: text keys + the last
                            `num_tokens` IP-Adapter image tokens through the processor's own `to_k_ip` / `to_v_ip`,
                            two softmaxes, `hidden + scale * ip_hidden`)
  * `Attention`           — the weight container diffusers 0.25.0 passes as `attn` (`to_q`, `to_k`, `to_v`, `to_out[0]`,
                            `heads`, `set_processor` / `get_processor`), restated for the SDXL configuration only.

Protocol: `processor(attn, hidden_states[B,T,C], encoder_hidden_states=None, attention_mask=None, temb=None, scale=1.0)
-> [B,T,C]`. All math runs in libb200vton.so (`b200vton_gemm_f16`, `b200vton_attention`, `b200vton_cross_attention`);
tensors must be CUDA fp16 and the cases the IDM-VTON UNets never produce (attention masks, spatial / group norm inside
the Attention module, 4-D inputs, head_dim != 64) raise instead of falling back to PyTorch.

The fused engine (engine.UNetEngine) implements exactly the semantics of these two classes inside its launch sequence
(fused QKV GEMM, garment K/V as a second segment, zero-K/V closed form); `unet.UNet2DConditionModel.set_attn_processor`
therefore accepts these classes only, takes the IP weights and `scale` from the installed processors, and
`tests/test_seams_gpu.py` checks the protocol path against the fused path and against the reference's own processors.
"""
import torch
import torch.nn as nn


def _lib():
    from . import lib
    lib.load()
    return lib


def _check_inputs(attn, hidden_states, attention_mask, who):
    if getattr(attn, "spatial_norm", None) is not None or getattr(attn, "group_norm", None) is not None:
        raise NotImplementedError(f"{who}: spatial_norm / group_norm inside Attention is not on the IDM-VTON path")
    if attention_mask is not None:
        raise NotImplementedError(f"{who}: attention masks are not on the IDM-VTON path (the reference passes None)")
    if hidden_states.ndim != 3:
        raise NotImplementedError(f"{who}: expects token-major [B, T, C] hidden states")
    if not hidden_states.is_cuda or hidden_states.dtype != torch.float16:
        raise RuntimeError(f"{who}: the engine's kernels need CUDA fp16 tensors (got {hidden_states.dtype} on "
                           f"{hidden_states.device}); there is no PyTorch fallback")
    if getattr(attn, "norm_cross", None):
        raise NotImplementedError(f"{who}: norm_cross is not on the IDM-VTON path")


def _w(linear):
    w = linear.weight
    if w.dtype != torch.float16 or not w.is_cuda:
        raise RuntimeError("attention weights must be CUDA fp16")
    return w


def _out_proj(L, attn, o, residual):
    """to_out[0] (+bias) -> dropout(p=0) -> optional residual -> / rescale_output_factor (:267-276)."""
    lin = attn.to_out[0]
    B, T, C = o.shape
    res = None
    if getattr(attn, "residual_connection", False):
        res = residual.reshape(B * T, -1)
    y = L.gemm(o.reshape(B * T, C), _w(lin), bias=getattr(lin, "bias", None), residual=res).view(B, T, -1)
    f = float(getattr(attn, "rescale_output_factor", 1.0))
    if f != 1.0:
        y = y / f
    return y


class AttnProcessor2_0(nn.Module):
    """Scaled-dot-product attention processor (ip_adapter/attention_processor.py:189-278) on `b200vton_attention`."""

    def __init__(self, hidden_size=None, cross_attention_dim=None):
        super().__init__()

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None, scale=1.0):
        _check_inputs(attn, hidden_states, attention_mask, "AttnProcessor2_0")
        L = _lib()
        B, T, C = hidden_states.shape
        x = hidden_states.contiguous().view(B * T, C)
        wq, wk, wv = _w(attn.to_q), _w(attn.to_k), _w(attn.to_v)
        inner = wq.shape[0]
        heads = attn.heads
        if inner != heads * 64:
            raise NotImplementedError("AttnProcessor2_0: head_dim must be 64")
        if encoder_hidden_states is None:
            # self-attention: one fused [3*inner, C] projection (cached per weight version), q/k/v are column views
            key = (wq.data_ptr(), wq._version, wk.data_ptr(), wk._version, wv.data_ptr(), wv._version)
            cache = getattr(attn, "_b200_wqkv", None)
            if cache is None or cache[0] != key:
                cache = (key, torch.cat([wq, wk, wv], 0).contiguous())
                attn._b200_wqkv = cache
            qkv = L.gemm(x, cache[1]).view(B, T, 3 * inner)
            q, k, v = qkv[..., :inner], qkv[..., inner:2 * inner], qkv[..., 2 * inner:]
        else:
            e = encoder_hidden_states
            if not e.is_cuda or e.dtype != torch.float16:
                raise RuntimeError("AttnProcessor2_0: encoder_hidden_states must be CUDA fp16")
            Te = e.shape[1]
            e2 = e.contiguous().view(B * Te, -1)
            q = L.gemm(x, wq).view(B, T, inner)
            k = L.gemm(e2, wk).view(B, Te, inner)
            v = L.gemm(e2, wv).view(B, Te, inner)
        o = L.attention(q, k, v, heads=heads)
        return _out_proj(L, attn, o, hidden_states)


class IPAttnProcessor2_0(nn.Module):
    """IP-Adapter decoupled cross-attention (ip_adapter/attention_processor.py:1879-2010) on `b200vton_cross_attention`:
    text keys and the last `num_tokens` image tokens of `encoder_hidden_states` in ONE launch, two independent
    softmaxes, `fp16(o_text) + fp16(scale * fp16(o_ip))`. Owns `to_k_ip` / `to_v_ip` (state-dict keys
    `...attn2.processor.to_k_ip.weight`, :1904-1905). The reference also stores `self.attn_map` (:1989-1990), a tensor
    nothing ever reads (and whose formula applies the softmax to K^T before the product); it is not materialised."""

    def __init__(self, hidden_size, cross_attention_dim=None, scale=1.0, num_tokens=4, device=None, dtype=None):
        super().__init__()
        self.hidden_size = hidden_size
        self.cross_attention_dim = cross_attention_dim
        self.scale = scale
        self.num_tokens = num_tokens
        self.to_k_ip = nn.Linear(cross_attention_dim or hidden_size, hidden_size, bias=False, device=device, dtype=dtype)
        self.to_v_ip = nn.Linear(cross_attention_dim or hidden_size, hidden_size, bias=False, device=device, dtype=dtype)

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None, scale=1.0):
        _check_inputs(attn, hidden_states, attention_mask, "IPAttnProcessor2_0")
        if encoder_hidden_states is None:
            # the reference would fail here too (ip_hidden_states undefined, :1976): this processor is cross-attention only
            raise ValueError("IPAttnProcessor2_0 needs encoder_hidden_states (text tokens followed by the IP tokens)")
        L = _lib()
        B, T, C = hidden_states.shape
        e = encoder_hidden_states
        if not e.is_cuda or e.dtype != torch.float16:
            raise RuntimeError("IPAttnProcessor2_0: encoder_hidden_states must be CUDA fp16")
        end_pos = e.shape[1] - self.num_tokens                                                      # :1949-1953
        txt = e[:, :end_pos, :].contiguous().view(B * end_pos, -1)
        ip = e[:, end_pos:, :].contiguous().view(B * self.num_tokens, -1)
        wq = _w(attn.to_q)
        inner = wq.shape[0]
        heads = attn.heads
        if inner != heads * 64:
            raise NotImplementedError("IPAttnProcessor2_0: head_dim must be 64")
        q = L.gemm(hidden_states.contiguous().view(B * T, C), wq).view(B, T, inner)
        kt = L.gemm(txt, _w(attn.to_k)).view(B, end_pos, inner)
        vt = L.gemm(txt, _w(attn.to_v)).view(B, end_pos, inner)
        ki = L.gemm(ip, _w(self.to_k_ip)).view(B, self.num_tokens, inner)
        vi = L.gemm(ip, _w(self.to_v_ip)).view(B, self.num_tokens, inner)
        if end_pos <= 80 and self.num_tokens <= 16:
            o = L.cross_attention(q, kt, vt, ki, vi, heads=heads, ip_scale=float(self.scale))
        else:
            if float(self.scale) != 1.0:
                raise NotImplementedError("IPAttnProcessor2_0: scale != 1 needs the fused kernel (<= 80 text, <= 16 IP tokens)")
            o = L.attention(q, kt, vt, heads=heads)
            L.attention(q, ki, vi, heads=heads, accumulate=True, out=o)
        return _out_proj(L, attn, o, hidden_states)


class _Weight(nn.Module):
    """A bias-free / biased linear's parameters under the reference's names (`.weight`, `.bias`)."""

    def __init__(self, out_f, in_f, bias, device=None, dtype=None):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(out_f, in_f, device=device, dtype=dtype), requires_grad=False)
        self.bias = nn.Parameter(torch.empty(out_f, device=device, dtype=dtype), requires_grad=False) if bias else None
        self.in_features, self.out_features = in_f, out_f

    def forward(self, x):
        L = _lib()
        shp = x.shape
        return L.gemm(x.reshape(-1, shp[-1]).contiguous(), self.weight, bias=self.bias).view(*shp[:-1], self.out_features)


class Attention(nn.Module):
    """diffusers 0.25.0 `Attention` as the SDXL UNets construct it (src/attentionhacked_tryon.py:201-210,231-240:
    `bias=False`, `out_bias=True`, `dim_head=64`, no norms): weights + processor dispatch."""

    def __init__(self, query_dim=None, cross_attention_dim=None, heads=8, dim_head=64, dropout=0.0, bias=False,
                 out_bias=True, processor=None, device=None, dtype=None, _empty=False):
        """`_empty=True` (used by the UNet facades): only the attributes; the weight children (`to_q.weight`, ...,
        `to_out.0.{weight,bias}`) are registered afterwards under the reference's state-dict names."""
        super().__init__()
        if dim_head != 64 or bias:
            raise NotImplementedError("the engine's attention kernels cover dim_head=64, bias-free q/k/v projections")
        self.inner_dim = dim_head * heads
        self.cross_attention_dim = cross_attention_dim if cross_attention_dim is not None else query_dim
        self.heads = heads
        self.scale = dim_head ** -0.5
        self.rescale_output_factor = 1.0
        self.residual_connection = False
        self.spatial_norm = self.group_norm = self.norm_cross = None
        if _empty:
            return
        self.to_q = _Weight(self.inner_dim, query_dim, False, device, dtype)
        self.to_k = _Weight(self.inner_dim, self.cross_attention_dim, False, device, dtype)
        self.to_v = _Weight(self.inner_dim, self.cross_attention_dim, False, device, dtype)
        self.to_out = nn.ModuleList([_Weight(query_dim, self.inner_dim, out_bias, device, dtype), nn.Dropout(dropout)])
        self.set_processor(processor if processor is not None else AttnProcessor2_0())

    def set_processor(self, processor, _remove_lora=False):
        if "processor" in self._modules and not isinstance(processor, nn.Module):
            self._modules.pop("processor")
        self.processor = processor

    def get_processor(self, return_deprecated_lora=False):
        return self.processor

    def forward(self, hidden_states, encoder_hidden_states=None, attention_mask=None, **cross_attention_kwargs):
        return self.processor(self, hidden_states, encoder_hidden_states=encoder_hidden_states,
                              attention_mask=attention_mask, **cross_attention_kwargs)
