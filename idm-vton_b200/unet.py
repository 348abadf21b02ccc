"""Host-side mirrors of the reference's two `UNet2DConditionModel` classes (seam B2 of SURVEY.md 8b).

  * same constructor-visible attributes the pipeline reads: `.config.{in_channels,time_cond_proj_dim,sample_size,
    addition_time_embed_dim,...}`, `.add_embedding.linear_1.in_features`, `.encoder_hid_proj(x)`, `.dtype`, `.device`
    (src/tryon_pipeline.py:493,1049,1606,1726,1755);
  * same parameter names, so `load_state_dict` ingests the reference checkpoints (SURVEY.md App. D.7);
  * same forward signatures: try-on `forward(sample, timestep, encoder_hidden_states, ..., added_cond_kwargs,
    return_dict, garment_features)` -> `(noise_pred,)` (src/unet_hacked_tryon.py:1006-1022); garment
    `forward(sample, timestep, encoder_hidden_states, return_dict)` -> `((sample,), garment_features)`
    (src/unet_hacked_garmnet.py:917-931,1281-1284).
All math runs in libb200vton.so through engine.UNetEngine; a missing library raises (no PyTorch fallback).
"""
import types

import torch
import torch.nn as nn

from .attention_processor import Attention, AttnProcessor2_0, IPAttnProcessor2_0
from .engine import CIN_PAD, SDXL_GARMENT, SDXL_TRYON, UNetEngine


# ------------------------------------------------------------------------------------------------
# parameter inventory (reference state-dict key names)
# ------------------------------------------------------------------------------------------------
def _resnet(p, cin, cout, temb):
    yield f"{p}.norm1.weight", (cin,)
    yield f"{p}.norm1.bias", (cin,)
    yield f"{p}.conv1.weight", (cout, cin, 3, 3)
    yield f"{p}.conv1.bias", (cout,)
    yield f"{p}.time_emb_proj.weight", (cout, temb)
    yield f"{p}.time_emb_proj.bias", (cout,)
    yield f"{p}.norm2.weight", (cout,)
    yield f"{p}.norm2.bias", (cout,)
    yield f"{p}.conv2.weight", (cout, cout, 3, 3)
    yield f"{p}.conv2.bias", (cout,)
    if cin != cout:
        yield f"{p}.conv_shortcut.weight", (cout, cin, 1, 1)
        yield f"{p}.conv_shortcut.bias", (cout,)


def _t2d(p, c, layers, cross, ip):
    for n, s in (("norm.weight", (c,)), ("norm.bias", (c,)), ("proj_in.weight", (c, c)), ("proj_in.bias", (c,))):
        yield f"{p}.{n}", s
    for k in range(layers):
        b = f"{p}.transformer_blocks.{k}"
        yield f"{b}.norm1.weight", (c,)
        yield f"{b}.norm1.bias", (c,)
        yield f"{b}.attn1.to_q.weight", (c, c)
        yield f"{b}.attn1.to_k.weight", (c, c)
        yield f"{b}.attn1.to_v.weight", (c, c)
        yield f"{b}.attn1.to_out.0.weight", (c, c)
        yield f"{b}.attn1.to_out.0.bias", (c,)
        yield f"{b}.norm2.weight", (c,)
        yield f"{b}.norm2.bias", (c,)
        yield f"{b}.attn2.to_q.weight", (c, c)
        yield f"{b}.attn2.to_k.weight", (c, cross)
        yield f"{b}.attn2.to_v.weight", (c, cross)
        yield f"{b}.attn2.to_out.0.weight", (c, c)
        yield f"{b}.attn2.to_out.0.bias", (c,)
        if ip:
            yield f"{b}.attn2.processor.to_k_ip.weight", (c, cross)
            yield f"{b}.attn2.processor.to_v_ip.weight", (c, cross)
        yield f"{b}.norm3.weight", (c,)
        yield f"{b}.norm3.bias", (c,)
        yield f"{b}.ff.net.0.proj.weight", (8 * c, c)
        yield f"{b}.ff.net.0.proj.bias", (8 * c,)
        yield f"{b}.ff.net.2.weight", (c, 4 * c)
        yield f"{b}.ff.net.2.bias", (c,)
    yield f"{p}.proj_out.weight", (c, c)
    yield f"{p}.proj_out.bias", (c,)


def _resampler(p, r):
    d, inner = r["dim"], r["dim_head"] * r["heads"]
    yield f"{p}.latents", (1, r["num_queries"], d)
    yield f"{p}.proj_in.weight", (d, r["embedding_dim"])
    yield f"{p}.proj_in.bias", (d,)
    yield f"{p}.proj_out.weight", (r["output_dim"], d)
    yield f"{p}.proj_out.bias", (r["output_dim"],)
    yield f"{p}.norm_out.weight", (r["output_dim"],)
    yield f"{p}.norm_out.bias", (r["output_dim"],)
    for i in range(r["depth"]):
        a, f = f"{p}.layers.{i}.0", f"{p}.layers.{i}.1"
        for n in ("norm1", "norm2"):
            yield f"{a}.{n}.weight", (d,)
            yield f"{a}.{n}.bias", (d,)
        yield f"{a}.to_q.weight", (inner, d)
        yield f"{a}.to_kv.weight", (2 * inner, d)
        yield f"{a}.to_out.weight", (d, inner)
        yield f"{f}.0.weight", (d,)
        yield f"{f}.0.bias", (d,)
        yield f"{f}.1.weight", (d * r["ff_mult"], d)
        yield f"{f}.3.weight", (d, d * r["ff_mult"])


def param_shapes(cfg):
    """{key: shape} for a UNet with this config, in the reference modules' naming."""
    ch = tuple(cfg["block_out_channels"])
    temb, cross, tl = ch[0] * 4, cfg["cross_attention_dim"], cfg["transformer_layers_per_block"]
    ip = cfg["ip_tokens"] > 0
    n = len(ch)
    out = {"conv_in.weight": (ch[0], cfg["in_channels"], 3, 3), "conv_in.bias": (ch[0],)}
    for i, (a, b) in enumerate(((ch[0], temb), (temb, temb)), start=1):
        out[f"time_embedding.linear_{i}.weight"] = (b, a)
        out[f"time_embedding.linear_{i}.bias"] = (b,)
    if cfg["text_time"]:
        for i, (a, b) in enumerate(((cfg["projection_class_embeddings_input_dim"], temb), (temb, temb)), start=1):
            out[f"add_embedding.linear_{i}.weight"] = (b, a)
            out[f"add_embedding.linear_{i}.bias"] = (b,)
    if cfg.get("resampler"):
        out.update(_resampler("encoder_hid_proj", cfg["resampler"]))
    prev = ch[0]
    for i, c in enumerate(ch):
        for j in range(cfg["layers_per_block"]):
            out.update(_resnet(f"down_blocks.{i}.resnets.{j}", prev if j == 0 else c, c, temb))
            if i > 0:
                out.update(_t2d(f"down_blocks.{i}.attentions.{j}", c, tl[i], cross, ip))
        if i < n - 1:
            out[f"down_blocks.{i}.downsamplers.0.conv.weight"] = (c, c, 3, 3)
            out[f"down_blocks.{i}.downsamplers.0.conv.bias"] = (c,)
        prev = c
    out.update(_resnet("mid_block.resnets.0", ch[-1], ch[-1], temb))
    out.update(_t2d("mid_block.attentions.0", ch[-1], tl[-1], cross, ip))
    out.update(_resnet("mid_block.resnets.1", ch[-1], ch[-1], temb))
    rch, rtl = ch[::-1], tuple(tl)[::-1]
    prev_out = rch[0]
    for i, c in enumerate(rch):
        skip_in = rch[min(i + 1, n - 1)]
        layers = cfg["layers_per_block"] + 1
        for j in range(layers):
            skip = skip_in if j == layers - 1 else c
            rin = prev_out if j == 0 else c
            out.update(_resnet(f"up_blocks.{i}.resnets.{j}", rin + skip, c, temb))
            if i < n - 1:
                out.update(_t2d(f"up_blocks.{i}.attentions.{j}", c, rtl[i], cross, ip))
        if i < n - 1:
            out[f"up_blocks.{i}.upsamplers.0.conv.weight"] = (c, c, 3, 3)
            out[f"up_blocks.{i}.upsamplers.0.conv.bias"] = (c,)
        prev_out = c
    out["conv_norm_out.weight"] = (ch[0],)
    out["conv_norm_out.bias"] = (ch[0],)
    out["conv_out.weight"] = (cfg["out_channels"], ch[0], 3, 3)
    out["conv_out.bias"] = (cfg["out_channels"],)
    return out


def random_state_dict(cfg, seed=0, device="cuda", dtype=torch.float16, residual_gain=0.25):
    """Seeded synthetic weights generated on `device` (the reference's ckpt/** are empty placeholders): uniform
    +-sqrt(3/fan_in) matrices, norm affine ~ (1 +- 0.1, +-0.1), residual-branch output layers scaled by
    `residual_gain` so the 70-block residual stream stays inside fp16 range."""
    g = torch.Generator(device=device).manual_seed(seed)
    sd = {}
    for k, shp in param_shapes(cfg).items():
        if len(shp) == 1 or k.endswith("latents"):
            is_norm = ".norm" in k or k.startswith("conv_norm_out") or (".layers." in k and k.split(".")[-2] == "0")
            w = torch.randn(shp, generator=g, device=device, dtype=torch.float32)
            if k.endswith("latents"):
                w = w / shp[-1] ** 0.5
            elif is_norm and k.endswith("weight"):
                w = 1.0 + 0.1 * w
            else:
                w = (0.1 if is_norm else 0.05) * w
        else:
            fan_in = 1
            for d in shp[1:]:
                fan_in *= d
            w = (torch.rand(shp, generator=g, device=device, dtype=torch.float32) * 2 - 1) * (3.0 / fan_in) ** 0.5
            if not k.startswith("encoder_hid_proj") and any(
                    t in k for t in ("to_out.0.weight", "ff.net.2.weight", "conv2.weight", "proj_out.weight")):
                w = w * residual_gain
        sd[k] = w.to(dtype)
    return sd


# ------------------------------------------------------------------------------------------------
# Resampler on the engine's kernels (ip_adapter/resampler.py:129-176)
# ------------------------------------------------------------------------------------------------
def resampler_forward(L, sd, p, r, x):
    """x: [B, T, embedding_dim] fp16 CLIP penultimate tokens -> [B, num_queries, output_dim]. PerceiverAttention's
    `cat((x, latents))` K/V is the attention kernel's two-segment stream (segment 0 = image tokens, 1 = latents)."""
    B, T, _ = x.shape
    d, heads, nq = r["dim"], r["heads"], r["num_queries"]
    f16 = torch.float16
    xx = L.gemm(x.reshape(B * T, -1).to(f16).contiguous(), sd[f"{p}.proj_in.weight"], bias=sd[f"{p}.proj_in.bias"])
    lat = sd[f"{p}.latents"].to(f16).repeat(B, 1, 1).reshape(B * nq, d).contiguous()
    inner = heads * r["dim_head"]
    for i in range(r["depth"]):
        a, f = f"{p}.layers.{i}.0", f"{p}.layers.{i}.1"
        xn = L.layernorm(xx, sd[f"{a}.norm1.weight"], sd[f"{a}.norm1.bias"])
        ln = L.layernorm(lat, sd[f"{a}.norm2.weight"], sd[f"{a}.norm2.bias"])
        q = L.gemm(ln, sd[f"{a}.to_q.weight"]).view(B, nq, inner)
        kv_x = L.gemm(xn, sd[f"{a}.to_kv.weight"]).view(B, T, 2 * inner)
        kv_l = L.gemm(ln, sd[f"{a}.to_kv.weight"]).view(B, nq, 2 * inner)
        o = L.attention(q, kv_x[..., :inner], kv_x[..., inner:], kv_l[..., :inner], kv_l[..., inner:], kv1_off=0,
                        heads=heads, scale=r["dim_head"] ** -0.5)
        lat = L.gemm(o.view(B * nq, inner), sd[f"{a}.to_out.weight"], residual=lat)
        h = L.layernorm(lat, sd[f"{f}.0.weight"], sd[f"{f}.0.bias"])
        h = L.gemm(h, sd[f"{f}.1.weight"], gelu=True)
        lat = L.gemm(h, sd[f"{f}.3.weight"], residual=lat)
    out = L.gemm(lat, sd[f"{p}.proj_out.weight"], bias=sd[f"{p}.proj_out.bias"])
    out = L.layernorm(out, sd[f"{p}.norm_out.weight"], sd[f"{p}.norm_out.bias"])
    return out.view(B, nq, r["output_dim"])


# ------------------------------------------------------------------------------------------------
# nn.Module facades
# ------------------------------------------------------------------------------------------------
class _Node(nn.Module):
    """Anonymous container so parameters can carry the reference's dotted names."""

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("container module")

    def __getitem__(self, i):          # `attn.to_out[0]` (a ModuleList in the reference)
        return self._modules[str(i)]


def _heads_of(cfg, key):
    """Attention heads of the block a parameter name belongs to (attention_head_dim per level, App. A)."""
    nh = tuple(cfg["num_heads"])
    if key.startswith("mid_block"):
        return nh[-1]
    if key.startswith("up_blocks."):
        return nh[::-1][int(key.split(".")[1])]
    return nh[int(key.split(".")[1])]


def _register(root, key, tensor, cfg=None):
    """Registers `tensor` under the reference's dotted parameter name. Path components `attn1` / `attn2` become
    `Attention` containers (seam B3) and `attn2.processor` an `IPAttnProcessor2_0` owning `to_k_ip` / `to_v_ip`."""
    parts = key.split(".")
    m = root
    for d, name in enumerate(parts[:-1]):
        if name not in m._modules:
            if name in ("attn1", "attn2") and cfg is not None and "transformer_blocks" in parts:
                child = Attention(heads=_heads_of(cfg, key), _empty=True)
            elif name == "processor" and isinstance(m, Attention):
                child = IPAttnProcessor2_0(hidden_size=tensor.shape[0], cross_attention_dim=tensor.shape[1], scale=1.0,
                                           num_tokens=cfg["ip_tokens"], device="meta")
            else:
                child = _Node()
            m.add_module(name, child)
        m = m._modules[name]
    m.register_parameter(parts[-1], nn.Parameter(tensor, requires_grad=False))


class _ResamplerProxy(_Node):
    """`unet.encoder_hid_proj(image_embeds)` (src/tryon_pipeline.py:1726) executed by the engine's kernels."""

    def forward(self, x):
        root = self._root()
        root._need_lib()
        sd = {k: v for k, v in root.state_dict().items() if k.startswith("encoder_hid_proj.")}
        return resampler_forward(root._lib, sd, "encoder_hid_proj", root._cfg["resampler"],
                                 x.to(root.device, torch.float16))


class _UNetBase(nn.Module):
    KIND = None

    def __init__(self, cfg, state_dict=None, device="cpu", dtype=torch.float16):
        super().__init__()
        self._cfg = dict(cfg)
        self._engine = None
        self._lib = None
        self._linear_precision = "fp16"
        shapes = param_shapes(cfg)
        for k, shp in shapes.items():
            if k.startswith("encoder_hid_proj.") and "encoder_hid_proj" not in self._modules:
                proxy = _ResamplerProxy()
                object.__setattr__(proxy, "_root", lambda s=self: s)
                self.add_module("encoder_hid_proj", proxy)
            t = state_dict[k].to(device=device, dtype=dtype) if state_dict is not None else torch.empty(
                shp, device=device, dtype=dtype)
            if tuple(t.shape) != tuple(shp):
                raise ValueError(f"{k}: expected shape {tuple(shp)}, got {tuple(t.shape)}")
            _register(self, k, t, self._cfg)
        for m in self.modules():
            if isinstance(m, Attention) and "processor" not in m._modules:
                m.set_processor(AttnProcessor2_0())
        if cfg["text_time"]:
            self.add_embedding.linear_1.in_features = cfg["projection_class_embeddings_input_dim"]
        ch = tuple(cfg["block_out_channels"])
        self.config = types.SimpleNamespace(
            in_channels=cfg["in_channels"], out_channels=cfg["out_channels"], block_out_channels=ch,
            cross_attention_dim=cfg["cross_attention_dim"], time_cond_proj_dim=None, sample_size=128,
            addition_time_embed_dim=cfg["addition_time_embed_dim"], center_input_sample=False,
            addition_embed_type="text_time" if cfg["text_time"] else None,
            encoder_hid_dim_type="ip_image_proj" if cfg.get("resampler") else None,
            projection_class_embeddings_input_dim=cfg["projection_class_embeddings_input_dim"])

    @property
    def dtype(self):
        return next(self.parameters()).dtype

    @property
    def device(self):
        return next(self.parameters()).device

    def _need_lib(self):
        if self._lib is None:
            from . import lib
            lib.load()
            self._lib = lib
        if self.device.type != "cuda" or self.dtype != torch.float16:
            raise RuntimeError("the engine needs the UNet on a CUDA device in fp16 "
                               f"(got {self.device}, {self.dtype}); there is no CPU / PyTorch fallback")

    def engine(self):
        """Pre-packs the weights on first use (after .to(device) / load_state_dict)."""
        self._need_lib()
        if self._engine is None:
            self._engine = UNetEngine(self._cfg, self.state_dict(), self.KIND, device=self.device,
                                      ip_scales=self._ip_scales(), fp8=self._linear_precision == "fp8")
        return self._engine

    LINEAR_PRECISIONS = ("fp16", "fp8")

    @property
    def linear_precision(self):
        return self._linear_precision

    def set_linear_precision(self, precision):
        """"fp16" (default) or "fp8": the arithmetic of the transformer blocks' per-token linears (attn1 QKV, attn2.to_q,
        the GEGLU projection), see UNetEngine(fp8=...). A change drops the packed engine; engine() re-packs."""
        if precision not in self.LINEAR_PRECISIONS:
            raise ValueError(f"linear precision must be one of {self.LINEAR_PRECISIONS}, got {precision!r}")
        if precision != self._linear_precision:
            self._linear_precision = precision
            self._engine = None

    def _apply(self, fn, *a, **k):
        self._engine = None      # weights moved / cast: re-pack lazily
        return super()._apply(fn, *a, **k)

    # ---- seam B3: the attention-processor protocol (src/unet_hacked_tryon.py:793-852) -------------------------------
    @property
    def attn_processors(self):
        """{"<attention module path>.processor": processor} for every Attention layer (src/unet_hacked_tryon.py:793-816)."""
        return {f"{name}.processor": m.get_processor() for name, m in self.named_modules() if isinstance(m, Attention)}

    def set_attn_processor(self, processor, _remove_lora=False):
        """src/unet_hacked_tryon.py:818-852: one processor for all layers, or a dict keyed like `attn_processors`.
        The fused engine implements the semantics of `AttnProcessor2_0` (self-attention; garment cross-attention) and
        `IPAttnProcessor2_0` (try-on cross-attention) of this package, so only those classes are accepted per slot;
        IP weights (`to_k_ip`, `to_v_ip`), `scale` and `num_tokens` are taken from the installed processors."""
        layers = {f"{name}.processor": m for name, m in self.named_modules() if isinstance(m, Attention)}
        count = len(layers)
        if isinstance(processor, dict) and len(processor) != count:
            raise ValueError(f"A dict of processors was passed, but the number of processors {len(processor)} does not match the"
                             f" number of attention layers: {count}. Please make sure to pass {count} processor classes.")
        ip = self._cfg["ip_tokens"] if self.KIND == "tryon" else 0
        todo = {}
        for name, attn in layers.items():
            proc = processor.pop(name) if isinstance(processor, dict) else processor
            want = IPAttnProcessor2_0 if (ip and name.endswith("attn2.processor")) else AttnProcessor2_0
            if type(proc) is not want:
                raise TypeError(f"{name}: the engine fuses {want.__name__} here (got {type(proc).__name__}); other "
                                "processors have no kernel and there is no PyTorch fallback")
            if want is IPAttnProcessor2_0:
                exp = (attn.to_q.weight.shape[0], attn.to_k.weight.shape[1])
                if tuple(proc.to_k_ip.weight.shape) != exp or tuple(proc.to_v_ip.weight.shape) != exp:
                    raise ValueError(f"{name}: to_k_ip / to_v_ip must be {exp}, got {tuple(proc.to_k_ip.weight.shape)}")
                if proc.num_tokens != ip:
                    raise ValueError(f"{name}: num_tokens {proc.num_tokens} != {ip} image tokens of this UNet")
            todo[name] = (attn, proc)
        for attn, proc in todo.values():
            attn.set_processor(proc, _remove_lora=_remove_lora)
        self._engine = None

    def _ip_scales(self):
        return {name[:-len(".attn2.processor")]: float(p.scale) for name, p in self.attn_processors.items()
                if isinstance(p, IPAttnProcessor2_0)}

    # Checkpoint keys the reference modules own but this UNet never executes. GarmentNet is the SDXL-base UNet built
    # WITH addition_embed_type="text_time" (train_xl.py:323-325 only nulls the config afterwards), so its checkpoint
    # carries add_embedding.linear_{1,2}.*, which the garment forward never reads (src/unet_hacked_garmnet.py).
    IGNORED_CHECKPOINT_PREFIXES = ()

    def load_state_dict(self, state_dict, strict=True, **k):
        self._engine = None
        drop = [key for key in state_dict if key.startswith(self.IGNORED_CHECKPOINT_PREFIXES)] \
            if self.IGNORED_CHECKPOINT_PREFIXES else []
        if drop:
            own = set(self.state_dict().keys())
            state_dict = {key: v for key, v in state_dict.items() if key in own or key not in drop}
        return super().load_state_dict(state_dict, strict=strict, **k)

    def _t_dev(self, timestep):
        if torch.is_tensor(timestep):
            return timestep.reshape(-1)[:1].to(self.device, torch.float32)
        return torch.tensor([float(timestep)], dtype=torch.float32, device=self.device)


class UNet2DConditionModel(_UNetBase):
    """Try-on UNet ("TryonNet", src/unet_hacked_tryon.py)."""
    KIND = "tryon"

    def __init__(self, cfg=None, state_dict=None, device="cpu", dtype=torch.float16):
        super().__init__(cfg or SDXL_TRYON, state_dict, device, dtype)
        self._garment_kv_precision = "fp16"
        self._freeu = None

    GARMENT_KV_PRECISIONS = ("fp16", "fp8")

    @property
    def garment_kv_precision(self):
        return self._garment_kv_precision

    def set_garment_kv_precision(self, precision):
        """"fp16" (default) or "fp8": the format the denoisers hold the hoisted garment K/V of this UNet in (e4m3 with
        one power-of-two exponent per token and head, INTEGRATION.md "FP8 garment K/V"). The weights are not re-packed;
        a denoiser allocates its garment K/V in the new format at its next prepare / configure."""
        if precision not in self.GARMENT_KV_PRECISIONS:
            raise ValueError(f"garment K/V precision must be one of {self.GARMENT_KV_PRECISIONS}, got {precision!r}")
        self._garment_kv_precision = precision
        if self._engine is not None:
            self._engine.garment_kv_format = precision

    def engine(self):
        eng = super().engine()
        eng.garment_kv_format = self._garment_kv_precision
        eng.freeu = self._freeu
        return eng

    @property
    def freeu(self):
        """(s1, s2, b1, b2) set by enable_freeu, or None."""
        return self._freeu

    def enable_freeu(self, s1, s2, b1, b2):
        """FreeU (https://arxiv.org/abs/2309.11497, src/unet_hacked_tryon.py:938-959): before every resnet of up stage 0
        the first half of the backbone channels is scaled by b1 and the skip feature's lowest frequencies by s1
        (stage 1: b2, s2). As in the reference, FreeU runs only while all four values are non-zero. The weights are not
        re-packed; a captured denoise step is re-captured at its next run."""
        self._freeu = tuple(None if v is None else float(v) for v in (s1, s2, b1, b2))
        if self._engine is not None:
            self._engine.freeu = self._freeu

    def disable_freeu(self):
        """Switches FreeU off (src/unet_hacked_tryon.py:961-967)."""
        self._freeu = None
        if self._engine is not None:
            self._engine.freeu = None

    @torch.no_grad()
    def forward(self, sample, timestep, encoder_hidden_states, class_labels=None, timestep_cond=None,
                attention_mask=None, cross_attention_kwargs=None, added_cond_kwargs=None,
                down_block_additional_residuals=None, mid_block_additional_residual=None,
                down_intrablock_additional_residuals=None, encoder_attention_mask=None, return_dict=True,
                garment_features=None):
        if any(v is not None for v in (class_labels, timestep_cond, attention_mask, down_block_additional_residuals,
                                       mid_block_additional_residual, down_intrablock_additional_residuals,
                                       encoder_attention_mask)):
            raise NotImplementedError("ControlNet / adapter residuals, masks and class labels are not on the "
                                      "IDM-VTON inference path")
        if added_cond_kwargs is None or "text_embeds" not in added_cond_kwargs or "time_ids" not in added_cond_kwargs \
                or "image_embeds" not in added_cond_kwargs:
            raise ValueError("added_cond_kwargs must provide text_embeds, time_ids and image_embeds "
                             "(src/unet_hacked_tryon.py:1174-1242)")
        if garment_features is None:
            raise ValueError("garment_features is required (src/attentionhacked_tryon.py:334)")
        if self._garment_kv_precision == "fp8":
            raise NotImplementedError("garment K/V precision 'fp8' with the module forward's reference-format "
                                      "garment_features: only hoisted garment K/V (the engine pipeline's denoiser) are "
                                      "held in the FP8 format")
        eng = self.engine()
        L = self._lib
        f16 = torch.float16
        B, C, h, w = sample.shape
        x = torch.zeros((B, h, w, CIN_PAD), dtype=f16, device=self.device)
        L.nchw_to_nhwc(sample.to(self.device, f16).contiguous(), x)
        ctx = eng.encode_context(encoder_hidden_states.to(self.device, f16),
                                 added_cond_kwargs["image_embeds"].to(self.device, f16))
        aug = eng.aug_embedding(added_cond_kwargs["text_embeds"].to(self.device, f16),
                                added_cond_kwargs["time_ids"].to(self.device))
        temb = eng.time_embedding(self._t_dev(timestep), B, aug)
        feats = [f.to(self.device, f16).contiguous() for f in garment_features]
        eps = eng.forward(x, temb, ctx, gfeats=feats, n_persons=B // 2)
        out = L.nhwc_to_nchw(eps, self._cfg["out_channels"])
        if not return_dict:
            return (out,)
        return types.SimpleNamespace(sample=out)


class UNet2DConditionModelGarment(_UNetBase):
    """Garment UNet ("GarmentNet", src/unet_hacked_garmnet.py): exports the post-norm1 activation of every block."""
    KIND = "garment"
    IGNORED_CHECKPOINT_PREFIXES = ("add_embedding.",)

    def __init__(self, cfg=None, state_dict=None, device="cpu", dtype=torch.float16):
        super().__init__(cfg or SDXL_GARMENT, state_dict, device, dtype)

    def enable_freeu(self, s1, s2, b1, b2):
        raise NotImplementedError("FreeU on the garment UNet is not supported: it would change the garment features, "
                                  "so the hoisted garment K/V, the GarmentKVCache keys and the pool pages would all "
                                  "depend on it. The reference pipeline's enable_freeu only touches the try-on UNet.")

    @torch.no_grad()
    def forward(self, sample, timestep, encoder_hidden_states, class_labels=None, timestep_cond=None,
                attention_mask=None, cross_attention_kwargs=None, added_cond_kwargs=None, return_dict=True, **kwargs):
        eng = self.engine()
        L = self._lib
        f16 = torch.float16
        B, C, h, w = sample.shape
        x = torch.zeros((B, h, w, CIN_PAD), dtype=f16, device=self.device)
        L.nchw_to_nhwc(sample.to(self.device, f16).contiguous(), x)
        ctx = eng.encode_context(encoder_hidden_states.to(self.device, f16))
        feats = []
        eng.forward(x, eng.time_embedding(self._t_dev(timestep), B), ctx, collect=feats)
        # The reference's first return value (`sample` before the skipped last up block) is dead: the pipeline discards
        # it (src/tryon_pipeline.py:1787). The engine stops after the last feature export and returns None for it.
        if not return_dict:
            return (None,), feats
        return types.SimpleNamespace(sample=None), feats
