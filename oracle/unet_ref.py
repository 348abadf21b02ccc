"""ORACLE (test infrastructure, not product): plain-PyTorch restatement of IDM-VTON's two UNets.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this module.
Nothing here is used by the product path (idm-vton_b200/), which must fail loudly when libb200vton.so is missing.

What it restates (reference file:line, relative to the reference):
  * try-on UNet forward            src/unet_hacked_tryon.py:1006-1395
  * garment UNet forward           src/unet_hacked_garmnet.py:917-1284   (returns the 70 garment features only)
  * block sequencing / skip cat    src/unet_block_hacked_tryon.py:724-781,1123-1201,1256-1289,2308-2397,2450-2507
  * Transformer2DModel.forward     src/transformerhacked_tryon.py:246-467
  * BasicTransformerBlock.forward  src/attentionhacked_tryon.py:284-415 (try-on: cat garment features into attn1,
                                   keep first N rows) / src/attentionhacked_garmnet.py:284-406 (export norm1 output)
  * AttnProcessor2_0               ip_adapter/attention_processor.py:203-278
  * IPAttnProcessor2_0             ip_adapter/attention_processor.py:1907-2010 (decoupled text / IP softmax, scale 1.0)
  * Resampler / PerceiverAttention ip_adapter/resampler.py:49-78,164-176
and, from the third-party dependency diffusers==0.25.0 (pinned environment.yaml:20, NOT vendored under
the reference — restated from its published semantics, SURVEY.md App. C): ResnetBlock2D, Downsample2D, Upsample2D,
Attention (weights only), GEGLU, Timesteps, TimestepEmbedding.

Pinning: oracle/make_golden.py runs the reference's own src/*.py + ip_adapter/*.py IN PLACE on the diffusers shim
(oracle/shim) with the same random weights and compares against this file (tests/test_oracle_pin.py re-checks the
committed fixtures). The in-repo logic is therefore pinned to the reference; the diffusers leaf ops are "parity
unpinned" (no upstream source, golden vectors or tests for them exist in the reference).

All functions are written with torch.nn.functional calls so that they run (i) on CPU in fp32 — the yard-stick and the
timed CPU baseline — and (ii) on CUDA under torch.autocast(fp16) with fp16 weights, which reproduces the reference's
rounding points (inference.py:223,339).
"""
import math

import torch
import torch.nn.functional as F

# ------------------------------------------------------------------------------------------------
# configurations
# ------------------------------------------------------------------------------------------------
SDXL_TRYON = dict(
    in_channels=13, out_channels=4, block_out_channels=(320, 640, 1280), layers_per_block=2,
    transformer_layers_per_block=(1, 2, 10), num_heads=(5, 10, 20), cross_attention_dim=2048,
    addition_time_embed_dim=256, projection_class_embeddings_input_dim=2816, text_time=True, ip_tokens=16,
    resampler=dict(dim=1280, depth=4, dim_head=64, heads=20, num_queries=16, embedding_dim=1280, output_dim=2048,
                   ff_mult=4),
)
SDXL_GARMENT = dict(
    in_channels=4, out_channels=4, block_out_channels=(320, 640, 1280), layers_per_block=2,
    transformer_layers_per_block=(1, 2, 10), num_heads=(5, 10, 20), cross_attention_dim=2048,
    addition_time_embed_dim=256, projection_class_embeddings_input_dim=2816, text_time=False, ip_tokens=0,
    resampler=None,
)


def tiny_config(kind):
    """Same topology as SDXL (3 levels, DownBlock2D + 2 CrossAttnDown, mid, 2 CrossAttnUp + UpBlock2D, head dim 64)
    at 1/5 width and depth: CPU-oracle friendly, used by the fast parity tests and the golden fixtures."""
    base = dict(SDXL_TRYON if kind == "tryon" else SDXL_GARMENT)
    base.update(block_out_channels=(64, 128, 256), transformer_layers_per_block=(1, 1, 2), num_heads=(1, 2, 4),
                cross_attention_dim=256, addition_time_embed_dim=64, projection_class_embeddings_input_dim=6 * 64 + 128)
    if kind == "tryon":
        # the reference hard-codes the Resampler geometry (src/unet_hacked_tryon.py:476-485); only the CLIP width
        # (encoder_hid_dim) and the output width (cross_attention_dim) follow the config
        base["resampler"] = dict(dim=1280, depth=4, dim_head=64, heads=20, num_queries=16, embedding_dim=192,
                                 output_dim=256, ff_mult=4)
    return base


# ------------------------------------------------------------------------------------------------
# state-dict enumeration with the reference's key names (SURVEY.md App. D.7)
# ------------------------------------------------------------------------------------------------
def _resnet_shapes(p, cin, cout, temb):
    s = {f"{p}.norm1.weight": (cin,), f"{p}.norm1.bias": (cin,), f"{p}.conv1.weight": (cout, cin, 3, 3),
         f"{p}.conv1.bias": (cout,), f"{p}.time_emb_proj.weight": (cout, temb), f"{p}.time_emb_proj.bias": (cout,),
         f"{p}.norm2.weight": (cout,), f"{p}.norm2.bias": (cout,), f"{p}.conv2.weight": (cout, cout, 3, 3),
         f"{p}.conv2.bias": (cout,)}
    if cin != cout:
        s[f"{p}.conv_shortcut.weight"] = (cout, cin, 1, 1)
        s[f"{p}.conv_shortcut.bias"] = (cout,)
    return s


def _t2d_shapes(p, c, layers, cross, ip):
    s = {f"{p}.norm.weight": (c,), f"{p}.norm.bias": (c,), f"{p}.proj_in.weight": (c, c), f"{p}.proj_in.bias": (c,),
         f"{p}.proj_out.weight": (c, c), f"{p}.proj_out.bias": (c,)}
    for k in range(layers):
        b = f"{p}.transformer_blocks.{k}"
        for n in ("norm1", "norm2", "norm3"):
            s[f"{b}.{n}.weight"] = (c,)
            s[f"{b}.{n}.bias"] = (c,)
        for a, kd in (("attn1", c), ("attn2", cross)):
            s[f"{b}.{a}.to_q.weight"] = (c, c)
            s[f"{b}.{a}.to_k.weight"] = (c, kd)
            s[f"{b}.{a}.to_v.weight"] = (c, kd)
            s[f"{b}.{a}.to_out.0.weight"] = (c, c)
            s[f"{b}.{a}.to_out.0.bias"] = (c,)
        if ip:
            s[f"{b}.attn2.processor.to_k_ip.weight"] = (c, cross)
            s[f"{b}.attn2.processor.to_v_ip.weight"] = (c, cross)
        s[f"{b}.ff.net.0.proj.weight"] = (8 * c, c)
        s[f"{b}.ff.net.0.proj.bias"] = (8 * c,)
        s[f"{b}.ff.net.2.weight"] = (c, 4 * c)
        s[f"{b}.ff.net.2.bias"] = (c,)
    return s


def _resampler_shapes(p, r):
    d, inner = r["dim"], r["dim_head"] * r["heads"]
    s = {f"{p}.latents": (1, r["num_queries"], d), f"{p}.proj_in.weight": (d, r["embedding_dim"]),
         f"{p}.proj_in.bias": (d,), f"{p}.proj_out.weight": (r["output_dim"], d), f"{p}.proj_out.bias": (r["output_dim"],),
         f"{p}.norm_out.weight": (r["output_dim"],), f"{p}.norm_out.bias": (r["output_dim"],)}
    for i in range(r["depth"]):
        a, f = f"{p}.layers.{i}.0", f"{p}.layers.{i}.1"
        for n in ("norm1", "norm2"):
            s[f"{a}.{n}.weight"] = (d,)
            s[f"{a}.{n}.bias"] = (d,)
        s[f"{a}.to_q.weight"] = (inner, d)
        s[f"{a}.to_kv.weight"] = (2 * inner, d)
        s[f"{a}.to_out.weight"] = (d, inner)
        s[f"{f}.0.weight"] = (d,)
        s[f"{f}.0.bias"] = (d,)
        s[f"{f}.1.weight"] = (d * r["ff_mult"], d)
        s[f"{f}.3.weight"] = (d, d * r["ff_mult"])
    return s


def unet_param_shapes(cfg):
    """Ordered {key: shape} of a UNet2DConditionModel state dict as the reference's modules would create it.
    (The garment UNet checkpoint also carries up_blocks.2 / conv_norm_out / conv_out, never used: App. D.7.)"""
    ch = cfg["block_out_channels"]
    temb = ch[0] * 4
    cross = cfg["cross_attention_dim"]
    tl = cfg["transformer_layers_per_block"]
    ip = cfg["ip_tokens"] > 0
    s = {"conv_in.weight": (ch[0], cfg["in_channels"], 3, 3), "conv_in.bias": (ch[0],),
         "time_embedding.linear_1.weight": (temb, ch[0]), "time_embedding.linear_1.bias": (temb,),
         "time_embedding.linear_2.weight": (temb, temb), "time_embedding.linear_2.bias": (temb,)}
    if cfg["text_time"]:
        s.update({"add_embedding.linear_1.weight": (temb, cfg["projection_class_embeddings_input_dim"]),
                  "add_embedding.linear_1.bias": (temb,), "add_embedding.linear_2.weight": (temb, temb),
                  "add_embedding.linear_2.bias": (temb,)})
    if cfg.get("resampler"):
        s.update(_resampler_shapes("encoder_hid_proj", cfg["resampler"]))
    # down
    out_c = ch[0]
    for i, c in enumerate(ch):
        in_c, out_c = out_c, c
        for j in range(cfg["layers_per_block"]):
            s.update(_resnet_shapes(f"down_blocks.{i}.resnets.{j}", in_c if j == 0 else out_c, out_c, temb))
            if i > 0:
                s.update(_t2d_shapes(f"down_blocks.{i}.attentions.{j}", out_c, tl[i], cross, ip))
        if i < len(ch) - 1:
            s[f"down_blocks.{i}.downsamplers.0.conv.weight"] = (out_c, out_c, 3, 3)
            s[f"down_blocks.{i}.downsamplers.0.conv.bias"] = (out_c,)
    # mid
    s.update(_resnet_shapes("mid_block.resnets.0", ch[-1], ch[-1], temb))
    s.update(_t2d_shapes("mid_block.attentions.0", ch[-1], tl[-1], cross, ip))
    s.update(_resnet_shapes("mid_block.resnets.1", ch[-1], ch[-1], temb))
    # up (reversed channels; skip channel bookkeeping as in src/unet_hacked_tryon.py:700-740)
    rev = list(reversed(ch))
    rtl = list(reversed(tl))
    out_c = rev[0]
    for i, c in enumerate(rev):
        prev_out, out_c = out_c, c
        in_c = rev[min(i + 1, len(ch) - 1)]
        n = cfg["layers_per_block"] + 1
        for j in range(n):
            res_skip = in_c if j == n - 1 else out_c
            res_in = prev_out if j == 0 else out_c
            s.update(_resnet_shapes(f"up_blocks.{i}.resnets.{j}", res_in + res_skip, out_c, temb))
            if i < len(ch) - 1:
                s.update(_t2d_shapes(f"up_blocks.{i}.attentions.{j}", out_c, rtl[i], cross, ip))
        if i < len(ch) - 1:
            s[f"up_blocks.{i}.upsamplers.0.conv.weight"] = (out_c, out_c, 3, 3)
            s[f"up_blocks.{i}.upsamplers.0.conv.bias"] = (out_c,)
    s["conv_norm_out.weight"] = (ch[0],)
    s["conv_norm_out.bias"] = (ch[0],)
    s["conv_out.weight"] = (cfg["out_channels"], ch[0], 3, 3)
    s["conv_out.bias"] = (cfg["out_channels"],)
    return s


def make_state_dict(cfg, seed=0, dtype=torch.float32, device="cpu", residual_gain=0.25):
    """Seeded synthetic weights (the reference's ckpt/** are 0-byte placeholders). PyTorch-default-like scale
    (uniform +-1/sqrt(fan_in)); norm affine ~ 1 +- 0.1 / +-0.1; the last layer of every residual branch is scaled by
    `residual_gain` so 70 residual blocks stay inside fp16 range (SURVEY.md 8d weight-scale guard)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shp in unet_param_shapes(cfg).items():
        if k.endswith("latents"):
            w = torch.randn(shp, generator=g) / shp[-1] ** 0.5
        elif ".norm" in k or k.startswith("conv_norm_out") or ".layers." in k and k.split(".")[-2] in ("0",) and len(shp) == 1:
            w = (1.0 + 0.1 * torch.randn(shp, generator=g)) if k.endswith("weight") else 0.1 * torch.randn(shp, generator=g)
        elif len(shp) == 1:
            w = 0.05 * torch.randn(shp, generator=g)
        else:
            fan_in = 1
            for d in shp[1:]:
                fan_in *= d
            w = (torch.rand(shp, generator=g) * 2 - 1) * (3.0 / fan_in) ** 0.5
            if any(t in k for t in ("to_out.0.weight", "ff.net.2.weight", "conv2.weight", "proj_out.weight")) and \
                    not k.startswith("encoder_hid_proj"):
                w = w * residual_gain
        sd[k] = w.to(dtype=dtype, device=device)
    return sd


# ------------------------------------------------------------------------------------------------
# diffusers 0.25.0 leaf ops (restated)
# ------------------------------------------------------------------------------------------------
def timesteps_proj(t, dim):
    """diffusers Timesteps(dim, flip_sin_to_cos=True, downscale_freq_shift=0): fp32 [cos | sin]."""
    half = dim // 2
    exponent = -math.log(10000) * torch.arange(half, dtype=torch.float32, device=t.device) / half
    emb = t[:, None].float() * torch.exp(exponent)[None, :]
    return torch.cat([torch.cos(emb), torch.sin(emb)], dim=-1)


def timestep_embedding(sd, p, x):
    x = F.linear(x, sd[f"{p}.linear_1.weight"], sd[f"{p}.linear_1.bias"])
    x = F.silu(x)
    return F.linear(x, sd[f"{p}.linear_2.weight"], sd[f"{p}.linear_2.bias"])


def resnet_block(sd, p, x, temb, eps=1e-5):
    """diffusers ResnetBlock2D (pre_norm, time_embedding_norm='default', output_scale_factor=1.0)."""
    h = F.group_norm(x, 32, sd[f"{p}.norm1.weight"], sd[f"{p}.norm1.bias"], eps)
    h = F.silu(h)
    h = F.conv2d(h, sd[f"{p}.conv1.weight"], sd[f"{p}.conv1.bias"], padding=1)
    t = F.linear(F.silu(temb), sd[f"{p}.time_emb_proj.weight"], sd[f"{p}.time_emb_proj.bias"])
    h = h + t[:, :, None, None]
    h = F.group_norm(h, 32, sd[f"{p}.norm2.weight"], sd[f"{p}.norm2.bias"], eps)
    h = F.silu(h)
    h = F.conv2d(h, sd[f"{p}.conv2.weight"], sd[f"{p}.conv2.bias"], padding=1)
    if f"{p}.conv_shortcut.weight" in sd:
        x = F.conv2d(x, sd[f"{p}.conv_shortcut.weight"], sd[f"{p}.conv_shortcut.bias"])
    return (x + h) / 1.0


def downsample(sd, p, x):
    return F.conv2d(x, sd[f"{p}.conv.weight"], sd[f"{p}.conv.bias"], stride=2, padding=1)


def upsample(sd, p, x):
    x = F.interpolate(x, scale_factor=2.0, mode="nearest")
    return F.conv2d(x, sd[f"{p}.conv.weight"], sd[f"{p}.conv.bias"], padding=1)


def _heads(x, h):
    b, n, c = x.shape
    return x.view(b, n, h, c // h).transpose(1, 2)


def _sdpa(q, k, v, heads):
    o = F.scaled_dot_product_attention(_heads(q, heads), _heads(k, heads), _heads(v, heads))
    b, h, n, d = o.shape
    return o.transpose(1, 2).reshape(b, n, h * d).to(q.dtype)


def attn_self(sd, p, x, heads):
    """AttnProcessor2_0 with encoder_hidden_states=None (ip_adapter/attention_processor.py:203-278)."""
    q = F.linear(x, sd[f"{p}.to_q.weight"])
    k = F.linear(x, sd[f"{p}.to_k.weight"])
    v = F.linear(x, sd[f"{p}.to_v.weight"])
    o = _sdpa(q, k, v, heads)
    return F.linear(o, sd[f"{p}.to_out.0.weight"], sd[f"{p}.to_out.0.bias"])


def attn_cross(sd, p, x, enc, heads, ip_tokens, ip_scale=1.0):
    """IPAttnProcessor2_0 (ip_adapter/attention_processor.py:1907-2010) when ip_tokens > 0, else AttnProcessor2_0."""
    q = F.linear(x, sd[f"{p}.to_q.weight"])
    if ip_tokens:
        end = enc.shape[1] - ip_tokens
        enc, ip = enc[:, :end], enc[:, end:]
    o = _sdpa(q, F.linear(enc, sd[f"{p}.to_k.weight"]), F.linear(enc, sd[f"{p}.to_v.weight"]), heads)
    if ip_tokens:
        o_ip = _sdpa(q, F.linear(ip, sd[f"{p}.processor.to_k_ip.weight"]),
                     F.linear(ip, sd[f"{p}.processor.to_v_ip.weight"]), heads)
        o = o + ip_scale * o_ip                                       # :1995, self.scale (1.0 at inference)
    return F.linear(o, sd[f"{p}.to_out.0.weight"], sd[f"{p}.to_out.0.bias"])


def feed_forward(sd, p, x):
    """FeedForward(GEGLU) (src/attentionhacked_tryon.py:621-679; diffusers GEGLU: value, gate = chunk(2); erf GELU)."""
    h = F.linear(x, sd[f"{p}.net.0.proj.weight"], sd[f"{p}.net.0.proj.bias"])
    h, gate = h.chunk(2, dim=-1)
    h = h * F.gelu(gate)
    return F.linear(h, sd[f"{p}.net.2.weight"], sd[f"{p}.net.2.bias"])


# ------------------------------------------------------------------------------------------------
# in-repo logic
# ------------------------------------------------------------------------------------------------
def transformer_block(sd, p, x, enc, heads, ip_tokens, garment_features, idx, collect, ip_scale=1.0):
    """BasicTransformerBlock.forward. collect=None: try-on variant (consume garment_features[idx]);
    collect=list: garment variant (append norm1 output)."""
    n1 = F.layer_norm(x, (x.shape[-1],), sd[f"{p}.norm1.weight"], sd[f"{p}.norm1.bias"], 1e-5)
    if collect is not None:
        collect.append(n1)                                   # src/attentionhacked_garmnet.py:321-322
        a = attn_self(sd, f"{p}.attn1", n1, heads)
        x = a + x
    else:
        mod = torch.cat([n1, garment_features[idx].to(n1.dtype)], dim=1)   # src/attentionhacked_tryon.py:334
        idx += 1
        a = attn_self(sd, f"{p}.attn1", mod, heads)
        x = a[:, :x.shape[-2], :] + x                        # :348
    n2 = F.layer_norm(x, (x.shape[-1],), sd[f"{p}.norm2.weight"], sd[f"{p}.norm2.bias"], 1e-5)
    x = attn_cross(sd, f"{p}.attn2", n2, enc, heads, ip_tokens, ip_scale) + x
    n3 = F.layer_norm(x, (x.shape[-1],), sd[f"{p}.norm3.weight"], sd[f"{p}.norm3.bias"], 1e-5)
    x = feed_forward(sd, f"{p}.ff", n3) + x
    return x, idx


def transformer_2d(sd, p, x, enc, heads, layers, ip_tokens, garment_features, idx, collect, ip_scale=1.0):
    """Transformer2DModel.forward, continuous input, use_linear_projection=True."""
    b, c, hh, ww = x.shape
    res = x
    h = F.group_norm(x, 32, sd[f"{p}.norm.weight"], sd[f"{p}.norm.bias"], 1e-6)
    h = h.permute(0, 2, 3, 1).reshape(b, hh * ww, c)
    h = F.linear(h, sd[f"{p}.proj_in.weight"], sd[f"{p}.proj_in.bias"])
    for k in range(layers):
        h, idx = transformer_block(sd, f"{p}.transformer_blocks.{k}", h, enc, heads, ip_tokens, garment_features, idx,
                                   collect, ip_scale)
    h = F.linear(h, sd[f"{p}.proj_out.weight"], sd[f"{p}.proj_out.bias"])
    h = h.reshape(b, hh, ww, c).permute(0, 3, 1, 2).contiguous()
    return h + res, idx


def _time_embed(sd, cfg, sample, timestep, added_cond):
    ch0 = cfg["block_out_channels"][0]
    t = timestep
    if not torch.is_tensor(t):
        t = torch.tensor([t], dtype=torch.float64 if isinstance(t, float) else torch.int64, device=sample.device)
    elif t.ndim == 0:
        t = t[None].to(sample.device)
    t = t.expand(sample.shape[0])
    t_emb = timesteps_proj(t, ch0).to(sample.dtype)
    emb = timestep_embedding(sd, "time_embedding", t_emb)
    if cfg["text_time"]:
        text_embeds, time_ids = added_cond["text_embeds"], added_cond["time_ids"]
        te = timesteps_proj(time_ids.flatten(), cfg["addition_time_embed_dim"]).reshape(text_embeds.shape[0], -1)
        add = torch.cat([text_embeds, te], dim=-1).to(emb.dtype)
        emb = emb + timestep_embedding(sd, "add_embedding", add)
    return emb


def _trunk(sd, cfg, sample, emb, enc, garment_features, collect, stop_after_up):
    ch = cfg["block_out_channels"]
    tl = cfg["transformer_layers_per_block"]
    nh = cfg["num_heads"]
    ip = cfg["ip_tokens"]
    ips = cfg.get("ip_scale", 1.0)      # IPAttnProcessor2_0.scale of every block (1.0 unless a test installs others)
    idx = 0
    x = F.conv2d(sample, sd["conv_in.weight"], sd["conv_in.bias"], padding=1)
    skips = [x]
    for i in range(len(ch)):
        for j in range(cfg["layers_per_block"]):
            x = resnet_block(sd, f"down_blocks.{i}.resnets.{j}", x, emb)
            if i > 0:
                x, idx = transformer_2d(sd, f"down_blocks.{i}.attentions.{j}", x, enc, nh[i], tl[i], ip,
                                        garment_features, idx, collect, ips)
            skips.append(x)
        if i < len(ch) - 1:
            x = downsample(sd, f"down_blocks.{i}.downsamplers.0", x)
            skips.append(x)
    x = resnet_block(sd, "mid_block.resnets.0", x, emb)
    x, idx = transformer_2d(sd, "mid_block.attentions.0", x, enc, nh[-1], tl[-1], ip, garment_features, idx, collect,
                            ips)
    x = resnet_block(sd, "mid_block.resnets.1", x, emb)
    rnh, rtl = list(reversed(nh)), list(reversed(tl))
    for i in range(len(ch)):
        if i >= stop_after_up:
            break
        for j in range(cfg["layers_per_block"] + 1):
            x = torch.cat([x, skips.pop()], dim=1)
            x = resnet_block(sd, f"up_blocks.{i}.resnets.{j}", x, emb)
            if i < len(ch) - 1:
                x, idx = transformer_2d(sd, f"up_blocks.{i}.attentions.{j}", x, enc, rnh[i], rtl[i], ip,
                                        garment_features, idx, collect, ips)
        if i < len(ch) - 1:
            x = upsample(sd, f"up_blocks.{i}.upsamplers.0", x)
    return x


def unet_tryon_forward(sd, cfg, sample, timestep, encoder_hidden_states, added_cond_kwargs, garment_features):
    """src/unet_hacked_tryon.py:1006-1395 -> noise_pred [2B,4,h,w]. image_embeds are already Resampler outputs
    (src/tryon_pipeline.py:1726) and are concatenated after the text tokens (:1242)."""
    emb = _time_embed(sd, cfg, sample, timestep, added_cond_kwargs)
    enc = torch.cat([encoder_hidden_states, added_cond_kwargs["image_embeds"]], dim=1)
    x = _trunk(sd, cfg, sample, emb, enc, garment_features, None, stop_after_up=len(cfg["block_out_channels"]))
    x = F.group_norm(x, 32, sd["conv_norm_out.weight"], sd["conv_norm_out.bias"], 1e-5)
    x = F.silu(x)
    return F.conv2d(x, sd["conv_out.weight"], sd["conv_out.bias"], padding=1)


def unet_garment_forward(sd, cfg, sample, timestep, encoder_hidden_states):
    """src/unet_hacked_garmnet.py:917-1284 -> list of garment features (post-norm1 activations, execution order).
    The reference stops after the last CrossAttnUpBlock2D (:1256-1278); its `sample` output is discarded by the
    pipeline (src/tryon_pipeline.py:1787), so only the features are returned."""
    emb = _time_embed(sd, cfg, sample, timestep, None)
    feats = []
    _trunk(sd, cfg, sample, emb, encoder_hidden_states, None, feats, stop_after_up=len(cfg["block_out_channels"]) - 1)
    return feats


def resampler_forward(sd, p, r, x):
    """ip_adapter/resampler.py:164-176 (Resampler) with PerceiverAttention :49-78 and FeedForward :13-20."""
    latents = sd[f"{p}.latents"].repeat(x.size(0), 1, 1)
    x = F.linear(x, sd[f"{p}.proj_in.weight"], sd[f"{p}.proj_in.bias"])
    heads = r["heads"]
    for i in range(r["depth"]):
        a, f = f"{p}.layers.{i}.0", f"{p}.layers.{i}.1"
        xn = F.layer_norm(x, (x.shape[-1],), sd[f"{a}.norm1.weight"], sd[f"{a}.norm1.bias"])
        ln = F.layer_norm(latents, (latents.shape[-1],), sd[f"{a}.norm2.weight"], sd[f"{a}.norm2.bias"])
        b, l, _ = ln.shape
        q = F.linear(ln, sd[f"{a}.to_q.weight"])
        k, v = F.linear(torch.cat((xn, ln), dim=-2), sd[f"{a}.to_kv.weight"]).chunk(2, dim=-1)
        q, k, v = _heads(q, heads), _heads(k, heads), _heads(v, heads)
        scale = 1 / math.sqrt(math.sqrt(r["dim_head"]))
        w = (q * scale) @ (k * scale).transpose(-2, -1)
        w = torch.softmax(w.float(), dim=-1).type(w.dtype)
        o = (w @ v).permute(0, 2, 1, 3).reshape(b, l, -1)
        latents = F.linear(o, sd[f"{a}.to_out.weight"]) + latents
        h = F.layer_norm(latents, (latents.shape[-1],), sd[f"{f}.0.weight"], sd[f"{f}.0.bias"])
        h = F.linear(F.gelu(F.linear(h, sd[f"{f}.1.weight"])), sd[f"{f}.3.weight"])
        latents = h + latents
    latents = F.linear(latents, sd[f"{p}.proj_out.weight"], sd[f"{p}.proj_out.bias"])
    return F.layer_norm(latents, (latents.shape[-1],), sd[f"{p}.norm_out.weight"], sd[f"{p}.norm_out.bias"])
