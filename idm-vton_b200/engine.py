"""UNet executors of the denoising engine: weight pre-packing + the launch sequence of both SDXL UNets.

Host orchestration is Python; all math is in libb200vton.so (see lib.py). One denoise step is a fixed launch sequence
over static buffers, so it is captured once into a CUDA graph and replayed for every step.
"""
import torch


# ------------------------------------------------------------------------------------------------
# weight packing (load time, plain torch)
# ------------------------------------------------------------------------------------------------
def pack_conv3x3(w):
    """[Cout, Cin, 3, 3] -> [9, Cout, Cin] (tap = ky*3+kx), the layout b200vton_conv3x3_nhwc streams by TMA."""
    cout, cin = w.shape[0], w.shape[1]
    return w.permute(2, 3, 0, 1).reshape(9, cout, cin).contiguous()


def pad_channels(w_packed, cin_to=None, cout_to=None):
    """Zero-pad a packed conv weight [9, Cout, Cin] (conv_in: Cin 13 -> 64; conv_out: Cout 4 -> 16)."""
    nine, cout, cin = w_packed.shape
    cin_to = cin_to or cin
    cout_to = cout_to or cout
    out = torch.zeros((nine, cout_to, cin_to), dtype=w_packed.dtype, device=w_packed.device)
    out[:, :cout, :cin] = w_packed
    return out


def pack_conv3x3_s2(w):
    """[Cout, Cin, 3, 3] -> [Cout, 9*Cin] with K ordered tap-major, matching b200vton_im2col3x3_s2_nhwc."""
    cout, cin = w.shape[0], w.shape[1]
    return w.permute(0, 2, 3, 1).reshape(cout, 9 * cin).contiguous()


def pack_geglu(w, b, bn):
    """GEGLU proj weight [8C, C] (rows = [value 4C | gate 4C], diffusers GEGLU.chunk order) -> rows interleaved per
    output tile of width bn: [value bn/2 | gate bn/2], so one accumulator tile holds both halves of its channels."""
    n2 = w.shape[0]
    n = n2 // 2
    hb = bn // 2
    assert n % hb == 0
    wv, wg = w[:n].reshape(n // hb, hb, -1), w[n:].reshape(n // hb, hb, -1)
    wp = torch.cat([wv, wg], dim=1).reshape(n2, -1).contiguous()
    bp = None
    if b is not None:
        bv, bg = b[:n].reshape(n // hb, hb), b[n:].reshape(n // hb, hb)
        bp = torch.cat([bv, bg], dim=1).reshape(n2).contiguous()
    return wp, bp


# ------------------------------------------------------------------------------------------------
# configuration (mirrors the fields of the reference's UNet2DConditionModel config that the path reads)
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

CIN_PAD = 64    # conv_in input channels are zero-padded to one 64-wide K slab
COUT_PAD = 16   # conv_out output channels are zero-padded to 16


class _Resnet:
    __slots__ = ("cin", "cout", "n1w", "n1b", "w1", "b1", "temb_off", "n2w", "n2b", "w2", "b2", "wsc", "bsc")


class _Block:
    __slots__ = ("ln1w", "ln1b", "wqkv", "wo1", "bo1", "ln2w", "ln2b", "wq2", "wkv_txt", "wkv_ip", "wo2", "bo2", "ln3w",
                 "ln3b", "wff1", "bff1", "wff2", "bff2", "c", "heads", "ff_bn", "ip_scale", "fp8")


class _T2D:
    __slots__ = ("nw", "nb", "win", "bin", "wout", "bout", "blocks", "c", "heads")


class _GarmentDone(Exception):
    """Raised inside the garment UNet's launch sequence once the last garment feature has been exported."""


def active_freeu(freeu):
    """The FreeU values (s1, s2, b1, b2) that run, or None. As in the reference's up blocks
    (src/unet_block_hacked_tryon.py:2322-2327), FreeU runs only if all four are truthy: a 0 switches it off."""
    return None if freeu is None or not all(freeu) else tuple(freeu)


class UNetEngine:
    """Launch sequence of one SDXL-family UNet (DownBlock2D, 2x CrossAttnDownBlock2D, mid, 2x CrossAttnUpBlock2D,
    UpBlock2D) over NHWC fp16 buffers. kind = "tryon" (src/unet_hacked_tryon.py) or "garment"
    (src/unet_hacked_garmnet.py). Weights come from a state dict with the reference's key names."""

    GEGLU_BN = 256

    def __init__(self, cfg, state_dict, kind, device="cuda", ip_scales=None, fp8=False):
        """ip_scales: optional {"<transformer block path>": scale} of the installed IPAttnProcessor2_0 instances
        (ip_adapter/attention_processor.py:1995 `hidden + self.scale * ip_hidden`; default 1.0).
        fp8: run attn1's QKV, attn2.to_q and the GEGLU projection of every BasicTransformerBlock as e4m3 GEMMs, their
        input quantized per token by the LayerNorm before them and the weights per output channel (INTEGRATION.md,
        "FP8 linears"). Every channel width with a transformer must then be a multiple of 128."""
        from . import lib
        lib.load()
        self.L = lib
        self.cfg = dict(cfg)
        self.kind = kind
        self.device = torch.device(device)
        self.ch = tuple(cfg["block_out_channels"])
        self.temb_dim = self.ch[0] * 4
        self.cross = cfg["cross_attention_dim"]
        self.ip_tokens = cfg["ip_tokens"] if kind == "tryon" else 0
        self.ip_scales = dict(ip_scales or {})
        self.fp8 = bool(fp8)
        # format of the hoisted garment K/V the denoisers keep for this (try-on) UNet: "fp16" or "fp8" (lib.GarmentKV8);
        # set by UNet2DConditionModel.set_garment_kv_precision
        self.garment_kv_format = "fp16"
        # FreeU of the try-on UNet's up stages 0 and 1: None or (s1, s2, b1, b2), set by UNet2DConditionModel.enable_freeu
        self.freeu = None
        self._kv_scratch = None
        if self.fp8:
            for name in ("b200vton_layernorm_e4m3", "b200vton_gemm_e4m3"):
                if not lib.has_symbol(name):
                    raise NotImplementedError(f"FP8 linears need {name}, which {lib.LIB_PATH} does not export: rebuild it "
                                              "(python idm-vton_b200/build.py --force)")
        self._pack(state_dict)

    # -------------------------------------------------------------------------------------------
    def _w(self, sd, key):
        t = sd[key]
        return t.to(device=self.device, dtype=torch.float16).contiguous()

    def _pack_resnet(self, sd, p, temb_ws, temb_bs):
        r = _Resnet()
        w1 = self._w(sd, f"{p}.conv1.weight")
        r.cout, r.cin = w1.shape[0], w1.shape[1]
        r.n1w, r.n1b = self._w(sd, f"{p}.norm1.weight"), self._w(sd, f"{p}.norm1.bias")
        r.w1, r.b1 = pack_conv3x3(w1), self._w(sd, f"{p}.conv1.bias")
        r.temb_off = sum(w.shape[0] for w in temb_ws)
        temb_ws.append(self._w(sd, f"{p}.time_emb_proj.weight"))
        temb_bs.append(self._w(sd, f"{p}.time_emb_proj.bias"))
        r.n2w, r.n2b = self._w(sd, f"{p}.norm2.weight"), self._w(sd, f"{p}.norm2.bias")
        r.w2, r.b2 = pack_conv3x3(self._w(sd, f"{p}.conv2.weight")), self._w(sd, f"{p}.conv2.bias")
        r.wsc = r.bsc = None
        if f"{p}.conv_shortcut.weight" in sd:
            r.wsc = self._w(sd, f"{p}.conv_shortcut.weight").reshape(r.cout, r.cin).contiguous()
            r.bsc = self._w(sd, f"{p}.conv_shortcut.bias")
        return r

    def _pack_t2d(self, sd, p, c, heads, layers):
        t = _T2D()
        t.c, t.heads = c, heads
        t.nw, t.nb = self._w(sd, f"{p}.norm.weight"), self._w(sd, f"{p}.norm.bias")
        t.win, t.bin = self._w(sd, f"{p}.proj_in.weight"), self._w(sd, f"{p}.proj_in.bias")
        t.wout, t.bout = self._w(sd, f"{p}.proj_out.weight"), self._w(sd, f"{p}.proj_out.bias")
        t.blocks = []
        for k in range(layers):
            b = f"{p}.transformer_blocks.{k}"
            blk = _Block()
            blk.c, blk.heads = c, heads
            blk.ln1w, blk.ln1b = self._w(sd, f"{b}.norm1.weight"), self._w(sd, f"{b}.norm1.bias")
            blk.wqkv = torch.cat([self._w(sd, f"{b}.attn1.to_q.weight"), self._w(sd, f"{b}.attn1.to_k.weight"),
                                  self._w(sd, f"{b}.attn1.to_v.weight")], 0).contiguous()
            blk.wo1, blk.bo1 = self._w(sd, f"{b}.attn1.to_out.0.weight"), self._w(sd, f"{b}.attn1.to_out.0.bias")
            blk.ln2w, blk.ln2b = self._w(sd, f"{b}.norm2.weight"), self._w(sd, f"{b}.norm2.bias")
            blk.wq2 = self._w(sd, f"{b}.attn2.to_q.weight")
            blk.wkv_txt = torch.cat([self._w(sd, f"{b}.attn2.to_k.weight"), self._w(sd, f"{b}.attn2.to_v.weight")],
                                    0).contiguous()
            blk.wkv_ip = None
            blk.ip_scale = float(self.ip_scales.get(b, 1.0))
            if self.ip_tokens:
                blk.wkv_ip = torch.cat([self._w(sd, f"{b}.attn2.processor.to_k_ip.weight"),
                                        self._w(sd, f"{b}.attn2.processor.to_v_ip.weight")], 0).contiguous()
            blk.wo2, blk.bo2 = self._w(sd, f"{b}.attn2.to_out.0.weight"), self._w(sd, f"{b}.attn2.to_out.0.bias")
            blk.ln3w, blk.ln3b = self._w(sd, f"{b}.norm3.weight"), self._w(sd, f"{b}.norm3.bias")
            bn = self.GEGLU_BN if (8 * c) % self.GEGLU_BN == 0 else 128
            blk.ff_bn = bn
            blk.wff1, blk.bff1 = pack_geglu(self._w(sd, f"{b}.ff.net.0.proj.weight"),
                                            self._w(sd, f"{b}.ff.net.0.proj.bias"), bn)
            blk.wff2, blk.bff2 = self._w(sd, f"{b}.ff.net.2.weight"), self._w(sd, f"{b}.ff.net.2.bias")
            blk.fp8 = self._pack_fp8(blk, b) if self.fp8 else None
            t.blocks.append(blk)
        return t

    def _pack_fp8(self, blk, path):
        """e4m3 weights and per-output-channel scales of the block's FP8 linears: {name: (w_q, w_scale)}. FF1 is quantized
        after pack_geglu, so every interleaved row carries its own scale. FF2 stays fp16: its input (the GEGLU output)
        would need a quantize pass of its own (BASELINE.md, "FP8 linears")."""
        if blk.c % 128:
            raise ValueError(f"{path}: FP8 linears need the channel width to be a multiple of 128 (got {blk.c}); there is "
                             "no fp16 fallback in FP8 mode")
        q = self.L.quantize_rows_e4m3
        return dict(qkv=q(blk.wqkv), q2=q(blk.wq2), ff1=q(blk.wff1))

    def _pack(self, sd):
        cfg, ch = self.cfg, self.ch
        tl, nh = cfg["transformer_layers_per_block"], cfg["num_heads"]
        n_lvl = len(ch)
        temb_ws, temb_bs = [], []
        self.w_in = pad_channels(pack_conv3x3(self._w(sd, "conv_in.weight")), cin_to=CIN_PAD)
        self.b_in = self._w(sd, "conv_in.bias")
        self.te = [self._w(sd, f"time_embedding.linear_{i}.{n}") for i in (1, 2) for n in ("weight", "bias")]
        self.ae = None
        if cfg["text_time"] and self.kind == "tryon":
            self.ae = [self._w(sd, f"add_embedding.linear_{i}.{n}") for i in (1, 2) for n in ("weight", "bias")]
        self.down = []
        for i in range(n_lvl):
            lvl = dict(res=[], attn=[], down=None)
            for j in range(cfg["layers_per_block"]):
                lvl["res"].append(self._pack_resnet(sd, f"down_blocks.{i}.resnets.{j}", temb_ws, temb_bs))
                if i > 0:
                    lvl["attn"].append(self._pack_t2d(sd, f"down_blocks.{i}.attentions.{j}", ch[i], nh[i], tl[i]))
            if i < n_lvl - 1:
                lvl["down"] = (pack_conv3x3(self._w(sd, f"down_blocks.{i}.downsamplers.0.conv.weight")),
                               self._w(sd, f"down_blocks.{i}.downsamplers.0.conv.bias"))
            self.down.append(lvl)
        self.mid_res = [self._pack_resnet(sd, f"mid_block.resnets.{j}", temb_ws, temb_bs) for j in (0, 1)]
        self.mid_attn = self._pack_t2d(sd, "mid_block.attentions.0", ch[-1], nh[-1], tl[-1])
        self.up = []
        rch, rnh, rtl = list(reversed(ch)), list(reversed(nh)), list(reversed(tl))
        n_up = n_lvl if self.kind == "tryon" else n_lvl - 1   # the garment UNet never runs its last up block
        for i in range(n_up):
            lvl = dict(res=[], attn=[], up=None)
            for j in range(cfg["layers_per_block"] + 1):
                lvl["res"].append(self._pack_resnet(sd, f"up_blocks.{i}.resnets.{j}", temb_ws, temb_bs))
                if i < n_lvl - 1:
                    lvl["attn"].append(self._pack_t2d(sd, f"up_blocks.{i}.attentions.{j}", rch[i], rnh[i], rtl[i]))
            if i < n_lvl - 1:
                lvl["up"] = (pack_conv3x3(self._w(sd, f"up_blocks.{i}.upsamplers.0.conv.weight")),
                             self._w(sd, f"up_blocks.{i}.upsamplers.0.conv.bias"))
            self.up.append(lvl)
        self.n_blocks = len(self.blocks())
        self.temb_w = torch.cat(temb_ws, 0).contiguous()
        self.temb_b = torch.cat(temb_bs, 0).contiguous()
        if self.kind == "tryon":
            self.no_w, self.no_b = self._w(sd, "conv_norm_out.weight"), self._w(sd, "conv_norm_out.bias")
            self.w_out = pad_channels(pack_conv3x3(self._w(sd, "conv_out.weight")), cout_to=COUT_PAD)
            self.b_out = torch.zeros(COUT_PAD, dtype=torch.float16, device=self.device)
            self.b_out[:cfg["out_channels"]] = self._w(sd, "conv_out.bias")

    def t2ds(self):
        """All Transformer2D stages in execution order (the order garment features are produced / consumed)."""
        out = []
        for lvl in self.down:
            out += lvl["attn"]
        out.append(self.mid_attn)
        for lvl in self.up:
            out += lvl["attn"]
        return out

    def blocks(self):
        return [b for t in self.t2ds() for b in t.blocks]

    def freeu_active(self):
        """(s1, s2, b1, b2) when FreeU runs in this UNet's forward (the try-on UNet only), else None (also for an engine
        object made without __init__, which has no `freeu`)."""
        return active_freeu(getattr(self, "freeu", None)) if self.kind == "tryon" else None

    # -------------------------------------------------------------------------------------------
    # step-invariant precompute (once per request): cross-attention K/V, aug_emb (SURVEY.md App. D.5)
    # -------------------------------------------------------------------------------------------
    def encode_context(self, text, ip=None, out=None):
        """text: [Bt,77,cross] fp16, ip: [Bt,16,cross] fp16 (Resampler output). Returns per-block (kv_txt, kv_ip),
        each [Bt, T, 2C] = [K | V] produced by attn2.to_k/to_v (and the processor's to_k_ip/to_v_ip). `out`: a list
        returned by an earlier call with the same shapes, overwritten in place (keeps a captured graph valid)."""
        L = self.L
        bt, nt, _ = text.shape
        t2 = text.reshape(bt * nt, -1).to(torch.float16).contiguous()
        i2 = None
        if ip is not None and self.ip_tokens:
            i2 = ip.reshape(bt * ip.shape[1], -1).to(torch.float16).contiguous()
        ctx = []
        for j, blk in enumerate(self.blocks()):
            o_t = out[j][0].view(bt * nt, 2 * blk.c) if out is not None else None
            kv_t = L.gemm(t2, blk.wkv_txt, out=o_t).view(bt, nt, 2 * blk.c)
            kv_i = None
            if i2 is not None:
                o_i = out[j][1].view(bt * ip.shape[1], 2 * blk.c) if out is not None else None
                kv_i = L.gemm(i2, blk.wkv_ip, out=o_i).view(bt, ip.shape[1], 2 * blk.c)
            ctx.append((kv_t, kv_i))
        return ctx

    def aug_embedding(self, text_embeds, time_ids, out=None):
        """add_embedding(concat(text_embeds, Timesteps(time_ids))) — step-invariant (src/unet_hacked_tryon.py:1174-1190)."""
        L = self.L
        b = text_embeds.shape[0]
        dim = self.cfg["addition_time_embed_dim"]
        te = L.timestep_embedding(time_ids.flatten().to(torch.float32).contiguous(), dim).view(b, -1)
        add = torch.cat([text_embeds.to(torch.float16), te], dim=-1).contiguous()
        if out is None:
            out = torch.empty((b, self.ae[2].shape[0]), dtype=torch.float16, device=self.device)
        for r0 in range(0, b, 16):                          # the skinny-linear kernel takes <= 16 rows per launch
            r1 = min(b, r0 + 16)
            h = L.skinny_linear(add[r0:r1], self.ae[0], self.ae[1], out_silu=True)
            L.skinny_linear(h, self.ae[2], self.ae[3], out=out[r0:r1])
        return out

    # -------------------------------------------------------------------------------------------
    # per-step pieces
    # -------------------------------------------------------------------------------------------
    def time_embedding(self, t_dev, batch, aug_emb=None):
        """t_dev: fp32 device tensor with 1 value (broadcast to `batch` rows) or `batch` values (one timestep per
        sample: the hoisted garment pass). Returns the per-resnet time_emb_proj outputs [batch, sum(Cout)]."""
        L = self.L
        n = t_dev.numel()
        assert n == 1 or n == batch
        t_emb = L.timestep_embedding(t_dev, self.ch[0], rows_repeat=batch if n == 1 else 1)
        out = torch.empty((batch, self.temb_w.shape[0]), dtype=torch.float16, device=self.device)
        for r0 in range(0, batch, 16):                      # the skinny-linear kernel takes <= 16 rows per launch
            r1 = min(batch, r0 + 16)
            h = L.skinny_linear(t_emb[r0:r1], self.te[0], self.te[1], out_silu=True)
            emb = L.skinny_linear(h, self.te[2], self.te[3], addend=None if aug_emb is None else aug_emb[r0:r1])
            L.skinny_linear(emb, self.temb_w, self.temb_b, in_silu=True, out=out[r0:r1])
        return out

    def _resnet(self, r, x0, x1, temb_all):
        L = self.L
        h = L.groupnorm(x0, r.n1w, r.n1b, 1e-5, True, x1=x1)
        h = L.conv3x3(h, r.w1, bias=r.b1, temb=temb_all[:, r.temb_off:r.temb_off + r.cout])
        h = L.groupnorm(h, r.n2w, r.n2b, 1e-5, True)
        if r.wsc is not None:
            return L.conv3x3(h, r.w2, bias=r.b2, sc0=x0, sc1=x1, w_sc=r.wsc, bias_sc=r.bsc)
        assert x1 is None
        return L.conv3x3(h, r.w2, bias=r.b2, residual=x0)

    def release_kv_scratch(self):
        """Drops the fp16 scratch of garment_kv's FP8 route (called after a run of hoisted passes, so the memory goes back
        to the allocator that the K/V budgets count as available)."""
        self._kv_scratch = None

    def garment_kv(self, blk, gfeat, out=None):
        """K/V of garment tokens as the TRY-ON UNet sees them: attn1.to_k / to_v applied to the garment UNet's
        post-norm1 feature (src/attentionhacked_tryon.py:334 + ip_adapter/attention_processor.py:247-248).
        gfeat [n, Ng, C] -> [n, Ng, 2C] = [K | V]. out may be a lib.GarmentKV8: the fp16 K/V then go to a scratch
        buffer reused across calls and are quantized into it (the same GEMM, so the same fp16 bits before the rule)."""
        n, ng, C = gfeat.shape
        if isinstance(out, self.L.GarmentKV8):
            need = n * ng * 2 * C
            if self._kv_scratch is None or self._kv_scratch.numel() < need:
                self._kv_scratch = None
                self._kv_scratch = torch.empty(need, dtype=torch.float16, device=self.device)
            kv = self.garment_kv(blk, gfeat, out=self._kv_scratch[:need].view(n, ng, 2 * C))
            return self.L.quantize_kv_e4m3(kv, out)
        o2 = None if out is None else out.view(n * ng, 2 * C)
        return self.L.gemm(gfeat.reshape(n * ng, C), blk.wqkv[C:], out=o2).view(n, ng, 2 * C)

    def _block(self, blk, h, B, N, ctx, gfeat, n_persons, collect, gkv_pre=None):
        """h: [B*N, C]. gfeat: garment feature for this block ([Bg,Ng,C], try-on fast path), a full [B,Ng,C] tensor
        (reference-format features through the module seam) or None (garment UNet). gkv_pre = (kv [T*Bg,Ng,2C],
        n_garments, step_base int32 device scalar): garment K/V precomputed for all denoise steps; or (pool [P*T,Ng,2C],
        rows int32 device [B - n_persons]): a pool of hoisted K/V pages, person sample j reading row rows[j] (negative:
        zero K/V, an idle slot). The hoisted K/V may be a lib.GarmentKV8 (FP8 garment K/V) in either form."""
        L = self.L
        C, H = blk.c, blk.heads
        f8 = blk.fp8
        if f8 is not None:
            # FP8 linears: each LayerNorm also writes its output quantized per row, the input of the e4m3 GEMM after it
            n1q, n1s, n1 = L.layernorm_e4m3(h, blk.ln1w, blk.ln1b, fp16_out=collect is not None)
        else:
            n1 = L.layernorm(h, blk.ln1w, blk.ln1b)
        if collect is not None:
            collect.append(n1.view(B, N, C))                 # src/attentionhacked_garmnet.py:321-322
            if len(collect) == self.n_blocks:
                # Last export of the garment UNet: everything after this norm1 (attn1/attn2/FF of this block, proj_out,
                # the upsampler) only feeds `sample`, which the pipeline discards (src/tryon_pipeline.py:1787).
                raise _GarmentDone()
        if f8 is not None:
            qkv = L.gemm_e4m3(n1q, n1s, *f8["qkv"]).view(B, N, 3 * C)
        else:
            qkv = L.gemm(n1, blk.wqkv).view(B, N, 3 * C)
        q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
        if gkv_pre is not None and len(gkv_pre) == 2:
            pool, rows = gkv_pre
            if isinstance(pool, L.GarmentKV8):
                a = L.attention_kv8(q, k, v, pool, kv1_off=n_persons, heads=H, kv1_rows=rows)
            else:
                a = L.attention_rows(q, k, v, pool[..., :C], pool[..., C:], rows, kv1_off=n_persons, heads=H)
        elif gkv_pre is not None:
            kv_all, n_g, base = gkv_pre
            if isinstance(kv_all, L.GarmentKV8):
                a = L.attention_kv8(q, k, v, kv_all, kv1_off=n_persons, heads=H, kv1_mod=n_g, kv1_base=base)
            else:
                a = L.attention(q, k, v, kv_all[..., :C], kv_all[..., C:], kv1_off=n_persons, heads=H, kv1_mod=n_g,
                                kv1_base=base)
        elif gfeat is None:
            a = L.attention(q, k, v, heads=H)
        else:
            bg, ng, _ = gfeat.shape
            gkv = self.garment_kv(blk, gfeat)
            off = 0 if bg == B else n_persons       # full-format features: every sample has its own segment 1
            a = L.attention(q, k, v, gkv[..., :C], gkv[..., C:], kv1_off=off, heads=H)
        h = L.gemm(a.view(B * N, C), blk.wo1, bias=blk.bo1, residual=h)
        if f8 is not None:
            n2q, n2s, _ = L.layernorm_e4m3(h, blk.ln2w, blk.ln2b)
            q2 = L.gemm_e4m3(n2q, n2s, *f8["q2"]).view(B, N, C)
        else:
            q2 = L.gemm(L.layernorm(h, blk.ln2w, blk.ln2b), blk.wq2).view(B, N, C)
        kv_t, kv_i = ctx
        if kv_t.shape[1] <= 80 and (kv_i is None or kv_i.shape[1] <= 16):
            # text + image-token cross-attention fused in one launch (both key sets fit one score tile)
            a2 = L.cross_attention(q2, kv_t[..., :C], kv_t[..., C:], None if kv_i is None else kv_i[..., :C],
                                   None if kv_i is None else kv_i[..., C:], heads=H, ip_scale=blk.ip_scale)
        else:
            a2 = L.attention(q2, kv_t[..., :C], kv_t[..., C:], heads=H)
            if kv_i is not None:
                assert blk.ip_scale == 1.0, "ip scale != 1 needs the fused cross-attention kernel"
                L.attention(q2, kv_i[..., :C], kv_i[..., C:], heads=H, accumulate=True, out=a2)
        h = L.gemm(a2.view(B * N, C), blk.wo2, bias=blk.bo2, residual=h)
        # force_bn: the tile width the GEGLU weights were packed for
        if f8 is not None:
            n3q, n3s, _ = L.layernorm_e4m3(h, blk.ln3w, blk.ln3b)
            ff = L.gemm_e4m3(n3q, n3s, *f8["ff1"], bias=blk.bff1, geglu=True, force_bn=blk.ff_bn)
        else:
            ff = L.gemm(L.layernorm(h, blk.ln3w, blk.ln3b), blk.wff1, bias=blk.bff1, geglu=True, force_bn=blk.ff_bn)
        return L.gemm(ff, blk.wff2, bias=blk.bff2, residual=h)

    def _t2d(self, t, x, state):
        L = self.L
        B, Hh, Ww, C = x.shape
        N = Hh * Ww
        hn = L.groupnorm(x, t.nw, t.nb, 1e-6, False)
        h = L.gemm(hn.view(B * N, C), t.win, bias=t.bin)
        for blk in t.blocks:
            i = state["idx"]
            gf = state["gfeats"][i] if state["gfeats"] is not None else None
            gp = None
            if state["gkv_pre"] is not None:
                gp = (state["gkv_pre"][0][i], *state["gkv_pre"][1:])
            h = self._block(blk, h, B, N, state["ctx"][i], gf, state["n_persons"], state["collect"], gp)
            state["idx"] = i + 1
        out = L.gemm(h, t.wout, bias=t.bout, residual=x.view(B * N, C))
        return out.view(B, Hh, Ww, C)

    def forward(self, x_in, temb_all, ctx, gfeats=None, n_persons=0, collect=None, gkv_pre=None):
        """x_in: [B,h,w,64] NHWC fp16 (input channels zero-padded). Returns the try-on eps [B,h,w,16] (first
        out_channels valid) or, for the garment UNet, None (features are appended to `collect`)."""
        try:
            return self._forward(x_in, temb_all, ctx, gfeats, n_persons, collect, gkv_pre)
        except _GarmentDone:
            return None

    def _forward(self, x_in, temb_all, ctx, gfeats, n_persons, collect, gkv_pre=None):
        L = self.L
        cfg = self.cfg
        n_lvl = len(self.ch)
        state = dict(idx=0, ctx=ctx, gfeats=gfeats, n_persons=n_persons, collect=collect, gkv_pre=gkv_pre)
        # forward_upsample_size (src/unet_hacked_tryon.py:1081-1091, src/unet_hacked_garmnet.py:994-1000): when this UNet's
        # own input is not a multiple of 2^num_upsamplers in either dimension, every upsampler resizes to the size of the
        # next skip it will be concatenated with instead of doubling (the stride-2 convolutions round up)
        div = 2 ** (n_lvl - 1)
        forward_upsample_size = x_in.shape[1] % div != 0 or x_in.shape[2] % div != 0
        if forward_upsample_size and getattr(L, "upsample_nearest", None) is None:
            # the resize to a skip's size is a kernel of its own (b200vton_upsample_nearest_nhwc): a binding without it
            # cannot run this size, and says so before the first launch instead of failing deep inside the up path
            raise NotImplementedError(f"latent size {tuple(x_in.shape[1:3])} is not a multiple of {div} (pixel size a "
                                      f"multiple of {8 * div}): the reference's `upsample_size` path needs the "
                                      "nearest-resize kernel b200vton_upsample_nearest_nhwc, which this library binding "
                                      "does not provide")
        x = L.conv3x3(x_in, self.w_in, bias=self.b_in)
        skips = [x]
        for i, lvl in enumerate(self.down):
            for j, r in enumerate(lvl["res"]):
                x = self._resnet(r, x, None, temb_all)
                if lvl["attn"]:
                    x = self._t2d(lvl["attn"][j], x, state)
                skips.append(x)
            if lvl["down"] is not None:
                # Downsample2D (conv3x3 stride 2 pad 1): the same implicit-GEMM kernel, its A map stepping 2 pixels per row
                x = L.conv3x3(x, lvl["down"][0], bias=lvl["down"][1], stride=2)
                skips.append(x)
        x = self._resnet(self.mid_res[0], x, None, temb_all)
        x = self._t2d(self.mid_attn, x, state)
        x = self._resnet(self.mid_res[1], x, None, temb_all)
        freeu = self.freeu_active()
        for i, lvl in enumerate(self.up):
            for j, r in enumerate(lvl["res"]):
                skip = skips.pop()
                if freeu is not None and i < 2:
                    # apply_freeu(resolution_idx=i) before the resnet's cat: stage 0 takes (b1, s1), stage 1 (b2, s2);
                    # x and skip are this step's own buffers, so both are rewritten in place
                    s1, s2, b1, b2 = freeu
                    L.freeu(x, skip, b1 if i == 0 else b2, s1 if i == 0 else s2)
                x = self._resnet(r, x, skip, temb_all)
                if lvl["attn"]:
                    x = self._t2d(lvl["attn"][j], x, state)
            if lvl["up"] is not None:
                # (the reference's upsample_size = down_block_res_samples[-1].shape[2:] after this block's pops, :1357-1362)
                up = L.upsample_nearest(x, skips[-1].shape[1:3]) if forward_upsample_size else L.upsample2x(x)
                x = L.conv3x3(up, lvl["up"][0], bias=lvl["up"][1])
        if self.kind != "tryon":
            return None
        h = L.groupnorm(x, self.no_w, self.no_b, 1e-5, True)
        return L.conv3x3(h, self.w_out, bias=self.b_out)
