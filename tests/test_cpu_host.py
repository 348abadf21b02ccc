"""CPU-side tests (no GPU): oracle pinning against the reference-module golden fixture, C-ABI export check, host logic
(weight packing, parameter inventory, scheduler, request sharding incl. a 2-rank gloo run), pipeline signature parity."""
import ast
import ctypes
import json
import math
import os
import re
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


# ------------------------------------------------------------------------------------------------
# oracle pinned to the reference
# ------------------------------------------------------------------------------------------------
def test_oracle_matches_reference_golden():
    """oracle/unet_ref.py (CPU fp32) reproduces the outputs of the reference's own modules (fixture written by
    oracle/make_golden.py from src/unet_hacked_*.py running on the diffusers shim)."""
    from oracle import unet_ref as R
    from oracle.make_golden import synth_inputs
    g = torch.load(os.path.join(GOLDEN, "unet_tiny_ref.pt"))
    cfg_t, cfg_g = R.tiny_config("tryon"), R.tiny_config("garment")
    sd_t, sd_g = R.make_state_dict(cfg_t, seed=11), R.make_state_dict(cfg_g, seed=22)
    x = synth_inputs(cfg_t, cfg_g, g["B"], g["h"], g["w"])
    with torch.no_grad():
        img = R.resampler_forward(sd_t, "encoder_hid_proj", cfg_t["resampler"], x["clip_tokens"])
        feats = R.unet_garment_forward(sd_g, cfg_g, x["cloth"], x["timestep"], x["text_embeds_cloth"])
        fc = [torch.cat([torch.zeros_like(d), d]) for d in feats]
        added = {"text_embeds": x["text_embeds"], "time_ids": x["time_ids"], "image_embeds": img}
        eps = R.unet_tryon_forward(sd_t, cfg_t, x["sample"], x["timestep"], x["prompt_embeds"], added, fc)
    # the fixture is stored in fp16: compare at fp16 resolution
    assert torch.allclose(img, g["image_embeds"].float(), atol=2e-3, rtol=2e-3)
    assert len(feats) == len(g["garment_feature_norms"]) == 17
    norms = torch.tensor([f.norm().item() for f in feats])
    assert torch.allclose(norms, g["garment_feature_norms"], rtol=1e-4)
    assert torch.allclose(feats[0], g["garment_feature_0"].float(), atol=2e-3, rtol=2e-3)
    assert torch.allclose(feats[-1], g["garment_feature_last"].float(), atol=2e-3, rtol=2e-3)
    assert torch.allclose(eps, g["noise_pred"].float(), atol=2e-3, rtol=2e-3)


def test_oracle_self_checks():
    """Independent invariants of the restated diffusers leaf ops (SURVEY.md App. D.8)."""
    from oracle import loop_ref as LR
    from oracle import unet_ref as R
    # sinusoidal embedding: [cos | sin], frequency 0 -> cos=1, sin=0; highest frequency index = 1/10000^(159/160)
    e = R.timesteps_proj(torch.tensor([0.0, 500.0]), 320)
    assert torch.allclose(e[0, :160], torch.ones(160)) and torch.allclose(e[0, 160:], torch.zeros(160))
    assert abs(e[1, 0].item() - math.cos(500.0)) < 1e-4 and abs(e[1, 160].item() - math.sin(500.0)) < 1e-4
    # scheduler: alphas_cumprod against the closed form for scaled-linear betas; 30 leading steps = 33k+1
    s = LR.DDPMRef()
    betas = torch.linspace(0.00085 ** 0.5, 0.012 ** 0.5, 1000, dtype=torch.float64) ** 2
    assert torch.allclose(s.alphas_cumprod.double(), torch.cumprod(1 - betas, 0), rtol=1e-5)
    ts = s.set_timesteps(30)
    assert ts.tolist() == [33 * k + 1 for k in range(29, -1, -1)]
    # zero-SNR rescale drives the terminal alpha-bar to 0
    z = LR.DDPMRef(rescale_betas_zero_snr=True)
    assert z.alphas_cumprod[-1].abs() < 1e-10 and abs(z.alphas_cumprod[0] - s.alphas_cumprod[0]) < 1e-6
    # zero garment features only add Ng * exp(-m) to the denominator (App. D.3)
    torch.manual_seed(0)
    q, k, v = torch.randn(1, 1, 8, 64).double(), torch.randn(1, 1, 24, 64).double(), torch.randn(1, 1, 24, 64).double()
    kz, vz = torch.cat([k, torch.zeros(1, 1, 16, 64).double()], 2), torch.cat([v, torch.zeros(1, 1, 16, 64).double()], 2)
    full = torch.softmax(q @ kz.transpose(-1, -2) / 8, -1) @ vz
    sc = q @ k.transpose(-1, -2) / 8
    m = torch.clamp(sc.max(-1, keepdim=True).values, min=0)
    p = torch.exp(sc - m)
    closed = (p @ v) / (p.sum(-1, keepdim=True) + 16 * torch.exp(-m))
    assert torch.allclose(full, closed, atol=1e-12)


def test_param_inventory_matches_oracle_and_reference_counts():
    from idm_vton_b200 import unet as U
    from oracle import unet_ref as R
    for prod, ora in ((U.SDXL_TRYON, R.SDXL_TRYON), (U.SDXL_GARMENT, R.SDXL_GARMENT),
                      (R.tiny_config("tryon"), R.tiny_config("tryon"))):
        a, b = U.param_shapes(prod), R.unet_param_shapes(ora)
        assert sorted(a.keys()) == sorted(b.keys())
        assert all(tuple(a[k]) == tuple(b[k]) for k in a)
    n_t = sum(math.prod(s) for s in U.param_shapes(U.SDXL_TRYON).values())
    n_g = sum(math.prod(s) for s in U.param_shapes(U.SDXL_GARMENT).values())
    # SDXL-base UNet has 2,567,463,684 params incl. add_embedding (5,245,440), which the garment UNet drops
    # (train_xl.py:323-325 addition_embed_type=None)
    assert n_g == 2_567_463_684 - 5_245_440
    assert 2.98e9 < n_t < 3.0e9
    assert len([k for k in U.param_shapes(U.SDXL_TRYON) if k.endswith("attn2.processor.to_k_ip.weight")]) == 70


def test_loop_oracle_pinned_by_reference_pipeline():
    """oracle/loop_ref.py (denoise_loop + DDPMRef) against the latents the REFERENCE pipeline produced
    (tests/golden/pipeline_call_ref.pt, made by oracle/make_golden_pipeline.py from src/tryon_pipeline.py itself): the loop
    oracle is pinned, not merely self-consistent. Also pins both schedulers' timestep lists and the host-side step()."""
    from idm_vton_b200.scheduler import DDPMScheduler
    from oracle import loop_ref as LR
    from oracle import unet_ref as R
    g = torch.load(os.path.join(ROOT, "tests", "golden", "pipeline_call_ref.pt"))
    cfg_t, cfg_g = R.tiny_config("tryon"), R.tiny_config("garment")
    sd_t = {k: v.half().float() for k, v in R.make_state_dict(cfg_t, seed=11).items()}
    sd_g = {k: v.half().float() for k, v in R.make_state_dict(cfg_g, seed=22).items()}
    steps = len(g["latents_per_step"])
    assert LR.DDPMRef().set_timesteps(steps).tolist() == g["timesteps"].tolist()
    s = DDPMScheduler()
    s.set_timesteps(steps)
    assert s.timesteps.tolist() == g["timesteps"].tolist()
    with torch.no_grad():
        for n in range(1, steps + 1):
            lat = LR.denoise_loop(sd_t, cfg_t, sd_g, cfg_g, g["loop_inputs"], steps, guidance_scale=2.0,
                                  noises=g["noises"], max_steps=n)
            ref = g["latents_per_step"][n - 1]
            assert (lat - ref).abs().max().item() <= 1e-4 * max(1.0, ref.abs().max().item())
    assert g["n_features"] == 17 and g["loop_inputs"]["mask"].shape[0] == 2 * g["loop_inputs"]["latents"].shape[0]


def test_garment_unet_ingests_sdxl_base_checkpoint_keys():
    """ADVICE r1: GarmentNet's checkpoint is the SDXL-base UNet (train_xl.py:323-325 nulls addition_embed_type only after
    construction), so it carries add_embedding.* which the garment forward never reads. strict loading must accept the full
    key set (and still reject keys that are neither used nor known-dead)."""
    from idm_vton_b200 import unet as U
    from oracle import unet_ref as R
    cfg = R.tiny_config("garment")
    sd = R.make_state_dict(cfg, seed=2)
    temb = cfg["block_out_channels"][0] * 4
    full = dict(sd)
    full.update({"add_embedding.linear_1.weight": torch.zeros(temb, cfg["projection_class_embeddings_input_dim"]),
                 "add_embedding.linear_1.bias": torch.zeros(temb), "add_embedding.linear_2.weight": torch.zeros(temb, temb),
                 "add_embedding.linear_2.bias": torch.zeros(temb)})
    net = U.UNet2DConditionModelGarment(cfg, dtype=torch.float32)
    res = net.load_state_dict(full, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    assert torch.equal(net.state_dict()["conv_in.weight"], sd["conv_in.weight"])
    with pytest.raises(RuntimeError, match="Unexpected key"):
        net.load_state_dict(dict(full, **{"controlnet_cond.weight": torch.zeros(1)}), strict=True)
    tnet = U.UNet2DConditionModel(R.tiny_config("tryon"), dtype=torch.float32)        # the try-on UNet uses add_embedding
    assert "add_embedding.linear_1.weight" in tnet.state_dict()


def test_serving_batches_by_garment_and_encodes_each_garment_once():
    """serving.TryOnServer (SURVEY.md 8f item 4) on a stand-in pipeline: requests are grouped by garment in arrival order of
    their oldest member, a batch never mixes garments or exceeds max_batch, every garment is VAE-encoded once and handed
    to the pipeline as latents + its cache key; tickets map results back to requests."""
    import types
    from idm_vton_b200.denoise import GarmentKVCache
    from idm_vton_b200.serving import TryOnRequest, TryOnServer
    calls, encodes = [], []

    class FakePipe:
        _execution_device = torch.device("cpu")
        unet = types.SimpleNamespace(dtype=torch.float32)
        garment_cache = None

        def _encode_vae_image(self, image, generator=None):
            encodes.append(tuple(image.shape))
            return image[:, :1].repeat(1, 4, 1, 1)[..., ::8, ::8] * 0 + image.mean()

        def __call__(self, **kw):
            B = kw["prompt_embeds"].shape[0]
            assert kw["cloth"].shape == (1, 4, 4, 4) and kw["text_embeds_cloth"].shape[0] == 1 and kw["ip_adapter_image"].shape[0] == 1
            calls.append((B, tuple(kw["garment_keys"]), float(kw["cloth"].mean())))
            return (kw["image"] + kw["cloth"].mean(),)

    srv = TryOnServer(FakePipe(), height=32, width=32, num_inference_steps=2, max_batch=2, seed=None)
    assert isinstance(srv.pipe.garment_cache, GarmentKVCache)

    def req(gid, val, with_garment=True):
        z = torch.zeros
        return TryOnRequest(garment_id=gid, image=z(3, 32, 32) + val, mask_image=z(1, 32, 32), pose_img=z(3, 32, 32),
                            prompt_embeds=z(77, 8), negative_prompt_embeds=z(77, 8), pooled_prompt_embeds=z(4),
                            negative_pooled_prompt_embeds=z(4), cloth=(z(3, 32, 32) + {"A": 1.0, "B": 2.0}[gid]) if with_garment else None,
                            ip_adapter_image=z(3, 224, 224) if with_garment else None, text_embeds_cloth=z(77, 8) if with_garment else None)

    with pytest.raises(ValueError, match="is new"):
        srv.submit(req("A", 0.0, with_garment=False))
    t = [srv.submit(req("A", 0.1)), srv.submit(req("B", 0.2)), srv.submit(req("A", 0.3)), srv.submit(req("A", 0.4, with_garment=False))]
    out = srv.run()
    assert calls == [(2, ("A",), 1.0), (1, ("B",), 2.0), (1, ("A",), 1.0)]          # A's oldest first, max_batch 2, then B, then A's rest
    assert encodes == [(1, 3, 32, 32)] * 2 and srv.stats["garments_encoded"] == 2 and srv.stats["images"] == 4
    assert sorted(out) == t and abs(float(out[t[3]].mean()) - 1.4) < 1e-6 and abs(float(out[t[1]].mean()) - 2.2) < 1e-6
    # LRU behaviour of the K/V cache itself
    c = GarmentKVCache(max_bytes=100)
    c.put("a", [torch.zeros(10, dtype=torch.float32)])
    c.put("b", [torch.zeros(10, dtype=torch.float32)])
    assert c.get("a") is not None
    c.put("c", [torch.zeros(10, dtype=torch.float32)])                            # evicts b (least recently used)
    assert c.get("b") is None and c.get("a") is not None and c.get("c") is not None and c.bytes == 80


def test_engine_rejects_latent_sizes_the_up_path_cannot_match():
    """Latent sizes that are not a multiple of the total downsampling factor need diffusers' `upsample_size` path
    (src/unet_hacked_tryon.py:1051-1064), which the engine does not implement: a clear error, not a shape mismatch deep
    inside the launch sequence."""
    import types
    from idm_vton_b200.engine import UNetEngine
    eng = object.__new__(UNetEngine)
    eng.L, eng.cfg, eng.ch, eng.kind = types.SimpleNamespace(), {}, (64, 128, 256), "tryon"
    with pytest.raises(NotImplementedError, match="multiple of 4"):
        eng._forward(torch.zeros(1, 18, 16, 64), None, None, None, 0, None)


def test_generic_scheduler_interface():
    """ADVICE r1: the denoiser derives its per-step coefficients from the generic DDPM interface (alphas_cumprod,
    config, num_inference_steps), so the caller's own scheduler object works; unsupported configs raise."""
    from idm_vton_b200.denoise import ddpm_step_coefficients
    from idm_vton_b200.scheduler import DDPMScheduler
    for kw in ({}, {"rescale_betas_zero_snr": True}):
        s = DDPMScheduler(**kw)
        s.set_timesteps(30)
        assert all(ddpm_step_coefficients(s, int(t)) == s.step_coefficients(int(t)) for t in s.timesteps)

    class Foreign:          # what a diffusers DDPMScheduler exposes (no step_coefficients / previous_timestep)
        def __init__(self, **over):
            self.alphas_cumprod = DDPMScheduler().alphas_cumprod
            self.config = dict(num_train_timesteps=1000, prediction_type="epsilon", variance_type="fixed_small",
                               clip_sample=False, **over)
            self.num_inference_steps = 30

    s = DDPMScheduler()
    s.set_timesteps(30)
    assert ddpm_step_coefficients(Foreign(), 967) == s.step_coefficients(967)
    with pytest.raises(NotImplementedError):
        ddpm_step_coefficients(Foreign(thresholding=True), 967)
    with pytest.raises(TypeError):
        ddpm_step_coefficients(object(), 967)


def test_attention_processor_seam_structure():
    """Seam B3 on the host: every Attention layer exposes a processor under the reference's names
    (src/unet_hacked_tryon.py:793-852), IP weights live in `...attn2.processor.to_{k,v}_ip.weight`
    (ip_adapter/attention_processor.py:1904-1905), set_attn_processor validates like the reference, and the processors
    refuse CPU tensors instead of falling back to PyTorch."""
    from idm_vton_b200 import unet as U
    from idm_vton_b200.attention_processor import Attention, AttnProcessor2_0, IPAttnProcessor2_0
    from oracle import unet_ref as R
    cfg_t, cfg_g = R.tiny_config("tryon"), R.tiny_config("garment")
    net = U.UNet2DConditionModel(cfg_t, R.make_state_dict(cfg_t, seed=1), dtype=torch.float32)
    gar = U.UNet2DConditionModelGarment(cfg_g, R.make_state_dict(cfg_g, seed=2), dtype=torch.float32)
    procs = net.attn_processors
    n_blocks = 17
    assert len(procs) == 2 * n_blocks and len(gar.attn_processors) == 2 * n_blocks
    assert all(k.endswith(".attn1.processor") or k.endswith(".attn2.processor") for k in procs)
    assert all(type(p) is (IPAttnProcessor2_0 if k.endswith("attn2.processor") else AttnProcessor2_0) for k, p in procs.items())
    assert all(type(p) is AttnProcessor2_0 for p in gar.attn_processors.values())
    assert sorted(net.state_dict()) == sorted(R.unet_param_shapes(cfg_t))       # registering processors adds no keys
    k0 = "down_blocks.1.attentions.0.transformer_blocks.0.attn2.processor"
    assert procs[k0].num_tokens == 16 and procs[k0].scale == 1.0
    assert procs[k0].to_k_ip.weight is net.state_dict(keep_vars=True)[k0 + ".to_k_ip.weight"]
    attn = dict(net.named_modules())[k0[:-len(".processor")]]
    assert isinstance(attn, Attention) and attn.heads == 2 and attn.to_out[0].bias is not None
    # reference error for a dict of the wrong size (src/unet_hacked_tryon.py:833-837)
    with pytest.raises(ValueError, match="does not match the number of attention layers: 34"):
        net.set_attn_processor({k0: procs[k0]})
    with pytest.raises(TypeError, match="IPAttnProcessor2_0"):
        net.set_attn_processor(AttnProcessor2_0())
    bad = {k: (IPAttnProcessor2_0(128, 256, num_tokens=4) if k == k0 else p) for k, p in procs.items()}
    with pytest.raises(ValueError, match="num_tokens"):
        net.set_attn_processor(bad)
    new = {k: (IPAttnProcessor2_0(p.hidden_size, p.cross_attention_dim, scale=0.25, num_tokens=16)
               if isinstance(p, IPAttnProcessor2_0) else AttnProcessor2_0()) for k, p in procs.items()}
    net.set_attn_processor(dict(new))
    assert net.attn_processors[k0] is new[k0] and net._ip_scales()[k0[:-len(".attn2.processor")]] == 0.25
    assert net.state_dict(keep_vars=True)[k0 + ".to_v_ip.weight"] is new[k0].to_v_ip.weight
    gar.set_attn_processor(AttnProcessor2_0())          # one processor for all layers
    # no CPU / PyTorch fallback behind the protocol
    a = Attention(query_dim=128, heads=2)
    with pytest.raises(RuntimeError, match="no PyTorch fallback"):
        a(torch.zeros(1, 8, 128))


# ------------------------------------------------------------------------------------------------
# C ABI
# ------------------------------------------------------------------------------------------------
def test_c_abi_exports_every_declared_symbol():
    from idm_vton_b200 import build, lib
    path = build.build()
    header = open(os.path.join(ROOT, "include", "b200vton.h")).read()
    declared = sorted(set(re.findall(r"\b(b200vton_\w+)\s*\(", header)))
    assert len(declared) >= 14
    so = ctypes.CDLL(path)
    for name in declared:
        assert hasattr(so, name), f"{name} declared in include/b200vton.h but not exported"
    assert set(lib.SIGNATURES) <= set(declared)
    l = lib.load()
    assert l.b200vton_version() == lib.ABI_VERSION
    # argument validation happens before any CUDA work: invalid shapes return an error code + message, no crash
    rc = l.b200vton_gemm_f16(None, 8, None, 8, None, 8, 16, 16, 60, None, None, 0, None, 0, 0, 0, 0, None)
    assert rc == 1 and b"multiple of 64" in l.b200vton_last_error()
    rc = l.b200vton_skinny_linear(None, 8, 17, 64, None, 64, 8, None, 0, 0, None, 0, None, 8, None)
    assert rc == 1 and b"out of range" in l.b200vton_last_error()


def test_clip_tower_packing_and_dispatch_on_cpu():
    """clip.ClipTower packs a transformers CLIP module's own state dict (fused QKV, zero-padded patch weight, class token +
    position 0); tower_for() leaves CPU / fp32 modules to the caller; the encoder-attention entry point validates its
    arguments before any CUDA work."""
    from transformers import CLIPTextConfig, CLIPTextModelWithProjection, CLIPVisionConfig, CLIPVisionModelWithProjection
    from idm_vton_b200 import lib
    from idm_vton_b200.clip import ClipTower, tower_for
    cfg = CLIPVisionConfig(hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=2, image_size=28,
                           patch_size=14, projection_dim=64, hidden_act="gelu")
    m = CLIPVisionModelWithProjection(cfg).eval()
    assert tower_for(m) is None                                   # CPU module: the caller's own path
    t = ClipTower(m.state_dict(), cfg, "vision", "cpu")
    sd = m.state_dict()
    assert t.D == 64 and t.K == 588 and t.Kp == 640 and t.w_patch.shape == (128, 640) and not t.w_patch[:, 588:].any()
    assert torch.equal(t.w_patch[:, :588], sd["vision_model.embeddings.patch_embedding.weight"].half().reshape(128, 588))
    assert torch.equal(t.blocks[1].wqkv[128:256], sd["vision_model.encoder.layers.1.self_attn.k_proj.weight"].half())
    assert torch.equal(t.blocks[0].bqkv[256:], sd["vision_model.encoder.layers.0.self_attn.v_proj.bias"].half())
    pos = sd["vision_model.embeddings.position_embedding.weight"].half()
    assert torch.equal(t.cls_pos0, sd["vision_model.embeddings.class_embedding"].half() + pos[0]) and t.pos_patches.shape == (4, 128)
    tc = CLIPTextConfig(vocab_size=100, hidden_size=64, intermediate_size=128, num_hidden_layers=1, num_attention_heads=1,
                        max_position_embeddings=77, projection_dim=32, hidden_act="quick_gelu", eos_token_id=99)
    tt = ClipTower(CLIPTextModelWithProjection(tc).state_dict(), tc, "text", "cpu")
    assert tt.act == {"quick_gelu": True} and tt.proj.shape == (32, 64) and tt.eos_token_id == 99
    with pytest.raises(ValueError):
        ClipTower(m.state_dict(), dict(hidden_size=96, num_attention_heads=4, num_hidden_layers=2, intermediate_size=192,
                                       hidden_act="gelu"), "vision", "cpu")
    l = lib.load()
    rc = l.b200vton_encoder_attention(None, 8, None, None, 8, None, 8, 1, 1, 16, 72, 1.0, 0, None)
    assert rc == 1 and b"head dim" in l.b200vton_last_error()


def test_clip_tower_control_flow_on_cpu(monkeypatch):
    """The towers' launch sequence (which hidden state index -2 is, class token / position wiring, causal text attention,
    EOS pooling, projection heads) checked on CPU: the lib wrappers are replaced by plain-torch stand-ins of the kernels'
    contracts (fp16 in, fp32 arithmetic, fp16 out) and the results compared with the transformers modules in fp32.
    (The kernels themselves: tests/test_clip_gpu.py.)"""
    import torch.nn.functional as F
    from transformers import CLIPTextConfig, CLIPTextModelWithProjection, CLIPVisionConfig, CLIPVisionModelWithProjection
    from idm_vton_b200 import clip as CL

    def gemm(a, w, bias=None, residual=None, gelu=False, quick_gelu=False, out=None, **k):
        y = a.float() @ w.float().t()
        if bias is not None:
            y = y + bias.float()
        if gelu:
            y = F.gelu(y)
        if quick_gelu:
            y = y * torch.sigmoid(1.702 * y)
        if residual is not None:
            y = y + residual.float()
        if out is not None:
            out.copy_(y)
            return out
        return y.half()

    def attention(q, k, v, heads, head_dim, scale=None, causal=False, out=None):
        B, N, _ = q.shape
        sp = lambda t: t.float().reshape(B, N, heads, head_dim).transpose(1, 2)
        o = F.scaled_dot_product_attention(sp(q), sp(k), sp(v), is_causal=causal, scale=scale)
        return o.transpose(1, 2).reshape(B, N, heads * head_dim).half()

    def patchify(x, P, ldk):
        a = F.unfold(x.float(), kernel_size=P, stride=P).transpose(1, 2).reshape(-1, x.shape[1] * P * P)
        return F.pad(a, (0, ldk - a.shape[1])).half()

    monkeypatch.setattr(CL.L, "gemm", gemm)
    monkeypatch.setattr(CL.L, "layernorm", lambda x, g, b, eps=1e-5, out=None:
                        F.layer_norm(x.float(), (x.shape[-1],), g.float(), b.float(), eps).half())
    monkeypatch.setattr(CL.L, "encoder_attention", attention)
    monkeypatch.setattr(CL.L, "patchify", patchify)
    monkeypatch.setattr(CL.L, "token_embedding",
                        lambda ids, tok, pos, T: (tok.float()[ids] + pos.float()[torch.arange(ids.numel()) % T]).half())
    monkeypatch.setattr(CL.L, "skinny_linear", lambda x, w, **k: (x.float() @ w.float().t()).half())

    def rounded(module):
        with torch.no_grad():
            for prm in module.parameters():
                prm.copy_(prm.half().float())          # the tower stores fp16 weights
        return module.eval()

    def close(a, b, tol=1e-2):
        return (a.float() - b).abs().max().item() <= tol * max(1.0, b.abs().max().item())
    torch.manual_seed(0)
    vc = CLIPVisionConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=3, num_attention_heads=2, image_size=28,
                          patch_size=14, projection_dim=32, hidden_act="gelu")
    m = rounded(CLIPVisionModelWithProjection(vc))
    t = CL.ClipTower(m.state_dict(), vc, "vision", "cpu")
    x = torch.randn(2, 3, 28, 28).half()
    with torch.no_grad():
        ref = m(x.float(), output_hidden_states=True)
    full = t.vision_forward(x, output_hidden_states=True)
    assert len(full.hidden_states) == 4 == len(ref.hidden_states)
    assert all(close(a, b) for a, b in zip(full.hidden_states, ref.hidden_states))
    assert close(t.vision_hidden(x, -2), ref.hidden_states[-2]) and not close(t.vision_hidden(x, -2), ref.hidden_states[-1])
    assert close(full.image_embeds, ref.image_embeds)
    with pytest.raises(ValueError, match="patches"):
        t.vision_hidden(torch.zeros(1, 3, 42, 42).half())
    for eos in (2, 99):                      # legacy argmax pooling / first-EOS pooling
        tc = CLIPTextConfig(vocab_size=100, hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=1,
                            max_position_embeddings=16, projection_dim=32, hidden_act="quick_gelu", eos_token_id=eos,
                            bos_token_id=0, pad_token_id=1)
        tm = rounded(CLIPTextModelWithProjection(tc))
        tt = CL.ClipTower(tm.state_dict(), tc, "text", "cpu")
        ids = torch.randint(3, 98, (3, 16))
        ids[0, 5], ids[1, 9], ids[2, 15] = 99, 99, 99
        ids[0, 6:] = 1
        with torch.no_grad():
            tr = tm(ids, output_hidden_states=True)
        to = tt.text_forward(ids)
        assert len(to.hidden_states) == 3 and all(close(a, b) for a, b in zip(to.hidden_states, tr.hidden_states))
        assert close(to.last_hidden_state, tr.last_hidden_state) and close(to.text_embeds, tr.text_embeds, 2e-2)


def test_product_does_not_import_oracle():
    """The product path must never route through the oracle or any CPU fallback."""
    pkg = os.path.join(ROOT, "idm-vton_b200")
    for fn in os.listdir(pkg):
        if fn.endswith(".py"):
            src = open(os.path.join(pkg, fn)).read()
            tree = ast.parse(src)
            for node in ast.walk(tree):
                mods = []
                if isinstance(node, ast.Import):
                    mods = [a.name for a in node.names]
                elif isinstance(node, ast.ImportFrom) and node.module:
                    mods = [node.module]
                assert not any(m == "oracle" or m.startswith("oracle.") for m in mods), f"{fn} imports the oracle"


def test_ops_fail_loudly_without_gpu():
    from idm_vton_b200 import unet as U
    from oracle import unet_ref as R
    cfg = R.tiny_config("garment")
    m = U.UNet2DConditionModelGarment(cfg, R.make_state_dict(cfg, seed=1))
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError, match="no CPU / PyTorch fallback"):
        m(torch.zeros(1, 4, 8, 8), 1, torch.zeros(1, 77, cfg["cross_attention_dim"]), return_dict=False)


# ------------------------------------------------------------------------------------------------
# host logic
# ------------------------------------------------------------------------------------------------
def test_weight_packing():
    from idm_vton_b200.engine import pack_conv3x3, pack_conv3x3_s2, pack_geglu, pad_channels
    w = torch.arange(2 * 3 * 9, dtype=torch.float32).reshape(2, 3, 3, 3)
    p = pack_conv3x3(w)
    assert p.shape == (9, 2, 3) and p[4, 1, 2] == w[1, 2, 1, 1] and p[2, 0, 1] == w[0, 1, 0, 2]
    assert pad_channels(p, cin_to=8, cout_to=4).shape == (9, 4, 8) and pad_channels(p, 8, 4)[:, 2:].abs().sum() == 0
    s2 = pack_conv3x3_s2(w)
    assert s2.shape == (2, 27) and s2[1, 5 * 3 + 2] == w[1, 2, 1, 2]
    C = 64
    wg = torch.randn(8 * C, C)
    bg = torch.randn(8 * C)
    x = torch.randn(5, C)
    wp, bp = pack_geglu(wg, bg, 128)
    ref = x @ wg.t() + bg
    pk = (x @ wp.t() + bp).reshape(5, 4 * C // 64, 2, 64)
    assert torch.allclose(pk[:, :, 0].reshape(5, -1), ref[:, :4 * C], atol=1e-5)
    assert torch.allclose(pk[:, :, 1].reshape(5, -1), ref[:, 4 * C:], atol=1e-5)


def test_scheduler_matches_oracle_and_formulas():
    from idm_vton_b200.scheduler import DDPMScheduler
    from oracle import loop_ref as LR
    for zsnr in (False, True):
        s, r = DDPMScheduler(rescale_betas_zero_snr=zsnr), LR.DDPMRef(rescale_betas_zero_snr=zsnr)
        s.set_timesteps(30)
        assert s.timesteps.tolist() == r.set_timesteps(30).tolist()
        assert torch.allclose(s.alphas_cumprod, r.alphas_cumprod)
        g = torch.Generator().manual_seed(0)
        x, eps, n = (torch.randn(2, 4, 8, 8, generator=g) for _ in range(3))
        for t in (958, 496, 1):
            sb, inv_sa, c0, c1, sigma = s.step_coefficients(t)
            mine = c0 * ((x - sb * eps) * inv_sa) + c1 * x + sigma * n
            assert torch.allclose(mine, r.step(eps, t, x, noise=n), atol=1e-4, rtol=1e-4)
    with pytest.raises(ValueError):
        DDPMScheduler().set_timesteps(2000)


def test_shard_requests_partition():
    from idm_vton_b200.parallel import shard_requests
    for n, w in ((64, 8), (10, 4), (3, 8), (0, 2)):
        parts = [list(shard_requests(n, w, r)) for r in range(w)]
        assert sum(parts, []) == list(range(n))
        assert max(len(p) for p in parts) - min(len(p) for p in parts) <= 1
    assert list(shard_requests(64, 8, 3)) == list(range(24, 32))
    with pytest.raises(ValueError):
        shard_requests(4, 2, 2)


def _gloo_worker(rank, world, port, out):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    sys.path.insert(0, ROOT)
    from idm_vton_b200.parallel import broadcast_state_dict, shard_requests
    g = torch.Generator().manual_seed(123)
    sd = {f"w{i}": (torch.randn(7 + i, 5, generator=g) if rank == 0 else torch.zeros(7 + i, 5)) for i in range(6)}
    sd["h"] = torch.randn(9, generator=g).half() if rank == 0 else torch.zeros(9).half()
    broadcast_state_dict(sd, src=0, bucket_bytes=200)
    # the path bench.py uses: one flat arena per UNet, views as the state dict, broadcast in place in buckets
    from idm_vton_b200.parallel import alloc_state_dict_arena, broadcast_arena
    shapes = {"a": (3, 5), "b": (130,), "c": (2, 2, 2)}
    views, flat = alloc_state_dict_arena(shapes, torch.float32, "cpu", align=8)
    assert all(v.data_ptr() % 32 == 0 and tuple(v.shape) == shapes[k] for k, v in views.items())
    for k, v in views.items():
        v.copy_(torch.randn(shapes[k], generator=g) if rank == 0 else torch.zeros(shapes[k]))
    broadcast_arena(flat, src=0, bucket_bytes=64)
    sd.update({f"arena_{k}": v for k, v in views.items()})
    chk = torch.tensor([sum(v.double().sum().item() for v in sd.values())], dtype=torch.float64)
    dist.all_reduce(chk, op=dist.ReduceOp.MAX)
    mine = list(shard_requests(10, world, rank))
    t = torch.tensor([float(len(mine))])
    dist.all_reduce(t)                       # every request is owned exactly once
    # device-time max over ranks, as bench.py reports it
    el = torch.tensor([1.0 + rank])
    dist.all_reduce(el, op=dist.ReduceOp.MAX)
    if rank == 0:
        out.put((chk.item(), t.item(), el.item(), sum(v.double().sum().item() for v in sd.values())))
    dist.destroy_process_group()


def test_two_rank_gloo_broadcast_and_sharding():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 2000
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    chk, n_owned, el, local = q.get(timeout=10)
    assert abs(chk - local) < 1e-9 and n_owned == 10 and el == 2.0


def test_bench_flop_model_matches_baseline_table():
    import bench
    from idm_vton_b200.engine import SDXL_GARMENT, SDXL_TRYON
    t = bench.unet_macs(SDXL_TRYON, 128, 96, tryon=True) / 1e9
    g = bench.unet_macs(SDXL_GARMENT, 128, 96, tryon=False) / 1e9
    assert abs(t - 2867) < 2 and abs(g - 2349) < 2                       # SURVEY.md App. B
    assert abs(bench.step_flops(SDXL_TRYON, SDXL_GARMENT, 128, 96, 2, 2) / 1e12 - 32.34) < 0.05   # BASELINE.md cfg 2
    assert abs(bench.unet_macs(SDXL_TRYON, 128, 128, tryon=True) / 1e9 - 4001) < 3                # 1024^2


# ------------------------------------------------------------------------------------------------
# drop-in surface
# ------------------------------------------------------------------------------------------------
def _sig(fn):
    a = fn.args
    names = [x.arg for x in a.args]
    return {"args": names, "defaults": [None] * (len(names) - len(a.defaults)) + [ast.unparse(d) for d in a.defaults],
            "kwarg": a.kwarg.arg if a.kwarg else None}


def test_pipeline_signatures_equal_reference():
    """__init__ / encode_prompt / __call__ / check_inputs: same parameter names, order, defaults and **kwargs as
    src/tryon_pipeline.py (golden extracted from the reference by oracle/make_signature_golden.py)."""
    gold = json.load(open(os.path.join(GOLDEN, "pipeline_signature.json")))["signatures"]
    tree = ast.parse(open(os.path.join(ROOT, "idm-vton_b200", "pipeline.py")).read())
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "StableDiffusionXLInpaintPipeline")
    mine = {f.name: _sig(f) for f in cls.body if isinstance(f, ast.FunctionDef) and f.name in gold}
    for name, g in gold.items():
        assert mine[name]["args"] == g["args"], name
        assert mine[name]["kwarg"] == g["kwarg"], name
        for arg, dm, dg in zip(g["args"], mine[name]["defaults"], g["defaults"]):
            assert dm == dg, f"{name}({arg}): default {dm} != reference {dg}"


def test_pipeline_check_inputs_errors():
    from idm_vton_b200.pipeline import StableDiffusionXLInpaintPipeline as P
    from idm_vton_b200.scheduler import DDPMScheduler
    from idm_vton_b200.vae import AutoencoderKL
    import types
    unet = types.SimpleNamespace(config=types.SimpleNamespace(time_cond_proj_dim=None, sample_size=128, in_channels=13),
                                 device=torch.device("cpu"))
    p = P(AutoencoderKL(block_out_channels=(32, 32), layers_per_block=1), None, None, None, None, unet, None, DDPMScheduler())
    assert p.vae_scale_factor == 2
    with pytest.raises(ValueError, match="divisible by 8"):
        p.check_inputs(None, None, None, None, 100, 64, 1.0, None, "pil", prompt_embeds=torch.zeros(1, 77, 8))
    with pytest.raises(ValueError, match="strength"):
        p.check_inputs(None, None, None, None, 64, 64, 1.5, None, "pil", prompt_embeds=torch.zeros(1, 77, 8))
    with pytest.raises(ValueError, match="Provide either"):
        p.check_inputs(None, None, None, None, 64, 64, 1.0, None, "pil")
    with pytest.raises(ValueError, match="Cannot forward both"):
        p.check_inputs("a", None, None, None, 64, 64, 1.0, None, "pil", prompt_embeds=torch.zeros(1, 77, 8))
    with pytest.raises(ValueError, match="same shape"):
        p.check_inputs(None, None, None, None, 64, 64, 1.0, None, "pil", prompt_embeds=torch.zeros(1, 77, 8),
                       negative_prompt_embeds=torch.zeros(1, 70, 8))


def test_vae_and_image_processor_plumbing():
    from idm_vton_b200.vae import AutoencoderKL, VaeImageProcessor
    torch.manual_seed(0)
    vae = AutoencoderKL(block_out_channels=(32, 64), layers_per_block=1)
    x = torch.rand(1, 3, 32, 32) * 2 - 1
    z = vae.encode(x).latent_dist.sample(torch.Generator().manual_seed(1))
    assert z.shape == (1, 4, 16, 16)
    assert vae.decode(z, return_dict=False)[0].shape == (1, 3, 32, 32)
    ip = VaeImageProcessor(vae_scale_factor=8)
    t = ip.preprocess(torch.rand(2, 3, 16, 16), height=16, width=16)
    assert t.min() >= -1 and t.max() <= 1 and t.min() < 0
    mp_ = VaeImageProcessor(vae_scale_factor=8, do_normalize=False, do_binarize=True, do_convert_grayscale=True)
    m = mp_.preprocess(torch.rand(2, 1, 16, 16), height=16, width=16)
    assert set(m.unique().tolist()) <= {0.0, 1.0}
    pil = ip.postprocess(torch.zeros(1, 3, 8, 8), output_type="pil")
    assert pil[0].size == (8, 8)


def test_library_options_and_argument_checks_without_gpu():
    """Every option name the header documents is accepted, unknown names are rejected with a message, and the new entry
    points validate their arguments before any CUDA work (error code 1 + message, no crash, no GPU needed)."""
    from idm_vton_b200 import lib
    l = lib.load()
    header = open(os.path.join(ROOT, "include", "b200vton.h")).read()
    block = header[header.index("/* library options:"):header.index("int b200vton_set_option")]
    names = sorted(set(re.findall(r'"([a-z0-9_]+)"', block)))
    assert {"gemm_2cta_auto", "gemm_cluster4", "programmatic_launch", "attention_pingpong", "attention_q_tiles",
            "attention_poly_exp"} <= set(names)
    defaults = {"gemm_2cta_auto": 1, "gemm_cluster4": 0, "programmatic_launch": 0, "attention_pingpong": 1,
                "attention_q_tiles": 0, "attention_poly_exp": 0}
    for n in names:
        assert n in defaults, f"option {n} documented in the header but not covered here"
        assert l.b200vton_set_option(n.encode(), defaults[n]) == 0
    assert l.b200vton_set_option(b"no_such_option", 1) != 0 and b"unknown option" in l.b200vton_last_error()
    # fused cross-attention: context sizes beyond one score tile are refused (the engine then uses the 2-launch path)
    rc = l.b200vton_cross_attention(None, 64, None, None, 64, 81, None, None, 0, 0, None, 64, 1, 1, 128, 0.125, 1.0, None)
    assert rc == 1 and b"Nt <= 80" in l.b200vton_last_error()
    rc = l.b200vton_cross_attention(None, 64, None, None, 64, 77, None, None, 64, 17, None, 64, 1, 1, 128, 0.125, 1.0, None)
    assert rc == 1
    # fp32/TF32 convolution: channel alignment
    rc = l.b200vton_conv3x3_nhwc_f32(None, 1, 16, 16, 48, None, 64, None, None, None, None)
    assert rc == 1 and b"multiples of 32" in l.b200vton_last_error()
    assert l.b200vton_split_tf32(None, 6, 1, 6, 1.0, None, None, None) == 1 and b"split_tf32" in l.b200vton_last_error()
    assert l.b200vton_softmax_split_tf32(None, 4, 6, None, None, None) == 1
    # operands the kernels access with 16-byte vectors (4-byte stores for attention's out) must be aligned, and the row
    # strides of residual / rowvec / temb multiples of 8 halves: refused before any tensor map is encoded or anything
    # launched (fake device addresses, never dereferenced)
    A, OK, BAD, BAD4 = 0x10000, 0x20000, 0x20008, 0x20002
    gemm = l.b200vton_gemm_f16
    for kw in ("out", "bias", "residual", "rowvec"):
        ptr = {k: OK for k in ("out", "bias", "residual", "rowvec")}
        ptr[kw] = BAD
        rc = gemm(A, 64, A, 64, ptr["out"], 64, 128, 64, 64, ptr["bias"], ptr["residual"], 64, ptr["rowvec"], 64, 128, 0,
                  0, None)
        assert rc == 1 and b"16-byte aligned" in l.b200vton_last_error(), kw
    assert gemm(A, 64, A, 64, OK, 64, 128, 64, 64, None, OK, 68, None, 0, 0, 0, 0, None) == 1
    assert b"ldr=68" in l.b200vton_last_error()
    assert gemm(A, 64, A, 64, OK, 64, 128, 64, 64, None, None, 0, OK, 36, 77, 0, 0, None) == 1
    assert b"ld_rowvec=36" in l.b200vton_last_error()
    conv = l.b200vton_conv3x3_nhwc
    for kw in ("out", "bias", "temb", "bias_sc", "residual"):
        ptr = {k: OK for k in ("out", "bias", "temb", "bias_sc", "residual")}
        ptr[kw] = BAD
        sc = kw == "bias_sc"          # a shortcut and an identity residual are exclusive
        rc = conv(A, 64, 1, 8, 8, 64, A, 64, ptr["bias"], ptr["temb"], 64, A if sc else None, 64 if sc else 0, None, 0,
                  A if sc else None, ptr["bias_sc"] if sc else None, None if sc else ptr["residual"], 64, ptr["out"], 64,
                  0, 1, None)
        assert rc == 1 and b"16-byte aligned" in l.b200vton_last_error(), kw
    assert conv(A, 64, 2, 8, 8, 64, A, 64, None, OK, 1284, None, 0, None, 0, None, None, None, 0, OK, 64, 0, 1, None) == 1
    assert b"ld_temb=1284" in l.b200vton_last_error()
    assert conv(A, 64, 1, 8, 8, 64, A, 64, None, None, 0, None, 0, None, 0, None, None, OK, 60, OK, 64, 0, 1, None) == 1
    assert b"ldr=60" in l.b200vton_last_error()
    rc = l.b200vton_attention(A, 64, A, A, 64, None, None, 0, BAD4, 64, 1, 1, 128, 128, 0, 0, 0, 0, None, 0.125, 0, None)
    assert rc == 1 and b"4-byte aligned" in l.b200vton_last_error()
    rc = l.b200vton_cross_attention(A, 64, A, A, 64, 77, None, None, 0, 0, BAD4, 64, 1, 1, 128, 0.125, 1.0, None)
    assert rc == 1 and b"4-byte aligned" in l.b200vton_last_error()
    rc = l.b200vton_encoder_attention(A, 64, A, A, 64, BAD4, 64, 1, 1, 77, 64, 0.125, 1, None)
    assert rc == 1 and b"4-byte aligned" in l.b200vton_last_error()
    for x0, x1, out in ((BAD, None, OK), (OK, BAD, OK), (OK, OK, BAD)):
        rc = l.b200vton_groupnorm(x0, 320, x1, 64 if x1 else 0, 1, 64, None, None, 1e-5, 1, OK, out, None)
        assert rc == 1 and b"16-byte aligned" in l.b200vton_last_error()
    for x, g, b, out in ((BAD, None, None, OK), (OK, BAD, None, OK), (OK, None, BAD, OK), (OK, None, None, BAD)):
        rc = l.b200vton_layernorm(x, 640, 4, 640, g, b, 1e-5, out, 640, None)
        assert rc == 1 and b"16-byte aligned" in l.b200vton_last_error()


def test_vae_conv_dispatch_and_weight_packing_on_cpu():
    """The VAE's engine-convolution switch never engages on CPU tensors (plain nn.Conv2d result), and the fp32 weight
    packing is the tap-major [9, Cout, Cin] layout the kernel's weight map expects."""
    import idm_vton_b200.vae as V
    from idm_vton_b200 import lib
    conv = torch.nn.Conv2d(32, 64, 3, padding=1)
    x = torch.randn(1, 32, 8, 8)
    assert torch.equal(V._conv(conv, x), conv(x))
    assert not lib.conv3x3_f32_supported(x, 32, 64)                       # CPU tensor
    wp = lib.pack_conv3x3_f32(conv.weight)
    assert wp.shape == (9, 64, 32) and wp.is_contiguous()
    for tap in (0, 4, 8):
        assert torch.equal(wp[tap], conv.weight[:, :, tap // 3, tap % 3])


def test_vae_nhwc_path_control_flow_on_cpu(monkeypatch):
    """The experimental NHWC route through the VAE (engine GroupNorm + TF32 convolution kernels, B200VTON_VAE_NHWC=1)
    with the two kernels replaced by PyTorch stand-ins that honour the same layout contract (channels_last in and
    out, packed [9,Cout,Cin] weights): layout handling, the token view of the mid-block attention and the residual
    adds must reproduce the default path."""
    import idm_vton_b200.vae as V
    from idm_vton_b200 import lib

    def fake_gn(x, gamma, beta, eps, silu, out_half=False):
        assert x.is_contiguous(memory_format=torch.channels_last)
        y = torch.nn.functional.group_norm(x, 32, gamma, beta, eps)
        y = torch.nn.functional.silu(y) if silu else y
        y = y.contiguous(memory_format=torch.channels_last)
        return y.half() if out_half else y

    def fake_conv16(x16, w_packed16, bias=None, residual=None):       # fp16 operands, fp32 arithmetic and output
        assert x16.dtype == torch.float16 and w_packed16.dtype == torch.float16
        assert x16.is_contiguous(memory_format=torch.channels_last)
        calls["conv16"] += 1
        return fake_conv(x16.float(), w_packed16.float(), bias, residual)

    def fake_conv(x, w_packed, bias=None, residual=None):
        cout, cin = w_packed.shape[1], w_packed.shape[2]
        w = w_packed.reshape(3, 3, cout, cin).permute(2, 3, 0, 1)
        y = torch.nn.functional.conv2d(x, w, bias, padding=1)
        if residual is not None:                       # the kernel's epilogue: (acc + bias) + residual
            calls["residual"] += 1
            y = y + residual
        return y.contiguous(memory_format=torch.channels_last)

    calls = {"conv": 0, "residual": 0, "conv16": 0}
    torch.manual_seed(0)
    vae = V.AutoencoderKL(block_out_channels=(32, 64), layers_per_block=1).eval()
    x = torch.rand(2, 3, 32, 24) * 2 - 1
    with torch.no_grad():
        ref_mean = vae.encode(x).latent_dist.mean
        z = torch.randn(2, 4, 16, 12)
        ref_img = vae.decode(z).sample
        monkeypatch.setattr(V, "_use_nhwc", lambda t: t.dim() == 4 and t.dtype == torch.float32)
        monkeypatch.setattr(V, "_ENGINE_NHWC", True)
        monkeypatch.setattr(lib, "groupnorm_f32_nhwc", fake_gn)
        monkeypatch.setattr(lib, "conv3x3_f32", fake_conv)
        monkeypatch.setattr(lib, "conv3x3_f32_supported", lambda t, cin, cout: cin % 32 == 0 and cout % 32 == 0 and cout >= 64)
        monkeypatch.setattr(V, "_conv_device_ok", lambda t: True)
        real_fake = fake_conv

        def counting_conv(x, w_packed, bias=None, residual=None):
            calls["conv"] += 1
            return real_fake(x, w_packed, bias, residual)

        monkeypatch.setattr(lib, "conv3x3_f32", counting_conv)
        monkeypatch.setattr(lib, "conv3x3_f16in", fake_conv16)
        monkeypatch.setattr(V, "_F16_ACT", False)
        got_mean = vae.encode(x).latent_dist.mean
        got_img = vae.decode(z).sample
        assert calls["conv"] > 0, "the engine-convolution route was not taken"
        assert calls["residual"] > 0, "the resnets' residual add did not ride in the convolution's epilogue"
        assert calls["conv16"] == 0
        assert got_mean.shape == ref_mean.shape and got_img.shape == ref_img.shape and got_img.is_contiguous()
        assert (got_mean - ref_mean).abs().max() < 1e-4
        assert (got_img - ref_img).abs().max() < 1e-4
        # GroupNorm(+SiLU) -> convolution with the fp16 hand-off (64-aligned input channels only): fp16 rounding of the operands
        monkeypatch.setattr(V, "_F16_ACT", True)
        h_mean = vae.encode(x).latent_dist.mean
        h_img = vae.decode(z).sample
        assert calls["conv16"] > 0, "the fp16 hand-off was not taken"
        assert (h_mean - ref_mean).abs().max() < 5e-3 * max(1.0, ref_mean.abs().max().item())
        assert (h_img - ref_img).abs().max() < 5e-3 * max(1.0, ref_img.abs().max().item())


def test_bench_emits_a_line_when_the_e2e_section_stalls():
    """bench.py's safety net: value / roofline are measured before the e2e section, and if that section does not return
    within B200VTON_E2E_TIMEOUT the line is still printed (e2e marked unavailable) and the process exits NON-ZERO (3): a
    hang must not surface as rc=0 (VERDICT r1)."""
    import json
    import subprocess
    import sys
    probe = os.path.join(ROOT, "tests", "helpers", "bench_guard_probe.py")
    r = subprocess.run([sys.executable, probe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 3, r.stderr[-2000:]
    lines = [l for l in r.stdout.strip().splitlines() if l.startswith("{")]
    assert len(lines) == 1 and "SHOULD NOT REACH" not in r.stdout
    d = json.loads(lines[0])
    assert d["value"] == 2.0 and d["e2e"]["value"] is None and "did not finish" in d["e2e"]["unavailable"]
    for key in ("metric", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
                "dtype", "data", "config", "roofline", "cpu_baseline", "gpu_launches", "clocks"):
        assert key in d
