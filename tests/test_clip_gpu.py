"""GPU parity of the CLIP towers on the engine's kernels (SURVEY.md 8f row 2; idm-vton_b200/clip.py, csrc/attn_enc.cu).

The reference calls `transformers` modules here (src/tryon_pipeline.py:468-470, 592-612); `transformers` is importable on
the GPU box, so the checker is the module itself: fp32 (TF32 off) = truth, fp16 = the reference's execution mode
(inference.py:268-274 loads the encoders with torch_dtype=float16). Contract as for the UNets (tests/test_fullsize_gpu.py): the
engine must not be further from the fp32 truth than the fp16 module is (+ slack), metric max|a-b| / max(1, max|b|).
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _err(a, b):
    a, b = a.float(), b.float()
    return (a - b).abs().max().item() / max(1.0, b.abs().max().item())


@pytest.fixture(autouse=True)
def _no_tf32():
    """fp32 truth without TF32; the process-wide switches are restored afterwards (later test files rely on the defaults)."""
    prev = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev


# ------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,N,D,causal", [
    (2, 16, 257, 80, False),    # ViT-H image encoder
    (3, 12, 77, 64, True),      # ViT-L text encoder
    (2, 20, 77, 64, True),      # bigG text encoder
    (1, 4, 300, 64, True),      # causal across three key tiles (later tiles fully masked for early rows)
    (2, 3, 130, 48, False),     # ragged second tile, head dim < 64
    (1, 5, 128, 96, False),     # the widest head the kernel takes
    (1, 2, 1, 80, True),        # one token
])
def test_encoder_attention_vs_fp32(B, H, N, D, causal):
    from idm_vton_b200 import lib as L
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + N + D)
    qkv = torch.randn(B, N, 3 * H * D, generator=g, device="cuda", dtype=torch.float16)
    C = H * D
    q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
    out = L.encoder_attention(q, k, v, H, D, causal=causal)
    sp = lambda t: t.float().view(B, N, H, D).transpose(1, 2)
    ref = torch.nn.functional.scaled_dot_product_attention(sp(q), sp(k), sp(v), is_causal=causal)
    ref = ref.transpose(1, 2).reshape(B, N, C)
    e = _err(out, ref)
    print(f"encoder_attention B={B} H={H} N={N} D={D} causal={causal}: {e:.2e}")
    assert torch.isfinite(out).all() and e < 2e-3


def test_encoder_attention_peaky_and_scale():
    """Large logits (max-subtraction matters) and an explicit scale."""
    from idm_vton_b200 import lib as L
    B, H, N, D = 1, 16, 257, 80
    g = torch.Generator(device="cuda").manual_seed(7)
    q = (4 * torch.randn(B, N, H * D, generator=g, device="cuda")).half()
    k = (4 * torch.randn(B, N, H * D, generator=g, device="cuda")).half()
    v = torch.randn(B, N, H * D, generator=g, device="cuda").half()
    out = L.encoder_attention(q, k, v, H, D, scale=0.25)
    sp = lambda t: t.float().view(B, N, H, D).transpose(1, 2)
    ref = torch.nn.functional.scaled_dot_product_attention(sp(q), sp(k), sp(v), scale=0.25).transpose(1, 2).reshape(B, N, H * D)
    assert _err(out, ref) < 3e-3


def test_gemm_quick_gelu_epilogue():
    from idm_vton_b200 import lib as L
    g = torch.Generator(device="cuda").manual_seed(1)
    for M in (154, 1024):      # one and several 128-row tiles
        a = torch.randn(M, 768, generator=g, device="cuda").half()
        w = (torch.randn(3072, 768, generator=g, device="cuda") * 0.05).half()
        b = torch.randn(3072, generator=g, device="cuda").half()
        x = (a.float() @ w.float().t() + b.float()).half().float()
        ref = x * torch.sigmoid(1.702 * x)
        assert _err(L.gemm(a, w, bias=b, quick_gelu=True), ref) < 2e-3
        ref_g = torch.nn.functional.gelu(x)
        assert _err(L.gemm(a, w, bias=b, gelu=True), ref_g) < 2e-3


def test_patchify_and_token_embedding_exact():
    from idm_vton_b200 import lib as L
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randn(2, 3, 224, 224, generator=g, device="cuda").half()
    a = L.patchify(x, 14, 640)
    ref = torch.nn.functional.unfold(x.float(), kernel_size=14, stride=14).transpose(1, 2).reshape(2 * 256, 588).half()
    assert torch.equal(a[:, :588], ref) and not a[:, 588:].any()
    tok = torch.randn(1000, 768, generator=g, device="cuda").half()
    pos = torch.randn(77, 768, generator=g, device="cuda").half()
    ids = torch.randint(0, 1000, (3, 77), generator=g, device="cuda")
    out = L.token_embedding(ids.view(-1), tok, pos, 77)
    ref = (tok[ids] + pos[None]).view(-1, 768)
    assert torch.equal(out, ref)


# ------------------------------------------------------------------------------------------------
# towers against the transformers modules
# ------------------------------------------------------------------------------------------------
def _seeded(module, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in module.named_parameters():
            if p.dim() >= 2 and "embedding" not in n:
                p.copy_(torch.randn(p.shape, generator=g) / math.sqrt(p[0].numel()))
            elif p.dim() >= 2 or "class_embedding" in n:
                p.copy_(torch.randn(p.shape, generator=g) * 0.5)
            elif n.endswith("bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
            else:   # LayerNorm scales
                p.copy_(1.0 + 0.1 * torch.randn(p.shape, generator=g))
    return module.eval()


def _report(name, eng, r16, r32, slack=5e-4, mult=1.5):
    e_eng, e_ref, e_x = _err(eng, r32), _err(r16, r32), _err(eng, r16)
    print(f"{name}: engine vs fp32 {e_eng:.2e}, module fp16 vs fp32 {e_ref:.2e}, engine vs module fp16 {e_x:.2e}")
    assert torch.isfinite(eng.float()).all()
    assert e_eng <= mult * e_ref + slack, f"{name}: engine {e_eng:.3e} vs the fp16 module's own error {e_ref:.3e}"


def test_vision_tower_vit_h_vs_transformers():
    """ViT-H/14 (the geometry of ckpt/image_encoder/config.json): hidden_states[-2] (what the pipeline feeds the Resampler,
    src/tryon_pipeline.py:468), every hidden state, pooled image_embeds."""
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection
    from idm_vton_b200 import lib as L
    from idm_vton_b200.clip import ClipTower, tower_for
    cfg = CLIPVisionConfig(hidden_size=1280, intermediate_size=5120, num_hidden_layers=32, num_attention_heads=16,
                           patch_size=14, image_size=224, projection_dim=1024, hidden_act="gelu")
    m32 = _seeded(CLIPVisionModelWithProjection(cfg), 5).cuda()
    # the same fp16-rounded weights everywhere
    with torch.no_grad():
        for p in m32.parameters():
            p.copy_(p.half().float())
    import copy
    m16 = copy.deepcopy(m32).half()
    x = torch.randn(2, 3, 224, 224, generator=torch.Generator().manual_seed(6)).half().cuda()
    with torch.no_grad():
        o32 = m32(x.float(), output_hidden_states=True)
        o16 = m16(x, output_hidden_states=True)
    tower = tower_for(m16)
    assert isinstance(tower, ClipTower) and tower.D == 80 and tower_for(m16) is tower
    n0 = L.launch_count()
    pen = tower.vision_hidden(x, -2)
    launches = L.launch_count() - n0
    assert launches > 31 * 7
    _report("ViT-H hidden_states[-2]", pen, o16.hidden_states[-2], o32.hidden_states[-2])
    full = tower.vision_forward(x, output_hidden_states=True)
    assert len(full.hidden_states) == 33
    assert torch.equal(full.hidden_states[-2], pen)
    for i in (0, 1, 16, 32):
        _report(f"ViT-H hidden_states[{i}]", full.hidden_states[i], o16.hidden_states[i], o32.hidden_states[i])
    _report("ViT-H image_embeds", full.image_embeds, o16.image_embeds, o32.image_embeds, slack=1e-3)


@pytest.mark.parametrize("name,hidden,inter,layers,heads,act,proj", [
    ("ViT-L text (text_encoder)", 768, 3072, 12, 12, "quick_gelu", None),
    ("bigG text (text_encoder_2)", 1280, 5120, 32, 20, "gelu", 1280),
])
def test_text_towers_vs_transformers(name, hidden, inter, layers, heads, act, proj):
    from transformers import CLIPTextConfig, CLIPTextModel, CLIPTextModelWithProjection
    from idm_vton_b200.clip import tower_for
    cfg = CLIPTextConfig(vocab_size=49408, hidden_size=hidden, intermediate_size=inter, num_hidden_layers=layers,
                         num_attention_heads=heads, max_position_embeddings=77, hidden_act=act,
                         projection_dim=proj or 768, bos_token_id=49406, eos_token_id=49407, pad_token_id=1)
    cls = CLIPTextModelWithProjection if proj else CLIPTextModel
    m32 = _seeded(cls(cfg), 8).cuda()
    with torch.no_grad():
        for p in m32.parameters():
            p.copy_(p.half().float())
    import copy
    m16 = copy.deepcopy(m32).half()
    g = torch.Generator().manual_seed(9)
    ids = torch.randint(0, 49406, (3, 77), generator=g)
    ids[:, 0] = 49406
    for b, n in enumerate((5, 30, 76)):      # EOS then padding, as the tokenizer produces
        ids[b, n] = 49407
        ids[b, n + 1:] = 1 if n < 76 else 49407
    ids = ids.cuda()
    with torch.no_grad():
        o32 = m32(ids, output_hidden_states=True)
        o16 = m16(ids, output_hidden_states=True)
    tower = tower_for(m16)
    assert tower is not None and tower.D == 64
    out = tower.text_forward(ids)
    assert len(out.hidden_states) == layers + 1
    _report(f"{name} hidden_states[-2]", out.hidden_states[-2], o16.hidden_states[-2], o32.hidden_states[-2])
    _report(f"{name} last_hidden_state", out.last_hidden_state, o16.last_hidden_state, o32.last_hidden_state, slack=1e-3)
    if proj:
        _report(f"{name} text_embeds", out.text_embeds, o16.text_embeds, o32.text_embeds, slack=1e-3)
    else:
        _report(f"{name} pooler_output", out.pooler_output, o16.pooler_output, o32.pooler_output, slack=1e-3)


def test_tower_for_declines_what_the_kernels_do_not_cover():
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection
    from idm_vton_b200.clip import tower_for
    cfg = CLIPVisionConfig(hidden_size=96, intermediate_size=192, num_hidden_layers=1, num_attention_heads=4, image_size=28,
                           patch_size=14)
    assert tower_for(CLIPVisionModelWithProjection(cfg).cuda().half()) is None      # hidden % 64 != 0
    cfg = CLIPVisionConfig(hidden_size=128, intermediate_size=256, num_hidden_layers=1, num_attention_heads=2, image_size=28,
                           patch_size=14)
    assert tower_for(CLIPVisionModelWithProjection(cfg).cuda()) is None             # fp32 module: the caller's own path
    m = CLIPVisionModelWithProjection(cfg).cuda().half()
    t = tower_for(m)
    assert t is not None
    with torch.no_grad():
        next(m.parameters()).add_(1.0)                                              # weights changed: re-packed
    assert tower_for(m) is not t
