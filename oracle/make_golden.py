"""Pins oracle/unet_ref.py against the REFERENCE's own modules and writes tests/golden/*.pt.

Needs a checkout of the original project (IDM_VTON_REFERENCE). The reference's src/*.py and ip_adapter/*.py are imported
UNMODIFIED and in place, on top of the test-only diffusers shim (oracle/shim), with seeded synthetic weights generated
by oracle.unet_ref.make_state_dict (loaded with strict=True: this also pins the state-dict key names / shapes).

Usage:  python oracle/make_golden.py            # compare + (re)write fixtures
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("IDM_VTON_REFERENCE", "")   # checkout of the original IDM-VTON project
GOLDEN = os.path.join(ROOT, "tests", "golden")


def import_reference():
    if not os.path.isdir(REF):
        raise RuntimeError("set IDM_VTON_REFERENCE to a checkout of the original project to regenerate the golden fixtures")
    sys.path.insert(0, os.path.join(ROOT, "oracle", "shim"))
    sys.path.insert(0, REF)
    import src.unet_hacked_tryon as ut  # noqa: E402
    import src.unet_hacked_garmnet as ug  # noqa: E402
    return ut, ug


def build_reference_unet(mod, cfg):
    kw = dict(
        sample_size=32, in_channels=cfg["in_channels"], out_channels=cfg["out_channels"],
        down_block_types=("DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"),
        up_block_types=("CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"),
        block_out_channels=tuple(cfg["block_out_channels"]), layers_per_block=cfg["layers_per_block"],
        cross_attention_dim=cfg["cross_attention_dim"],
        transformer_layers_per_block=list(cfg["transformer_layers_per_block"]),
        attention_head_dim=list(cfg["num_heads"]), use_linear_projection=True,
        projection_class_embeddings_input_dim=cfg["projection_class_embeddings_input_dim"],
        addition_time_embed_dim=cfg["addition_time_embed_dim"],
    )
    if cfg["text_time"]:
        kw["addition_embed_type"] = "text_time"
    if cfg.get("resampler"):
        kw["encoder_hid_dim"] = cfg["resampler"]["embedding_dim"]
        kw["encoder_hid_dim_type"] = "ip_image_proj"
    return mod.UNet2DConditionModel(**kw).eval()


def synth_inputs(cfg_t, cfg_g, B, h, w, seed=1234):
    """Synthetic step inputs for B persons (CFG => try-on batch 2B, garment batch B), latent h x w."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    cross = cfg_t["cross_attention_dim"]
    pooled = cfg_t["projection_class_embeddings_input_dim"] - 6 * cfg_t["addition_time_embed_dim"]
    return dict(
        sample=r(2 * B, cfg_t["in_channels"], h, w),
        timestep=torch.tensor(967),
        prompt_embeds=r(2 * B, 77, cross),
        text_embeds=r(2 * B, pooled),
        time_ids=torch.tensor([[h * 8.0, w * 8.0, 0.0, 0.0, h * 8.0, w * 8.0]]).repeat(2 * B, 1),
        clip_tokens=r(2 * B, 257, cfg_t["resampler"]["embedding_dim"]),
        cloth=r(B, cfg_g["in_channels"], h, w),
        text_embeds_cloth=r(B, 77, cfg_g["cross_attention_dim"]),
    )


def main():
    from oracle import unet_ref as R
    ut, ug = import_reference()
    os.makedirs(GOLDEN, exist_ok=True)
    torch.manual_seed(0)
    cfg_t, cfg_g = R.tiny_config("tryon"), R.tiny_config("garment")
    sd_t, sd_g = R.make_state_dict(cfg_t, seed=11), R.make_state_dict(cfg_g, seed=22)

    net_t, net_g = build_reference_unet(ut, cfg_t), build_reference_unet(ug, cfg_g)
    # strict=True pins key names and shapes. The garment reference module also owns the never-used tail
    # (up_blocks.2 / conv_norm_out / conv_out, App. D.7); our generated dict contains those keys too.
    missing_t = net_t.load_state_dict(sd_t, strict=True)
    missing_g = net_g.load_state_dict(sd_g, strict=True)
    print("state dict pinned:", len(sd_t), "try-on keys,", len(sd_g), "garment keys", missing_t, missing_g)

    B, h, w = 1, 16, 16
    x = synth_inputs(cfg_t, cfg_g, B, h, w)
    with torch.no_grad():
        # ---- Resampler (once per request; src/tryon_pipeline.py:1726)
        img_ref = net_t.encoder_hid_proj(x["clip_tokens"])
        img_ora = R.resampler_forward(sd_t, "encoder_hid_proj", cfg_t["resampler"], x["clip_tokens"])
        print("resampler      max|d| =", (img_ref - img_ora).abs().max().item())
        # ---- garment UNet -> 70-style feature list
        _, feats_ref = net_g(x["cloth"], x["timestep"], x["text_embeds_cloth"], return_dict=False)
        feats_ora = R.unet_garment_forward(sd_g, cfg_g, x["cloth"], x["timestep"], x["text_embeds_cloth"])
        assert len(feats_ref) == len(feats_ora), (len(feats_ref), len(feats_ora))
        d_feat = max((a - b).abs().max().item() for a, b in zip(feats_ref, feats_ora))
        print(f"garment UNet   {len(feats_ref)} features, max|d| = {d_feat}")
        # ---- CFG zero-padding of the features (src/tryon_pipeline.py:1796) + try-on UNet
        feats_cfg = [torch.cat([torch.zeros_like(d), d]) for d in feats_ref]
        added = {"text_embeds": x["text_embeds"], "time_ids": x["time_ids"], "image_embeds": img_ref}
        out_ref = net_t(x["sample"], x["timestep"], encoder_hidden_states=x["prompt_embeds"],
                        added_cond_kwargs=added, return_dict=False, garment_features=feats_cfg)[0]
        out_ora = R.unet_tryon_forward(sd_t, cfg_t, x["sample"], x["timestep"], x["prompt_embeds"], added, feats_cfg)
        d_out = (out_ref - out_ora).abs().max().item()
        print("try-on UNet    max|d| =", d_out, " |out|max =", out_ref.abs().max().item())
    tol = 2e-5
    assert (img_ref - img_ora).abs().max().item() < tol * max(1, img_ref.abs().max().item())
    assert d_feat < 1e-4 and d_out < 1e-4, "oracle restatement deviates from the reference modules"

    torch.save({
        "note": "outputs of the REFERENCE modules (src/unet_hacked_*.py on the diffusers shim), CPU fp32, tiny config; "
                "weights = oracle.unet_ref.make_state_dict(tiny_config(kind), seed=11 (tryon) / 22 (garment)); "
                "inputs = oracle.make_golden.synth_inputs(B=1, h=16, w=16, seed=1234)",
        "B": B, "h": h, "w": w,
        "image_embeds": img_ref.half(),
        "garment_feature_0": feats_ref[0].half(), "garment_feature_last": feats_ref[-1].half(),
        "garment_feature_norms": torch.tensor([f.float().norm().item() for f in feats_ref]),
        "noise_pred": out_ref.half(),
    }, os.path.join(GOLDEN, "unet_tiny_ref.pt"))
    print("wrote", os.path.join(GOLDEN, "unet_tiny_ref.pt"))


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    main()
