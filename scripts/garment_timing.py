"""Garment photos and descriptions: the GPU preparation of a garment photo (photo.prepare_garments: resize to the server
size with `cloth`, CLIP resize, CLIP pixels) against the demo's host path, and the two prompt encodes of a description,
per garment, at 3024 x 4032 (a phone photo), 1080 x 1920 and 768 x 1024, for a 768 x 1024 server.

GPU times: CUDA events around prepare_garments with the photo starting as a host uint8 tensor (staged through pinned
memory, so the H2D copy is included) and as a uint8 tensor already on the device; the median over --iters runs after
--warmup. Host times on one thread, the median over --iters: Pillow's resize to the server size, ToTensor + Normalize of
it (torchvision's arithmetic in torch), and transformers' CLIPImageProcessorPil on it.
Prompt encodes: serving.encode_description (the demo's person prompt with CFG and garment prompt) on SDXL-geometry CLIP
text encoders with random fp16 weights (ViT-L/14 text: 768 wide, 12 layers; bigG: 1280 wide, 32 layers, projection
1280) on the engine's CLIP kernels, timed with CUDA events. The tokenizer is byte-level (no merges); every prompt is
padded to 77 tokens, so the encoders' work does not depend on it.
Prints one JSON line per photo size and one for the encodes, with the card's name and power limit read in the same run.

    python scripts/garment_timing.py [--iters 20] [--warmup 3]
"""
import argparse
import json
import os
import sys
import tempfile
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import idm_vton_b200  # noqa: E402,F401
from idm_vton_b200 import photo as P  # noqa: E402
from scripts.photo_timing import _events, _wall  # noqa: E402
from scripts.schedule_timing import card  # noqa: E402


def _byte_tokenizer(d):
    """A CLIPTokenizer over the 2 x 256 byte symbols and the two special tokens (no merges), written to `d`."""
    from transformers import CLIPTokenizer
    bs = list(range(ord("!"), ord("~") + 1)) + list(range(ord("¡"), ord("¬") + 1)) + list(range(ord("®"), ord("ÿ") + 1))
    cs, n = bs[:], 0
    for b in range(256):
        if b not in bs:
            bs.append(b)
            cs.append(256 + n)
            n += 1
    symbols = [chr(c) for _, c in sorted(zip(bs, cs))]
    vocab = {s: i for i, s in enumerate(symbols)}
    vocab.update({s + "</w>": 256 + i for i, s in enumerate(symbols)})
    vocab.update({"<|startoftext|>": 512, "<|endoftext|>": 513})
    with open(os.path.join(d, "vocab.json"), "w") as f:
        json.dump(vocab, f)
    open(os.path.join(d, "merges.txt"), "w").close()
    return CLIPTokenizer(os.path.join(d, "vocab.json"), os.path.join(d, "merges.txt"), model_max_length=77)


def _text_pipeline(dev, tmp):
    """The pipeline's encode_prompt with SDXL-geometry text encoders (random fp16 weights) and a byte-level tokenizer."""
    from transformers import CLIPTextConfig, CLIPTextModel, CLIPTextModelWithProjection
    from idm_vton_b200.pipeline import StableDiffusionXLInpaintPipeline
    common = dict(vocab_size=49408, max_position_embeddings=77, bos_token_id=512, eos_token_id=513, pad_token_id=513)
    te1 = CLIPTextModel(CLIPTextConfig(hidden_size=768, intermediate_size=3072, num_hidden_layers=12,
                                       num_attention_heads=12, hidden_act="quick_gelu", **common))
    te2 = CLIPTextModelWithProjection(CLIPTextConfig(hidden_size=1280, intermediate_size=5120, num_hidden_layers=32,
                                                     num_attention_heads=20, hidden_act="gelu", projection_dim=1280,
                                                     **common))
    tok = _byte_tokenizer(tmp)
    vae = types.SimpleNamespace(config=types.SimpleNamespace(block_out_channels=(1, 2, 3, 4)))
    unet = types.SimpleNamespace(device=dev, dtype=torch.float16)
    return StableDiffusionXLInpaintPipeline(vae=vae, text_encoder=te1.to(dev, torch.float16).eval(),
                                            text_encoder_2=te2.to(dev, torch.float16).eval(), tokenizer=tok,
                                            tokenizer_2=tok, unet=unet, unet_encoder=None, scheduler=None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    the_card = card()
    import PIL.Image
    from transformers import CLIPImageProcessorPil
    h, w = 1024, 768
    processor = CLIPImageProcessorPil()
    g = np.random.default_rng(0)
    for W, H in ((3024, 4032), (1080, 1920), (768, 1024)):
        a = g.integers(0, 256, (H, W, 3), dtype=np.uint8)
        host = torch.from_numpy(a)
        dev = host.cuda()
        gpu_host = _events(lambda: P.prepare_garments([host], h, w), args.iters, args.warmup)
        gpu_dev = _events(lambda: P.prepare_garments([dev], h, w), args.iters, args.warmup)
        img = PIL.Image.fromarray(a)
        garm = img.resize((w, h))

        def to_tensor():
            x = torch.from_numpy(np.array(garm)).permute(2, 0, 1).contiguous().float().div(255)
            return (x - 0.5) / 0.5
        pil_resize = _wall(lambda: img.convert("RGB").resize((w, h)), args.iters, args.warmup)
        tensor = _wall(to_tensor, args.iters, args.warmup)
        clip = _wall(lambda: processor(garm, return_tensors="np"), args.iters, args.warmup)
        print(json.dumps(dict(garment=f"{W}x{H}", server=f"{w}x{h}", card=the_card,
                              gpu_prepare_from_host_ms=round(gpu_host, 3), gpu_prepare_on_device_ms=round(gpu_dev, 3),
                              pillow_convert_resize_ms=round(pil_resize, 2), to_tensor_normalize_ms=round(tensor, 2),
                              clip_image_processor_pil_ms=round(clip, 2),
                              host_total_ms=round(pil_resize + tensor + clip, 2))), flush=True)
    from idm_vton_b200.serving import encode_description
    dev = torch.device("cuda", 0)
    with tempfile.TemporaryDirectory() as tmp, torch.no_grad():
        pipe = _text_pipeline(dev, tmp)
        enc = _events(lambda: encode_description(pipe, "a red striped shirt with long sleeves", dev), args.iters,
                      args.warmup)
        t0 = time.perf_counter()
        encode_description(pipe, "a denim jacket", dev)
        torch.cuda.synchronize()
        once = (time.perf_counter() - t0) * 1e3
    print(json.dumps(dict(prompt_encodes="encode_description: person prompt with CFG (2 x 2 encoders) + garment prompt "
                                         "(2 encoders), SDXL-geometry CLIP text encoders, random fp16 weights",
                          card=the_card, gpu_encode_ms=round(enc, 3), wall_one_call_ms=round(once, 3))), flush=True)


if __name__ == "__main__":
    main()
