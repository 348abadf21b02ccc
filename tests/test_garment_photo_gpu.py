"""Garment photos and descriptions on the GPU:
  * photo.prepare_garments equals the demo's host path bit for bit on the sweep of tests/test_garment_photo_cpu.py:
    Pillow's convert + resize (image_u8), ToTensor + Normalize (cloth) and CLIPImageProcessorPil (clip_pixels); a ragged
    batch of five garments in one call (three calls, five launches) equals each garment prepared alone;
  * the servers (tiny config at 256 x 192, so the CLIP centre crop is exercised, with tiny fp16 CLIP text encoders on
    the engine's kernels): a request with garment_photo and garment_description gives final latents bit-identical to
    the same request with every garment and prompt tensor made on the host the demo's way, in TryOnServer and in
    ContinuousTryOnServer (default and pool mode); a second request for the garment encodes nothing and gets the same
    bits; a request with a person photo and a garment photo runs beside a plain tensor request in one batch.
"""
import json

import numpy as np
import pytest
import torch

from test_garment_photo_cpu import PIL, SWEEP, _case_id, clip_pil, demo_cloth, demo_garment, garment_photo

pytestmark = pytest.mark.gpu

H, W = 256, 192
DESC = "a red striped shirt with long sleeves"


@pytest.mark.parametrize("case", SWEEP, ids=_case_id)
def test_prepare_garments_equals_the_demos_host_path(case):
    from idm_vton_b200 import photo as P
    (gw, gh, mode), (h, w) = case
    photo = garment_photo(gw, gh, mode)
    garm = demo_garment(photo, h, w)
    e = P.prepare_garments([photo], h, w)[0]
    assert np.array_equal(e.image_u8.cpu().numpy(), np.asarray(garm))
    assert e.cloth.dtype == torch.float32 and torch.equal(e.cloth.cpu(), demo_cloth(garm))
    assert e.clip_pixels.dtype == torch.float32 and np.array_equal(e.clip_pixels.cpu().numpy(), clip_pil(garm))


def test_ragged_batch_in_one_call_equals_each_alone():
    from idm_vton_b200 import lib, photo as P
    photos = [garment_photo(3024, 4032, "RGB", 1), garment_photo(1080, 1920, "RGBA", 2), garment_photo(77, 91, "P", 3),
              garment_photo(1, 1, "RGB", 4), garment_photo(500, 300, "L", 5)]
    inputs = [photos[0], torch.from_numpy(np.asarray(photos[1].convert("RGB")).copy()), photos[2],
              torch.from_numpy(np.asarray(photos[3])).cuda(), photos[4]]            # PIL, CPU and CUDA tensors
    n0 = lib.launch_count()
    batch = P.prepare_garments(inputs, 397, 301)
    assert lib.launch_count() - n0 == 5          # two resample calls of two passes each, one CLIP-pixels launch
    for x, b in zip(inputs, batch):
        alone = P.prepare_garments([x], 397, 301)[0]
        for f in ("image_u8", "cloth", "clip_pixels"):
            assert torch.equal(getattr(b, f), getattr(alone, f)), f


# ------------------------------------------------------------------------------------------------
# the servers (tiny config)
# ------------------------------------------------------------------------------------------------
from test_continuous_gpu import _drive, tiny_modules  # noqa: E402,F401


def _bytes_to_unicode():
    """GPT-2's byte-to-symbol table (the one CLIP's BPE vocabulary is written in)."""
    bs = list(range(ord("!"), ord("~") + 1)) + list(range(ord("¡"), ord("¬") + 1)) + list(range(ord("®"), ord("ÿ") + 1))
    cs, n = bs[:], 0
    for b in range(256):
        if b not in bs:
            bs.append(b)
            cs.append(256 + n)
            n += 1
    return [chr(c) for _, c in sorted(zip(bs, cs))]


@pytest.fixture(scope="module")
def text_pipe(tiny_modules, tmp_path_factory):
    """The tiny pipeline with a byte-level CLIPTokenizer (no merges: one token per byte) and two fp16 CLIP text encoders
    on the GPU: hidden 128 + 128 = the tiny UNet's cross_attention_dim 256, projection 128 = its pooled width."""
    from transformers import CLIPTextConfig, CLIPTextModel, CLIPTextModelWithProjection, CLIPTokenizer
    from oracle import make_golden_pipeline as MG
    from idm_vton_b200.clip import tower_for
    from idm_vton_b200.pipeline import StableDiffusionXLInpaintPipeline
    from idm_vton_b200.scheduler import DDPMScheduler
    d = tmp_path_factory.mktemp("tokenizer")
    symbols = _bytes_to_unicode()
    vocab = {s: i for i, s in enumerate(symbols)}
    vocab.update({s + "</w>": 256 + i for i, s in enumerate(symbols)})
    vocab.update({"<|startoftext|>": 512, "<|endoftext|>": 513})
    (d / "vocab.json").write_text(json.dumps(vocab))
    (d / "merges.txt").write_text("")
    tok = CLIPTokenizer(str(d / "vocab.json"), str(d / "merges.txt"), model_max_length=77)
    cfg = dict(vocab_size=514, hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=2,
               max_position_embeddings=77, bos_token_id=512, eos_token_id=513, pad_token_id=513)
    te1 = MG.seeded_fill_(CLIPTextModel(CLIPTextConfig(hidden_act="quick_gelu", **cfg)), seed=41)
    te2 = MG.seeded_fill_(CLIPTextModelWithProjection(CLIPTextConfig(hidden_act="gelu", projection_dim=128, **cfg)),
                          seed=42)
    te1, te2 = te1.to("cuda", torch.float16).eval(), te2.to("cuda", torch.float16).eval()
    assert tower_for(te1) is not None and tower_for(te2) is not None      # the engine's CLIP kernels
    return StableDiffusionXLInpaintPipeline(
        vae=MG.make_vae().to("cuda", torch.float16), text_encoder=te1, text_encoder_2=te2, tokenizer=tok,
        tokenizer_2=tok, unet=tiny_modules["net_t"], unet_encoder=tiny_modules["net_g"], scheduler=DDPMScheduler(),
        image_encoder=MG.make_image_encoder(tiny_modules["cfg_t"]["resampler"]["embedding_dim"]).to("cuda",
                                                                                                     torch.float16))


def _person(seed):
    g = torch.Generator().manual_seed(seed)
    mask = torch.zeros(1, H, W)
    mask[:, H // 4: 3 * H // 4, W // 8: 5 * W // 8] = 1.0
    return dict(image=torch.rand(3, H, W, generator=g).cuda(), mask_image=mask.cuda(),
                pose_img=(torch.rand(3, H, W, generator=g) * 2 - 1))


def _pair(pipe, gid="A", person_seed=50, photo=(600, 800, "RGBA"), desc=DESC):
    """(request with garment_photo and garment_description, the same request with every garment and prompt tensor
    made on the host the demo's way: Pillow, ToTensor + Normalize, CLIPImageProcessorPil, the demo's encode_prompt)."""
    from idm_vton_b200.serving import (GARMENT_PROMPT, NEGATIVE_PROMPT, PERSON_PROMPT, PROMPT_FIELDS,
                                       TryOnRequest)
    p = garment_photo(*photo)
    garm = demo_garment(p, H, W)
    with torch.no_grad():
        person = pipe.encode_prompt(PERSON_PROMPT + desc, num_images_per_prompt=1, do_classifier_free_guidance=True,
                                    negative_prompt=NEGATIVE_PROMPT)
        cloth_text = pipe.encode_prompt([GARMENT_PROMPT + desc], num_images_per_prompt=1,
                                        do_classifier_free_guidance=False, negative_prompt=[NEGATIVE_PROMPT])[0]
    derived = TryOnRequest(garment_id=gid, garment_photo=p, garment_description=desc, seed=7, **_person(person_seed))
    host = TryOnRequest(garment_id=gid, cloth=demo_cloth(garm), ip_adapter_image=torch.from_numpy(clip_pil(garm)),
                        text_embeds_cloth=cloth_text[0], seed=7, **_person(person_seed),
                        **{f: t[0] for f, t in zip(PROMPT_FIELDS, person)})
    return derived, host


def _plain(pipe, gid, person_seed):
    """A request in today's tensor form (its own prompt embeddings and garment tensors)."""
    from idm_vton_b200.serving import TryOnRequest
    g = torch.Generator().manual_seed(person_seed + 1000)
    r = lambda *s: torch.randn(*s, generator=g).half().float()  # noqa: E731
    return TryOnRequest(garment_id=gid, prompt_embeds=r(77, 256), negative_prompt_embeds=r(77, 256),
                        pooled_prompt_embeds=r(128), negative_pooled_prompt_embeds=r(128),
                        cloth=(torch.rand(3, H, W, generator=g) * 2 - 1), ip_adapter_image=r(3, 224, 224),
                        text_embeds_cloth=r(77, 256), seed=7, **_person(person_seed))


def _batch_server(pipe, max_batch=1):
    from idm_vton_b200.serving import TryOnServer
    return TryOnServer(pipe, height=H, width=W, num_inference_steps=3, guidance_scale=2.0, max_batch=max_batch, seed=7,
                       garment_cache_bytes=0, output_type="latent")


def test_tryon_server_garment_photo_and_description(text_pipe):
    res = {}
    for name in ("derived", "host"):
        derived, host = _pair(text_pipe)
        srv = _batch_server(text_pipe)
        t = srv.submit(derived if name == "derived" else host)
        res[name] = (srv.run()[t], text_pipe._last_latents.clone())
        if name == "derived":
            assert srv.stats["garment_photos_prepared"] == 1 and srv.stats["descriptions_encoded"] == 1
            # a second request for the garment, with neither garment fields nor prompts: nothing is encoded again
            from idm_vton_b200.serving import TryOnRequest
            t2 = srv.submit(TryOnRequest(garment_id="A", seed=7, **_person(50)))
            second = srv.run()[t2]
            assert srv.stats["garments_encoded"] == 1 and srv.stats["garment_photos_prepared"] == 1
            assert srv.stats["descriptions_encoded"] == 1 and torch.equal(second, res["derived"][0])
    assert torch.equal(res["derived"][0], res["host"][0]) and torch.equal(res["derived"][1], res["host"][1])


def test_tryon_server_photo_and_garment_photo_beside_a_plain_request(text_pipe):
    """One batch of a request with a full-resolution person photo and a garment photo and a plain tensor request of the
    same garment: the bits of the same batch with the person image made by Pillow and the garment tensors on the host."""
    from idm_vton_b200 import photo as P
    from test_photo_cpu import _photo
    a = _photo(301, 397, "RGB", 3)
    crop = PIL.fromarray(a).crop(P.crop_box((301, 397), H, W)).resize((W, H), 3)
    out = {}
    for name in ("derived", "host"):
        derived, host = _pair(text_pipe)
        plain = _plain(text_pipe, "A", 60)
        plain.cloth = plain.ip_adapter_image = plain.text_embeds_cloth = None       # the garment comes from the first
        first = derived if name == "derived" else host
        if name == "derived":
            first.image, first.photo = None, torch.from_numpy(a)
        else:
            first.image = torch.from_numpy(np.asarray(crop, np.float32) / 255).permute(2, 0, 1).contiguous().cuda()
        srv = _batch_server(text_pipe, max_batch=2)
        tickets = [srv.submit(first), srv.submit(plain)]
        res = srv.run()
        assert srv.stats["batches"] == 1 and not srv.failed
        out[name] = ([res[t] for t in tickets], text_pipe._last_latents.clone())
    # a photo request's "latent" result is its row of the final latents; the plain request gets the pipeline's own output
    assert torch.equal(out["derived"][1], out["host"][1]) and torch.equal(out["derived"][0][0], out["host"][1][0])
    assert torch.equal(out["derived"][0][1], out["host"][0][1])


@pytest.mark.parametrize("pool", [False, True], ids=["default", "pool"])
def test_continuous_server_garment_photo_and_description(text_pipe, pool):
    from idm_vton_b200.serving import PROMPT_FIELDS, ContinuousTryOnServer, TryOnRequest

    def server():
        srv = ContinuousTryOnServer(text_pipe, height=H, width=W, slots=3, num_inference_steps=3, guidance_scale=2.0,
                                    seed=7, output_type="latent", garment_kv_bytes=0 if pool else None)
        if pool:
            srv.garment_kv_bytes = 3 * srv.page_bytes()
        return srv
    lat = {}
    for name in ("derived", "host"):
        derived, host = _pair(text_pipe)
        b_derived, b_host = _pair(text_pipe, "B", 51, photo=(1080, 1920, "P"), desc="a denim jacket")
        srv = server()
        # two new garments (one admission) beside a plain tensor request of a third
        script = [([derived, b_derived, _plain(text_pipe, "C", 52)], 1)] if name == "derived" else \
            [([host, b_host, _plain(text_pipe, "C", 52)], 1)]
        # a later request for garment A without garment fields, and without prompts where A has a description
        later = TryOnRequest(garment_id="A", seed=7, **_person(50))
        if name == "host":
            for f in PROMPT_FIELDS:
                setattr(later, f, getattr(host, f))
        script.append(([later], 0))
        _, lat[name], _ = _drive(srv, script)
        if name == "derived":
            assert srv.stats["garment_photos_prepared"] == 2 and srv.stats["descriptions_encoded"] == 2
            assert srv.stats["garments_encoded"] == 3 and not srv.failed
    assert sorted(lat["derived"]) == sorted(lat["host"]) == [0, 1, 2, 3]
    for t in range(4):
        assert torch.equal(lat["derived"][t], lat["host"][t]), t
    assert torch.equal(lat["derived"][3], lat["derived"][0])
