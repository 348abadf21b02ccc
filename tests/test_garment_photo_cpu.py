"""Garment photos and descriptions without a GPU: the numpy restatement of CLIPImageProcessor's Pillow path (the CLIP
resize of the server-size garment, the centre crop and the 3 x 256 table) equals transformers' CLIPImageProcessorPil on
the sweep, and each mutant of it differs somewhere on the same sweep; the table is transformers' rescale and normalize;
the prompt strings are the demo's; the submit refusals and the drop of a garment whose preparation fails in both
servers; the C-ABI entry point (declared, exported, argument checks, refused by the binding when missing)."""
import collections
import ctypes
import os
import types

import numpy as np
import pytest
import torch

PIL = pytest.importorskip("PIL.Image")
transformers = pytest.importorskip("transformers")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# garment photos (W, H, mode), from a phone photo down to one pixel, and server sizes (height, width): 397 x 301 gives
# a CLIP resize of 224 x 295, an odd crop offset (35.5 rounded down)
GARMENTS = [(3024, 4032, "RGB"), (1080, 1920, "RGBA"), (768, 1024, "P"), (500, 300, "L"), (77, 91, "RGB"),
            (1, 1, "RGB")]
SERVER_SIZES = [(1024, 768), (1024, 1024), (256, 192), (397, 301)]
SWEEP = [(g, s) for g in GARMENTS for s in SERVER_SIZES]


def _case_id(c):
    (W, H, mode), (h, w) = c
    return f"{W}x{H}-{mode}-at-{w}x{h}"


def garment_photo(W, H, mode, seed=0):
    """A gradient with noise and hard edges, in `mode` (P: an adaptive palette, RGBA: a varying alpha)."""
    g = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W]
    base = (x * 255 // max(W - 1, 1) + y * 127 // max(H - 1, 1)) % 256
    a = (base[..., None] + g.integers(-40, 41, (H, W, 3))).clip(0, 255).astype(np.uint8)
    a[H // 3: H // 3 + 3] = 255
    a[:, W // 2: W // 2 + 2] = 0
    img = PIL.fromarray(a)
    if mode == "RGBA":
        img.putalpha(PIL.fromarray((base * 7 % 256).astype(np.uint8)))
    elif mode == "P":
        img = img.convert("P", palette=PIL.Palette.ADAPTIVE, colors=64)
    elif mode == "L":
        img = img.convert("L")
    return img


def demo_garment(photo, h, w):
    """The demo's garm_img: photo.convert("RGB").resize((w, h)) (BICUBIC, Pillow's default for RGB)."""
    return photo.convert("RGB").resize((w, h))


def demo_cloth(garm):
    """ToTensor + Normalize([0.5], [0.5]) of garm, as the demo's tensor_transfrom computes it: fp32, and contiguous
    like ToTensor's output (the VAE's result depends on its input's layout, so the layout is part of the recipe)."""
    x = torch.from_numpy(np.asarray(garm).copy()).permute(2, 0, 1).contiguous().float().div(255)
    return (x - 0.5) / 0.5


def clip_pil(garm):
    """CLIPImageProcessor's Pillow path (the reference's transformers), the truth."""
    return transformers.CLIPImageProcessorPil()(garm, return_tensors="np").pixel_values[0]


def restated_clip(garm, mutant=None, photo=None):
    """The restatement prepare_garments runs: Pillow's bicubic resize to clip_resize's size, the centre crop at its
    origin, the 3 x 256 table. Mutants: "f32_rescale", "reciprocal_normalize", "from_photo" (the CLIP resize from the
    original photo), "crop_round_up"."""
    from idm_vton_b200 import photo as P
    src = photo.convert("RGB") if mutant == "from_photo" else garm
    nw, nh, left, top = P.clip_resize(*src.size)
    if mutant == "crop_round_up":
        left, top = (nw - P.CLIP_SIZE + 1) // 2, (nh - P.CLIP_SIZE + 1) // 2
    a = np.asarray(src.resize((nw, nh), PIL.BICUBIC))[top:top + P.CLIP_SIZE, left:left + P.CLIP_SIZE]
    return np.stack([table(mutant)[c][a[..., c]] for c in range(3)])


def table(mutant=None):
    from idm_vton_b200 import photo as P
    mean, std = np.array(P.CLIP_MEAN, np.float32), np.array(P.CLIP_STD, np.float32)
    if mutant == "f32_rescale":
        x = np.arange(256, dtype=np.float32) * np.float32(1 / 255)
        return (x[None] - mean[:, None]) / std[:, None]
    if mutant == "reciprocal_normalize":
        x = (np.arange(256) * (1 / 255)).astype(np.float32)
        return (x[None] - mean[:, None]) * (np.float32(1) / std[:, None])
    return P.clip_table()


@pytest.fixture(scope="module")
def expected():
    """case -> (photo, garm, CLIPImageProcessorPil's pixels)."""
    out, photos = {}, {}
    for c in SWEEP:
        (W, H, mode), (h, w) = c
        photo = photos.setdefault((W, H, mode), garment_photo(W, H, mode))
        garm = demo_garment(photo, h, w)
        out[_case_id(c)] = (photo, garm, clip_pil(garm))
    return out


@pytest.mark.parametrize("case", SWEEP, ids=_case_id)
def test_restatement_equals_clip_image_processor_pil(case, expected):
    photo, garm, ref = expected[_case_id(case)]
    got = restated_clip(garm)
    assert got.dtype == ref.dtype == np.float32 and got.shape == ref.shape == (3, 224, 224)
    assert np.array_equal(got, ref)


def test_table_is_transformers_rescale_and_normalize():
    from idm_vton_b200 import photo as P
    p = transformers.CLIPImageProcessorPil()
    assert tuple(p.image_mean) == P.CLIP_MEAN and tuple(p.image_std) == P.CLIP_STD and p.rescale_factor == 1 / 255
    v = np.arange(256, dtype=np.uint8).reshape(16, 16)
    ref = p.normalize(p.rescale(np.stack([v, v, v]), p.rescale_factor), p.image_mean, p.image_std)
    assert ref.dtype == np.float32 and np.array_equal(ref.reshape(3, 256), P.clip_table())
    # the two arithmetic mutants are far from harmless: that many of the 768 entries differ
    assert (table("f32_rescale") != P.clip_table()).sum() == 325
    assert (table("reciprocal_normalize") != P.clip_table()).sum() == 191


@pytest.mark.parametrize("mutant", ["f32_rescale", "reciprocal_normalize", "torchvision", "from_photo",
                                    "crop_round_up"])
def test_each_mutant_differs_on_the_sweep(mutant, expected):
    differs = []
    for c in SWEEP:
        photo, garm, ref = expected[_case_id(c)]
        if mutant == "torchvision":
            got = transformers.CLIPImageProcessor()(garm, return_tensors="np").pixel_values[0]
        else:
            got = restated_clip(garm, mutant, photo)
        if got.shape != ref.shape or not np.array_equal(got, ref):
            differs.append(_case_id(c))
    assert differs, f"mutant {mutant} equals CLIPImageProcessorPil on the whole sweep"


def test_clip_resize_is_transformers_shortest_edge_rule():
    from idm_vton_b200 import photo as P
    assert P.clip_resize(768, 1024) == (224, 298, 0, 37)
    assert P.clip_resize(1024, 768) == (298, 224, 37, 0)
    assert P.clip_resize(301, 397) == (224, 295, 0, 35)
    assert P.clip_resize(224, 224) == (224, 224, 0, 0)


def test_prompt_strings_are_the_demos():
    from idm_vton_b200 import serving as S
    assert S.PERSON_PROMPT + "x" == "model is wearing x"          # gradio_demo/app.py:178
    assert S.GARMENT_PROMPT + "x" == "a photo of x"               # :193
    assert S.NEGATIVE_PROMPT == "monochrome, lowres, bad anatomy, worst quality, low quality"   # :179, 194
    calls = []

    class Pipe:
        def encode_prompt(self, prompt, **kw):
            calls.append((prompt, kw))
            t = torch.full((1, 77, 8), float(len(calls)))
            return t, t + 10, t[:, 0], t[:, 0] + 10
    emb = S.encode_description(Pipe(), "a red shirt", "cpu")
    assert calls[0] == ("model is wearing a red shirt", dict(device="cpu", num_images_per_prompt=1,
                                                             do_classifier_free_guidance=True,
                                                             negative_prompt=S.NEGATIVE_PROMPT))
    assert calls[1] == (["a photo of a red shirt"], dict(device="cpu", num_images_per_prompt=1,
                                                         do_classifier_free_guidance=False,
                                                         negative_prompt=[S.NEGATIVE_PROMPT]))
    assert emb["prompt_embeds"].shape == (77, 8) and float(emb["prompt_embeds"][0, 0]) == 1
    assert float(emb["negative_prompt_embeds"][0, 0]) == 11 and emb["pooled_prompt_embeds"].shape == (8,)
    assert float(emb["text_embeds_cloth"][0, 0]) == 2 and emb["text_embeds_cloth"].shape == (77, 8)


# ------------------------------------------------------------------------------------------------------------------
# the servers, on stubs
# ------------------------------------------------------------------------------------------------------------------
H, W = 64, 48
BAD = 13            # a stub garment photo this many rows high fails its preparation


def _req(gid="g", prompts=True, **kw):
    from idm_vton_b200.serving import TryOnRequest
    z = torch.zeros
    args = dict(garment_id=gid, image=z(3, H, W), mask_image=z(1, H, W), pose_img=z(3, H, W))
    if prompts:
        args.update(prompt_embeds=z(77, 8), negative_prompt_embeds=z(77, 8), pooled_prompt_embeds=z(4),
                    negative_pooled_prompt_embeds=z(4))
    args.update(kw)
    return TryOnRequest(**args)


def _photo_req(gid, rows=20, desc="a shirt", **kw):
    return _req(gid, prompts=False, garment_photo=torch.zeros(rows, 10, 3, dtype=torch.uint8),
                garment_description=desc, **kw)


class _Pipe:
    """The pipeline surface the servers use, on the CPU. encode_prompt fills with len(prompt) so a test can tell which
    description a tensor came from."""
    vae_scale_factor = 8
    _execution_device = torch.device("cpu")
    tokenizer = tokenizer_2 = text_encoder = text_encoder_2 = object()

    def __init__(self):
        self.unet = types.SimpleNamespace(dtype=torch.float32, encoder_hid_proj=lambda e: e)
        self.calls = []

    def encode_prompt(self, prompt, **kw):
        n = float(len(prompt if isinstance(prompt, str) else prompt[0]))
        t = torch.full((1, 77, 8), n)
        return t, -t, t[:, 0, :4], -t[:, 0, :4]

    def _encode_vae_image(self, cloth, generator=None):
        return cloth[:, :1]

    def prepare_ip_adapter_image_embeds(self, image, device, n):
        return image

    def __call__(self, image, **kw):
        self.calls.append(kw)
        return (list(image),)


@pytest.fixture
def stub_garments(monkeypatch):
    """photo.prepare_garments on the CPU: raises for a photo BAD rows high, else cloth = its height; records calls."""
    from idm_vton_b200 import photo as P
    calls = []

    def prepare(garments, height, width):
        calls.append(len(garments))
        for g in garments:
            P.check_garment(g)
            if g.shape[0] == BAD:
                raise ValueError("stub: this garment photo cannot be prepared")
        return [P.PreparedGarment(image_u8=torch.zeros(height, width, 3, dtype=torch.uint8),
                                  cloth=torch.full((3, height, width), float(g.shape[0])),
                                  clip_pixels=torch.zeros(3, 224, 224)) for g in garments]
    monkeypatch.setattr(P, "prepare_garments", prepare)
    return calls


def _servers(pipe=None):
    from idm_vton_b200.serving import ContinuousTryOnServer, TryOnServer
    pipe = pipe or types.SimpleNamespace(vae_scale_factor=8)
    return [TryOnServer(pipe, height=H, width=W, garment_cache_bytes=0),
            ContinuousTryOnServer(pipe, height=H, width=W, slots=2)]


def test_garment_requests_are_checked_at_submit():
    z, u8 = torch.zeros, torch.uint8
    tensors = dict(cloth=z(3, H, W), ip_adapter_image=z(3, 224, 224), text_embeds_cloth=z(77, 8))
    photo = z(20, 10, 3, dtype=u8)
    bad = [
        (dict(), "is new"),
        (dict(cloth=z(3, H, W), text_embeds_cloth=z(77, 8)), "is new"),
        (dict(cloth=z(3, H, W), ip_adapter_image=z(3, 224, 224)), "is new"),
        (dict(tensors, garment_photo=photo), "garment_photo replaces"),
        (dict(tensors, ip_adapter_image=None, garment_photo=photo), "garment_photo replaces"),
        (dict(tensors, garment_description="x"), "garment_description replaces"),
        (dict(tensors, text_embeds_cloth=None, garment_photo=None, garment_description=5), "str"),
        (dict(garment_photo=z(20, 10, 3), text_embeds_cloth=z(77, 8)), "uint8"),
        (dict(garment_photo=z(20, 10, 4, dtype=u8), text_embeds_cloth=z(77, 8)), "uint8"),
        (dict(garment_photo=np.zeros((20, 10, 3), np.uint8), text_embeds_cloth=z(77, 8)), "PIL image"),
        (dict(garment_photo=z(0, 10, 3, dtype=u8), text_embeds_cloth=z(77, 8)), "empty"),
        (dict(garment_photo=PIL.new("RGB", (0, 5)), text_embeds_cloth=z(77, 8)), "empty"),
        (dict(tensors, prompt_embeds=None), "all four"),
    ]
    for srv in _servers(_Pipe()):
        for kw, match in bad:
            with pytest.raises(ValueError, match=match):
                srv.submit(_req(**kw))
        # no prompt embeddings: the garment needs a description, on a pipeline that can encode it
        with pytest.raises(ValueError, match="no prompt embeddings"):
            srv.submit(_req(prompts=False, **tensors))
        assert srv.pending() == 0
        srv.submit(_req("p", **dict(tensors, text_embeds_cloth=None), garment_description="a shirt"))
        srv.submit(_req("p", prompts=False))            # pending garment "p" has a description
        srv.submit(_req("q", **tensors))
        with pytest.raises(ValueError, match="no prompt embeddings"):
            srv.submit(_req("q", prompts=False))         # pending garment "q" has none
        srv.submit(_req("r", prompts=False, garment_photo=PIL.new("P", (30, 40)), garment_description="x"))
        srv.submit(_req("s", garment_photo=photo, text_embeds_cloth=z(77, 8)))
        assert srv.pending() == 5
    for srv in _servers():                               # a pipeline without tokenizers or text encoders
        with pytest.raises(ValueError, match="tokenizers and text encoders"):
            srv.submit(_req(garment_photo=photo, garment_description="a shirt"))


def test_prepare_garments_refuses_before_any_device_work():
    from idm_vton_b200 import photo as P
    ok = torch.zeros(4, 4, 3, dtype=torch.uint8)
    for bad, match in ((torch.zeros(4, 4, 3), "uint8"), (torch.zeros(0, 4, 3, dtype=torch.uint8), "empty"),
                       ("photo.png", "PIL image")):
        with pytest.raises(ValueError, match=match):
            P.prepare_garments([ok, bad], 64, 48)
    with pytest.raises(ValueError, match="empty server size"):
        P.prepare_garments([ok], 0, 48)
    assert P.prepare_garments([], 64, 48) == []


def test_batch_server_drops_a_garment_whose_preparation_fails(stub_garments):
    from idm_vton_b200.serving import TryOnServer
    pipe = _Pipe()
    srv = TryOnServer(pipe, height=H, width=W, garment_cache_bytes=0, max_batch=1)
    bad = [srv.submit(_photo_req("X", BAD)), srv.submit(_req("X", prompts=False))]   # the second waits behind it
    good = [srv.submit(_photo_req("Y", 20, desc="a long red shirt")), srv.submit(_req("Y", prompts=False))]
    out = srv.run()
    assert sorted(out) == good and sorted(srv.failed) == bad and srv.pending() == 0
    assert all(isinstance(srv.failed[t], ValueError) for t in bad) and srv.stats["failed"] == 2
    assert "X" not in srv.garments
    with pytest.raises(ValueError, match="is new"):       # the id is unknown again
        srv.submit(_req("X"))
    # garment Y: one preparation and one encode for both requests; the person prompt comes from its description
    assert srv.stats["garment_photos_prepared"] == 1 and srv.stats["descriptions_encoded"] == 1
    assert srv.stats["garments_encoded"] == 1 and stub_garments == [1, 1, 1]      # X, X alone again, Y
    n = len("model is wearing a long red shirt")
    for kw in pipe.calls:
        assert torch.equal(kw["prompt_embeds"], torch.full((1, 77, 8), float(n)))
        assert torch.equal(kw["negative_prompt_embeds"], torch.full((1, 77, 8), -float(n)))
        assert torch.equal(kw["text_embeds_cloth"], torch.full((1, 77, 8), float(len("a photo of a long red shirt"))))
        assert torch.equal(kw["cloth"], torch.full((1, 1, H, W), 20.0))
    # a later request brings garment X again and runs
    t = srv.submit(_photo_req("X", 21))
    assert list(srv.run()) == [t]


def _continuous(pipe, S=2, T=2):
    from idm_vton_b200.serving import ContinuousTryOnServer
    from test_continuous_cpu import _FakeDen

    class Srv(ContinuousTryOnServer):
        def _configure(self):
            self.den, self.T, self._configured = _FakeDen(S, T), T, True

        def _prepare_request(self, req, gen, entry=None):
            from idm_vton_b200.serving import _prompts
            self.prompts = getattr(self, "prompts", {})
            self.prompts[req.ticket] = _prompts(req, self.garments.get(req.garment_id))
            return dict(latents=torch.tensor(float(req.ticket)))

        def _decode(self, latents):
            return latents
    return Srv(pipe, height=H, width=W, slots=S, num_inference_steps=T, seed=1)


def test_continuous_server_drops_a_garment_whose_preparation_fails(stub_garments):
    srv = _continuous(_Pipe(), S=2)
    bad = [srv.submit(_photo_req("X", BAD)), srv.submit(_req("X", prompts=False))]
    good = [srv.submit(_photo_req("Y", 20, desc="a shirt")), srv.submit(_photo_req("Z", 22, desc="a coat")),
            srv.submit(_req("Y", prompts=False))]
    srv.step()
    # the heads were both X's requests: X failed in the admission's call and alone, and took its waiting request with
    # it; the heads taken again, Y and Z, are prepared in one call
    assert stub_garments == [1, 1, 2]
    assert sorted(srv.failed) == bad and all(isinstance(srv.failed[t], ValueError) for t in bad)
    assert [e["req"].ticket for e in srv.slots] == good[:2] and "X" not in srv.garments
    out = srv.run()
    assert sorted(out) == good and srv.pending() == 0 and srv.stats["failed"] == 2
    assert srv.stats["garments_encoded"] == 2 and srv.stats["descriptions_encoded"] == 2
    assert srv.stats["garment_photos_prepared"] == 2
    assert float(srv.prompts[good[2]][0][0, 0]) == len("model is wearing a shirt")
    assert float(srv.prompts[good[1]][0][0, 0]) == len("model is wearing a coat")
    with pytest.raises(ValueError, match="is new"):
        srv.submit(_req("X"))


def test_continuous_admission_prepares_new_garments_in_one_call(stub_garments):
    srv = _continuous(_Pipe(), S=3)
    tickets = [srv.submit(_photo_req(g, 20 + i)) for i, g in enumerate("ABC")]
    srv.submit(_req("A", prompts=False))
    srv.step()
    assert stub_garments == [3] and srv.stats["garment_photos_prepared"] == 3 and not srv._prepared_garments
    srv.run()
    assert stub_garments == [3] and srv.stats["garments_encoded"] == 3 and tickets == [0, 1, 2]


# ------------------------------------------------------------------------------------------------------------------
# the C ABI
# ------------------------------------------------------------------------------------------------------------------
def test_clip_pixels_entry_point_declared_exported_and_validated():
    from idm_vton_b200 import build, lib
    name = "b200vton_clip_pixels_u8"
    header = open(os.path.join(ROOT, "include", "b200vton.h")).read()
    so = ctypes.CDLL(build.build())
    assert f"int {name}(" in header and hasattr(so, name) and name in lib.OPTIONAL_SIGNATURES
    assert "#define B200VTON_CLIP_SIZE 224" in header and lib.CLIP_SIZE == 224
    raw = lib.load()
    assert lib.has_symbol(name)
    n0 = lib.launch_count()

    def call(descs=1, dev=64, n=1, tab=64, out=64, **kw):
        d = dict(src=64, src_pitch=3 * 300, src_w=300, src_h=224, crop_x=38, crop_y=0)
        d.update(kw)
        arr = (lib.ClipDesc * 1)(lib.ClipDesc(**d))
        return raw.b200vton_clip_pixels_u8(arr if descs else None, dev, n, tab, out, None)
    for kw, msg in ((dict(src=None), b"null src"), (dict(src_w=0), b"empty"), (dict(src_pitch=899), b"pitch"),
                    (dict(crop_x=77), b"crop"), (dict(crop_x=-1), b"crop"), (dict(src_h=223), b"crop"),
                    (dict(crop_y=1), b"crop"), (dict(tab=None), b"table"), (dict(out=66), b"aligned"),
                    (dict(dev=60), b"aligned"), (dict(n=0), b"descriptors"), (dict(n=5000), b"descriptors"),
                    (dict(descs=0), b"descriptors")):
        assert call(**kw) == 1 and msg in raw.b200vton_last_error(), kw
    assert lib.launch_count() == n0


def test_library_without_the_clip_entry_point_refuses_in_the_binding():
    from idm_vton_b200 import lib
    lib.load()
    present = set(lib._present)
    try:
        lib._present.discard("b200vton_clip_pixels_u8")
        with pytest.raises(NotImplementedError, match="b200vton_clip_pixels_u8"):
            lib.clip_pixels_u8([], None, None)
    finally:
        lib._present.update(present)


def test_request_fields_keep_existing_constructions():
    """The positional order of the existing fields is unchanged; the new ones default to None."""
    from idm_vton_b200.serving import TryOnRequest
    z = torch.zeros
    r = TryOnRequest("g", z(3), z(1), z(3), z(77, 8), z(77, 8), z(4), z(4), z(3), z(3), z(77, 8))
    assert r.text_embeds_cloth.shape == (77, 8) and r.garment_photo is None and r.garment_description is None
    r = TryOnRequest("g", z(3), z(1), z(3))
    assert all(getattr(r, f) is None for f in ("prompt_embeds", "negative_prompt_embeds", "pooled_prompt_embeds",
                                               "negative_pooled_prompt_embeds"))
    assert collections.Counter(f.name for f in TryOnRequest.__dataclass_fields__.values())["garment_photo"] == 1
