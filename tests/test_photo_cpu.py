"""Full-resolution photos without a GPU: the numpy restatement of the resampler (host coefficients and the two integer
passes), the crop and the paste equal Pillow byte for byte on the sweep; each mutant of the restatement differs from
Pillow somewhere on the same sweep; crop_box is the demo's arithmetic; the submit-time refusals; the two C-ABI entry
points (declared, exported, argument checks, refused by the binding when missing)."""
import ctypes
import importlib.util
import os
import types

import numpy as np
import pytest
import torch

PIL = pytest.importorskip("PIL.Image")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ("b200vton_resample_u8", "b200vton_paste_u8")


def _load_ref():
    spec = importlib.util.spec_from_file_location("photo_ref", os.path.join(ROOT, "tests", "helpers", "photo_ref.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


R = _load_ref()

# (photo W, H, server width, height, filter, mode): a phone photo down to 768 x 1024 and back; ratios near 1 both ways;
# odd sizes and 1-pixel outputs; every filter; "L"; crop boxes at half pixels (W - tw odd: left = 116.5 rounds to 116
# (even), 117.5 to 118 and is pasted back at 117).
SWEEP = [
    (3024, 4032, 768, 1024, "bicubic", "RGB"),
    (770, 1027, 768, 1024, "bicubic", "RGB"),
    (767, 1023, 768, 1024, "bicubic", "RGB"),
    (768, 1030, 768, 1024, "bicubic", "RGB"),     # unchanged width: the horizontal pass is skipped
    (37, 53, 1, 1, "bicubic", "RGB"),
    (53, 37, 3, 1, "lanczos", "L"),
    (5, 9, 7, 11, "bilinear", "RGB"),
    (601, 799, 240, 320, "box", "RGB"),
    (601, 799, 240, 320, "bilinear", "L"),
    (601, 799, 240, 320, "hamming", "RGB"),
    (601, 799, 240, 320, "lanczos", "RGB"),
    (1001, 1024, 768, 1024, "bicubic", "L"),
    (1003, 1024, 768, 1024, "hamming", "RGB"),
    (99, 131, 64, 48, "bicubic", "RGB"),
]


def _case_id(c):
    return f"{c[0]}x{c[1]}-{c[2]}x{c[3]}-{c[4]}-{c[5]}"


def _photo(W, H, mode, seed):
    """A smooth gradient with noise: edges and flat areas, so clipping and rounding both matter."""
    g = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W]
    base = (x * 255 // max(W - 1, 1) + y * 127 // max(H - 1, 1)) % 256
    C = 3 if mode == "RGB" else 1
    a = (base[..., None] + g.integers(-40, 41, (H, W, C))).clip(0, 255).astype(np.uint8)
    a[H // 3: H // 3 + 3] = 255                     # hard edges: overshoot beyond 255 and below 0
    a[:, W // 2: W // 2 + 2] = 0
    return a


def _pil(a):
    return PIL.fromarray(a[..., 0] if a.shape[2] == 1 else a)


def _np(img):
    a = np.asarray(img)
    return a[..., None] if a.ndim == 2 else a


def _expected(case, seed=0):
    """Pillow: crop, resize to the server size; an output of that size resized back to the crop size and pasted."""
    W, H, w, h, filt, mode = case
    photo = _photo(W, H, mode, seed)
    box = R.P.crop_box((W, H), h, w)
    crop = _pil(photo).crop(box)
    down = _np(crop.resize((w, h), R.P.PIL_FILTERS[filt]))
    out = _photo(w, h, mode, seed + 1)
    back = _pil(out).resize(crop.size, R.P.PIL_FILTERS[filt])
    full = _pil(photo)
    full.paste(back, (int(box[0]), int(box[1])))
    return photo, box, out, down, _np(back), _np(full)


def _restated(photo, box, out, case, mutant=None):
    W, H, w, h, filt, _ = case
    x0, y0, x1, y1 = R.crop_pixels(box, mutant)
    down = R.resample(photo, (x0, y0, x1, y1), w, h, filt, mutant)
    x0, y0, x1, y1 = R.P.crop_pixels(box)
    back = R.resample(out, (0, 0, w, h), x1 - x0, y1 - y0, filt, mutant)
    return down, back, R.paste(photo, back, box, mutant) if photo.shape[2] == 3 else None


@pytest.fixture(scope="module")
def expected():
    return {_case_id(c): _expected(c) for c in SWEEP}


@pytest.mark.parametrize("case", SWEEP, ids=_case_id)
def test_restatement_equals_pillow(case, expected):
    photo, box, out, down, back, full = expected[_case_id(case)]
    d, b, f = _restated(photo, box, out, case)
    assert d.shape == down.shape and np.array_equal(d, down)
    assert b.shape == back.shape and np.array_equal(b, back)
    if f is not None:
        assert np.array_equal(f, full)


@pytest.mark.parametrize("mutant", R.MUTANTS)
def test_each_mutant_differs_from_pillow_on_the_sweep(mutant, expected):
    differs = []
    for case in SWEEP:
        photo, box, out, down, back, full = expected[_case_id(case)]
        try:
            d, b, f = _restated(photo, box, out, case, mutant)
        except (IndexError, ValueError):
            differs.append(_case_id(case))
            continue
        if d.shape != down.shape or not np.array_equal(d, down) or not np.array_equal(b, back) or \
                (f is not None and not np.array_equal(f, full)):
            differs.append(_case_id(case))
    assert differs, f"mutant {mutant} equals Pillow on the whole sweep"


def test_crop_box_is_the_demos_arithmetic():
    from idm_vton_b200 import photo as P
    assert 768 / 1024 == 3 / 4 and 1024 / 768 == 4 / 3      # so the server's ratios are the demo's doubles

    def demo(width, height):                                # gradio_demo/app.py:137-143
        target_width = int(min(width, height * (3 / 4)))
        target_height = int(min(height, width * (4 / 3)))
        return ((width - target_width) / 2, (height - target_height) / 2, (width + target_width) / 2,
                (height + target_height) / 2)
    g = np.random.default_rng(5)
    sizes = [(3024, 4032), (4032, 3024), (1080, 1920), (1920, 1080), (768, 1024), (1, 1), (1, 5000), (5000, 1)]
    sizes += [tuple(int(v) for v in g.integers(1, 20000, 2)) for _ in range(20000)]
    for W, H in sizes:
        assert P.crop_box((W, H), 1024, 768) == demo(W, H), (W, H)
    # the product, not W / 0.75: the two differ in the last bit for some widths (their int agrees)
    prod = [W for W in range(1, 20000) if W * (4 / 3) != W / 0.75]
    assert prod and all(int(W * (4 / 3)) == int(W / 0.75) for W in prod)


def test_pillow_crop_and_paste_quirks():
    from idm_vton_b200 import photo as P
    img = PIL.new("RGB", (10, 10))
    assert img.crop((0.5, 1.5, 5.5, 6.5)).size == (6, 4)
    assert P.crop_pixels((0.5, 1.5, 5.5, 6.5)) == (0, 2, 6, 6)
    box = P.crop_box((1003, 1024), 1024, 768)
    assert box[0] == 117.5 and P.crop_pixels(box)[0] == 118 and P.paste_offset(box) == (117, 0)


def test_coefficient_tables_are_cached_and_fixed_point():
    from idm_vton_b200 import photo as P
    P._tables.cache_clear()
    b, k = P._tables(4032, 1024, "bicubic")
    assert P._tables(4032, 1024, "bicubic")[1] is k and P._tables.cache_info().hits == 1
    assert k.dtype == np.int32 and b.shape == (1024, 2) and k.shape[1] == 2 * 8 + 1
    assert np.all(np.abs(k.sum(1) - (1 << 22)) <= k.shape[1])    # each row sums to 1 in 22-bit fixed point


# ------------------------------------------------------------------------------------------------------------------
# refusals
# ------------------------------------------------------------------------------------------------------------------
def _req(**kw):
    from idm_vton_b200.serving import TryOnRequest
    z = torch.zeros
    args = dict(garment_id="g", image=None, mask_image=z(1, 64, 48), pose_img=z(3, 64, 48), prompt_embeds=z(77, 8),
                negative_prompt_embeds=z(77, 8), pooled_prompt_embeds=z(8), negative_pooled_prompt_embeds=z(8),
                cloth=z(3, 64, 48), ip_adapter_image=z(3, 224, 224), text_embeds_cloth=z(77, 8),
                photo=torch.zeros(100, 90, 3, dtype=torch.uint8))
    args.update(kw)
    return TryOnRequest(**args)


def _servers():
    from idm_vton_b200.serving import ContinuousTryOnServer, TryOnServer
    pipe = types.SimpleNamespace(vae_scale_factor=8)
    return [TryOnServer(pipe, height=64, width=48, garment_cache_bytes=0),
            ContinuousTryOnServer(pipe, height=64, width=48, slots=2)]


def test_photo_requests_are_checked_at_submit():
    u8 = torch.uint8
    bad = [
        (dict(image=torch.zeros(3, 64, 48)), "photo.*image"),
        (dict(photo=PIL.new("RGBA", (90, 100))), "mode"),
        (dict(photo=torch.zeros(100, 90, 3)), "uint8"),
        (dict(photo=torch.zeros(100, 90, 4, dtype=u8)), "uint8"),
        (dict(mask_image=torch.zeros(1, 50, 50)), "mask_image"),
        (dict(mask_image=PIL.new("RGB", (90, 100))), "mode"),
        (dict(mask_image=torch.zeros(100, 91, dtype=u8)), "mask_image"),
        (dict(pose_img=torch.zeros(3, 100, 90)), "pose_img"),
        (dict(pose_img=torch.zeros(100, 90, 3)), "pose_img"),
        (dict(mask_image=None), "mask"),
        (dict(paste="blend"), "paste"),
        # empty crops: 4 x 2 at 3 : 4 is the box (1.5, 0, 2.5, 2), rounded to zero width; a 1-pixel-high photo
        (dict(photo=torch.zeros(2, 4, 3, dtype=u8)), "empty crop"),
        (dict(photo=PIL.new("RGB", (50, 1))), "empty crop"),
        # at the server size only the format of requests without a photo: float [1, h, w] masks, [3, h, w] poses
        (dict(mask_image=torch.zeros(1, 64, 48, dtype=u8)), "mask_image"),
        (dict(mask_image=torch.zeros(1, 64, 48, dtype=torch.bool)), "mask_image"),
        (dict(mask_image=torch.zeros(64, 48)), "mask_image"),
        (dict(pose_img=torch.zeros(3, 64, 48, dtype=u8)), "pose_img"),
    ]
    for srv in _servers():
        for kw, match in bad:
            with pytest.raises(ValueError, match=match):
                srv.submit(_req(**kw))
        assert srv.pending() == 0
        # at photo size and at server size, each is accepted
        for kw in (dict(), dict(mask_image=torch.zeros(100, 90, dtype=torch.bool), pose_img=torch.zeros(100, 90, 3, dtype=u8)),
                   dict(mask_image=PIL.new("L", (90, 100)), pose_img=PIL.new("RGB", (90, 100)), paste="mask"),
                   dict(photo=PIL.new("RGB", (90, 100)), mask_image=PIL.new("1", (90, 100)))):
            srv.submit(_req(**kw))
        assert srv.pending() == 4


def test_server_size_inputs_are_decided_alike_at_submit_and_at_run_time():
    """What submit accepts as a server-size mask or pose is what the server feeds to the pipeline (not the entry's)."""
    from idm_vton_b200 import photo as P
    from idm_vton_b200.serving import _person_inputs
    e = P.PreparedPhoto(photo=torch.zeros(100, 90, 3, dtype=torch.uint8), box=(0.0, 10.0, 90.0, 90.0),
                        crop=(0, 10, 90, 90), image=torch.zeros(3, 64, 48), image_u8=torch.zeros(64, 48, 3))
    for dt in (torch.float32, torch.float16):
        r = _req(mask_image=torch.zeros(1, 64, 48, dtype=dt), pose_img=torch.zeros(3, 64, 48, dtype=dt))
        for srv in _servers():
            srv.submit(r)
        image, mask, pose = _person_inputs(r, e)
        assert image is e.image and mask is r.mask_image and pose is r.pose_img


def test_paste_back_and_prepare_refuse_bad_arguments():
    from idm_vton_b200 import photo as P
    with pytest.raises(ValueError, match="filter"):
        P.prepare_photos([torch.zeros(10, 10, 3, dtype=torch.uint8)], 8, 6, filter="nearest")
    with pytest.raises(ValueError, match="empty crop"):        # refused before any device work
        P.prepare_photos([torch.zeros(2, 4, 3, dtype=torch.uint8)], 1024, 768)
    with pytest.raises(ValueError, match="mode"):
        P.paste_back([None], torch.zeros(1, 8, 6, 3, dtype=torch.uint8), mode="blend")


def _bad_photo_request(srv, garment="A"):
    """A photo request with an empty crop placed in the queue as if its submit check had passed. A 4 x 1 photo has an
    empty crop at any aspect: at 1 : 1 its box is (1.5, 0, 2.5, 1), rounded to zero width."""
    h, w = srv.height, srv.width
    r = _req(garment_id=garment, photo=torch.zeros(1, 4, 3, dtype=torch.uint8), mask_image=torch.zeros(1, h, w),
             pose_img=torch.zeros(3, h, w))
    with pytest.raises(ValueError, match="empty crop"):
        srv.submit(r)
    r.ticket = srv._next_ticket
    srv._next_ticket += 1
    return r


def test_continuous_admission_drops_a_photo_request_whose_preparation_fails():
    from test_continuous_cpu import _fake_server
    from test_continuous_cpu import _req as plain
    srv = _fake_server(S=2, T=3)
    bad = _bad_photo_request(srv)
    srv.waiting.append(bad)
    good = [srv.submit(plain("A")), srv.submit(plain("B")), srv.submit(plain("C"))]
    srv.step()
    assert list(srv.failed) == [bad.ticket] and isinstance(srv.failed[bad.ticket], ValueError)
    assert srv.stats["failed"] == 1 and [e["req"].ticket for e in srv.slots] == good[:2]
    out = srv.run()
    assert sorted(out) == good and srv.pending() == 0


def test_batch_mode_drops_a_photo_request_whose_preparation_fails():
    from idm_vton_b200.serving import TryOnServer

    class Pipe:
        vae_scale_factor = 8
        _execution_device = torch.device("cpu")
        unet = types.SimpleNamespace(dtype=torch.float32)

        def __call__(self, image, **kw):
            self.batch = image.shape[0]
            return (list(image),)

    class Srv(TryOnServer):
        def _garment(self, gid, batch, device, dtype):
            return dict(latents=None, ip_adapter_image=None, text_embeds_cloth=None)

    srv = Srv(Pipe(), height=64, width=48, garment_cache_bytes=0, max_batch=4)
    bad = _bad_photo_request(srv)
    srv.queue.setdefault(("A", None), __import__("collections").deque()).append(bad)
    good = srv.submit(_req(garment_id="A", photo=None, image=torch.ones(3, 64, 48)))
    out = srv.run()
    assert list(out) == [good] and torch.equal(out[good], torch.ones(3, 64, 48)) and srv.pipe.batch == 1
    assert list(srv.failed) == [bad.ticket] and srv.stats["failed"] == 1 and srv.pending() == 0


# ------------------------------------------------------------------------------------------------------------------
# the C ABI
# ------------------------------------------------------------------------------------------------------------------
def test_photo_entry_points_declared_exported_and_validated():
    from idm_vton_b200 import build, lib
    header = open(os.path.join(ROOT, "include", "b200vton.h")).read()
    so = ctypes.CDLL(build.build())
    for name in SYMBOLS:
        assert f"int {name}(" in header and hasattr(so, name) and name in lib.OPTIONAL_SIGNATURES, name
    raw = lib.load()
    assert all(lib.has_symbol(n) for n in SYMBOLS)
    n0 = lib.launch_count()

    def rs(**kw):
        d = dict(src=64, src_pitch=30, src_w=10, src_h=10, crop_x=0, crop_y=0, crop_w=10, crop_h=10, dst=64,
                 dst_pitch=15, out_w=5, out_h=5, channels=3, need_x=1, need_y=1, bounds_x=0, coefs_x=10, ksize_x=5,
                 bounds_y=0, coefs_y=10, ksize_y=5, tmp_first=0, tmp_rows=10)
        d.update(kw)
        arr = (lib.ResampleDesc * 1)(lib.ResampleDesc(**d))
        return raw.b200vton_resample_u8(arr, 64, 1, 64, 35, 64, 1 << 10, None)
    for kw, msg in ((dict(channels=2), b"channels"), (dict(crop_x=1), b"crop"), (dict(src_pitch=20), b"pitch"),
                    (dict(need_x=0), b"need_x"), (dict(ksize_x=6), b"horizontal tables"),
                    (dict(tmp_rows=11), b"intermediate"), (dict(tmp_offset=1000), b"intermediate"),
                    (dict(src=None), b"null")):
        assert rs(**kw) == 1 and msg in raw.b200vton_last_error(), kw
    assert raw.b200vton_resample_u8(None, 64, 1, 64, 35, 64, 1 << 10, None) == 1

    def ps(**kw):
        d = dict(photo=64, photo_pitch=30, dst=64, dst_pitch=30, image=64, image_pitch=15, width=10, height=10,
                 box_x=2, box_y=2, box_w=5, box_h=5)
        d.update(kw)
        arr = (lib.PasteDesc * 1)(lib.PasteDesc(**d))
        return raw.b200vton_paste_u8(arr, 64, 1, None)
    for kw, msg in ((dict(box_x=6), b"box"), (dict(image_pitch=14), b"box"), (dict(photo=None), b"null"),
                    (dict(mask=64, mask_x=3, mask_w=10, mask_h=10, mask_pitch=10), b"mask")):
        assert ps(**kw) == 1 and msg in raw.b200vton_last_error(), kw
    assert lib.launch_count() == n0


def test_library_without_the_photo_entry_points_refuses_in_the_binding():
    from idm_vton_b200 import lib
    lib.load()
    present = set(lib._present)
    try:
        for name, call in (("b200vton_resample_u8", lambda: lib.resample_u8([], None, None)),
                           ("b200vton_paste_u8", lambda: lib.paste_u8([], None))):
            lib._present.discard(name)
            with pytest.raises(NotImplementedError, match=name):
                call()
    finally:
        lib._present.update(present)
