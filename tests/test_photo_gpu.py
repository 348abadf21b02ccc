"""Full-resolution photos on the GPU:
  * b200vton_resample_u8 equals Pillow byte for byte on the sweep of tests/test_photo_cpu.py (crop + resize down, the
    output resized back), for "RGB" and "L" and every filter; a ragged batch of five photos in one call (two launches)
    equals Pillow per photo;
  * paste-back: crop mode equals Pillow's crop / resize / paste; in mask mode every pixel outside the mask is the
    photo's and every pixel inside is the resampled output's;
  * the fused fp32 outputs equal np.asarray(img, np.float32) / 255 and the demo's ToTensor + Normalize(0.5, 0.5);
  * the servers (tiny config): a photo request's final latents are bit-identical to the same request with `image` made
    by Pillow on the host, in TryOnServer and in ContinuousTryOnServer (default and pool mode); its full-resolution
    result equals Pillow's paste-back of its own server-size output; beside requests of other photo sizes in a
    continuous batch it gets the same bits as alone.
"""
import numpy as np
import pytest
import torch

from test_photo_cpu import PIL, SWEEP, _case_id, _expected, _np, _photo, _pil

pytestmark = pytest.mark.gpu


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _resample_gpu(src, crop, w, h, filt):
    from idm_vton_b200 import photo as P
    x0, y0, x1, y1 = crop
    dst = torch.empty((h, w, src.shape[2]), dtype=torch.uint8, device="cuda")
    P._resample([(src, (x0, y0, x1 - x0, y1 - y0), dst, None, 0, filt)], src.device)
    return dst.cpu().numpy()


@pytest.mark.parametrize("case", SWEEP, ids=_case_id)
def test_resample_kernel_equals_pillow(case):
    from idm_vton_b200 import photo as P
    photo, box, out, down, back, full = _expected(case)
    W, H, w, h, filt, mode = case
    crop = P.crop_pixels(box)
    assert np.array_equal(_resample_gpu(_cuda(photo), crop, w, h, filt), down)
    assert np.array_equal(_resample_gpu(_cuda(out), (0, 0, w, h), crop[2] - crop[0], crop[3] - crop[1], filt), back)
    if mode == "RGB":        # the public path: prepare, then paste back that output
        e = P.prepare_photos([_cuda(photo)], h, w, filter=filt)[0]
        assert np.array_equal(e.image_u8.cpu().numpy(), down)
        assert np.array_equal(e.image.cpu().numpy(), np.asarray(down, np.float32).transpose(2, 0, 1) / 255)
        assert np.array_equal(P.paste_back([e], _cuda(out)[None])[0].cpu().numpy(), full)


def test_ragged_batch_in_one_call():
    from idm_vton_b200 import lib, photo as P
    sizes = [(3024, 4032), (1080, 1920), (4032, 3024), (801, 1067), (768, 1024)]
    photos = [_photo(W, H, "RGB", 10 + i) for i, (W, H) in enumerate(sizes)]
    inputs = [_pil(photos[0]), torch.from_numpy(photos[1])] + [_cuda(p) for p in photos[2:]]   # PIL, CPU, CUDA
    n0 = lib.launch_count()
    prep = P.prepare_photos(inputs, 1024, 768)
    assert lib.launch_count() - n0 == 2                           # one launch per pass for the five photos
    for a, e in zip(photos, prep):
        ref = _np(_pil(a).crop(P.crop_box((a.shape[1], a.shape[0]), 1024, 768)).resize((768, 1024), 3))
        assert np.array_equal(e.image_u8.cpu().numpy(), ref)
    outs = torch.stack([_cuda(_photo(768, 1024, "RGB", 20 + i)) for i in range(5)])
    n0 = lib.launch_count()
    full = P.paste_back(prep, outs)
    assert lib.launch_count() - n0 == 3                           # two resample passes and the paste
    for a, e, o, f in zip(photos, prep, outs, full):
        img = _pil(a)
        back = _pil(o.cpu().numpy()).resize((e.crop[2] - e.crop[0], e.crop[3] - e.crop[1]), 3)
        img.paste(back, P.paste_offset(e.box))
        assert np.array_equal(f.cpu().numpy(), np.asarray(img))


def test_mask_mode_paste_and_fused_outputs():
    from idm_vton_b200 import photo as P
    W, H, w, h = 1003, 1411, 768, 1024
    photo = _photo(W, H, "RGB", 3)
    g = np.random.default_rng(4)
    mask = np.zeros((H, W), np.uint8)
    mask[300:900, 200:800] = 255
    mask[g.random((H, W)) < 0.05] = 127                            # just below the 128 threshold
    mask[g.random((H, W)) < 0.05] = 128
    pose = _photo(W, H, "RGB", 5)
    e = P.prepare_photos([_pil(photo)], h, w, masks=[PIL.fromarray(mask, "L")], poses=[torch.from_numpy(pose)])[0]
    box = P.crop_box((W, H), h, w)
    m_u8 = _np(PIL.fromarray(mask, "L").crop(box).resize((w, h), 3))[..., 0]
    p_u8 = _np(_pil(pose).crop(box).resize((w, h), 3))
    assert np.array_equal(e.mask.cpu().numpy()[0], m_u8.astype(np.float32) / 255)
    ref = (p_u8.astype(np.float32) / np.float32(255) - np.float32(0.5)) / np.float32(0.5)
    assert np.array_equal(e.pose.cpu().numpy(), ref.transpose(2, 0, 1))
    out = _photo(w, h, "RGB", 6)
    full = P.paste_back([e], _cuda(out)[None], mode="mask")[0].cpu().numpy()
    back = _np(_pil(out).resize((e.crop[2] - e.crop[0], e.crop[3] - e.crop[1]), 3))
    px, py = P.paste_offset(box)
    resampled = photo.copy()
    resampled[py:py + back.shape[0], px:px + back.shape[1]] = back
    in_box = np.zeros((H, W), bool)
    in_box[py:py + back.shape[0], px:px + back.shape[1]] = True
    inside = (mask >= 128) & in_box
    assert inside.sum() > 1000 and (~inside).sum() > 1000
    assert np.array_equal(full[~inside], photo[~inside]) and np.array_equal(full[inside], resampled[inside])
    # a server-size mask: binarised (>= 0.5) x 255, resampled to the crop size, set where >= 128
    e2 = P.prepare_photos([_cuda(photo)], h, w)[0]
    sm = torch.from_numpy((g.random((1, h, w)) < 0.5).astype(np.float32))
    sm[:, :h // 2] = 0.5
    full2 = P.paste_back([e2], _cuda(out)[None], mode="mask", masks=[sm])[0].cpu().numpy()
    big = _np(PIL.fromarray(((sm[0].numpy() >= 0.5) * 255).astype(np.uint8), "L").resize(back.shape[1::-1], 3))[..., 0]
    sel = np.zeros((H, W), bool)
    sel[py:py + back.shape[0], px:px + back.shape[1]] = big >= 128
    assert sel.sum() > 1000 and np.array_equal(full2[~sel], photo[~sel]) and np.array_equal(full2[sel], resampled[sel])


# ------------------------------------------------------------------------------------------------
# the servers (tiny config)
# ------------------------------------------------------------------------------------------------
from test_continuous_gpu import _drive, _pipe, _request, _server, tiny_modules  # noqa: E402,F401


def _photo_pair(tiny, size, person_seed=40, garment="A", photo_seed=0):
    """(photo request, the same request with `image` made by Pillow on the host, the photo)."""
    from oracle import make_golden_pipeline as MG
    from idm_vton_b200 import photo as P
    W, H = size
    a = _photo(W, H, "RGB", photo_seed)
    crop = _pil(a).crop(P.crop_box((W, H), MG.H, MG.W)).resize((MG.W, MG.H), 3)
    host = torch.from_numpy(np.asarray(crop, np.float32) / 255).permute(2, 0, 1).contiguous()
    ph, ref = _request(tiny, person_seed, garment), _request(tiny, person_seed, garment)
    ph.image, ph.photo = None, torch.from_numpy(a)
    ref.image = host.cuda()
    return ph, ref, a


def _pillow_paste(a, server_u8, size):
    from oracle import make_golden_pipeline as MG
    from idm_vton_b200 import photo as P
    box = P.crop_box(size, MG.H, MG.W)
    x0, y0, x1, y1 = P.crop_pixels(box)
    img = _pil(a)
    img.paste(PIL.fromarray(server_u8).resize((x1 - x0, y1 - y0), 3), P.paste_offset(box))
    return np.asarray(img)


def _server_u8(pt):
    """The uint8 bytes of a "pt" image, as the postprocess kernel makes them for "pil"."""
    return (pt.permute(1, 2, 0) * 255).round().to(torch.uint8).cpu().numpy()


def test_tryon_server_photo_request(tiny_modules):
    from oracle import make_golden_pipeline as MG
    from idm_vton_b200.serving import TryOnServer
    size = (301, 397)
    pipe = _pipe(tiny_modules)
    res = {}
    for name, out_type in (("photo", "latent"), ("ref", "latent"), ("photo_pt", "pt"), ("ref_pil", "pil")):
        ph, ref, a = _photo_pair(tiny_modules, size)
        srv = TryOnServer(pipe, height=MG.H, width=MG.W, num_inference_steps=3, guidance_scale=2.0, max_batch=1,
                          seed=7, garment_cache_bytes=0, output_type=out_type)
        t = srv.submit(ph if name.startswith("photo") else ref)
        res[name] = (srv.run()[t], pipe._last_latents.clone())
    assert torch.equal(res["photo"][0], res["ref"][1][0]) and torch.equal(res["photo"][1], res["ref"][1])
    full = res["photo_pt"][0]
    assert full.dtype == torch.uint8 and full.is_cuda and tuple(full.shape) == (size[1], size[0], 3)
    assert np.array_equal(full.cpu().numpy(), _pillow_paste(a, np.asarray(res["ref_pil"][0]), size))


@pytest.mark.parametrize("pool", [False, True], ids=["default", "pool"])
def test_continuous_server_photo_requests(tiny_modules, pool):
    from test_continuous_pool_gpu import _pool_server
    size = (301, 397)

    def server():
        return _pool_server(tiny_modules, pages=3, steps=3) if pool else _server(tiny_modules, steps=3)
    ph, ref, a = _photo_pair(tiny_modules, size)
    img_p, lat_p, _ = _drive(server(), [([ph], 0)])
    img_r, lat_r, _ = _drive(server(), [([ref], 0)])
    assert torch.equal(lat_p[0], lat_r[0])
    full = img_p[0]
    assert tuple(full.shape) == (size[1], size[0], 3)
    assert np.array_equal(full.cpu().numpy(), _pillow_paste(a, _server_u8(img_r[0]), size))
    # beside requests of other photo sizes and a request without a photo: the same bits as alone
    b, b_ref, _ = _photo_pair(tiny_modules, (512, 300), 41, "B", photo_seed=1)
    ph2, _, _ = _photo_pair(tiny_modules, size)
    img_m, lat_m, _ = _drive(server(), [([b, _request(tiny_modules, 42, "C")], 1), ([ph2], 0)])
    assert torch.equal(lat_m[2], lat_p[0]) and torch.equal(img_m[2], full)
    assert tuple(img_m[0].shape) == (300, 512, 3)
    # the request without a photo (ticket 1) decoded beside a photo request: the bits it gets in the same run without
    # photos (b's twin with its image made by Pillow has b's latents, so the two decodes see the same batch)
    img_n, lat_n, _ = _drive(server(), [([b_ref, _request(tiny_modules, 42, "C")], 1),
                                        ([_photo_pair(tiny_modules, size)[1]], 0)])
    assert torch.equal(lat_n[0], lat_m[0]) and torch.equal(lat_n[1], lat_m[1])
    assert img_n[1].dtype == torch.float32 and torch.equal(img_n[1], img_m[1])


def test_tryon_server_mixed_batch(tiny_modules):
    """A batch of a photo request and a request without one: the latter's image is the bits it gets in the same batch
    without photos (where the pipeline decodes), the former's result Pillow's paste-back of its twin's output."""
    from oracle import make_golden_pipeline as MG
    from idm_vton_b200.serving import TryOnServer
    size = (301, 397)
    pipe = _pipe(tiny_modules)
    out = {}
    for name in ("photo", "plain"):
        ph, ref, a = _photo_pair(tiny_modules, size)
        srv = TryOnServer(pipe, height=MG.H, width=MG.W, num_inference_steps=3, guidance_scale=2.0, max_batch=2,
                          seed=7, garment_cache_bytes=0, output_type="pt")
        tickets = [srv.submit(ph if name == "photo" else ref), srv.submit(_request(tiny_modules, 42, "A"))]
        res = srv.run()
        assert srv.stats["batches"] == 1
        out[name] = ([res[t] for t in tickets], pipe._last_latents.clone())
    assert torch.equal(out["photo"][1], out["plain"][1])
    assert torch.equal(out["photo"][0][1], out["plain"][0][1])
    assert np.array_equal(out["photo"][0][0].cpu().numpy(), _pillow_paste(a, _server_u8(out["plain"][0][0]), size))
