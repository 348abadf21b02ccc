"""Full-resolution photos on the GPU: the reference demo's "auto-crop & resizing" (gradio_demo/app.py:135-147, 236-239)
generalised to the server geometry, for any photo size:

  1. centre-crop the photo to the server's aspect (crop_box, then Pillow's crop of the float box);
  2. resample the crop to width x height with a Pillow convolution filter (BICUBIC by default, Pillow's default for RGB);
  3. denoise (the caller: the pipeline, or a server);
  4. resample the server-size output back to the crop size with the same filter;
  5. paste it into the photo (paste_back): the result has the photo's size, and every pixel outside the box keeps its own
     bytes.

Steps 2 and 4 run b200vton_resample_u8, Pillow's ImagingResample restated in integers: the same bytes as
`PIL.Image.resize`. Step 5 runs b200vton_paste_u8. Two reference quirks are kept on purpose:
  * the crop box is float and Pillow's `crop` rounds it with Python's round (half to even): crop((0.5, 1.5, 5.5, 6.5)) is
    6 x 4 pixels;
  * the demo pastes at (int(left), int(top)), which truncates: a crop taken at x = round(1.5) = 2 goes back at x = 1.

Around a plain pipeline call:  p = prepare_photos([photo], 1024, 768);  pipe(image=p.images, ...,
output_type="pil") ... then paste_back(p, uint8 [B, 1024, 768, 3] of the outputs). The try-on servers do both steps for
requests that carry `photo` (serving.TryOnRequest).

Garment photos (prepare_garments) follow the demo's garm_img: the whole photo resized to the server size (BICUBIC), its
ToTensor + Normalize as `cloth`, and CLIPImageProcessor's Pillow path on it as the IP-Adapter's pixels (the CLIP resize
by b200vton_resample_u8, the centre crop and the 3 x 256 rescale / normalize table by b200vton_clip_pixels_u8).
"""
import dataclasses
import functools
import math
from typing import Optional

import numpy as np
import torch

from . import lib as L

PRECISION_BITS = 32 - 8 - 2        # Pillow's fixed-point precision for 8-bit images (Resample.c)


# ------------------------------------------------------------------------------------------------
# Pillow's filters and coefficient precomputation (Resample.c), restated in Python doubles
# ------------------------------------------------------------------------------------------------
def _box(x):
    return 1.0 if -0.5 < x <= 0.5 else 0.0


def _bilinear(x):
    if x < 0.0:
        x = -x
    return 1.0 - x if x < 1.0 else 0.0


_F054, _F046 = float(np.float32(0.54)), float(np.float32(0.46))     # Pillow writes them as float literals


def _hamming(x):
    if x < 0.0:
        x = -x
    if x == 0.0:
        return 1.0
    if x >= 1.0:
        return 0.0
    x = x * math.pi
    return math.sin(x) / x * (_F054 + _F046 * math.cos(x))


def _bicubic(x):
    a = -0.5
    if x < 0.0:
        x = -x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def _sinc(x):
    if x == 0.0:
        return 1.0
    x = x * math.pi
    return math.sin(x) / x


def _lanczos(x):
    return _sinc(x) * _sinc(x / 3) if -3.0 <= x < 3.0 else 0.0


# name -> (filter, support); PIL_FILTERS: the matching PIL.Image.Resampling values
FILTERS = {"box": (_box, 0.5), "bilinear": (_bilinear, 1.0), "hamming": (_hamming, 1.0), "bicubic": (_bicubic, 2.0),
           "lanczos": (_lanczos, 3.0)}
PIL_FILTERS = {"box": 4, "bilinear": 2, "hamming": 5, "bicubic": 3, "lanczos": 1}
PASTE_MODES = ("crop", "mask")


def _check_filter(name):
    if name not in FILTERS:
        raise ValueError(f"unknown resampling filter {name!r}; offered: {list(FILTERS)}")


def resample_coefficients(in_size, out_size, filter="bicubic"):
    """Pillow's precompute_coeffs for an axis of in_size pixels resampled to out_size (the whole axis: the crop is the
    image). Returns (bounds int32 [out, 2] = (first tap, tap count), kk float64 [out, ksize]): support x max(scale, 1),
    centres at (x + 0.5) * scale, taps clipped to the input, normalised by their sum. Same doubles as Pillow's C."""
    _check_filter(filter)
    fn, support = FILTERS[filter]
    scale = filterscale = in_size / out_size
    if filterscale < 1.0:
        filterscale = 1.0
    support = support * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    ss = 1.0 / filterscale
    bounds = np.zeros((out_size, 2), np.int32)
    kk = np.zeros((out_size, ksize), np.float64)
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        w = [fn((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for v in w:                    # sequential sum, as the C loop (Python's sum() compensates)
            ww += v
        kk[xx, :xmax] = [v / ww for v in w] if ww != 0.0 else w
        bounds[xx] = (xmin, xmax)
    return bounds, kk


def fixed_point(kk):
    """Pillow's normalize_coeffs_8bpc: (int)(k * 2^22 +- 0.5), rounding half away from zero."""
    s = kk * (1 << PRECISION_BITS)
    return np.where(kk < 0, np.trunc(-0.5 + s), np.trunc(0.5 + s)).astype(np.int32)


@functools.lru_cache(maxsize=256)
def _tables(in_size, out_size, filter):
    """(bounds, fixed-point coefficients) of one axis, cached by (in, out, filter): photos of one size reuse them."""
    bounds, kk = resample_coefficients(in_size, out_size, filter)
    return bounds, fixed_point(kk)


# ------------------------------------------------------------------------------------------------
# the crop box
# ------------------------------------------------------------------------------------------------
def crop_box(photo_size, height, width):
    """The demo's centre crop of a photo of photo_size = (W, H) to the aspect width : height, as its float box
    (left, top, right, bottom). Products in Python doubles, as the demo writes them: for 768 x 1024, width / height and
    height / width are the same doubles as its 3 / 4 and 4 / 3, so the box is the demo's bit for bit."""
    W, H = photo_size
    tw = int(min(W, H * (width / height)))
    th = int(min(H, W * (height / width)))
    return (W - tw) / 2, (H - th) / 2, (W + tw) / 2, (H + th) / 2


def crop_pixels(box):
    """The pixels Pillow's `crop` takes for a float box: each edge rounded with Python's round (half to even)."""
    return tuple(int(round(v)) for v in box)


def paste_offset(box):
    """Where the demo pastes the output back: (int(left), int(top)), truncated (not the crop's rounded corner)."""
    return int(box[0]), int(box[1])


# ------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------
def _is_pil(x):
    try:
        import PIL.Image
    except ImportError:
        return False
    return isinstance(x, PIL.Image.Image)


def _upload(t, device):
    """A uint8 tensor on `device`: CUDA tensors as they are (made contiguous), host tensors through pinned staging."""
    if t.is_cuda:
        return t.contiguous()
    return t.contiguous().pin_memory().to(device, non_blocking=True)


def _pil_u8(img, device):
    a = np.asarray(img)
    staged = torch.empty(a.shape, dtype=torch.uint8, pin_memory=True)
    staged.numpy()[...] = a
    return staged.to(device, non_blocking=True)


def photo_size(photo):
    """(W, H) of a photo: a PIL image, a uint8 [H, W, 3] tensor or a PreparedPhoto."""
    if isinstance(photo, PreparedPhoto):
        return photo.size
    if _is_pil(photo):
        return photo.size
    return int(photo.shape[1]), int(photo.shape[0])


def check_photo(photo):
    """ValueError unless `photo` is a PIL RGB image, a uint8 [H, W, 3] tensor or a PreparedPhoto."""
    if isinstance(photo, PreparedPhoto):
        return
    if _is_pil(photo):
        if photo.mode != "RGB":
            raise ValueError(f"photo: unsupported image mode {photo.mode!r} (RGB is supported)")
        return
    if not (torch.is_tensor(photo) and photo.dtype == torch.uint8 and photo.dim() == 3 and photo.shape[2] == 3):
        raise ValueError("photo must be a PIL RGB image or a uint8 [H, W, 3] tensor, got "
                         f"{type(photo).__name__} {getattr(photo, 'dtype', '')} {tuple(getattr(photo, 'shape', ()))}")


def check_crop(size, height, width):
    """ValueError when the crop of a photo of size = (W, H) to width x height has no pixels. Pillow's rounding of the
    float box can leave an empty crop: a 4 x 2 photo at 3 : 4 has the box (1.5, 0, 2.5, 2) and the crop (2, 0, 2, 2);
    a photo one pixel high has a crop 0 pixels wide."""
    x0, y0, x1, y1 = crop_pixels(crop_box(size, height, width))
    if x1 <= x0 or y1 <= y0:
        raise ValueError(f"a {size[0]}x{size[1]} photo has an empty crop at the aspect {width}:{height} (pixels "
                         f"{(x0, y0, x1, y1)})")


def mask_size(mask, size, height, width):
    """'photo' for a mask at photo size = (W, H) (PIL "L" / "1", or a uint8 / bool [H, W] or [1, H, W] tensor), 'server'
    for a floating-point [1, height, width] tensor (the format of requests without a photo); ValueError otherwise."""
    W, H = size
    if _is_pil(mask):
        if mask.mode not in ("L", "1"):
            raise ValueError(f"mask_image: unsupported image mode {mask.mode!r} (L and 1 are supported)")
        if mask.size == (W, H):
            return "photo"
    elif torch.is_tensor(mask):
        if (mask.dtype in (torch.uint8, torch.bool) and tuple(mask.shape[-2:]) == (H, W) and
                (mask.dim() == 2 or mask.dim() == 3 and mask.shape[0] == 1)):
            return "photo"
        if mask.is_floating_point() and tuple(mask.shape) == (1, height, width):
            return "server"
    raise ValueError(f"mask_image must be at the photo's size {W}x{H} (PIL L/1, or uint8/bool [H, W]) or a float "
                     f"[1, {height}, {width}] tensor, got {type(mask).__name__} "
                     f"{getattr(mask, 'size', None) if _is_pil(mask) else (mask.dtype, tuple(mask.shape)) if torch.is_tensor(mask) else ''}")


def pose_size(pose, size, height, width):
    """'photo' for a pose image at photo size (PIL RGB or a uint8 [H, W, 3] tensor), 'server' for a floating-point
    [3, height, width] tensor (the format of requests without a photo); ValueError otherwise."""
    W, H = size
    if _is_pil(pose):
        if pose.mode != "RGB":
            raise ValueError(f"pose_img: unsupported image mode {pose.mode!r} (RGB is supported)")
        if pose.size == (W, H):
            return "photo"
    elif torch.is_tensor(pose):
        if pose.dtype == torch.uint8 and tuple(pose.shape) == (H, W, 3):
            return "photo"
        if pose.is_floating_point() and tuple(pose.shape) == (3, height, width):
            return "server"
    raise ValueError(f"pose_img must be at the photo's size {W}x{H} (PIL RGB, or uint8 [H, W, 3]) or a float [3, "
                     f"{height}, {width}] tensor, got {type(pose).__name__} "
                     f"{getattr(pose, 'size', None) if _is_pil(pose) else (pose.dtype, tuple(pose.shape)) if torch.is_tensor(pose) else ''}")


def _mask_u8(mask, device):
    """A photo-size mask as uint8 [H, W] on the device (bool and mode "1" as 0 / 255)."""
    if _is_pil(mask):
        return _pil_u8(mask.convert("L") if mask.mode == "1" else mask, device)
    m = mask.reshape(mask.shape[-2:])
    if m.dtype == torch.bool:
        m = m.to(torch.uint8) * 255
    return _upload(m, device)


def _rgb_u8(img, device):
    return _pil_u8(img, device) if _is_pil(img) else _upload(img, device)


# ------------------------------------------------------------------------------------------------
# prepared photos
# ------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class PreparedPhoto:
    """One photo at the server size. `image` is what the pipeline takes as `image` (fp32 [3, height, width] CUDA,
    bit-identical to np.asarray(pil_crop_resized, np.float32) / 255); `image_u8` its uint8 [height, width, 3]."""
    photo: torch.Tensor                   # uint8 [H, W, 3] CUDA: the photo (paste-back keeps its pixels)
    box: tuple                            # crop_box's float (left, top, right, bottom)
    crop: tuple                           # the pixels cropped, (x0, y0, x1, y1) (crop_pixels)
    image: torch.Tensor
    image_u8: torch.Tensor
    filter: str = "bicubic"
    mask: Optional[torch.Tensor] = None        # fp32 [1, height, width]: a photo-size mask resampled, / 255
    pose: Optional[torch.Tensor] = None        # fp32 [3, height, width]: a photo-size pose resampled, (x/255 - .5)/.5
    photo_mask: Optional[torch.Tensor] = None  # uint8 [H, W] CUDA: the photo-size mask (paste="mask": set where >= 128)

    @property
    def size(self):
        return int(self.photo.shape[1]), int(self.photo.shape[0])


class PreparedPhotos(list):
    """The PreparedPhoto entries of prepare_photos, in input order."""

    @property
    def images(self):
        """[B, 3, height, width] fp32: the pipeline's `image` for the whole batch."""
        return torch.stack([e.image for e in self])


def _resample(jobs, device):
    """One b200vton_resample_u8 call for jobs of (src uint8 [h, w, C] CUDA, crop (x, y, cw, ch), dst uint8
    [out_h, out_w, C] contiguous, fp32 NCHW out or None, f32_mode, filter)."""
    chunks, where, descs, tmp = [], {}, [], 0
    n_tab = 0

    def table(size_in, size_out, filt):
        nonlocal n_tab
        key = (size_in, size_out, filt)
        if key not in where:
            bounds, coefs = _tables(size_in, size_out, filt)
            where[key] = (n_tab, n_tab + bounds.size, coefs.shape[1])
            chunks.extend((bounds.ravel(), coefs.ravel()))
            n_tab += bounds.size + coefs.size
        return where[key]

    for src, (cx, cy, cw, ch), dst, f32, mode, filt in jobs:
        oh, ow, C = dst.shape
        assert src.dim() == 3 and src.shape[2] == C and src.stride(2) == 1 and src.stride(1) == C and dst.is_contiguous()
        d = L.ResampleDesc(src=src.data_ptr(), src_pitch=src.stride(0), src_w=src.shape[1], src_h=src.shape[0],
                           crop_x=cx, crop_y=cy, crop_w=cw, crop_h=ch, dst=dst.data_ptr(), dst_pitch=ow * C,
                           out_f32=None if f32 is None else f32.data_ptr(), out_w=ow, out_h=oh, channels=C,
                           f32_mode=mode, need_x=int(ow != cw), need_y=int(oh != ch))
        if d.need_x:
            d.bounds_x, d.coefs_x, d.ksize_x = table(cw, ow, filt)
        if d.need_y:
            d.bounds_y, d.coefs_y, d.ksize_y = table(ch, oh, filt)
        if d.need_x and d.need_y:          # the crop rows the vertical pass reads (Pillow's ybox_first .. ybox_last)
            bounds_y = _tables(ch, oh, filt)[0]
            d.tmp_first = int(bounds_y[0, 0])
            d.tmp_rows = int(bounds_y[-1, 0] + bounds_y[-1, 1]) - d.tmp_first
            d.tmp_offset = tmp
            tmp += -(-d.tmp_rows * ow * C // 16) * 16
        elif d.need_x:
            d.tmp_first, d.tmp_rows = 0, ch
        descs.append(d)
    host = np.concatenate(chunks) if chunks else np.zeros(1, np.int32)
    tables = torch.from_numpy(host).pin_memory().to(device, non_blocking=True)
    workspace = torch.empty(max(tmp, 16), dtype=torch.uint8, device=device)
    L.resample_u8(descs, tables, workspace)


def prepare_photos(photos, height, width, filter="bicubic", masks=None, poses=None):
    """Photos -> PreparedPhotos at the server size height x width, in one b200vton_resample_u8 call.

    photos: PIL RGB images, uint8 [H, W, 3] CPU (staged through pinned memory) or CUDA tensors, or PreparedPhoto
    entries (not resampled again). masks / poses: None, or one entry per photo, each None or at photo size (masks: PIL
    "L" / "1", uint8 / bool [H, W]; poses: PIL RGB, uint8 [H, W, 3]): cropped and resampled like the photo, the mask as
    x / 255 (the pipeline binarises it at 0.5), the pose as (x / 255 - 0.5) / 0.5 (the demo's ToTensor + Normalize)."""
    _check_filter(filter)
    n = len(photos)
    masks = [None] * n if masks is None else list(masks)
    poses = [None] * n if poses is None else list(poses)
    if len(masks) != n or len(poses) != n:
        raise ValueError(f"prepare_photos: {n} photos, {len(masks)} masks and {len(poses)} poses")
    for photo, mask, pose in zip(photos, masks, poses):        # every refusal before any upload or launch
        check_photo(photo)
        size = photo_size(photo)
        if isinstance(photo, PreparedPhoto):
            if photo.image.shape[-2:] != (height, width):
                raise ValueError(f"a photo prepared at {tuple(photo.image.shape[-2:])} is used at ({height}, {width})")
        else:
            check_crop(size, height, width)
        if mask is not None and mask_size(mask, size, height, width) != "photo":
            raise ValueError("prepare_photos takes masks at photo size (server-size masks go to the pipeline as they are)")
        if pose is not None and pose_size(pose, size, height, width) != "photo":
            raise ValueError("prepare_photos takes poses at photo size")
    device = torch.device("cuda", torch.cuda.current_device())
    jobs, out = [], PreparedPhotos()
    for photo, mask, pose in zip(photos, masks, poses):
        if isinstance(photo, PreparedPhoto):
            e = dataclasses.replace(photo)
        else:
            p = _rgb_u8(photo, device)
            box = crop_box((p.shape[1], p.shape[0]), height, width)
            e = PreparedPhoto(photo=p, box=box, crop=crop_pixels(box),
                              image=torch.empty((3, height, width), dtype=torch.float32, device=device),
                              image_u8=torch.empty((height, width, 3), dtype=torch.uint8, device=device), filter=filter)
            jobs.append((p, _crop_rect(e), e.image_u8, e.image, 0, filter))
        if mask is not None:
            e.photo_mask = _mask_u8(mask, device)
            e.mask = torch.empty((1, height, width), dtype=torch.float32, device=device)
            jobs.append((e.photo_mask[..., None], _crop_rect(e),
                         torch.empty((height, width, 1), dtype=torch.uint8, device=device), e.mask, 0, e.filter))
        if pose is not None:
            e.pose = torch.empty((3, height, width), dtype=torch.float32, device=device)
            jobs.append((_rgb_u8(pose, device), _crop_rect(e),
                         torch.empty((height, width, 3), dtype=torch.uint8, device=device), e.pose, 1, e.filter))
        out.append(e)
    if jobs:
        _resample(jobs, device)
    return out


def _crop_rect(e):
    x0, y0, x1, y1 = e.crop
    return x0, y0, x1 - x0, y1 - y0


# ------------------------------------------------------------------------------------------------
# garment photos: the demo's garm_img (gradio_demo/app.py:132, 215, 232)
# ------------------------------------------------------------------------------------------------
CLIP_SIZE = L.CLIP_SIZE
CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)     # CLIPImageProcessor's defaults (OpenAI CLIP)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


def clip_table():
    """float32 [3, 256]: CLIPImageProcessor's rescale and normalize of every uint8 value, as transformers computes it:
    x = float32(float64(v) * (1 / 255)), then (x - mean) / std in float32 with the float32 mean and std."""
    x = (np.arange(256, dtype=np.float64) * (1 / 255)).astype(np.float32)
    mean, std = np.array(CLIP_MEAN, np.float32), np.array(CLIP_STD, np.float32)
    return (x[None, :] - mean[:, None]) / std[:, None]


@functools.lru_cache(maxsize=8)
def _clip_table_on(device):
    return torch.from_numpy(clip_table()).to(device)


def clip_resize(width, height):
    """CLIPImageProcessor's geometry for a width x height image: (new_w, new_h, left, top). The short side becomes 224
    and the long side int(224 * long / short) (transformers' shortest-edge rule); the 224 x 224 centre crop starts at
    left = (new_w - 224) // 2, top = (new_h - 224) // 2."""
    short, long = min(width, height), max(width, height)
    new_long = int(CLIP_SIZE * long / short)
    new_w, new_h = (CLIP_SIZE, new_long) if width <= height else (new_long, CLIP_SIZE)
    return new_w, new_h, (new_w - CLIP_SIZE) // 2, (new_h - CLIP_SIZE) // 2


def check_garment(garment):
    """ValueError unless `garment` is a PIL image of any mode (converted with .convert("RGB"), as the demo does) or a
    uint8 [H, W, 3] tensor, with at least one pixel."""
    if _is_pil(garment):
        size = garment.size
    elif torch.is_tensor(garment) and garment.dtype == torch.uint8 and garment.dim() == 3 and garment.shape[2] == 3:
        size = (int(garment.shape[1]), int(garment.shape[0]))
    else:
        raise ValueError("garment_photo must be a PIL image or a uint8 [H, W, 3] tensor, got "
                         f"{type(garment).__name__} {getattr(garment, 'dtype', '')} {tuple(getattr(garment, 'shape', ()))}")
    if size[0] < 1 or size[1] < 1:
        raise ValueError(f"garment_photo is empty ({size[0]}x{size[1]})")


@dataclasses.dataclass
class PreparedGarment:
    """One garment at the server size, as the demo prepares garm_img:
      image_u8: uint8 [height, width, 3] CUDA, Pillow's garm_img.convert("RGB").resize((width, height)) (BICUBIC);
      cloth: fp32 [3, height, width] CUDA, ToTensor + Normalize([0.5], [0.5]) of it (the pipeline's `cloth`);
      clip_pixels: fp32 [3, 224, 224] CUDA, CLIPImageProcessor()(image).pixel_values with transformers' Pillow path
      (the pipeline's `ip_adapter_image`)."""
    image_u8: torch.Tensor
    cloth: torch.Tensor
    clip_pixels: torch.Tensor


def prepare_garments(garments, height, width):
    """Garment photos -> PreparedGarment entries at the server size height x width, in three calls for the whole list:
    one b200vton_resample_u8 call to the server size (writing `cloth` as it goes), one from there to the CLIP size
    (Pillow's CLIP resize starts from the resized image, not from the photo) and one b200vton_clip_pixels_u8 launch.

    garments: PIL images of any mode (converted to RGB on the host) or uint8 [H, W, 3] tensors on the CPU (staged
    through pinned memory) or the GPU. Every input is checked before anything is uploaded or launched. For a plain
    pipeline call: pipe(cloth=g.cloth[None].half(), ip_adapter_image=g.clip_pixels[None], ...)."""
    garments = list(garments)
    for g in garments:
        check_garment(g)
    if height < 1 or width < 1:
        raise ValueError(f"prepare_garments: empty server size {width}x{height}")
    if not garments:
        return []
    device = torch.device("cuda", torch.cuda.current_device())
    srcs = [(_pil_u8(g if g.mode == "RGB" else g.convert("RGB"), device) if _is_pil(g) else _upload(g, device))
            for g in garments]
    n = len(srcs)
    image_u8 = torch.empty((n, height, width, 3), dtype=torch.uint8, device=device)
    cloth = torch.empty((n, 3, height, width), dtype=torch.float32, device=device)
    _resample([(s, (0, 0, s.shape[1], s.shape[0]), image_u8[i], cloth[i], 1, "bicubic") for i, s in enumerate(srcs)],
              device)
    cw, ch, left, top = clip_resize(width, height)
    small = torch.empty((n, ch, cw, 3), dtype=torch.uint8, device=device)
    _resample([(image_u8[i], (0, 0, width, height), small[i], None, 0, "bicubic") for i in range(n)], device)
    pixels = torch.empty((n, 3, CLIP_SIZE, CLIP_SIZE), dtype=torch.float32, device=device)
    L.clip_pixels_u8([L.ClipDesc(src=small[i].data_ptr(), src_pitch=3 * cw, src_w=cw, src_h=ch, crop_x=left,
                                 crop_y=top) for i in range(n)], _clip_table_on(device), pixels)
    return [PreparedGarment(image_u8=image_u8[i], cloth=cloth[i], clip_pixels=pixels[i]) for i in range(n)]


def paste_back(prepared, images_u8, mode="crop", masks=None):
    """The full-resolution results: images_u8 (uint8 [B, height, width, 3] CUDA, the bytes the pipeline's "pil" output
    is made of) resampled back to each crop's size with its filter, then pasted into its photo at paste_offset, in one
    resample call and one b200vton_paste_u8 launch. Returns a list of uint8 [H, W, 3] CUDA tensors.

    mode (one for all, or one per entry): "crop" replaces the whole box (the demo); "mask" replaces only the pixels
    where the mask is set and keeps every other byte of the photo. The mask is the entry's photo-size mask (set where
    >= 128), else masks[i], the server-size mask of the request ([1, height, width], binarised at 0.5 as the pipeline
    does, x 255, resampled to the crop size with the same filter, set where >= 128)."""
    n = len(prepared)
    modes = [mode] * n if isinstance(mode, str) else list(mode)
    if len(modes) != n or any(m not in PASTE_MODES for m in modes):
        raise ValueError(f"paste_back: mode must be one of {PASTE_MODES} (or one per photo), got {mode!r}")
    if images_u8.dtype != torch.uint8 or not images_u8.is_cuda or images_u8.dim() != 4 or images_u8.shape[0] != n or \
            images_u8.shape[3] != 3:
        raise ValueError(f"paste_back: images_u8 must be uint8 CUDA [{n}, height, width, 3], got {images_u8.dtype} "
                         f"{tuple(images_u8.shape)} on {images_u8.device}")
    device = images_u8.device
    images_u8 = images_u8.contiguous()
    h, w = images_u8.shape[1:3]
    jobs, pastes, dsts = [], [], []
    for i, (e, m) in enumerate(zip(prepared, modes)):
        x0, y0, x1, y1 = e.crop
        cw, ch = x1 - x0, y1 - y0
        px, py = paste_offset(e.box)
        back = torch.empty((ch, cw, 3), dtype=torch.uint8, device=device)
        jobs.append((images_u8[i], (0, 0, w, h), back, None, 0, e.filter))
        mask, mx, my = None, 0, 0
        if m == "mask":
            if e.photo_mask is not None:
                mask = e.photo_mask
            else:
                sm = None if masks is None else masks[i]
                if sm is None or not torch.is_tensor(sm) or tuple(sm.shape[-2:]) != (h, w) or sm.numel() != h * w:
                    raise ValueError(f"paste_back: photo {i} has no photo-size mask; mode 'mask' needs its server-size "
                                     f"[1, {h}, {w}] mask in masks")
                binary = ((sm.reshape(h, w, 1).to(device=device, dtype=torch.float32) >= 0.5).to(torch.uint8) * 255)
                mask = torch.empty((ch, cw), dtype=torch.uint8, device=device)
                jobs.append((binary, (0, 0, w, h), mask[..., None], None, 0, e.filter))
                mx, my = px, py
        dst = torch.empty_like(e.photo)
        W, H = e.size
        pastes.append(L.PasteDesc(photo=e.photo.data_ptr(), photo_pitch=3 * W, dst=dst.data_ptr(), dst_pitch=3 * W,
                                  image=back.data_ptr(), image_pitch=3 * cw,
                                  mask=None if mask is None else mask.data_ptr(),
                                  mask_pitch=0 if mask is None else mask.shape[1], width=W, height=H, box_x=px,
                                  box_y=py, box_w=cw, box_h=ch, mask_x=mx, mask_y=my,
                                  mask_w=0 if mask is None else mask.shape[1], mask_h=0 if mask is None else mask.shape[0]))
        dsts.append(dst)
    _resample(jobs, device)
    L.paste_u8(pastes, device)
    return dsts
