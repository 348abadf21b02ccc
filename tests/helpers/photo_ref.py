"""numpy restatement of the full-resolution photo path (idm_vton_b200.photo, include/b200vton.h b200vton_resample_u8 /
b200vton_paste_u8): host coefficients, the two integer passes, the crop and the paste — with named mutants, each a
plausible bug, so a test can show that its sweep tells them apart from Pillow.

Mutants: "float_intermediate" (no uint8 rounding between the passes), "vertical_first", "photo_taps" (taps clipped to
the photo instead of the crop: Pillow's resize of the whole photo with a box), "truncated_coefs" (fixed point by
truncation), "round_half_up_crop" (crop edges rounded half up), "rounded_paste" (paste at the crop's rounded corner).
"""
import math

import numpy as np

from idm_vton_b200 import photo as P

MUTANTS = ("float_intermediate", "vertical_first", "photo_taps", "truncated_coefs", "round_half_up_crop",
           "rounded_paste")
SHIFT = P.PRECISION_BITS


def _photo_axis(photo_len, c0, c1, out, filt):
    """Pillow's precompute_coeffs with a box [c0, c1) of a photo axis of photo_len pixels (taps clipped to the photo)."""
    fn, support = P.FILTERS[filt]
    scale = filterscale = (c1 - c0) / out
    filterscale = max(filterscale, 1.0)
    support = support * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out, 2), np.int32)
    kk = np.zeros((out, ksize))
    for xx in range(out):
        center = c0 + (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), photo_len) - xmin
        w = [fn((x + xmin - center + 0.5) * (1.0 / filterscale)) for x in range(xmax)]
        ww = 0.0
        for v in w:
            ww += v
        kk[xx, :xmax] = [v / ww for v in w] if ww else w
        bounds[xx] = (xmin, xmax)
    return bounds, kk


def _axis(photo_len, c0, c1, out, filt, mutant):
    """(first tap in photo coordinates, tap count, fixed-point coefficients) of one axis."""
    if mutant == "photo_taps":
        bounds, kk = _photo_axis(photo_len, c0, c1, out, filt)
    else:
        bounds, kk = P.resample_coefficients(c1 - c0, out, filt)
        bounds = bounds.copy()
        bounds[:, 0] += c0
    k = np.trunc(kk * (1 << SHIFT)).astype(np.int64) if mutant == "truncated_coefs" else P.fixed_point(kk).astype(np.int64)
    return bounds, k


def _clip8(acc):
    return np.clip(acc >> SHIFT, 0, 255).astype(np.uint8)


def _pass(a, bounds, k, axis, src_len, as_float=False):
    """One pass along `axis` (1 = columns, 0 = rows) of a [rows, cols, C] array; taps from absolute source indices."""
    out = bounds.shape[0]
    shape = list(a.shape)
    shape[axis] = out
    acc = np.zeros(shape, np.float64 if as_float else np.int64)
    if not as_float:
        acc += 1 << (SHIFT - 1)
    for t in range(k.shape[1]):
        idx = np.minimum(bounds[:, 0] + t, src_len - 1)
        kt = np.where(t < bounds[:, 1], k[:, t], 0)
        g = np.take(a, idx, axis=axis).astype(acc.dtype)
        acc += g * (kt[None, :, None] if axis == 1 else kt[:, None, None])
    return acc


def resample(photo, crop, out_w, out_h, filt="bicubic", mutant=None):
    """photo uint8 [H, W, C]; crop (x0, y0, x1, y1) integer pixels -> uint8 [out_h, out_w, C]: Pillow's
    photo.crop(crop).resize((out_w, out_h), filt)."""
    H, W = photo.shape[:2]
    x0, y0, x1, y1 = crop
    need_x, need_y = out_w != x1 - x0, out_h != y1 - y0
    if mutant == "photo_taps":
        need_x = need_y = True
    bx, kx = _axis(W, x0, x1, out_w, filt, mutant)
    by, ky = _axis(H, y0, y1, out_h, filt, mutant)
    if not need_x:
        bx, kx = np.stack([np.arange(x0, x1), np.ones(out_w)], 1).astype(np.int32), np.full((out_w, 1), 1 << SHIFT)
    if not need_y:
        by, ky = np.stack([np.arange(y0, y1), np.ones(out_h)], 1).astype(np.int32), np.full((out_h, 1), 1 << SHIFT)
    if mutant == "vertical_first":
        v = _clip8(_pass(photo, by, ky, 0, H))
        bx = bx.copy()
        return _clip8(_pass(v, bx, kx, 1, W))
    if mutant == "float_intermediate":
        h = _pass(photo, bx, kx, 1, W, as_float=True) / (1 << SHIFT)
        acc = _pass(h, by, ky, 0, H, as_float=True)
        return np.clip(np.floor((acc + (1 << (SHIFT - 1))) / (1 << SHIFT)), 0, 255).astype(np.uint8)
    h = _clip8(_pass(photo, bx, kx, 1, W))
    return _clip8(_pass(h, by, ky, 0, H))


def crop_pixels(box, mutant=None):
    if mutant == "round_half_up_crop":
        return tuple(int(math.floor(v + 0.5)) for v in box)
    return P.crop_pixels(box)


def paste(photo, back, box, mutant=None, mask=None):
    """The photo with `back` (the crop-size output) pasted at the demo's offset; with mask [h, w] of the photo's size,
    only where mask >= 128."""
    out = photo.copy()
    px, py = (int(round(box[0])), int(round(box[1]))) if mutant == "rounded_paste" else P.paste_offset(box)
    h, w = back.shape[:2]
    region = out[py:py + h, px:px + w]
    if mask is None:
        region[...] = back
    else:
        sel = mask[py:py + h, px:px + w] >= 128
        region[sel] = back[sel]
    return out
