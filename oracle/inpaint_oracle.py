"""Restatement of the byte-level steps of AnyEdit's inpainting edits (local_pipeline_tool.py background_change / replace and
diffusers' StableDiffusionInpaintPipeline processors) in numpy.  TEST INFRASTRUCTURE: pinned to live Pillow / OpenCV by
tests/test_inpaint_host.py, and the reference of the kernels in csrc/inpaint.cu.

  Pillow Image.resize, 8 bits per channel (src/libImaging/Resample.c): per axis, output x has centre (x + 0.5) * in / out,
  support = filter support * max(in / out, 1), taps [int(centre - support + 0.5), int(centre + support + 0.5)) clipped to the
  image, weights filter((tap - centre + 0.5) / max(scale, 1)) normalised in double and rounded to 22-bit fixed point away
  from zero; the horizontal pass first, clipped to bytes, then the vertical one; an axis that keeps its size is skipped.
  NEAREST (forced for mode "1", Geometry.c ImagingScaleAffine): a double source position from in / out * 0.5 in steps of
  in / out, truncated.  Live Pillow 12.2 runs the vertical pass first for some narrow, tall images (width below 7 and a few
  hundred rows or more, both axes resized); this restatement and the kernel always run the horizontal pass first.
  OpenCV GaussianBlur((5, 5), 0) of 8-bit images: sigma 0 selects the fixed kernel [1 4 6 4 1] / 16 (8.8 fixed-point rows,
  16.16 columns, one rounding); BORDER_REFLECT_101.  BGR2GRAY: (1868 B + 9617 G + 4899 R) / 2^14 as OpenCV's 15-bit
  (3735, 19235, 9798) fixed point.
"""
import math

import numpy as np

PREC = 22


def bicubic(x):
    a = -0.5
    x = abs(x)
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1.0
    if x < 2.0:
        return (((x - 5.0) * x + 8.0) * x - 4.0) * a
    return 0.0


def _sinc(x):
    if x == 0.0:
        return 1.0
    x = x * math.pi
    return math.sin(x) / x


def lanczos(x):
    return _sinc(x) * _sinc(x / 3) if -3.0 <= x < 3.0 else 0.0


FILTERS = {"bicubic": (bicubic, 2.0), "lanczos": (lanczos, 3.0)}


def axis_coeffs(filt, n_in, n_out):
    """Per output position (first tap, int32 weights) of one axis, as Resample.c precompute_coeffs + normalize_coeffs_8bpc."""
    fn, fs = FILTERS[filt]
    scale = n_in / n_out
    filterscale = max(scale, 1.0)
    support = fs * filterscale
    out = []
    for xx in range(n_out):
        center = (xx + 0.5) * scale
        ss = 1.0 / filterscale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), n_in) - xmin
        k = [fn((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for w in k:
            ww += w
        if ww != 0.0:
            k = [w / ww for w in k]
        out.append((xmin, [int(-0.5 + w * (1 << PREC)) if w < 0 else int(0.5 + w * (1 << PREC)) for w in k]))
    return out


def nearest_index(n_in, n_out):
    """Source index of every output position of Pillow's NEAREST resize (Geometry.c ImagingScaleAffine: a double position
    from in / out * 0.5 in steps of in / out, truncated)."""
    a = n_in / n_out
    pos, out = a * 0.5, []
    for _ in range(n_out):
        out.append(int(pos))
        pos += a
    return np.array(out, np.int64)


def _pass(img, coeffs, axis):
    """One convolution pass along ``axis`` (0 rows, 1 columns) of uint8 HWC -> clipped uint8."""
    x = np.moveaxis(img.astype(np.int64), axis, 0)
    out = np.empty((len(coeffs),) + x.shape[1:], np.int64)
    for i, (first, w) in enumerate(coeffs):
        acc = np.full(x.shape[1:], 1 << (PREC - 1), np.int64)
        for k, c in enumerate(w):
            acc += x[first + k] * c
        out[i] = acc
    out = np.clip(out >> PREC, 0, 255).astype(np.uint8)
    return np.moveaxis(out, 0, axis)


def resize(img, size, filt):
    """Image.fromarray(img).resize((W, H), filt) for uint8 [H, W] or [H, W, 3]; size = (H, W); filt "lanczos", "bicubic",
    "nearest"."""
    squeeze = img.ndim == 2
    x = img[..., None] if squeeze else img
    H, W = size
    if filt == "nearest":
        x = x[nearest_index(x.shape[0], H)][:, nearest_index(x.shape[1], W)]
    else:
        if W != x.shape[1]:
            x = _pass(x, axis_coeffs(filt, x.shape[1], W), 1)
        if H != x.shape[0]:
            x = _pass(x, axis_coeffs(filt, x.shape[0], H), 0)
    return x[..., 0] if squeeze else x


def resize_mask(mask, size):
    """The mask processor's resize + convert("L") of a mode "1" (bool) or mode "L" (uint8) mask -> uint8 [H, W]."""
    if mask.dtype == np.bool_:
        return resize(mask.astype(np.uint8) * 255, size, "nearest")
    return resize(mask, size, "lanczos")


def prepare(image, mask, size=512):
    """StableDiffusionInpaintPipeline's processors + prepare_mask_latents (strength 1): -> (masked image float32 [3, S, S],
    binarised mask float32 [1, S, S], mask latent float32 [1, S / 8, S / 8], mask count)."""
    img = resize(image, (size, size), "lanczos")
    x = img.astype(np.float32) / 255.0
    x = (2.0 * x - 1.0).transpose(2, 0, 1)
    m = resize_mask(mask, (size, size)).astype(np.float32) / 255.0
    m = np.where(m < 0.5, np.float32(0), np.float32(1))[None]
    masked = x * (m < 0.5)
    return masked, m, m[:, ::8, ::8].copy(), int(m.sum())


def _reflect101(p, n):
    if n == 1:
        return 0
    while p < 0 or p >= n:
        p = -p if p < 0 else 2 * n - 2 - p
    return p


def gaussian5(img):
    """cv2.GaussianBlur(img, (5, 5), 0) of uint8 [H, W, C]."""
    H, W = img.shape[:2]
    w = np.array([1, 4, 6, 4, 1], np.int64)
    ys = np.array([[_reflect101(y + d, H) for d in range(-2, 3)] for y in range(H)])
    xs = np.array([[_reflect101(x + d, W) for d in range(-2, 3)] for x in range(W)])
    x = img.astype(np.int64)
    rows = sum(w[k] * x[:, xs[:, k]] for k in range(5))
    cols = sum(w[k] * rows[ys[:, k]] for k in range(5))
    return ((cols + 128) >> 8).astype(np.uint8)


def bgr2gray(img):
    x = img.astype(np.int64)
    return ((x[..., 0] * 3735 + x[..., 1] * 19235 + x[..., 2] * 9798 + (1 << 14)) >> 15).astype(np.uint8)


def background_mask(fore_bgr):
    """local_pipeline_tool.py:496-499: bool [H, W] = gray(GaussianBlur(fore, (5, 5), 0)) == 0."""
    return bgr2gray(gaussian5(fore_bgr)) == 0
