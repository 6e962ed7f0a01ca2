"""Numpy restatement of AnyDoor's pair preparation and crop-back (AnyEdit_Collection/adaptive_editing_pipelines:
visual_reference_tool.py ``process_pairs`` / ``crop_back``, tools/tool.py ``sobel`` and the box helpers) with the OpenCV
calls written out as arithmetic (TEST INFRASTRUCTURE, see oracle/__init__.py).  It documents the formulas csrc/anydoor.cu
implements:

  resize_u8   cv2.resize(INTER_LINEAR) of uint8 images.  Per axis, f = float32((d + 0.5) * (1 / (out / in)) - 0.5) in double,
              s = floor(f), f -= s; the weights are round(2048 (1 - f)), round(2048 f).  Along x a source index outside
              [0, in - 1] is clamped and its fraction zeroed; along y it is NOT: the two rows are clamped but the weights are
              kept, which is what makes the first and last rows of an upscale differ from a clamped formula.  Horizontal pass
              S = p0 a0 + p1 a1 (exact int); vertical pass (((S0 >> 4) b0 >> 16) + ((S1 >> 4) b1 >> 16) + 2) >> 2 -- the
              vectorised formula, which OpenCV's exact-2x INTER_AREA branch also equals (weights 1024 / 1024).
  resize_f64  the same coefficients unrounded (float32), passes in double: the mask of ``sobel``.
  resize_f32  the same in float32: ``crop_back``.  No FMA here; OpenCV's SIMD may fuse, so live cv2 can differ in the last bit.
  nearest     s = min(floor(d * (1 / (out / in))), in - 1) in double.
  sobel       mask > 0.5 of the float64 resize, a 9 x 9 erode with the border ignored (= two 5 x 5 erodes), the 3 x 3 Sobel x / y
              with BORDER_REFLECT_101, rint(|v|) saturated, addWeighted 0.5 / 0.5 = rint((a + b) / 2) half to even, channel max
              times mask, < thresh -> 0, uint8(float32(s) / 255 * float32(img)) truncated.
  jpg, hint   float32(x) / 127.5 - 1 in float32; ref = float32(x / 255 in double).

``tests/golden/make_golden_anydoor.py`` pins it against the reference's own functions; the tests also hold it against live cv2.
"""
import numpy as np

SIZE_REF, SIZE_HF, SIZE_OUT, MARGIN = 224, 256, 512, 5


# ---- OpenCV resizes ----------------------------------------------------------------------------------------------------------
def _axis(n_in, n_out, clamp):
    scale = 1.0 / (n_out / n_in)
    f = ((np.arange(n_out, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    if clamp:
        lo, hi = s < 0, s >= n_in - 1
        f[lo | hi] = 0
        s[lo], s[hi] = 0, n_in - 1
    return s, np.clip(s, 0, n_in - 1), np.clip(s + 1, 0, n_in - 1), (np.float32(1) - f).astype(np.float32), f


def _hwc(img):
    return img.reshape(img.shape[0], img.shape[1], -1)


def resize_u8(img, size):
    """cv2.resize(img, size) of a uint8 [H, W] or [H, W, C] image, size = (out_w, out_h)."""
    ow, oh = size
    x = _hwc(img).astype(np.int64)
    ih, iw = x.shape[:2]
    _, x0, x1, a0, a1 = _axis(iw, ow, True)
    _, y0, y1, b0, b1 = _axis(ih, oh, False)
    q = lambda w: np.rint(w.astype(np.float32) * np.float32(2048)).astype(np.int64)
    a0, a1, b0, b1 = q(a0), q(a1), q(b0), q(b1)
    S = x[:, x0] * a0[None, :, None] + x[:, x1] * a1[None, :, None]
    out = (((S[y0] >> 4) * b0[:, None, None] >> 16) + ((S[y1] >> 4) * b1[:, None, None] >> 16) + 2) >> 2
    return out.astype(np.uint8).reshape((oh, ow) + img.shape[2:])


def _resize_float(img, size, dt):
    ow, oh = size
    x = _hwc(img).astype(dt)
    ih, iw = x.shape[:2]
    _, x0, x1, a0, a1 = _axis(iw, ow, True)
    _, y0, y1, b0, b1 = _axis(ih, oh, False)
    a0, a1, b0, b1 = (w.astype(dt) for w in (a0, a1, b0, b1))
    S = x[:, x0] * a0[None, :, None] + x[:, x1] * a1[None, :, None]
    out = S[y0] * b0[:, None, None] + S[y1] * b1[:, None, None]
    return out.astype(dt).reshape((oh, ow) + img.shape[2:])


def resize_f64(img, size):
    return _resize_float(img, size, np.float64)


def resize_f32(img, size):
    return _resize_float(img, size, np.float32)


def resize_nearest(img, size):
    ow, oh = size
    ih, iw = img.shape[:2]
    ys = np.minimum(np.floor(np.arange(oh) * (1.0 / (oh / ih))).astype(np.int64), ih - 1)
    xs = np.minimum(np.floor(np.arange(ow) * (1.0 / (ow / iw))).astype(np.int64), iw - 1)
    return img[ys][:, xs]


# ---- tools/tool.py ---------------------------------------------------------------------------------------------------------
def _reflect101(n):
    i = np.arange(-1, n + 1)
    i = np.where(i < 0, -i, i)
    i = np.where(i >= n, 2 * n - 2 - i, i)
    return np.clip(i, 0, n - 1)


def erode9(m):
    """Minimum over the 9 x 9 window inside the image (the border is ignored)."""
    H, W = m.shape
    p = np.pad(m, 4, constant_values=255)
    out = np.full_like(m, 255)
    for dy in range(9):
        for dx in range(9):
            out = np.minimum(out, p[dy:dy + H, dx:dx + W])
    return out


def sobel(img, mask, thresh=50):
    """tool.py sobel: uint8 [H, W, 3] image, float64 [H, W] mask (values / 255) -> the uint8 high-frequency map [H, W, 3]."""
    H, W = img.shape[:2]
    im = resize_u8(img, (SIZE_HF, SIZE_HF))
    m = (resize_f64(mask, (SIZE_HF, SIZE_HF)) > 0.5).astype(np.uint8)
    m = erode9(m)
    p = im.astype(np.int64)[_reflect101(SIZE_HF)][:, _reflect101(SIZE_HF)]
    c = lambda dy, dx: p[1 + dy:1 + dy + SIZE_HF, 1 + dx:1 + dx + SIZE_HF]
    gx = (c(-1, 1) - c(-1, -1)) + 2 * (c(0, 1) - c(0, -1)) + (c(1, 1) - c(1, -1))
    gy = (c(1, -1) - c(-1, -1)) + 2 * (c(1, 0) - c(-1, 0)) + (c(1, 1) - c(-1, 1))
    ax, ay = np.minimum(np.abs(gx), 255), np.minimum(np.abs(gy), 255)
    s = np.rint((ax + ay).astype(np.float64) * 0.5).astype(np.int64).max(-1) * m
    s[s < thresh] = 0
    s3 = np.repeat(s[:, :, None], 3, -1)
    hf = ((s3.astype(np.float32) / np.float32(255)) * im.astype(np.float32)).astype(np.uint8)
    return resize_u8(hf, (W, H))


def get_bbox_from_mask(mask):
    h, w = mask.shape
    if mask.sum() < 10:
        return 0, h, 0, w
    ys, xs = np.nonzero(mask)
    return int(ys.min()), int(ys.max()), int(xs.min()), int(xs.max())


def expand_bbox(shape, yyxx, ratio):
    y1, y2, x1, x2 = yyxx
    ratio = np.random.randint(ratio[0] * 10, ratio[1] * 10) / 10
    H, W = shape[:2]
    xc, yc = 0.5 * (x1 + x2), 0.5 * (y1 + y2)
    h, w = ratio * (y2 - y1 + 1), ratio * (x2 - x1 + 1)
    x1, x2, y1, y2 = int(xc - w * 0.5), int(xc + w * 0.5), int(yc - h * 0.5), int(yc + h * 0.5)
    return max(0, y1), min(H, y2), max(0, x1), min(W, x2)


def box2square(shape, box):
    H, W = shape[:2]
    y1, y2, x1, x2 = box
    cx, cy = (x1 + x2) // 2, (y1 + y2) // 2
    h, w = y2 - y1, x2 - x1
    if h >= w:
        x1, x2 = cx - h // 2, cx + h // 2
    else:
        y1, y2 = cy - w // 2, cy + w // 2
    return max(0, y1), min(H, y2), max(0, x1), min(W, x2)


def pad_square(img, value):
    H, W = img.shape[:2]
    if H == W:
        return img
    p = abs(H - W)
    p1 = int(p / 2)
    pad = ((0, 0), (p1, p - p1)) if H > W else ((p1, p - p1), (0, 0))
    return np.pad(img, pad + ((0, 0),) * (img.ndim - 2), constant_values=value)


def process_pairs(ref_image, ref_mask, tar_image, tar_mask, stages=None):
    """visual_reference_tool.py process_pairs; ``stages`` (a dict) receives the uint8 intermediates."""
    st = stages if stages is not None else {}
    y1, y2, x1, x2 = get_bbox_from_mask(ref_mask)
    m3 = ref_mask[:, :, None].astype(np.int64)
    masked = (ref_image * m3 + 255 * (1 - m3))[y1:y2, x1:x2].astype(np.uint8)
    crop_mask = ref_mask[y1:y2, x1:x2]
    ratio = np.random.randint(11, 13) / 10
    h, w = masked.shape[:2]
    H, W = int(h * ratio), int(w * ratio)
    h1, w1 = int((H - h) // 2), int((W - w) // 2)
    masked = np.pad(masked, ((h1, H - h - h1), (w1, W - w - w1), (0, 0)), constant_values=255)
    crop_mask = np.pad(crop_mask, ((h1, H - h - h1), (w1, W - w - w1)), constant_values=0)
    ref = resize_u8(pad_square(masked, 255), (SIZE_REF, SIZE_REF))
    rmask = resize_u8(pad_square(crop_mask * np.uint8(255), 0), (SIZE_REF, SIZE_REF))
    hf = sobel(ref, rmask / 255)
    st.update(ref_u8=ref, ref_mask_u8=rmask, hf=hf)

    box = expand_bbox(tar_mask.shape, get_bbox_from_mask(tar_mask), [1.1, 1.2])
    crop = box2square(tar_image.shape, expand_bbox(tar_image.shape, box, [1.5, 3]))
    cy1, cy2, cx1, cx2 = crop
    target = tar_image[cy1:cy2, cx1:cx2]
    by1, by2, bx1, bx2 = box[0] - cy1, box[1] - cy1, box[2] - cx1, box[3] - cx1
    collage = target.copy()
    collage[by1:by2, bx1:bx2] = resize_u8(hf, (bx2 - bx1, by2 - by1))
    cmask = np.zeros(target.shape[:2], np.uint8)
    cmask[by1:by2, bx1:bx2] = 1
    H1, W1 = target.shape[:2]
    target, collage, cmask = pad_square(target, 0), pad_square(collage, 0), pad_square(cmask, 255)
    H2, W2 = collage.shape[:2]
    t512, c512 = resize_u8(target, (SIZE_OUT, SIZE_OUT)), resize_u8(collage, (SIZE_OUT, SIZE_OUT))
    m512 = (resize_nearest(cmask, (SIZE_OUT, SIZE_OUT)) > 0.5).astype(np.float32)
    st.update(target_u8=t512, collage_u8=c512)
    norm = lambda x: x.astype(np.float32) / np.float32(127.5) - np.float32(1.0)
    return dict(ref=(ref / 255).astype(np.float32), jpg=norm(t512), hint=np.concatenate([norm(c512), m512[:, :, None]], -1),
                extra_sizes=np.array([H1, W1, H2, W2]), tar_box_yyxx_crop=np.array(crop))


def crop_back(pred, tar_image, extra_sizes, tar_box_yyxx_crop):
    """visual_reference_tool.py crop_back on float32 pred [511, 512, 3]; returns a new image (the caller's is left alone)."""
    H1, W1, H2, W2 = (int(v) for v in extra_sizes)
    y1, y2, x1, x2 = (int(v) for v in tar_box_yyxx_crop)
    pred = resize_f32(pred, (W2, H2))
    m = MARGIN
    if W1 < W2:
        p1 = int((W2 - W1) / 2)
        pred = pred[:, p1:p1 + W1]
    elif H1 < H2:
        p1 = int((H2 - H1) / 2)
        pred = pred[p1:p1 + H1]
    out = tar_image.copy()
    out[y1 + m:y2 - m, x1 + m:x2 - m] = pred[m:-m, m:-m]
    return out


def decode_to_pred(x):
    """visual_reference_tool.py:221-227 on one decoded image [3, H, W] fp32: clip(x * 127.5 + 127.5, 0, 255)[1:] as HWC fp32."""
    y = np.transpose(x, (1, 2, 0)).astype(np.float32) * np.float32(127.5) + np.float32(127.5)
    return np.clip(y, 0, 255)[1:]


# ---- seeded cases (tests/golden/make_golden_anydoor.py) --------------------------------------------------------------------
# name: (ref image size, ref mask ellipse (cy, cx, ry, rx) in fractions of the size, tar size, tar ellipse, seed)
CASES = {
    "blob512": ((512, 512), (0.45, 0.55, 0.25, 0.2), (512, 512), (0.5, 0.4, 0.15, 0.2), 1),
    "edges": ((512, 512), (0.1, 0.05, 0.3, 0.3), (512, 512), (0.95, 0.9, 0.25, 0.3), 2),
    "edges_tr": ((512, 512), (0.95, 0.98, 0.2, 0.3), (512, 512), (0.02, 0.97, 0.2, 0.1), 3),
    "tiny": ((512, 512), (0.5, 0.5, 0.003, 0.003), (512, 512), (0.3, 0.3, 0.004, 0.003), 4),
    "wide": ((512, 512), (0.5, 0.5, 0.04, 0.4), (512, 512), (0.6, 0.5, 0.03, 0.35), 5),
    "tall": ((512, 512), (0.5, 0.5, 0.4, 0.05), (512, 512), (0.45, 0.5, 0.4, 0.04), 6),
    "square": ((512, 512), (0.5, 0.5, 0.1, 0.1), (512, 512), (0.5, 0.5, 0.1, 0.1), 8),
    "odd": ((300, 417), (0.4, 0.6, 0.2, 0.15), (333, 289), (0.5, 0.5, 0.12, 0.2), 9),
}


def blob(size, e):
    H, W = size
    cy, cx, ry, rx = e[0] * H, e[1] * W, max(e[2] * H, 0.5), max(e[3] * W, 0.5)
    yy, xx = np.mgrid[0:H, 0:W]
    return ((((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2) <= 1).astype(np.uint8)


def case_inputs(name):
    """(ref_image, ref_mask, tar_image, tar_mask, seed) of a named case: uint8 RGB images and 0/1 uint8 masks."""
    from oracle import sketch_oracle
    rs, re, ts, te, seed = CASES[name]
    return (sketch_oracle.images(rs, 1000 + seed)[0], blob(rs, re), sketch_oracle.images(ts, 2000 + seed)[0], blob(ts, te), seed)


def case_pred(seed):
    """A seeded decoded image [3, 512, 512] fp32, slightly outside [-1, 1] so that the clip is exercised."""
    return np.random.default_rng(3000 + seed).uniform(-1.05, 1.05, (3, SIZE_OUT, SIZE_OUT)).astype(np.float32)
