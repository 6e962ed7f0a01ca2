"""Integer restatement of AnyEdit's Canny sketch annotator (visual_condition_tool.py ``img2sketch``: cvtColor(BGR2GRAY),
GaussianBlur((3, 3), 0), Canny(low, high) with a 3x3 aperture and the L1 gradient, bitwise_not) in numpy (TEST
INFRASTRUCTURE, see oracle/__init__.py).  Every step is integer arithmetic, so it is meant to equal OpenCV on every pixel:

  grey   (B 3735 + G 19235 + R 9798 + 2^14) >> 15
  blur   [1, 2, 1] along x, then along y, then (v + 8) >> 4; BORDER_REFLECT_101 (an axis of length 1 reflects onto itself)
  sobel  3x3 dx, dy on the blurred image, BORDER_REPLICATE; m = |dx| + |dy|
  nms    m outside the image is 0; t = |dx| 13573: |dy| << 15 < t keeps m > left, m >= right; |dy| << 15 > t + (|dx| << 16)
         keeps m > up, m >= down; otherwise the diagonal through (up, x - s) and (down, x + s), s = -1 if dx ^ dy < 0 else 1,
         both strict.  A kept pixel with m > low is a candidate; with m > high also strong.
  hyst   255 on every candidate whose 8-connected candidate component holds a strong pixel, then inverted.

``tests/golden/make_golden_sketch.py`` pins it against the reference's own ``img2sketch``; the tests also hold it against the
live cv2 chain.
"""
import numpy as np
from scipy import ndimage

GOLDEN_SIZES = ((48, 64), (61, 93), (17, 200), (1, 37), (512, 512))


def _reflect101(n):
    """Index map of the positions -1 .. n onto 0 .. n - 1 (BORDER_REFLECT_101; an axis of length 1 maps onto itself)."""
    i = np.arange(-1, n + 1)
    i = np.where(i < 0, -i, i)
    i = np.where(i >= n, 2 * n - 2 - i, i)
    return np.clip(i, 0, n - 1)


def grey(img):
    """uint8 [..., H, W, 3] BGR -> int32 [..., H, W]."""
    b, g, r = (img[..., c].astype(np.int32) for c in range(3))
    return (b * 3735 + g * 19235 + r * 9798 + (1 << 14)) >> 15


def blur(gr):
    """GaussianBlur((3, 3), 0) of an integer image [H, W]."""
    H, W = gr.shape
    p = gr[_reflect101(H)][:, _reflect101(W)]
    h = p[:, :-2] + 2 * p[:, 1:-1] + p[:, 2:]
    v = h[:-2] + 2 * h[1:-1] + h[2:]
    return (v + 8) >> 4


def sobel(bl):
    """3x3 Sobel dx, dy of an integer image [H, W] with replicated borders."""
    p = np.pad(bl, 1, mode="edge")
    dx = (p[:-2, 2:] - p[:-2, :-2]) + 2 * (p[1:-1, 2:] - p[1:-1, :-2]) + (p[2:, 2:] - p[2:, :-2])
    dy = (p[2:, :-2] - p[:-2, :-2]) + 2 * (p[2:, 1:-1] - p[:-2, 1:-1]) + (p[2:, 2:] - p[:-2, 2:])
    return dx, dy


def classes(img, low=50, high=150):
    """uint8 [H, W, 3] BGR -> uint8 [H, W]: 0 not a candidate, 1 weak candidate, 2 strong."""
    dx, dy = sobel(blur(grey(img)))
    H, W = dx.shape
    m = np.abs(dx) + np.abs(dy)
    mp = np.pad(m, 1)                                   # the magnitude outside the image is 0
    nb = lambda oy, ox: mp[1 + oy:1 + oy + H, 1 + ox:1 + ox + W]
    xs, ys = np.abs(dx), np.abs(dy)
    t = xs * 13573
    horiz = (ys << 15) < t
    vert = ~horiz & ((ys << 15) > t + (xs << 16))
    diag = ~horiz & ~vert
    neg = (dx ^ dy) < 0                                 # s = -1: up-right and down-left; s = +1: up-left and down-right
    keep = np.where(horiz, (m > nb(0, -1)) & (m >= nb(0, 1)), False)
    keep |= vert & (m > nb(-1, 0)) & (m >= nb(1, 0))
    keep |= diag & np.where(neg, (m > nb(-1, 1)) & (m > nb(1, -1)), (m > nb(-1, -1)) & (m > nb(1, 1)))
    cand = keep & (m > low)
    return (cand.astype(np.uint8) + (cand & (m > high))).astype(np.uint8)


def hysteresis(cls):
    """Class map [H, W] -> Canny's uint8 edge map: 255 on the 8-connected candidate components holding a strong pixel."""
    lab, n = ndimage.label(cls > 0, structure=np.ones((3, 3), dtype=int))
    keep = np.zeros(n + 1, dtype=bool)
    keep[np.unique(lab[cls == 2])] = True
    keep[0] = False
    return np.where(keep[lab], 255, 0).astype(np.uint8)


def sketch(img, low=50, high=150):
    """img2sketch's array: uint8 [H, W, 3] BGR -> uint8 [H, W], 255 - Canny(GaussianBlur(grey))."""
    if not (isinstance(img, np.ndarray) and img.dtype == np.uint8 and img.ndim == 3 and img.shape[2] == 3):
        raise ValueError("sketch: expects a uint8 BGR image [H, W, 3]")
    if not (0 <= low <= high):
        raise ValueError(f"sketch: thresholds must satisfy 0 <= low <= high (got {low}, {high})")
    return 255 - hysteresis(classes(img, low, high))


def images(size, seed, B=1):
    """Seeded structured uint8 BGR images [B, H, W, 3]: a smooth colour field with fine noise, plus drawn discs, bars and a
    ring.  Low-contrast shapes give weak-only edge components, high-contrast ones strong components, and shapes laid over the
    field's ramp change contrast along their outline, so they mix the two."""
    rng = np.random.default_rng(seed)
    H, W = size
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    out = np.empty((B, H, W, 3), dtype=np.uint8)
    for b in range(B):
        img = np.zeros((H, W, 3))
        for c in range(3):
            fy, fx, ph = rng.uniform(0.5, 3.0), rng.uniform(0.5, 3.0), rng.uniform(0, 2 * np.pi)
            img[..., c] = 110 + 50 * np.sin(2 * np.pi * (fy * yy / max(H, 8) + fx * xx / max(W, 8)) + ph)
        img += 60 * (xx / max(W - 1, 1) - 0.5)[..., None]          # a ramp: shapes over it change contrast along their edge
        for _ in range(max(3, H * W // 1500)):
            cy, cx = rng.uniform(0, H), rng.uniform(0, W)
            r = rng.uniform(2, max(3, min(H, W) / 4))
            contrast = rng.choice([12.0, 25.0, 45.0, 90.0]) * rng.choice([-1, 1])
            kind = rng.integers(3)
            if kind == 0:
                mask = (yy - cy) ** 2 + (xx - cx) ** 2 < r * r
            elif kind == 1:
                mask = (np.abs(yy - cy) < r / 3) & (np.abs(xx - cx) < r * 1.5)
            else:
                d = np.sqrt((yy - cy) ** 2 + (xx - cx) ** 2)
                mask = np.abs(d - r) < 1.5
            img[mask] += contrast * rng.uniform(0.7, 1.3, 3)
        img += rng.normal(0, 3.0, img.shape)
        out[b] = np.clip(np.rint(img), 0, 255).astype(np.uint8)
    return out
