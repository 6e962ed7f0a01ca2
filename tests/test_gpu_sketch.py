"""The Canny sketch annotator on the GPU (``sketch.detect`` / ``sketch.img2sketch``, kernels in csrc/sketch.cu): every comparison is
``np.array_equal`` against OpenCV, with no tolerance.

* the reference's golden (tests/golden/make_golden_sketch.py) and the live cv2 chain at real, odd and degenerate sizes and at
  several (low, high) pairs, including low == high and (0, 0);
* hysteresis stress images, each first checked on OpenCV's output for the situation it claims: a weak spiral across many tiles
  kept by a strong inner end, a weak snake that meets a strong edge only in its last tile, weak and strong patches, a noise
  image with 40 % of its pixels candidates and few strong ones, a flat image;
* batch independence, two calls alike (the atomics do not reach the output), a CUDA-graph replay (no host synchronisation) and
  the PNG bytes ``img2sketch`` writes.
"""
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import sketch_oracle as O

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu

G = os.path.join(os.path.dirname(__file__), "golden")
TILE = 32


@pytest.fixture(scope="module")
def sk():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from anyedit_b200 import ops, sketch
    assert tuple(ops.device_info())[1:] == (9, 0), "sm_90a kernels need a Hopper GPU (H100)"
    return sketch


def cv2_sketch(img, low=50, high=150):
    grey = cv2.cvtColor(img, cv2.COLOR_BGR2GRAY)
    return cv2.bitwise_not(cv2.Canny(cv2.GaussianBlur(grey, (3, 3), 0), low, high))


def components(cls):
    from scipy import ndimage
    return ndimage.label(cls > 0, structure=np.ones((3, 3), dtype=int))


def tiles_touched(mask):
    ys, xs = np.nonzero(mask)
    return len(set(zip((ys // TILE).tolist(), (xs // TILE).tolist())))


def same(got, want, name):
    d = int((got != want).sum())
    print(f"{name}: {d} of {want.size} pixels differ from OpenCV, {int((want == 0).sum())} edge pixels")
    return d == 0


# ---- against the reference and live OpenCV ---------------------------------------------------------------------------------
def test_vs_reference_golden(sk):
    g = np.load(os.path.join(G, "sketch_golden.npz"))
    for i, (H, W) in enumerate(O.GOLDEN_SIZES):
        s = f"{H}x{W}"
        img = O.images((H, W), int(g["seed"]) + i)[0]
        if f"img{s}" in g:
            assert np.array_equal(img, g[f"img{s}"])
        else:
            assert hashlib.sha256(img.tobytes()).hexdigest() == str(g[f"imgsha{s}"])
        assert same(sk.detect(img[None])[0], g[f"sketch{s}"], f"[sketch golden] {s}")


SIZES = [(480, 640), (512, 512), (1024, 1024), (97, 131), (33, 65), (1, 200), (200, 1), (1, 1), (2, 2), (3, 5), (31, 33)]


@pytest.mark.parametrize("H,W", SIZES)
def test_vs_live_cv2(sk, H, W):
    img = O.images((H, W), 7 * H + W, B=2)
    got = sk.detect(img)
    for b in range(2):
        assert same(got[b], cv2_sketch(img[b]), f"[sketch live] {H}x{W} image {b}")


@pytest.mark.parametrize("low,high", [(50, 150), (0, 0), (100, 100), (10, 40), (150, 400), (0, 255)])
def test_thresholds(sk, low, high):
    img = O.images((300, 411), 41, B=2)
    got = sk.detect(torch.from_numpy(img).cuda(), low, high).cpu().numpy()
    for b in range(2):
        assert same(got[b], cv2_sketch(img[b], low, high), f"[sketch thresholds] ({low}, {high}) image {b}")


# ---- hysteresis stress -----------------------------------------------------------------------------------------------------
def spiral(n=1024, turns=9, d=20, fade=400, steps=40):
    """A 2-pixel spiral of contrast d, too weak to be strong anywhere, whose inner end fades in from full contrast."""
    img = np.full((n, n, 3), 128, np.uint8)
    t = np.linspace(0, 2 * np.pi * turns, 20000)
    r = 20 + (n / 2 - 30) * t / t[-1]
    pts = np.stack([n / 2 + r * np.cos(t), n / 2 + r * np.sin(t)], 1).round().astype(np.int32)
    cv2.polylines(img, [pts], False, (128 + d,) * 3, 2)
    for k in range(steps):
        a, b = k * fade // steps, (k + 1) * fade // steps + 1
        cv2.polylines(img, [pts[a:b]], False, (int(round(255 - (127 - d) * k / (steps - 1))),) * 3, 2)
    return img


def snake(h=512, w=768, d=30, pitch=24, fade=24, steps=12):
    """A weak serpentine from the first tile down the whole image; only its last few pixels fade in to full contrast."""
    img = np.full((h, w, 3), 128, np.uint8)
    pts = []
    for i, y in enumerate(range(12, h - 12, pitch)):
        xs = (12, w - 12) if i % 2 == 0 else (w - 12, 12)
        pts += [(xs[0], y), (xs[1], y)]
    pts = np.array(pts, np.int32)
    cv2.polylines(img, [pts], False, (128 + d,) * 3, 2)
    (px, y), (ex, _) = pts[-2], pts[-1]
    step = 1 if ex > px else -1
    for k in range(steps):
        x0, x1 = ex - step * (fade - k * fade // steps), ex - step * (fade - (k + 1) * fade // steps)
        cv2.line(img, (int(x0), int(y)), (int(x1), int(y)), (int(round(128 + d + (127 - d) * (k + 1) / steps)),) * 3, 2)
    return img


def patches(n=512, cell=32, weak=30, strong=90):
    img = np.full((n, n, 3), 128, np.uint8)
    for i, y in enumerate(range(4, n - cell, cell)):
        for j, x in enumerate(range(4, n - cell, cell)):
            cv2.rectangle(img, (x, y), (x + cell - 10, y + cell - 10), (128 + (strong if (i + j) % 2 else weak),) * 3, -1)
    return img


def check_spiral(img, cls, want):
    lab, n = components(cls)
    big = np.bincount(lab.ravel())[1:].argmax() + 1
    comp = lab == big
    assert int((cls[comp] == 2).sum()) < 100 and int((cls[comp] == 1).sum()) > 30000, "the spiral should be weak but for its end"
    assert tiles_touched(comp) > 200 and bool((want[comp] == 0).all()), "OpenCV should keep the whole spiral"


def check_snake(img, cls, want):
    lab, n = components(cls)
    assert int(np.nonzero(cls == 2)[0].min()) >= img.shape[0] - 2 * TILE, "only the square at the snake's end should be strong"
    comp = lab == lab[np.nonzero(cls == 2)][0]
    assert tiles_touched(comp) > 150 and bool((want[comp] == 0).all()), "OpenCV should keep the whole snake"
    assert bool(comp[:TILE, :TILE].any()), "the snake should start in the first tile"


def check_patches(img, cls, want):
    lab, n = components(cls)
    strong = np.bincount(lab.ravel(), weights=(cls == 2).ravel(), minlength=n + 1)[1:]
    assert int((strong == 0).sum()) > 50 and int((strong > 0).sum()) > 50, "want both weak-only and strong patches"
    kept = np.bincount(lab.ravel(), weights=(want == 0).ravel(), minlength=n + 1)[1:]
    assert bool((kept[strong == 0] == 0).all()) and bool((kept[strong > 0] > 0).all())


def check_dense(img, cls, want):
    lab, n = components(cls)
    frac, kept = float((cls > 0).mean()), float((want[cls > 0] == 0).mean())
    print(f"[sketch dense] {frac:.3f} of pixels are candidates in {n} components, {kept:.3f} of them kept")
    assert frac > 0.35, "non-maximum suppression lets through at most about 40 % of a noise image"
    assert 0 < int((cls == 2).sum()) < 0.01 * cls.size and kept > 0.5, "a few strong pixels should keep most candidates"
    sizes = np.bincount(lab.ravel())[1:]
    assert tiles_touched(lab == sizes.argmax() + 1) > 50, "the largest component should cross many tiles"


def check_flat(img, cls, want):
    assert not cls.any() and bool((want == 255).all())


STRESS = {
    "spiral": (spiral, 50, 150, check_spiral),
    "snake": (snake, 50, 150, check_snake),
    "patches": (patches, 50, 150, check_patches),
    "dense": (lambda: np.random.default_rng(5).integers(0, 256, (512, 512, 3), dtype=np.uint8), 0, 400, check_dense),
    "flat": (lambda: np.full((256, 320, 3), 77, np.uint8), 50, 150, check_flat),
}


@pytest.mark.parametrize("name", list(STRESS))
def test_hysteresis_stress(sk, name):
    make, low, high, check = STRESS[name]
    img = make()
    want = cv2_sketch(img, low, high)
    cls = O.classes(img, low, high)
    assert np.array_equal(O.hysteresis(cls), 255 - want), "the oracle's classes should explain OpenCV's output"
    check(img, cls, want)
    assert same(sk.detect(img[None], low, high)[0], want, f"[sketch stress] {name}")


# ---- determinism, batches, graphs, files ------------------------------------------------------------------------------------
def test_batch_independence_and_repeatability(sk):
    imgs = np.concatenate([O.images((256, 384), 61, B=3), spiral(n=768)[None, :256, :384]])
    x = torch.from_numpy(imgs).cuda()
    four = sk.detect(x)
    assert torch.equal(sk.detect(x), four), "two calls differ"
    for i in range(4):
        assert torch.equal(sk.detect(x[i:i + 1])[0], four[i]), f"image {i}: batch 1 != batch 4"
        assert np.array_equal(four[i].cpu().numpy(), cv2_sketch(imgs[i]))


def test_cuda_graph_replay(sk):
    imgs = O.images((480, 640), 71, B=2)
    x = torch.from_numpy(imgs).cuda()
    eager = sk.detect(x)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        sk.detect(x)                                   # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = sk.detect(x)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
    x.copy_(torch.from_numpy(O.images((480, 640), 72, B=2)).cuda())
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, sk.detect(x)), "a replay on new pixels differs from the eager call"


def test_img2sketch_png_bytes(sk, tmp_path):
    g = np.load(os.path.join(G, "sketch_golden.npz"))
    src, dst = str(tmp_path / "in.png"), str(tmp_path / "out.png")
    assert cv2.imwrite(src, g["img61x93"])
    sk.img2sketch(src, dst)
    assert open(dst, "rb").read() == g["png61x93"].tobytes(), "img2sketch should write the reference's PNG bytes"
