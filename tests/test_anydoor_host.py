"""AnyDoor's pair preparation without a GPU: the numpy restatement (oracle/anydoor_oracle.py) against the reference's own
``process_pairs`` / ``sobel`` / ``crop_back`` bytes (tests/golden/make_golden_anydoor.py) and against live OpenCV; the host box
geometry of ``anyedit_b200.anydoor`` against the oracle's; the refusals and the absence of a CPU fallback."""
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import anydoor_oracle as O

G = os.path.join(os.path.dirname(__file__), "golden")


def sha(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(G, "anydoor_golden.npz"))


@pytest.mark.parametrize("name", list(O.CASES))
def test_oracle_matches_reference(gold, name):
    ri, rm, ti, tm, seed = O.case_inputs(name)
    assert sha(ri, rm, ti, tm) == str(gold[f"{name}/in"]), "the seeded inputs changed"
    st = {}
    np.random.seed(seed)
    item = O.process_pairs(ri, rm, ti, tm, stages=st)
    for k in ("ref", "jpg", "hint"):
        assert item[k].dtype == np.float32 and sha(item[k]) == str(gold[f"{name}/{k}"]), k
    assert np.array_equal(item["extra_sizes"], gold[f"{name}/extra_sizes"])
    assert np.array_equal(item["tar_box_yyxx_crop"], gold[f"{name}/tar_box_yyxx_crop"])
    assert sha(O.sobel(st["ref_u8"], st["ref_mask_u8"] / 255)) == str(gold[f"{name}/hf"])
    back = O.crop_back(O.decode_to_pred(O.case_pred(seed)), ti, item["extra_sizes"], item["tar_box_yyxx_crop"])
    assert sha(back) == str(gold[f"{name}/crop_back"])
    print(f"[anydoor oracle] {name}: every fp32 bit of ref / jpg / hint and every byte of the high-frequency map and of crop_back "
          f"equal the reference's (OpenCV {gold['cv2_version']})")


SIZES = [((224, 224), (256, 256)), ((256, 256), (224, 224)), ((480, 640), (512, 512)), ((417, 300), (512, 512)),
         ((35, 900), (512, 512)), ((1000, 1000), (512, 512)), ((224, 224), (112, 112)), ((511, 512), (289, 289)),
         ((61, 93), (7, 200)), ((1, 5), (3, 1)), ((37, 1), (9, 4))]


@pytest.mark.parametrize("src,dst", SIZES)
@pytest.mark.parametrize("ch", [1, 3])
def test_resizes_match_live_cv2(src, dst, ch):
    """uint8 linear and nearest equal OpenCV on every byte, with its optimised paths on and off (upscales, downscales, the exact
    2x that OpenCV sends to INTER_AREA, lines); float64 and float32 equal OpenCV's own arithmetic on every bit.  The default build
    sends float32 through Intel IPP, whose weights differ slightly: reported, not asserted."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(sum(src) * 7 + sum(dst) + ch)
    shape = src + ((3,) if ch == 3 else ())
    img = rng.integers(0, 256, shape, dtype=np.uint8)
    f32 = rng.uniform(0, 255, shape).astype(np.float32)
    size = (dst[1], dst[0])
    was = cv2.useOptimized()
    try:
        for optimized in (True, False):
            cv2.setUseOptimized(optimized)
            assert np.array_equal(O.resize_u8(img, size), cv2.resize(img, size))
            assert np.array_equal(O.resize_nearest(img, size), cv2.resize(img, size, interpolation=cv2.INTER_NEAREST))
        if (src[0], src[1]) == (2 * dst[0], 2 * dst[1]):
            return                      # floats at exact 2x go to INTER_AREA; no float resize here is ever one
        assert np.array_equal(O.resize_f64(img / 255, size), cv2.resize(img / 255, size))
        assert np.array_equal(O.resize_f32(f32, size), cv2.resize(f32, size))
        cv2.setUseOptimized(True)
        d = np.abs(O.resize_f32(f32, size).astype(np.float64) - cv2.resize(f32, size))
        print(f"[resize f32] {src}->{dst} x{ch}: default build differs on {int((d > 0).sum())} of {d.size} values, "
              f"by at most {d.max():.2e}")
    finally:
        cv2.setUseOptimized(was)


@pytest.mark.parametrize("name", list(O.CASES))
def test_sobel_vs_live_cv2(gold, name):
    """Live OpenCV through the reference's ``sobel`` steps equals the restatement on every byte; the default build's crop_back
    (IPP) is within one of OpenCV's own arithmetic on every byte (recorded in the golden)."""
    cv2 = pytest.importorskip("cv2")
    ri, rm, ti, tm, seed = O.case_inputs(name)
    st = {}
    np.random.seed(seed)
    item = O.process_pairs(ri, rm, ti, tm, stages=st)
    ref, mask = st["ref_u8"], st["ref_mask_u8"] / 255
    im = cv2.resize(ref, (256, 256))
    m = cv2.erode((cv2.resize(mask, (256, 256)) > 0.5).astype(np.uint8), np.ones((5, 5), np.uint8), iterations=2)
    sx, sy = cv2.Sobel(im, cv2.CV_64F, 1, 0, ksize=3), cv2.Sobel(im, cv2.CV_64F, 0, 1, ksize=3)
    s = np.max(cv2.addWeighted(cv2.convertScaleAbs(sx), 0.5, cv2.convertScaleAbs(sy), 0.5, 0), -1) * m
    s[s < 50] = 0
    s = (np.stack([s] * 3, -1).astype(np.float32) / 255 * im.astype(np.float32)).astype(np.uint8)
    assert np.array_equal(O.sobel(ref, mask), cv2.resize(s, (224, 224)))
    assert int(gold[f"{name}/crop_back_ipp"][1]) <= 1
    print(f"[crop_back] {name}: the default OpenCV build (IPP float32 resize) differs from its own arithmetic on "
          f"{int(gold[f'{name}/crop_back_ipp'][0])} pasted bytes, by at most {int(gold[f'{name}/crop_back_ipp'][1])}")


def test_geometry_matches_oracle():
    """The host box arithmetic of anyedit_b200.anydoor (with the device bounding box replaced by numpy's) draws the same random
    numbers in the same order and gives the oracle's boxes and sizes, including int() truncation toward zero of negatives."""
    from anyedit_b200 import anydoor as A
    rng = np.random.default_rng(0)
    for it in range(300):
        H, W = (512, 512) if it % 3 else tuple(int(v) for v in rng.integers(40, 700, 2))
        ref_mask, tar_mask = (np.zeros((H, W), np.uint8) for _ in range(2))
        for m in (ref_mask, tar_mask):
            y0, x0 = rng.integers(0, H - 1), rng.integers(0, W - 1)
            m[y0:y0 + rng.integers(2, H), x0:x0 + rng.integers(2, W)] = 1
            if it % 17 == 0:
                m[:] = 0
                m[y0, x0] = 1
        s = int(rng.integers(1 << 30))
        np.random.seed(s)
        item = O.process_pairs(rng.integers(0, 256, (H, W, 3), dtype=np.uint8), ref_mask,
                               rng.integers(0, 256, (H, W, 3), dtype=np.uint8), tar_mask)
        np.random.seed(s)
        g = A.pair_geometry(A.bbox_numpy(ref_mask), A.bbox_numpy(tar_mask), (H, W), (H, W))
        assert list(item["extra_sizes"]) == [g.H1, g.W1, g.H2, g.W2]
        assert list(item["tar_box_yyxx_crop"]) == list(g.crop)


def test_refusals_and_no_cpu_path():
    from anyedit_b200 import anydoor as A
    img, m = np.zeros((64, 64, 3), np.uint8), np.ones((64, 64), np.uint8)
    for bad in ((img.astype(np.float32), m, img, m), (img, m * 2, img, m), (img, m[:32], img, m), (img[..., :2], m, img, m)):
        with pytest.raises(ValueError):
            A.process_pairs(*bad)
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="CUDA"):
            A.process_pairs(img, m, img, m)
        with pytest.raises(RuntimeError, match="CUDA"):
            A.crop_back(np.zeros((511, 512, 3), np.float32), img, np.array([64, 64, 64, 64]), np.array([0, 64, 0, 64]))
