"""The Canny sketch annotator without a GPU: the integer oracle (oracle/sketch_oracle.py) against the reference's own
``img2sketch`` (tests/golden/make_golden_sketch.py) and against the live cv2 chain with OpenCV's optimised paths on and off, on
every pixel; the tiny shapes; the refusals and the absence of a CPU fallback."""
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import sketch_oracle as O

G = os.path.join(os.path.dirname(__file__), "golden")
TINY = [(1, 1), (1, 7), (7, 1), (2, 2), (2, 9), (3, 5)]


def cv2_sketch(img, low=50, high=150):
    import cv2
    grey = cv2.cvtColor(img, cv2.COLOR_BGR2GRAY)
    return cv2.bitwise_not(cv2.Canny(cv2.GaussianBlur(grey, (3, 3), 0), low, high))


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(G, "sketch_golden.npz"))


def golden_image(g, i, size):
    s = f"{size[0]}x{size[1]}"
    img = O.images(size, int(g["seed"]) + i)[0]
    if f"img{s}" in g:
        assert np.array_equal(img, g[f"img{s}"]), f"{s}: the seeded image changed"
    else:
        assert hashlib.sha256(img.tobytes()).hexdigest() == str(g[f"imgsha{s}"]), f"{s}: the seeded image changed"
    return img


def test_oracle_matches_reference(gold):
    for i, size in enumerate(O.GOLDEN_SIZES):
        s = f"{size[0]}x{size[1]}"
        got = O.sketch(golden_image(gold, i, size))
        print(f"[sketch oracle] {s}: {int((got == 0).sum())} edge pixels, identical to the reference: "
              f"{np.array_equal(got, gold[f'sketch{s}'])} (golden from OpenCV {gold['cv2_version']})")
        assert np.array_equal(got, gold[f"sketch{s}"])


@pytest.mark.parametrize("optimized", [True, False])
def test_oracle_matches_live_cv2(optimized):
    cv2 = pytest.importorskip("cv2")
    was = cv2.useOptimized()
    cv2.setUseOptimized(optimized)
    try:
        for i, size in enumerate([(40, 40), (33, 71), (97, 64), (130, 161)]):
            img = O.images(size, 900 + i)[0]
            for low, high in ((50, 150), (0, 0), (80, 80), (20, 300)):
                assert np.array_equal(O.sketch(img, low, high), cv2_sketch(img, low, high)), (size, low, high)
    finally:
        cv2.setUseOptimized(was)


@pytest.mark.parametrize("size", TINY)
def test_tiny_shapes(size):
    pytest.importorskip("cv2")
    for seed in range(4):
        img = np.random.default_rng(seed).integers(0, 256, (*size, 3), dtype=np.uint8)
        for low, high in ((50, 150), (0, 0), (10, 30)):
            assert np.array_equal(O.sketch(img, low, high), cv2_sketch(img, low, high)), (size, seed, low, high)


def test_refusals_and_no_cpu_fallback():
    from anyedit_b200 import sketch
    ok = np.zeros((1, 8, 8, 3), dtype=np.uint8)
    for bad in (np.zeros((1, 8, 8, 3), dtype=np.float32), np.zeros((1, 8, 8, 4), dtype=np.uint8),
                np.zeros((8, 8, 3), dtype=np.uint8), torch.zeros(1, 8, 8, 1, dtype=torch.uint8),
                torch.zeros(1, 8, 8, 3, dtype=torch.int16)):
        with pytest.raises(ValueError):
            sketch.detect(bad)
    for low, high in ((151, 150), (-1, 150), (-5, -1), (50.0, 150), (50, 150.5)):
        with pytest.raises(ValueError):
            sketch.detect(ok, low, high)
    for low, high in ((151, 150), (-1, 150)):
        with pytest.raises(ValueError):
            O.sketch(ok[0], low, high)
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="CUDA"):
            sketch.detect(ok)
        with pytest.raises(RuntimeError, match="CUDA"):
            sketch.detect(torch.from_numpy(ok))
    else:
        with pytest.raises(RuntimeError, match="CUDA"):
            sketch.detect(torch.from_numpy(ok))


def test_ops_refuses_cpu_tensors():
    from anyedit_b200 import _lib, ops
    with pytest.raises(_lib.AnysdError, match="CUDA"):
        ops.sketch(torch.zeros(1, 8, 8, 3, dtype=torch.uint8), torch.zeros(1, 8, 8, dtype=torch.uint8))
