#!/usr/bin/env python
"""Golden vectors for AnyEdit's Canny sketch annotator, from the reference's own ``img2sketch``
(AnyEdit_Collection/adaptive_editing_pipelines/visual_condition_tool.py:33-45).

That file imports GroundingDINO and SAM at module level, so it cannot be imported: the one function is taken out of its syntax
tree with ``ast`` and executed with ``cv2``, ``os`` and ``np`` in scope (nothing is copied into this repository).  Each seeded
structured image (oracle.sketch_oracle.images) goes in and comes out as a PNG in a temporary directory, at 48 x 64, 61 x 93,
17 x 200, 1 x 37 and 512 x 512.  Written to sketch_golden.npz: per size s, ``img{s}`` (uint8 BGR HWC) and ``sketch{s}`` (the uint8
map the reference wrote), except that the 512 x 512 image is kept as ``imgsha{s}``, the SHA-256 of its bytes, and
regenerated from its seed; ``png{s}``, the bytes of the PNG the reference wrote for the 61 x 93 image; ``seed``; ``cv2_version``.
Usage: python tests/golden/make_golden_sketch.py"""
import ast
import hashlib
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..", "..")))

from oracle import sketch_oracle as O  # noqa: E402
from oracle.ref_import import SRC_ROOT  # noqa: E402

SEED = 131
PNG_SIZE = (61, 93)
BIG = (512, 512)                         # kept as its seed and a SHA-256 of its bytes, not as pixels


def reference_img2sketch():
    import cv2
    path = os.path.join(SRC_ROOT, "AnyEdit_Collection", "adaptive_editing_pipelines", "visual_condition_tool.py")
    tree = ast.parse(open(path).read(), path)
    fn = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "img2sketch"]
    assert len(fn) == 1, "img2sketch not found in the reference"
    scope = {"cv2": cv2, "os": os, "np": np}
    exec(compile(ast.Module(body=fn, type_ignores=[]), path, "exec"), scope)
    return scope["img2sketch"]


def component_kinds(cls):
    """Counts of 8-connected candidate components that are weak only, that mix weak and strong pixels, and that are strong only."""
    from scipy import ndimage
    lab, n = ndimage.label(cls > 0, structure=np.ones((3, 3), dtype=int))
    weak = ndimage.sum(cls == 1, lab, np.arange(1, n + 1))
    strong = ndimage.sum(cls == 2, lab, np.arange(1, n + 1))
    return {"weak": int(((weak > 0) & (strong == 0)).sum()), "mixed": int(((weak > 0) & (strong > 0)).sum()),
            "strong": int(((weak == 0) & (strong > 0)).sum())}


def main():
    import cv2
    img2sketch = reference_img2sketch()
    out = {"seed": np.int64(SEED), "cv2_version": np.array(cv2.__version__)}
    with tempfile.TemporaryDirectory() as tmp:
        for i, size in enumerate(O.GOLDEN_SIZES):
            s = f"{size[0]}x{size[1]}"
            img = O.images(size, SEED + i)[0]
            src, dst = os.path.join(tmp, f"in{s}.png"), os.path.join(tmp, f"out{s}.png")
            assert cv2.imwrite(src, img)
            img2sketch(src, dst)
            sk = cv2.imread(dst, cv2.IMREAD_UNCHANGED)
            assert sk.shape == size and sk.dtype == np.uint8
            kinds = component_kinds(O.classes(img))
            print(f"{s}: {int((sk == 0).sum())} edge pixels; candidate components: {kinds}")
            if size != (1, 37):
                assert kinds["weak"] > 0 and kinds["mixed"] > 0, f"{s}: want both dropped and kept weak pixels"
            out[f"sketch{s}"] = sk
            if size == BIG:
                out[f"imgsha{s}"] = np.array(hashlib.sha256(img.tobytes()).hexdigest())
            else:
                out[f"img{s}"] = img
            if size == PNG_SIZE:
                out[f"png{s}"] = np.frombuffer(open(dst, "rb").read(), dtype=np.uint8)
    np.savez_compressed(os.path.join(HERE, "sketch_golden.npz"), **out)
    print({k: (v.shape if hasattr(v, "shape") else v) for k, v in out.items()})


if __name__ == "__main__":
    main()
