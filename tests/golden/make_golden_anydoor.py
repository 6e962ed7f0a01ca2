#!/usr/bin/env python
"""Golden vectors for AnyDoor's pair preparation and crop-back, from the reference's own functions:
``process_pairs`` and ``crop_back`` (AnyEdit_Collection/adaptive_editing_pipelines/visual_reference_tool.py) and the helpers they
call from tools/tool.py (``sobel``, ``expand_image_mask``, ``get_bbox_from_mask``, ``expand_bbox``, ``box2squre``,
``pad_to_square``, ``box_in_box``).

Both modules import GroundingDINO and SAM at module level, so they cannot be imported: the functions are taken out of their
syntax trees with ``ast`` and executed with ``cv2`` and ``np`` in scope (nothing is copied into this repository).  Each case of
``oracle.anydoor_oracle.CASES`` is regenerated from its seed; ``process_pairs`` runs under ``np.random.seed(seed)``, and
``crop_back`` takes the seeded decoded image ``case_pred(seed)`` through the reference's clip-and-drop-a-row
(visual_reference_tool.py:221-227).  The arrays are large, so the fixture keeps, per case ``c``:
  ``c/in``        SHA-256 of the four input arrays' bytes (the seeded images and masks must not drift);
  ``c/ref`` ``c/jpg`` ``c/hint``  SHA-256 of the reference's fp32 arrays (C order);
  ``c/hf``        SHA-256 of the reference's ``sobel`` of the 224 x 224 reference image and mask;
  ``c/extra_sizes`` ``c/tar_box_yyxx_crop``  the integer geometry itself;
  ``c/crop_back`` SHA-256 of the uint8 image ``crop_back`` returns with OpenCV's own arithmetic (``cv2.setUseOptimized(False)``);
  ``c/crop_back_ipp``  how many bytes of that image, and by how much at most, the default build differs: its float32 resize goes
                  through Intel IPP, whose weights differ from OpenCV's by up to ~6e-3, so a truncated byte can differ by one;
plus ``cv2_version`` and ``cv2_cpu``, the OpenCV build the bytes came from.  ``process_pairs`` gives the same bytes with and
without the optimised paths (checked here).
Usage: python tests/golden/make_golden_anydoor.py"""
import ast
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..", "..")))

from oracle import anydoor_oracle as O  # noqa: E402
from oracle.ref_import import SRC_ROOT  # noqa: E402

PIPE = os.path.join(SRC_ROOT, "AnyEdit_Collection", "adaptive_editing_pipelines")
TOOL_FNS = ("sobel", "expand_image_mask", "get_bbox_from_mask", "expand_bbox", "box2squre", "pad_to_square", "box_in_box")


def sha(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return np.array(h.hexdigest())


def reference_functions():
    import cv2
    scope = {"cv2": cv2, "np": np}
    for path, names in ((os.path.join(PIPE, "tools", "tool.py"), TOOL_FNS),
                        (os.path.join(PIPE, "visual_reference_tool.py"), ("process_pairs", "crop_back"))):
        tree = ast.parse(open(path).read(), path)
        fns = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in names]
        assert sorted(f.name for f in fns) == sorted(names), f"{path}: expected {names}"
        exec(compile(ast.Module(body=fns, type_ignores=[]), path, "exec"), scope)
    return scope


def main():
    import cv2
    ref = reference_functions()
    out = {"cv2_version": np.array(cv2.__version__), "cv2_cpu": np.array(cv2.getCPUFeaturesLine())}
    for name in O.CASES:
        ri, rm, ti, tm, seed = O.case_inputs(name)
        out[f"{name}/in"] = sha(ri, rm, ti, tm)
        items = []
        for optimized in (True, False):
            cv2.setUseOptimized(optimized)
            np.random.seed(seed)
            items.append(ref["process_pairs"](ri, rm, ti.copy(), tm))
        cv2.setUseOptimized(True)
        item = items[0]
        assert all(np.array_equal(items[0][k], items[1][k]) for k in item)
        assert item["ref"].dtype == np.float64 and item["jpg"].dtype == item["hint"].dtype == np.float32
        for k in ("ref", "jpg", "hint"):                       # ref as the model gets it: .float() of the float64 array
            out[f"{name}/{k}"] = sha(item[k].astype(np.float32))
        u8 = np.rint(item["ref"] * 255).astype(np.uint8)                         # ref is x / 255 of a uint8 image
        assert np.array_equal(u8 / 255, item["ref"])
        st = {}
        np.random.seed(seed)
        O.process_pairs(ri, rm, ti, tm, stages=st)
        assert np.array_equal(st["ref_u8"], u8)
        out[f"{name}/hf"] = sha(ref["sobel"](u8, st["ref_mask_u8"] / 255))
        out[f"{name}/extra_sizes"] = np.asarray(item["extra_sizes"], dtype=np.int64)
        out[f"{name}/tar_box_yyxx_crop"] = np.asarray(item["tar_box_yyxx_crop"], dtype=np.int64)
        pred = O.decode_to_pred(O.case_pred(seed))
        ipp = ref["crop_back"](pred, ti.copy(), item["extra_sizes"], item["tar_box_yyxx_crop"])
        cv2.setUseOptimized(False)
        back = ref["crop_back"](pred, ti.copy(), item["extra_sizes"], item["tar_box_yyxx_crop"])
        cv2.setUseOptimized(True)
        out[f"{name}/crop_back"] = sha(back)
        d = np.abs(ipp.astype(np.int64) - back)
        out[f"{name}/crop_back_ipp"] = np.array([int((d > 0).sum()), int(d.max())])
        print(f"{name}: extra_sizes {item['extra_sizes'].tolist()}, crop {item['tar_box_yyxx_crop'].tolist()}, "
              f"crop_back bytes differing under IPP: {out[f'{name}/crop_back_ipp'].tolist()}")
    np.savez_compressed(os.path.join(HERE, "anydoor_golden.npz"), **out)


if __name__ == "__main__":
    main()
