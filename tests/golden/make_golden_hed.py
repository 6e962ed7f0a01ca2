#!/usr/bin/env python
"""Golden vectors for AnyEdit's HED scribble annotator (AnyEdit_Collection/other_modules/HED/__init__.py), from the reference module
itself (imported from the reference tree, never copied; it needs only cv2, einops and torch).

The reference's own ``HEDdetector.__call__`` runs on the CPU: ``nn.Module.cuda`` and ``Tensor.cuda`` are patched to no-ops, the
seeded state dict is written to a temporary file for its ``torch.load``, and each image goes in and comes out as a PNG in a temporary
directory.  Weights (oracle.hed_oracle.seeded_state_dict) are at the real width; images (oracle.hed_oracle.images) are seeded and
structured, at 48 x 64 (even at every pool), 61 x 93 (odd sides, floored by the pools) and 17 x 200 (block 5 is one pixel tall).  Written to
hed_golden.npz: per size s, ``img{s}`` (uint8 HWC), ``side{s}_{k}`` (the five fp32 side maps [h, w]) and ``edge{s}`` (the uint8
map); ``wsum``, the weights' checksum.  And to hed_keys.json: the seeds, the sizes and the reference's key / shape pairs.
Usage: python tests/golden/make_golden_hed.py"""
import importlib.util
import json
import os
import sys
import tempfile
from unittest import mock

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..", "..")))

from oracle import hed_oracle as O, weights  # noqa: E402
from oracle.ref_import import SRC_ROOT  # noqa: E402

SEED, IMG_SEED = 101, 102


def import_reference():
    path = os.path.join(SRC_ROOT, "AnyEdit_Collection", "other_modules", "HED", "__init__.py")
    spec = importlib.util.spec_from_file_location("reference_hed", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    import cv2
    ref = import_reference()
    torch.set_grad_enabled(False)
    sd = O.seeded_state_dict(SEED)
    keys = {k: list(v.shape) for k, v in ref.ControlNetHED_Apache2().state_dict().items()}
    out = {"wsum": weights.checksum(sd)}
    with tempfile.TemporaryDirectory() as tmp, mock.patch.object(torch.nn.Module, "cuda", lambda self, *a, **k: self), \
            mock.patch.object(torch.Tensor, "cuda", lambda self, *a, **k: self):
        wpath = os.path.join(tmp, "ControlNetHED.pth")
        torch.save(sd, wpath)
        det = ref.HEDdetector(wpath)
        for i, size in enumerate(O.GOLDEN_SIZES):
            s = f"{size[0]}x{size[1]}"
            img = O.images(size, IMG_SEED + i)[0]
            src, dst = os.path.join(tmp, f"in{s}.png"), os.path.join(tmp, f"out{s}.png")
            assert cv2.imwrite(src, img)
            det(src, dst)
            edge = cv2.imread(dst, cv2.IMREAD_UNCHANGED)
            assert edge.shape == size and edge.dtype == np.uint8
            assert len(np.unique(edge)) >= 40, f"{s}: the edge map is nearly constant ({len(np.unique(edge))} values)"
            x = torch.from_numpy(img.copy()).float().permute(2, 0, 1)[None]
            for k, e in enumerate(det.netNetwork(x)):
                out[f"side{s}_{k}"] = e[0, 0].numpy()
            out[f"img{s}"], out[f"edge{s}"] = img, edge
    with open(os.path.join(HERE, "hed_keys.json"), "w") as fh:
        json.dump({"seeds": [SEED, IMG_SEED], "sizes": [list(s) for s in O.GOLDEN_SIZES], "keys": keys}, fh)
    np.savez_compressed(os.path.join(HERE, "hed_golden.npz"), **out)
    print({k: (v.shape if hasattr(v, "shape") else v) for k, v in out.items()}, len(keys), sum(int(np.prod(s)) for s in keys.values()))


if __name__ == "__main__":
    main()
