#!/usr/bin/env python
"""Golden vectors for AnyEdit's segmentation annotator (AnyEdit_Collection/other_modules/uniformer: the UniFormer backbone, UPerHead,
FCNHead, mmcv's imrescale / imnormalize and mmseg's resize), from the reference modules themselves (imported from the reference
tree, never copied).

The vendored mmseg stack imports timm, addict, yapf and matplotlib, none of which the annotator's forward uses: ``uniformer`` is
registered as a namespace package (its ``__init__`` would import matplotlib), ``timm.models.layers`` is stubbed with the three
names uniformer.py imports (DropPath is never built at drop_path_rate 0), and the other three are mocked.

Seeded tiny configuration (oracle.segment_oracle): embed_dim [64, 128, 192, 256], layers [1, 1, 2, 1], head_dim 64, UPerHead with
channels 128 and 150 classes, every BatchNorm with random statistics.  Written to segment_tiny.npz:
  out{i}              the four backbone outputs for the first of two seeded 68 x 100 BGR images (imnormalize'd), run
                      as one batch
  logits              UPerHead logits at 1/4 resolution (17 x 25) for the first image of that batch
  infer_*             inference_segmentor's path on a seeded 60 x 90 image: imrescale to 512 x 768 (shape and sha256 of the uint8
                      image, sha256 of the imnormalize'd fp32 input), labels [60, 90] and the fp32 top-two margin of the final
                      logits per pixel
and to segment_keys.json: the seeds, the tiny key shapes, and the key / shape pairs of the real configuration (UniFormer-S,
UPerHead, FCNHead auxiliary head) with mmseg's prefixes.
Usage: python tests/golden/make_golden_segment.py"""
import hashlib
import json
import os
import sys
import types
from unittest import mock

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..", "..")))

from oracle import segment_oracle as O, weights  # noqa: E402
from oracle.ref_import import SRC_ROOT  # noqa: E402

SEED, IMG_SEED, RAW_SEED = 81, 82, 83


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def import_reference():
    class DropPath(nn.Identity):
        def __init__(self, *a, **k):
            super().__init__()

    def stub(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m

    stub("timm")
    stub("timm.models")
    stub("timm.models.layers", DropPath=DropPath, to_2tuple=lambda x: x if isinstance(x, tuple) else (x, x),
         trunc_normal_=lambda t, std=1.0, **k: nn.init.trunc_normal_(t, std=std))
    for n in ("addict", "yapf", "yapf.yapflib", "yapf.yapflib.yapf_api", "matplotlib", "matplotlib.pyplot"):
        sys.modules[n] = mock.MagicMock()
    pkg = types.ModuleType("uniformer")
    pkg.__path__ = [os.path.join(SRC_ROOT, "AnyEdit_Collection", "other_modules", "uniformer")]
    sys.modules["uniformer"] = pkg
    from uniformer.mmseg.models.backbones.uniformer import UniFormer
    from uniformer.mmseg.models.decode_heads.uper_head import UPerHead
    from uniformer.mmseg.models.decode_heads.fcn_head import FCNHead
    from uniformer.mmcv.image import imnormalize, imrescale
    from uniformer.mmseg.ops import resize
    return UniFormer, UPerHead, FCNHead, imrescale, imnormalize, resize


def build(UniFormer, UPerHead, FCNHead, bb, hd):
    norm_cfg = dict(type="BN", requires_grad=True)
    loss = dict(type="CrossEntropyLoss", use_sigmoid=False, loss_weight=1.0)
    m = nn.Module()
    m.backbone = UniFormer(embed_dim=bb["embed_dim"], layers=bb["layers"], head_dim=64, mlp_ratio=4.0, qkv_bias=True,
                           drop_path_rate=0.0, windows=False, hybrid=False)
    m.decode_head = UPerHead(in_channels=bb["embed_dim"], in_index=[0, 1, 2, 3], pool_scales=(1, 2, 3, 6), channels=hd["channels"],
                             dropout_ratio=0.1, num_classes=hd["num_classes"], norm_cfg=norm_cfg, align_corners=False, loss_decode=loss)
    m.auxiliary_head = FCNHead(in_channels=bb["embed_dim"][2], in_index=2, channels=hd["channels"] // 2, num_convs=1, concat_input=False,
                               dropout_ratio=0.1, num_classes=hd["num_classes"], norm_cfg=norm_cfg, align_corners=False, loss_decode=loss)
    return m.eval()


def main():
    UniFormer, UPerHead, FCNHead, imrescale, imnormalize, resize = import_reference()
    torch.set_grad_enabled(False)
    real = {k: list(v.shape) for k, v in build(UniFormer, UPerHead, FCNHead, O.REAL_BACKBONE, O.REAL_HEAD).state_dict().items()}
    m = build(UniFormer, UPerHead, FCNHead, O.TINY_BACKBONE, O.TINY_HEAD)
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    sd = O.seeded_state_dict(shapes, SEED)
    m.load_state_dict(sd, strict=True)
    mean, std = np.array(O.MEAN), np.array(O.STD)

    def prep(img):
        return torch.from_numpy(np.ascontiguousarray(imnormalize(img, mean, std, to_rgb=True).transpose(2, 0, 1)))[None]

    out = {"wsum": weights.checksum({k: v for k, v in sd.items() if v.is_floating_point()})}
    raw = O.tiny_raw_images(O.TINY_SIZE, IMG_SEED)
    x = torch.cat([prep(r) for r in raw])
    feats = m.backbone(x)
    for i, f in enumerate(feats):
        out[f"out{i}"] = f[:1].numpy()
    out["logits"] = m.decode_head(feats)[:1].numpy()

    img = O.tiny_raw_images(O.TINY_RAW, RAW_SEED, B=1)[0]
    rescaled = imrescale(img, O.IMG_SCALE)
    xi = prep(rescaled)
    out["infer_shape"] = np.array(rescaled.shape)
    out["infer_img_sha256"] = sha(rescaled)
    out["infer_x_sha256"] = sha(xi.numpy())
    seg = resize(m.decode_head(m.backbone(xi)), size=xi.shape[2:], mode="bilinear", align_corners=False)
    seg = resize(seg, size=img.shape[:2], mode="bilinear", align_corners=False)[0]
    out["infer_labels"] = torch.softmax(seg, 0).argmax(0).numpy()
    out["infer_margin"] = O.top2_margin(seg).numpy()
    with open(os.path.join(HERE, "segment_keys.json"), "w") as fh:
        json.dump({"seeds": [SEED, IMG_SEED, RAW_SEED], "keys": {k: list(v) for k, v in shapes.items()}, "real_keys": real}, fh)
    np.savez(os.path.join(HERE, "segment_tiny.npz"), **out)
    print({k: (v.shape if hasattr(v, "shape") else v) for k, v in out.items()}, len(real),
          sum(int(np.prod(s)) for k, s in real.items() if k.startswith("backbone.")),
          sum(int(np.prod(s)) for k, s in real.items() if k.startswith("decode_head.")))


if __name__ == "__main__":
    main()
