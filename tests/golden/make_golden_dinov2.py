#!/usr/bin/env python
"""Golden vectors for AnyDoor's reference-image encoder (``FrozenDinoV2Encoder``, ldm/modules/encoders/modules.py:279-315).

The encoder's DINOv2 ViT comes from the DINOv2 hub, which is not in the reference tree; transformers' ``Dinov2Model`` with
``use_swiglu_ffn=True`` computes the same blocks (this image has the version printed below).  On the seeded tiny configuration
``oracle.dinov2_oracle.TINY`` (hidden 192, 3 heads of 64, 3 layers, 9 x 9 position grid, LayerScale away from 1.0) it produces:
ImageNet-normalised images of two sizes (81 and 145 tokens) -> last_hidden_state -> a seeded Linear(192, 64) projector; and
the position tables transformers interpolates for both grids (its ``size=(gh, gw)`` form = offset 0.0 here).
Weights and images are regenerated from seeds by the tests (oracle.dinov2_oracle.seeded_state_dict / tiny_images).
Usage: python tests/golden/make_golden_dinov2.py"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..", "..")))

from oracle import dinov2_oracle as O, weights  # noqa: E402

SEED, PROJ_SEED, IMG_SEED = 91, 92, 93


def main():
    import transformers
    from transformers import Dinov2Config, Dinov2Model
    torch.set_grad_enabled(False)
    m = Dinov2Model(Dinov2Config(**O.TINY)).eval()
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    sd = O.seeded_state_dict(shapes, SEED)
    m.load_state_dict(sd, strict=True)
    pshapes = {"projector.weight": (O.TINY_PROJ, O.TINY["hidden_size"]), "projector.bias": (O.TINY_PROJ,)}
    psd = weights.make_state_dict(pshapes, PROJ_SEED)
    mean, std = torch.tensor(O.MEAN).view(1, 3, 1, 1), torch.tensor(O.STD).view(1, 3, 1, 1)
    out = {"transformers": transformers.__version__, "wsum": weights.checksum({**sd, **psd})}
    for i, (H, W) in enumerate(O.TINY_SIZES):
        x = O.tiny_images((H, W), IMG_SEED + i)
        h = m(pixel_values=(x - mean) / std).last_hidden_state
        out[f"out_{H}x{W}"] = torch.nn.functional.linear(h, psd["projector.weight"], psd["projector.bias"]).numpy()
        gh, gw = H // O.TINY["patch_size"], W // O.TINY["patch_size"]
        emb = torch.zeros(1, gh * gw + 1, O.TINY["hidden_size"])
        out[f"pos_{gh}x{gw}"] = m.embeddings.interpolate_pos_encoding(emb, H, W)[0].numpy()
    with open(os.path.join(HERE, "dinov2_tiny_keys.json"), "w") as f:
        json.dump({"config": O.TINY, "projection_dim": O.TINY_PROJ, "seeds": [SEED, PROJ_SEED, IMG_SEED],
                   "keys": {k: list(v) for k, v in shapes.items()}, "projector_keys": {k: list(v) for k, v in pshapes.items()}}, f)
    np.savez(os.path.join(HERE, "dinov2_tiny.npz"), **out)
    print({k: (v.shape if hasattr(v, "shape") else v) for k, v in out.items()})


if __name__ == "__main__":
    main()
