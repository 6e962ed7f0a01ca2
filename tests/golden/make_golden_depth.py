#!/usr/bin/env python
"""Golden vectors for Depth Anything V2 (AnyEdit_Collection/other_modules/depth_anything_v2: dpt.py, dinov2.py, util/blocks.py),
from the reference modules themselves (imported from the reference tree, never copied).

Seeded tiny configuration (oracle.depth_oracle): a hub ``DinoVisionTransformer`` with D 192 (3 heads of 64), 4 GELU-MLP blocks
read at [0, 1, 2, 3], a 9 x 9 position table (img_size 126), LayerScale, offset 0.1; ``DPTHead(192, features=128,
out_channels=[64, 128, 256, 256])``; the last head conv's bias set to 0.5.  Written to depth_anything_tiny.npz:
  depth_{H}x{W}       DepthAnythingV2.forward for B = 2 seeded normalised images, 126 x 126 (the table's own grid) and 98 x 182
                      (7 x 13 patches: the position table is interpolated)
  tok{i} / cls{i}     get_intermediate_layers(x, [0, 1, 2, 3], return_class_token=True) for the first 126 x 126 image
  pos_{gh}x{gw}       interpolate_pos_encoding of the tiny table; the 37 x 56 grid as the sha256 of its fp32 bytes
  infer_*             infer_image(raw, input_size=126) on a seeded 60 x 90 BGR uint8 image (+ image2tensor's shape and hash)
  swiglu_*            forward_features of a tiny ffn_layer="swiglufused" hub ViT (2 blocks) on a 98 x 182 image: the backbone of
                      encoders.FrozenDinoV2Encoder pinned against the hub class
and to depth_anything_tiny_keys.json: the tiny key shapes, the seeds, and the 407 key / shape pairs of DepthAnythingV2('vitl').
Usage: python tests/golden/make_golden_depth.py"""
import hashlib
import json
import os
import sys
from functools import partial

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..", "..")))

from oracle import dinov2_oracle, depth_oracle as O, weights  # noqa: E402
from oracle.ref_import import SRC_ROOT  # noqa: E402

SEED, IMG_SEED, SWIGLU_SEED, RAW_SEED = 71, 72, 73, 74


def sha(t):
    return hashlib.sha256(np.ascontiguousarray(t.detach().float().numpy()).tobytes()).hexdigest()


def main():
    sys.path.insert(0, os.path.join(SRC_ROOT, "AnyEdit_Collection", "other_modules"))
    from depth_anything_v2.dinov2 import DinoVisionTransformer
    from depth_anything_v2.dinov2_layers import MemEffAttention, NestedTensorBlock as Block
    from depth_anything_v2.dpt import DepthAnythingV2, DPTHead
    torch.set_grad_enabled(False)

    def backbone(c):
        return DinoVisionTransformer(img_size=c["image_size"], patch_size=14, embed_dim=c["hidden_size"], depth=c["num_hidden_layers"],
                                     num_heads=c["num_attention_heads"], mlp_ratio=4, block_fn=partial(Block, attn_class=MemEffAttention),
                                     init_values=1.0, ffn_layer="swiglufused" if c["use_swiglu_ffn"] else "mlp", block_chunks=0,
                                     num_register_tokens=0, interpolate_antialias=False, interpolate_offset=0.1).eval()

    vitl = {k: list(v.shape) for k, v in DepthAnythingV2(encoder="vitl").state_dict().items()}
    m = DepthAnythingV2(encoder="vits", **O.TINY_HEAD)
    m.pretrained = backbone(O.TINY_BACKBONE)
    m.depth_head = DPTHead(O.TINY_BACKBONE["hidden_size"], O.TINY_HEAD["features"], False, out_channels=O.TINY_HEAD["out_channels"])
    m.intermediate_layer_idx["vits"] = O.TINY_LAYERS
    m.eval()
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    sd = O.seeded_state_dict(shapes, SEED)
    m.load_state_dict(sd, strict=True)
    out = {"wsum": weights.checksum(sd)}
    for i, size in enumerate(O.TINY_SIZES):
        x = O.tiny_images(size, IMG_SEED + i)
        out["depth_%dx%d" % size] = m(x).numpy()
    x = O.tiny_images(O.TINY_SIZES[0], IMG_SEED)[:1]
    for i, (t, c) in enumerate(m.pretrained.get_intermediate_layers(x, O.TINY_LAYERS, return_class_token=True)):
        out[f"tok{i}"], out[f"cls{i}"] = t.numpy(), c.numpy()
    D = O.TINY_BACKBONE["hidden_size"]
    for gh, gw in O.POS_GRIDS + (O.POS_GRID_HASHED,):
        t = m.pretrained.interpolate_pos_encoding(torch.zeros(1, gh * gw + 1, D), gh * 14, gw * 14)[0]
        if (gh, gw) == O.POS_GRID_HASHED:
            out[f"pos_{gh}x{gw}_sha256"] = sha(t)
        else:
            out[f"pos_{gh}x{gw}"] = t.numpy()
    raw = O.raw_image(RAW_SEED)
    img, hw = m.image2tensor(raw, 126)
    out["infer_i2t_shape"], out["infer_i2t_sha256"] = np.array(img.shape), sha(img)
    out["infer_depth"] = m.infer_image(raw, 126)
    sw = backbone(O.TINY_SWIGLU)
    ssd = dinov2_oracle.seeded_state_dict({k: tuple(v.shape) for k, v in sw.state_dict().items()}, SWIGLU_SEED)
    sw.load_state_dict(ssd, strict=True)
    f = sw.forward_features(O.tiny_images(O.TINY_SIZES[1], SWIGLU_SEED, B=1))
    out["swiglu_wsum"] = weights.checksum(ssd)
    out["swiglu_x_norm"] = torch.cat([f["x_norm_clstoken"][:, None], f["x_norm_patchtokens"]], 1).numpy()
    with open(os.path.join(HERE, "depth_anything_tiny_keys.json"), "w") as fh:
        json.dump({"seeds": [SEED, IMG_SEED, SWIGLU_SEED, RAW_SEED], "keys": {k: list(v) for k, v in shapes.items()},
                   "swiglu_keys": {k: list(v.shape) for k, v in sw.state_dict().items()}, "vitl_keys": vitl}, fh)
    np.savez(os.path.join(HERE, "depth_anything_tiny.npz"), **out)
    print({k: (v.shape if hasattr(v, "shape") else v) for k, v in out.items()}, len(vitl))


if __name__ == "__main__":
    main()
