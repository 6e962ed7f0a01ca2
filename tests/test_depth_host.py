"""Depth Anything V2 without a GPU: the fp32 oracle (oracle/depth_oracle.py) against the reference modules' golden
(tests/golden/make_golden_depth.py), the hub position-table resize bit for bit, the vitl parameter tree, ``image2tensor``,
the refusals and the absence of a CPU fallback."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from oracle import depth_oracle as O, dinov2_oracle, weights

G = os.path.join(os.path.dirname(__file__), "golden")


def rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).norm() / b.norm())


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(G, "depth_anything_tiny.npz")), json.load(open(os.path.join(G, "depth_anything_tiny_keys.json")))


def tiny_state_dict(meta):
    return O.seeded_state_dict({k: tuple(v) for k, v in meta["keys"].items()}, meta["seeds"][0])


def test_oracle_matches_reference(gold):
    g, meta = gold
    sd = tiny_state_dict(meta)
    assert weights.checksum(sd) == pytest.approx(float(g["wsum"]), rel=1e-12)
    for i, size in enumerate(O.TINY_SIZES):
        got = O.depth(sd, O.tiny_images(size, meta["seeds"][1] + i), O.TINY_LAYERS, O.TINY_HEADS)
        want = g["depth_%dx%d" % size]
        e = rel(got, want)
        print(f"[depth oracle {size}] rel-L2 vs reference {e:.2e}, positive {float((got > 0).float().mean()):.3f}")
        assert tuple(got.shape) == want.shape and e <= 2e-6
        assert (want > 0).mean() > 0.5, "the golden's depth maps should be mostly positive"
    hub = {k[len("pretrained."):]: v for k, v in sd.items() if k.startswith("pretrained.")}
    x = O.tiny_images(O.TINY_SIZES[0], meta["seeds"][1])[:1]
    for i, (t, c) in enumerate(O.intermediate_layers(hub, x, O.TINY_LAYERS, O.TINY_HEADS)):
        assert rel(t, g[f"tok{i}"]) <= 2e-6 and rel(c, g[f"cls{i}"]) <= 2e-6, i


def test_oracle_swiglu_backbone_matches_hub(gold):
    """The SwiGLU ViT restated by oracle/dinov2_oracle.py (which the FrozenDinoV2Encoder tests use) against the hub class."""
    g, meta = gold
    sd = dinov2_oracle.seeded_state_dict({k: tuple(v) for k, v in meta["swiglu_keys"].items()}, meta["seeds"][2])
    assert weights.checksum(sd) == pytest.approx(float(g["swiglu_wsum"]), rel=1e-12)
    x = O.tiny_images(O.TINY_SIZES[1], meta["seeds"][2], B=1)
    e = rel(dinov2_oracle.forward_features(sd, x, O.TINY_HEADS, offset=0.1), g["swiglu_x_norm"])
    print(f"[dinov2 SwiGLU oracle] rel-L2 vs hub {e:.2e}")
    assert e <= 2e-6
    assert rel(O.forward_features(sd, x, O.TINY_HEADS), g["swiglu_x_norm"]) <= 2e-6


def test_pos_table_bit_exact_vs_hub(gold):
    from anyedit_b200.encoders import dinov2_pos_table
    g, meta = gold
    pos = tiny_state_dict(meta)["pretrained.pos_embed"]
    for gh, gw in O.POS_GRIDS:
        assert torch.equal(dinov2_pos_table(pos, gh, gw, 0.1), torch.from_numpy(g[f"pos_{gh}x{gw}"])), (gh, gw)
    gh, gw = O.POS_GRID_HASHED
    t = dinov2_pos_table(pos, gh, gw, 0.1)
    assert hashlib.sha256(t.numpy().tobytes()).hexdigest() == str(g[f"pos_{gh}x{gw}_sha256"])


def test_vitl_parameter_tree(gold):
    from anyedit_b200.depth import DepthAnythingV2
    _, meta = gold
    with torch.device("meta"):
        m = DepthAnythingV2(encoder="vitl", features=256, out_channels=[256, 512, 1024, 1024])
    got = {k: list(v.shape) for k, v in m.state_dict().items()}
    assert len(meta["vitl_keys"]) == 407 and got == meta["vitl_keys"]
    with torch.device("meta"):
        t = DepthAnythingV2(encoder="vits", **O.TINY_HEAD, config=O.TINY_BACKBONE, layer_idx=O.TINY_LAYERS)
    assert {k: list(v.shape) for k, v in t.state_dict().items()} == meta["keys"]


def test_named_backbones():
    from anyedit_b200.encoders import DINOV2_CONFIGS, Dinov2Model
    want = {"vits": (384, 6, 12, "fc1"), "vitb": (768, 12, 12, "fc1"), "vitl": (1024, 16, 24, "fc1"), "vitg": (1536, 24, 40, "w12")}
    for name, (D, heads, layers, mlp) in want.items():
        with torch.device("meta"):
            m = Dinov2Model(DINOV2_CONFIGS[name])
        c = m.config
        assert (c.hidden_size, c.num_attention_heads, len(m.blocks), c.image_size, c.patch_size) == (D, heads, layers, 518, 14)
        assert hasattr(m.blocks[0].mlp, mlp) and tuple(m.pos_embed.shape) == (1, 37 * 37 + 1, D)
    with torch.device("meta"):
        assert tuple(Dinov2Model(DINOV2_CONFIGS["vitl"]).blocks[0].mlp.fc1.weight.shape) == (4096, 1024)


def test_image2tensor(gold):
    """dpt.py:202-221 on the host: the reference's tensor bit for bit on the golden image; aspect-keeping lower-bound sizes."""
    pytest.importorskip("cv2")
    from anyedit_b200.depth import DepthAnythingV2, _lower_bound_size
    g, meta = gold
    m = DepthAnythingV2(encoder="vits", **O.TINY_HEAD, config=O.TINY_BACKBONE, layer_idx=O.TINY_LAYERS)
    x, hw = m.image2tensor(O.raw_image(meta["seeds"][3]), 126)
    assert hw == (60, 90) and x.dtype == torch.float32 and tuple(x.shape) == tuple(g["infer_i2t_shape"]) == (1, 3, 126, 196)
    assert hashlib.sha256(x.numpy().tobytes()).hexdigest() == str(g["infer_i2t_sha256"])
    # (w, h) -> (w', h'): both sides >= 518, multiples of 14, aspect kept up to the rounding
    assert _lower_bound_size(640, 480, 518, 14) == (686, 518)
    assert _lower_bound_size(480, 640, 518, 14) == (518, 686)
    assert _lower_bound_size(518, 518, 518, 14) == (518, 518)
    assert _lower_bound_size(1000, 1000, 518, 14) == (518, 518)


def test_refusals():
    from anyedit_b200.depth import DepthAnythingV2
    with pytest.raises(NotImplementedError):
        DepthAnythingV2(encoder="vits", use_bn=True)
    with pytest.raises(NotImplementedError):
        DepthAnythingV2(encoder="vits", use_clstoken=True)
    with pytest.raises(ValueError):
        DepthAnythingV2(encoder="vith")


def test_no_cpu_fallback():
    from anyedit_b200.depth import DepthAnythingV2
    m = DepthAnythingV2(encoder="vits", **O.TINY_HEAD, config=O.TINY_BACKBONE, layer_idx=O.TINY_LAYERS)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.rand(1, 3, 126, 126))
