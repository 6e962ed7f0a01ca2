"""AnyDoor's reference-image encoder without a GPU: the fp32 oracle (oracle/dinov2_oracle.py) against transformers' own
``Dinov2Model`` golden (tests/golden/make_golden_dinov2.py), the transformers -> hub key map, both position-table
interpolation forms, the ``ldm`` alias path, and the absence of a CPU fallback."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import dinov2_oracle as O, weights

G = os.path.join(os.path.dirname(__file__), "golden")


def rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).norm() / b.norm())


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(G, "dinov2_tiny.npz")), json.load(open(os.path.join(G, "dinov2_tiny_keys.json")))


def tiny_hub_state_dict(meta):
    """The golden's weights under the names FrozenDinoV2Encoder loads (``model.*`` hub names + ``projector.*``)."""
    from anyedit_b200.encoders import dinov2_from_transformers
    seed, pseed, _ = meta["seeds"]
    hf = O.seeded_state_dict({k: tuple(v) for k, v in meta["keys"].items()}, seed)
    proj = weights.make_state_dict({k: tuple(v) for k, v in meta["projector_keys"].items()}, pseed)
    return {**{"model." + k: v for k, v in dinov2_from_transformers(hf).items()}, **proj}, weights.checksum({**hf, **proj})


def test_oracle_matches_transformers(gold):
    g, meta = gold
    sd, wsum = tiny_hub_state_dict(meta)
    assert wsum == pytest.approx(float(g["wsum"]), rel=1e-12)
    for i, (H, W) in enumerate(O.TINY_SIZES):
        got = O.encoder(sd, O.tiny_images((H, W), meta["seeds"][2] + i), O.TINY["num_attention_heads"], offset=0.0)
        e = rel(got, g[f"out_{H}x{W}"])
        print(f"[dinov2 oracle {H}x{W}] rel-L2 vs transformers {e:.2e}")
        assert e <= 2e-6, (H, W, e)


def test_key_map_round_trip(gold):
    from anyedit_b200.encoders import FrozenDinoV2Encoder, dinov2_from_transformers, dinov2_to_transformers
    _, meta = gold
    hf = O.seeded_state_dict({k: tuple(v) for k, v in meta["keys"].items()}, 5)
    hub = dinov2_from_transformers(hf)
    back = dinov2_to_transformers(hub)
    assert back.keys() == hf.keys() and all(torch.equal(back[k], hf[k]) for k in hf)
    enc = FrozenDinoV2Encoder(config=dict(meta["config"], projection_dim=meta["projection_dim"]))
    want = {"model." + k: tuple(v.shape) for k, v in hub.items()}
    want.update({k: tuple(v) for k, v in meta["projector_keys"].items()})
    assert {k: tuple(v.shape) for k, v in enc.state_dict().items()} == want
    assert "blocks.0.attn.qkv.weight" in hub and hub["blocks.0.attn.qkv.weight"].shape[0] == 3 * O.TINY["hidden_size"]
    with pytest.raises(KeyError):
        dinov2_from_transformers({"pooler.dense.weight": torch.zeros(1)})


def test_position_table_forms(gold):
    from anyedit_b200.encoders import dinov2_pos_table
    g, _ = gold
    pos = weights.fill_tensor("pos", (1, 82, 192), 3)
    for (H, W) in O.TINY_SIZES:
        gh, gw = H // 14, W // 14
        grid = pos[0, 1:].reshape(1, 9, 9, 192).permute(0, 3, 1, 2)
        want = F.interpolate(grid, scale_factor=((gh + 0.1) / 9, (gw + 0.1) / 9), mode="bicubic").permute(0, 2, 3, 1).reshape(-1, 192)
        t = dinov2_pos_table(pos, gh, gw)
        assert torch.equal(t[0], pos[0, 0]) and torch.equal(t[1:], want)
        assert torch.equal(t, O.pos_table(pos, gh, gw, 0.1))
    _, meta = gold
    sd, _ = tiny_hub_state_dict(meta)
    for (H, W) in O.TINY_SIZES:
        gh, gw = H // 14, W // 14
        t = dinov2_pos_table(sd["model.pos_embed"], gh, gw, interpolate_offset=0.0)
        assert torch.equal(t, torch.from_numpy(g[f"pos_{gh}x{gw}"])), (gh, gw)
    assert torch.equal(dinov2_pos_table(pos, 9, 9), pos[0])          # the trained grid is used as it is


def test_alias_and_instantiate_from_config(gold):
    from anyedit_b200.encoders import FrozenCLIPEmbedder, FrozenDinoV2Encoder
    from anyedit_b200.ldm.modules.encoders import modules
    from anyedit_b200.ldm.util import instantiate_from_config
    assert modules.FrozenDinoV2Encoder is FrozenDinoV2Encoder and modules.FrozenCLIPEmbedder is FrozenCLIPEmbedder
    _, meta = gold
    enc = instantiate_from_config({"target": "anyedit_b200.ldm.modules.encoders.modules.FrozenDinoV2Encoder",
                                   "params": {"config": meta["config"]}})
    assert isinstance(enc, FrozenDinoV2Encoder)
    assert not any(p.requires_grad for p in enc.model.parameters())
    assert tuple(enc.projector.weight.shape) == (1024, O.TINY["hidden_size"])


def test_no_cpu_fallback(gold):
    from anyedit_b200.encoders import FrozenDinoV2Encoder
    _, meta = gold
    enc = FrozenDinoV2Encoder(config=meta["config"])
    with pytest.raises(RuntimeError, match="CUDA"):
        enc(torch.rand(1, 3, 112, 112))
