"""The HED scribble annotator without a GPU: the fp32 oracle (oracle/hed_oracle.py) against the reference module's golden
(tests/golden/make_golden_hed.py), the reference's parameter tree with a strict load, the refusals and the absence of a CPU
fallback."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import hed_oracle as O, weights

G = os.path.join(os.path.dirname(__file__), "golden")


def rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).norm() / b.norm())


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(G, "hed_golden.npz")), json.load(open(os.path.join(G, "hed_keys.json")))


def test_oracle_matches_reference(gold):
    g, meta = gold
    sd = O.seeded_state_dict(meta["seeds"][0])
    assert weights.checksum(sd) == pytest.approx(float(g["wsum"]), rel=1e-12)
    for i, (H, W) in enumerate(meta["sizes"]):
        s = f"{H}x{W}"
        img = O.images((H, W), meta["seeds"][1] + i)
        assert np.array_equal(img[0], g[f"img{s}"]), f"{s}: the seeded image changed"
        sides = O.side_maps(sd, img)
        for k, e in enumerate(sides):
            err = rel(e[0, 0], g[f"side{s}_{k}"])
            assert tuple(e.shape[2:]) == g[f"side{s}_{k}"].shape and err <= 2e-6, (s, k, err)
        edge = O.edge_map(sides, H, W)[0]
        print(f"[hed oracle] {s}: side maps within 2e-6 of the reference, edge map identical: {np.array_equal(edge, g[f'edge{s}'])}, "
              f"{len(np.unique(edge))} distinct values")
        assert np.array_equal(edge, g[f"edge{s}"])
    assert g["side17x200_4"].shape[0] == 1, "the golden should have a one-pixel-tall block 5"


def test_parameter_tree_matches_reference(gold):
    from anyedit_b200.hed import ControlNetHED_Apache2
    _, meta = gold
    m = ControlNetHED_Apache2()
    got = {k: list(v.shape) for k, v in m.state_dict().items()}
    assert got == meta["keys"] and len(got) == 37
    assert got == {k: list(v) for k, v in O.param_shapes().items()}
    assert sum(p.numel() for p in m.parameters()) == 14716168
    m.load_state_dict(O.seeded_state_dict(meta["seeds"][0]), strict=True)


def test_refusals_and_no_cpu_fallback():
    from anyedit_b200.hed import ControlNetHED_Apache2
    m = ControlNetHED_Apache2()
    for bad in (torch.zeros(1, 32, 32, 3, dtype=torch.float32), torch.zeros(1, 32, 32, 4, dtype=torch.uint8),
                torch.zeros(32, 32, 3, dtype=torch.uint8), torch.zeros(1, 15, 64, 3, dtype=torch.uint8),
                torch.zeros(1, 64, 15, 3, dtype=torch.uint8)):
        with pytest.raises(ValueError):
            m(bad)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros(1, 16, 16, 3, dtype=torch.uint8))
    with pytest.raises(RuntimeError, match="CUDA"):
        m.edge_map(torch.zeros(1, 16, 16, 3, dtype=torch.uint8))
