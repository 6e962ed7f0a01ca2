"""The segmentation annotator without a GPU: the fp32 oracle (oracle/segment_oracle.py) against the reference modules' golden
(tests/golden/make_golden_segment.py), the mmseg parameter tree, the host preprocessing, the refusals and the absence of a CPU
fallback."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from oracle import segment_oracle as O, weights

G = os.path.join(os.path.dirname(__file__), "golden")


def rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).norm() / b.norm())


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(G, "segment_tiny.npz")), json.load(open(os.path.join(G, "segment_keys.json")))


def tiny_state_dict(meta):
    return O.seeded_state_dict({k: tuple(v) for k, v in meta["keys"].items()}, meta["seeds"][0])


def test_oracle_matches_reference(gold):
    g, meta = gold
    sd = tiny_state_dict(meta)
    assert weights.checksum({k: v for k, v in sd.items() if v.is_floating_point()}) == pytest.approx(float(g["wsum"]), rel=1e-12)
    raw = O.tiny_raw_images(O.TINY_SIZE, meta["seeds"][1])
    x = torch.cat([O.normalize(r) for r in raw])
    feats = O.backbone(sd, x)
    for i, f in enumerate(feats):
        e = rel(f[:1], g[f"out{i}"])
        print(f"[segment oracle] backbone out{i} {tuple(f.shape)} rel-L2 vs reference {e:.2e}")
        assert tuple(f[:1].shape) == g[f"out{i}"].shape and e <= 2e-6
    lg = O.decode(sd, feats)
    e = rel(lg[:1], g["logits"])
    print(f"[segment oracle] logits {tuple(lg.shape)} rel-L2 vs reference {e:.2e}")
    assert tuple(lg[:1].shape) == g["logits"].shape and e <= 2e-6
    assert g["out3"].shape[2] < 6, "the golden should exercise overlapping adaptive-pool bins"


def test_oracle_inference_matches_reference(gold):
    g, meta = gold
    sd = tiny_state_dict(meta)
    img = O.tiny_raw_images(O.TINY_RAW, meta["seeds"][2], B=1)[0]
    labels, out, size = O.inference(sd, img)
    assert size == tuple(g["infer_shape"][:2])
    margin = torch.from_numpy(g["infer_margin"])
    sure = margin > 1e-4
    agree = (labels == torch.from_numpy(g["infer_labels"]))
    print(f"[segment oracle] inference labels agree on {float(agree.float().mean()):.5f}, {int(sure.sum())} of {margin.numel()} "
          f"pixels with margin > 1e-4, {len(torch.unique(labels))} classes present")
    assert bool(agree[sure].all())
    assert rel(O.top2_margin(out), margin) <= 1e-5
    assert len(torch.unique(labels)) >= 3, "the golden's label map should not be trivial"


def test_preprocessing_matches_mmcv(gold):
    """imrescale (2048, 512) keep_ratio with cv2 INTER_LINEAR and imnormalize(to_rgb=True), pinned by hash."""
    g, meta = gold
    img = O.tiny_raw_images(O.TINY_RAW, meta["seeds"][2], B=1)[0]
    r = O.imrescale(img)
    assert r.shape == tuple(g["infer_shape"]) and r.shape[:2] == (512, 768)
    assert hashlib.sha256(np.ascontiguousarray(r).tobytes()).hexdigest() == str(g["infer_img_sha256"])
    x = O.normalize(r)
    assert hashlib.sha256(np.ascontiguousarray(x.numpy()).tobytes()).hexdigest() == str(g["infer_x_sha256"])
    from anyedit_b200 import segment
    assert segment.rescale(img).tobytes() == r.tobytes()
    # mmcv rescale_size: min(long / max(h, w), short / min(h, w)), then int(x s + 0.5)
    assert O.rescale_size(480, 640) == (512, 683) and O.rescale_size(640, 480) == (683, 512)
    assert O.rescale_size(100, 5000) == (41, 2048) and O.rescale_size(513, 513) == (512, 512)


def test_parameter_tree_matches_mmseg(gold):
    """UniFormerSegmentor's state dict has mmseg's keys and shapes at AnyEdit's config (upernet_global_small), BN buffers included,
    so that load_state_dict(torch.load(ckpt)["state_dict"], strict=True) takes the released checkpoint."""
    from anyedit_b200.segment import UniFormerSegmentor
    _, meta = gold
    want = meta["real_keys"]
    got = {k: list(v.shape) for k, v in UniFormerSegmentor().state_dict().items()}
    assert got == want
    assert any(k.startswith("auxiliary_head.") for k in got) and sum(k.endswith("num_batches_tracked") for k in got) > 0
    tiny = UniFormerSegmentor(embed_dim=O.TINY_BACKBONE["embed_dim"], layers=O.TINY_BACKBONE["layers"], channels=O.TINY_HEAD["channels"])
    assert {k: list(v.shape) for k, v in tiny.state_dict().items()} == meta["keys"]
    sd = tiny_state_dict(meta)
    tiny.load_state_dict(sd, strict=True)


def test_refusals_and_no_cpu_fallback():
    from anyedit_b200.segment import UniFormerSegmentor, show_result_pyplot
    for kw in (dict(windows=True), dict(hybrid=True)):
        with pytest.raises(NotImplementedError):
            UniFormerSegmentor(**kw)
    m = UniFormerSegmentor(embed_dim=[64, 128, 192, 256], layers=[1, 1, 1, 1], channels=64)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros(1, 64, 64, 3, dtype=torch.uint8))
    with pytest.raises(NotImplementedError):
        show_result_pyplot(m, np.zeros((4, 4, 3), np.uint8), [np.zeros((4, 4), np.int64)], np.zeros((150, 3), np.uint8), opacity=0.5)
