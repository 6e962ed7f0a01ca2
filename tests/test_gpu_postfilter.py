"""AnyEdit's post-filter scores on the GPU: the preprocess kernel against live Pillow / CLIPImageProcessorPil / torchvision bit
for bit, the wrapped L1 against numpy, and ``CLIPModel`` + the scores against the golden vectors
(tests/golden/make_golden_postfilter.py) at tiny and real widths.

Bounds of the model checks.  The towers run fp16 activations with fp32 accumulation against the golden's fp32 CPU run.  Each
fp16 rounding is 2^-11 relative; the errors of a pre-LN tower stay near that size relative to the residual stream, which the
final LayerNorm renormalises, so the projected features carry a relative error of order 1e-3 (measured: see DESIGN §10.10).
A cosine of features with relative error e moves by at most about 2e, so the CLIP score (cos * exp(logit_scale) / 100 ~ cos)
gets 4e-3 and the feature bounds 1e-2 (tiny) / 3e-2 (32 and 24 layers).  The directional cosine divides by the norms of
the feature differences, which are a fraction f of the features' norms (f ~ 0.3 for these edits), so its error is about
2e / f: bound 2e-2 (tiny) / 5e-2 (real)."""
import json
import os

import numpy as np
import pytest
import torch
from PIL import Image

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
LONG = 320


def pil_crop(img, crop):
    H, W = img.shape[:2]
    if W <= H:
        h, w = int(224 * H / W), 224
    else:
        h, w = 224, int(224 * W / H)
    r = np.asarray(Image.fromarray(img).resize((w, h), Image.BICUBIC))
    t, l = ((h - 224) // 2, (w - 224) // 2) if crop == "floor" else (int(round((h - 224) / 2)), int(round((w - 224) / 2)))
    return r[t:t + 224, l:l + 224]


def rows_to_pixels(rows, B, patch):
    g = 224 // patch
    x = rows[:, : 3 * patch * patch].reshape(B, g, g, 3, patch, patch)
    return x.permute(0, 3, 1, 4, 2, 5).reshape(B, 3, 224, 224)


def preprocess(images, crop, patch, crop_u8=True):
    from anyedit_b200 import ops
    from anyedit_b200.postfilter import pixel_lut
    dev = torch.device("cuda")
    t = [torch.from_numpy(np.ascontiguousarray(im)).to(dev) for im in images]
    cu8 = torch.empty(len(t), 224, 224, 3, dtype=torch.uint8, device=dev) if crop_u8 else None
    rows = ops.clip_preprocess(t, pixel_lut(crop, dev), patch, crop, crop_u8=cu8)
    torch.cuda.synchronize()
    return rows, cu8


@pytest.mark.parametrize("crop,patch", [("floor", 14), ("round", 32)])
def test_preprocess_sweep_ragged_equals_pillow(crop, patch):
    """Every short side 1..300 against a long side of 320, both orientations, plus upscales and extreme aspects: one ragged
    launch; the crop bytes equal Pillow's and the fp16 rows equal the processor's table of those bytes, padding zero."""
    from anyedit_b200.postfilter import pixel_lut
    rng = np.random.default_rng(11)
    sizes = [(s, LONG) for s in range(1, 301)] + [(LONG, s) for s in range(1, 301)] + [(3, 2000), (2000, 3), (1, 1), (4000, 300)]
    images = [rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for H, W in sizes]
    rows, cu8 = preprocess(images, crop, patch)
    got = cu8.cpu().numpy()
    bad = [sizes[i] for i, im in enumerate(images) if not np.array_equal(got[i], pil_crop(im, crop))]
    assert not bad, f"{len(bad)} sizes differ from Pillow, e.g. {bad[:8]}"
    lut = pixel_lut(crop, "cuda")
    want = lut[torch.arange(3, device="cuda")[None, :, None, None], cu8.permute(0, 3, 1, 2).long()]
    assert torch.equal(rows_to_pixels(rows, len(sizes), patch).view(torch.int16), want.view(torch.int16))
    if rows.shape[1] > 3 * patch * patch:
        assert not rows[:, 3 * patch * patch:].float().abs().sum()


def test_preprocess_rows_equal_the_live_processors():
    from torchvision import transforms as T
    from transformers import CLIPImageProcessorPil
    proc = CLIPImageProcessorPil()
    tv = T.Compose([T.Resize(224, interpolation=T.InterpolationMode.BICUBIC), T.CenterCrop(224), T.ToTensor(),
                    T.Normalize(proc.image_mean, proc.image_std)])
    rng = np.random.default_rng(12)
    sizes = [(427, 640), (640, 427), (300, 451), (512, 512), (480, 640), (225, 224), (224, 224), (97, 300), (1, 300), (300, 1)]
    images = [rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for H, W in sizes]
    for crop, patch, ref in (("floor", 14, lambda im: np.asarray(proc(images=[Image.fromarray(im)], return_tensors="np")["pixel_values"])[0]),
                             ("floor", 32, lambda im: np.asarray(proc(images=[Image.fromarray(im)], return_tensors="np")["pixel_values"])[0]),
                             ("round", 32, lambda im: tv(Image.fromarray(im)).numpy()),
                             ("round", 14, lambda im: tv(Image.fromarray(im)).numpy())):
        rows, _ = preprocess(images, crop, patch, crop_u8=False)
        px = rows_to_pixels(rows, len(images), patch).cpu()
        for i, im in enumerate(images):
            want = torch.from_numpy(ref(im)).half()
            assert torch.equal(px[i].view(torch.int16), want.view(torch.int16)), (crop, patch, sizes[i])


def test_preprocess_batch_independence():
    rng = np.random.default_rng(13)
    images = [rng.integers(0, 256, s + (3,), dtype=np.uint8) for s in [(480, 640), (512, 512), (3000, 200), (230, 231)]]
    rows_all, cu8_all = preprocess(images, "floor", 14)
    g = 16 * 16
    for i, im in enumerate(images):
        rows, cu8 = preprocess([im], "floor", 14)
        assert torch.equal(rows.view(torch.int16), rows_all[i * g:(i + 1) * g].view(torch.int16))
        assert torch.equal(cu8[0], cu8_all[i])


def test_l1_bit_equal_to_numpy():
    from anyedit_b200.postfilter import l1_distance
    rng = np.random.default_rng(14)
    pairs = [(np.array([[[10, 200, 0]]], np.uint8), np.array([[[20, 100, 255]]], np.uint8))]
    for H, W in [(480, 640), (512, 512), (1, 1), (7, 13), (1000, 333)]:
        pairs.append(tuple(rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for _ in range(2)))
    a = [torch.from_numpy(p[0]).cuda() for p in pairs]
    b = [torch.from_numpy(p[1]).cuda() for p in pairs]
    got = l1_distance(a, b).cpu().numpy()
    for i, (x, y) in enumerate(zip(a, b)):
        x, y = x.cpu().numpy(), y.cpu().numpy()
        ref = np.sum(np.abs(x - y)) / (x.shape[0] * x.shape[1] * x.shape[2]) / 255
        assert got[i] == ref, (i, got[i], ref)
    u8 = torch.zeros(1000, dtype=torch.uint8, device="cuda")
    a2, b2 = u8[1:301].view(10, 10, 3), u8[3:303].view(10, 10, 3)      # storage offsets off 16 bytes: the byte path
    u8.copy_(torch.arange(1000, device="cuda") * 7 % 256)
    assert float(l1_distance([a2], [b2])[0]) == np.sum(np.abs(a2.cpu().numpy() - b2.cpu().numpy())) / 300 / 255
    with pytest.raises(ValueError):
        l1_distance([a[0]], [torch.zeros(2, 2, 3, dtype=torch.uint8, device="cuda")])


def test_refusals():
    from anyedit_b200 import ops
    from anyedit_b200.postfilter import pixel_lut
    lut = pixel_lut("floor", "cuda")
    im = torch.zeros(10, 10, 3, dtype=torch.uint8, device="cuda")
    with pytest.raises(ValueError):
        ops.clip_preprocess([im], lut, 14, "ceil")
    with pytest.raises(ValueError):
        ops.clip_preprocess([im], lut, 16, "floor")
    with pytest.raises(ValueError):
        ops.clip_preprocess([torch.zeros(10, 10, 4, dtype=torch.uint8, device="cuda")], lut, 14, "floor")
    with pytest.raises(ValueError):
        ops.clip_preprocess([torch.zeros(0, 10, 3, dtype=torch.uint8, device="cuda")], lut, 14, "floor")
    with pytest.raises(ValueError):
        ops.clip_preprocess([], lut, 14, "floor")
    with pytest.raises(ValueError):
        ops.l1_wrapped_sum([], [])


# ---- models and scores against the golden ------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(HERE, "golden", "postfilter_tiny.npz")), json.load(open(os.path.join(HERE, "golden", "postfilter_keys.json")))


def _model(meta, name):
    from anyedit_b200.encoders import CLIPModel
    from oracle import weights
    m = CLIPModel(meta["configs"][name])
    sd = weights.make_state_dict({k: tuple(v) for k, v in meta["keys"][name].items()}, meta["seeds"][name])
    sd["logit_scale"] = torch.tensor(meta["logit_scale"])
    m.load_state_dict(sd, strict=False)
    return m.cuda(), sd


def _ids(name, meta):
    import sys
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import make_golden_postfilter as mg
    cfg = meta["configs"][name]
    return mg, cfg


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / b.norm())


@pytest.mark.parametrize("tag,feat_tol,dir_tol", [("tiny", 1e-2, 2e-2), ("real", 3e-2, 5e-2)])
def test_scores_against_golden(gold, tag, feat_tol, dir_tol):
    from anyedit_b200.encoders import openai_clip_to_transformers, transformers_to_openai_clip
    from anyedit_b200.postfilter import directional_clip, score_pairs
    g, meta = gold
    nh, nb = f"{tag}_h", f"{tag}_b32"
    mg, _ = _ids(nh, meta)
    m_h, _ = _model(meta, nh)
    m_b, sd_b = _model(meta, nb)
    # the ViT-B/32 weights through the OpenAI layout and back, as a ``clip.load`` checkpoint arrives
    m_b.load_state_dict(openai_clip_to_transformers(transformers_to_openai_clip(sd_b)), strict=False)
    m_b.invalidate()
    orig, edit = mg.images()
    to = lambda xs: [torch.from_numpy(x).cuda() for x in xs]
    ids_h = mg.token_ids(meta["configs"][nh], 5, [12, 40])
    ids_in, ids_out = mg.token_ids(meta["configs"][nb], 6, [9, 30]), mg.token_ids(meta["configs"][nb], 7, [15, 21])
    s = score_pairs(m_h, m_b, to(orig), to(edit), ids_in, ids_h, output_ids_b32=ids_out)
    from anyedit_b200.postfilter import image_features
    fh = image_features(m_h, to(edit), "floor")
    th = m_h.get_text_features(ids_h)
    fa, fb = image_features(m_b, to(orig), "round"), image_features(m_b, to(edit), "round")
    errs = {"img_h": _rel(fh, g[f"{tag}_img_h"]), "txt_h": _rel(th, g[f"{tag}_txt_h"]), "img_a": _rel(fa, g[f"{tag}_img_a"]),
            "img_b": _rel(fb, g[f"{tag}_img_b"]), "txt_a": _rel(m_b.get_text_features(ids_in), g[f"{tag}_txt_a"]),
            "txt_b": _rel(m_b.get_text_features(ids_out), g[f"{tag}_txt_b"])}
    dc = np.abs(s["clip"].numpy() - g[f"{tag}_clip"]).max()
    dd = np.abs(s["directional"].numpy() - g[f"{tag}_directional"]).max()
    print(f"{tag}: feature rel-L2 {errs}; |clip - golden| {dc:.2e} (golden {g[f'{tag}_clip']}); |directional - golden| {dd:.2e} "
          f"(golden {g[f'{tag}_directional']})")
    assert max(errs.values()) < feat_tol, errs
    assert dc < 4e-3 and dd < dir_tol
    assert np.array_equal(s["l1"].numpy(), g[f"{tag}_l1"])
    # directional_clip alone equals score_pairs' column; an unchanged pair scores exactly 0
    assert torch.equal(directional_clip(m_b, to(orig), to(edit), ids_in, ids_out), s["directional"])
    same = directional_clip(m_b, to(orig), to(orig), ids_in, ids_out)
    assert same.tolist() == [0.0, 0.0]


def test_padded_ids_equal_unpadded(gold):
    _, meta = gold
    for name in ("tiny_h", "tiny_b32"):
        m, _ = _model(meta, name)
        mg, cfg = _ids(name, meta)
        ids = mg.token_ids(cfg, 8, [10, 20])
        full = m.get_text_features(ids)
        short = m.get_text_features(ids[:, :24].contiguous())
        assert _rel(short, full) < 2e-3, name


def test_patch_rows_equal_pixel_path(gold):
    """get_image_features from the kernel's rows equals the pixel path on the processor's fp16 pixels, bit for bit."""
    from transformers import CLIPImageProcessorPil
    from anyedit_b200.postfilter import image_features
    _, meta = gold
    m, _ = _model(meta, "tiny_h")
    rng = np.random.default_rng(15)
    images = [rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for H, W in [(427, 640), (512, 512)]]
    px = np.asarray(CLIPImageProcessorPil()(images=[Image.fromarray(x) for x in images], return_tensors="np")["pixel_values"])
    a = m.get_image_features(pixel_values=torch.from_numpy(px).half().cuda())
    b = image_features(m, [torch.from_numpy(x).cuda() for x in images], "floor")
    assert torch.equal(a, b)
