"""AnyEdit's post-filter scores, host side (no GPU): the numpy restatement of Pillow's bicubic resize and of the two CLIP
preprocessors against the live libraries, the launch plan the preprocess kernel reads (emulated here) against Pillow, the
wrapped L1 against utils.py's numpy expression, the float64 OpenAI CLIP restatement and the key mapping against
``transformers``, and ``keep`` against post_filter.py's truth table."""
import itertools

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import postfilter_oracle as O

LONG = 320


def pil_crop(img, crop):
    H, W = img.shape[:2]
    h, w = O.resize_size(H, W)
    r = np.asarray(Image.fromarray(img).resize((w, h), Image.BICUBIC))
    t, l = O.crop_offsets(h, w, crop)
    return r[t:t + 224, l:l + 224]


def sweep_sizes():
    return [(s, LONG) for s in range(1, 301)] + [(LONG, s) for s in range(1, 301)]


def test_resize_size_sweep_equals_pillow():
    rng = np.random.default_rng(1)
    bad = []
    for H, W in sweep_sizes() + [(224, 224), (225, 224), (224, 225), (3, 2000), (2000, 3), (1, 1), (480, 640), (427, 640), (300, 451)]:
        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        crop = "floor" if (H + W) % 2 else "round"
        if not np.array_equal(O.preprocess_u8(img, crop), pil_crop(img, crop)):
            bad.append((H, W))
    assert not bad, f"resize differs from Pillow at {bad[:10]}"


def content_images():
    out = []
    for H, W in [(37, 61), (300, 451), (640, 480), (231, 229)]:
        for y, x in [(0, 0), (H // 2, W // 3), (H - 1, W - 1)]:          # impulses expose the coefficients
            im = np.zeros((H, W, 3), np.uint8)
            im[y, x] = (255, 128, 1)
            out.append(im)
        out += [np.full((H, W, 3), v, np.uint8) for v in (0, 1, 254, 255)]                   # constants
        for p in (1, 2, 3):                                                                  # 0/255 checkerboards: clipping
            yy, xx = np.mgrid[0:H, 0:W]
            out.append(np.repeat((((yy // p + xx // p) % 2) * 255).astype(np.uint8)[..., None], 3, -1))
    return out


def test_resize_content_equals_pillow():
    for img, crop in itertools.product(content_images(), ("floor", "round")):
        assert np.array_equal(O.preprocess_u8(img, crop), pil_crop(img, crop)), (img.shape, crop)
        h, w = O.resize_size(*img.shape[:2])
        full = np.asarray(Image.fromarray(img).resize((w, h), Image.BICUBIC))
        assert np.array_equal(O.pillow_resize_bicubic(img, (w, h)), full)


def emulate_kernel(img, table, b):
    """The preprocess kernel's integer arithmetic on the plan's table, in numpy: horizontal pass to uint8, vertical pass."""
    g = table[b * 8: b * 8 + 8]
    H, W, ox_, sx, oy_, sy = (int(v) for v in g[:6])
    tx = table[ox_: ox_ + 224 * sx].reshape(224, sx).astype(np.int64)
    ty = table[oy_: oy_ + 224 * sy].reshape(224, sy).astype(np.int64)

    def one(src, t, axis):
        x = np.moveaxis(src.astype(np.int64), axis, 0)
        acc = np.full((224,) + x.shape[1:], 1 << 21, np.int64)
        for k in range(t.shape[1] - 2):
            use = k < t[:, 1]
            idx = np.where(use, t[:, 0] + k, 0)
            acc += x[idx] * np.where(use, t[:, 2 + k], 0).reshape((-1,) + (1,) * (x.ndim - 1))
        return np.moveaxis(np.clip(acc >> 22, 0, 255).astype(np.uint8), 0, axis)

    return one(one(img, tx, 1), ty, 0)


@pytest.mark.parametrize("crop", ["floor", "round"])
def test_kernel_plan_equals_pillow(crop):
    from anyedit_b200 import ops
    rng = np.random.default_rng(2)
    sizes = [(s, LONG) for s in range(1, 301, 7)] + [(LONG, s) for s in range(2, 301, 11)] + [(427, 640), (225, 224), (224, 224),
                                                                                             (4000, 300), (1, 1)]
    table, R, sm = ops.clip_preprocess_plan(sizes, crop, 14)
    table = table.numpy()
    assert 1 <= R <= 16 and 0 < sm <= 200 * 1024
    for b, (H, W) in enumerate(sizes):
        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        assert np.array_equal(emulate_kernel(img, table, b), pil_crop(img, crop)), (H, W)


def test_plan_refusals():
    from anyedit_b200 import ops
    with pytest.raises(ValueError):
        ops.clip_preprocess_plan([(10, 10)], "ceil", 14)
    with pytest.raises(ValueError):
        ops.clip_preprocess_plan([(10, 10)], "floor", 16)
    with pytest.raises(ValueError):
        ops.clip_preprocess_plan([(10, 10)], "floor", 14, channels=4)
    with pytest.raises(ValueError):
        ops.clip_preprocess_plan([(0, 10)], "floor", 14)
    with pytest.raises(ValueError):
        ops.clip_preprocess_plan([(10, 0)], "floor", 32)
    with pytest.raises(ValueError):
        ops.clip_preprocess_plan([], "floor", 32)


SIZES = [(427, 640), (640, 427), (300, 451), (512, 512), (480, 640), (225, 224), (224, 224), (97, 300), (300, 97)]


def test_crop_rules_and_pixels_equal_the_processors():
    from torchvision import transforms as T
    from transformers import CLIPImageProcessorPil
    proc = CLIPImageProcessorPil()
    tv = T.Compose([T.Resize(224, interpolation=T.InterpolationMode.BICUBIC), T.CenterCrop(224), T.ToTensor(),
                    T.Normalize(proc.image_mean, proc.image_std)])
    rng = np.random.default_rng(3)
    for H, W in SIZES:
        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        ref_h = np.asarray(proc(images=[Image.fromarray(img)], return_tensors="np")["pixel_values"])[0]
        ref_b = tv(Image.fromarray(img)).numpy()
        assert np.array_equal(O.pixel_values(O.preprocess_u8(img, "floor"), "floor"), ref_h), (H, W)
        assert np.array_equal(O.pixel_values(O.preprocess_u8(img, "round"), "round"), ref_b), (H, W)
    # the offsets differ where (h - 224) / 2 is a half: 427 x 640 -> 224 x 335, left 55 (floor) vs 56 (round)
    assert O.crop_offsets(224, 335, "floor") == (0, 55) and O.crop_offsets(224, 335, "round") == (0, 56)


def test_pixel_lut_equals_the_processors_on_every_byte():
    from torchvision import transforms as T
    from transformers import CLIPImageProcessorPil
    from anyedit_b200.postfilter import pixel_lut
    proc = CLIPImageProcessorPil()
    img = np.zeros((224, 224, 3), np.uint8)                  # 224 x 224: no resize, an identity crop
    img.reshape(-1, 3)[:256] = np.arange(256)[:, None]
    ref_h = torch.from_numpy(np.asarray(proc(images=[Image.fromarray(img)], return_tensors="np")["pixel_values"])[0])
    tv = T.Compose([T.ToTensor(), T.Normalize(proc.image_mean, proc.image_std)])
    ref_b = tv(Image.fromarray(img))
    for crop, ref in (("floor", ref_h), ("round", ref_b)):
        lut = pixel_lut(crop, "cpu")
        got = lut[:, torch.from_numpy(img.reshape(-1, 3)[:256, 0].astype(np.int64))]
        want = ref.reshape(3, -1)[:, :256].half()
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), crop


def utils_l1(a, b):
    """utils.py get_L1_distance on the RGB arrays."""
    l1_distance = np.sum(np.abs(a - b))
    num_pixels = a.shape[0] * a.shape[1] * a.shape[2]
    return l1_distance / num_pixels / 255


def test_l1_equals_the_numpy_expression():
    a = np.array([[[10, 200, 0]]], np.uint8)
    b = np.array([[[20, 100, 255]]], np.uint8)
    assert int(((a.astype(int) - b) % 256).sum()) == 246 + 100 + 1
    assert O.l1_distance(a, b) == utils_l1(a, b)
    rng = np.random.default_rng(4)
    for H, W in [(1, 1), (3, 5), (480, 640), (512, 512)]:
        a, b = (rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for _ in range(2))
        assert O.l1_distance(a, b) == utils_l1(a, b)
        assert O.l1_distance(a, a) == 0.0
    with pytest.raises(ValueError):
        O.l1_distance(np.zeros((2, 2, 3), np.uint8), np.zeros((2, 3, 3), np.uint8))


def _tiny_transformers(cfg_name):
    import json
    import os
    from transformers import CLIPConfig, CLIPModel
    from oracle import weights
    meta = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "postfilter_keys.json")))
    m = CLIPModel(CLIPConfig(**meta["configs"][cfg_name])).eval().double()
    sd = weights.make_state_dict({k: tuple(v) for k, v in meta["keys"][cfg_name].items()}, meta["seeds"][cfg_name])
    sd["logit_scale"] = torch.tensor(meta["logit_scale"])
    m.load_state_dict(sd, strict=False)
    return m, sd, meta["configs"][cfg_name]


def test_openai_restatement_equals_transformers_through_the_key_mapping():
    from anyedit_b200.encoders import transformers_to_openai_clip
    torch.set_grad_enabled(False)
    m, sd, cfg = _tiny_transformers("tiny_b32")
    osd = transformers_to_openai_clip(sd)
    g = torch.Generator().manual_seed(5)
    px = torch.randn(2, 3, 224, 224, generator=g, dtype=torch.float64)
    ids = torch.randint(10, 998, (2, 77), generator=g)
    ids[0, 9], ids[0, 10:], ids[1, 30], ids[1, 31:] = 999, 0, 999, 0
    vi = cfg["vision_config"]["num_attention_heads"]
    ti = cfg["text_config"]["num_attention_heads"]
    ref_i = m.get_image_features(pixel_values=px)
    ref_t = m.get_text_features(input_ids=ids)
    ref_i, ref_t = (getattr(t, "pooler_output", t) for t in (ref_i, ref_t))
    torch.testing.assert_close(O.openai_encode_image(osd, px, vi), ref_i, rtol=1e-9, atol=1e-9)
    torch.testing.assert_close(O.openai_encode_text(osd, ids, ti), ref_t, rtol=1e-9, atol=1e-9)


def test_key_mapping_round_trip():
    from anyedit_b200.encoders import CLIPModel, openai_clip_to_transformers, transformers_to_openai_clip
    _, sd, cfg = _tiny_transformers("tiny_b32")
    osd = transformers_to_openai_clip(sd)
    assert "visual.proj" in osd and "visual.transformer.resblocks.0.attn.in_proj_weight" in osd and "text_projection" in osd
    assert osd["visual.proj"].shape == sd["visual_projection.weight"].shape[::-1]
    back = openai_clip_to_transformers({**osd, "input_resolution": torch.tensor(224)})
    assert set(back) == set(sd) and all(torch.equal(back[k], sd[k]) for k in sd)
    model = CLIPModel(cfg)
    missing, unexpected = model.load_state_dict(back, strict=False)
    assert not unexpected and not [k for k in missing if "position_ids" not in k]


# post_filter.py:40-53 with the scorers replaced by the given values: (clip, l1, directional) -> decision
def ref_action_change(c, l, d):
    if c > 0.3:
        return d > 0.05


def ref_appearance_alter(c, l, d):
    if c > 0.25:
        if l > 0.3:
            return d > 0.06
    return False


def ref_tone_transfer(c, l, d):
    if c > 0.25:
        l1_score = l
        return l1_score > 0.2 and l1_score < 0.8


def test_keep_truth_table():
    from anyedit_b200.postfilter import keep
    refs = {"action_change": ref_action_change, "appearance_alter": ref_appearance_alter, "tone_transfer": ref_tone_transfer}
    vals = [0.0, 0.05, 0.06, 0.1, 0.2, 0.25, 0.26, 0.3, 0.31, 0.5, 0.8, 0.81, 1.0]
    for t, ref in refs.items():
        for c, l, d in itertools.product(vals, vals, [-0.1, 0.0, 0.05, 0.0500001, 0.06, 0.07]):
            assert keep(t, {"clip": c, "l1": l, "directional": d}) is ref(c, l, d), (t, c, l, d)
        got = keep(t, {"clip": torch.tensor([0.1, 0.4]), "l1": torch.tensor([0.5, 0.5]), "directional": torch.tensor([0.1, 0.1])})
        assert got == [ref(0.1, 0.5, 0.1), ref(0.4, 0.5, 0.1)]
    for t, needs in (("color_alter", "BLIP-2"), ("background_change", "BLIP-2"), ("textual_change", "GOT-OCR2"),
                     ("add", "GroundingDINO"), ("remove", "GroundingDINO"), ("replace", "SAM")):
        with pytest.raises(NotImplementedError, match=needs):
            keep(t, {"clip": 1.0, "l1": 0.5, "directional": 1.0})
