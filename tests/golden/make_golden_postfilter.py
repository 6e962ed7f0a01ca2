#!/usr/bin/env python
"""Golden vectors for AnyEdit's post-filter scores (AnyEdit_Collection/filter_tool/utils.py get_clip_score,
get_directional_clip, get_L1_distance).

The scorers' arithmetic lives in third-party libraries of the reference: ``transformers.CLIPModel`` + ``CLIPProcessor`` (the
PIL backend, ``CLIPImageProcessorPil``) for the CLIP score, OpenAI's ``clip`` ViT-B/32 with its torchvision transform for the
directional score (the ``clip`` package is not installed: its model is a ``transformers.CLIPModel`` with QuickGELU, whose
weights map one to one onto the ``clip.load`` layout).  Everything here runs those libraries' own code in fp32 on the CPU with
weights from ``oracle.weights`` seeds; the images are regenerated from ``images()`` by the tests.
Configurations: an H-like tiny model (patch 14, GELU, the first-eos pooling of a non-legacy eos id), a B/32-like tiny model
(patch 32, QuickGELU, the argmax pooling of eos id 2), and one pair at the real widths (ViT-H/14 + its 1024-wide text tower,
ViT-B/32) at B = 2.
Usage: python tests/golden/make_golden_postfilter.py"""
import json
import math
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..", "..")))

from oracle import weights  # noqa: E402

TINY_H = dict(text_config=dict(vocab_size=1000, hidden_size=128, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2,
                               max_position_embeddings=77, hidden_act="gelu", eos_token_id=7),
              vision_config=dict(hidden_size=160, intermediate_size=640, num_hidden_layers=2, num_attention_heads=2, image_size=224,
                                 patch_size=14, hidden_act="gelu"),
              projection_dim=64)
TINY_B32 = dict(text_config=dict(vocab_size=1000, hidden_size=128, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2,
                                 max_position_embeddings=77, hidden_act="quick_gelu", eos_token_id=2),
                vision_config=dict(hidden_size=128, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2, image_size=224,
                                   patch_size=32, hidden_act="quick_gelu"),
                projection_dim=48)
REAL_H = dict(text_config=dict(vocab_size=49408, hidden_size=1024, intermediate_size=4096, num_hidden_layers=24, num_attention_heads=16,
                               max_position_embeddings=77, hidden_act="gelu", eos_token_id=2),
              vision_config=dict(hidden_size=1280, intermediate_size=5120, num_hidden_layers=32, num_attention_heads=16, image_size=224,
                                 patch_size=14, hidden_act="gelu"),
              projection_dim=1024)
REAL_B32 = dict(text_config=dict(vocab_size=49408, hidden_size=512, intermediate_size=2048, num_hidden_layers=12, num_attention_heads=8,
                                 max_position_embeddings=77, hidden_act="quick_gelu", eos_token_id=2),
                vision_config=dict(hidden_size=768, intermediate_size=3072, num_hidden_layers=12, num_attention_heads=12, image_size=224,
                                   patch_size=32, hidden_act="quick_gelu"),
                projection_dim=512)
CONFIGS = {"tiny_h": (TINY_H, 91), "tiny_b32": (TINY_B32, 92), "real_h": (REAL_H, 93), "real_b32": (REAL_B32, 94)}
LOGIT_SCALE = math.log(100.0) - 0.03
# (original size, edited size) per pair; the edited image of pair 0 is the original with a band changed (wrapping bytes)
SIZES = [((427, 640), (427, 640)), ((512, 512), (512, 512))]


def images():
    """-> (originals, edited): uint8 HWC RGB numpy images, smooth enough that the scores are not noise."""
    rng = np.random.default_rng(2024)
    orig, edit = [], []
    for (H, W), _ in SIZES:
        y, x = np.mgrid[0:H, 0:W]
        base = np.stack([128 + 100 * np.sin(x / 37.0 + c) * np.cos(y / 53.0 - c) for c in range(3)], -1)
        a = np.clip(base + rng.normal(0, 12, base.shape), 0, 255).astype(np.uint8)
        b = a.copy()
        b[H // 4: H // 2] = (b[H // 4: H // 2].astype(np.int64) + 60).astype(np.uint8)          # wraps above 195
        b[:, : W // 3, 1] = 255 - b[:, : W // 3, 1]
        orig.append(a)
        edit.append(b)
    return orig, edit


def token_ids(cfg, seed, lengths):
    """[B, 77] ids: random tokens, the end-of-text token at lengths[i], padding after it."""
    tc = cfg["text_config"]
    V, eos = tc["vocab_size"], tc["eos_token_id"]
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(10, V - 1, (len(lengths), 77), generator=g)
    for i, n in enumerate(lengths):
        if eos == 2:                       # legacy id: pooled at the argmax -> the end-of-text token is the largest id, pad 0
            ids[i, n], ids[i, n + 1:] = V - 1, 0
        else:                              # first occurrence of eos_token_id; pad with the same id, as CLIPTokenizer does
            ids[i, n:] = eos
    return ids


def build(name):
    from transformers import CLIPConfig, CLIPModel
    cfg, seed = CONFIGS[name]
    m = CLIPModel(CLIPConfig(**cfg)).eval()
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items() if v.dtype.is_floating_point}
    sd = weights.make_state_dict(shapes, seed)
    sd["logit_scale"] = torch.tensor(LOGIT_SCALE)
    m.load_state_dict(sd, strict=False)
    return m, shapes, sd


def processors():
    from PIL import Image
    from torchvision import transforms as T
    from transformers import CLIPImageProcessorPil
    proc = CLIPImageProcessorPil()
    mean, std = proc.image_mean, proc.image_std
    tv = T.Compose([T.Resize(224, interpolation=T.InterpolationMode.BICUBIC), T.CenterCrop(224), T.ToTensor(), T.Normalize(mean, std)])
    h = lambda a: torch.as_tensor(np.asarray(proc(images=[Image.fromarray(x) for x in a], return_tensors="pt")["pixel_values"]))
    b32 = lambda a: torch.stack([tv(Image.fromarray(x).convert("RGB")) for x in a])
    return h, b32


def scores(m_h, m_b, orig, edit, ids_h, ids_in, ids_out):
    """utils.py's three scores (the directional score in fp32 here; the reference's CUDA model runs it in fp16)."""
    F = torch.nn.functional
    pre_h, pre_b = processors()
    px_h, px_a, px_b = pre_h(edit), pre_b(orig), pre_b(edit)
    out = m_h(input_ids=ids_h, pixel_values=px_h)
    clip = torch.diagonal(out.logits_per_image).double() / 100
    fa, fb = m_b.get_image_features(pixel_values=px_a), m_b.get_image_features(pixel_values=px_b)
    ta, tb = m_b.get_text_features(input_ids=ids_in), m_b.get_text_features(input_ids=ids_out)
    fa, fb, ta, tb = (getattr(t, "pooler_output", t) for t in (fa, fb, ta, tb))
    d = F.cosine_similarity(F.normalize(fb - fa, p=2, dim=-1), F.normalize(tb - ta, p=2, dim=-1), dim=1).double()
    l1 = []
    for a, b in zip(orig, edit):
        s = np.sum(np.abs(a - b))
        l1.append(s / (a.shape[0] * a.shape[1] * a.shape[2]) / 255)
    feats = lambda f: getattr(f, "pooler_output", f)
    return dict(img_h=feats(m_h.get_image_features(pixel_values=px_h)).numpy(), txt_h=feats(m_h.get_text_features(input_ids=ids_h)).numpy(),
                img_a=fa.numpy(), img_b=fb.numpy(), txt_a=ta.numpy(), txt_b=tb.numpy(),
                clip=clip.numpy(), directional=d.numpy(), l1=np.array(l1, np.float64))


def main():
    import transformers
    torch.set_grad_enabled(False)
    orig, edit = images()
    out, keys = {"transformers": transformers.__version__}, {}
    for tag, (nh, nb) in {"tiny": ("tiny_h", "tiny_b32"), "real": ("real_h", "real_b32")}.items():
        m_h, keys[nh], sd_h = build(nh)
        m_b, keys[nb], sd_b = build(nb)
        ids_h = token_ids(CONFIGS[nh][0], 5, [12, 40])
        ids_in, ids_out = token_ids(CONFIGS[nb][0], 6, [9, 30]), token_ids(CONFIGS[nb][0], 7, [15, 21])
        for k, v in scores(m_h, m_b, orig, edit, ids_h, ids_in, ids_out).items():
            out[f"{tag}_{k}"] = v
        out[f"{tag}_h_wsum"], out[f"{tag}_b32_wsum"] = weights.checksum(sd_h), weights.checksum(sd_b)
        print(tag, {k: out[f"{tag}_{k}"] for k in ("clip", "directional", "l1")}, flush=True)
        del m_h, m_b, sd_h, sd_b
    with open(os.path.join(HERE, "postfilter_keys.json"), "w") as f:
        json.dump({"configs": {k: v[0] for k, v in CONFIGS.items()}, "seeds": {k: v[1] for k, v in CONFIGS.items()},
                   "logit_scale": LOGIT_SCALE, "keys": {n: {k: list(v) for k, v in d.items()} for n, d in keys.items()}}, f)
    np.savez_compressed(os.path.join(HERE, "postfilter_tiny.npz"), **out)
    print({k: (v.shape if hasattr(v, "shape") else v) for k, v in out.items()})


if __name__ == "__main__":
    main()
