"""AnyEdit's post-filter scores on the kernels (AnyEdit_Collection/filter_tool/utils.py, post_filter.py; DESIGN.md §10.10).

  ``clip_score(model_h, edited, output_ids)``            get_clip_score: exp(logit_scale) cos(image, caption) / 100 of a
                                                         ``encoders.CLIPModel`` (laion CLIP-ViT-H-14 in the reference)
  ``directional_clip(model_b32, original, edited, input_ids, output_ids)``   get_directional_clip: the cosine of the image
                                                         and caption feature differences (OpenAI ViT-B/32, mapped with
                                                         ``encoders.openai_clip_to_transformers``); 0 for an unchanged pair
  ``l1_distance(original, edited)``                      get_L1_distance: sum((a - b) mod 256) / N / 255 in float64
  ``score_pairs(...)``                                   all three for B pairs, one preprocess launch per model
  ``keep(edit_type, scores)``                            post_filter.py's decisions for action_change, appearance_alter and
                                                         tone_transfer

Images are lists of CUDA uint8 HWC RGB tensors of any sizes (the bytes of ``Image.convert('RGB')``); token ids come from the
caller (tokenisation and utils.py's caption-shortening ladder stay outside, as for ``FrozenCLIPEmbedder``), padded to one
length: the causal mask makes the padded tail invisible to the end-of-text token.  Preprocessing is Pillow's bicubic resize
and the processors' centre crop on the device: CLIPProcessor's (crop offset floored) for CLIP-H, ``clip``'s torchvision
transform (offset rounded half to even) for ViT-B/32; the fp16 pixels equal fp16 of the processors' float32 output.
"""
import numpy as np
import torch

from . import ops

OPENAI_MEAN = (0.48145466, 0.4578275, 0.40821073)
OPENAI_STD = (0.26862954, 0.26130258, 0.27577711)
# post_filter.py: the crop rule of each scorer's preprocessor
CLIP_H_CROP, CLIP_B32_CROP = "floor", "round"

_LUT = {}


def pixel_lut(crop, device):
    """fp16 [3, 256]: each byte's normalised value as the preprocessor computes it in float32, rounded to fp16.
    "floor": CLIPImageProcessorPil (rescale: byte * (1 / 255) in float64, cast to float32; (x - mean) / std in float32).
    "round": torchvision ToTensor + Normalize (byte / 255 in float32; (x - mean) / std in float32)."""
    key = (crop, str(device))
    if key not in _LUT:
        v = np.arange(256)
        if crop == "floor":
            x = (v.astype(np.float64) * (1 / 255)).astype(np.float32)
        elif crop == "round":
            x = v.astype(np.float32) / np.float32(255)
        else:
            raise ValueError(f"crop={crop!r}: 'floor' (transformers) or 'round' (torchvision)")
        mean = np.array(OPENAI_MEAN, np.float32)[:, None]
        std = np.array(OPENAI_STD, np.float32)[:, None]
        lut = ((x[None, :] - mean) / std).astype(np.float32)
        _LUT[key] = torch.from_numpy(lut).to(torch.float16).contiguous().to(device)
    return _LUT[key]


def _check_images(images, what):
    if not isinstance(images, (list, tuple)) or not images:
        raise ValueError(f"{what}: a non-empty list of uint8 HWC RGB CUDA tensors")
    for im in images:
        if not isinstance(im, torch.Tensor) or im.dtype != torch.uint8 or im.dim() != 3 or im.shape[2] != 3 or not im.is_cuda:
            raise ValueError(f"{what}: images are uint8 [H, W, 3] CUDA tensors")
    return [im.contiguous() for im in images]


def image_features(model, images, crop):
    """Preprocess B images in one launch and run the vision tower + projection -> fp32 [B, projection_dim]."""
    images = _check_images(images, "image_features")
    rows = ops.clip_preprocess(images, pixel_lut(crop, images[0].device), model.patch_size, crop)
    return model.get_image_features(patch_rows=rows)


def _ids(ids, B, what):
    ids = torch.as_tensor(ids)
    if ids.dim() != 2 or ids.shape[0] != B:
        raise ValueError(f"{what}: token ids [B = {B}, n]")
    return ids


def clip_score(model_h, edited, output_ids):
    """get_clip_score for B pairs -> float64 CPU tensor [B]."""
    edited = _check_images(edited, "clip_score")
    return _scores(model_h, None, edited, edited, None, output_ids, None)[:, 0].double()


def directional_clip(model_b32, original, edited, input_ids, output_ids):
    """get_directional_clip for B pairs -> float64 CPU tensor [B]."""
    original, edited = _check_images(original, "directional_clip"), _check_images(edited, "directional_clip")
    return _scores(None, model_b32, original, edited, input_ids, None, output_ids)[:, 1].double()


def l1_distance(original, edited):
    """get_L1_distance for B pairs -> float64 CUDA tensor [B]; shapes must match pair by pair (ValueError, as numpy)."""
    original, edited = _check_images(original, "l1_distance"), _check_images(edited, "l1_distance")
    s = ops.l1_wrapped_sum(original, edited)
    n = torch.tensor([a.numel() for a in original], dtype=torch.float64).to(s.device, non_blocking=True)
    return s.double() / n / 255


def _scores(model_h, model_b32, original, edited, input_ids, output_ids_h, output_ids_b):
    B = len(edited)
    if len(original) != B:
        raise ValueError("original and edited lists differ in length")
    dev = edited[0].device
    out = torch.zeros(B, 2, dtype=torch.float32, device=dev)
    feats = {}
    if model_h is not None:
        feats.update(img_h=image_features(model_h, edited, CLIP_H_CROP),
                     txt_h=model_h.get_text_features(_ids(output_ids_h, B, "output_ids")),
                     logit_scale=model_h.logit_scale_value())
    if model_b32 is not None:
        both = image_features(model_b32, list(original) + list(edited), CLIP_B32_CROP)
        ia, ob = _ids(input_ids, B, "input_ids"), _ids(output_ids_b, B, "output_ids")
        if ia.shape[1] != ob.shape[1]:
            raise ValueError("input_ids and output_ids: pad both to one length")
        txt = model_b32.get_text_features(torch.cat([ia, ob], 0))
        feats.update(img_a=both[:B].contiguous(), img_b=both[B:].contiguous(), txt_a=txt[:B].contiguous(), txt_b=txt[B:].contiguous())
    ops.postfilter_scores(out, **feats)
    return out.cpu()


def score_pairs(model_h, model_b32, original, edited, input_ids, output_ids, output_ids_b32=None):
    """All three scores for B pairs: one preprocess launch for CLIP-H's B edited images, one for ViT-B/32's 2B images.
    ``output_ids`` are CLIP-H's tokens of the output caption, ``input_ids`` / ``output_ids_b32`` ViT-B/32's of the input and
    output captions (``output_ids_b32`` defaults to ``output_ids``, for tokenisers that agree).
    -> {"clip": float64 [B], "directional": float64 [B], "l1": float64 [B]} on the CPU."""
    original, edited = _check_images(original, "score_pairs"), _check_images(edited, "score_pairs")
    l1 = l1_distance(original, edited)
    s = _scores(model_h, model_b32, original, edited, input_ids, output_ids,
                output_ids if output_ids_b32 is None else output_ids_b32).double()
    return {"clip": s[:, 0], "directional": s[:, 1], "l1": l1.cpu()}


_NEEDS = {"color_alter": "BLIP-2", "background_change": "BLIP-2", "textual_change": "GOT-OCR2",
          "add": "GroundingDINO + SAM", "remove": "GroundingDINO + SAM", "replace": "GroundingDINO + SAM"}


def _keep_one(edit_type, clip, l1, directional):
    if edit_type == "action_change":                 # post_filter.py:40-42
        if clip > 0.3:
            return directional > 0.05
        return None
    if edit_type == "appearance_alter":              # post_filter.py:44-48
        if clip > 0.25 and l1 > 0.3:
            return directional > 0.06
        return False
    if edit_type == "tone_transfer":                 # post_filter.py:50-53
        if clip > 0.25:
            return 0.2 < l1 < 0.8
        return None
    if edit_type in _NEEDS:
        raise NotImplementedError(f"{edit_type}: its post-filter needs {_NEEDS[edit_type]}, which does not run here")
    raise NotImplementedError(f"{edit_type}: no post-filter decision here (action_change, appearance_alter, tone_transfer)")


def keep(edit_type, scores):
    """post_filter.py's decision per pair from ``score_pairs``' scores (or one pair's scalars): True / False, or None where the
    reference function returns None below its CLIP gate (treated as "drop")."""
    clip, l1, d = scores["clip"], scores.get("l1"), scores.get("directional")
    if not isinstance(clip, torch.Tensor) or clip.dim() == 0:
        return _keep_one(edit_type, float(clip), None if l1 is None else float(l1), None if d is None else float(d))
    return [_keep_one(edit_type, float(clip[i]), None if l1 is None else float(l1[i]), None if d is None else float(d[i]))
            for i in range(len(clip))]
