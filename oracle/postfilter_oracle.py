"""AnyEdit's post-filter scores (AnyEdit_Collection/filter_tool/utils.py get_clip_score, get_directional_clip, get_L1_distance)
restated in numpy (TEST INFRASTRUCTURE, see oracle/__init__.py).

  ``pillow_resize_bicubic``  PIL.Image.resize(BICUBIC) of uint8 HWC images as integer numpy: bicubic a = -0.5, support
                             2 max(scale, 1), per-output coefficients in double normalised to sum 1 and rounded half away from
                             zero to 22-bit fixed point, each pass an int32 sum on a 1 << 21 bias shifted right by 22 and
                             clipped to uint8, horizontal pass first, a pass of unchanged size skipped
  ``resize_size``            short side 224, long side int(224 * long / short)
  ``crop_offsets``           transformers' center_crop ((h - 224) // 2) or torchvision's (round((h - 224) / 2), half to even)
  ``pixel_values``           rescale + normalise of the two processors (float32)
  ``l1_distance``            sum((a - b) mod 256) / N / 255 in float64, utils.py's uint8 numpy expression
  ``clip_score`` / ``directional``   the float64 scores of the features
  ``openai_encode_image`` / ``openai_encode_text``   OpenAI CLIP's ``encode_image`` / ``encode_text`` in float64 from the
                             ``clip.load`` state-dict layout (VisionTransformer: conv1, class + positional embedding, ln_pre,
                             resblocks, ln_post on the class token, @ proj; text: token + positional embedding, causal
                             resblocks, ln_final, the features at argmax(ids) @ text_projection; QuickGELU)
"""
import math

import numpy as np
import torch

OPENAI_MEAN = (0.48145466, 0.4578275, 0.40821073)
OPENAI_STD = (0.26862954, 0.26130258, 0.27577711)
PREC = 22


def _bicubic(x):
    a = -0.5
    x = np.abs(x)
    return np.where(x < 1.0, ((a + 2.0) * x - (a + 3.0)) * x * x + 1.0,
                    np.where(x < 2.0, (((x - 5.0) * x + 8.0) * x - 4.0) * a, 0.0))


def _coeffs(n_in, n_out):
    """-> (xmin [n_out], fixed-point coefficients [n_out, ksize]) with zeros past each output's support."""
    scale = n_in / n_out
    fs = max(scale, 1.0)
    support = 2.0 * fs
    ksize = int(math.ceil(support)) * 2 + 1
    center = (np.arange(n_out) + 0.5) * scale
    xmin = np.maximum((center - support + 0.5).astype(np.int64), 0)      # C (int) truncation; negatives clamp to 0 either way
    xmax = np.minimum((center + support + 0.5).astype(np.int64), n_in) - xmin
    x = np.arange(ksize)[None, :]
    valid = x < xmax[:, None]
    w = np.where(valid, _bicubic((x + xmin[:, None] - center[:, None] + 0.5) * (1.0 / fs)), 0.0)
    ww = np.zeros(n_out)
    for j in range(ksize):          # Pillow sums the weights left to right
        ww = ww + w[:, j]
    w = np.where(ww[:, None] != 0.0, w / np.where(ww == 0.0, 1.0, ww)[:, None], w)
    k = np.where(w < 0, np.trunc(-0.5 + w * (1 << PREC)), np.trunc(0.5 + w * (1 << PREC))).astype(np.int64)
    return xmin, k


def _pass(img, n_out, axis, first=0, n=None):
    """One pass to n_out along axis; only outputs [first, first + n) are computed (each depends only on its own coefficients)."""
    n_in = img.shape[axis]
    n = n_out - first if n is None else n
    if n_in == n_out:
        return np.take(img, np.arange(first, first + n), axis)
    xmin, k = _coeffs(n_in, n_out)
    xmin, k = xmin[first:first + n], k[first:first + n]
    x = np.moveaxis(img.astype(np.int64), axis, 0)
    idx = np.minimum(xmin[:, None] + np.arange(k.shape[1])[None, :], n_in - 1)       # clamped taps carry coefficient 0
    acc = (x[idx] * k.reshape(k.shape + (1,) * (x.ndim - 1))).sum(1) + (1 << (PREC - 1))
    return np.moveaxis(np.clip(acc >> PREC, 0, 255).astype(np.uint8), 0, axis)


def pillow_resize_bicubic(img, size):
    """uint8 [H, W, C] -> uint8 [h, w, C] with size = (w, h) as PIL takes it."""
    w, h = size
    return _pass(_pass(np.asarray(img, np.uint8), w, 1), h, 0)


def resize_size(H, W, short=224):
    if W <= H:
        return int(short * H / W), short
    return short, int(short * W / H)


def crop_offsets(h, w, crop, size=224):
    if crop == "floor":
        return (h - size) // 2, (w - size) // 2
    assert crop == "round"
    return int(round((h - size) / 2.0)), int(round((w - size) / 2.0))


def preprocess_u8(img, crop):
    """-> the 224 x 224 uint8 crop the processor normalises (only the crop's columns and rows are computed)."""
    H, W = img.shape[:2]
    h, w = resize_size(H, W)
    t, l = crop_offsets(h, w, crop)
    return _pass(_pass(np.asarray(img, np.uint8), w, 1, l, 224), h, 0, t, 224)


def pixel_values(crop_u8, crop):
    """The processor's fp32 [3, 224, 224] from the crop's bytes: transformers rescales in float64 then casts (floor
    convention, CLIPImageProcessorPil), torchvision divides in float32 (round convention, ToTensor)."""
    x = np.asarray(crop_u8).transpose(2, 0, 1)
    if crop == "floor":
        x = (x.astype(np.float64) * (1 / 255)).astype(np.float32)
    else:
        x = x.astype(np.float32) / np.float32(255)
    mean = np.array(OPENAI_MEAN, np.float32)[:, None, None]
    std = np.array(OPENAI_STD, np.float32)[:, None, None]
    return (x - mean) / std


def l1_distance(a, b):
    a, b = np.asarray(a, np.uint8), np.asarray(b, np.uint8)
    if a.shape != b.shape:
        raise ValueError(f"shapes {a.shape} and {b.shape} differ")
    s = int(((a.astype(np.int64) - b.astype(np.int64)) % 256).sum())
    return float(np.float64(s) / a.size / 255)


def clip_score(img, txt, logit_scale):
    img, txt = np.asarray(img, np.float64), np.asarray(txt, np.float64)
    cos = (img * txt).sum(-1) / (np.linalg.norm(img, axis=-1) * np.linalg.norm(txt, axis=-1))
    return math.exp(float(logit_scale)) * cos / 100


def directional(img_a, img_b, txt_a, txt_b):
    di = np.asarray(img_b, np.float64) - np.asarray(img_a, np.float64)
    dt = np.asarray(txt_b, np.float64) - np.asarray(txt_a, np.float64)
    ni, nt = np.linalg.norm(di, axis=-1), np.linalg.norm(dt, axis=-1)
    ok = (ni > 0) & (nt > 0)
    return np.where(ok, (di * dt).sum(-1) / np.where(ok, ni * nt, 1.0), 0.0)


# ---- OpenAI CLIP (clip/model.py, public architecture) in float64 -----------------------------------------------------------
def _ln(x, sd, p, eps=1e-5):
    return torch.nn.functional.layer_norm(x, x.shape[-1:], sd[p + "weight"].double(), sd[p + "bias"].double(), eps)


def _resblocks(x, sd, prefix, heads, causal):
    F = torch.nn.functional
    i = 0
    while f"{prefix}{i}.ln_1.weight" in sd:
        p = f"{prefix}{i}."
        B, n, D = x.shape
        h = _ln(x, sd, p + "ln_1.")
        qkv = h @ sd[p + "attn.in_proj_weight"].double().T + sd[p + "attn.in_proj_bias"].double()
        q, k, v = (t.reshape(B, n, heads, D // heads).transpose(1, 2) for t in qkv.chunk(3, -1))
        s = q @ k.transpose(-1, -2) / math.sqrt(D // heads)
        if causal:
            s = s + torch.full((n, n), float("-inf"), dtype=s.dtype).triu(1)
        a = (s.softmax(-1) @ v).transpose(1, 2).reshape(B, n, D)
        x = x + a @ sd[p + "attn.out_proj.weight"].double().T + sd[p + "attn.out_proj.bias"].double()
        h = _ln(x, sd, p + "ln_2.") @ sd[p + "mlp.c_fc.weight"].double().T + sd[p + "mlp.c_fc.bias"].double()
        h = h * torch.sigmoid(1.702 * h)
        x = x + h @ sd[p + "mlp.c_proj.weight"].double().T + sd[p + "mlp.c_proj.bias"].double()
        i += 1
    return x


def openai_encode_image(sd, pixels, heads):
    """pixels float [B, 3, H, W] -> float64 [B, embed]."""
    x = torch.nn.functional.conv2d(pixels.double(), sd["visual.conv1.weight"].double(), stride=sd["visual.conv1.weight"].shape[-1])
    x = x.flatten(2).transpose(1, 2)
    cls = sd["visual.class_embedding"].double().expand(x.shape[0], 1, -1)
    x = torch.cat([cls, x], 1) + sd["visual.positional_embedding"].double()
    x = _ln(x, sd, "visual.ln_pre.")
    x = _resblocks(x, sd, "visual.transformer.resblocks.", heads, causal=False)
    return _ln(x[:, 0], sd, "visual.ln_post.") @ sd["visual.proj"].double()


def openai_encode_text(sd, ids, heads):
    """ids int [B, n] -> float64 [B, embed] (pooled at argmax of the ids, the end-of-text token)."""
    n = ids.shape[1]
    x = sd["token_embedding.weight"].double()[ids] + sd["positional_embedding"].double()[:n]
    x = _resblocks(x, sd, "transformer.resblocks.", heads, causal=True)
    x = _ln(x, sd, "ln_final.")
    return x[torch.arange(x.shape[0]), ids.argmax(-1)] @ sd["text_projection"].double()
