"""fp32 CPU restatement of AnyEdit's segmentation annotator: UniFormer (uniformer/mmseg/models/backbones/uniformer.py) + UPerHead
(decode_heads/uper_head.py, psp_head.py) and mmseg's whole-image test (apis/inference.py, segmentors/encoder_decoder.py) on the
reference's parameter names (TEST INFRASTRUCTURE, see oracle/__init__.py).  BatchNorm runs as BatchNorm (eval statistics), the
input normalisation as mmcv's ``imnormalize``: nothing is folded here.

``tests/golden/make_golden_segment.py`` pins it against the reference modules themselves on the tiny configuration below; it is the
reference wherever no golden exists (the real-width tests).
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import weights

MEAN = (123.675, 116.28, 103.53)           # configs/_base_/datasets/ade20k.py img_norm_cfg (RGB), to_rgb=True
STD = (58.395, 57.12, 57.375)
IMG_SCALE = (2048, 512)                    # the test pipeline's Resize(keep_ratio=True)
HEAD_DIM = 64
BN_EPS = 1e-5

# the golden's tiny configuration: every channel count a multiple of 64, 150 classes as at the real width
TINY_BACKBONE = dict(embed_dim=[64, 128, 192, 256], layers=[1, 1, 2, 1])
TINY_HEAD = dict(channels=128, num_classes=150)
TINY_SIZE = (68, 100)                      # not multiples of 32: patch crops at stages 2 and 3
TINY_RAW = (60, 90)                        # the inference case: rescaled to 512 x 768
REAL_BACKBONE = dict(embed_dim=[64, 128, 320, 512], layers=[3, 4, 8, 3])
REAL_HEAD = dict(channels=512, num_classes=150)
# residual-branch outputs drawn at 0.3 of unit gain, so that the residual stream of the 18-block real backbone stays well inside
# fp16 range (a trained network's branches are small too)
_BRANCH_OUT = ("pos_embed.weight", "conv2.weight", "mlp.fc2.weight", "attn.proj.weight")


def seeded_state_dict(shapes, seed):
    """Name-keyed seeded weights (oracle.weights.fill_tensor); every BatchNorm gets random running statistics and affine terms, so
    that folding it is not the identity."""
    sd = {}
    for k, s in shapes.items():
        if k.endswith("num_batches_tracked"):
            sd[k] = torch.zeros((), dtype=torch.int64)
            continue
        sd[k] = weights.fill_tensor(k, s, seed, gain=0.3 if k.endswith(_BRANCH_OUT) else 1.0)
    for k in shapes:
        if k.endswith(".running_var"):
            p, n = k[: -len("running_var")], int(np.prod(shapes[k]))
            u = lambda name: torch.from_numpy(weights._uniform(p + name, n, seed + 1))          # U(-1, 1)
            sd[p + "weight"] = 1.0 + 0.25 * u("weight")
            sd[p + "bias"] = 0.2 * u("bias")
            sd[p + "running_mean"] = 0.3 * u("running_mean")
            sd[p + "running_var"] = 1.0 + 0.5 * u("running_var")
    return sd


def tiny_raw_images(size, seed, B=2):
    """Seeded BGR uint8 images [B, H, W, 3]: a smooth colour field plus noise, so that the labels form regions."""
    rng = np.random.default_rng(seed)
    H, W = size
    yy, xx = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
    out = []
    for _ in range(B):
        f = rng.uniform(1, 4, size=(3, 2))
        ph = rng.uniform(0, 6.3, size=3)
        base = np.stack([np.sin(2 * np.pi * (f[c, 0] * yy + f[c, 1] * xx) + ph[c]) for c in range(3)], -1)
        img = 128 + 90 * base + rng.normal(0, 20, size=(H, W, 3))
        out.append(np.clip(img, 0, 255).astype(np.uint8))
    return np.stack(out)


def rescale_size(h, w, scale=IMG_SCALE):
    """mmcv rescale_size((w, h), scale) for a (long, short) bound -> (new_h, new_w)."""
    s = min(max(scale) / max(h, w), min(scale) / min(h, w))
    return int(h * s + 0.5), int(w * s + 0.5)


def imrescale(img, scale=IMG_SCALE):
    """mmcv imrescale(img, scale) with keep_ratio: cv2 INTER_LINEAR on the uint8 HWC image."""
    import cv2
    nh, nw = rescale_size(img.shape[0], img.shape[1], scale)
    return cv2.resize(img, (nw, nh), interpolation=cv2.INTER_LINEAR)


def normalize(img):
    """mmcv imnormalize(img, mean, std, to_rgb=True) -> fp32 NCHW [1, 3, H, W]."""
    import cv2
    x = np.ascontiguousarray(img[..., ::-1]).astype(np.float32)
    x = cv2.multiply(cv2.subtract(x, np.array(MEAN, np.float64).reshape(1, -1)), 1.0 / np.array(STD, np.float64).reshape(1, -1))
    return torch.from_numpy(np.ascontiguousarray(x.transpose(2, 0, 1)))[None]


def _bn(sd, p, x):
    return F.batch_norm(x, sd[p + "running_mean"], sd[p + "running_var"], sd[p + "weight"], sd[p + "bias"], False, 0.0, BN_EPS)


def _conv(sd, p, x, **kw):
    return F.conv2d(x, sd[p + "weight"], sd.get(p + "bias"), **kw)


def _patch_embed(sd, p, x, r):
    x = _conv(sd, p + "proj.", x, stride=r)
    C = x.shape[1]
    return F.layer_norm(x.permute(0, 2, 3, 1), (C,), sd[p + "norm.weight"], sd[p + "norm.bias"], 1e-5).permute(0, 3, 1, 2)


def _cblock(sd, p, x):
    C = x.shape[1]
    x = x + _conv(sd, p + "pos_embed.", x, padding=1, groups=C)
    y = _conv(sd, p + "conv1.", _bn(sd, p + "norm1.", x))
    x = x + _conv(sd, p + "conv2.", _conv(sd, p + "attn.", y, padding=2, groups=C))
    y = F.gelu(_conv(sd, p + "mlp.fc1.", _bn(sd, p + "norm2.", x)))
    return x + _conv(sd, p + "mlp.fc2.", y)


def _sablock(sd, p, x):
    B, C, H, W = x.shape
    heads = C // HEAD_DIM
    x = x + _conv(sd, p + "pos_embed.", x, padding=1, groups=C)
    t = x.flatten(2).transpose(1, 2)
    y = F.layer_norm(t, (C,), sd[p + "norm1.weight"], sd[p + "norm1.bias"], 1e-6)
    qkv = F.linear(y, sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"]).reshape(B, -1, 3, heads, HEAD_DIM).permute(2, 0, 3, 1, 4)
    a = torch.softmax((qkv[0] @ qkv[1].transpose(-2, -1)) * HEAD_DIM ** -0.5, -1) @ qkv[2]
    t = t + F.linear(a.transpose(1, 2).reshape(B, -1, C), sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"])
    y = F.layer_norm(t, (C,), sd[p + "norm2.weight"], sd[p + "norm2.bias"], 1e-6)
    t = t + F.linear(F.gelu(F.linear(y, sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"])), sd[p + "mlp.fc2.weight"],
                     sd[p + "mlp.fc2.bias"])
    return t.transpose(1, 2).reshape(B, C, H, W)


def _blocks(sd, stage):
    n = 0
    while f"backbone.blocks{stage}.{n}.pos_embed.weight" in sd:
        n += 1
    return n


def backbone(sd, x):
    """UniFormer.forward_features (windows=False, hybrid=False): the four normed stage outputs, NCHW fp32."""
    outs = []
    for s in range(1, 5):
        x = _patch_embed(sd, f"backbone.patch_embed{s}.", x, 4 if s == 1 else 2)
        for i in range(_blocks(sd, s)):
            p = f"backbone.blocks{s}.{i}."
            x = _cblock(sd, p, x) if s <= 2 else _sablock(sd, p, x)
        C = x.shape[1]
        n = f"backbone.norm{s}."
        outs.append(F.layer_norm(x.permute(0, 2, 3, 1), (C,), sd[n + "weight"], sd[n + "bias"], 1e-6).permute(0, 3, 1, 2))
    return outs


def _convmodule(sd, p, x, **kw):
    return F.relu(_bn(sd, p + "bn.", _conv(sd, p + "conv.", x, **kw)))


def _resize(x, size):
    return F.interpolate(x, size=tuple(size), mode="bilinear", align_corners=False)


def decode(sd, inputs, pool_scales=(1, 2, 3, 6)):
    """UPerHead.forward (align_corners=False): logits NCHW fp32 at the first input's resolution."""
    h = "decode_head."
    x = inputs[-1]
    psp = [x] + [_resize(_convmodule(sd, f"{h}psp_modules.{k}.1.", F.adaptive_avg_pool2d(x, s)), x.shape[2:])
                 for k, s in enumerate(pool_scales)]
    lat = [_convmodule(sd, f"{h}lateral_convs.{i}.", inputs[i]) for i in range(len(inputs) - 1)]
    lat.append(_convmodule(sd, h + "bottleneck.", torch.cat(psp, 1), padding=1))
    for i in range(len(lat) - 1, 0, -1):
        lat[i - 1] = lat[i - 1] + _resize(lat[i], lat[i - 1].shape[2:])
    fpn = [_convmodule(sd, f"{h}fpn_convs.{i}.", lat[i], padding=1) for i in range(len(lat) - 1)] + [lat[-1]]
    fpn = [fpn[0]] + [_resize(f, fpn[0].shape[2:]) for f in fpn[1:]]
    y = _convmodule(sd, h + "fpn_bottleneck.", torch.cat(fpn, 1), padding=1)
    return _conv(sd, h + "conv_seg.", y)


def logits(sd, x):
    return decode(sd, backbone(sd, x))


def inference(sd, raw):
    """inference_segmentor on one BGR uint8 image: (labels int64 [h, w], final fp32 logits [classes, h, w], network input size)."""
    img = imrescale(raw)
    x = normalize(img)
    out = _resize(logits(sd, x), x.shape[2:])
    out = _resize(out, raw.shape[:2])[0]
    return torch.softmax(out, 0).argmax(0), out, tuple(x.shape[2:])


def top2_margin(out):
    """Per-pixel gap between the largest and the second largest class value of [classes, h, w]."""
    t = out.topk(2, dim=0).values
    return t[0] - t[1]
