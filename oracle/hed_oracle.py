"""fp32 restatement of AnyEdit's HED scribble annotator (other_modules/HED/__init__.py: ControlNetHED_Apache2 and
HEDdetector.__call__) on the reference's parameter names (TEST INFRASTRUCTURE, see oracle/__init__.py).  The network runs as
F.conv2d / F.max_pool2d on whatever device the weights are on; the post-processing is the reference's, written out with cv2 and
numpy on the host: cv2.resize(INTER_LINEAR) of each side map, np.mean, a float64 sigmoid, uint8 truncation, cv2.bitwise_not.

``tests/golden/make_golden_hed.py`` pins it against the reference module itself at the real width; it is the reference wherever no
golden exists (the real-size GPU tests).
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import weights

# (cin, cout, number of 3x3 convs) of block1..block5
BLOCKS = ((3, 64, 2), (64, 128, 2), (128, 256, 3), (256, 512, 3), (512, 512, 3))
GOLDEN_SIZES = ((48, 64), (61, 93), (17, 200))     # even at every pool; odd sides floored by the pools; block 5 one pixel tall
# Seeded weights: He-scaled convs (13 ReLU layers neither vanish nor blow up), a per-channel norm around 115, and side projections
# drawn small enough that the mean of the five maps lands in the sigmoid's live range.
CONV_GAIN = 2.0 ** 0.5
PROJ_GAIN = 0.02


def param_shapes():
    """The reference's 37 tensors: norm, block{1..5}.convs.{i}.{weight,bias}, block{1..5}.projection.{weight,bias}."""
    shapes = {"norm": (1, 3, 1, 1)}
    for b, (cin, cout, n) in enumerate(BLOCKS, 1):
        for i in range(n):
            shapes[f"block{b}.convs.{i}.weight"] = (cout, cin if i == 0 else cout, 3, 3)
            shapes[f"block{b}.convs.{i}.bias"] = (cout,)
        shapes[f"block{b}.projection.weight"] = (1, cout, 1, 1)
        shapes[f"block{b}.projection.bias"] = (1,)
    return shapes


def seeded_state_dict(seed, conv_gain=CONV_GAIN, proj_gain=PROJ_GAIN):
    sd = {}
    for k, s in param_shapes().items():
        if k == "norm":
            sd[k] = torch.from_numpy(115.0 + 15.0 * weights._uniform(k, 3, seed)).reshape(s)
        else:
            sd[k] = weights.fill_tensor(k, s, seed, gain=proj_gain if ".projection." in k else conv_gain)
    return sd


def _box(a, r):
    """Box blur of radius r along the first two axes, edges replicated."""
    for ax in (0, 1):
        n = a.shape[ax]
        p = np.pad(a, [(r, r) if i == ax else (0, 0) for i in range(a.ndim)], mode="edge")
        c = np.cumsum(p, axis=ax)
        c = np.concatenate([np.zeros_like(np.take(c, [0], axis=ax)), c], axis=ax)
        a = (np.take(c, np.arange(2 * r + 1, 2 * r + 1 + n), axis=ax) - np.take(c, np.arange(n), axis=ax)) / (2 * r + 1)
    return a


def images(size, seed, B=1):
    """Seeded structured uint8 images [B, H, W, 3]: smoothed colour noise, a few filled rectangles and discs, fine noise."""
    rng = np.random.default_rng(seed)
    H, W = size
    yy, xx = np.mgrid[:H, :W]
    out = []
    for _ in range(B):
        base = _box(_box(rng.normal(0.0, 1.0, (H, W, 3)), max(1, min(H, W) // 10)), 2)
        img = 128.0 + 45.0 * base / base.std()
        for _ in range(4):
            col = rng.uniform(0, 255, 3)
            cy, cx = rng.uniform(0, H), rng.uniform(0, W)
            if rng.random() < 0.5:
                hy, hx = rng.uniform(0.1, 0.35) * H, rng.uniform(0.1, 0.35) * W
                mask = (np.abs(yy - cy) < hy) & (np.abs(xx - cx) < hx)
            else:
                r = rng.uniform(0.1, 0.3) * min(H, W)
                mask = (yy - cy) ** 2 + (xx - cx) ** 2 < r * r
            img[mask] = col
        img += rng.normal(0.0, 4.0, img.shape)
        out.append(np.clip(img, 0, 255).astype(np.uint8))
    return np.stack(out)


def side_maps(sd, img):
    """ControlNetHED_Apache2.__call__ on uint8 HWC images [B, H, W, 3] (numpy or tensor; channels as given, no swap) -> the five
    side maps, fp32 [B, 1, h, w], on the weights' device."""
    dev = sd["norm"].device
    # NCHW-contiguous, as the reference's rearranged single image is: a channels-last input would pick other conv kernels
    x = torch.as_tensor(np.asarray(img) if not isinstance(img, torch.Tensor) else img).to(dev).float().permute(0, 3, 1, 2).contiguous()
    h = x - sd["norm"]
    outs = []
    for b, (_, _, n) in enumerate(BLOCKS, 1):
        if b > 1:
            h = F.max_pool2d(h, kernel_size=(2, 2), stride=(2, 2))
        for i in range(n):
            h = F.relu(F.conv2d(h, sd[f"block{b}.convs.{i}.weight"], sd[f"block{b}.convs.{i}.bias"], padding=1))
        outs.append(F.conv2d(h, sd[f"block{b}.projection.weight"], sd[f"block{b}.projection.bias"]))
    return outs


def post_sigmoid(sides, H, W):
    """Per image: 255 sigmoid(mean of the cv2-resized side maps) in float64, before the uint8 cast, [B, H, W]."""
    import cv2
    out = []
    for i in range(sides[0].shape[0]):
        edges = [e[i, 0].detach().cpu().numpy().astype(np.float32) for e in sides]
        edges = np.stack([cv2.resize(e, (W, H), interpolation=cv2.INTER_LINEAR) for e in edges], axis=2)
        out.append(1 / (1 + np.exp(-np.mean(edges, axis=2).astype(np.float64))) * 255.0)
    return np.stack(out)


def edge_map(sides, H, W):
    """HEDdetector.__call__'s post-processing -> uint8 [B, H, W]."""
    import cv2
    return np.stack([cv2.bitwise_not(v.clip(0, 255).astype(np.uint8)) for v in post_sigmoid(sides, H, W)])


def detect(sd, img):
    img = np.asarray(img) if not isinstance(img, torch.Tensor) else img
    return edge_map(side_maps(sd, img), img.shape[1], img.shape[2])
