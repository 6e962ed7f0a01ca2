"""fp32 CPU restatement of Depth Anything V2 (AnyEdit_Collection/other_modules/depth_anything_v2/dpt.py, dinov2.py,
util/blocks.py) on the reference's parameter names (TEST INFRASTRUCTURE, see oracle/__init__.py).

``tests/golden/make_golden_depth.py`` pins it against the reference modules themselves on the tiny configuration below; it is
the reference wherever no golden exists (the real-width tests).
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import dinov2_oracle

# the golden's tiny configuration: D 192 (3 heads of 64), 4 blocks read at [0, 1, 2, 3], a 9 x 9 position table (img_size 126),
# features 128, out_channels [64, 128, 256, 256] -- channel counts at which every head conv takes the wgmma path
TINY_BACKBONE = dict(hidden_size=192, num_attention_heads=3, num_hidden_layers=4, image_size=126, use_swiglu_ffn=False)
TINY_HEAD = dict(features=128, out_channels=[64, 128, 256, 256])
TINY_LAYERS = [0, 1, 2, 3]
TINY_HEADS = 3
TINY_SWIGLU = dict(hidden_size=192, num_attention_heads=3, num_hidden_layers=2, image_size=126, use_swiglu_ffn=True)
TINY_SIZES = ((126, 126), (98, 182))
POS_GRIDS = ((7, 13), (9, 9), (12, 5))
POS_GRID_HASHED = (37, 56)
OUT_BIAS = "depth_head.scratch.output_conv2.2.bias"


def seeded_state_dict(shapes, seed):
    """Name-keyed seeded weights (dinov2_oracle.seeded_state_dict: LayerScale in [0.3, 1.5], unit position table) with the last
    head conv's bias positive, so that the depth maps are not all zero after the final ReLU."""
    sd = dinov2_oracle.seeded_state_dict(shapes, seed)
    if OUT_BIAS in sd:
        sd[OUT_BIAS] = torch.full_like(sd[OUT_BIAS], 0.5)
    return sd


def tiny_images(size, seed, B=2):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, 3, size[0], size[1], generator=g)


def raw_image(seed):
    """The BGR uint8 60 x 90 image of the golden's ``infer_image`` case."""
    return np.random.default_rng(seed).integers(0, 256, size=(60, 90, 3), dtype=np.uint8)


def _block(sd, pre, t, heads, eps):
    p = lambda name: sd[f"{pre}{name}"]
    B, n, D = t.shape
    d = D // heads
    y = F.layer_norm(t, (D,), p("norm1.weight"), p("norm1.bias"), eps)
    qkv = F.linear(y, p("attn.qkv.weight"), p("attn.qkv.bias")).reshape(B, n, 3, heads, d).permute(2, 0, 3, 1, 4)
    s = torch.softmax((qkv[0] * d ** -0.5) @ qkv[1].transpose(-1, -2), -1)
    a = (s @ qkv[2]).transpose(1, 2).reshape(B, n, D)
    t = t + p("ls1.gamma") * F.linear(a, p("attn.proj.weight"), p("attn.proj.bias"))
    y = F.layer_norm(t, (D,), p("norm2.weight"), p("norm2.bias"), eps)
    if f"{pre}mlp.fc1.weight" in sd:
        m = F.linear(F.gelu(F.linear(y, p("mlp.fc1.weight"), p("mlp.fc1.bias"))), p("mlp.fc2.weight"), p("mlp.fc2.bias"))
    else:
        x1, x2 = F.linear(y, p("mlp.w12.weight"), p("mlp.w12.bias")).chunk(2, -1)
        m = F.linear(F.silu(x1) * x2, p("mlp.w3.weight"), p("mlp.w3.bias"))
    return t + p("ls2.gamma") * m


def intermediate_layers(sd, x, blocks, heads, patch=14, eps=1e-6, offset=0.1):
    """DinoVisionTransformer.get_intermediate_layers(x, blocks, return_class_token=True, norm=True) on hub names (no prefix):
    -> [(patch tokens [B, gh*gw, D], class token [B, D])]."""
    sd = {k: v.float() for k, v in sd.items()}
    B, _, H, W = x.shape
    gh, gw = H // patch, W // patch
    t = F.conv2d(x.float(), sd["patch_embed.proj.weight"], sd["patch_embed.proj.bias"], stride=patch).flatten(2).transpose(1, 2)
    D = t.shape[-1]
    t = torch.cat([sd["cls_token"].expand(B, 1, D), t], 1) + dinov2_oracle.pos_table(sd["pos_embed"], gh, gw, offset)[None]
    out = []
    for i in range(max(blocks) + 1):
        t = _block(sd, f"blocks.{i}.", t, heads, eps)
        if i in blocks:
            y = F.layer_norm(t, (D,), sd["norm.weight"], sd["norm.bias"], eps)
            out.append((y[:, 1:], y[:, 0]))
    return out


def forward_features(sd, x, heads, patch=14, eps=1e-6, offset=0.1):
    """DinoVisionTransformer.forward_features -> x_norm [B, 1 + gh*gw, D] (class token first)."""
    n = 0
    while f"blocks.{n}.norm1.weight" in sd:
        n += 1
    (p, c), = intermediate_layers(sd, x, [n - 1], heads, patch, eps, offset)
    return torch.cat([c[:, None], p], 1)


def _rcu(sd, pre, x):
    out = F.conv2d(F.relu(x), sd[pre + "conv1.weight"], sd[pre + "conv1.bias"], padding=1)
    out = F.conv2d(F.relu(out), sd[pre + "conv2.weight"], sd[pre + "conv2.bias"], padding=1)
    return out + x


def _fusion(sd, pre, *xs, size=None):
    out = xs[0]
    if len(xs) == 2:
        out = out + _rcu(sd, pre + "resConfUnit1.", xs[1])
    out = _rcu(sd, pre + "resConfUnit2.", out)
    kw = {"scale_factor": 2} if size is None else {"size": size}
    out = F.interpolate(out, **kw, mode="bilinear", align_corners=True)
    return F.conv2d(out, sd[pre + "out_conv.weight"], sd[pre + "out_conv.bias"])


def head(sd, feats, gh, gw):
    """DPTHead.forward (use_clstoken=False) on ``depth_head.*`` names; feats = [(patch tokens, class token)] -> [B, 1, 14gh, 14gw]."""
    h = "depth_head."
    out = []
    for i, (x, _) in enumerate(feats):
        x = x.permute(0, 2, 1).reshape(x.shape[0], x.shape[-1], gh, gw)
        x = F.conv2d(x, sd[f"{h}projects.{i}.weight"], sd[f"{h}projects.{i}.bias"])
        if i == 0:
            x = F.conv_transpose2d(x, sd[f"{h}resize_layers.0.weight"], sd[f"{h}resize_layers.0.bias"], stride=4)
        elif i == 1:
            x = F.conv_transpose2d(x, sd[f"{h}resize_layers.1.weight"], sd[f"{h}resize_layers.1.bias"], stride=2)
        elif i == 3:
            x = F.conv2d(x, sd[f"{h}resize_layers.3.weight"], sd[f"{h}resize_layers.3.bias"], stride=2, padding=1)
        out.append(x)
    rn = [F.conv2d(x, sd[f"{h}scratch.layer{k + 1}_rn.weight"], padding=1) for k, x in enumerate(out)]
    s = h + "scratch."
    p4 = _fusion(sd, s + "refinenet4.", rn[3], size=rn[2].shape[2:])
    p3 = _fusion(sd, s + "refinenet3.", p4, rn[2], size=rn[1].shape[2:])
    p2 = _fusion(sd, s + "refinenet2.", p3, rn[1], size=rn[0].shape[2:])
    p1 = _fusion(sd, s + "refinenet1.", p2, rn[0])
    o = F.conv2d(p1, sd[s + "output_conv1.weight"], sd[s + "output_conv1.bias"], padding=1)
    o = F.interpolate(o, (int(gh * 14), int(gw * 14)), mode="bilinear", align_corners=True)
    o = F.relu(F.conv2d(o, sd[s + "output_conv2.0.weight"], sd[s + "output_conv2.0.bias"], padding=1))
    return F.relu(F.conv2d(o, sd[s + "output_conv2.2.weight"], sd[s + "output_conv2.2.bias"]))


def depth(sd, x, blocks, heads):
    """DepthAnythingV2.forward: x [B, 3, H, W] (normalised) -> fp32 [B, H, W]."""
    sd = {k: v.float() for k, v in sd.items()}
    hub = {k[len("pretrained."):]: v for k, v in sd.items() if k.startswith("pretrained.")}
    gh, gw = x.shape[-2] // 14, x.shape[-1] // 14
    feats = intermediate_layers(hub, x, blocks, heads)
    return F.relu(head(sd, feats, gh, gw)).squeeze(1)


def resize_depth(d, h, w):
    """infer_image's final resize: [B, H, W] -> [B, h, w]."""
    return F.interpolate(d[:, None], (h, w), mode="bilinear", align_corners=True)[:, 0]
