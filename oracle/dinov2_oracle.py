"""fp32 CPU restatement of AnyDoor's ``FrozenDinoV2Encoder`` (ldm/modules/encoders/modules.py:279-315) on the DINOv2 hub's
parameter names (TEST INFRASTRUCTURE, see oracle/__init__.py).

The encoder's arithmetic lives in the DINOv2 hub (``hubconf.dinov2_vitg14``), which is not in the reference tree: what is
restated here is the published ``DinoVisionTransformer.forward_features`` with the SwiGLU MLP (ImageNet normalisation, 14 x 14
patch conv, class token, bicubic position-table resize, pre-LN blocks with LayerScale, final LayerNorm), then the projector.
``tests/golden/make_golden_dinov2.py`` pins it against transformers' ``Dinov2Model`` at the offset-0.0 interpolation.
"""
import math

import torch
import torch.nn.functional as F

from . import weights

MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)

# the golden's tiny configuration (transformers Dinov2Config names): 9 x 9 position grid, 3 heads of 64, SwiGLU hidden 512
TINY = dict(hidden_size=192, num_hidden_layers=3, num_attention_heads=3, mlp_ratio=4, image_size=126, patch_size=14,
            layer_norm_eps=1e-6, use_swiglu_ffn=True)
TINY_PROJ = 64
TINY_SIZES = ((112, 140), (168, 168))       # 8 x 10 patches = 81 tokens (short-sequence attention), 12 x 12 = 145 (wgmma)


def seeded_state_dict(shapes, seed):
    """Name-keyed seeded weights (oracle.weights) with the position table at unit scale, the final LayerNorm gain around 1
    and every LayerScale in [0.3, 1.5] -- away from the hub's 1.0 and from 0, so that both branches of a block count."""
    sd = weights.make_state_dict(shapes, seed)
    for k, s in shapes.items():
        if k.endswith(("lambda1", "gamma")):
            lo, span = 0.9, 0.6
        elif k.endswith(("position_embeddings", "pos_embed")):
            lo, span = 0.0, 1.0
        elif k in ("layernorm.weight", "norm.weight", "model.norm.weight"):
            lo, span = 1.0, 0.2
        else:
            continue
        u = weights.fill_tensor(k, s, seed + 1)
        sd[k] = lo + span * (u / u.abs().max())
    return sd


def tiny_images(size, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(2, 3, size[0], size[1], generator=g)


def pos_table(pos_embed, gh, gw, offset):
    """[1, 1 + m*m, D] -> [1 + gh*gw, D]: hub ``interpolate_pos_encoding`` (offset 0.1: scale_factor form; 0: size form)."""
    pos = pos_embed.float().reshape(-1, pos_embed.shape[-1])
    m = int(math.isqrt(pos.shape[0] - 1))
    if gh == m and gw == m:
        return pos
    grid = pos[1:].reshape(1, m, m, -1).permute(0, 3, 1, 2)
    kw = {"scale_factor": ((gh + offset) / m, (gw + offset) / m)} if offset else {"size": (gh, gw)}
    g = F.interpolate(grid, mode="bicubic", align_corners=False, **kw)
    return torch.cat([pos[:1], g.permute(0, 2, 3, 1).reshape(gh * gw, -1)], 0)


def forward_features(sd, x, heads, patch=14, eps=1e-6, offset=0.1):
    """DinoVisionTransformer.forward_features on an already normalised image [B, 3, H, W] -> x_norm [B, 1 + gh*gw, D]."""
    sd = {k: v.float() for k, v in sd.items()}
    B, _, H, W = x.shape
    gh, gw = H // patch, W // patch
    t = F.conv2d(x.float(), sd["patch_embed.proj.weight"], sd["patch_embed.proj.bias"], stride=patch).flatten(2).transpose(1, 2)
    D = t.shape[-1]
    t = torch.cat([sd["cls_token"].expand(B, 1, D), t], 1) + pos_table(sd["pos_embed"], gh, gw, offset)[None]
    n, d = t.shape[1], D // heads
    i = 0
    while f"blocks.{i}.norm1.weight" in sd:
        p = lambda name: sd[f"blocks.{i}.{name}"]
        y = F.layer_norm(t, (D,), p("norm1.weight"), p("norm1.bias"), eps)
        qkv = F.linear(y, p("attn.qkv.weight"), p("attn.qkv.bias")).reshape(B, n, 3, heads, d).permute(2, 0, 3, 1, 4)
        s = torch.softmax((qkv[0] * d ** -0.5) @ qkv[1].transpose(-1, -2), -1)
        a = (s @ qkv[2]).transpose(1, 2).reshape(B, n, D)
        t = t + p("ls1.gamma") * F.linear(a, p("attn.proj.weight"), p("attn.proj.bias"))
        y = F.layer_norm(t, (D,), p("norm2.weight"), p("norm2.bias"), eps)
        x1, x2 = F.linear(y, p("mlp.w12.weight"), p("mlp.w12.bias")).chunk(2, -1)
        t = t + p("ls2.gamma") * F.linear(F.silu(x1) * x2, p("mlp.w3.weight"), p("mlp.w3.bias"))
        i += 1
    return F.layer_norm(t, (D,), sd["norm.weight"], sd["norm.bias"], eps)


def encoder(sd, image, heads, patch=14, eps=1e-6, offset=0.1):
    """FrozenDinoV2Encoder.forward: state dict with ``model.*`` and ``projector.*`` keys, image [B, 3, H, W] in [0, 1]."""
    mean, std = torch.tensor(MEAN).view(1, 3, 1, 1), torch.tensor(STD).view(1, 3, 1, 1)
    model = {k[len("model."):]: v for k, v in sd.items() if k.startswith("model.")}
    t = forward_features(model, (image.float() - mean) / std, heads, patch, eps, offset)
    return F.linear(t, sd["projector.weight"].float(), sd["projector.bias"].float())
