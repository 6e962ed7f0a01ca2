"""UniFormer-S + UPerNet on the H100 kernels: the ADE20K segmentation annotator of AnyEdit's ``visual_segment`` edits
(AnyEdit_Collection/adaptive_editing_pipelines/visual_condition_tool.py:137-143, 176-182).

  ``UniFormerSegmentor``   mmseg's EncoderDecoder at other_modules/uniformer/configs/_base_/models/upernet_uniformer.py with
                           seg_config.py's overrides: ``backbone`` (UniFormer, mmseg/models/backbones/uniformer.py), ``decode_head``
                           (UPerHead, decode_heads/uper_head.py + psp_head.py) and ``auxiliary_head`` (FCNHead, held for the
                           checkpoint, never run).  The parameter tree is mmseg's, BN buffers included, so an
                           ``upernet_global_small`` checkpoint loads with ``load_state_dict(ckpt["state_dict"], strict=True)``.
  ``init_segmentor`` / ``inference_segmentor`` / ``show_result_pyplot``   the mmseg.apis names the annotator calls.

Launch plan (DESIGN.md §10.5); activations are NHWC fp16 token rows, every step a library kernel:
  patch_embed{s}   space_to_depth (kernel = stride = 4 | 2, remainders cropped; patch_embed1 straight from the uint8 BGR image) ->
                   one contraction -> LayerNorm (eps 1e-5).  Normalize(mean, std, to_rgb) is folded into patch_embed1's packed
                   weight and bias: the conv sees every pixel exactly once (no padding), so W (x - m) / s + b = (W / s) x + b'.
  CBlock           dwconv3 (pos_embed) + residual; conv1 with BN norm1 folded in; dwconv5 (attn); conv2 + residual;
                   mlp.fc1 with BN norm2 folded in and GELU; mlp.fc2 + residual
  SABlock          dwconv3 + residual; LayerNorm (1e-6); qkv; wgmma attention (d 64, scale 1/8); proj + residual;
                   LayerNorm; fc1 + GELU; fc2 + residual
  norm{s}          LayerNorm (1e-6) -> the head's input s; the stage continues from the un-normalised map
  UPerHead         every ConvModule = conv with its BN folded in + ReLU (act 6).  PPM: adaptive pool -> 1x1 -> half-pixel
                   resize into its channel slice of the [x, p1, p2, p3, p6] concat (x itself by the identity-size resize, which is
                   exact); bottleneck 3x3; laterals 1x1; top-down sums as resizes with an addend; fpn_convs (level 0 straight into
                   the second concat), each coarser level resized into its slice; fpn_bottleneck 3x3; conv_seg with its class
                   rows zero-padded to a multiple of 8, fp32 out.
  labels           seg_labels: both of mmseg's half-pixel resizes and the argmax per original pixel, with the palette lookup.
``windows`` / ``hybrid`` (windowed stage-3 attention; off in AnyEdit's config) raise.  CUDA only, no CPU fallback.
"""
import numpy as np
import torch
import torch.nn as nn

from . import ops
from .encoders import _Packable

IMG_SCALE = (2048, 512)                              # configs/_base_/datasets/ade20k.py test pipeline, Resize(keep_ratio=True)
IMG_MEAN = (123.675, 116.28, 103.53)                 # img_norm_cfg (RGB), to_rgb=True
IMG_STD = (58.395, 57.12, 57.375)
HEAD_DIM = 64


class _PatchEmbed(nn.Module):
    def __init__(self, cin, cout, r):
        super().__init__()
        self.norm = nn.LayerNorm(cout)
        self.proj = nn.Conv2d(cin, cout, r, stride=r)


class _CMlp(nn.Module):
    def __init__(self, dim, hidden, conv):
        super().__init__()
        self.fc1 = nn.Conv2d(dim, hidden, 1) if conv else nn.Linear(dim, hidden)
        self.fc2 = nn.Conv2d(hidden, dim, 1) if conv else nn.Linear(hidden, dim)


class _CBlock(nn.Module):
    def __init__(self, dim, mlp_ratio):
        super().__init__()
        self.pos_embed = nn.Conv2d(dim, dim, 3, padding=1, groups=dim)
        self.norm1 = nn.BatchNorm2d(dim)
        self.conv1 = nn.Conv2d(dim, dim, 1)
        self.conv2 = nn.Conv2d(dim, dim, 1)
        self.attn = nn.Conv2d(dim, dim, 5, padding=2, groups=dim)
        self.norm2 = nn.BatchNorm2d(dim)
        self.mlp = _CMlp(dim, int(dim * mlp_ratio), conv=True)


class _Attention(nn.Module):
    def __init__(self, dim, qkv_bias):
        super().__init__()
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.proj = nn.Linear(dim, dim)


class _SABlock(nn.Module):
    def __init__(self, dim, mlp_ratio, qkv_bias):
        super().__init__()
        self.pos_embed = nn.Conv2d(dim, dim, 3, padding=1, groups=dim)
        self.norm1 = nn.LayerNorm(dim, eps=1e-6)
        self.attn = _Attention(dim, qkv_bias)
        self.norm2 = nn.LayerNorm(dim, eps=1e-6)
        self.mlp = _CMlp(dim, int(dim * mlp_ratio), conv=False)


class UniFormer(nn.Module):
    """uniformer.py UniFormer parameter holder (windows=False, hybrid=False)."""

    def __init__(self, layers, embed_dim, head_dim, mlp_ratio, qkv_bias):
        super().__init__()
        self.embed_dim, self.head_dim = list(embed_dim), head_dim
        for s in range(4):
            cin = 3 if s == 0 else embed_dim[s - 1]
            setattr(self, f"patch_embed{s + 1}", _PatchEmbed(cin, embed_dim[s], 4 if s == 0 else 2))
        for s in range(4):
            blk = (lambda: _CBlock(embed_dim[s], mlp_ratio)) if s < 2 else (lambda: _SABlock(embed_dim[s], mlp_ratio, qkv_bias))
            setattr(self, f"blocks{s + 1}", nn.ModuleList([blk() for _ in range(layers[s])]))
            setattr(self, f"norm{s + 1}", nn.LayerNorm(embed_dim[s], eps=1e-6))


class _ConvModule(nn.Module):
    """mmcv ConvModule with norm_cfg BN and ReLU: a bias-free conv, BatchNorm, ReLU."""

    def __init__(self, cin, cout, k):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, k, padding=k // 2, bias=False)
        self.bn = nn.BatchNorm2d(cout)


class UPerHead(nn.Module):
    """uper_head.py UPerHead parameter holder (BaseDecodeHead's conv_seg; the PPM as psp_modules.{i}.1)."""

    def __init__(self, in_channels, channels, pool_scales, num_classes, align_corners):
        super().__init__()
        self.pool_scales, self.align_corners, self.num_classes = tuple(pool_scales), align_corners, num_classes
        self.conv_seg = nn.Conv2d(channels, num_classes, 1)
        self.psp_modules = nn.ModuleList([nn.Sequential(nn.AdaptiveAvgPool2d(s), _ConvModule(in_channels[-1], channels, 1))
                                          for s in pool_scales])
        self.bottleneck = _ConvModule(in_channels[-1] + len(pool_scales) * channels, channels, 3)
        self.lateral_convs = nn.ModuleList([_ConvModule(c, channels, 1) for c in in_channels[:-1]])
        self.fpn_convs = nn.ModuleList([_ConvModule(channels, channels, 3) for _ in in_channels[:-1]])
        self.fpn_bottleneck = _ConvModule(len(in_channels) * channels, channels, 3)


class FCNHead(nn.Module):
    """fcn_head.py FCNHead parameter holder (num_convs=1, concat_input=False): the training-time auxiliary head."""

    def __init__(self, in_channels, channels, num_classes):
        super().__init__()
        self.conv_seg = nn.Conv2d(channels, num_classes, 1)
        self.convs = nn.Sequential(_ConvModule(in_channels, channels, 3))


def _bn_fold(bn, dev):
    """BatchNorm2d (eval) as a per-channel fp64 (scale, shift)."""
    s = bn.weight.detach().to(dev, torch.float64) / torch.sqrt(bn.running_var.detach().to(dev, torch.float64) + bn.eps)
    return s, bn.bias.detach().to(dev, torch.float64) - bn.running_mean.detach().to(dev, torch.float64) * s


def _pack_w(w, dev):
    """Conv weight [co, ci, k, k] (or Linear [co, ci]) in fp64 -> [co, (ky, kx, ci)] fp16."""
    w = w.detach().to(dev, torch.float64)
    if w.dim() == 4:
        w = w.permute(0, 2, 3, 1)
    return w.reshape(w.shape[0], -1).half().contiguous()


def _b32(b, dev):
    return b.detach().to(dev, torch.float32).contiguous()


def _pre_bn(bn, conv, dev):
    """conv(BN(x)) for a 1x1 conv: W diag(s), W t + b."""
    s, t = _bn_fold(bn, dev)
    w = conv.weight.detach().to(dev, torch.float64).reshape(conv.weight.shape[0], -1)
    return _pack_w(w * s[None], dev), _b32(w @ t + conv.bias.detach().to(dev, torch.float64), dev)


def _post_bn(cm, dev):
    """ConvModule: BN(conv(x)) with a bias-free conv: s[co] W, t."""
    s, t = _bn_fold(cm.bn, dev)
    w = cm.conv.weight.detach().to(dev, torch.float64)
    return _pack_w(w * s.view(-1, *([1] * (w.dim() - 1))), dev), _b32(t, dev)


def _ln(m, dev):
    return _b32(m.weight, dev), _b32(m.bias, dev), m.eps


class UniFormerSegmentor(_Packable):
    """EncoderDecoder(UniFormer, UPerHead, FCNHead) at AnyEdit's configuration.  ``forward(img)``: uint8 BGR images [B, H, W, 3] on
    the GPU (one size per batch; the network input, i.e. already rescaled) -> fp32 logits [B, num_classes, H // 4, W // 4]."""

    def __init__(self, embed_dim=(64, 128, 320, 512), layers=(3, 4, 8, 3), head_dim=HEAD_DIM, mlp_ratio=4.0, qkv_bias=True, channels=512,
                 pool_scales=(1, 2, 3, 6), num_classes=150, align_corners=False, windows=False, hybrid=False):
        super().__init__()
        if windows or hybrid:
            raise NotImplementedError("UniFormerSegmentor: windowed / hybrid stage-3 attention is not implemented (AnyEdit's "
                                      "seg_config.py sets windows=False, hybrid=False)")
        if align_corners:
            raise NotImplementedError("UniFormerSegmentor: align_corners=True is not implemented (upernet_uniformer.py: False)")
        if head_dim != HEAD_DIM or any(c % HEAD_DIM for c in embed_dim[2:]) or any(c % 8 for c in embed_dim) or channels % 64:
            raise ValueError(f"UniFormerSegmentor: needs head_dim 64, stage-3/4 widths divisible by 64, all widths by 8 and channels "
                             f"by 64 (got head_dim={head_dim}, embed_dim={list(embed_dim)}, channels={channels})")
        self.backbone = UniFormer(list(layers), list(embed_dim), head_dim, mlp_ratio, qkv_bias)
        self.decode_head = UPerHead(list(embed_dim), channels, pool_scales, num_classes, align_corners)
        self.auxiliary_head = FCNHead(embed_dim[2], channels // 2, num_classes)
        self.align_corners = align_corners
        self.eval()

    def _packed(self):
        # the BatchNorm statistics are buffers, which the parameter versions do not cover: a load_state_dict repacks
        key = sum(b._version for b in self.buffers())
        if key != getattr(self, "_buffer_key", None):
            self.invalidate()
            self._buffer_key = key
        return super()._packed()

    def _build_pack(self, dev):
        bb, hd = self.backbone, self.decode_head
        w1 = bb.patch_embed1.proj.weight.detach().to(dev, torch.float64)              # [co, RGB, 4, 4]
        mean = torch.tensor(IMG_MEAN, dtype=torch.float64, device=dev)
        std = torch.tensor(IMG_STD, dtype=torch.float64, device=dev)
        b1 = bb.patch_embed1.proj.bias.detach().to(dev, torch.float64) - (w1 * (mean / std).view(1, 3, 1, 1)).sum((1, 2, 3))
        w1 = (w1 / std.view(1, 3, 1, 1)).flip(1)                                     # the image is BGR: channel order reversed
        pe = [(_pack_w(w1, dev), _b32(b1, dev), _ln(bb.patch_embed1.norm, dev))]
        for s in (2, 3, 4):
            p = getattr(bb, f"patch_embed{s}")
            pe.append((_pack_w(p.proj.weight, dev), _b32(p.proj.bias, dev), _ln(p.norm, dev)))
        blocks = []
        for s in range(1, 5):
            st = []
            for b in getattr(bb, f"blocks{s}"):
                d = {"pos": (ops.pack_dwconv(b.pos_embed.weight, dev), _b32(b.pos_embed.bias, dev))}
                if s <= 2:
                    d["conv1"] = _pre_bn(b.norm1, b.conv1, dev)
                    d["attn"] = (ops.pack_dwconv(b.attn.weight, dev), _b32(b.attn.bias, dev))
                    d["conv2"] = (_pack_w(b.conv2.weight, dev), _b32(b.conv2.bias, dev))
                    d["fc1"] = _pre_bn(b.norm2, b.mlp.fc1, dev)
                else:
                    d["ln1"], d["ln2"] = _ln(b.norm1, dev), _ln(b.norm2, dev)
                    d["qkv"] = (_pack_w(b.attn.qkv.weight, dev), _b32(b.attn.qkv.bias, dev))
                    d["proj"] = (_pack_w(b.attn.proj.weight, dev), _b32(b.attn.proj.bias, dev))
                    d["fc1"] = (_pack_w(b.mlp.fc1.weight, dev), _b32(b.mlp.fc1.bias, dev))
                d["fc2"] = (_pack_w(b.mlp.fc2.weight, dev), _b32(b.mlp.fc2.bias, dev))
                st.append(d)
            blocks.append(st)
        K = hd.num_classes
        Kp = (K + 7) // 8 * 8
        ws = torch.zeros(Kp, hd.conv_seg.weight.shape[1], dtype=torch.float16, device=dev)
        ws[:K] = _pack_w(hd.conv_seg.weight, dev)
        bs = torch.zeros(Kp, dtype=torch.float32, device=dev)
        bs[:K] = _b32(hd.conv_seg.bias, dev)
        return {"pe": pe, "blocks": blocks, "norm": [_ln(getattr(bb, f"norm{s}"), dev) for s in range(1, 5)],
                "psp": [_post_bn(m[1], dev) for m in hd.psp_modules], "bottleneck": _post_bn(hd.bottleneck, dev),
                "lateral": [_post_bn(m, dev) for m in hd.lateral_convs], "fpn": [_post_bn(m, dev) for m in hd.fpn_convs],
                "fpn_bottleneck": _post_bn(hd.fpn_bottleneck, dev), "seg": (ws, bs)}

    # ---- backbone ----------------------------------------------------------------------------------------------------------
    @staticmethod
    def _cblock(x, d):
        B, H, W, C = x.shape
        x1 = torch.empty_like(x)
        ops.dwconv(x, *d["pos"], x1, residual=x)
        u = torch.empty_like(x)
        ops.gemm(x1.view(-1, C), d["conv1"][0], u.view(-1, C), bias=d["conv1"][1])
        v = torch.empty_like(x)
        ops.dwconv(u, *d["attn"], v)
        x2 = torch.empty_like(x)
        ops.gemm(v.view(-1, C), d["conv2"][0], x2.view(-1, C), bias=d["conv2"][1], residual=x1.view(-1, C))
        return UniFormerSegmentor._mlp(x2, x2.view(-1, C), d)

    @staticmethod
    def _mlp(x, a, d):
        """x + fc2(GELU(fc1(a))) on the rows of x."""
        C = x.shape[-1]
        h = torch.empty(a.shape[0], d["fc1"][0].shape[0], dtype=torch.float16, device=x.device)
        ops.gemm(a, d["fc1"][0], h, bias=d["fc1"][1], act=3)
        out = torch.empty_like(x)
        ops.gemm(h, d["fc2"][0], out.view(-1, C), bias=d["fc2"][1], residual=x.view(-1, C))
        return out

    @staticmethod
    def _sablock(x, d):
        B, H, W, C = x.shape
        n, heads = H * W, C // HEAD_DIM
        x1 = torch.empty_like(x)
        ops.dwconv(x, *d["pos"], x1, residual=x)
        y = torch.empty(B * n, C, dtype=torch.float16, device=x.device)
        ops.layernorm(x1.view(-1, C), d["ln1"][0], d["ln1"][1], y, d["ln1"][2])
        qkv = torch.empty(B * n, 3 * C, dtype=torch.float16, device=x.device)
        ops.gemm(y, d["qkv"][0], qkv, bias=d["qkv"][1])
        a = torch.empty(B * n, C, dtype=torch.float16, device=x.device)
        ops.attention(qkv, qkv[:, C:], qkv[:, 2 * C:], a, B, heads, n, n, HEAD_DIM, 3 * C, 3 * C, 3 * C, C, scale=HEAD_DIM ** -0.5)
        x2 = torch.empty_like(x)
        ops.gemm(a, d["proj"][0], x2.view(-1, C), bias=d["proj"][1], residual=x1.view(-1, C))
        ops.layernorm(x2.view(-1, C), d["ln2"][0], d["ln2"][1], y, d["ln2"][2])
        return UniFormerSegmentor._mlp(x2, y, d)

    def _backbone(self, img, P):
        """uniformer.py forward_features on uint8 BGR [B, H, W, 3] -> the four normed maps, NHWC fp16."""
        B = img.shape[0]
        dev = img.device
        x, outs = img, []
        for s in range(4):
            r = 4 if s == 0 else 2
            w, b, (g, beta, eps) = P["pe"][s]
            Ho, Wo = x.shape[1] // r, x.shape[2] // r
            if Ho < 1 or Wo < 1:
                raise ValueError(f"UniFormerSegmentor: image {tuple(img.shape[1:3])} too small for four patch stages")
            cols = torch.empty(B * Ho * Wo, r * r * x.shape[3], dtype=torch.float16, device=dev)
            ops.space_to_depth(x, cols, r)
            t = torch.empty(B * Ho * Wo, w.shape[0], dtype=torch.float16, device=dev)
            ops.gemm(cols, w, t, bias=b)
            x = torch.empty(B, Ho, Wo, w.shape[0], dtype=torch.float16, device=dev)
            ops.layernorm(t, g, beta, x.view(-1, w.shape[0]), eps)
            for d in P["blocks"][s]:
                x = self._cblock(x, d) if s < 2 else self._sablock(x, d)
            g, beta, eps = P["norm"][s]
            o = torch.empty_like(x)
            ops.layernorm(x.view(-1, x.shape[3]), g, beta, o.view(-1, x.shape[3]), eps)
            outs.append(o)
        return outs

    # ---- head --------------------------------------------------------------------------------------------------------------
    def _decode(self, feats, P):
        """uper_head.py UPerHead.forward -> fp32 NHWC logits [B, h, w, num_classes rounded up to 8]."""
        hd = self.decode_head
        x = feats[-1]
        B, h4, w4, C4 = x.shape
        dev = x.device
        f16 = dict(dtype=torch.float16, device=dev)
        Ch = P["bottleneck"][0].shape[0]
        cat = torch.empty(B, h4, w4, C4 + len(hd.pool_scales) * Ch, **f16)
        ops.resize_bilinear(x, cat[..., :C4], align_corners=False)                    # identity size: an exact copy
        for k, s in enumerate(hd.pool_scales):                                        # PPM (psp_head.py:44-55)
            pooled = torch.empty(B, s, s, C4, **f16)
            ops.adaptive_avg_pool(x, pooled)
            y = torch.empty(B, s, s, Ch, **f16)
            ops.gemm(pooled.view(-1, C4), P["psp"][k][0], y.view(-1, Ch), bias=P["psp"][k][1], act=6)
            c0 = C4 + k * Ch
            ops.resize_bilinear(y, cat[..., c0:c0 + Ch], align_corners=False)
        lat = []
        for i in range(len(feats) - 1):                                               # lateral_convs
            f = feats[i]
            y = torch.empty(*f.shape[:3], Ch, **f16)
            ops.gemm(f.view(-1, f.shape[3]), P["lateral"][i][0], y.view(-1, Ch), bias=P["lateral"][i][1], act=6)
            lat.append(y)
        top = torch.empty(B, h4, w4, Ch, **f16)
        ops.conv3x3(cat, P["bottleneck"][0], top.view(-1, Ch), bias=P["bottleneck"][1], act=6)
        lat.append(top)
        for i in range(len(lat) - 1, 0, -1):                                          # laterals[i - 1] += resize(laterals[i])
            ops.resize_bilinear(lat[i], lat[i - 1], addend=lat[i - 1], align_corners=False)
        h1, w1 = lat[0].shape[1:3]
        L = len(lat)
        cat2 = torch.empty(B, h1, w1, L * Ch, **f16)
        for i in range(L - 1):                                                        # fpn_convs; level 0 straight into the concat
            wf, bf = P["fpn"][i]
            if i == 0:
                ops.conv3x3(lat[0], wf, cat2.view(-1, L * Ch)[:, :Ch], bias=bf, act=6)
            else:
                y = torch.empty_like(lat[i])
                ops.conv3x3(lat[i], wf, y.view(-1, Ch), bias=bf, act=6)
                ops.resize_bilinear(y, cat2[..., i * Ch:(i + 1) * Ch], align_corners=False)
        ops.resize_bilinear(lat[-1], cat2[..., (L - 1) * Ch:], align_corners=False)
        fb = torch.empty(B, h1, w1, Ch, **f16)
        ops.conv3x3(cat2, P["fpn_bottleneck"][0], fb.view(-1, Ch), bias=P["fpn_bottleneck"][1], act=6)
        ws, bs = P["seg"]
        logits = torch.empty(B, h1, w1, ws.shape[0], dtype=torch.float32, device=dev)
        ops.gemm(fb.view(-1, Ch), ws, logits.view(-1, ws.shape[0]), bias=bs)
        return logits

    def _check(self, img):
        if not (isinstance(img, torch.Tensor) and img.dtype == torch.uint8 and img.dim() == 4 and img.shape[3] == 3):
            raise ValueError("UniFormerSegmentor: expects uint8 BGR images [B, H, W, 3]")
        P = self._packed()
        if not img.is_cuda:
            raise RuntimeError("UniFormerSegmentor runs on CUDA only (no CPU fallback); move the image to the model's device")
        return P, img.contiguous()

    @torch.no_grad()
    def logits_nhwc(self, img):
        """fp32 logits [B, H // 4, W // 4, num_classes rounded up to 8] (the padding classes are zero)."""
        P, img = self._check(img)
        return self._decode(self._backbone(img, P), P)

    @torch.no_grad()
    def backbone_features(self, img):
        """The four normed backbone maps (UniFormer.forward), NHWC fp16."""
        P, img = self._check(img)
        return self._backbone(img, P)

    @torch.no_grad()
    def forward(self, img):
        lg = self.logits_nhwc(img)
        B, h, w, _ = lg.shape
        out = torch.empty(B, self.decode_head.num_classes, h, w, dtype=torch.float32, device=lg.device)
        ops.nhwc_to_nchw(lg, out)
        return out

    @torch.no_grad()
    def labels(self, img, out_size, palette=None):
        """mmseg's simple_test labels for the rescaled image(s) ``img`` of original size ``out_size`` (h, w): int64 [B, h, w], and
        with ``palette`` (uint8 [num_classes, 3] on the device) also the colour map uint8 [B, h, w, 3]."""
        lg = self.logits_nhwc(img)
        B = lg.shape[0]
        lab = torch.empty(B, int(out_size[0]), int(out_size[1]), dtype=torch.int64, device=lg.device)
        rgb = torch.empty(*lab.shape, 3, dtype=torch.uint8, device=lg.device) if palette is not None else None
        ops.seg_labels(lg, self.decode_head.num_classes, img.shape[1:3], lab, palette=palette, rgb=rgb)
        return lab if palette is None else (lab, rgb)


def rescale(img, scale=IMG_SCALE):
    """mmcv imrescale(img, scale) with keep_ratio (the test pipeline's Resize): s = min(long / max(h, w), short / min(h, w)),
    size int(x s + 0.5), cv2 INTER_LINEAR on the uint8 image."""
    import cv2
    h, w = img.shape[:2]
    s = min(max(scale) / max(h, w), min(scale) / min(h, w))
    return cv2.resize(img, (int(w * s + 0.5), int(h * s + 0.5)), interpolation=cv2.INTER_LINEAR)


def init_segmentor(config=None, checkpoint=None, device="cuda"):
    """mmseg.apis.init_segmentor for AnyEdit's config: ``config`` is accepted for the caller's signature and not read (the
    constructor's defaults are seg_config.py); ``checkpoint``: an mmseg checkpoint whose ``state_dict`` loads strictly."""
    model = UniFormerSegmentor()
    if checkpoint is not None:
        ck = torch.load(checkpoint, map_location="cpu")
        model.load_state_dict(ck.get("state_dict", ck), strict=True)
        meta = ck.get("meta", {}) if isinstance(ck, dict) else {}
        model.CLASSES, model.PALETTE = meta.get("CLASSES"), meta.get("PALETTE")
    return model.to(device).eval()


def inference_segmentor(model, img):
    """mmseg.apis.inference_segmentor on one BGR uint8 image (HWC numpy, as cv2.imread gives): [int64 label map [h, w]]."""
    dev = next(model.parameters()).device
    x = torch.from_numpy(np.ascontiguousarray(rescale(img)))[None].to(dev)
    return [model.labels(x, img.shape[:2])[0].cpu().numpy()]


def show_result_pyplot(model, img, result, palette=None, fig_size=(15, 10), opacity=0.5, title="", block=True):
    """mmseg.apis.show_result_pyplot at opacity 1 (the annotator's only value): show_result paints palette[label] over the image,
    then bgr2rgb -> palette[label], uint8 [h, w, 3].  ``palette`` ([num_classes, 3]) comes from the caller."""
    if opacity != 1:
        raise NotImplementedError("show_result_pyplot: only opacity=1 is implemented (the annotator's value)")
    if palette is None:
        raise ValueError("show_result_pyplot: pass the palette (e.g. get_palette('ade'))")
    pal = np.asarray(palette, dtype=np.uint8)
    seg = np.asarray(result[0])
    if seg.shape != tuple(img.shape[:2]):
        raise ValueError(f"show_result_pyplot: label map {seg.shape} does not match the image {img.shape[:2]}")
    return pal[seg]
