"""Depth Anything V2 on the H100 kernels: the depth annotator of AnyEdit's ``visual_depth`` edits
(AnyEdit_Collection/adaptive_editing_pipelines/visual_condition_tool.py:111-135, 190-195, 290).

  ``DepthAnythingV2``   other_modules/depth_anything_v2/dpt.py:153-221: a DINOv2 ViT (``encoders.Dinov2Model``, ``pretrained.*``
                        in the hub's names) read at four intermediate blocks, and the DPT head (``depth_head.*``, dpt.py:40-150,
                        util/blocks.py).  The parameter tree is the reference's (407 tensors for vitl), so the released
                        checkpoint loads with ``load_state_dict`` unchanged.

Launch plan of the head (DESIGN.md §10.4); every step is a library kernel, activations NHWC fp16:
  projects[i]         one contraction on the normed patch rows [B*gh*gw, D] (1x1 conv)
  resize_layers[0/1]  ConvTranspose2d(k = stride = 4 / 2) = a contraction with the weight packed [(ky, kx, co), ci] and the
                      bias repeated r^2 times, then ``depth_to_space``; [2] identity; [3] the stride-2 3x3 conv
  layer{k}_rn         3x3 conv, no bias
  ResidualConvUnit    ``relu`` copy -> 3x3 conv + ReLU epilogue -> 3x3 conv with the unit's input as residual
  FeatureFusionBlock  out_conv (1x1) runs BEFORE the bilinear upsample: both are linear and every output's bilinear weights sum
                      to 1, so they commute (bias included) and the 1x1 conv runs on 4x fewer pixels.  The resize kernel adds
                      the next level's layer_rn as its addend: ``path + layer_rn`` is the residual of the next block's
                      resConfUnit1.conv2, so ``path + RCU1(layer_rn)`` comes out of that conv's epilogue.
  output_conv1 at 2x the finest level, resize to 14 (gh, gw), 3x3 conv + ReLU, 1x1 conv 32 -> 1 + ReLU (weight rows zero-padded
  to 8, fp32 output; the first channel is read out by ``nhwc_to_nchw``).
``use_bn`` / ``use_clstoken`` (no AnyEdit caller, no released V2 checkpoint) raise.  CUDA only, no CPU fallback.
"""
import numpy as np
import torch
import torch.nn as nn

from . import ops
from .encoders import DINOV2_CONFIGS, IMAGENET_MEAN, IMAGENET_STD, Dinov2Model, _Packable
from .unet import _Param, _f, _h, _pack_conv3

INTERMEDIATE_LAYER_IDX = {"vits": [2, 5, 8, 11], "vitb": [2, 5, 8, 11], "vitl": [4, 11, 17, 23], "vitg": [9, 19, 29, 39]}


class _RCU(nn.Module):
    """util/blocks.py ResidualConvUnit (bn=False)."""

    def __init__(self, f):
        super().__init__()
        self.conv1, self.conv2 = _Param((f, f, 3, 3), kind="conv"), _Param((f, f, 3, 3), kind="conv")


class _Fusion(nn.Module):
    """util/blocks.py FeatureFusionBlock (expand=False, align_corners=True)."""

    def __init__(self, f):
        super().__init__()
        self.out_conv = _Param((f, f, 1, 1), kind="conv")
        self.resConfUnit1, self.resConfUnit2 = _RCU(f), _RCU(f)


class _DPTHead(nn.Module):
    """dpt.py DPTHead parameter holder (use_bn=False, use_clstoken=False)."""

    def __init__(self, in_channels, features, out_channels):
        super().__init__()
        oc = out_channels
        self.projects = nn.ModuleList([_Param((c, in_channels, 1, 1), kind="conv") for c in oc])
        self.resize_layers = nn.ModuleList([_Param((oc[0], oc[0], 4, 4), kind="conv"), _Param((oc[1], oc[1], 2, 2), kind="conv"),
                                            nn.Identity(), _Param((oc[3], oc[3], 3, 3), kind="conv")])
        s = self.scratch = nn.Module()
        for k in range(4):
            setattr(s, f"layer{k + 1}_rn", _Param((features, oc[k], 3, 3), bias=False, kind="conv"))
        for k in range(4):
            setattr(s, f"refinenet{k + 1}", _Fusion(features))
        s.output_conv1 = _Param((features // 2, features, 3, 3), kind="conv")
        s.output_conv2 = nn.Sequential(_Param((32, features // 2, 3, 3), kind="conv"), nn.Identity(), _Param((1, 32, 1, 1), kind="conv"),
                                       nn.Identity(), nn.Identity())


def _pack_1x1(p, dev):
    return _h(p.weight.reshape(p.weight.shape[0], -1), dev), _f(p.bias, dev)


def _pack_deconv(p, dev):
    """ConvTranspose2d weight [ci, co, r, r] -> [(ky, kx, co), ci] fp16, bias repeated r^2 times."""
    ci, co, r, _ = p.weight.shape
    w = p.weight.detach().to(dev).float().permute(2, 3, 1, 0).reshape(r * r * co, ci)
    return w.half().contiguous(), _f(p.bias, dev).repeat(r * r).contiguous(), r


class DepthAnythingV2(_Packable):
    """dpt.py:153-221.  ``forward(x)`` (x [B, 3, H, W], normalised, H and W multiples of 14) -> fp32 depth [B, H, W];
    ``infer_image(raw_image, input_size=518)`` -> numpy [h, w] for a BGR uint8 image; ``image2tensor`` as the reference.
    ``config`` (dict, optional): overrides of the backbone's ``Dinov2Model`` configuration; ``layer_idx``: the blocks the head
    reads (default: the reference's ``intermediate_layer_idx[encoder]``)."""

    def __init__(self, encoder="vitl", features=256, out_channels=(256, 512, 1024, 1024), use_bn=False, use_clstoken=False,
                 config=None, layer_idx=None):
        super().__init__()
        if use_bn or use_clstoken:
            raise NotImplementedError("DepthAnythingV2: use_bn / use_clstoken are not implemented (no AnyEdit caller or released "
                                      "V2 checkpoint uses them)")
        if encoder not in DINOV2_CONFIGS:
            raise ValueError(f"encoder must be one of {sorted(DINOV2_CONFIGS)}, got {encoder!r}")
        self.encoder = encoder
        self.layer_idx = list(layer_idx if layer_idx is not None else INTERMEDIATE_LAYER_IDX[encoder])
        cfg = dict(DINOV2_CONFIGS[encoder], image_size=518, patch_size=14)
        cfg.update(config or {})
        self.pretrained = Dinov2Model(cfg, interpolate_offset=0.1)
        self.depth_head = _DPTHead(self.pretrained.config.hidden_size, features, list(out_channels))

    def _build_pack(self, dev):
        h, s = self.depth_head, self.depth_head.scratch
        o2a, o2b = s.output_conv2[0], s.output_conv2[2]
        wb = torch.zeros(8, o2b.weight.shape[1], device=dev)
        wb[:1] = o2b.weight.detach().to(dev).float().reshape(1, -1)
        bb = torch.zeros(8, device=dev)
        bb[:1] = o2b.bias.detach().to(dev).float()
        fus = []
        for k in range(4):
            r = getattr(s, f"refinenet{k + 1}")
            rcu = lambda u: (_pack_conv3(u.conv1.weight, dev), _f(u.conv1.bias, dev), _pack_conv3(u.conv2.weight, dev), _f(u.conv2.bias, dev))
            fus.append({"out": _pack_1x1(r.out_conv, dev), "rcu1": rcu(r.resConfUnit1), "rcu2": rcu(r.resConfUnit2)})
        return {"proj": [_pack_1x1(p, dev) for p in h.projects],
                "deconv": [_pack_deconv(h.resize_layers[0], dev), _pack_deconv(h.resize_layers[1], dev)],
                "down": (_pack_conv3(h.resize_layers[3].weight, dev), _f(h.resize_layers[3].bias, dev)),
                "rn": [_pack_conv3(getattr(s, f"layer{k + 1}_rn").weight, dev) for k in range(4)], "fusion": fus,
                "oc1": (_pack_conv3(s.output_conv1.weight, dev), _f(s.output_conv1.bias, dev)),
                "oc2a": (_pack_conv3(o2a.weight, dev), _f(o2a.bias, dev)), "oc2b": (wb.half().contiguous(), bb)}

    @staticmethod
    def _rcu(x, w, residual):
        """ResidualConvUnit's convs on NHWC x: conv2(relu(conv1(relu(x)))) + residual."""
        B, H, W, F = x.shape
        t = torch.empty_like(x)
        ops.relu(x, t)
        u = torch.empty_like(x)
        ops.conv3x3(t, w[0], u.view(-1, F), bias=w[1], act=6)
        out = torch.empty_like(x)
        ops.conv3x3(u, w[2], out.view(-1, F), bias=w[3], residual=residual.view(-1, F))
        return out

    @torch.no_grad()
    def forward(self, x):
        P = self._packed()
        tokens, B, gh, gw = self.pretrained.intermediate_patches(x, self.layer_idx)
        dev = tokens[0].device
        f16 = dict(dtype=torch.float16, device=dev)
        M = B * gh * gw
        layers = []
        for i, t in enumerate(tokens):                         # projects + resize_layers (dpt.py:117-131)
            w, b = P["proj"][i]
            y = torch.empty(B, gh, gw, w.shape[0], **f16)
            ops.gemm(t, w, y.view(M, -1), bias=b)
            if i < 2:
                wd, bd, r = P["deconv"][i]
                g = torch.empty(M, wd.shape[0], **f16)
                ops.gemm(y.view(M, -1), wd, g, bias=bd)
                y = torch.empty(B, gh * r, gw * r, wd.shape[1], **f16)
                ops.depth_to_space(g, y, r)
            elif i == 3:
                wc, bc = P["down"]
                Ho, Wo = (gh - 1) // 2 + 1, (gw - 1) // 2 + 1
                z = torch.empty(B, Ho, Wo, wc.shape[0], **f16)
                ops.conv3x3(y, wc, z.view(-1, wc.shape[0]), bias=bc, stride=2)
                y = z
            layers.append(y)
        rn = []
        for k, y in enumerate(layers):                         # scratch.layer{k}_rn
            w = P["rn"][k]
            z = torch.empty(*y.shape[:3], w.shape[0], **f16)
            ops.conv3x3(y, w, z.view(-1, w.shape[0]))
            rn.append(z)
        F = rn[0].shape[-1]
        path = None                                            # refinenet4 .. refinenet1 (dpt.py:140-143)
        for k in (3, 2, 1, 0):
            fz = P["fusion"][k]
            # path already holds upsample(previous) + layer_rn (the resize addend) = the residual of resConfUnit1.conv2
            h = rn[k] if path is None else self._rcu(rn[k], fz["rcu1"], path)
            h = self._rcu(h, fz["rcu2"], h)
            o = torch.empty_like(h)
            ops.gemm(h.view(-1, F), fz["out"][0], o.view(-1, F), bias=fz["out"][1])
            H, W = h.shape[1:3]
            size = rn[k - 1].shape[1:3] if k > 0 else (2 * H, 2 * W)
            path = torch.empty(B, size[0], size[1], F, **f16)
            ops.resize_bilinear(o, path, addend=rn[k - 1] if k > 0 else None)
        w1, b1 = P["oc1"]
        c1 = torch.empty(*path.shape[:3], w1.shape[0], **f16)
        ops.conv3x3(path, w1, c1.view(-1, w1.shape[0]), bias=b1)
        Ho, Wo = 14 * gh, 14 * gw
        up = torch.empty(B, Ho, Wo, c1.shape[-1], **f16)
        ops.resize_bilinear(c1, up)
        wa, ba = P["oc2a"]
        c2 = torch.empty(B, Ho, Wo, wa.shape[0], **f16)
        ops.conv3x3(up, wa, c2.view(-1, wa.shape[0]), bias=ba, act=6)
        wb, bb = P["oc2b"]
        d8 = torch.empty(B, Ho, Wo, 8, dtype=torch.float32, device=dev)
        ops.gemm(c2.view(-1, wa.shape[0]), wb, d8.view(-1, 8), bias=bb, act=6)
        depth = torch.empty(B, 1, Ho, Wo, dtype=torch.float32, device=dev)
        ops.nhwc_to_nchw(d8, depth)
        return depth.view(B, Ho, Wo)

    @torch.no_grad()
    def infer_image(self, raw_image, input_size=518):
        image, (h, w) = self.image2tensor(raw_image, input_size)
        depth = self.forward(image)
        out = torch.empty(depth.shape[0], h, w, dtype=torch.float32, device=depth.device)
        ops.resize_bilinear(depth, out)
        return out[0].cpu().numpy()

    def image2tensor(self, raw_image, input_size=518):
        """dpt.py:202-221 on the host: BGR -> RGB in [0, 1], aspect-keeping resize to at least ``input_size`` on both sides with
        multiples of 14 (bicubic), ImageNet normalisation -> (fp32 [1, 3, H', W'] on the model's device, (h, w))."""
        import cv2
        h, w = raw_image.shape[:2]
        image = cv2.cvtColor(raw_image, cv2.COLOR_BGR2RGB) / 255.0
        nw, nh = _lower_bound_size(w, h, input_size, 14)
        image = cv2.resize(image, (nw, nh), interpolation=cv2.INTER_CUBIC)
        image = (image - np.array(IMAGENET_MEAN)) / np.array(IMAGENET_STD)
        image = np.ascontiguousarray(np.transpose(image, (2, 0, 1))).astype(np.float32)
        dev = next(self.parameters()).device
        return torch.from_numpy(image).unsqueeze(0).to(dev), (h, w)


def _lower_bound_size(width, height, size, multiple):
    """util/transform.py Resize.get_size with keep_aspect_ratio=True, resize_method="lower_bound" -> (new_width, new_height)."""
    sh, sw = size / height, size / width
    if sw > sh:
        sh = sw
    else:
        sw = sh

    def fit(x):
        y = (np.round(x / multiple) * multiple).astype(int)
        if y < size:
            y = (np.ceil(x / multiple) * multiple).astype(int)
        return int(y)
    return fit(sw * width), fit(sh * height)
