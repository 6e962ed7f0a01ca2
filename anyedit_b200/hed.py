"""ControlNet's HED edge network on the H100 kernels: the scribble annotator of AnyEdit's ``visual_scribble`` edits
(AnyEdit_Collection/other_modules/HED/__init__.py; built at adaptive_editing_pipelines/visual_condition_tool.py:183-188).

  ``ControlNetHED_Apache2``   the reference's parameter tree (``norm``, ``block{1..5}.convs.{i}``, ``block{1..5}.projection``:
                              37 tensors), so ``ControlNetHED.pth`` loads with ``load_state_dict(..., strict=True)``.  ``forward(img)``:
                              uint8 images [B, H, W, 3] on the GPU, channels as ``cv2.imread`` gives them (BGR, fed as is, as the
                              reference does) -> the five fp32 side maps [B, 1, h, w].
  ``HEDdetector(path)``       the reference's detector: ``__call__(image_path, output_path)`` and the batched ``detect(images)``.

Launch plan (DESIGN.md §10.6); activations are NHWC fp16 token rows, every step a library kernel:
  input        hed_input: K = 32 im2col rows fp16(s (x - norm)) of the uint8 image, zero-padded after the subtraction
  block1       convs.0 as one dense K = 32 contraction + bias + ReLU; convs.1 as a 3x3 conv + bias + ReLU
  block2..5    max_pool2 (2x2, stride 2, floor), then each conv as a 3x3 conv + bias + ReLU
  projections  1x1 conv C -> 1 as a contraction onto weight rows zero-padded to 8, fp32 out (column 0 is the side map)
  edges        hed_edges: cv2's INTER_LINEAR resize of each side map, the mean, the fp64 sigmoid and the inversion, per pixel
The network has no normalisation layer, so its fp16 activations carry a fixed power-of-two scale S: convs, ReLU and max-pool are
positively homogeneous once every bias is scaled too, so S goes into the input kernel and every conv bias, and 1 / S into the
projection weights, which puts the fp32 side maps back at their true scale.  Exact up to fp16 subnormals.  CUDA only.
"""
import numpy as np
import torch
import torch.nn as nn

from . import ops
from .encoders import _Packable

# Scale of the fp16 activations: the input is 0..255 minus ``norm``.  Not fitted to the released checkpoint's activation range
# (DESIGN.md §10.6).
S = 2.0 ** -8
MIN_SIDE = 16                                        # four 2x2 pools leave block 5 at least one pixel


class _DoubleConvBlock(nn.Module):
    def __init__(self, cin, cout, n):
        super().__init__()
        self.convs = nn.Sequential(*[nn.Conv2d(cin if i == 0 else cout, cout, 3, padding=1) for i in range(n)])
        self.projection = nn.Conv2d(cout, 1, 1)


class ControlNetHED_Apache2(_Packable):
    """HED/__init__.py ControlNetHED_Apache2 on the kernels.  ``forward(img)``: uint8 [B, H, W, 3] on the GPU (both sides >= 16)
    -> tuple of the five side maps, fp32 [B, 1, H >> k, W >> k] (floored at each pool)."""

    def __init__(self):
        super().__init__()
        self.norm = nn.Parameter(torch.zeros(1, 3, 1, 1))
        for b, (cin, cout, n) in enumerate(((3, 64, 2), (64, 128, 2), (128, 256, 3), (256, 512, 3), (512, 512, 3)), 1):
            setattr(self, f"block{b}", _DoubleConvBlock(cin, cout, n))
        self.eval()

    def _build_pack(self, dev):
        f64 = dict(device=dev, dtype=torch.float64)
        blocks = []
        for b in range(1, 6):
            blk = getattr(self, f"block{b}")
            convs = []
            for conv in blk.convs:
                w = conv.weight.detach().to(**f64).permute(0, 2, 3, 1).reshape(conv.weight.shape[0], -1)     # [co, (ky, kx, ci)]
                if w.shape[1] == 27:                                                  # block1.convs.0: K = 32
                    w = torch.nn.functional.pad(w, (0, 5))
                convs.append((w.half().contiguous(), (conv.bias.detach().to(**f64) * S).float().contiguous()))
            p = blk.projection
            wp = torch.zeros(8, p.weight.shape[1], **f64)
            wp[0] = p.weight.detach().to(**f64).reshape(-1) / S
            bp = torch.zeros(8, device=dev, dtype=torch.float32)
            bp[0] = p.bias.detach().to(dev, torch.float32)[0]
            if not bool(wp.abs().max() < 65504):
                raise ValueError(f"ControlNetHED_Apache2: block{b}.projection weights exceed the fp16 range once scaled by 1 / S")
            blocks.append({"convs": convs, "proj": (wp.half().contiguous(), bp)})
        return {"norm": self.norm.detach().to(dev, torch.float32).reshape(3).contiguous(), "blocks": blocks}

    def _check(self, img):
        if not (isinstance(img, torch.Tensor) and img.dtype == torch.uint8 and img.dim() == 4 and img.shape[3] == 3):
            raise ValueError("ControlNetHED_Apache2: expects uint8 images [B, H, W, 3]")
        if min(img.shape[1], img.shape[2]) < MIN_SIDE:
            raise ValueError(f"ControlNetHED_Apache2: image {tuple(img.shape[1:3])} has a side shorter than {MIN_SIDE} (the fifth "
                             f"max-pool would be empty)")
        P = self._packed()
        if not img.is_cuda:
            raise RuntimeError("ControlNetHED_Apache2 runs on CUDA only (no CPU fallback); move the image to the model's device")
        return P, img.contiguous()

    def _sides(self, img, P):
        """The five side maps as fp32 [B, h, w, 8] buffers (column 0 is the map, the rest are zero)."""
        B, H, W, _ = img.shape
        dev = img.device
        cols = torch.empty(B * H * W, 32, dtype=torch.float16, device=dev)
        ops.hed_input(img, P["norm"], cols, S)
        x, sides = None, []
        for b, blk in enumerate(P["blocks"]):
            if b > 0:
                y = torch.empty(B, x.shape[1] // 2, x.shape[2] // 2, x.shape[3], dtype=torch.float16, device=dev)
                ops.max_pool2(x, y)
                x = y
            for i, (w, bias) in enumerate(blk["convs"]):
                h, wd = (H, W) if x is None else x.shape[1:3]
                y = torch.empty(B, h, wd, w.shape[0], dtype=torch.float16, device=dev)
                if x is None:
                    ops.gemm(cols, w, y.view(-1, w.shape[0]), bias=bias, act=6)
                else:
                    ops.conv3x3(x, w, y.view(-1, w.shape[0]), bias=bias, act=6)
                x = y
            wp, bp = blk["proj"]
            d = torch.empty(*x.shape[:3], 8, dtype=torch.float32, device=dev)
            ops.gemm(x.view(-1, x.shape[3]), wp, d.view(-1, 8), bias=bp)
            sides.append(d)
        return sides

    @torch.no_grad()
    def forward(self, img):
        P, img = self._check(img)
        return tuple(d.permute(0, 3, 1, 2)[:, :1] for d in self._sides(img, P))

    @torch.no_grad()
    def edge_map(self, img):
        """HEDdetector's uint8 edge map [B, H, W] of uint8 images [B, H, W, 3] on the GPU."""
        P, img = self._check(img)
        sides = self._sides(img, P)
        out = torch.empty(img.shape[:3], dtype=torch.uint8, device=img.device)
        ops.hed_edges([d[..., 0] for d in sides], out)
        return out


class HEDdetector:
    """HED/__init__.py HEDdetector: ``path`` is the ``ControlNetHED.pth`` state dict, loaded strictly."""

    def __init__(self, path):
        self.netNetwork = ControlNetHED_Apache2().float().cuda().eval()
        self.netNetwork.load_state_dict(torch.load(path, map_location="cpu"), strict=True)

    def detect(self, images):
        """uint8 [B, H, W, 3] (numpy, or a CUDA tensor) of same-size images -> the uint8 edge maps [B, H, W], numpy for numpy input
        and a CUDA tensor for a tensor."""
        if isinstance(images, np.ndarray):
            x = torch.from_numpy(np.ascontiguousarray(images)).to(next(self.netNetwork.parameters()).device)
            return self.netNetwork.edge_map(x).cpu().numpy()
        return self.netNetwork.edge_map(images)

    def __call__(self, image_path, output_path):
        import cv2
        input_image = cv2.imread(image_path)
        assert input_image.ndim == 3
        cv2.imwrite(output_path, self.detect(input_image[None])[0])
