"""AnyDoor's visual-reference edit on the H100 kernels (AnyEdit_Collection/adaptive_editing_pipelines/visual_reference_tool.py):
the pair preparation, the high-frequency collage and the crop-back run in csrc/anydoor.cu, equal to the reference's OpenCV and
numpy arithmetic; the models are the package's ``ControlDenoiser`` (ControlNet + UNet), ``FrozenDinoV2Encoder`` and
``DDIMSampler``.

  ``process_pairs(ref_image, ref_mask, tar_image, tar_mask)``   the reference's dict (numpy in, numpy out; CUDA in, CUDA out)
  ``sobel(img, mask, thresh=50)``                             tools/tool.py sobel (the high-frequency map)
  ``crop_back(pred, tar_image, extra_sizes, tar_box_yyxx_crop)``  the reference's function; the caller's image is left alone
  ``inference_single_image(model, ddim_sampler, ...)``        the reference's request, with an optional fixed ``x_T``
  ``edit_pairs(model, sampler, ref_images, ...)``             B pairs in one DINOv2 call and one sampler run of batch B

The host keeps only the integer box geometry (``pair_geometry``), in the reference's float64 / ``int()`` arithmetic and with its
``np.random`` draws in its order: ``randint(11, 13)`` for the reference's expansion, then ``randint(11, 12)`` and
``randint(15, 30)`` for the two target boxes, pair after pair.  The masks' bounding boxes come from one device reduction; reading
them back is the only synchronisation.  CUDA only.  DESIGN.md §10.8.
"""
from dataclasses import dataclass

import numpy as np
import torch

from . import ops

REF, OUT, P = 224, 512, 18           # P: the geometry row, ANYDOOR_P in include/anysd_b200.h


@dataclass
class PairGeometry:
    ry0: int
    rx0: int
    rh: int
    rw: int
    roy: int
    rox: int
    rs: int
    cy1: int
    cx1: int
    hc: int
    wc: int
    by1: int
    bx1: int
    bh: int
    bw: int
    qy: int
    qx: int
    s2: int

    def row(self):
        return [self.ry0, self.rx0, self.rh, self.rw, self.roy, self.rox, self.rs, self.cy1, self.cx1, self.hc, self.wc,
                self.by1, self.bx1, self.bh, self.bw, self.qy, self.qx, self.s2]

    @property
    def H1(self):
        return self.hc

    @property
    def W1(self):
        return self.wc

    @property
    def H2(self):
        return self.s2

    @property
    def W2(self):
        return self.s2

    @property
    def crop(self):
        return (self.cy1, self.cy1 + self.hc, self.cx1, self.cx1 + self.wc)


def bbox_numpy(mask):
    """(sum, first row, last row, first column, last column) of a mask, as the device reduction gives it."""
    ys, xs = np.nonzero(mask)
    if len(ys) == 0:
        return (0, 0, -1, 0, -1)
    return (int(mask.sum()), int(ys.min()), int(ys.max()), int(xs.min()), int(xs.max()))


def _box(bb, H, W):
    """tool.py get_bbox_from_mask: inclusive last row / column, used by the callers as slice ends; fewer than 10 pixels: all."""
    s, y1, y2, x1, x2 = bb
    return (0, H, 0, W) if s < 10 else (y1, y2, x1, x2)


def _expand(box, lo, hi, H, W):
    """tool.py expand_bbox: the ratio from np.random.randint(lo, hi) / 10, int() truncating toward zero before the clamp."""
    y1, y2, x1, x2 = box
    ratio = np.random.randint(lo, hi) / 10
    xc, yc = 0.5 * (x1 + x2), 0.5 * (y1 + y2)
    h, w = ratio * (y2 - y1 + 1), ratio * (x2 - x1 + 1)
    return max(0, int(yc - h * 0.5)), min(H, int(yc + h * 0.5)), max(0, int(xc - w * 0.5)), min(W, int(xc + w * 0.5))


def _pad_offsets(h, w):
    """tool.py pad_to_square (random=False): (rows before, columns before, side)."""
    p1 = int(abs(h - w) / 2)
    return (0, p1, h) if h > w else ((p1, 0, w) if w > h else (0, 0, h))


def pair_geometry(ref_bb, tar_bb, ref_size, tar_size):
    """The integer geometry of one pair from its masks' bounding boxes (``bbox_numpy`` layout) and the (H, W) of the reference
    and target images, drawing the reference's random numbers in the reference's order."""
    y1, y2, x1, x2 = _box(ref_bb, *ref_size)
    H, W = tar_size
    rh, rw = y2 - y1, x2 - x1
    if rh <= 0 or rw <= 0:
        raise ValueError(f"anydoor: the reference mask's box {(y1, y2, x1, x2)} crops an empty image (the mask spans one row or "
                         "column)")
    ratio = np.random.randint(11, 13) / 10
    eh, ew = int(rh * ratio), int(rw * ratio)
    h1, w1 = int((eh - rh) // 2), int((ew - rw) // 2)
    py, px, rs = _pad_offsets(eh, ew)

    box = _expand(_box(tar_bb, H, W), 11, 12, H, W)
    cy1, cy2, cx1, cx2 = _expand(box, 15, 30, H, W)
    cx, cy = (cx1 + cx2) // 2, (cy1 + cy2) // 2                     # tool.py box2squre
    if cy2 - cy1 >= cx2 - cx1:
        cx1, cx2 = cx - (cy2 - cy1) // 2, cx + (cy2 - cy1) // 2
    else:
        cy1, cy2 = cy - (cx2 - cx1) // 2, cy + (cx2 - cx1) // 2
    cy1, cy2, cx1, cx2 = max(0, cy1), min(H, cy2), max(0, cx1), min(W, cx2)
    hc, wc = cy2 - cy1, cx2 - cx1
    by1, by2, bx1, bx2 = box[0] - cy1, box[1] - cy1, box[2] - cx1, box[3] - cx1
    if not (0 <= by1 < by2 <= hc and 0 <= bx1 < bx2 <= wc):
        raise ValueError(f"anydoor: the target box {box} does not lie inside its crop {(cy1, cy2, cx1, cx2)}")
    qy, qx, s2 = _pad_offsets(hc, wc)
    return PairGeometry(y1, x1, rh, rw, py + h1, px + w1, rs, cy1, cx1, hc, wc, by1, bx1, by2 - by1, bx2 - bx1, qy, qx, s2)


# ---- input handling ----------------------------------------------------------------------------------------------------------
def _require_cuda():
    if not torch.cuda.is_available():
        raise RuntimeError("anydoor runs on CUDA only (no CPU fallback)")


def _dev(x):
    if isinstance(x, np.ndarray):
        return torch.from_numpy(np.ascontiguousarray(x)).cuda()
    if not x.is_cuda:
        raise RuntimeError("anydoor runs on CUDA only (no CPU fallback); move the tensors to the GPU")
    return x.contiguous()


def _check(ref_images, ref_masks, tar_images, tar_masks, batched):
    nd = 4 if batched else 3
    for name, x, want in (("ref_image", ref_images, nd), ("ref_mask", ref_masks, nd - 1), ("tar_image", tar_images, nd),
                          ("tar_mask", tar_masks, nd - 1)):
        if not isinstance(x, (np.ndarray, torch.Tensor)) or x.dtype not in (np.uint8, torch.uint8) or x.ndim != want:
            raise ValueError(f"anydoor: {name} must be a uint8 array with {want} dimensions")
    for img, mask in ((ref_images, ref_masks), (tar_images, tar_masks)):
        shape = tuple(img.shape)
        if shape[-1] != 3 or shape[-3] < 1 or shape[-2] < 1:
            raise ValueError(f"anydoor: images must be [..., H, W, 3] (got {shape})")
        if tuple(mask.shape) != shape[:-1]:
            raise ValueError(f"anydoor: a mask must have its image's H x W (got {tuple(mask.shape)} for {shape})")
    if batched and ref_images.shape[0] != tar_images.shape[0]:
        raise ValueError("anydoor: as many reference images as target images")
    for m in (ref_masks, tar_masks):                  # CUDA masks are checked by the bounding-box reduction
        if isinstance(m, np.ndarray) and m.size and m.max() > 1:
            raise ValueError("anydoor: mask values must be 0 or 1")
    _require_cuda()


def _prepare(ref_images, ref_masks, tar_images, tar_masks):
    """Batched process_pairs on CUDA tensors [B, H, W, 3] / [B, H, W] -> (stage tensors, geometries, device geometry rows)."""
    ref_images, ref_masks, tar_images, tar_masks = (_dev(x) for x in (ref_images, ref_masks, tar_images, tar_masks))
    B = ref_images.shape[0]
    dev = ref_images.device
    bb = torch.empty(2 * B, 6, dtype=torch.int32, device=dev)
    ops.anydoor_bbox(ref_masks, bb[:B])
    ops.anydoor_bbox(tar_masks, bb[B:])
    bb = bb.cpu().tolist()                                          # the one synchronisation
    if max(r[5] for r in bb) > 1:
        raise ValueError("anydoor: mask values must be 0 or 1")
    geoms = [pair_geometry(bb[i][:5], bb[B + i][:5], ref_images.shape[1:3], tar_images.shape[1:3]) for i in range(B)]
    g = torch.tensor([gm.row() for gm in geoms], dtype=torch.int32).to(dev, non_blocking=True)
    u8 = dict(dtype=torch.uint8, device=dev)
    f32 = dict(dtype=torch.float32, device=dev)
    st = {"ref_u8": torch.empty(B, REF, REF, 3, **u8), "mask_u8": torch.empty(B, REF, REF, **u8),
          "img256": torch.empty(B, 256, 256, 3, **u8), "m256": torch.empty(B, 256, 256, **u8),
          "hf256": torch.empty(B, 256, 256, 3, **u8), "hf224": torch.empty(B, REF, REF, 3, **u8),
          "ref": torch.empty(B, REF, REF, 3, **f32), "jpg": torch.empty(B, OUT, OUT, 3, **f32),
          "hint": torch.empty(B, OUT, OUT, 4, **f32)}
    ops.anydoor_prepare(ref_images, ref_masks, tar_images, g, st)
    return st, geoms, g


@torch.no_grad()
def process_pairs(ref_image, ref_mask, tar_image, tar_mask):
    """visual_reference_tool.py process_pairs of one pair: uint8 images [H, W, 3], uint8 0/1 masks [H, W] -> dict(ref, jpg, hint,
    extra_sizes, tar_box_yyxx_crop).  numpy input gives the reference's dtypes (ref float64 = x / 255, jpg / hint float32);
    CUDA tensors give CUDA tensors (ref float32, as the model takes it)."""
    _check(ref_image, ref_mask, tar_image, tar_mask, batched=False)
    st, (g,), _ = _prepare(*(x[None] for x in (ref_image, ref_mask, tar_image, tar_mask)))
    sizes, crop = [g.H1, g.W1, g.H2, g.W2], list(g.crop)
    if isinstance(ref_image, np.ndarray):
        return dict(ref=st["ref_u8"][0].cpu().numpy() / 255, jpg=st["jpg"][0].cpu().numpy(), hint=st["hint"][0].cpu().numpy(),
                    extra_sizes=np.array(sizes), tar_box_yyxx_crop=np.array(crop))
    dev = st["ref"].device
    return dict(ref=st["ref"][0], jpg=st["jpg"][0], hint=st["hint"][0], extra_sizes=torch.tensor(sizes, device=dev),
                tar_box_yyxx_crop=torch.tensor(crop, device=dev))


@torch.no_grad()
def sobel(img, mask, thresh=50):
    """tools/tool.py sobel of the 224 x 224 reference crop: uint8 [224, 224, 3] image and its mask / 255 (float, [224, 224]) ->
    the uint8 high-frequency map [224, 224, 3].  The mask is taken as the uint8 it was divided from (values k / 255)."""
    if not (isinstance(img, (np.ndarray, torch.Tensor)) and img.dtype in (np.uint8, torch.uint8) and tuple(img.shape) == (REF, REF, 3)):
        raise ValueError("anydoor.sobel: expects a uint8 [224, 224, 3] image (the size process_pairs gives it)")
    if tuple(mask.shape) != (REF, REF) or thresh != 50:
        raise ValueError("anydoor.sobel: expects a [224, 224] mask and thresh=50")
    m = np.asarray(mask.cpu() if isinstance(mask, torch.Tensor) else mask, dtype=np.float64)
    mu8 = np.rint(np.clip(m, 0, 1) * 255).astype(np.uint8)
    if not np.array_equal(mu8 / 255, m):
        raise ValueError("anydoor.sobel: mask values must be k / 255 for integers k in [0, 255]")
    _require_cuda()
    x = _dev(img)[None]
    st = {k: torch.empty(s, dtype=torch.uint8, device=x.device) for k, s in
          (("img256", (1, 256, 256, 3)), ("m256", (1, 256, 256)), ("hf256", (1, 256, 256, 3)), ("hf224", (1, REF, REF, 3)))}
    ops.anydoor_sobel(x, torch.from_numpy(mu8)[None].cuda(), st)
    out = st["hf224"][0]
    return out.cpu().numpy() if isinstance(img, np.ndarray) else out


def _crop_row(extra_sizes, box):
    H1, W1, H2, W2 = (int(v) for v in extra_sizes)
    y1, y2, x1, x2 = (int(v) for v in box)
    if H2 != W2 or max(H1, W1) != H2 or y2 - y1 != H1 or x2 - x1 != W1:
        raise ValueError(f"anydoor.crop_back: extra_sizes {extra_sizes} do not fit the crop box {box}")
    qy, qx, _ = _pad_offsets(H1, W1)
    return [0] * 7 + [y1, x1, H1, W1, 0, 0, 0, 0, qy, qx, H2]


@torch.no_grad()
def crop_back(pred, tar_image, extra_sizes, tar_box_yyxx_crop):
    """visual_reference_tool.py crop_back: float32 pred [511, 512, 3] (the decoded image * 127.5 + 127.5, clipped, first row
    dropped) resized to the padded crop, un-padded and pasted into a copy of uint8 tar_image [H, W, 3] with a 5-pixel margin."""
    if not (isinstance(pred, (np.ndarray, torch.Tensor)) and pred.dtype in (np.float32, torch.float32)
            and tuple(pred.shape) == (OUT - 1, OUT, 3)):
        raise ValueError("anydoor.crop_back: pred must be float32 [511, 512, 3]")
    if not (isinstance(tar_image, (np.ndarray, torch.Tensor)) and tar_image.dtype in (np.uint8, torch.uint8)
            and tar_image.ndim == 3 and tar_image.shape[2] == 3):
        raise ValueError("anydoor.crop_back: tar_image must be uint8 [H, W, 3]")
    row = _crop_row(extra_sizes, tar_box_yyxx_crop)
    y1, y2, x1, x2 = (int(v) for v in tar_box_yyxx_crop)
    if y1 < 0 or x1 < 0 or y2 > tar_image.shape[0] or x2 > tar_image.shape[1]:
        raise ValueError("anydoor.crop_back: the crop box leaves the image")
    _require_cuda()
    t = _dev(tar_image)[None]
    out = torch.empty_like(t)
    ops.anydoor_crop_back(_dev(pred)[None], t, torch.tensor([row], dtype=torch.int32, device=t.device), out)
    return out[0].cpu().numpy() if isinstance(tar_image, np.ndarray) else out[0]


# ---- the request -------------------------------------------------------------------------------------------------------------
def _sample(model, sampler, st, steps, guidance_scale, strength, num, x_T, rep):
    """visual_reference_tool.py:194-221 for the prepared pairs, each repeated ``rep`` times -> decoded fp32 [num, 3, 512, 512]."""
    control = st["hint"].permute(0, 3, 1, 2).repeat_interleave(rep, 0).contiguous()
    refs = st["ref"].permute(0, 3, 1, 2).repeat_interleave(rep, 0)
    emb = model.get_learned_conditioning(torch.cat([refs, torch.zeros_like(refs)]).contiguous())   # [ref ; zeros]: one call
    cond = {"c_concat": [control], "c_crossattn": [emb[:num]]}
    un_cond = {"c_concat": [control], "c_crossattn": [emb[num:]]}
    model.control_scales = [strength] * 13
    samples, _ = sampler.sample(steps, num, (4, OUT // 8, OUT // 8), cond, verbose=False, eta=0.0,
                                unconditional_guidance_scale=guidance_scale, unconditional_conditioning=un_cond, x_T=x_T)
    return model.decode_first_stage(samples).float().contiguous()


def _check_x_T(x_T, num):
    if x_T is not None and tuple(x_T.shape) != (num, 4, OUT // 8, OUT // 8):
        raise ValueError(f"anydoor: x_T must be [{num}, 4, {OUT // 8}, {OUT // 8}] (got {tuple(x_T.shape)})")


@torch.no_grad()
def inference_single_image(model, ddim_sampler, ref_image, ref_mask, tar_image, tar_mask, args, x_T=None):
    """visual_reference_tool.py inference_single_image: ``args.num_samples`` copies of the pair, control scales
    ``[args.strength] * 13``, the unconditional context = DINOv2 of zero images, ``args.ddim_steps`` DDIM steps (eta 0) with
    ``args.guidance_scale``; sample 0 is composited back into tar_image.  ``model`` is a ``ControlDenoiser`` whose
    ``cond_stage_model`` is a ``FrozenDinoV2Encoder`` and whose ``first_stage_model`` decodes; ``x_T`` [num_samples, 4, 64, 64]
    fixes the noise (``None``: the sampler draws it)."""
    _check(ref_image, ref_mask, tar_image, tar_mask, batched=False)
    if (args.H, args.W) != (OUT, OUT):
        raise ValueError(f"anydoor: H, W must be {OUT} = 8 x the hint's latent size (got {args.H}, {args.W})")
    num = int(args.num_samples)
    _check_x_T(x_T, num)
    st, _, g = _prepare(*(x[None] for x in (ref_image, ref_mask, tar_image, tar_mask)))
    dec = _sample(model, ddim_sampler, st, args.ddim_steps, args.guidance_scale, args.strength, num, x_T, num)
    t = _dev(tar_image)[None]
    out = torch.empty_like(t)
    ops.anydoor_crop_back(dec[:1], t, g, out)
    return out[0].cpu().numpy() if isinstance(tar_image, np.ndarray) else out[0]


@torch.no_grad()
def edit_pairs(model, sampler, ref_images, ref_masks, tar_images, tar_masks, steps=50, guidance_scale=7.5, strength=1.0, x_T=None):
    """B visual-reference edits at once: uint8 images [B, H, W, 3] and uint8 0/1 masks [B, H, W] (numpy or CUDA; the reference
    images share one size, the target images another) -> the composited uint8 images, the target images' shape.  One DINOv2 call and one sampler run of batch B; pair i equals ``inference_single_image`` of that
    pair with one sample, given the same random boxes and ``x_T[i]``."""
    _check(ref_images, ref_masks, tar_images, tar_masks, batched=True)
    B = ref_images.shape[0]
    _check_x_T(x_T, B)
    st, _, g = _prepare(ref_images, ref_masks, tar_images, tar_masks)
    dec = _sample(model, sampler, st, steps, guidance_scale, strength, B, x_T, 1)
    t = _dev(tar_images)
    out = torch.empty_like(t)
    ops.anydoor_crop_back(dec, t, g, out)
    return out.cpu().numpy() if isinstance(tar_images, np.ndarray) else out
