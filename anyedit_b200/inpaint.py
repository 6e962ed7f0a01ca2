"""AnyEdit's inpainting edits on the kernels: ``background_change`` and the second stage of ``replace``
(AnyEdit_Collection/adaptive_editing_pipelines/local_pipeline_tool.py:440-450, 482-522), which run diffusers'
``StableDiffusionInpaintPipeline`` on the ``sd-inpaint`` checkpoint: ldm's ``LatentInpaintDiffusion``, a UNet of 9 input
channels (the latent, the latent-sized mask, the masked image's latent).

  ``background_mask(fore_bgr)``                     the tool's mask post-processing of the foreground mask it reads back with
                                                    ``cv2.imread``: GaussianBlur((5, 5), 0), BGR2GRAY, == 0 -> bool masks and
                                                    their pixel counts
  ``prepare(images, masks)``                        the pipeline's image and mask processors and its conditioning: Pillow's
                                                    LANCZOS resize to 512^2 of the image, of a mode "L" mask (uint8) or NEAREST
                                                    of a mode "1" mask (bool), binarisation, the masked image as the encoder's
                                                    input rows, the 64^2 mask latent
  ``inpaint_latents(model, sampler, ...)``          B requests of any sizes in one sampler run of batch B -> final latents
  ``inpaint(model, sampler, ...)``                  the same, decoded, post-processed and resized back with LANCZOS
  ``background_change(model, sampler, ...)``        the tool's steps 1-5 for B requests, ``None`` for the skipped ones

Every byte-level step is a kernel of ``csrc/inpaint.cu`` equal to Pillow / OpenCV on every byte; the model is the package's
UNet, ``AutoencoderKL`` and ``PLMSSampler``.  Prompts come in as text embeddings (there is no tokenizer here).  The mask and
masked-image latents are the same tensors in both CFG halves, so the sampler runs the UNet's shared-halves path.  Reading the
coverage counts back is the only synchronisation before sampling.  CUDA only.  DESIGN.md §10.11.
"""
import numpy as np
import torch

from . import ops

SIZE = 512                   # StableDiffusionInpaintPipeline: height = width = unet.sample_size * vae_scale_factor
MIN_COVERAGE = 0.05          # local_pipeline_tool.py:510: skip a background mask under 5 % of the image


def _require_cuda():
    if not torch.cuda.is_available():
        raise RuntimeError("anyedit_b200.inpaint runs on CUDA only (no CPU fallback)")


def _dev(x):
    if isinstance(x, np.ndarray):
        return torch.from_numpy(np.ascontiguousarray(x)).cuda()
    if not x.is_cuda:
        raise RuntimeError("anyedit_b200.inpaint runs on CUDA only (no CPU fallback); move the tensors to the GPU")
    return x.contiguous()


def _images(images, what, channels=3):
    if not isinstance(images, (list, tuple)) or not images:
        raise ValueError(f"{what}: a non-empty list of images")
    for im in images:
        if not isinstance(im, (np.ndarray, torch.Tensor)) or im.dtype not in (np.uint8, torch.uint8) or im.ndim != 3 \
                or im.shape[2] != channels or im.shape[0] < 1 or im.shape[1] < 1:
            raise ValueError(f"{what}: images are uint8 [H, W, {channels}] arrays or tensors")
    _require_cuda()
    return [_dev(im) for im in images]


def _masks(masks, B):
    if not isinstance(masks, (list, tuple)) or len(masks) != B:
        raise ValueError(f"prepare: one mask per image ({B})")
    out, filters = [], []
    for m in masks:
        if not isinstance(m, (np.ndarray, torch.Tensor)) or m.ndim != 2 or m.shape[0] < 1 or m.shape[1] < 1:
            raise ValueError("prepare: masks are [H, W] arrays or tensors")
        if m.dtype in (np.bool_, torch.bool):             # a mode "1" image: Pillow resizes it NEAREST
            out.append(_dev(m).view(torch.uint8))
            filters.append("mode1")
        elif m.dtype in (np.uint8, torch.uint8):         # a mode "L" image: LANCZOS, ringing included
            out.append(_dev(m))
            filters.append("lanczos")
        else:
            raise ValueError("prepare: a mask is bool (mode \"1\") or uint8 (mode \"L\")")
    return out, filters


@torch.no_grad()
def background_mask(fore_bgr):
    """local_pipeline_tool.py:494-499 for B foreground masks: BGR uint8 [H, W, 3] (``cv2.imread`` of the saved ``fore | face``
    mask; any sizes) -> (bool CUDA masks [H, W]: ``cvtColor(GaussianBlur(m, (5, 5), 0), BGR2GRAY) == 0``, int64 CPU tensor of
    their True counts).  One launch; reading the counts back is the synchronisation."""
    imgs = _images(fore_bgr, "background_mask")
    outs = [torch.empty(im.shape[:2], dtype=torch.uint8, device=im.device) for im in imgs]
    counts = torch.empty(len(imgs), dtype=torch.int32, device=imgs[0].device)
    ops.background_mask(imgs, outs, counts)
    return [o.view(torch.bool) for o in outs], counts.cpu().long()


@torch.no_grad()
def prepare(images, masks, size=SIZE, row_channels=64):
    """The inpaint pipeline's processors for B requests (diffusers VaeImageProcessor + prepare_mask_latents, strength 1):
    uint8 RGB images [H, W, 3] and masks [h, w] (bool: mode "1", NEAREST; uint8: mode "L", LANCZOS), each of any size ->
    dict of CUDA tensors:
      image     uint8 [B, size, size, 3]  Image.resize((size, size), LANCZOS)
      mask      uint8 [B, size, size]     the mask's resize, then convert("L")
      masked    fp16 [B, size, size, row_channels]  (x / 255 * 2 - 1) * (mask < 128) in float32, zero channels after 3: the
                                                    encoder's input rows (``AutoencoderKL.encode_rows``)
      mask_latent  fp32 [B, 1, size / 8, size / 8]  mask[8i, 8j] >= 128 (F.interpolate, nearest)
      counts    int32 [B]                 mask bytes >= 128
    Three launches: the images' resize, the masks' resize, the conditioning."""
    imgs = _images(images, "prepare")
    B = len(imgs)
    ms, filters = _masks(masks, B)
    if size % 8 or size < 8:
        raise ValueError(f"prepare: size {size} is not a positive multiple of 8")
    dev = imgs[0].device
    st = {"image": torch.empty(B, size, size, 3, dtype=torch.uint8, device=dev),
          "mask": torch.empty(B, size, size, dtype=torch.uint8, device=dev),
          "masked": torch.empty(B, size, size, row_channels, dtype=torch.float16, device=dev),
          "mask_latent": torch.empty(B, 1, size // 8, size // 8, dtype=torch.float32, device=dev),
          "counts": torch.empty(B, dtype=torch.int32, device=dev)}
    ops.pil_resize(imgs, list(st["image"]), ["lanczos"] * B)
    ops.pil_resize([m[..., None] for m in ms], [m[..., None] for m in st["mask"]], filters)
    ops.inpaint_prepare(st["image"], st["mask"], st["masked"], st["mask_latent"], st["counts"])
    return st


def _embeddings(cond, uncond, B, dev):
    if not (isinstance(cond, torch.Tensor) and cond.dim() == 3 and cond.shape[0] == B):
        raise ValueError(f"inpaint: cond must be [B = {B}, L, D] text embeddings, got {tuple(getattr(cond, 'shape', ()))}")
    L, D = cond.shape[1:]
    if not (isinstance(uncond, torch.Tensor) and tuple(uncond.shape) in ((L, D), (B, L, D))):
        raise ValueError(f"inpaint: uncond must be [L, D] or [B, L, D] = {(B, L, D)}, got {tuple(getattr(uncond, 'shape', ()))}")
    uc = uncond.to(dev).expand(B, L, D) if uncond.dim() == 2 else uncond.to(dev)
    return cond.to(dev).contiguous(), uc.contiguous()


@torch.no_grad()
def inpaint_latents(model, sampler, images, masks, cond, uncond, steps=50, guidance_scale=7.5, x_T=None, posterior_noise=None,
                    size=SIZE):
    """StableDiffusionInpaintPipeline.__call__ up to the final latents for B requests in one sampler run of batch B.
    ``model``: a ``LatentInpaintDenoiser`` (or any hybrid ``LatentDenoiser`` with a 9-channel UNet) with ``first_stage_model``
    and ``scale_factor``; ``sampler``: its ``PLMSSampler`` (the pipeline's PNDM with skip_prk_steps, DESIGN.md §10.11);
    ``cond`` [B, L, D] the prompts' embeddings, ``uncond`` [L, D] or [B, L, D] the negative prompt's; ``x_T`` [B, 4, h, w]
    the start latents and ``posterior_noise`` [B, 4, h, w] the masked image's posterior draw (default: ``randn``).
    -> fp32 [B, 4, size / 8, size / 8].  Request i equals the single request with ``x_T[i]`` and ``posterior_noise[i]``."""
    if not isinstance(images, (list, tuple)) or not images:
        raise ValueError("inpaint: a non-empty list of images")
    B = len(images)
    h = size // 8
    dev = model.device
    c, uc = _embeddings(cond, uncond, B, dev)
    for name, t in (("x_T", x_T), ("posterior_noise", posterior_noise)):
        if t is not None and tuple(t.shape) != (B, 4, h, h):
            raise ValueError(f"inpaint: {name} must be [{B}, 4, {h}, {h}], got {tuple(t.shape)}")
    vae = model.first_stage_model
    st = prepare(images, masks, size, vae.input_row_channels)
    masked_latents = model.get_first_stage_encoding(vae.encode_rows(st["masked"]), noise=posterior_noise)
    c_concat = torch.cat([st["mask_latent"], masked_latents], 1)       # concat_keys = ("mask", "masked_image")
    cfg = guidance_scale != 1.0
    cond_d = {"c_concat": [c_concat], "c_crossattn": [c]}
    uncond_d = {"c_concat": [c_concat], "c_crossattn": [uc]}          # the same tensor: the CFG halves share the prefix
    if x_T is None:
        x_T = torch.randn(B, 4, h, h, device=dev)
    lat, _ = sampler.sample(steps, B, (4, h, h), cond_d, verbose=False, x_T=x_T.to(dev, torch.float32), eta=0.0,
                            unconditional_guidance_scale=guidance_scale, unconditional_conditioning=uncond_d if cfg else None)
    return lat


@torch.no_grad()
def inpaint(model, sampler, images, masks, cond, uncond, steps=50, guidance_scale=7.5, x_T=None, posterior_noise=None,
            out_sizes=None, size=SIZE):
    """``inpaint_latents``, then ``decode_first_stage``, round(clamp(x / 2 + 1/2, 0, 1) * 255) and Image.resize(out_size,
    LANCZOS) of every request -> list of uint8 [H, W, 3] at ``out_sizes`` ((H, W) per request; default: the images' sizes),
    numpy for numpy images, CUDA tensors otherwise.  A 9-channel UNet gets no paste-back."""
    lat = inpaint_latents(model, sampler, images, masks, cond, uncond, steps, guidance_scale, x_T, posterior_noise, size)
    B = lat.shape[0]
    if out_sizes is None:
        out_sizes = [tuple(im.shape[:2]) for im in images]
    if len(out_sizes) != B:
        raise ValueError(f"inpaint: one out size per request ({B})")
    dec = model.decode_first_stage(lat).float().contiguous()
    u8 = torch.empty(B, size, size, 3, dtype=torch.uint8, device=dec.device)
    ops.image_to_u8(dec, u8)
    outs = [torch.empty(int(hh), int(ww), 3, dtype=torch.uint8, device=dec.device) for hh, ww in out_sizes]
    ops.pil_resize(list(u8), outs, ["lanczos"] * B)
    return [o.cpu().numpy() for o in outs] if isinstance(images[0], np.ndarray) else outs


@torch.no_grad()
def background_change(model, sampler, images, fore_bgr, cond, uncond, steps=50, guidance_scale=7.5, x_T=None, posterior_noise=None,
                      size=SIZE):
    """local_pipeline_tool.py:482-522 after GroundingDINO + SAM, for B requests: RGB uint8 images [H, W, 3] and the BGR
    foreground masks read back from JPEG at the same sizes; ``cond`` [B, L, D] the new backgrounds' embeddings, ``uncond`` the
    fixed negative prompt's.  -> list of B entries: ``None`` where the background covers under 5 % of the image (the tool
    skips the request), else (edited uint8 [H, W, 3] at the original size, the bool background mask [H, W]).  The kept
    requests run in one sampler run; request i equals its single run given ``x_T[i]`` and ``posterior_noise[i]``."""
    masks, counts = background_mask(fore_bgr)
    if len(images) != len(masks):
        raise ValueError("background_change: one foreground mask per image")
    keep = [i for i, m in enumerate(masks) if not int(counts[i]) / m.numel() < MIN_COVERAGE]
    out = [None] * len(masks)
    if not keep:
        return out
    pick = lambda t: None if t is None else t[keep]
    ks = torch.tensor(keep)
    uc = uncond if uncond.dim() == 2 else uncond[ks.to(uncond.device)]
    edited = inpaint(model, sampler, [images[i] for i in keep], [masks[i] for i in keep], cond[ks.to(cond.device)], uc, steps,
                     guidance_scale, pick(x_T), pick(posterior_noise), size=size)
    numpy_out = isinstance(images[0], np.ndarray)
    for j, i in enumerate(keep):
        out[i] = (edited[j], masks[i].cpu().numpy() if numpy_out else masks[i])
    return out
