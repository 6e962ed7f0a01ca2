#!/usr/bin/env python
"""Golden vectors of the SD inpainting model (AnyEdit's background_change / replace), from the reference's own modules on CPU.

Run in the build container only (needs the reference checkout):

    python tests/golden/make_golden_inpaint.py

Two requests of different sizes, one with a mode "1" (bool) mask and one with a mode "L" (uint8, JPEG round-tripped) mask,
go through diffusers' processors written with live Pillow and numpy (resize LANCZOS, x / 255 * 2 - 1; the mask resized, then
convert("L"), / 255, binarised; masked image = image * (mask < 0.5); mask latent = nearest to size / 8).  The masked image is
encoded by the reference's ``Encoder`` + quant_conv (ldm/modules/diffusionmodules/model.py) and drawn from its
``DiagonalGaussianDistribution`` with stored noise, times 0.18215.  The reference's ``UNetModel(in_channels=9)`` and its
``PLMSSampler`` (CPU subclass) then sample through ``ref_import.RefModelShim`` with ``hybrid`` conditioning: the shim
receives the CFG-batched context tensor (the reference PLMS concatenates tensor conditionings only) and prepends the
requests' ``c_concat`` = [mask latent, masked-image latent] per CFG half.  CFG 7.5 and no guidance, 6 steps.

Writes ``inpaint_tiny.npz`` (inputs, prepared tensors, posterior noise, latents) and ``inpaint_keys.json`` (both configs and
state-dict shapes; weights come from ``oracle.weights`` with the stored seeds).
"""
import io
import json
import os
import sys

import numpy as np
import torch
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..", "..")))

from oracle import ddim_oracle, ref_import, weights  # noqa: E402

UNET = dict(image_size=16, in_channels=9, model_channels=32, out_channels=4, num_res_blocks=1, attention_resolutions=[1],
            channel_mult=[1, 2], num_heads=2, use_spatial_transformer=True, transformer_depth=1, context_dim=32, legacy=False)
VAE = dict(double_z=True, z_channels=4, resolution=128, in_channels=3, out_ch=3, ch=64, ch_mult=[1, 1, 2, 2], num_res_blocks=1,
           attn_resolutions=[], dropout=0.0)
SEED_U, SEED_V, SIZE, S, SCALE = 61, 62, 128, 6, 7.5


def requests():
    rng = np.random.default_rng(9)
    img0 = rng.integers(0, 256, (150, 201, 3), dtype=np.uint8)
    img1 = rng.integers(0, 256, (90, 160, 3), dtype=np.uint8)
    m0 = np.zeros((150, 201), bool)
    m0[30:110, 40:120] = True
    m1 = np.zeros((90, 160), np.uint8)
    m1[20:70, 30:90] = 255
    buf = io.BytesIO()
    Image.fromarray(m1).save(buf, "JPEG")                         # the tool's masks pass through JPEG files
    m1 = np.asarray(Image.open(buf).convert("L")).copy()
    return [img0, img1], [m0, m1]


def processors(img, mask):
    x = np.asarray(Image.fromarray(img).resize((SIZE, SIZE), Image.LANCZOS)).astype(np.float32) / 255.0
    x = (2.0 * x - 1.0).transpose(2, 0, 1)
    m = np.asarray(Image.fromarray(mask).resize((SIZE, SIZE), Image.LANCZOS).convert("L")).astype(np.float32) / 255.0
    m[m < 0.5] = 0
    m[m >= 0.5] = 1
    m = m[None]
    masked = x * (m < 0.5)
    ml = torch.nn.functional.interpolate(torch.from_numpy(m)[None], size=(SIZE // 8, SIZE // 8))[0].numpy()
    return masked, ml


def main():
    UNetModel, _, _ = ref_import.load()
    sys.path.insert(0, ref_import.REF_ROOT)
    from ldm.models.diffusion.plms import PLMSSampler
    from ldm.modules.diffusionmodules import model as M
    from ldm.modules.distributions.distributions import DiagonalGaussianDistribution
    torch.set_grad_enabled(False)

    class PLMSSamplerCPU(PLMSSampler):
        def register_buffer(self, name, attr):
            setattr(self, name, attr)

    torch.manual_seed(0)
    net = UNetModel(**UNET).eval()
    shapes_u = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    sd_u = weights.make_state_dict(shapes_u, SEED_U)
    net.load_state_dict(sd_u)
    enc, quant = M.Encoder(**VAE).eval(), torch.nn.Conv2d(8, 8, 1)
    dec, post = M.Decoder(**VAE).eval(), torch.nn.Conv2d(4, 4, 1)
    shapes_v = {}
    for pre, m in (("encoder.", enc), ("decoder.", dec), ("quant_conv.", quant), ("post_quant_conv.", post)):
        shapes_v.update({pre + k: tuple(v.shape) for k, v in m.state_dict().items()})
    sd_v = weights.make_state_dict(shapes_v, SEED_V)
    for pre, m in (("encoder.", enc), ("decoder.", dec), ("quant_conv.", quant), ("post_quant_conv.", post)):
        m.load_state_dict({k[len(pre):]: v for k, v in sd_v.items() if k.startswith(pre)})

    imgs, masks = requests()
    B = len(imgs)
    gen = torch.Generator().manual_seed(9)
    ctx = torch.randn(B, 7, 32, generator=gen)
    uctx = torch.randn(7, 32, generator=gen)
    x_T = torch.randn(B, 4, SIZE // 8, SIZE // 8, generator=gen)
    noise = torch.randn(B, 4, SIZE // 8, SIZE // 8, generator=gen)
    masked, ml = zip(*(processors(i, m) for i, m in zip(imgs, masks)))
    masked, ml = np.stack(masked), np.stack(ml)
    dist = DiagonalGaussianDistribution(quant(enc(torch.from_numpy(masked))))
    z = 0.18215 * (dist.mean + dist.std * noise)
    cc = torch.cat([torch.from_numpy(ml), z], 1)

    sched = ddim_oracle.register_schedule("linear", 1000, 0.00085, 0.012)

    class InpaintShim(ref_import.RefModelShim):
        def apply_model(self, x, t, c):
            return super().apply_model(x, t, {"c_concat": [cc.repeat(x.shape[0] // B, 1, 1, 1)], "c_crossattn": [c]})

    sampler = PLMSSamplerCPU(InpaintShim(net, sched, "hybrid"))
    res = {"img0": imgs[0], "img1": imgs[1], "mask0": masks[0], "mask1": masks[1], "ctx": ctx.numpy(), "uctx": uctx.numpy(),
           "x_T": x_T.numpy(), "noise": noise.numpy(), "masked": masked, "mask_latent": ml, "c_concat": cc.numpy()}
    for scale in (SCALE, 1.0):
        out, _ = sampler.sample(S, B, (4, SIZE // 8, SIZE // 8), ctx, verbose=False, x_T=x_T.clone(), eta=0.0,
                                unconditional_guidance_scale=scale,
                                unconditional_conditioning=uctx[None].expand(B, -1, -1).contiguous() if scale != 1.0 else None)
        res[f"final_{scale:g}"] = out.numpy()
        print(f"scale {scale}: final latent |x| max {float(out.abs().max()):.3f}")
    res.update(seed_u=SEED_U, seed_v=SEED_V, size=SIZE, steps=S, scale=SCALE, wsum_u=weights.checksum(sd_u), wsum_v=weights.checksum(sd_v))
    np.savez_compressed(os.path.join(HERE, "inpaint_tiny.npz"), **res)
    with open(os.path.join(HERE, "inpaint_keys.json"), "w") as f:
        json.dump({"unet": UNET, "vae": VAE, "unet_keys": {k: list(v) for k, v in shapes_u.items()},
                   "vae_keys": {k: list(v) for k, v in shapes_v.items()}}, f)
    print("golden vectors written to", HERE)


if __name__ == "__main__":
    main()
