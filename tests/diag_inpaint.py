#!/usr/bin/env python
"""Timing of AnyEdit's inpainting edits on one GPU -- a diagnostic, not a test.  Prints the card and its power limit with the
numbers.
  * the byte kernels at B = 1 and 8 from 640 x 480 images and masks, each launch alone (plans and pointer tables made once):
    the image resize, the mask resize, the conditioning, the background mask; the host plan of the image resize; the whole
    ``prepare`` call: CUDA events over repeated windows, median;
  * ``inpaint`` end to end at 512^2 (prepare, SD VAE encode, ``--steps`` PLMS steps with CFG 7.5 on the SD-1.5-inpainting
    UNet with seeded weights, decode, bytes, LANCZOS back to 640 x 480) at B = 1 and 8, requests/s, and the share of the time
    spent outside ``sampler.sample``;
  * the host arm: Pillow / OpenCV on this machine's CPU for the same byte steps of one request (the tool's path).
Usage: python tests/diag_inpaint.py [--windows 5] [--iters 20] [--steps 50] [--reps 2]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))

H, W = 480, 640


def timed(fn, windows, iters):
    times = []
    for _ in range(windows):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / iters)
    return sorted(times)[len(times) // 2]


def requests(B, seed=0):
    rng = np.random.default_rng(seed)
    imgs = [torch.from_numpy(rng.integers(0, 256, (H, W, 3), dtype=np.uint8)).cuda() for _ in range(B)]
    masks, fores = [], []
    for i in range(B):
        m = np.zeros((H, W), np.uint8)
        m[H // 4:3 * H // 4, W // 5:W // 2 + 10 * i] = 255
        masks.append(torch.from_numpy(m > 0 if i % 2 == 0 else m).cuda())
        fores.append(torch.from_numpy(np.repeat(m[..., None], 3, -1)).cuda())
    return imgs, masks, fores


def _resize_launch(srcs, outs, filters):
    """The plan, its upload and the pointer tables made once; returns the bare kernel launch."""
    from anyedit_b200 import _lib, ops
    C = srcs[0].shape[2]
    table, R, sm, nb = ops.pil_resize_plan([(*a.shape[:2], *o.shape[:2]) for a, o in zip(srcs, outs)], filters, C)
    keep = [table.cuda(), ops._ptr_table(srcs, "cuda"), ops._ptr_table(outs, "cuda")]
    lib = _lib.load()
    return lambda: _lib.check(lib.anysd_pil_resize_u8(ops._ptr(keep[1]), ops._ptr(keep[2]), ops._ptr(keep[0]), len(srcs), C, R, sm, nb,
                                                      ops._stream()), "pil_resize")


def kernel_leg(a):
    from anyedit_b200 import _lib, inpaint, ops
    print("byte kernels (ms, CUDA events, median of windows): each launch alone, then whole calls with host plans and uploads:")
    for B in (1, 8):
        imgs, masks, fores = requests(B)
        st = inpaint.prepare(imgs, masks)
        ms = [m.view(torch.uint8)[..., None] if m.dtype == torch.bool else m[..., None] for m in masks]
        filters = ["mode1" if m.dtype == torch.bool else "lanczos" for m in masks]
        k_img = _resize_launch(imgs, list(st["image"]), ["lanczos"] * B)
        k_mask = _resize_launch(ms, [m[..., None] for m in st["mask"]], filters)
        k_prep = lambda: ops.inpaint_prepare(st["image"], st["mask"], st["masked"], st["mask_latent"], st["counts"])
        outs = [torch.empty(H, W, dtype=torch.uint8, device="cuda") for _ in fores]
        counts = torch.empty(B, dtype=torch.int32, device="cuda")
        hw = torch.tensor([v for f in fores for v in f.shape[:2]], dtype=torch.int32).cuda()
        src, dst = ops._ptr_table(fores, "cuda"), ops._ptr_table(outs, "cuda")
        lib = _lib.load()
        k_bg = lambda: _lib.check(lib.anysd_background_mask_u8(ops._ptr(src), ops._ptr(dst), ops._ptr(hw), B, H, W, ops._ptr(counts),
                                                               ops._stream()), "background_mask")
        t = {name: timed(fn, a.windows, a.iters) for name, fn in (("resize images", k_img), ("resize masks", k_mask),
                                                                   ("conditioning", k_prep), ("background mask", k_bg))}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(a.iters):
            ops.pil_resize_plan([(H, W, 512, 512)] * B, ["lanczos"] * B, 3)
        plan = (time.perf_counter() - t0) / a.iters * 1e3
        whole = timed(lambda: inpaint.prepare(imgs, masks), a.windows, a.iters)
        mb = B * 512 * 512 * 64 * 2 / 1e6
        print(f"  B={B}: " + ", ".join(f"{k} {v:.3f}" for k, v in t.items()) +
              f" (conditioning writes {mb:.0f} MB: {mb / 1e3 / t['conditioning']:.2f} TB/s); host plan of the image resize "
              f"{plan:.3f}; whole prepare() {whole:.3f}")


def host_leg(reps):
    import cv2
    from PIL import Image
    rng = np.random.default_rng(1)
    img = Image.fromarray(rng.integers(0, 256, (H, W, 3), dtype=np.uint8))
    m = np.zeros((H, W), np.uint8)
    m[H // 4:3 * H // 4, W // 5:W // 2] = 255
    fore = np.repeat(m[..., None], 3, -1)
    out512 = Image.fromarray(rng.integers(0, 256, (512, 512, 3), dtype=np.uint8))

    def one():
        back = cv2.cvtColor(cv2.GaussianBlur(fore, (5, 5), 0), cv2.COLOR_BGR2GRAY) == 0
        mk = Image.fromarray(back)
        im = img.resize((512, 512), Image.LANCZOS)
        x = np.asarray(im).astype(np.float32) / 255.0 * 2.0 - 1.0
        mm = (np.asarray(mk.resize((512, 512), Image.LANCZOS).convert("L")).astype(np.float32) / 255.0 >= 0.5)
        _ = x * (~mm)[..., None]
        _ = out512.resize((W, H), Image.LANCZOS)
    one()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        one()
        t.append(time.perf_counter() - t0)
    print(f"host arm (Pillow / OpenCV / numpy, one request: mask, resizes to 512^2, processors, resize back): "
          f"{1e3 * sorted(t)[len(t) // 2]:.2f} ms on this machine's CPU")


def sd_inpaint():
    from anyedit_b200.autoencoder import AutoencoderKL
    from anyedit_b200.diffusion import LatentInpaintDenoiser
    from anyedit_b200.unet import UNetModel
    from oracle import weights
    meta = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "sd15_keys.json")))
    cfg = dict(meta["config"], in_channels=9)
    with torch.device("cuda"):
        net = UNetModel(**cfg)
    net.load_state_dict(weights.make_state_dict({k: tuple(v.shape) for k, v in net.state_dict().items()}, 3, scheme="torch"))
    vae = AutoencoderKL(dict(double_z=True, z_channels=4, resolution=256, in_channels=3, out_ch=3, ch=128, ch_mult=[1, 2, 4, 4],
                             num_res_blocks=2, attn_resolutions=[], dropout=0.0), embed_dim=4)
    vae.load_state_dict(weights.make_state_dict({k: tuple(v.shape) for k, v in vae.state_dict().items()}, 54, scheme="torch"))
    return LatentInpaintDenoiser(net, first_stage_model=vae.cuda(), scale_factor=0.18215).cuda()


def run_leg(a):
    from anyedit_b200 import inpaint
    from anyedit_b200.plms import PLMSSampler
    model = sd_inpaint()
    smp = PLMSSampler(model)
    inner = {"t": 0.0}
    orig = smp.sample

    def timed_sample(*args, **kw):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = orig(*args, **kw)
        torch.cuda.synchronize()
        inner["t"] += time.perf_counter() - t0
        return out
    smp.sample = timed_sample
    print(f"inpaint end to end at 512^2, {a.steps} PLMS steps, CFG 7.5, SD-1.5-inpainting widths, seeded weights "
          f"(median of {a.reps}):")
    for B in (1, 8):
        imgs, masks, _ = requests(B)
        gen = torch.Generator().manual_seed(B)
        cond = torch.randn(B, 77, 768, generator=gen).cuda()
        uncond = torch.randn(77, 768, generator=gen).cuda()
        inpaint.inpaint(model, smp, imgs, masks, cond, uncond, steps=2)            # warm-up: graphs, packs, plans
        ts, share = [], []
        for _ in range(a.reps):
            inner["t"] = 0.0
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            inpaint.inpaint(model, smp, imgs, masks, cond, uncond, steps=a.steps)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            ts.append(dt)
            share.append(1.0 - inner["t"] / dt)
        t = sorted(ts)[len(ts) // 2]
        print(f"  B={B}: {t:.3f} s per call, {B / t:.3f} requests/s, outside sampler.sample {100 * sorted(share)[len(share) // 2]:.2f} %")


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--windows", type=int, default=5)
    p.add_argument("--iters", type=int, default=20)
    p.add_argument("--steps", type=int, default=50)
    p.add_argument("--reps", type=int, default=2)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("diag_inpaint needs a GPU")
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True,
                         text=True).stdout.strip())
    kernel_leg(a)
    host_leg(5)
    run_leg(a)


if __name__ == "__main__":
    main()
