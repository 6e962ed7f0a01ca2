#!/usr/bin/env python
"""Timing of AnyDoor's visual-reference edit on one GPU -- a diagnostic, not a test.  Prints the card and its power limit with
the numbers.
  * the pixel kernels (csrc/anydoor.cu): ``anydoor_prepare`` (five launches) and ``anydoor_crop_back`` at B = 1 and 8, CUDA events
    over repeated windows, median; and ``_prepare`` from host arrays (upload, bounding boxes, the one read-back, geometry, kernels)
    on the host clock;
  * the reference's host work for one pair: its OpenCV calls in its order (cv2.resize, erode, Sobel, convertScaleAbs,
    addWeighted, and the numpy padding and casts), restated with the same OpenCV calls, host clock, cv2's thread count;
  * the whole request at 512 x 512, CFG DDIM (``--steps``, default 50) with the AnyDoor ControlNet + UNet geometry
    (tests/golden/anydoor_keys.json, hint 4 channels), DINOv2 ViT-g/14 + projector and the SD VAE decoder, seeded weights, fp16
    kernels: ``edit_pairs`` at B = 1 and 8 pairs, images/s, and the share of the time outside the sampler (everything but
    ``sampler.sample``).
Usage: python tests/diag_anydoor.py [--windows 5] [--iters 20] [--steps 50] [--skip-request]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
from oracle import anydoor_oracle as O  # noqa: E402


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


def host_ms(fn, reps):
    fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return sorted(t)[len(t) // 2]


def reference_host(cv2, ri, rm, ti, tm, pred):
    """The reference's host work for one pair with its own OpenCV calls (process_pairs + sobel + crop_back)."""
    y1, y2, x1, x2 = O.get_bbox_from_mask(rm)
    m3 = np.stack([rm] * 3, -1)
    img = (ri * m3 + np.ones_like(ri) * 255 * (1 - m3))[y1:y2, x1:x2]
    msk = rm[y1:y2, x1:x2]
    img = O.pad_square(np.pad(img, ((4, 4), (4, 4), (0, 0)), constant_values=255), 255)
    msk = O.pad_square(np.stack([np.pad(msk, 4)] * 3, -1) * 255, 0)
    ref = cv2.resize(img.astype(np.uint8), (224, 224))
    rmask = cv2.resize(msk.astype(np.uint8), (224, 224))[:, :, 0]
    im = cv2.resize(ref, (256, 256))
    m = cv2.erode((cv2.resize(rmask / 255, (256, 256)) > 0.5).astype(np.uint8), np.ones((5, 5), np.uint8), iterations=2)
    s = cv2.addWeighted(cv2.convertScaleAbs(cv2.Sobel(im, cv2.CV_64F, 1, 0, ksize=3)), 0.5,
                        cv2.convertScaleAbs(cv2.Sobel(im, cv2.CV_64F, 0, 1, ksize=3)), 0.5, 0)
    s = np.max(s, -1) * m
    s[s < 50] = 0
    hf = cv2.resize((np.stack([s] * 3, -1).astype(np.float32) / 255 * im.astype(np.float32)).astype(np.uint8), (224, 224))
    crop = ti[100:400, 80:420]
    col = crop.copy()
    col[50:250, 60:280] = cv2.resize(hf, (220, 200))
    cm = crop * 0.0
    cm[50:250, 60:280] = 1.0
    crop, col, cm = O.pad_square(crop, 0).astype(np.uint8), O.pad_square(col, 0).astype(np.uint8), O.pad_square(cm, -1).astype(np.uint8)
    jpg = cv2.resize(crop, (512, 512)).astype(np.float32) / 127.5 - 1.0
    hint = np.concatenate([cv2.resize(col, (512, 512)).astype(np.float32) / 127.5 - 1.0,
                           (cv2.resize(cm, (512, 512), interpolation=cv2.INTER_NEAREST).astype(np.float32) > 0.5)[:, :, :1]], -1)
    p = cv2.resize(pred, (340, 340))[20:320]
    out = ti.copy()
    out[105:395, 85:415] = p[5:-5, 5:-5]
    return ref / 255, jpg, hint, out


def full_models(steps):
    from anyedit_b200.autoencoder import AutoencoderKL
    from anyedit_b200.cldm import ControlDenoiser, ControlledUnetModel, ControlNet
    from anyedit_b200.ddim import DDIMSampler
    from anyedit_b200.encoders import FrozenDinoV2Encoder
    from oracle import weights
    cfg = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "anydoor_keys.json")))["config"]
    cn = ControlNet(**dict({k: v for k, v in cfg.items() if k != "out_channels"}, hint_channels=4))
    un = ControlledUnetModel(**cfg)
    enc = FrozenDinoV2Encoder()
    vae = AutoencoderKL(dict(double_z=True, z_channels=4, resolution=256, in_channels=3, out_ch=3, ch=128, ch_mult=[1, 2, 4, 4],
                             num_res_blocks=2, attn_resolutions=[], dropout=0.0), embed_dim=4)
    for i, net in enumerate((cn, un, enc, vae)):
        net.load_state_dict(weights.make_state_dict({k: tuple(v.shape) for k, v in net.state_dict().items()}, 51 + i,
                                                    scheme="torch"), strict=True)
    model = ControlDenoiser(un.cuda(), cn.cuda(), cond_stage_model=enc.cuda(), first_stage_model=vae.cuda(),
                            scale_factor=0.18215).cuda()
    return model, DDIMSampler(model)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--skip-request", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "diag_anydoor needs a CUDA device"
    from anyedit_b200 import anydoor as A, ops
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    print(f"device: {torch.cuda.get_device_name(0)} | nvidia-smi name, power limit, max SM clock: {q[0] if q else 'n/a'}")
    names = ["blob512", "edges", "edges_tr", "tiny", "wide", "tall", "square", "blob512"]
    ins = [O.case_inputs(n) for n in names]
    for B in (1, 8):
        ri, rm, ti, tm = (np.stack([x[i] for x in ins[:B]]) for i in range(4))
        np.random.seed(0)
        st, _, g = A._prepare(ri, rm, ti, tm)
        dev = [torch.from_numpy(x).cuda() for x in (ri, rm, ti)]
        t_prep = timed(lambda: ops.anydoor_prepare(*dev, g, st), a.windows, a.iters)
        dec = torch.from_numpy(np.stack([O.case_pred(i) for i in range(B)])).cuda()
        out = torch.empty_like(dev[2])
        t_back = timed(lambda: ops.anydoor_crop_back(dec, dev[2], g, out), a.windows, a.iters)
        t_host = host_ms(lambda: (np.random.seed(0), A._prepare(ri, rm, ti, tm), torch.cuda.synchronize()), 2 * a.windows)
        print(f"B={B}: anydoor_prepare {t_prep * 1e3:.1f} us ({t_prep * 1e3 / B:.1f} us/pair), crop_back {t_back * 1e3:.1f} us "
              f"({t_back * 1e3 / B:.1f} us/pair); _prepare from host arrays {t_host:.2f} ms")
    import cv2
    ri, rm, ti, tm, seed = ins[0]
    pred = O.decode_to_pred(O.case_pred(seed))
    t_ref = host_ms(lambda: reference_host(cv2, ri, rm, ti, tm, pred), 10)
    print(f"reference host process_pairs + sobel + crop_back (its OpenCV calls), one pair: {t_ref:.2f} ms "
          f"(cv2 threads {cv2.getNumThreads()}, OpenCV {cv2.__version__})")
    if a.skip_request:
        return
    model, sampler = full_models(a.steps)
    orig = sampler.sample
    spent = {"s": 0.0}

    def timed_sample(*args, **kw):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = orig(*args, **kw)
        torch.cuda.synchronize()
        spent["s"] += time.perf_counter() - t0
        return r

    sampler.sample = timed_sample
    for B in (1, 8):
        ri, rm, ti, tm = (np.stack([x[i] for x in ins[:B]]) for i in range(4))
        np.random.seed(0)
        A.edit_pairs(model, sampler, ri, rm, ti, tm, steps=a.steps)                 # warm-up (graph capture, packing)
        torch.cuda.synchronize()
        spent["s"] = 0.0
        reps = 2
        t0 = time.perf_counter()
        for _ in range(reps):
            np.random.seed(0)
            A.edit_pairs(model, sampler, ri, rm, ti, tm, steps=a.steps)
        torch.cuda.synchronize()
        dt = (time.perf_counter() - t0) / reps
        print(f"edit_pairs 512x512, {a.steps} CFG DDIM steps, B={B}: {dt * 1e3:.0f} ms per call, {B / dt:.2f} images/s, "
              f"{100 * (1 - spent['s'] / reps / dt):.1f} % of the time outside the sampler")


if __name__ == "__main__":
    main()
