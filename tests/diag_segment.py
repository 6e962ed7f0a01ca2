#!/usr/bin/env python
"""Timing of the UniFormer-S + UPerNet segmentation annotator (``segment.UniFormerSegmentor``) on one GPU -- a diagnostic, not a
test.  Seeded weights (the arithmetic does not depend on their values); B = 1 and 4 at 512 x 683 (a 480 x 640 image after the test
pipeline's rescale); median over repeated timed windows after warm-up, CUDA events; rate = FLOPs counted from the shapes
(2 M N K per contraction and conv, 2 k^2 per depthwise output, 4 n^2 d per head for attention) over the median time.  Also
``inference_segmentor`` end to end on the 480 x 640 image (host rescale, upload, network, labels, download), and the fp32 eager
restatement of oracle/segment_oracle.py on the same GPU for scale (the reference's mmseg stack does not import here: not measured).
Prints the card and its power limit with the numbers.
Usage: python tests/diag_segment.py [--windows 7] [--iters 5]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))


def flops_per_image(H=512, W=683, dims=(64, 128, 320, 512), layers=(3, 4, 8, 3), Ch=512, classes=150, pools=(1, 2, 3, 6)):
    """(backbone contractions, attention, depthwise, head convs) in FLOPs."""
    lin = attn = dw = 0
    h, w, cin = H, W, 3
    sizes = []
    for s, (C, L) in enumerate(zip(dims, layers)):
        r = 4 if s == 0 else 2
        h, w = h // r, w // r
        n = h * w
        lin += 2 * n * C * cin * r * r
        for _ in range(L):
            dw += 2 * n * C * 9
            if s < 2:
                lin += 2 * n * C * C * 2 + 2 * n * C * 4 * C * 2
                dw += 2 * n * C * 25
            else:
                lin += 2 * n * C * 3 * C + 2 * n * C * C + 2 * n * C * 4 * C * 2
                attn += 4 * n * n * C
        sizes.append((h, w))
        cin = C
    (h1, w1), (h4, w4) = sizes[0], sizes[3]
    head = sum(2 * p * p * dims[3] * Ch for p in pools) + 2 * h4 * w4 * (dims[3] + len(pools) * Ch) * Ch * 9
    head += sum(2 * hh * ww * c * Ch for (hh, ww), c in zip(sizes[:3], dims[:3]))
    head += sum(2 * hh * ww * Ch * Ch * 9 for (hh, ww) in sizes[:3])
    head += 2 * h1 * w1 * 4 * Ch * Ch * 9 + 2 * h1 * w1 * Ch * classes
    return lin, attn, dw, head


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
    return sorted(times)[len(times) // 2], min(times), max(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "diag_segment needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    print(f"device: {torch.cuda.get_device_name(0)} | nvidia-smi name, power limit, max SM clock: {q[0] if q else 'n/a'}")
    from anyedit_b200 import segment
    from oracle import segment_oracle as O
    m = segment.UniFormerSegmentor()
    sd = O.seeded_state_dict({k: tuple(v.shape) for k, v in m.state_dict().items()}, 95)
    m.load_state_dict(sd, strict=True)
    m = m.cuda()
    lin, attn, dw, head = flops_per_image()
    total = lin + attn + dw + head
    print(f"512x683 counted per image: backbone contractions {lin / 1e9:.1f} GFLOP, attention {attn / 1e9:.1f}, depthwise "
          f"{dw / 1e9:.2f}, head {head / 1e9:.1f}, total {total / 1e9:.1f} GFLOP")
    img = O.tiny_raw_images((480, 640), 96, B=1)[0]
    for B in (1, 4):
        x = torch.from_numpy(np.ascontiguousarray(segment.rescale(img)))[None].repeat(B, 1, 1, 1).cuda()
        for _ in range(3):
            m(x)
        torch.cuda.synchronize()
        med, lo, hi = timed(lambda: m(x), args.windows, args.iters)
        print(f"forward B={B} 512x683: median {med:.2f} ms per call (min {lo:.2f}, max {hi:.2f}; {args.windows} windows x {args.iters} "
              f"calls), {med / B:.2f} ms per image, {B * total / (med * 1e-3) / 1e12:.0f} TFLOP/s counted")
    for _ in range(3):
        segment.inference_segmentor(m, img)
    ts = []
    for _ in range(args.windows * args.iters):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        segment.inference_segmentor(m, img)          # ends in a device-to-host copy of the labels
        ts.append((time.perf_counter() - t0) * 1e3)
    ts.sort()
    print(f"inference_segmentor 480x640 (rescale on the host, upload, network, labels, download): median {ts[len(ts) // 2]:.2f} ms "
          f"(min {ts[0]:.2f}, max {ts[-1]:.2f}; {len(ts)} calls, host clock)")
    sdc = {k: v.cuda() for k, v in sd.items()}
    xo = O.normalize(segment.rescale(img)).cuda()
    with torch.no_grad():
        for _ in range(2):
            O.logits(sdc, xo)
        torch.cuda.synchronize()
        med, lo, hi = timed(lambda: O.logits(sdc, xo), 3, 2)
    print(f"fp32 eager restatement (oracle/segment_oracle.py, not the reference) B=1 512x683: median {med:.2f} ms per call "
          f"(min {lo:.2f}, max {hi:.2f}); the reference's mmseg stack: not measured")


if __name__ == "__main__":
    main()
