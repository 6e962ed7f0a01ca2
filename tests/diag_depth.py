#!/usr/bin/env python
"""Timing of the Depth Anything V2 ViT-L depth annotator (``depth.DepthAnythingV2``) on one GPU -- a diagnostic, not a test.
Seeded weights (the arithmetic does not depend on their values); B = 1 and 4 at 518 x 518, B = 1 at 518 x 784; median over
repeated timed windows after warm-up, CUDA events; rate = FLOPs counted from the shapes (2 M N K per contraction and conv,
4 n^2 d per head for attention) over the median time.  Prints the card and its power limit with the numbers.
Usage: python tests/diag_depth.py [--windows 7] [--iters 5]"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))


def flops_per_image(H=518, W=518, D=1024, layers=24, heads=16, F=256, oc=(256, 512, 1024, 1024)):
    gh, gw = H // 14, W // 14
    n = gh * gw + 1
    lin = 2 * n * (3 * D * D + D * D + 2 * 4 * D * D) * layers
    attn = 4 * n * n * (D // heads) * heads * layers
    P = gh * gw
    sizes = [(4 * gh, 4 * gw), (2 * gh, 2 * gw), (gh, gw), ((gh - 1) // 2 + 1, (gw - 1) // 2 + 1)]
    conv = 2 * P * D * 588 + sum(2 * P * D * c for c in oc) + 2 * sizes[3][0] * sizes[3][1] * oc[3] * oc[3] * 9       # patch embedding, projects, resize_layers[3]
    conv += sum(2 * h * w * c * F * 9 for (h, w), c in zip(sizes, oc))                               # layer{k}_rn
    outs = [(2 * sizes[0][0], 2 * sizes[0][1])] + sizes[:3]       # out_conv of refinenet{k+1} runs at the next level (reference order)
    for k, (h, w) in enumerate(sizes):
        conv += (2 if k == 3 else 4) * 2 * h * w * F * F * 9 + 2 * outs[k][0] * outs[k][1] * F * F  # residual conv units, out_conv
    h1, w1 = outs[0]
    conv += 2 * h1 * w1 * F * (F // 2) * 9 + 2 * H * W * (F // 2) * 32 * 9 + 2 * H * W * 32        # output_conv1, output_conv2
    tconv = 2 * P * (oc[0] * oc[0] * 16 + oc[1] * oc[1] * 4)
    return lin, attn, conv, tconv


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "diag_depth needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    print(f"device: {torch.cuda.get_device_name(0)} | nvidia-smi name, power limit, max SM clock: {q[0] if q else 'n/a'}")
    from anyedit_b200.depth import DepthAnythingV2
    torch.manual_seed(0)
    m = DepthAnythingV2(encoder="vitl").cuda().eval()
    for B, H, W in ((1, 518, 518), (4, 518, 518), (1, 518, 784)):
        lin, attn, conv, tconv = flops_per_image(H, W)
        total = lin + attn + conv + tconv
        print(f"{H}x{W} counted per image: linears {lin / 1e9:.1f} GFLOP, attention {attn / 1e9:.1f}, convolutions {conv / 1e9:.1f}, "
              f"transposed convs {tconv / 1e9:.1f}, total {total / 1e12:.3f} TFLOP")
        x = torch.randn(B, 3, H, W, device="cuda")
        for _ in range(3):
            m(x)
        torch.cuda.synchronize()
        times = []
        for _ in range(args.windows):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.iters):
                m(x)
            b.record()
            b.synchronize()
            times.append(a.elapsed_time(b) / args.iters)
        med = sorted(times)[len(times) // 2]
        print(f"B={B} {H}x{W}: median {med:.2f} ms per call (min {min(times):.2f}, max {max(times):.2f}; {args.windows} windows x "
              f"{args.iters} calls), {med / B:.2f} ms per image, {B * total / (med * 1e-3) / 1e12:.0f} TFLOP/s counted")


if __name__ == "__main__":
    main()
