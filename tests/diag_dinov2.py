#!/usr/bin/env python
"""Timing of AnyDoor's reference-image encoder (``encoders.FrozenDinoV2Encoder``: DINOv2 ViT-g/14 + projector) on one GPU --
a diagnostic, not a test.  Seeded weights (the arithmetic does not depend on their values), 224 x 224 images, B = 1 and 8;
median over repeated timed windows after warm-up, CUDA events; rate = FLOPs counted from the shapes (2 M N K per contraction,
4 n^2 d per head for attention) over the median time.  Prints the card and its power limit with the numbers.
Usage: python tests/diag_dinov2.py [--windows 7] [--iters 5]"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))


def flops_per_image(D=1536, layers=40, heads=24, hidden=4096, n=257, patch_k=588, proj=1024):
    lin = 2 * n * (D * 3 * D + D * D + D * 2 * hidden + hidden * D) * layers
    attn = 4 * n * n * (D // heads) * heads * layers
    edge = 2 * (n - 1) * D * patch_k + 2 * n * D * proj
    return lin, attn, edge


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "diag_dinov2 needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    print(f"device: {torch.cuda.get_device_name(0)} | nvidia-smi name, power limit, max SM clock: {q[0] if q else 'n/a'}")
    from anyedit_b200.encoders import FrozenDinoV2Encoder
    torch.manual_seed(0)
    with torch.device("cuda"):
        enc = FrozenDinoV2Encoder()
    lin, attn, edge = flops_per_image()
    print(f"counted per image: linears {lin / 1e9:.1f} GFLOP, attention {attn / 1e9:.1f} GFLOP, patch + projector "
          f"{edge / 1e9:.2f} GFLOP, total {(lin + attn + edge) / 1e12:.3f} TFLOP")
    for B in (1, 8):
        x = torch.rand(B, 3, 224, 224, device="cuda")
        for _ in range(3):
            enc(x)
        torch.cuda.synchronize()
        times = []
        for _ in range(args.windows):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.iters):
                enc(x)
            b.record()
            b.synchronize()
            times.append(a.elapsed_time(b) / args.iters)
        med = sorted(times)[len(times) // 2]
        rate = B * (lin + attn + edge) / (med * 1e-3) / 1e12
        print(f"B={B}: median {med:.2f} ms per call (min {min(times):.2f}, max {max(times):.2f}; {args.windows} windows x "
              f"{args.iters} calls), {med / B:.2f} ms per image, {rate:.0f} TFLOP/s counted")


if __name__ == "__main__":
    main()
