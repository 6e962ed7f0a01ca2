#!/usr/bin/env python
"""Timing of the HED scribble annotator (``hed.ControlNetHED_Apache2.edge_map``: network and edge kernel) on one GPU -- a
diagnostic, not a test.  Seeded weights (the arithmetic does not depend on their values); B = 1 and 8 at 512 x 512, B = 1 at
480 x 640 and 1024 x 1024; median over repeated timed windows after warm-up, CUDA events; rate = FLOPs counted from the shapes
(2 h w Cin Cout 9 per 3x3 conv, 2 h w C per side projection) over the median time.  Also ``HEDdetector.detect`` from a uint8 numpy
image to the uint8 numpy map (upload, network, edges, download; host clock), and the fp32 eager restatement of oracle/hed_oracle.py
on the same GPU with TF32 at torch's default (the reference's configuration): the network alone (CUDA events) and with the
reference's host post-processing (host clock).  Prints the card and its power limit with the numbers.
Usage: python tests/diag_hed.py [--windows 7] [--iters 5]"""
import argparse
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))

BLOCKS = ((3, 64, 2), (64, 128, 2), (128, 256, 3), (256, 512, 3), (512, 512, 3))


def flops_per_image(H, W):
    total = 0
    for b, (cin, cout, n) in enumerate(BLOCKS):
        if b:
            H, W = H // 2, W // 2
        for i in range(n):
            total += 2 * H * W * (cin if i == 0 else cout) * cout * 9
        total += 2 * H * W * cout
    return total


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


def host_timed(fn, n):
    ts = []
    for _ in range(n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()                                          # ends in a device-to-host copy
        ts.append((time.perf_counter() - t0) * 1e3)
    ts.sort()
    return ts[len(ts) // 2], ts[0], ts[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "diag_hed needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    print(f"device: {torch.cuda.get_device_name(0)} | nvidia-smi name, power limit, max SM clock: {q[0] if q else 'n/a'}")
    from anyedit_b200 import hed
    from oracle import hed_oracle as O
    sd = O.seeded_state_dict(121)
    m = hed.ControlNetHED_Apache2()
    m.load_state_dict(sd, strict=True)
    m = m.cuda()
    for (H, W), B in (((512, 512), 1), ((512, 512), 8), ((480, 640), 1), ((1024, 1024), 1)):
        x = torch.from_numpy(O.images((H, W), 122, B=B)).cuda()
        for _ in range(3):
            m.edge_map(x)
        torch.cuda.synchronize()
        med, lo, hi = timed(lambda: m.edge_map(x), args.windows, args.iters)
        fl = flops_per_image(H, W)
        print(f"edge_map B={B} {H}x{W}: median {med:.2f} ms per call (min {lo:.2f}, max {hi:.2f}; {args.windows} windows x "
              f"{args.iters} calls), {med / B:.2f} ms per image, {fl / 1e9:.1f} GFLOP counted per image, "
              f"{B * fl / (med * 1e-3) / 1e12:.0f} TFLOP/s counted")
    det = hed.HEDdetector.__new__(hed.HEDdetector)
    det.netNetwork = m
    img = O.images((512, 512), 123)
    for _ in range(3):
        det.detect(img)
    med, lo, hi = host_timed(lambda: det.detect(img), args.windows * args.iters)
    print(f"HEDdetector.detect 512x512 (uint8 numpy in, upload, network, edges, uint8 numpy out): median {med:.2f} ms "
          f"(min {lo:.2f}, max {hi:.2f}; host clock)")
    sdc = {k: v.cuda() for k, v in sd.items()}
    xo = torch.from_numpy(img).cuda()
    print(f"torch TF32 defaults: cudnn.allow_tf32={torch.backends.cudnn.allow_tf32}, "
          f"cuda.matmul.allow_tf32={torch.backends.cuda.matmul.allow_tf32}")
    with torch.no_grad():
        for _ in range(2):
            O.side_maps(sdc, xo)
        torch.cuda.synchronize()
        med, lo, hi = timed(lambda: O.side_maps(sdc, xo), 3, 3)
        print(f"fp32 eager restatement (oracle/hed_oracle.py) B=1 512x512, network only: median {med:.2f} ms per call "
              f"(min {lo:.2f}, max {hi:.2f})")
        med, lo, hi = host_timed(lambda: O.edge_map(O.side_maps(sdc, xo), 512, 512), 7)
        print(f"fp32 eager restatement with the reference's host post-processing (cv2 / numpy) 512x512: median {med:.2f} ms "
              f"(min {lo:.2f}, max {hi:.2f}; host clock)")


if __name__ == "__main__":
    main()
