#!/usr/bin/env python
"""Timing of the Canny sketch annotator (``sketch.detect``: csrc/sketch.cu's four launches) on one GPU -- a diagnostic, not a
test.  Seeded structured images (oracle/sketch_oracle.py) at B = 1 and 8 for 512 x 512 and 1024 x 1024; median over repeated
timed windows after warm-up, CUDA events around the kernels on preallocated tensors, called eagerly and replayed from a CUDA
graph of the same calls (the replay leaves out the host's launch path); bytes counted from the shapes, per pixel:
3 read (BGR); the out byte written as the class by the tile kernel, read by the flag and output passes and rewritten (4); the
int32 label written by the tile kernel, read and written by the flag pass and read by the output pass (16); the root flag
written and read (2); so 25 bytes per pixel, with every pixel counted as a candidate; rate over the median time against the
H100 SXM's 3.35 TB/s.  Also ``detect`` from a uint8 numpy image to the uint8 numpy map (upload, kernels, download; host clock)
and the reference's four cv2 calls on the host, with cv2's thread count.  Prints the card and its power limit with the numbers.
Checks every timed output against cv2 once.
Usage: python tests/diag_sketch.py [--windows 7] [--iters 20]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))

BYTES_PER_PIXEL = 3 + 4 + 16 + 2
HBM = 3.35e12


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
    times.sort()
    return times[len(times) // 2], times[0], times[-1]


def host_timed(fn, n):
    ts = []
    for _ in range(n):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    ts.sort()
    return ts[len(ts) // 2], ts[0], ts[-1]


def cv2_sketch(img):
    import cv2
    grey = cv2.cvtColor(img, cv2.COLOR_BGR2GRAY)
    return cv2.bitwise_not(cv2.Canny(cv2.GaussianBlur(grey, (3, 3), 0), 50, 150))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "diag_sketch needs a CUDA device"
    import cv2
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    print(f"device: {torch.cuda.get_device_name(0)} | nvidia-smi name, power limit, max SM clock: {q[0] if q else 'n/a'}")
    from anyedit_b200 import ops, sketch
    from oracle import sketch_oracle as O
    for (H, W) in ((512, 512), (1024, 1024)):
        for B in (1, 8):
            imgs = O.images((H, W), 151, B=B)
            x = torch.from_numpy(imgs).cuda()
            out = torch.empty(B, H, W, dtype=torch.uint8, device="cuda")
            for _ in range(3):
                ops.sketch(x, out)
            torch.cuda.synchronize()
            got = out.cpu().numpy()
            assert all(np.array_equal(got[b], cv2_sketch(imgs[b])) for b in range(B)), "output differs from cv2"
            nbytes = B * H * W * BYTES_PER_PIXEL
            # eager calls (host launch path included), then the same calls replayed from a CUDA graph (device time alone)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                for _ in range(args.iters):
                    ops.sketch(x, out)
            for name, fn, n in (("eager", lambda: ops.sketch(x, out), args.iters), ("graph", g.replay, 1)):
                med, lo, hi = timed(fn, args.windows, n)
                med, lo, hi = (v / (args.iters if name == "graph" else 1) for v in (med, lo, hi))
                print(f"kernels {name} B={B} {H}x{W}: median {med * 1e3:.1f} us per call (min {lo * 1e3:.1f}, max {hi * 1e3:.1f}; "
                      f"{args.windows} windows x {args.iters} calls), {med * 1e3 / B:.1f} us per image, {nbytes / 1e6:.2f} MB "
                      f"counted, {nbytes / (med * 1e-3) / 1e12:.3f} TB/s = {nbytes / (med * 1e-3) / HBM:.3f} of 3.35 TB/s")
            assert np.array_equal(out.cpu().numpy(), got), "graph replay differs"
    for (H, W) in ((512, 512), (1024, 1024)):
        img = O.images((H, W), 152)
        for _ in range(3):
            sketch.detect(img)
        med, lo, hi = host_timed(lambda: sketch.detect(img), args.windows * 5)
        print(f"sketch.detect {H}x{W} B=1 (uint8 numpy in, upload, kernels, uint8 numpy out): median {med:.3f} ms "
              f"(min {lo:.3f}, max {hi:.3f}; host clock)")
        for _ in range(3):
            cv2_sketch(img[0])
        med, lo, hi = host_timed(lambda: cv2_sketch(img[0]), args.windows * 5)
        print(f"reference's four cv2 calls {H}x{W} on the host (OpenCV {cv2.__version__}, cv2.getNumThreads() = "
              f"{cv2.getNumThreads()}, {os.cpu_count()} CPUs visible): median {med:.3f} ms (min {lo:.3f}, max {hi:.3f})")


if __name__ == "__main__":
    main()
