#!/usr/bin/env python
"""Diagnostic (not a pytest file): the 8x8-level contractions under ANYSD_GEMM_SPLITK=0|2|3|4 (one process per setting; the
GPU is kept busy ahead of the timed launches so that host launch latency does not leak into the CUDA-event intervals)."""
import os
import sys

import torch

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
from anyedit_b200 import ops  # noqa: E402


def timeit(fn, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    torch.cuda._sleep(int(2e7))                      # ~10 ms of GPU work queued first: the host runs ahead
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e-3


def main():
    B = 16
    g = torch.Generator(device="cuda").manual_seed(2)
    print("ANYSD_GEMM_SPLITK =", os.environ.get("ANYSD_GEMM_SPLITK"), "ANYSD_GEMM_BN =", os.environ.get("ANYSD_GEMM_BN"), flush=True)
    for (Cin, Cout, H, W, res) in ((1280, 1280, 8, 8, True), (2560, 1280, 8, 8, False), (1280, 1280, 16, 16, True)):
        x = torch.randn(B, H, W, Cin, device="cuda", generator=g).half()
        w = (torch.randn(Cout, 9 * Cin, device="cuda", generator=g) * (9 * Cin) ** -0.5).half()
        bias = torch.randn(Cout, device="cuda", generator=g) * 0.1
        r = torch.randn(B * H * W, Cout, device="cuda", generator=g).half() if res else None
        out = torch.empty(B * H * W, Cout, dtype=torch.float16, device="cuda")
        t = timeit(lambda: ops.conv3x3(x, w, out, bias=bias, residual=r, stats=True))
        fl = 2.0 * B * H * W * 9 * Cin * Cout
        print(f"conv  N={B} {Cin:4d}->{Cout:4d} @{H}x{W} res={int(res)}: {t * 1e6:8.1f} us  {fl / t / 1e12:7.1f} TFLOP/s", flush=True)
    for (M, N, K, rpb) in ((1024, 1280, 5120, 64), (1024, 1280, 2560, 64), (1024, 1280, 1280, 64)):
        A = torch.randn(M, K, device="cuda", generator=g).half()
        W_ = (torch.randn(N, K, device="cuda", generator=g) * K ** -0.5).half()
        out = torch.empty(M, N, dtype=torch.float16, device="cuda")
        r = torch.randn(M, N, device="cuda", generator=g).half()
        t = timeit(lambda: ops.gemm(A, W_, out, residual=r, rows_per_batch=rpb))
        print(f"gemm  M={M} N={N} K={K} rows/image={rpb}: {t * 1e6:8.1f} us  {2.0 * M * N * K / t / 1e12:7.1f} TFLOP/s", flush=True)


if __name__ == "__main__":
    main()
