#!/usr/bin/env python
"""Diagnostic (not a pytest file): steady-state attention kernel time at the UNet's shapes.

Each shape is warmed up, then timed as the median of WINDOWS windows of LAUNCHES back-to-back launches (CUDA events), so
that clocks have settled and one slow window does not move the result.  Counted FLOPs are 4 B heads n_q n_kv d (d, not
the padded head width).  --aux runs the d % 16 == 8 shapes with the aux_cols operands the UNet packs.
    python tests/diag_attn_steady.py [--aux]"""
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
from anyedit_b200 import ops  # noqa: E402
from anyedit_b200.unet import head_stride_for  # noqa: E402

WINDOWS, LAUNCHES = 7, 50
SHAPES = ((16, 8, 4096, 4096, 40), (16, 8, 1024, 1024, 80), (16, 8, 256, 256, 160), (16, 8, 4096, 77, 40))


def run(B, heads, n, nkv, d, aux):
    aux = aux and d % 16 == 8
    hs = head_stride_for(d)
    C, Cp = heads * d, heads * hs
    g = torch.Generator(device="cuda").manual_seed(0)

    def mk(rows):
        t = torch.zeros(B, rows, heads, hs, dtype=torch.float16, device="cuda")
        t[..., :d] = torch.randn(B, rows, heads, d, device="cuda", generator=g).half()
        return t.reshape(B, rows, Cp)

    q, k, v = mk(n), mk(nkv), mk(nkv)
    if aux:                                  # operand contract of anysd_attn_params::aux_cols
        q = (q.float() * (d ** -0.5 * 1.4426950408889634)).half()
        k.view(B, nkv, heads, hs)[..., d:d + 2] = 1.0
        v.view(B, nkv, heads, hs)[..., d] = 1.0
    out = torch.empty(B, n, C, dtype=torch.float16, device="cuda")
    fn = lambda: ops.attention(q, k, v, out, B, heads, n, nkv, d, Cp, Cp, Cp, C, head_stride=hs, aux_cols=aux)
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(WINDOWS):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(LAUNCHES):
            fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / LAUNCHES * 1e-3)
    t = statistics.median(times)
    fl = 4.0 * B * heads * n * nkv * d
    print(f"attn aux={int(aux)} B={B} h={heads} n={n} kv={nkv} d={d}: {t * 1e6:9.1f} us {fl / t / 1e12:7.1f} TFLOP/s "
          f"(median of {WINDOWS} x {LAUNCHES}, spread {(max(times) - min(times)) / t:.1%})", flush=True)


if __name__ == "__main__":
    print(torch.cuda.get_device_name())
    for shape in SHAPES:
        run(*shape, aux="--aux" in sys.argv)
