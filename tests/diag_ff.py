"""Kernel time of the 320-channel feed-forward at the UNet's row counts: the fused kernel (ops.geglu_ff) against the three
launches it replaces (ln3 -> ff1 + GEGLU -> ff2 + bias + residual), both fed the same LayerNorm output.

Both paths run interleaved in one process: per M, 7 windows of 50 launches of each, CUDA events around every window; the
median window is reported, with the FLOP rate of the two products (161 GFLOP at M = 65536).  The fused path's LayerNorm is
timed with it, so both columns cover the same work.

    python tests/diag_ff.py [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)

from anyedit_b200 import ops  # noqa: E402
from anyedit_b200.unet import ff1_chunk_order  # noqa: E402

C, HID = 320, 1280
WINDOWS, LAUNCHES = 7, 50


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name()
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(0)
    u = lambda shape, fan_in: (torch.rand(shape, generator=g) * 2 - 1) / fan_in ** 0.5
    w1, b1, w2, b2 = u((2 * HID, C), C), u((2 * HID,), C), u((C, HID), HID), u((C,), HID)
    ff1_w = torch.stack([w1[:HID], w1[HID:]], 1).reshape(2 * HID, C).half()
    ff1_b = torch.stack([b1[:HID], b1[HID:]], 1).reshape(-1).float()
    perm = ff1_chunk_order(HID)
    W = dict(ff1_w=ff1_w.to(dev), ff1_b=ff1_b.to(dev), ff2_w=w2.half().to(dev), ff2_b=b2.float().to(dev),
             ff1p_w=ff1_w[perm].contiguous().to(dev), ff1p_b=ff1_b[perm].contiguous().to(dev),
             ff2t_w=w2.half().t().contiguous().to(dev))
    ln_w, ln_b = torch.ones(C, device=dev), torch.zeros(C, device=dev)
    card = _card()
    print("card:", card)
    rows = []
    for M in (65536, 36864):
        t3 = torch.randn(M, C, generator=g).half().to(dev)
        ln3 = torch.empty_like(t3)
        hid = torch.empty(M, HID, dtype=torch.float16, device=dev)
        o3, of = torch.empty_like(t3), torch.empty_like(t3)

        def three():
            ops.layernorm(t3, ln_w, ln_b, ln3)
            ops.gemm(ln3, W["ff1_w"], hid, bias=W["ff1_b"], act=2)
            ops.gemm(hid, W["ff2_w"], o3, bias=W["ff2_b"], residual=t3)

        def fused():
            ops.layernorm(t3, ln_w, ln_b, ln3)
            ops.geglu_ff(ln3, W["ff1p_w"], W["ff1p_b"], W["ff2t_w"], W["ff2_b"], t3, of)

        def ln_only():
            ops.layernorm(t3, ln_w, ln_b, ln3)

        paths = {"three_launch": three, "fused": fused, "layernorm": ln_only}
        for f in paths.values():
            for _ in range(5):
                f()
        torch.cuda.synchronize()
        times = {k: [] for k in paths}
        for _ in range(WINDOWS):
            for k, f in paths.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(LAUNCHES):
                    f()
                e1.record()
                e1.synchronize()
                times[k].append(e0.elapsed_time(e1) * 1e3 / LAUNCHES)
        flop = 2.0 * M * 2 * HID * C + 2.0 * M * C * HID
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        same = bool(torch.equal(o3, of))
        row = {"M": M, "gflop": flop / 1e9, "bit_identical": same,
               "us": med, "spread_us": {k: [min(v), max(v)] for k, v in times.items()},
               "tflops_products": {k: flop / ((med[k] - med["layernorm"]) * 1e-6) / 1e12 for k in ("three_launch", "fused")}}
        rows.append(row)
        print(f"M={M}: three launches {med['three_launch']:.1f} us, fused {med['fused']:.1f} us (layernorm {med['layernorm']:.1f} us); "
              f"products at {row['tflops_products']['three_launch']:.0f} / {row['tflops_products']['fused']:.0f} TFLOP/s; "
              f"speed-up {med['three_launch'] / med['fused']:.2f}x; bit-identical: {same}")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "diag_ff.json"), "w") as f:
            json.dump({"card": card, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
