"""Kernel time of the 320-channel transformer blocks' span from the self-attention's output projection to the feed-forward's
LayerNorm, at the UNet's row counts: the six launches the UNet runs there, each on its own and as one chain.

    t2 = a1 Wo1^T + bo1 + t      (gemm + bias + residual)
    l2 = LayerNorm2(t2)
    q  = l2 Wq^T                 (8 heads padded to 48 columns, softmax scale and log2(e) folded into Wq)
    a2 = softmax(q K^T) V        (77 context keys per image, d = 40, aux_cols operands)
    t3 = a2 Wo2^T + bo2 + t2     (gemm + bias + residual)
    l3 = LayerNorm3(t3)

The fused kernel (ops.xattn_block) does the same work in one launch.  Per M: 7 windows of 50 launches of every path,
interleaved, CUDA events around every window; the median window is reported with the spread.  The context K/V are
computed once (the sampler keeps them across steps) and not timed.

    python tests/diag_xattn.py [--out DIR]
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
from anyedit_b200.unet import LOG2E, aux_bias, pad_heads  # noqa: E402

C, HEADS, D, HS, L, CTX = 320, 8, 40, 48, 77, 768
CP = HEADS * HS
WINDOWS, LAUNCHES = 7, 50
SHAPES = ((16, 4096), (4, 9216))       # (images, rows per image): M = 65536 and 36864


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name()
    return q


def weights(dev, g):
    u = lambda shape, fan_in: (torch.rand(shape, generator=g) * 2 - 1) / fan_in ** 0.5
    wq = pad_heads(u((C, C), C) * (D ** -0.5 * LOG2E), HEADS, D, HS)
    wkv = torch.cat([pad_heads(u((C, CTX), CTX), HEADS, D, HS), pad_heads(u((C, CTX), CTX), HEADS, D, HS)], 0)
    kv_b = torch.cat([aux_bias(HEADS, D, HS, 2), aux_bias(HEADS, D, HS, 1)])
    h, f = (lambda t: t.half().contiguous().to(dev)), (lambda t: t.float().contiguous().to(dev))
    return dict(o1_w=h(u((C, C), C)), o1_b=f(u((C,), C)), ln2_w=f(1 + 0.1 * torch.randn(C, generator=g)),
                ln2_b=f(0.1 * torch.randn(C, generator=g)), q_w=h(wq), kv_w=h(wkv), kv_b=f(kv_b),
                o2_w=h(u((C, C), C)), o2_b=f(u((C,), C)), ln3_w=f(1 + 0.1 * torch.randn(C, generator=g)),
                ln3_b=f(0.1 * torch.randn(C, generator=g)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(0)
    W = weights(dev, g)
    card = _card()
    print("card:", card)
    rows = []
    for B, n in SHAPES:
        M = B * n
        a1 = torch.randn(M, C, generator=g).half().to(dev)
        t = torch.randn(M, C, generator=g).half().to(dev)
        ctx = torch.randn(B * L, CTX, generator=g).half().to(dev)
        kv = torch.empty(B * L, 2 * CP, dtype=torch.float16, device=dev)
        ops.gemm(ctx, W["kv_w"], kv, bias=W["kv_b"])
        t2, l2, t3, l3 = (torch.empty_like(t) for _ in range(4))
        q = torch.empty(M, CP, dtype=torch.float16, device=dev)
        a2 = torch.empty(M, C, dtype=torch.float16, device=dev)

        steps = {
            "to_out1": lambda: ops.gemm(a1, W["o1_w"], t2, bias=W["o1_b"], residual=t),
            "layernorm2": lambda: ops.layernorm(t2, W["ln2_w"], W["ln2_b"], l2),
            "to_q2": lambda: ops.gemm(l2, W["q_w"], q),
            "xattn": lambda: ops.attention(q, kv, kv[:, CP:], a2, B, HEADS, n, L, D, CP, 2 * CP, 2 * CP, C,
                                           head_stride=HS, aux_cols=True),
            "to_out2": lambda: ops.gemm(a2, W["o2_w"], t3, bias=W["o2_b"], residual=t2),
            "layernorm3": lambda: ops.layernorm(t3, W["ln3_w"], W["ln3_b"], l3),
        }

        def chain():
            for f in steps.values():
                f()

        f2, f3, fl3 = (torch.empty_like(t) for _ in range(3))

        def fused():
            ops.xattn_block(a1, t, W["o1_w"], W["o1_b"], W["ln2_w"], W["ln2_b"], W["q_w"], kv, L, W["o2_w"], W["o2_b"],
                            W["ln3_w"], W["ln3_b"], f2, f3, fl3, n, HEADS, D, HS)

        paths = dict(steps, chain=chain, fused=fused)
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
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        row = {"M": M, "B": B, "n": n, "us": med, "spread_us": {k: [min(v), max(v)] for k, v in times.items()},
               "sum_of_launches_us": sum(med[k] for k in steps),
               "bit_identical": bool(torch.equal(t2, f2) and torch.equal(t3, f3) and torch.equal(l3, fl3))}
        rows.append(row)
        print(f"M={M} (B={B}, n={n}): " + ", ".join(f"{k} {med[k]:.1f}" for k in steps) +
              f" us; sum {row['sum_of_launches_us']:.1f} us; chain {med['chain']:.1f} us "
              f"(spread {min(times['chain']):.1f}-{max(times['chain']):.1f}); fused {med['fused']:.1f} us "
              f"(spread {min(times['fused']):.1f}-{max(times['fused']):.1f}); speed-up {med['chain'] / med['fused']:.2f}x; "
              f"bit-identical: {row['bit_identical']}")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "diag_xattn.json"), "w") as f:
            json.dump({"card": card, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
