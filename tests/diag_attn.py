#!/usr/bin/env python
"""Diagnostic (not a pytest file): attention kernel timing on the UNet's shapes. ANYSD_ATTN=mma|wgmma selects the kernel."""
import os
import sys

import torch

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
from anyedit_b200 import ops  # noqa: E402
from anyedit_b200.unet import head_stride_for  # noqa: E402


def run(B, heads, n, nkv, d, check=True):
    aux = "--aux" in sys.argv and d % 16 == 8
    hs = head_stride_for(d)
    C, Cp = heads * d, heads * hs
    g = torch.Generator(device="cuda").manual_seed(0)
    def mk(rows):
        t = torch.zeros(B, rows, heads, hs, dtype=torch.float16, device="cuda")
        t[..., :d] = torch.randn(B, rows, heads, d, device="cuda", generator=g).half()
        return t.reshape(B, rows, Cp)
    q, k, v = mk(n), mk(nkv), mk(nkv)
    qa = q
    if aux:                                  # operand contract of anysd_attn_params::aux_cols
        qa = (q.float() * (d ** -0.5 * 1.4426950408889634)).half()
        k.view(B, nkv, heads, hs)[..., d:d + 2] = 1.0
        v.view(B, nkv, heads, hs)[..., d] = 1.0
    out = torch.empty(B, n, C, dtype=torch.float16, device="cuda")
    fn = lambda: ops.attention(qa, k, v, out, B, heads, n, nkv, d, Cp, Cp, Cp, C, head_stride=hs, aux_cols=aux)
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        fn()
    e1.record()
    torch.cuda.synchronize()
    t = e0.elapsed_time(e1) / 5 * 1e-3
    err = float("nan")
    if check:
        qq = q.view(B, n, heads, hs)[..., :d].permute(0, 2, 1, 3).float()
        kk = k.view(B, nkv, heads, hs)[..., :d].permute(0, 2, 1, 3).float()
        vv = v.view(B, nkv, heads, hs)[..., :d].permute(0, 2, 1, 3).float()
        ref = torch.nn.functional.scaled_dot_product_attention(qq[:1], kk[:1], vv[:1])
        ref = ref.permute(0, 2, 1, 3).reshape(1, n, C)
        err = float((out[:1].float() - ref).norm() / ref.norm())
    fl = 4.0 * B * heads * n * nkv * d
    print(f"attn aux={int(aux)} B={B} h={heads} n={n} kv={nkv} d={d}: {t * 1e6:9.1f} us {fl / t / 1e12:7.1f} TFLOP/s rel={err:.2e}", flush=True)


if __name__ == "__main__" and "--experts" not in sys.argv:
    print("ANYSD_ATTN =", os.environ.get("ANYSD_ATTN"))
    if "--l0" in sys.argv:                       # only the d = 40 / 4096-token level (experiments on the paired kernel)
        run(16, 8, 4096, 4096, 40, check="--nocheck" not in sys.argv)
        sys.exit(0)
    for c in ((1, 2, 128, 128, 64), (1, 2, 256, 256, 40), (2, 8, 300, 77, 40), (1, 8, 256, 256, 80), (1, 8, 256, 256, 160)):
        run(*c)
    if "--quick" not in sys.argv:
        for c in ((16, 8, 4096, 4096, 40), (16, 8, 1024, 1024, 80), (16, 8, 256, 256, 160), (16, 8, 4096, 77, 40)):
            run(*c)


def run_experts(B=16, heads=8, n=4096, nvis=16, d=40, E=11):
    """python tests/diag_attn.py --experts: the AnySD expert streams of one layer (expert_attention) at the 64x64 level."""
    hs = head_stride_for(d)
    C, Cp = heads * d, heads * hs
    g = torch.Generator(device="cuda").manual_seed(0)
    q = torch.zeros(B, n, heads, hs, dtype=torch.float16, device="cuda")
    q[..., :d] = torch.randn(B, n, heads, d, device="cuda", generator=g).half()
    ekv = torch.zeros(B, nvis, E, 2, heads, hs, dtype=torch.float16, device="cuda")
    ekv[..., :d] = torch.randn(B, nvis, E, 2, heads, d, device="cuda", generator=g).half()
    gates = torch.rand(B, E, device="cuda", generator=g)
    out = torch.zeros(B, n, C, dtype=torch.float16, device="cuda")
    fn = lambda: ops.expert_attention(q.view(B * n, Cp), ekv.view(B * nvis, E * 2 * Cp), gates, out, B, heads, n, nvis, d, E, Cp, E * 2 * Cp, C,
                                      2 * Cp, Cp, d ** -0.5, head_stride=hs)
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        fn()
    e1.record()
    torch.cuda.synchronize()
    print(f"expert_attention B={B} h={heads} n={n} nvis={nvis} d={d} E={E}: {e0.elapsed_time(e1) / 5 * 1e3:.1f} us")


if "--experts" in sys.argv:
    run_experts()
