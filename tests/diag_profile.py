#!/usr/bin/env python
"""Diagnostic (not a pytest file): the three dominant kernels on their bench shapes, each launched twice, for
   ncu --set full --clock-control none --import-source on -k regex:"attention_wgmma|gemm_wgmma|bwd_d" -o prof python tests/diag_profile.py"""
import os
import sys

import torch

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))
from anyedit_b200 import ops  # noqa: E402

B = 16
g = torch.Generator(device="cuda").manual_seed(0)
rn = lambda *s: torch.randn(*s, device="cuda", generator=g)

# 1. level-0 self-attention: 16 x 8 heads, 4096 tokens, d = 40 (head stride 48)
hs, heads, n, d = 48, 8, 4096, 40
qkv = torch.zeros(B, n, 3, heads, hs, dtype=torch.float16, device="cuda")
qkv[..., :d] = rn(B, n, 3, heads, d).half()
qkv[:, :, 0, :, :d] *= d ** -0.5 * 1.4426950408889634      # aux_cols contract: q pre-scaled, ones in K/V padding
qkv[:, :, 1, :, d:d + 2] = 1.0
qkv[:, :, 2, :, d] = 1.0
qkv = qkv.view(B * n, 3 * heads * hs)
Cp = heads * hs
out = torch.empty(B * n, heads * d, dtype=torch.float16, device="cuda")
for _ in range(2):
    ops.attention(qkv, qkv[:, Cp:], qkv[:, 2 * Cp:], out, B, heads, n, n, d, 3 * Cp, 3 * Cp, 3 * Cp, heads * d, head_stride=hs,
                  aux_cols=True)
# 2. conv3x3 320 -> 320 @ 64x64 with time-embedding row add and residual
x = rn(B, 64, 64, 320).half()
w = (rn(320, 9 * 320) * (2880 ** -0.5)).half()
bias, emb = rn(320) * 0.1, rn(B, 320)
res = rn(B * 4096, 320).half()
o2 = torch.empty(B * 4096, 320, dtype=torch.float16, device="cuda")
for _ in range(2):
    ops.conv3x3(x, w, o2, bias=bias, rowadd=emb, residual=res)
# 3. GEGLU projection 320 -> 2560 on 65536 tokens
a = rn(B * 4096, 320).half()
wg = (rn(2560, 320) * (320 ** -0.5)).half()
bg = rn(2560) * 0.1
o3 = torch.empty(B * 4096, 1280, dtype=torch.float16, device="cuda")
for _ in range(2):
    ops.gemm(a, wg, o3, bias=bg, act=2)
# 4. backward of 1. (the forward keeps its log-sum-exp)
lse = torch.empty(B, heads, n, dtype=torch.float32, device="cuda")
ops.attention(qkv, qkv[:, Cp:], qkv[:, 2 * Cp:], out, B, heads, n, n, d, 3 * Cp, 3 * Cp, 3 * Cp, heads * d, head_stride=hs, aux_cols=True, lse=lse)
d_out = (rn(B * n, heads * d) * 0.1).half()
dqkv = torch.empty_like(qkv)
for _ in range(2):
    ops.attention_bwd(qkv, qkv[:, Cp:], qkv[:, 2 * Cp:], d_out, dqkv, dqkv[:, Cp:], dqkv[:, 2 * Cp:], B, heads, n, n, d, 3 * Cp, 3 * Cp, 3 * Cp,
                      heads * d, 3 * Cp, 3 * Cp, 3 * Cp, qk_scale=0.6931471805599453, head_stride=hs, out=out, ld_o=heads * d, lse=lse)
torch.cuda.synchronize()
print("done")
