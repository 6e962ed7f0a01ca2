"""GroupNorm(+SiLU) and LayerNorm (anyedit_b200/csrc/norm.cu, backward.cu) on every path, element by element against a float64
reference of the same fp16 inputs with two-pass statistics, plus the invariants the rest of the suite relies on:

* the two-launch GroupNorm (ANYSD_GN_FUSED=0) writes the same bits as the cooperative one-launch kernel;
* every output bit is independent of the batch position and size and of the run, on every path;
* a workspace zero-filled once can be reused by calls of any batch size, in any order, on every path;
* widths the kernels cannot launch are refused.

The switches (ANYSD_GN_RES, ANYSD_GN_FUSED, ANYSD_GNBWD_CLUSTER) are read once per process, so every forced setting runs in a
child process (this file with ``--worker``): the parent saves the inputs once, the child runs the cases through
``anyedit_b200.ops`` and saves what they wrote, the parent compares.  The natural selection runs in-process.

Forward bound per element, from the fp16 input x with group (row) statistics m, sigma, rstd = 1 / sqrt(sigma^2 + eps),
kappa = E[x^2] / sigma^2 of the group, z = (x - m) rstd gamma + beta and y = z or silu(z):

    e    = s (|gamma| rstd (dm + |x - m| dr) + 4u (|beta| + |z| + |gamma| rstd (|x| + |m|))) + [SiLU] 2^-20 (1 + |z|) |y|
    |out - y| <= e + 2^-11 (|y| + e) + 2^-25

u = 2^-24; s = 1.1 (the steepest slope of SiLU) when SiLU is fused, else 1; the 4u term is the fp32 apply (a = rstd gamma,
b = beta - m a, fma(x, a, b)); 2^-20 (1 + |z|) covers silu_fast (ex2.approx of an argument rounded relative to |z|, rcp.approx).
The statistics terms, with c the longest fp32 addition chain of the kernel (each addition rounds once relative to the running
sum, which is bounded by the sum of magnitudes):

    dm = c u (|m| + sigma)                       (mean|x| <= |m| + sigma)
    dr = c u             two-pass statistics     (register-resident GroupNorm, LayerNorm)
    dr = 2 c u kappa     single-pass chunks      (var = E[x^2] - m^2: |dvar| <= c u E[x^2] + 2 |m| c u mean|x| <= 3 c u kappa var,
                                                  halved by the square root, + the fp32 store of rstd)

    register-resident (gn_res_kernel): c = V (rows per thread) + 8 (row-lane fold) + ceil(cpg P / 32) (lane-strided group
        loop, P = RL / 8) + 5 (shuffle tree) + 4 (inv_cnt, the product, rsqrtf's 2 ulp)
    chunks (gn_stats_block): c = ceil(rows_per_block / R) (rows per thread) + R (fold 1) + cpg (fold 2) + 2; the fold over the
        chunks and the mean / variance are in double
    epilogue statistics: c = 32 + 2 (one 32-row slab per fp32 cell, folded in double), and the statistics are of the
        contraction's fp32 values, not of the fp16 x: dm += 1.01 2^-11 (|m| + sigma), dr += 1.01 2^-11 sqrt(kappa)
    LayerNorm (layernorm_row_stats): c = 8 VPL + log2(LPR) + 4

Backward bound per (image, group) -- per row for LayerNorm -- normwise, because dx = rstd (w - mean(w) - xhat mean(w xhat))
cancels (w = dy [silu'(z)] gamma); the reference is float64 autograd.  Over the group's n elements:

    ||dx - ref|| <= 2^-11 ||ref|| + 2^-25 sqrt(n) + c u (2 S + sqrt(kappa) T)
    S = rstd (||w|| + sqrt(n) (|mean(w)| + |mean(w xhat)|))          the terms before the cancellation; rstd's error
    T = rstd (sqrt(n) |mean(w xhat)| + [SiLU] 1/2 ||dy gamma^2 (1 + |xhat|)||)    the mean's error through xhat (|silu''| <= 1/2)

    gn_bwd_kernel: c = ceil(ceil(HW / CS) / RL) + RL + cpg + CS + 8 (two-pass mean and variance, RL = 256 / VC row lanes)
    ln_bwd_kernel: c = 8 ceil(C / 256) + 5 + 8
"""
import math
import os
import subprocess
import sys
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
U = 2.0 ** -24
H11 = 2.0 ** -11
SILU_SLOPE = 1.1
SENTINEL = 0x7E5A                   # an fp16 NaN no kernel writes
KAPPAS = (1, 256, 4096)
CS_FORCED = (1, 2, 4, 8)
ENV_SWITCHES = ("ANYSD_GN_RES", "ANYSD_GN_FUSED", "ANYSD_GNBWD_CLUSTER", "ANYSD_GN_EPILOGUE")


def _cdiv(a, b):
    return -(-a // b)


# ---- restated geometry (norm.cu / backward.cu): which path a shape takes and its longest fp32 chain ------------------------
def _res_plan(C, HW, G=32):                                  # gn_res_plan
    cpg = C // G
    gpc = 1
    while (gpc * cpg) % 8:
        gpc += 1
    VC = gpc * cpg // 8
    if G % gpc or VC > 16:
        return None
    RL = 64 if VC * 64 <= 512 else 32
    v = _cdiv(HW, RL)
    if v > 8:
        return None
    V = 1
    while V < v:
        V <<= 1
    return dict(VC=VC, RL=RL, gpc=gpc, V=V)


def _chunks(C, HW):                                          # anysd_groupnorm_nhwc_f16: rows per chunk, chunks per image, R
    R = max(1, 512 // (C // 8))
    batch = 8 * R
    rpb = batch * _cdiv(HW, batch * 64)
    return rpb, _cdiv(HW, rpb), R


def _c_gn(path, C, HW, G):
    cpg = C // G
    if path == "res":
        p = _res_plan(C, HW, G)
        return p["V"] + 8 + _cdiv(cpg * p["RL"] // 8, 32) + 5 + 4
    if path == "chunks":
        rpb, _, R = _chunks(C, HW)
        return _cdiv(rpb, R) + R + cpg + 2
    return 32 + 2                                            # epilogue statistics


def _gn_path(C, HW, G=32):
    return "res" if _res_plan(C, HW, G) else "chunks"


def _ln_inst(C):                                             # anysd_layernorm_f16: (LPR, VPL)
    CV = C // 8
    if CV <= 40:
        return (8, 1) if CV <= 8 else (8, 2) if CV <= 16 else (8, 3) if CV <= 24 else (8, 5)
    return (16, 5) if CV <= 80 else (32, 5) if CV <= 160 else (32, 8)


def _c_gn_bwd(C, HW, CS, G=32):
    cpg = C // G
    gpc = 1
    while (gpc * cpg) % 8:
        gpc += 1
    RL = 256 // (gpc * cpg // 8)
    return _cdiv(_cdiv(HW, CS), RL) + RL + cpg + CS + 8


def _natural_cs(HW):
    return 8 if HW >= 2048 else 1


# ---- case matrices ----------------------------------------------------------------------------------------------------
def _fwd(name, N, HW, C1, C2=0, kappa=1, silu=True, eps=1e-5, edge=False, G=32):
    return dict(name=name, N=N, HW=HW, C1=C1, C2=C2, C=C1 + C2, kappa=kappa, silu=silu, eps=eps, edge=edge, G=G)


def _fwd_cases():
    c = []
    # register-resident, every plan: C = 32 / 64 / 128 (gpc 8 / 4 / 2, VC 1), 320 (VC 5, RL 64), 640 | 320 (cpg 30: a group
    # straddles the sources, VC 15, RL 32), 2560 (VC 10), 4096 (VC 16, the limit); HW on both sides of every V boundary and
    # the first HW that leaves the path (8 RL + 1)
    for C1, C2 in ((32, 0), (64, 0), (128, 0), (320, 0), (640, 320), (2560, 0), (4096, 0)):
        RL = _res_plan(C1 + C2, 1)["RL"]
        for i, HW in enumerate((1, RL - 1, RL, RL + 1, 2 * RL, 2 * RL + 1, 4 * RL, 4 * RL + 1, 8 * RL, 8 * RL + 1)):
            c.append(_fwd(f"res{C1}+{C2}_hw{HW}", 3, HW, C1, C2, silu=i % 2 == 0, eps=1e-5 if i % 3 else 1e-6))
    # cooperative one-launch (and two-launch): the VAE and UNet sizes; N = 8 at 64^2 x 320 is 344 chunks
    for HW, C1, C2, N in ((513, 128, 0, 3), (576, 320, 0, 3), (1024, 640, 640, 3), (1024, 1280, 640, 3), (576, 1280, 1280, 1),
                          (4096, 320, 0, 3), (4096, 320, 0, 8), (9216, 320, 0, 1), (4096, 128, 0, 1), (65536, 256, 0, 1),
                          (65536, 512, 0, 1), (262144, 128, 0, 1), (1024, 4096, 0, 1)):
        c.append(_fwd(f"coop{C1}+{C2}_hw{HW}_n{N}", N, HW, C1, C2, silu=HW % 2 == 0))
    # DC offsets (kappa = 256, 4096) and the edges: a constant group, var ~ eps, |x| up to 6e4, an all-zero group
    for kappa in KAPPAS[1:]:
        for HW, C1, C2 in ((256, 320, 0), (64, 2560, 0), (4096, 320, 0), (1024, 640, 640)):
            for silu in (True, False):
                c.append(_fwd(f"k{kappa}_{C1}+{C2}_hw{HW}_{'silu' if silu else 'id'}", 3, HW, C1, C2, kappa=kappa, silu=silu))
    for eps in (1e-5, 1e-6):
        for HW, C1, C2 in ((256, 320, 0), (64, 2560, 0), (4096, 320, 0), (1024, 640, 320)):
            c.append(_fwd(f"edge{eps:g}_{C1}+{C2}_hw{HW}", 3, HW, C1, C2, eps=eps, edge=True, silu=HW != 64))
    return c


FWD = _fwd_cases()
FWD_BY = {c["name"]: c for c in FWD}
assert len(FWD_BY) == len(FWD)
RES_NAMES = [c["name"] for c in FWD if _gn_path(c["C"], c["HW"]) == "res"]
CHUNK_NAMES = [c["name"] for c in FWD if _gn_path(c["C"], c["HW"]) == "chunks"]


def _bwd_cases():
    c = []
    for C1, C2 in ((32, 0), (64, 0), (128, 0), (320, 0), (640, 320), (2560, 0)):
        for i, HW in enumerate((1, 9, 60, 2047, 2048, 4096, 9216)):
            if C1 == 2560 and HW == 9216:
                continue
            c.append(dict(name=f"bwd{C1}+{C2}_hw{HW}", N=2, HW=HW, C1=C1, C2=C2, C=C1 + C2, kappa=1, silu=i % 2 == 1, eps=1e-5))
    for kappa in KAPPAS[1:]:
        for C1, C2, HW in ((320, 0, 4096), (640, 320, 2048), (2560, 0, 60), (32, 0, 9)):
            for silu in (True, False):
                c.append(dict(name=f"bwd_k{kappa}_{C1}+{C2}_hw{HW}_{'silu' if silu else 'id'}", N=2, HW=HW, C1=C1, C2=C2,
                              C=C1 + C2, kappa=kappa, silu=silu, eps=1e-6 if silu else 1e-5))
    return c


BWD = _bwd_cases()
BWD_BY = {c["name"]: c for c in BWD}
LN_WIDTHS = (8, 64, 72, 128, 136, 192, 200, 320, 328, 512, 640, 648, 768, 1024, 1280, 1288, 1536, 2048)
LN_ROWS = (1, 31, 32, 33, 77, 4097)


# ---- inputs -----------------------------------------------------------------------------------------------------------
def _grouped(g, N, HW, G, cpg, kappa):
    """x [N, HW, G, cpg]: per (image, group) sigma in [0.5, 2] and a mean of +-sigma sqrt(kappa - 1)."""
    sig = 0.5 + 1.5 * torch.rand(N, 1, G, 1, generator=g)
    sign = torch.randint(0, 2, (N, 1, G, 1), generator=g) * 2.0 - 1.0
    return sign * sig * math.sqrt(kappa - 1) + sig * torch.randn(N, HW, G, cpg, generator=g)


def _gn_inputs(c, seed):
    g = torch.Generator().manual_seed(seed)
    N, HW, C, G = c["N"], c["HW"], c["C"], c["G"]
    x = _grouped(g, N, HW, G, C // G, c["kappa"])
    if c["edge"]:
        x[:, :, 0] = torch.tensor([0.75, -3.0, 1.0 / 3.0])[:N].view(N, 1, 1)     # constant groups: var = 0
        x[:, :, 1] = math.sqrt(c["eps"]) * torch.randn(N, HW, C // G, generator=g)   # var ~ eps
        x[:, :, 2] = (3e4 * torch.randn(N, HW, C // G, generator=g)).clamp(-6e4, 6e4)
        x[0, :, 3] = 0.0
    T = dict(x=x.reshape(N, HW, C).half(), gamma=1 + 0.3 * torch.randn(C, generator=g), beta=0.2 * torch.randn(C, generator=g))
    if c["edge"]:
        T["gamma"][: 2 * (C // G)] = torch.linspace(-1.5, 1.5, 2 * (C // G))   # negative gammas on the constant / tiny groups
    return T


def _gn_bwd_inputs(c, seed):
    g = torch.Generator().manual_seed(seed)
    N, HW, C = c["N"], c["HW"], c["C"]
    x = _grouped(g, N, HW, 32, C // 32, c["kappa"]).reshape(N, HW, C).half()
    return dict(x=x, dy=torch.randn(N, HW, C, generator=g).half(), gamma=1 + 0.3 * torch.randn(C, generator=g),
                beta=0.2 * torch.randn(C, generator=g))


def _ln_inputs(M, C, seed):
    """Rows cycle through kappa = 1, 256, 4096 (a mean of +-sigma sqrt(kappa - 1), sigma in [0.5, 2])."""
    g = torch.Generator().manual_seed(seed)
    sig = 0.5 + 1.5 * torch.rand(M, 1, generator=g)
    kap = torch.tensor(KAPPAS, dtype=torch.float32)[torch.arange(M) % 3].view(M, 1)
    sign = torch.randint(0, 2, (M, 1), generator=g) * 2.0 - 1.0
    x = (sign * sig * (kap - 1).sqrt() + sig * torch.randn(M, C, generator=g)).half()
    return dict(x=x, dy=torch.randn(M, C, generator=g).half(), gamma=1 + 0.3 * torch.randn(C, generator=g),
                beta=0.2 * torch.randn(C, generator=g))


def _fill(t):
    t.view(torch.int16).fill_(SENTINEL)
    return t


def _is_sent(t):
    return t.view(torch.int16) == SENTINEL


def _same(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


# ---- references and bounds --------------------------------------------------------------------------------------------
def _moments(x, dims):
    """Two-pass float64 mean, variance (population) and kappa = E[x^2] / var over ``dims`` (kappa 0 where var = 0)."""
    m = x.mean(dims, keepdim=True)
    var = ((x - m) ** 2).mean(dims, keepdim=True)
    kappa = torch.where(var > 0, (m * m + var) / var.clamp_min(1e-300), torch.zeros_like(var))
    return m, var, kappa


def _fwd_ratio(x, m, var, kappa, gamma, beta, eps, silu, out, c, two_pass, epi=False):
    """Worst err / bound over one tensor (shapes broadcast: x [.., k] with statistics reduced over the normalised dims)."""
    sig = var.sqrt()
    rstd = 1.0 / (var + eps).sqrt()
    z = (x - m) * rstd * gamma + beta
    y = z * torch.sigmoid(z) if silu else z
    dm = c * U * (m.abs() + sig)
    dr = c * U if two_pass else 2 * c * U * kappa
    if epi:
        dm = dm + 1.01 * H11 * (m.abs() + sig)
        dr = dr + 1.01 * H11 * kappa.sqrt()
    pre = gamma.abs() * rstd * (dm + (x - m).abs() * dr) + 4 * U * (beta.abs() + z.abs() + gamma.abs() * rstd * (x.abs() + m.abs()))
    e = SILU_SLOPE * pre + 2.0 ** -20 * (1 + z.abs()) * y.abs() if silu else pre
    bound = e + H11 * (y.abs() + e) + 2.0 ** -25
    err = (out.double() - y).abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
    worst = float(ratio.max())
    if not worst <= 1.0:
        bad = (ratio > 1) | ratio.isnan()
        idx = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError(f"{int(bad.sum())} elements out of bound, worst err/bound {worst:.3g}; first {idx} got "
                             f"{float(out[idx])!r} want {float(y[idx])!r}")
    return worst


def _check_gn(c, T, y, path):
    """Every image of a GroupNorm output against the float64 reference, one image at a time (memory)."""
    G, C, HW = c["G"], c["C"], c["HW"]
    cpg, cc = C // G, _c_gn(path, C, HW, G)
    gamma, beta = T["gamma"].double().view(1, G, cpg), T["beta"].double().view(1, G, cpg)
    worst = 0.0
    for n in range(c["N"]):
        x = T["x"][n].double().view(HW, G, cpg)
        m, var, kappa = _moments(x, (0, 2))
        try:
            worst = max(worst, _fwd_ratio(x, m, var, kappa, gamma, beta, c["eps"], c["silu"], y[n].view(HW, G, cpg), cc,
                                          path == "res", path == "epilogue"))
        except AssertionError as e:
            raise AssertionError(f"{c['name']} image {n}: {e}") from None
    return worst


def _check_all(names, check, label, note=lambda name: ""):
    """``check(name)`` on every case, so that one run reports every failing case; prints the worst err / bound per case."""
    failures = []
    for name in names:
        try:
            worst = f"{check(name):.3f}"
        except AssertionError as e:
            worst = "FAIL"
            failures.append(f"{label}: {str(e).splitlines()[0]}")
        print(f"{label:10s} {name:34s} worst err/bound {worst:6s} {note(name)}")
    return failures


def _gn_bwd_ref(c, T):
    """float64 autograd dx and the per-(image, group) quantities of the bound."""
    N, HW, C = c["N"], c["HW"], c["C"]
    x = T["x"].double().permute(0, 2, 1).requires_grad_(True)
    gamma, beta = T["gamma"].double(), T["beta"].double()
    y = F.group_norm(x, 32, gamma, beta, c["eps"])
    if c["silu"]:
        y = F.silu(y)
    dy = T["dy"].double().permute(0, 2, 1)
    y.backward(dy)
    dx = x.grad.permute(0, 2, 1).reshape(N, HW, 32, C // 32)
    xv = T["x"].double().view(N, HW, 32, C // 32)
    dyv = T["dy"].double().view(N, HW, 32, C // 32)
    gv, bv = gamma.view(32, C // 32), beta.view(32, C // 32)
    m, var, kappa = _moments(xv, (1, 3))
    rstd = 1.0 / (var + c["eps"]).sqrt()
    xh = (xv - m) * rstd
    return _bwd_terms(dx, dyv, xh, rstd, kappa, gv, bv, c["silu"], (1, 3))


def _bwd_terms(dx, dy, xh, rstd, kappa, gamma, beta, silu, dims):
    n = 1
    for d in dims:
        n *= dx.shape[d]
    w = dy * gamma
    if silu:
        z = xh * gamma + beta
        s = torch.sigmoid(z)
        w = w * s * (1 + z * (1 - s))
    nrm = lambda t: t.pow(2).sum(dims, keepdim=True).sqrt()
    mw, mwx = w.mean(dims, keepdim=True), (w * xh).mean(dims, keepdim=True)
    S = rstd * (nrm(w) + math.sqrt(n) * (mw.abs() + mwx.abs()))
    T = rstd * math.sqrt(n) * mwx.abs()
    if silu:
        T = T + rstd * 0.5 * nrm(dy * gamma * gamma * (1 + xh.abs()))
    return SimpleNamespace(dx=dx, ref_norm=nrm(dx), S=S, T=T, kappa=kappa, n=n, dims=dims)


def _bwd_ratio(r, got, cc):
    err = (got.double().view_as(r.dx) - r.dx).pow(2).sum(r.dims, keepdim=True).sqrt()
    bound = H11 * r.ref_norm + 2.0 ** -25 * math.sqrt(r.n) + cc * U * (2 * r.S + r.kappa.sqrt() * r.T)
    ratio = err / bound
    worst = float(ratio.max())
    if not worst <= 1.0:
        raise AssertionError(f"{int((ratio > 1).sum())} groups out of bound, worst err/bound {worst:.3g} at "
                             f"{tuple(int(v) for v in (ratio == ratio.max()).nonzero()[0])}")
    return worst


# ---- runs -------------------------------------------------------------------------------------------------------------
def _gn(ops, x, T, c, N, y, ws, G=None, stats=None):
    C1 = c["C1"]
    x1, x2 = (x[..., :C1].contiguous(), x[..., C1:].contiguous()) if c["C2"] else (x, None)
    ops.groupnorm(x1, T["gamma"], T["beta"], y, N, c["HW"], c["eps"], c["silu"], ws, x2=x2, G=G or c["G"], stats=stats)


def _run_fwd(ops, names, inputs):
    """Each case: y (an NaN-filled guard image follows it), a second run, and every image alone at batch 1."""
    out = {}
    for name in names:
        c = FWD_BY[name]
        T = {k: v.cuda() for k, v in inputs[name].items()}
        x = T["x"]
        N = c["N"]
        buf = _fill(torch.empty(N + 1, c["HW"], c["C"], dtype=torch.float16, device="cuda"))
        _gn(ops, x, T, c, N, buf[:N], ops.groupnorm_workspace(N))
        again = _fill(torch.empty_like(x))
        _gn(ops, x, T, c, N, again, ops.groupnorm_workspace(N))
        alone = _fill(torch.empty_like(x))
        for i in range(N):
            _gn(ops, x[i:i + 1], T, c, 1, alone[i:i + 1], ops.groupnorm_workspace(1))
        torch.cuda.synchronize()
        y = buf[:N]
        out[name] = dict(y=y.cpu(), guard=bool(_is_sent(buf[N]).all()), repeat=_same(y, again), alone=_same(y, alone))
    return out


def _run_bwd(ops, names, inputs):
    out = {}
    for name in names:
        c = BWD_BY[name]
        T = {k: v.cuda() for k, v in inputs[name].items()}
        C1, x = c["C1"], T["x"]
        x1, x2 = (x[..., :C1].contiguous(), x[..., C1:].contiguous()) if c["C2"] else (x, None)
        dx, dx2 = _fill(torch.empty_like(x)), _fill(torch.empty_like(x))
        for d in (dx, dx2):
            ops.groupnorm_bwd(x1, T["gamma"], T["beta"], T["dy"], d, c["N"], c["HW"], c["eps"], c["silu"], x2=x2)
        torch.cuda.synchronize()
        out[name] = dict(dx=dx.cpu(), repeat=_same(dx, dx2))
    return out


REUSE_STEPS = ((8, 32), (3, 32), (8, 32), (1, 32), (5, 32), (3, 64), (8, 32))


def _run_reuse(ops):
    """One workspace sized for N = 8 (G = 32), zero-filled once, used by the REUSE_STEPS calls in order on each path; every
    result must be bit-equal to the same call on a fresh workspace.  Returns the failures."""
    g = torch.Generator().manual_seed(77)
    failures = []
    old_min, ops.GN_EPILOGUE_MIN_ROWS = ops.GN_EPILOGUE_MIN_ROWS, 0
    try:
        for path, HW in (("resident", 256), ("statistics + apply", 4096), ("epilogue statistics", 1024)):
            c = _fwd("reuse", 8, HW, 320)
            T = {k: v.cuda() for k, v in _gn_inputs(c, 78 + HW).items()}
            stats = None
            if path == "epilogue statistics":
                A = torch.randn(8 * HW, 64, generator=g).half().cuda()
                W = (torch.randn(320, 64, generator=g) / 8).half().cuda()
                T["x"] = torch.empty(8, HW, 320, dtype=torch.float16, device="cuda")
                stats = ops.gemm(A, W, T["x"].view(-1, 320), bias=torch.randn(320, generator=g).cuda(), rows_per_batch=HW,
                                 stats_images=8)
                assert stats is not None, "no epilogue statistics for the reuse case"
            ws = ops.groupnorm_workspace(8, 32)
            for step, (N, G) in enumerate(REUSE_STEPS):
                st = stats if G == 32 else None
                y, y_fresh = _fill(torch.empty(N, HW, 320, dtype=torch.float16, device="cuda")), _fill(torch.empty(N, HW, 320, dtype=torch.float16, device="cuda"))
                _gn(ops, T["x"][:N], T, c, N, y, ws, G=G, stats=st)
                _gn(ops, T["x"][:N], T, c, N, y_fresh, ops.groupnorm_workspace(N, G), G=G, stats=st)
                torch.cuda.synchronize()
                if not _same(y, y_fresh):
                    bad = int((y.view(torch.int16) != y_fresh.view(torch.int16)).sum())
                    failures.append(f"{path}: step {step} (N={N}, G={G}) on the reused workspace differs from a fresh "
                                    f"workspace in {bad} of {y.numel()} elements")
    finally:
        ops.GN_EPILOGUE_MIN_ROWS = old_min
    return failures


# ---- fixtures ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from anyedit_b200 import ops as o
    sms, major, minor = o.device_info()
    assert (major, minor) == (9, 0), f"sm_90a kernels need a Hopper GPU (H100), got cc {major}.{minor}"
    return o


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    d = tmp_path_factory.mktemp("norm")
    fwd = {c["name"]: _gn_inputs(c, 1000 + i) for i, c in enumerate(FWD)}
    bwd = {c["name"]: _gn_bwd_inputs(c, 5000 + i) for i, c in enumerate(BWD)}
    torch.save(fwd, d / "fwd.pt")
    torch.save(bwd, d / "bwd.pt")
    refs = {}

    def bwd_ref(name):                                       # computed once, shared by every cluster size
        if name not in refs:
            refs[name] = _gn_bwd_ref(BWD_BY[name], bwd[name])
        return refs[name]
    return SimpleNamespace(dir=d, fwd=fwd, bwd=bwd, bwd_ref=bwd_ref)


@pytest.fixture(scope="module")
def natural(ops, data):
    return _run_fwd(ops, [c["name"] for c in FWD], data.fwd)


def _child(data, tag, env, job, names=()):
    """One child process with the switches ``env``; returns what its cases wrote."""
    out = data.dir / f"out_{tag}.pt"
    e = {k: v for k, v in os.environ.items() if k not in ENV_SWITCHES}
    e.update(env)
    cmd = [sys.executable, *(["-s"] if sys.flags.no_user_site else []), os.path.abspath(__file__), "--worker", job,
           str(data.dir), str(out), ",".join(names)]
    r = subprocess.run(cmd, env=e, cwd=ROOT, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, f"worker {tag} failed:\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"
    return torch.load(out)


def _bits_failures(c_names, got, label):
    f = []
    for n in c_names:
        g = got[n]
        if not g["guard"]:
            f.append(f"{label} {n}: the guard image after y was written")
        if not g["repeat"]:
            f.append(f"{label} {n}: two runs differ")
        if not g["alone"]:
            f.append(f"{label} {n}: an image alone at batch 1 differs from the batch")
    return f


def _coop_note(sms):
    def note(name):
        c = FWD_BY[name]
        if _gn_path(c["C"], c["HW"]) == "res":
            p = _res_plan(c["C"], c["HW"])
            return f"resident VC={p['VC']} RL={p['RL']} gpc={p['gpc']} V={p['V']}"
        rpb, S, R = _chunks(c["C"], c["HW"])
        return f"chunks N*S={c['N'] * S} (P <= 2 x {sms} SMs = {2 * sms}) rows/chunk={rpb} R={R}"
    return note


# ---- GroupNorm forward ------------------------------------------------------------------------------------------------
def test_groupnorm_natural_against_fp64(ops, data, natural):
    """Every case on the path the shape selects (register-resident or cooperative): the bound, the guard image, run-to-run
    bits, and each image's bits at batch 1."""
    names = [c["name"] for c in FWD]
    check = lambda n: _check_gn(FWD_BY[n], data.fwd[n], natural[n]["y"], _gn_path(FWD_BY[n]["C"], FWD_BY[n]["HW"]))
    failures = _check_all(names, check, "natural", _coop_note(ops.device_info()[0]))
    failures += _bits_failures(names, natural, "natural")
    assert not failures, "\n".join(failures)


def test_groupnorm_two_launch_bit_identical(data, natural):
    """ANYSD_GN_FUSED=0: gn_stats_kernel + gn_apply_kernel write the cooperative kernel's bits (and so meet its bound)."""
    got = _child(data, "two_launch", {"ANYSD_GN_FUSED": "0"}, "fwd", CHUNK_NAMES)
    failures = _bits_failures(CHUNK_NAMES, got, "two-launch")
    differ = [n for n in CHUNK_NAMES if not _same(got[n]["y"], natural[n]["y"])]
    for n in CHUNK_NAMES:
        print(f"two-launch {n:34s} bit-identical to the cooperative kernel: {n not in differ}")
    assert not differ, f"two-launch differs from the cooperative kernel: {differ}"
    assert not failures, "\n".join(failures)


def test_groupnorm_resident_off(data, natural):
    """ANYSD_GN_RES=0: the resident shapes through the cooperative kernel (single-pass statistics: their own bound)."""
    got = _child(data, "res_off", {"ANYSD_GN_RES": "0"}, "fwd", RES_NAMES)
    check = lambda n: _check_gn(FWD_BY[n], data.fwd[n], got[n]["y"], "chunks")
    failures = _check_all(RES_NAMES, check, "res=0") + _bits_failures(RES_NAMES, got, "res=0")
    assert not failures, "\n".join(failures)
    assert any(not _same(got[n]["y"], natural[n]["y"]) for n in RES_NAMES), "ANYSD_GN_RES=0 did not change any result"


# (HW, N, parts, kappa): N * cdiv(HW, 4 R nb) against 2 x 132 SMs gives the apply chunking nb = 1, 2, 4, 8 at C = 320 (R = 12)
EPI_CASES = ((32, 1, 1, 1), (9216, 3, 1, 256), (4096, 16, 1, 1), (9216, 16, 1, 4096), (1024, 2, 2, 1), (4096, 2, 2, 4096),
             (1024, 16, 2, 256))


def _epi_nb(C, HW, N, sms):                                  # anysd_groupnorm_apply_nhwc_f16
    batch = 4 * max(1, 512 // (C // 8))
    nb = 8
    while nb > 1 and N * _cdiv(HW, batch * nb) < 2 * sms:
        nb >>= 1
    return nb


def test_groupnorm_epilogue_statistics(ops):
    """Statistics from the producing contraction's epilogue (one producer, and two for a channel concat 320 | 640 whose group
    10 straddles them) against the fp64 bound of that path; the same tensor through the statistics-computing path too."""
    sms = ops.device_info()[0]
    g = torch.Generator().manual_seed(99)
    failures, nbs = [], set()
    old, ops.GN_EPILOGUE_MIN_ROWS = ops.GN_EPILOGUE_MIN_ROWS, 0
    try:
        for HW, N, parts, kappa in EPI_CASES:
            widths = (320,) if parts == 1 else (320, 640)
            outs, sts = [], []
            for Cp in widths:
                A = torch.randn(N * HW, 64, generator=g).half().cuda()
                W = (torch.randn(Cp, 64, generator=g) / 8).half().cuda()
                sign = torch.randint(0, 2, (Cp,), generator=g) * 2.0 - 1.0
                bias = sign * math.sqrt(kappa - 1) + 0.1 * torch.randn(Cp, generator=g)   # the output's sigma is ~1
                o = torch.empty(N * HW, Cp, dtype=torch.float16, device="cuda")
                st = ops.gemm(A, W, o, bias=bias.cuda(), rows_per_batch=HW, stats_images=N)
                assert st is not None and st.S * 32 == HW
                outs.append(o)
                sts.append(st)
            C = sum(widths)
            x = torch.cat(outs, 1) if parts == 2 else outs[0]
            stats = sts[0] if parts == 1 else ops.GnStats(sts[0].parts + sts[1].parts, sts[0].S)
            c = _fwd(f"epi_hw{HW}_n{N}_p{parts}_k{kappa}", N, HW, C, 0, kappa=kappa, silu=HW != 1024, eps=1e-5)
            T = dict(x=x.view(N, HW, C), gamma=(1 + 0.3 * torch.randn(C, generator=g)).cuda(),
                     beta=(0.2 * torch.randn(C, generator=g)).cuda())
            y_epi, y_own = (_fill(torch.empty(N, HW, C, dtype=torch.float16, device="cuda")) for _ in range(2))
            _gn(ops, T["x"], T, c, N, y_epi, ops.groupnorm_workspace(N), stats=stats)
            _gn(ops, T["x"], T, c, N, y_own, ops.groupnorm_workspace(N))
            torch.cuda.synchronize()
            Tc = {k: v.cpu() for k, v in T.items()}
            nb = _epi_nb(C, HW, N, sms)
            nbs.add(nb)
            for label, y, path in (("epilogue", y_epi, "epilogue"), ("own", y_own, _gn_path(C, HW))):
                try:
                    worst = f"{_check_gn(c, Tc, y.cpu(), path):.3f}"
                except AssertionError as e:
                    worst = "FAIL"
                    failures.append(f"{label}: {e}")
                print(f"{label:10s} {c['name']:34s} worst err/bound {worst:6s} "
                      + (f"nb={nb}" if label == "epilogue" else f"path={path}"))
    finally:
        ops.GN_EPILOGUE_MIN_ROWS = old
    assert not failures, "\n".join(failures)
    print(f"apply chunkings exercised: nb in {sorted(nbs)}")


def test_groupnorm_workspace_reuse(ops):
    """Resident, cooperative and epilogue-statistics paths on one workspace reused across batch sizes (and group counts)."""
    failures = _run_reuse(ops)
    assert not failures, "\n".join(failures)


def test_groupnorm_workspace_reuse_two_launch(data):
    """The same on the two-launch path, whose per-image completion counters live in the workspace."""
    failures = _child(data, "reuse_two_launch", {"ANYSD_GN_FUSED": "0"}, "reuse")
    assert not failures, "\n".join(failures)


def test_groupnorm_width_limits(ops):
    """C = 4096 runs on the resident and the cooperative paths (natural cases res4096+0_*, coop4096+0_*); wider is refused
    up front (ANYSD_EUNSUPPORTED, raised as ValueError): the statistics + apply kernels give a row's C / 8 channel vectors one
    thread each (<= 512)."""
    for C in (4128, 8192):
        for HW in (256, 1024):
            x = torch.zeros(1, HW, C, dtype=torch.float16, device="cuda")
            gam, bet = torch.ones(C, device="cuda"), torch.zeros(C, device="cuda")
            with pytest.raises(ValueError, match="at most 4096"):
                ops.groupnorm(x, gam, bet, torch.empty_like(x), 1, HW, 1e-5, True, ops.groupnorm_workspace(1))
        st = ops.GnStats([(torch.zeros(1, 1024 // 32, C, 2, device="cuda"), C)], 1024 // 32)
        x = torch.zeros(1, 1024, C, dtype=torch.float16, device="cuda")
        with pytest.raises(ValueError, match="at most 4096"):
            ops.groupnorm(x, gam, bet, torch.empty_like(x), 1, 1024, 1e-5, True, ops.groupnorm_workspace(1), stats=st)
    assert _res_plan(4096, 256) and not _res_plan(4096, 1024)
    assert {"res4096+0_hw256", "coop4096+0_hw1024_n1"} <= set(FWD_BY)


# ---- GroupNorm backward -----------------------------------------------------------------------------------------------
def _check_bwd(data, got, cs_of, label):
    names = [c["name"] for c in BWD]

    def check(n):
        c = BWD_BY[n]
        if not got[n]["repeat"]:
            raise AssertionError(f"{n}: two runs differ")
        try:
            return _bwd_ratio(data.bwd_ref(n), got[n]["dx"], _c_gn_bwd(c["C"], c["HW"], cs_of(c)))
        except AssertionError as e:
            raise AssertionError(f"{n}: {e}") from None
    return _check_all(names, check, label, lambda n: f"CS={cs_of(BWD_BY[n])} kappa={BWD_BY[n]['kappa']}")


def test_groupnorm_backward_natural(ops, data):
    got = _run_bwd(ops, [c["name"] for c in BWD], data.bwd)
    failures = _check_bwd(data, got, lambda c: _natural_cs(c["HW"]), "bwd")
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("cs", CS_FORCED)
def test_groupnorm_backward_forced_cluster(data, cs):
    """ANYSD_GNBWD_CLUSTER: CS CTAs per span of groups (at HW = 9 with CS = 8 the trailing CTAs get no rows)."""
    got = _child(data, f"cs{cs}", {"ANYSD_GNBWD_CLUSTER": str(cs)}, "bwd", [c["name"] for c in BWD])
    failures = _check_bwd(data, got, lambda c: cs, f"bwd CS={cs}")
    assert not failures, "\n".join(failures)


# ---- LayerNorm --------------------------------------------------------------------------------------------------------
def test_layernorm_every_instantiation(ops):
    """Forward (element-wise) and backward (per-row normwise) at every (LPR, VPL), full and partly filled, rows with
    kappa up to 4096, and M across the 8-warp block edges."""
    failures, seen = [], set()
    for i, C in enumerate(LN_WIDTHS):
        LPR, VPL = _ln_inst(C)
        seen.add((LPR, VPL))
        for j, M in enumerate(LN_ROWS):
            T = _ln_inputs(M, C, 300 + 10 * i + j)
            Tg = {k: v.cuda() for k, v in T.items()}
            y, dx = _fill(torch.empty(M + 1, C, dtype=torch.float16, device="cuda")), _fill(torch.empty(M + 1, C, dtype=torch.float16, device="cuda"))
            ops.layernorm(Tg["x"], Tg["gamma"], Tg["beta"], y[:M])
            ops.layernorm_bwd(Tg["x"], Tg["gamma"], Tg["dy"], dx[:M])
            torch.cuda.synchronize()
            y, dx = y.cpu(), dx.cpu()
            name = f"ln{C}_m{M}"
            try:
                assert _is_sent(y[M]).all() and _is_sent(dx[M]).all(), "the guard row after the output was written"
                x = T["x"].double()
                m, var, kappa = _moments(x, (1,))
                fw = _fwd_ratio(x, m, var, kappa, T["gamma"].double(), T["beta"].double(), 1e-5, False, y[:M], 8 * VPL + 5 + 4,
                                True)
                xr = x.clone().requires_grad_(True)
                F.layer_norm(xr, (C,), T["gamma"].double(), T["beta"].double(), 1e-5).backward(T["dy"].double())
                rstd = 1.0 / (var + 1e-5).sqrt()
                r = _bwd_terms(xr.grad, T["dy"].double(), (x - m) * rstd, rstd, kappa, T["gamma"].double(), None, False, (1,))
                bw = _bwd_ratio(r, dx[:M], 8 * _cdiv(C, 256) + 5 + 8)
                res = f"fwd {fw:.3f} bwd {bw:.3f}"
            except AssertionError as e:
                res = "FAIL"
                failures.append(f"{name}: {e}")
            print(f"layernorm  {name:14s} (LPR, VPL) = ({LPR}, {VPL}) worst err/bound {res}")
    assert seen == {(8, 1), (8, 2), (8, 3), (8, 5), (16, 5), (32, 5), (32, 8)}
    assert not failures, "\n".join(failures)


def test_layernorm_refusals(ops):
    """Wider than 2048 or not a multiple of 8: refused (ANYSD_EINVAL, raised as ValueError); the backward needs C % 8 == 0."""
    for C in (2056, 12):
        x = torch.zeros(4, C, dtype=torch.float16, device="cuda")
        g = torch.ones(C, device="cuda")
        with pytest.raises(ValueError, match="multiple of 8 and <= 2048"):
            ops.layernorm(x, g, torch.zeros(C, device="cuda"), torch.empty_like(x))
    x = torch.zeros(4, 12, dtype=torch.float16, device="cuda")
    with pytest.raises(ValueError, match="C % 8 == 0"):
        ops.layernorm_bwd(x, torch.ones(12, device="cuda"), x, torch.empty_like(x))


def _worker(argv):
    job, d, outp, names = argv[0], argv[1], argv[2], [n for n in argv[3].split(",") if n] if len(argv) > 3 else []
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from anyedit_b200 import ops
    if job == "fwd":
        res = _run_fwd(ops, names, torch.load(os.path.join(d, "fwd.pt")))
    elif job == "bwd":
        res = _run_bwd(ops, names, torch.load(os.path.join(d, "bwd.pt")))
    else:
        res = _run_reuse(ops)
    torch.save(res, outp)
    return 0


if __name__ == "__main__" and sys.argv[1:2] == ["--worker"]:
    sys.exit(_worker(sys.argv[2:]))
