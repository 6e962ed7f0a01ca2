"""The persistent wgmma contraction (anyedit_b200/csrc/gemm_wgmma.cu) at every tile width and epilogue, element by element
against a float64 CPU reference, plus the invariants the rest of the suite relies on without stating them:

* one output element (and its GroupNorm / LayerNorm statistics) is bit-identical whatever tile width the cost model picks
  -- the whole-UNet batch-independence test silently depends on it, because the width depends on the batch size;
* split-K (the natural rule and forced uneven splits) meets the same bound, is batch-independent and re-arms its counters;
* the mma.sync fallback (ANYSD_GEMM=mma) meets the bound on its own, and the switch really selects it;
* requests a kernel cannot serve are refused loudly, or answered with ``None`` where the API says so.

The width (ANYSD_GEMM_BN), the split count (ANYSD_GEMM_SPLITK) and the kernel (ANYSD_GEMM) are read once per process, so every
forced setting runs in a child process (this file with ``--worker``): the parent saves the inputs once, the child runs the
cases through ``anyedit_b200.ops`` and saves what they wrote, the parent compares.  The natural selection runs in-process.

Bound per output element, from the fp16-rounded operands (``_reference``):

    |out - ref| <= 2^-11 |ref| + 2^-25            (fp16 output: round to nearest, incl. the subnormal half step)
                 + s * C_ACC 2^-24 (K (|A| |W|^T) + |bias| + |rowadd|)
                 + activation slack             (1.2e-5 for the fitted GELU of fp16 outputs, x |a| for GEGLU)

with s = 1.13, the steepest slope of SiLU / GELU / QuickGELU (1 without an activation).  C_ACC = 4: the tensor cores add
their fp32 partial sums with truncation, not round-to-nearest, so one addition may lose a full ulp (2 x 2^-24 relative, the
worst case K (|A| |W|^T) term with c = 2); the other factor 2 covers the fp32 epilogue additions (bias, row add, residual),
each rounding once relative to the running magnitude.
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
WIDTHS = (64, 128, 192, 256)
SPLITS = (2, 5, 8)
GUARD = 16                         # sentinel rows above and below every output window
COL0 = 8                           # first column of the output / residual / row-add window inside its wider buffer
SENTINEL = {torch.float16: (torch.int16, 0x7E5A), torch.float32: (torch.int32, 0x7FA5A5A5)}   # NaNs no kernel writes
U = 2.0 ** -24
C_ACC = 4
SLOPE = 1.13
P_GELU_FIT = 1.2e-5                # |x Phi(x) - p_gelu(x)| (gemm_wgmma.cu), used by the fp16-output GELU / GEGLU epilogues


# ---- the case matrix ------------------------------------------------------------------------------------------------
def _dense(name, M, N, K, act=0, f32=False, bias=True, rpb=0, rowadd=False, res=False, a_slice=False, w_slice=False,
           stats=False, row_stats=False, ln=False):
    return dict(name=name, kind="dense", M=M, N=N, K=K, act=act, f32=f32, bias=bias, rpb=rpb, rowadd=rowadd, res=res,
                a_slice=a_slice, w_slice=w_slice, stats=stats, row_stats=row_stats, ln=ln, pad_rb=False)


def _conv(name, Nimg, H, W, Cin, Cout, stride=1, up=0, pad_rb=False, act=0, f32=False, rowadd=True, res=True, stats=False,
          live_cout=None):
    return dict(name=name, kind="conv", Nimg=Nimg, H=H, W=W, Cin=Cin, N=Cout, K=9 * Cin, stride=stride, up=up, pad_rb=pad_rb,
                act=act, f32=f32, bias=True, rowadd=rowadd, res=res, stats=stats, live_cout=live_cout, row_stats=False, ln=False)


def _main_cases():
    c = []
    # M = 1000: ragged (8 row tiles, the last one 104 rows); N = 448: a partial last column tile at every width
    # (7 x 64, 3 x 128 + 64, 2 x 192 + 64, 256 + 192); K = 392 = 6 x 64 + 8: a K tail, and 7 k-blocks per unit -- coprime to
    # both stage counts (6 at BN 64 / 128, 4 at BN 192 / 256), so the operand ring's phase wraps across unit boundaries.
    # K = 8: one k-block that is all tail; the accumulation term is small there, so the activation slack is what bites.
    M, N, K = 1000, 448, 392
    for f32 in (False, True):
        t = "f32" if f32 else "f16"
        c.append(_dense(f"dense_bias_{t}", M, N, K, f32=f32))
        c.append(_dense(f"dense_rowadd_res_{t}", M, N, K, f32=f32, rpb=200, rowadd=True, res=True))
        for act in (1, 3, 4):
            c.append(_dense(f"dense_act{act}_{t}", M, N, K, act=act, f32=f32, rpb=200, rowadd=True, res=True))
            c.append(_dense(f"dense_k8_act{act}_{t}", 300, 320, 8, act=act, f32=f32, res=True))
        c.append(_dense(f"dense_geglu_{t}", M, N, K, act=2, f32=f32, rpb=200, rowadd=True))
        c.append(_dense(f"dense_geglu_res_{t}", M, N, K, act=2, f32=f32, rpb=200, rowadd=True, res=True))
        c.append(_dense(f"dense_k8_geglu_res_{t}", 300, 320, 8, act=2, f32=f32, res=True))
        c.append(_dense(f"dense_strided_{t}", M, N, K, f32=f32, rpb=200, rowadd=True, res=True, a_slice=True, w_slice=True))
    # 71 row tiles x 2..5 column tiles: 142..355 units on 132 SMs at every width (several units per CTA)
    c.append(_dense("dense_many_units", 9001, 320, 264, rpb=200, rowadd=True, res=True))
    # statistics: GroupNorm (9 images of 1024 rows, 144..360 units), LayerNorm row statistics, the LayerNorm-fold consumer
    c.append(_dense("dense_gn_stats", 9216, 320, 264, rpb=1024, res=True, stats=True))
    c.append(_dense("dense_row_stats_320", 1000, 320, 392, res=True, row_stats=True))
    c.append(_dense("dense_row_stats_640", 1000, 640, 264, res=True, row_stats=True))
    for act in (0, 1, 2):
        c.append(_dense(f"dense_ln_fold_act{act}", 1000, 448, 320, act=act, ln=True, res=act == 0))
    # conv: one patch geometry per branch of p_pick_extent (64 -> 64x2, 96 -> 32x4, 48 -> 16x8, 24 / 40 / 8 -> 8x8x2,
    # 4x8 -> 8x4x4, 12x20 -> 4x4x8, overshooting 6x10 / 9x7 stride 2 / 13x11 right-bottom padded), upsample, odd batches
    c += [_conv("conv_64sq_cin64", 2, 64, 64, 64, 320, stats=True),
          _conv("conv_96sq", 1, 96, 96, 64, 128, stats=True),
          _conv("conv_48sq_cin128", 2, 48, 48, 128, 320, stats=True),
          _conv("conv_24sq_b3", 3, 24, 24, 64, 192, stats=True),
          _conv("conv_40sq_b3", 3, 40, 40, 64, 64, stats=True),
          _conv("conv_8sq_b5_cin320", 5, 8, 8, 320, 320, stats=True),
          _conv("conv_4x8_b5", 5, 4, 8, 64, 128, stats=True),
          _conv("conv_12x20", 2, 12, 20, 128, 128),
          _conv("conv_6x10_overshoot", 2, 6, 10, 64, 64),
          _conv("conv_s2_9x7_b3", 3, 9, 7, 64, 96, stride=2),
          _conv("conv_up_8x12", 2, 8, 12, 128, 128, up=1, stats=True),
          _conv("conv_pad_rb_16sq", 2, 16, 16, 64, 64, stride=2, pad_rb=True, stats=True),
          _conv("conv_pad_rb_13x11_b3", 3, 13, 11, 64, 64, stride=2, pad_rb=True),
          _conv("conv_silu", 2, 16, 16, 64, 128, act=1),
          # the UNet's output conv: 4 channels padded to 8 with zero weights, fp32 output, bias only
          _conv("conv_out_f32", 2, 32, 32, 320, 8, f32=True, rowadd=False, res=False, live_cout=4)]
    return c


# Forced splits need rows_per_image <= 128; 90 k-blocks (Cin 640) and 71 (K = 70 x 64 + 8) leave an uneven last split
SPLIT_CASES = [_conv("split_conv_cin640", 3, 8, 8, 640, 320, stats=True),
               _dense("split_dense_rpb96", 480, 320, 4488, rpb=96, rowadd=True, res=True, stats=True)]
MAIN_CASES = _main_cases()
ALL = MAIN_CASES + SPLIT_CASES
CASES = {c["name"]: c for c in ALL}
assert len(CASES) == len(ALL)
MMA_NAMES = [c["name"] for c in ALL if not (c["row_stats"] or c["ln"] or c["pad_rb"])]


def _conv_out(c):
    Hl, Wl = c["H"] << c["up"], c["W"] << c["up"]
    if c["pad_rb"]:
        return (Hl - 2) // 2 + 1, (Wl - 2) // 2 + 1
    return (Hl - 1) // c["stride"] + 1, (Wl - 1) // c["stride"] + 1


def _rows(c):
    if c["kind"] == "dense":
        return c["M"]
    Ho, Wo = _conv_out(c)
    return c["Nimg"] * Ho * Wo


def _n_out(c):
    return c["N"] // 2 if c["act"] == 2 else c["N"]


def _rows_per_image(c):
    if c["kind"] == "dense":
        return c["rpb"]
    Ho, Wo = _conv_out(c)
    return Ho * Wo


def _cdiv(a, b):
    return -(-a // b)


def _pick_extent(n, cap):          # gemm_wgmma.cu p_pick_extent
    lim = 1
    while lim < n:
        lim <<= 1
    lim = min(lim, cap)
    e = lim
    while e >= 4:
        if n % e == 0:
            return e
        e >>= 1
    return lim


def _natural_width(c, sms):
    """The width and split count p_select picks for a case (only printed: the tests cannot observe the choice)."""
    if c["kind"] == "conv":
        Ho, Wo = _conv_out(c)
        bw = _pick_extent(Wo, 128)
        bh = _pick_extent(Ho, 128 // bw)
        nb = 128 // (bw * bh)
        tiles_m, num_kb = _cdiv(Wo, bw) * _cdiv(Ho, bh) * _cdiv(c["Nimg"], nb), 9 * c["Cin"] // 64
    else:
        tiles_m, num_kb = _cdiv(c["M"], 128), _cdiv(c["K"], 64)
    sp = 3 if (c["kind"] == "conv" and num_kb >= 256 and 0 < _rows_per_image(c) <= 128 and not c["f32"] and c["act"] != 2) else 1
    best, bn = None, 256
    for w in (256, 192, 128, 64):
        cost = _cdiv(tiles_m * _cdiv(c["N"], w) * sp, sms) * (w + 270) * (_cdiv(num_kb, sp) + (8 if sp > 1 else 0))
        if best is None or cost < best:
            best, bn = cost, w
    return bn, sp


# ---- inputs, runs, references ---------------------------------------------------------------------------------------
def _make_inputs(c, seed):
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g)
    N, K, rows, n_out = c["N"], c["K"], _rows(c), _n_out(c)
    T = {}
    wscale = 1.5 * K ** -0.5                       # pre-activations ~ N(0, 1.5^2): the activations' curved range
    if c["kind"] == "dense":
        M = c["M"]
        T["A"] = (rn(M, K + 64 if c["a_slice"] else K) + (0.5 if c["ln"] else 0.0)).half()
        T["W"] = (rn(N, K + 64 if c["w_slice"] else K) * wscale).half()
        if c["ln"]:                                # per-(64-column slab, row) moments of A: what a producer's row_stats holds
            a = T["A"].double().view(M, K // 64, 64)
            T["ln_stats"] = torch.stack([a.sum(-1), (a * a).sum(-1)], -1).permute(1, 0, 2).float().contiguous()
            T["colsum"] = T["W"].float().sum(1)
        n_img = _cdiv(M, c["rpb"]) if c["rpb"] else 1
    else:
        T["x"] = rn(c["Nimg"], c["H"], c["W"], c["Cin"]).half()
        T["W"] = (rn(N, K) * wscale).half()
        n_img = c["Nimg"]
    T["bias"] = 0.1 * rn(N)
    if c.get("live_cout"):
        T["W"][c["live_cout"]:] = 0
        T["bias"][c["live_cout"]:] = 0
    if c["rowadd"]:
        T["rowadd"] = rn(n_img, N + 16)
    if c["res"]:
        T["res"] = rn(rows, n_out + 16).half()
    return T


def _fill_sentinel(t):
    dt, v = SENTINEL[t.dtype]
    t.view(dt).fill_(v)
    return t


def _is_sentinel(t):
    dt, v = SENTINEL[t.dtype]
    return t.view(dt) == v


def _run_cases(ops, cases, inputs):
    """Run every case through anyedit_b200.ops on cuda:0.  Outputs are windows of sentinel-filled buffers; the statistics
    buffers are sentinel-filled too (ops._want_stats wrapped), so a slab no unit wrote shows."""
    want_stats, want_splitk, min_rows = ops._want_stats, ops._want_splitk, ops.GN_EPILOGUE_MIN_ROWS
    split = []

    def stats_sentinel(p, images, dev, reuse=None):
        st = want_stats(p, images, dev, reuse)
        if st is not None:
            _fill_sentinel(st.parts[0][0])
        return st

    def splitk_seen(p, dev):
        ws = want_splitk(p, dev)
        split.append(ws is not None)
        return ws

    ops._want_stats, ops._want_splitk, ops.GN_EPILOGUE_MIN_ROWS = stats_sentinel, splitk_seen, 0
    results = {}
    try:
        for c in cases:
            T = {k: v.cuda() for k, v in inputs[c["name"]].items()}
            N, K, rows, n_out = c["N"], c["K"], _rows(c), _n_out(c)
            odt = torch.float32 if c["f32"] else torch.float16
            buf = _fill_sentinel(torch.empty(rows + 2 * GUARD, COL0 + n_out + 16, dtype=odt, device="cuda"))
            out = buf[GUARD:GUARD + rows, COL0:COL0 + n_out]
            rowadd = T["rowadd"][:, COL0:COL0 + N] if c["rowadd"] else None
            res = T["res"][:, COL0:COL0 + n_out] if c["res"] else None
            del split[:]
            rs = None
            if c["kind"] == "dense":
                A = T["A"][:, 64:] if c["a_slice"] else T["A"]
                W = T["W"][:, 32:32 + K] if c["w_slice"] else T["W"]
                if c["row_stats"]:
                    rs = _fill_sentinel(ops.row_stats_buffer(c["M"], N, "cuda"))
                ln = (T["ln_stats"], T["colsum"], 1e-5) if c["ln"] else None
                st = ops.gemm(A, W, out, bias=T["bias"], rowadd=rowadd, rows_per_batch=c["rpb"], residual=res, act=c["act"],
                              stats_images=c["M"] // c["rpb"] if c["stats"] else 0, row_stats=rs, ln=ln)
            else:
                st = ops.conv3x3(T["x"], T["W"], out, bias=T["bias"], rowadd=rowadd, residual=res, stride=c["stride"],
                                 upsample=c["up"], act=c["act"], pad_rb=c["pad_rb"], stats=c["stats"])
                st = st if c["stats"] else None
            torch.cuda.synchronize()
            cnt = ops._splitk_counters.get(out.device)
            results[c["name"]] = dict(
                out=buf.cpu(), stats=st.parts[0][0].cpu() if st is not None else None,
                row_stats=rs.cpu() if rs is not None else None, split=any(split),
                counters_nonzero=int(cnt.count_nonzero()) if cnt is not None else 0)
    finally:
        ops._want_stats, ops._want_splitk, ops.GN_EPILOGUE_MIN_ROWS = want_stats, want_splitk, min_rows
    return results


def _probe_mma(ops, inputs):
    """Under ANYSD_GEMM=mma: the error message of each request only the wgmma kernel can serve ('' when none was raised)."""
    got = {}
    for name in ("dense_row_stats_320", "dense_ln_fold_act1"):
        try:
            _run_cases(ops, [CASES[name]], inputs)
            got[name] = ""
        except ValueError as e:
            got[name] = str(e) or "ValueError"
    return got


def _gelu(v):
    return 0.5 * v * (1.0 + torch.erf(v * 0.5 ** 0.5))


def _reference(c, T):
    """float64 reference of one case from the fp16 operands: (y, e), y [rows, n_out] the exact result, e the bound on the
    kernel's fp32 value before any fp16 rounding (what the statistics are taken of)."""
    N, K = c["N"], c["K"]
    W = T["W"].double()
    if c["kind"] == "dense":
        A = T["A"].double()
        A = A[:, 64:] if c["a_slice"] else A
        W = W[:, 32:32 + K] if c["w_slice"] else W
        acc, P = A @ W.t(), A.abs() @ W.abs().t()
        rpb = c["rpb"]
    else:
        Cin = c["Cin"]
        x = T["x"].double().permute(0, 3, 1, 2)
        w = W.view(N, 3, 3, Cin).permute(0, 3, 1, 2)
        if c["up"]:
            x = F.interpolate(x, scale_factor=2, mode="nearest")
        pad = 1
        if c["pad_rb"]:
            x, pad = F.pad(x, (0, 1, 0, 1)), 0
        nhwc = lambda t: t.permute(0, 2, 3, 1).reshape(-1, N)
        acc = nhwc(F.conv2d(x, w, stride=c["stride"], padding=pad))
        P = nhwc(F.conv2d(x.abs(), w.abs(), stride=c["stride"], padding=pad))
        rpb = _rows_per_image(c)
    bias = T["bias"].double()
    if c["ln"]:                                     # out = rstd (acc - mean colsum) + bias, moments from the given slabs
        s = T["ln_stats"].double().sum(0)
        mean = s[:, 0] / K
        rstd = 1.0 / torch.sqrt(s[:, 1] / K - mean * mean + 1e-5)
        cs = T["colsum"].double()
        core = rstd[:, None] * (acc - mean[:, None] * cs[None, :])
        pre = core + bias
        # + the fp32 row-moment combine and rsqrtf (a few ulp of rstd) and the fmaf chain: 2^-19 of the terms
        e_pre = rstd[:, None] * C_ACC * U * K * P + 2.0 ** -19 * rstd[:, None] * (acc.abs() + (mean[:, None] * cs[None, :]).abs()) \
            + C_ACC * U * bias.abs()
    else:
        pre, mag = acc + bias, bias.abs().expand_as(acc)
        if c["rowadd"]:
            ra = T["rowadd"].double()[:, COL0:COL0 + N][torch.arange(acc.shape[0]) // rpb]
            pre, mag = pre + ra, mag + ra.abs()
        e_pre = C_ACC * U * (K * P + mag)
    f16 = not c["f32"]
    slack = lambda v, fitted: P_GELU_FIT if fitted else 2.0 ** -21 * (1.0 + v.abs())   # fitted GELU / libm-grade fp32
    act = c["act"]
    if act == 0:
        y, e = pre, e_pre
    elif act == 2:                                  # interleaved (a, gate) columns -> a * GELU(gate)
        a, gt, ea, eg = pre[:, 0::2], pre[:, 1::2], e_pre[:, 0::2], e_pre[:, 1::2]
        y = a * _gelu(gt)
        e = _gelu(gt).abs() * ea + (a.abs() + ea) * (SLOPE * eg + slack(gt, f16))
    else:
        y = {1: lambda v: v * torch.sigmoid(v), 3: _gelu, 4: lambda v: v * torch.sigmoid(1.702 * v)}[act](pre)
        e = SLOPE * e_pre + slack(pre, act == 3 and f16)
    if c["res"]:
        r = T["res"].double()[:, COL0:COL0 + _n_out(c)]
        y = y + r
        e = e + C_ACC * U * (y.abs() + r.abs())
    return y, e


def _ratio(err, bound):
    """err / bound, 0 where both are 0 (exact zeros: the zero-padded channels of the output conv); NaN stays NaN."""
    return torch.where(err == 0, torch.zeros_like(err), err / bound)


def _check(c, T, ref, got, label):
    """Asserts the bound, the sentinels and the statistics of one case; returns the worst err / bound ratio of the output."""
    y, e = ref
    rows, n_out = y.shape
    buf = got["out"]
    sent = _is_sentinel(buf)
    inside = sent[GUARD:GUARD + rows, COL0:COL0 + n_out].clone()
    assert not inside.any(), f"{label} {c['name']}: {int(inside.sum())} output elements were not written"
    sent[GUARD:GUARD + rows, COL0:COL0 + n_out] = True
    assert sent.all(), f"{label} {c['name']}: {int((~sent).sum())} elements outside the output window were overwritten"
    out = buf[GUARD:GUARD + rows, COL0:COL0 + n_out].double()
    bound = e if c["f32"] else e + 2.0 ** -11 * (y.abs() + e) + 2.0 ** -25
    ratio = _ratio((out - y).abs(), bound)
    worst = float(ratio.max())
    if not worst <= 1.0:
        bad = (ratio > 1) | ratio.isnan()
        r_, c_ = [int(v) for v in bad.nonzero()[0]]
        cols = sorted({int(v) for v in bad.nonzero()[:, 1]})
        raise AssertionError(f"{label} {c['name']}: {int(bad.sum())} elements out of bound, worst err/bound {worst:.3g}; "
                             f"first ({r_}, {c_}) got {float(out[r_, c_])!r} want {float(y[r_, c_])!r}; columns {cols[:8]}...")
    if got["stats"] is not None:                    # [slots, S, N, 2] per-(image, 32-row slab, channel) {sum, sum of squares}
        n_img, hw = rows // _rows_per_image(c), _rows_per_image(c)
        st = got["stats"][:n_img]
        assert st.shape[1] == hw // 32 and not _is_sentinel(st).any(), f"{label} {c['name']}: statistics slabs not written"
        s = st.double().sum(1)
        yi, ei = y.view(n_img, hw, -1), e.view(n_img, hw, -1)
        for k, (want, tol) in enumerate(((yi.sum(1), ei.sum(1) + 32 * C_ACC * U * yi.abs().sum(1)),
                                         ((yi * yi).sum(1), (2 * yi.abs() * ei + ei * ei).sum(1) + 32 * C_ACC * U * (yi * yi).sum(1)))):
            r = float(_ratio((s[..., k] - want).abs(), tol).max())
            assert r <= 1.0, f"{label} {c['name']}: GroupNorm statistics moment {k + 1} err/bound {r:.3g}"
    if got["row_stats"] is not None:                # [N / 64, M, 2] per-(64-column slab, row) {sum, sum of squares}
        rs = got["row_stats"]
        assert not _is_sentinel(rs).any(), f"{label} {c['name']}: row statistics cells not written"
        ys, es = y.view(rows, -1, 64).transpose(0, 1), e.view(rows, -1, 64).transpose(0, 1)
        for k, (want, tol) in enumerate(((ys.sum(-1), es.sum(-1) + 64 * C_ACC * U * ys.abs().sum(-1)),
                                         ((ys * ys).sum(-1), (2 * ys.abs() * es + es * es).sum(-1) + 64 * C_ACC * U * (ys * ys).sum(-1)))):
            r = float(_ratio((rs[..., k].double() - want).abs(), tol).max())
            assert r <= 1.0, f"{label} {c['name']}: row statistics moment {k + 1} err/bound {r:.3g}"
    return worst


def _bits(t):
    return t.view(SENTINEL[t.dtype][0])


def _same_bits(a, b):
    """Bitwise equality of everything a run wrote (output buffer with its guards, GroupNorm and row statistics)."""
    for k in ("out", "stats", "row_stats"):
        if (a[k] is None) != (b[k] is None):
            return False
        if a[k] is not None and not torch.equal(_bits(a[k]), _bits(b[k])):
            return False
    return True


# ---- fixtures -------------------------------------------------------------------------------------------------------
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
    inputs = {c["name"]: _make_inputs(c, 1000 + i) for i, c in enumerate(ALL)}
    d = tmp_path_factory.mktemp("contraction")
    torch.save(inputs, d / "inputs.pt")
    refs = {}

    def ref(name):                                  # computed once per module, shared by every width and kernel
        if name not in refs:
            refs[name] = _reference(CASES[name], inputs[name])
        return refs[name]
    return SimpleNamespace(inputs=inputs, dir=d, ref=ref)


@pytest.fixture(scope="module")
def natural(ops, data):
    return _run_cases(ops, ALL, data.inputs)


def _child(data, tag, env, names, probe=False):
    """One child process with the forced setting ``env``; returns what its cases wrote."""
    out = data.dir / f"out_{tag}.pt"
    e = {k: v for k, v in os.environ.items() if not k.startswith("ANYSD_GEMM")}
    e.update(env)
    cmd = [sys.executable, *(["-s"] if sys.flags.no_user_site else []), os.path.abspath(__file__), "--worker",
           str(data.dir / "inputs.pt"), str(out), ",".join(names), *(["--probe-mma"] if probe else [])]
    r = subprocess.run(cmd, env=e, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, f"worker {tag} failed:\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"
    return torch.load(out)


def _check_all(data, names, got, label, note=lambda name: ""):
    """_check on every case, so that one run reports every failing case; prints the worst err / bound per case."""
    failures = []
    for name in names:
        try:
            worst = f"{_check(CASES[name], data.inputs[name], data.ref(name), got[name], label):.3f}"
        except AssertionError as e:
            worst = "FAIL"
            failures.append(str(e).splitlines()[0])
        print(f"{label:9s} {name:24s} worst err/bound {worst:6s} {note(name)}")
    return failures


# ---- tests ----------------------------------------------------------------------------------------------------------
def test_natural_selection_against_fp64(ops, data, natural):
    sms = ops.device_info()[0]
    names = [c["name"] for c in ALL]
    failures = _check_all(data, names, natural, "natural", lambda n: "BN=%d splits=%d (p_select restated)" % _natural_width(CASES[n], sms))
    assert not failures, "\n".join(failures)
    assert not any(natural[n]["split"] for n in names), "a case expected to run unsplit ran split-K"


@pytest.mark.parametrize("bn", WIDTHS)
def test_forced_width_against_fp64_and_bit_identical(data, natural, bn):
    """Every case at one forced tile width: the fp64 bound, and bit for bit what the natural width wrote."""
    names = [c["name"] for c in ALL]
    got = _child(data, f"bn{bn}", {"ANYSD_GEMM_BN": str(bn)}, names)
    same = {n: _same_bits(got[n], natural[n]) for n in names}
    failures = _check_all(data, names, got, f"BN={bn}", lambda n: f"bit-identical to natural: {same[n]}")
    assert not failures, "\n".join(failures)
    assert not any(got[n]["split"] for n in names), "a case expected to run unsplit ran split-K"
    differ = [n for n in names if not same[n]]
    assert not differ, f"BN={bn}: not bit-identical to the natural width: {differ}"


@pytest.mark.parametrize("splits", SPLITS)
def test_forced_split_k(data, splits):
    """ANYSD_GEMM_SPLITK: uneven K ranges (the last one short), partials added in split order by the last unit to arrive,
    with statistics and every epilogue add; the arrival counters read zero after every launch."""
    names = [c["name"] for c in SPLIT_CASES]
    got = _child(data, f"sk{splits}", {"ANYSD_GEMM_SPLITK": str(splits)}, names)
    failures = _check_all(data, names, got, f"splitk={splits}")
    assert not failures, "\n".join(failures)
    for n in names:
        assert got[n]["split"], f"{n}: ANYSD_GEMM_SPLITK={splits} did not split K"
        assert got[n]["counters_nonzero"] == 0, f"{n}: {got[n]['counters_nonzero']} split-K arrival counters left armed"


def test_split_k_natural_rule_batch_independent(ops):
    """The 8x8 2560 -> 1280 conv splits K into 3 by geometry alone: every image bit-identical at batch 1, 2 and 5 (output and
    GroupNorm statistics), two runs bitwise equal, the counters re-armed, batch 1 within the fp64 bound."""
    c5 = _conv("split_natural_b5", 5, 8, 8, 2560, 1280, rowadd=False, stats=True)
    T5 = _make_inputs(c5, 7)

    def run(n, lo=0):
        c = dict(c5, name=f"split_natural_{n}_{lo}", Nimg=n)
        T = dict(T5, x=T5["x"][lo:lo + n].contiguous(), res=T5["res"][lo * 64:(lo + n) * 64].contiguous())
        return c, T, _run_cases(ops, [c], {c["name"]: T})[c["name"]]

    b5, b5_again, b2 = run(5)[2], run(5)[2], run(2)[2]
    ones = [run(1, i) for i in range(5)]
    assert _same_bits(b5, b5_again), "two runs of the split-K conv differ"
    for r in (b5, b5_again, b2, *(o for _, _, o in ones)):
        assert r["split"], "the 8x8 2560 -> 1280 conv is expected to run split-K"
        assert r["counters_nonzero"] == 0, "split-K arrival counters left armed"
    win = lambda r, n: _bits(r["out"][GUARD:GUARD + n * 64, COL0:COL0 + 1280]).view(n, 64, 1280)
    for i, (_, _, o) in enumerate(ones):
        assert torch.equal(win(o, 1)[0], win(b5, 5)[i]), f"image {i}: batch 1 != batch 5"
        assert torch.equal(_bits(o["stats"][0]), _bits(b5["stats"][i])), f"image {i}: statistics batch 1 != batch 5"
        if i < 2:
            assert torch.equal(win(o, 1)[0], win(b2, 2)[i]), f"image {i}: batch 1 != batch 2"
            assert torch.equal(_bits(o["stats"][0]), _bits(b2["stats"][i])), f"image {i}: statistics batch 1 != batch 2"
    c1, T1, o1 = ones[0]
    worst = _check(c1, T1, _reference(c1, T1), o1, "natural split")
    print(f"natural split-K conv 8x8 2560->1280: worst err/bound {worst:.3f} (batch 1, image 0)")


def test_mma_against_fp64_and_distinct(data, natural):
    """ANYSD_GEMM=mma: the mma.sync kernel on every case it supports meets the same bound on its own; its fp16 GELU results
    are not bitwise the wgmma kernel's (the switch took effect); statistics requests return None, row statistics and the
    LayerNorm fold are refused."""
    got = _child(data, "mma", {"ANYSD_GEMM": "mma"}, MMA_NAMES, probe=True)
    same = {n: _same_bits(got[n], dict(natural[n], stats=None)) for n in MMA_NAMES}
    failures = _check_all(data, MMA_NAMES, got, "mma", lambda n: f"bitwise equal to wgmma: {same[n]}")
    assert not failures, "\n".join(failures)
    for n in MMA_NAMES:
        assert got[n]["stats"] is None, f"{n}: ANYSD_GEMM=mma returned statistics"
        assert not got[n]["split"]
    # Measured on the H100: both kernels add the k16 products in K order into fp32 accumulators and give the same bits
    # wherever their epilogues agree.  They differ by design in the GELU of fp16 outputs (erf in the mma kernel, the fitted
    # p_gelu in the wgmma kernel): those cases must differ, which shows the switch took effect.
    gelu16 = [n for n in MMA_NAMES if not CASES[n]["f32"] and CASES[n]["act"] in (2, 3)]
    print(f"mma: bitwise equal to wgmma on {sum(same.values())} of {len(same)} cases")
    assert gelu16 and not any(same[n] for n in gelu16), \
        f"ANYSD_GEMM=mma gave the wgmma kernel's fp16 GELU bits (did the switch take effect?): {[n for n in gelu16 if same[n]]}"
    for name, msg in got["__probe__"].items():
        assert "wgmma" in msg, f"ANYSD_GEMM=mma, {name}: expected a refusal naming the wgmma path, got {msg!r}"


def test_unservable_requests(ops):
    """pad_rb needs the wgmma kernel (Cin % 64 == 0): refused otherwise.  Statistics of a shape that cannot produce them
    (rows per image not a multiple of 32, GEGLU, fp32 output, conv patches overshooting the image) come back as None."""
    dev = "cuda"
    x = torch.randn(1, 16, 16, 32, device=dev).half()
    w = torch.randn(64, 9 * 32, device=dev).half()
    o = torch.empty(64, 64, dtype=torch.float16, device=dev)
    with pytest.raises(ValueError, match="right/bottom padding"):
        ops.conv3x3(x, w, o, stride=2, pad_rb=True)
    old, ops.GN_EPILOGUE_MIN_ROWS = ops.GN_EPILOGUE_MIN_ROWS, 0
    try:
        A, W = torch.randn(3 * 48, 64, device=dev).half(), torch.randn(64, 64, device=dev).half()
        assert ops.gemm(A, W, torch.empty(3 * 48, 64, dtype=torch.float16, device=dev), rows_per_batch=48, stats_images=3) is None
        A = torch.randn(3 * 64, 64, device=dev).half()
        assert ops.gemm(A, W, torch.empty(3 * 64, 32, dtype=torch.float16, device=dev), act=2, rows_per_batch=64,
                        stats_images=3) is None
        assert ops.gemm(A, W, torch.empty(3 * 64, 64, dtype=torch.float32, device=dev), rows_per_batch=64, stats_images=3) is None
        assert ops.gemm(A, W, torch.empty(3 * 64, 64, dtype=torch.float16, device=dev), rows_per_batch=64, stats_images=3) is not None
        xc = torch.randn(2, 6, 10, 64, device=dev).half()
        wc = torch.randn(64, 9 * 64, device=dev).half()
        assert ops.conv3x3(xc, wc, torch.empty(2 * 60, 64, dtype=torch.float16, device=dev), stats=True) is None
    finally:
        ops.GN_EPILOGUE_MIN_ROWS = old
    torch.cuda.synchronize()


def _worker(argv):
    inp, outp, names = argv[0], argv[1], argv[2].split(",")
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from anyedit_b200 import ops
    inputs = torch.load(inp)
    res = _run_cases(ops, [CASES[n] for n in names], inputs)
    if "--probe-mma" in argv:
        res["__probe__"] = _probe_mma(ops, inputs)
    torch.save(res, outp)
    return 0


if __name__ == "__main__" and sys.argv[1:2] == ["--worker"]:
    sys.exit(_worker(sys.argv[2:]))
