"""Per-op parity of the training-step kernels (SURVEY.md a24) against torch autograd on fp32 CPU copies of the same
fp16-rounded operands.  Called through the C ABI (anyedit_b200.ops)."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from anyedit_b200 import ops as o
    return o


def randn(seed, *shape, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g) * scale


def h16(t):
    return t.half().float()


@pytest.mark.parametrize("B,heads,nq,nkv,d,self_attn,gated,ln2", [
    (2, 3, 100, 77, 40, False, True, False), (1, 2, 130, 130, 64, True, False, False), (2, 2, 70, 70, 160, True, False, False),
    (1, 3, 65, 16, 24, False, True, True), (2, 8, 256, 256, 40, True, False, True), (1, 2, 200, 300, 80, False, False, False)])
def test_attention_backward(ops, B, heads, nq, nkv, d, self_attn, gated, ln2):
    """dq, dk, dv and the gate gradient of softmax(c q k^T) v * gate vs autograd; padded head stride; ln2 = the
    aux_cols packing where q already carries scale*log2(e) and the natural-log factor is ln 2."""
    from anyedit_b200.unet import head_stride_for
    hs = head_stride_for(d)
    C, Cp = heads * d, heads * hs
    scale = d ** -0.5
    q, k, v = h16(randn(1, B, nq, heads, d)), h16(randn(2, B, nkv, heads, d)), h16(randn(3, B, nkv, heads, d))
    if ln2:
        q = h16(q * scale * math.log2(math.e))
    c = math.log(2.0) if ln2 else scale
    dO = h16(randn(4, B, nq, heads, d) * 0.1)
    gate = torch.rand(B, generator=torch.Generator().manual_seed(5)) + 0.25 if gated else None
    qr, kr, vr = (t.clone().requires_grad_(True) for t in (q, k, v))
    gr = gate.clone().requires_grad_(True) if gated else None
    s = torch.einsum("bihd,bjhd->bhij", qr, kr) * c
    o = torch.einsum("bhij,bjhd->bihd", s.softmax(-1), vr)
    if gated:
        o = o * gr.view(B, 1, 1, 1)
    o.backward(dO)

    def pad(t):
        out = torch.zeros(B, t.shape[1], heads, hs, dtype=torch.float16)
        out[..., :d] = t
        return out.reshape(B, t.shape[1], Cp).cuda().contiguous()

    q16, k16, v16 = pad(q), pad(k), pad(v)
    dO16 = dO.reshape(B, nq, C).half().cuda().contiguous()
    dq = torch.full((B, nq, Cp), float("nan"), dtype=torch.float16, device="cuda")
    dk = torch.full((B, nkv, Cp), float("nan"), dtype=torch.float16, device="cuda")
    dv = torch.full((B, nkv, Cp), float("nan"), dtype=torch.float16, device="cuda")
    g_dev = gate.cuda() if gated else None
    dg = torch.zeros(B, device="cuda") if gated else None
    ops.attention_bwd(q16, k16, v16, dO16, dq, dk, dv, B, heads, nq, nkv, d, Cp, Cp, Cp, C, Cp, Cp, Cp, qk_scale=c, gate=g_dev,
                      d_gate=dg, head_stride=hs)
    torch.cuda.synchronize()
    unpad = lambda t, n: t.float().cpu().reshape(B, n, heads, hs)
    for name, got, ref, n in (("dq", dq, qr.grad, nq), ("dk", dk, kr.grad, nkv), ("dv", dv, vr.grad, nkv)):
        g4 = unpad(got, n)
        assert torch.isfinite(g4).all(), name
        assert float(g4[..., d:].abs().max()) == 0.0 if hs > d else True, name       # padding columns stay zero
        e = rel(g4[..., :d], ref)
        assert e < 4e-3, (name, e)
    if gated:
        e = rel(dg, gr.grad)
        assert e < 4e-3, ("d_gate", e)
    if not gated:
        # with the forward output supplied (self-attention): same gradients, one sweep less
        o16 = torch.einsum("bhij,bjhd->bihd", (torch.einsum("bihd,bjhd->bhij", q, k) * c).softmax(-1), v).reshape(B, nq, C).half().cuda()
        dq3, dk3, dv3 = torch.empty_like(dq), torch.empty_like(dk), torch.empty_like(dv)
        ops.attention_bwd(q16, k16, v16, dO16, dq3, dk3, dv3, B, heads, nq, nkv, d, Cp, Cp, Cp, C, Cp, Cp, Cp, qk_scale=c, head_stride=hs,
                          out=o16.contiguous(), ld_o=C)
        for name, got, ref, n in (("dq", dq3, qr.grad, nq), ("dk", dk3, kr.grad, nkv), ("dv", dv3, vr.grad, nkv)):
            e = rel(unpad(got, n)[..., :d], ref)
            assert e < 4e-3, (name + " (with out)", e)
    # frozen K/V (text cross-attention): dq only, accumulated onto an existing gradient
    dq2 = dq.clone()
    ops.attention_bwd(q16, k16, v16, dO16, dq2, None, None, B, heads, nq, nkv, d, Cp, Cp, Cp, C, Cp, qk_scale=c, gate=g_dev,
                      head_stride=hs, accumulate_dq=True)
    e = rel(unpad(dq2, nq)[..., :d], 2 * qr.grad)
    assert e < 4e-3, ("dq accumulate", e)


@pytest.mark.parametrize("B,heads,nq,nkv,d,aux", [(2, 3, 256, 256, 40, True), (1, 2, 128, 512, 40, True), (1, 2, 384, 128, 24, False),
                                                  (1, 8, 1024, 1024, 40, True)])
def test_attention_backward_wgmma(ops, monkeypatch, B, heads, nq, nkv, d, aux):
    """The wgmma backward (attention_wgmma.cu): the forward hands over its base-2 log-sum-exp (anysd_attn_params::lse), the
    backward recomputes P = 2^(s - lse) and forms dS, dQ, dK, dV on the tensor cores.  Checked against autograd, against the
    mma.sync kernels on the same inputs, and the log-sum-exp against torch.logsumexp."""
    from anyedit_b200.unet import head_stride_for
    hs = head_stride_for(d)
    assert hs == (d + 15) // 16 * 16
    C, Cp = heads * d, heads * hs
    scale = d ** -0.5
    q, k, v = h16(randn(11, B, nq, heads, d)), h16(randn(12, B, nkv, heads, d)), h16(randn(13, B, nkv, heads, d))
    if aux:
        q = h16(q * scale * math.log2(math.e))
    c = math.log(2.0) if aux else scale
    dO = h16(randn(14, B, nq, heads, d) * 0.1)
    qr, kr, vr = (t.clone().requires_grad_(True) for t in (q, k, v))
    s = torch.einsum("bihd,bjhd->bhij", qr, kr) * c
    o = torch.einsum("bhij,bjhd->bihd", s.softmax(-1), vr)
    o.backward(dO)

    def pad(t, ones=0):
        out = torch.zeros(B, t.shape[1], heads, hs, dtype=torch.float16)
        out[..., :d] = t
        out[..., d:d + ones] = 1.0
        return out.reshape(B, t.shape[1], Cp).cuda().contiguous()

    q16, k16, v16 = pad(q), pad(k, 2 if aux else 0), pad(v, 1 if aux else 0)
    out = torch.empty(B, nq, C, dtype=torch.float16, device="cuda")
    lse = torch.full((B, heads, nq), float("nan"), device="cuda")
    ops.attention(q16, k16, v16, out, B, heads, nq, nkv, d, Cp, Cp, Cp, C, head_stride=hs, aux_cols=aux, scale=scale, lse=lse)
    assert rel(out.float().cpu().view(B, nq, heads, d), o.detach()) < 2e-3
    lse_ref = torch.logsumexp(s.detach(), -1) / math.log(2.0)                      # [B, h, nq], base 2
    assert float((lse.cpu() - lse_ref).abs().max()) < 2e-3
    dO16 = dO.reshape(B, nq, C).half().cuda().contiguous()
    res = {}
    for mode in ("wgmma", "mma"):
        if mode == "mma":
            lse_arg = None
        else:
            lse_arg = lse
        dq = torch.full((B, nq, Cp), float("nan"), dtype=torch.float16, device="cuda")
        dk = torch.full((B, nkv, Cp), float("nan"), dtype=torch.float16, device="cuda")
        dv = torch.full((B, nkv, Cp), float("nan"), dtype=torch.float16, device="cuda")
        ops.attention_bwd(q16, k16, v16, dO16, dq, dk, dv, B, heads, nq, nkv, d, Cp, Cp, Cp, C, Cp, Cp, Cp, qk_scale=c, head_stride=hs,
                          out=out, ld_o=C, lse=lse_arg)
        torch.cuda.synchronize()
        res[mode] = (dq, dk, dv)
    unpad = lambda t, n: t.float().cpu().reshape(B, n, heads, hs)
    for mode, (dq, dk, dv) in res.items():
        for name, got, ref, n in (("dq", dq, qr.grad, nq), ("dk", dk, kr.grad, nkv), ("dv", dv, vr.grad, nkv)):
            g4 = unpad(got, n)
            assert torch.isfinite(g4).all(), (mode, name)
            assert float(g4[..., d:].abs().max()) == 0.0, (mode, name)            # padding columns stay zero
            e = rel(g4[..., :d], ref)
            print(f"attention backward {mode} B={B} h={heads} nq={nq} nkv={nkv} d={d} {name}: {e:.2e}")
            assert e < 4e-3, (mode, name, e)
    assert not torch.equal(res["wgmma"][0], res["mma"][0])                        # the two really are different kernels
    # frozen K/V, accumulated onto an existing gradient
    dq2 = res["wgmma"][0].clone()
    ops.attention_bwd(q16, k16, v16, dO16, dq2, None, None, B, heads, nq, nkv, d, Cp, Cp, Cp, C, Cp, qk_scale=c, head_stride=hs,
                      out=out, ld_o=C, lse=lse, accumulate_dq=True)
    assert rel(unpad(dq2, nq)[..., :d], 2 * qr.grad) < 4e-3


@pytest.mark.parametrize("N,HW,C1,C2,silu", [(2, 60, 64, 0, True), (3, 35, 96, 32, True), (2, 16, 320, 0, False), (1, 100, 64, 128, False),
                                              (2, 4096, 64, 0, True), (1, 1030, 96, 32, True), (2, 200, 320, 0, False)])   # 8 / 4 / 2 CTAs per slab
def test_groupnorm_backward(ops, N, HW, C1, C2, silu):
    C = C1 + C2
    x = h16(randn(11, N, HW, C) * 1.5 + 0.3)
    gamma, beta = randn(12, C) * 0.5 + 1.0, randn(13, C) * 0.2
    dy = h16(randn(14, N, HW, C) * 0.1)
    xr = x.clone().requires_grad_(True)
    y = F.group_norm(xr.permute(0, 2, 1), 32, gamma, beta, eps=1e-5)
    if silu:
        y = F.silu(y)
    y.backward(dy.permute(0, 2, 1))
    x1 = x[..., :C1].contiguous().half().cuda()
    x2 = x[..., C1:].contiguous().half().cuda() if C2 else None
    dx = torch.empty(N, HW, C, dtype=torch.float16, device="cuda")
    ops.groupnorm_bwd(x1, gamma.cuda(), beta.cuda(), dy.half().cuda(), dx, N, HW, 1e-5, silu, x2=x2)
    e = rel(dx, xr.grad)
    assert e < 3e-3, e


@pytest.mark.parametrize("M,C", [(50, 64), (33, 320), (9, 1280)])
def test_layernorm_backward(ops, M, C):
    x = h16(randn(21, M, C) * 2.0 + 0.5)
    gamma = randn(22, C) * 0.5 + 1.0
    dy = h16(randn(23, M, C) * 0.1)
    xr = x.clone().requires_grad_(True)
    F.layer_norm(xr, (C,), gamma, torch.zeros(C), 1e-5).backward(dy)
    dx = torch.empty(M, C, dtype=torch.float16, device="cuda")
    ops.layernorm_bwd(x.half().cuda(), gamma.cuda(), dy.half().cuda(), dx)
    e = rel(dx, xr.grad)
    assert e < 3e-3, e


def test_geglu_forward_backward(ops):
    M, inner = 37, 64
    pre = h16(randn(31, M, inner, 2) * 1.5)                    # [..., 0] = a, [..., 1] = gate (interleaved columns)
    dy = h16(randn(32, M, inner) * 0.1)
    pr = pre.clone().requires_grad_(True)
    out = pr[..., 0] * F.gelu(pr[..., 1])
    out.backward(dy)
    pre16 = pre.reshape(M, 2 * inner).half().cuda()
    o = torch.empty(M, inner, dtype=torch.float16, device="cuda")
    ops.geglu(pre16, o)
    assert rel(o, out.detach()) < 1e-3
    dpre = torch.empty(M, 2 * inner, dtype=torch.float16, device="cuda")
    ops.geglu_bwd(pre16, dy.half().cuda(), dpre)
    assert rel(dpre.view(M, inner, 2), pr.grad) < 2e-3


def test_conv_and_linear_input_gradients_reuse_the_forward_contraction(ops):
    """dX of conv3x3 (stride 1, stride 2 via zero insertion, after nearest x2 via sum pooling) and of a linear layer are
    anysd_gemm_f16 launches on rotated / transposed weight packs (anyedit_b200.training)."""
    from anyedit_b200 import training as T
    N, H, W, Ci, Co = 2, 8, 12, 64, 128
    x = h16(randn(41, N, Ci, H, W))
    w = h16(randn(42, Co, Ci, 3, 3) * (9 * Ci) ** -0.5)
    to_nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous().half().cuda()
    from_nhwc = lambda t, n, h, ww: t.float().cpu().view(n, h, ww, -1).permute(0, 3, 1, 2)
    wb = T.pack_conv3_dx(w, "cuda")
    # stride 1
    xr = x.clone().requires_grad_(True)
    y = F.conv2d(xr, w, padding=1)
    dy = h16(randn(43, *y.shape) * 0.1)
    y.backward(dy)
    dx = torch.empty(N * H * W, Ci, dtype=torch.float16, device="cuda")
    ops.conv3x3(to_nhwc(dy), wb, dx)
    assert rel(from_nhwc(dx, N, H, W), xr.grad) < 2e-3
    # stride 2 (Downsample)
    xr = x.clone().requires_grad_(True)
    y = F.conv2d(xr, w, padding=1, stride=2)
    dy = h16(randn(44, *y.shape) * 0.1)
    y.backward(dy)
    up = torch.empty(N, H, W, Co, dtype=torch.float16, device="cuda")
    ops.zero_insert2x(to_nhwc(dy), up)
    ops.conv3x3(up, wb, dx)
    assert rel(from_nhwc(dx, N, H, W), xr.grad) < 2e-3
    # nearest x2 then conv (Upsample)
    xr = x.clone().requires_grad_(True)
    y = F.conv2d(F.interpolate(xr, scale_factor=2, mode="nearest"), w, padding=1)
    dy = h16(randn(45, *y.shape) * 0.1)
    y.backward(dy)
    dbig = torch.empty(N * 2 * H * 2 * W, Ci, dtype=torch.float16, device="cuda")
    ops.conv3x3(to_nhwc(dy), wb, dbig)
    dsm = torch.empty(N, H, W, Ci, dtype=torch.float16, device="cuda")
    ops.sumpool2x(dbig.view(N, 2 * H, 2 * W, Ci), dsm)
    assert rel(from_nhwc(dsm, N, H, W), xr.grad) < 2e-3
    # linear
    M, K, Nn = 70, 96, 160
    a, wl = h16(randn(46, M, K)), h16(randn(47, Nn, K) * K ** -0.5)
    ar = a.clone().requires_grad_(True)
    dyl = h16(randn(48, M, Nn) * 0.1)
    F.linear(ar, wl).backward(dyl)
    dxl = torch.empty(M, K, dtype=torch.float16, device="cuda")
    ops.gemm(dyl.half().cuda(), T.pack_linear_dx(wl, "cuda"), dxl)
    assert rel(dxl, ar.grad) < 2e-3


def test_small_training_kernels(ops):
    from oracle import ddim_oracle, train_oracle
    # q_sample
    sched = ddim_oracle.register_schedule("linear", 1000, 0.00085, 0.012)
    x0, noise = randn(51, 3, 4, 8, 8), randn(52, 3, 4, 8, 8)
    t = torch.tensor([0, 500, 999])
    out = torch.empty(3, 4, 8, 8, device="cuda")
    ops.q_sample(x0.cuda(), noise.cuda(), t.cuda(), sched["sqrt_alphas_cumprod"].cuda(), sched["sqrt_one_minus_alphas_cumprod"].cuda(), out)
    ref = train_oracle.q_sample(x0, noise, t, sched["alphas_cumprod"])
    assert float((out.cpu() - ref).abs().max()) < 1e-6
    # mse loss + gradient in the padded NHWC layout
    pred, target = randn(53, 2, 4, 6, 5), randn(54, 2, 4, 6, 5)
    pr = pred.clone().requires_grad_(True)
    loss_ref = F.mse_loss(pr, target)
    loss_ref.backward()
    dp = torch.empty(2, 30, 64, dtype=torch.float16, device="cuda")
    loss = torch.zeros(1, device="cuda")
    ops.mse_loss(pred.cuda(), target.cuda(), dp, loss, grad_scale=256.0)
    assert float(loss) == pytest.approx(float(loss_ref.detach()), rel=1e-5)
    got = dp.float().cpu().view(2, 6, 5, 64)
    assert float(got[..., 4:].abs().max()) == 0.0
    assert rel(got[..., :4].permute(0, 3, 1, 2) / 256.0, pr.grad) < 1e-3
    # colsum / add / split
    x = h16(randn(55, 3, 50, 72))
    cs = torch.zeros(3, 100, device="cuda")
    ops.colsum(x.half().cuda(), cs, 3, 50)
    assert rel(cs[:, :72], x.sum(1)) < 1e-5 and float(cs[:, 72:].abs().max()) == 0.0
    ops.colsum(x.half().cuda(), cs, 3, 50, accumulate=True)
    assert rel(cs[:, :72], 2 * x.sum(1)) < 1e-5
    y = h16(randn(56, 40, 64))
    yy = y.half().cuda()
    ops.add_(yy, y.half().cuda())
    assert torch.equal(yy.cpu(), (2 * y).half())
    src = h16(randn(57, 33, 24 + 40)).half().cuda()
    a, b = torch.empty(33, 24, dtype=torch.float16, device="cuda"), torch.empty(33, 40, dtype=torch.float16, device="cuda")
    ops.split_channels(src, a, b)
    assert torch.equal(torch.cat([a, b], 1), src)
    # silu backward (fp32)
    xs, ds = randn(58, 5, 64), randn(59, 5, 64)
    xr = xs.clone().requires_grad_(True)
    F.silu(xr).backward(ds)
    dxs = torch.empty(5, 64, device="cuda")
    ops.silu_bwd_f32(xs.cuda(), ds.cuda(), dxs)
    assert rel(dxs, xr.grad) < 1e-5
    # weight gradient with padded heads
    M, heads, d, hs, Kb = 48, 3, 24, 32, 40
    A = h16(randn(60, M, heads, d))
    Bm = h16(randn(61, M, Kb))
    Ap = torch.zeros(M, heads, hs)
    Ap[..., :d] = A
    outw = torch.zeros(heads * d, Kb, device="cuda")
    ops.gemm_tn(Ap.reshape(M, heads * hs).half().cuda(), Bm.half().cuda(), outw, M, heads * d, Kb, alpha=0.5, head_d=d, head_stride=hs)
    assert rel(outw, 0.5 * A.reshape(M, heads * d).t() @ Bm) < 1e-5
    # two "experts" side by side (group mapping): rows [e*C, (e+1)*C) of out read columns e*group_stride + ...
    A2 = torch.cat([Ap.reshape(M, heads * hs), torch.zeros(M, 8), 2 * Ap.reshape(M, heads * hs), torch.zeros(M, 8)], 1)
    outg = torch.zeros(2 * heads * d, Kb, device="cuda")
    ops.gemm_tn(A2.half().cuda(), Bm.half().cuda(), outg, M, 2 * heads * d, Kb, head_d=d, head_stride=hs, group_c=heads * d,
                group_stride=heads * hs + 8)
    refw = A.reshape(M, heads * d).t() @ Bm
    assert rel(outg, torch.cat([refw, 2 * refw], 0)) < 1e-5
    # the same gradient on the tensor cores: gather + transpose both operands to K-major, then anysd_gemm_f16 (fp32 out)
    Mp = (M + 7) // 8 * 8
    At = torch.full((2 * heads * d, Mp + 8), float("nan"), dtype=torch.float16, device="cuda")[:, :Mp]     # ldo > M, strided rows
    At = torch.empty(2 * heads * d, Mp, dtype=torch.float16, device="cuda")
    Bt = torch.empty(Kb, Mp, dtype=torch.float16, device="cuda")
    ops.gather_transpose(A2.half().cuda(), At, M, 2 * heads * d, head_d=d, head_stride=hs, group_c=heads * d, group_stride=heads * hs + 8)
    ops.gather_transpose(Bm.half().cuda(), Bt, M, Kb)
    assert torch.equal(Bt[:, :M].cpu(), Bm.half().t()) and float(Bt[:, M:].float().abs().max() if Mp > M else 0.0) == 0.0
    outt = torch.empty(2 * heads * d, Kb, device="cuda")
    ops.gemm(At, Bt, outt)
    assert rel(outt, torch.cat([refw, 2 * refw], 0)) < 1e-3
    # AdamW
    p0, g0 = randn(62, 1000), randn(63, 1000) * 0.1
    p, m, v = p0.clone().cuda(), torch.zeros(1000, device="cuda"), torch.zeros(1000, device="cuda")
    q, mq, vq = p0.clone(), torch.zeros(1000), torch.zeros(1000)
    for step in (1, 2, 3):
        ops.adamw_(p, (g0 * 128).cuda(), m, v, step, 1e-3, 0.9, 0.999, 1e-8, 1e-2, grad_scale=1 / 128)
        q, mq, vq = train_oracle.adamw_step(q, g0, mq, vq, step, 1e-3, 0.9, 0.999, 1e-8, 1e-2)
    assert float((p.cpu() - q).abs().max()) < 1e-6


def test_router_backward_and_scatter(ops):
    N, L, E, D, T = 5, 3, 4, 64, 7
    table = randn(71, T, D)
    idx = torch.tensor([0, 3, 3, 6, 1])
    W = h16(randn(72, L, E, D) * 0.2)
    b = randn(73, L, E) * 0.1
    dg = randn(74, N, L, E)
    tr = table.clone().requires_grad_(True)
    Wr, br = W.clone().requires_grad_(True), b.clone().requires_grad_(True)
    te = tr[idx]
    gates = torch.einsum("led,nd->nle", Wr, te) + br
    gates = gates.softmax(-1)
    gates.backward(dg)
    dW, db, dte = torch.zeros(L, E, D, device="cuda"), torch.zeros(L, E, device="cuda"), torch.zeros(N, D, device="cuda")
    ops.router_bwd(gates.detach().cuda(), dg.cuda(), table[idx].cuda(), W.half().cuda(), dW, db, dte)
    assert rel(dW, Wr.grad) < 1e-4 and rel(db, br.grad) < 1e-4
    dtab = torch.zeros(T, D, device="cuda")
    ops.scatter_add_rows(dte, idx.cuda(), dtab)
    assert rel(dtab, tr.grad) < 1e-4


@pytest.mark.parametrize("B,heads,nq,nvis,d,E,ln2", [(2, 3, 100, 16, 40, 4, True), (1, 2, 130, 5, 64, 3, False), (2, 2, 70, 64, 160, 2, False),
                                                     (3, 4, 64, 7, 16, 11, False)])
def test_expert_attention_forward_backward(ops, B, heads, nq, nvis, d, E, ln2):
    """All E expert streams of a layer in one launch: out += sum_e g[b,e] softmax(c q K_e^T) V_e, and its backward
    (dq accumulated, dK_e / dV_e in the fused [K_e | V_e] layout, gate gradients) vs autograd."""
    from anyedit_b200.unet import head_stride_for
    hs = head_stride_for(d)
    C, Cp = heads * d, heads * hs
    scale = d ** -0.5
    q = h16(randn(81, B, nq, heads, d))
    if ln2:
        q = h16(q * scale * math.log2(math.e))
    c = math.log(2.0) if ln2 else scale
    k, v = h16(randn(82, B, nvis, E, heads, d)), h16(randn(83, B, nvis, E, heads, d))
    gates = torch.rand(B, 3, E, generator=torch.Generator().manual_seed(84))          # [B, layers, E]: layer 1 is used
    base = h16(randn(85, B, nq, C) * 0.5)
    dO = h16(randn(86, B, nq, heads, d) * 0.1)
    qr, kr, vr, gr = (t.clone().requires_grad_(True) for t in (q, k, v, gates))
    s = torch.einsum("bihd,bjehd->behij", qr, kr) * c
    o = torch.einsum("behij,bjehd->behid", s.softmax(-1), vr)
    o = (o * gr[:, 1].view(B, E, 1, 1, 1)).sum(1).permute(0, 2, 1, 3)                 # [B, nq, heads, d]
    o.backward(dO)

    def padq(t):
        out = torch.zeros(B, nq, heads, hs, dtype=torch.float16)
        out[..., :d] = t
        return out.reshape(B, nq, Cp).cuda().contiguous()

    ekv = torch.zeros(B, nvis, E, 2, heads, hs, dtype=torch.float16)
    ekv[:, :, :, 0, :, :d] = k
    ekv[:, :, :, 1, :, :d] = v
    ekv = ekv.reshape(B * nvis, E * 2 * Cp).cuda().contiguous()
    out = base.half().cuda().contiguous()
    g_dev = gates.cuda()
    q16 = padq(q)
    ops.expert_attention(q16, ekv, g_dev[:, 1], out, B, heads, nq, nvis, d, E, Cp, E * 2 * Cp, C, 2 * Cp, Cp, c, head_stride=hs)
    assert rel(out.float().cpu() - base, o.detach().reshape(B, nq, C)) < 3e-3
    dq = torch.zeros(B, nq, Cp, dtype=torch.float16, device="cuda")
    dekv = torch.full_like(ekv, float("nan"))
    dg = torch.zeros_like(g_dev)
    ops.expert_attention_bwd(q16, ekv, g_dev[:, 1], dO.reshape(B, nq, C).half().cuda().contiguous(), dq, dekv, dg[:, 1], B, heads, nq, nvis, d,
                             E, Cp, E * 2 * Cp, C, Cp, 2 * Cp, Cp, c, head_stride=hs)
    torch.cuda.synchronize()
    assert rel(dq.float().cpu().view(B, nq, heads, hs)[..., :d], qr.grad) < 4e-3
    d5 = dekv.float().cpu().view(B, nvis, E, 2, heads, hs)
    assert torch.isfinite(d5).all()
    assert rel(d5[:, :, :, 0, :, :d], kr.grad) < 4e-3 and rel(d5[:, :, :, 1, :, :d], vr.grad) < 4e-3
    if hs > d:
        assert float(d5[..., d:].abs().max()) == 0.0
    assert rel(dg[:, 1], gr.grad[:, 1]) < 4e-3 and float(dg[:, 0].abs().max()) == 0.0
