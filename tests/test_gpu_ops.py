"""Kernel-level parity: each CUDA op, called through the C ABI, against a fp32 CPU reference of the
same op (oracle / plain torch fp32) on seeded inputs, plus the golden KATs generated from the
reference's own module classes.  Tolerances: fp16 operands with fp32 accumulation -> relative L2
error a small multiple of 2^-11; integer / fp32 elementwise work is checked bit-exactly."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

G = os.path.join(os.path.dirname(__file__), "golden")


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from anyedit_b200 import ops as o
    sms, major, minor = o.device_info()
    assert (major, minor) == (9, 0), f"sm_90a kernels need a Hopper GPU (H100), got cc {major}.{minor}"
    return o


@pytest.fixture
def stats_everywhere(ops):
    """The product asks for epilogue statistics from 1024 pixels per image on (a measured break-even); the kernel path itself
    works from 32: the op tests exercise it on small maps too."""
    old, ops.GN_EPILOGUE_MIN_ROWS = ops.GN_EPILOGUE_MIN_ROWS, 0
    yield
    ops.GN_EPILOGUE_MIN_ROWS = old


def randn(seed, *shape, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g) * scale


def to_nhwc16(x):
    return x.permute(0, 2, 3, 1).contiguous().half().cuda()


def from_nhwc(y, N, H, W):
    return y.float().cpu().reshape(N, H, W, -1).permute(0, 3, 1, 2)


def test_layout_roundtrip(ops):
    x = randn(1, 3, 5, 7, 9)
    dst = torch.zeros(3, 7, 9, 8, dtype=torch.float16, device="cuda")
    ops.nchw_to_nhwc(x.cuda(), dst, 2)
    ref = torch.zeros(3, 7, 9, 8)
    ref[..., 2:7] = x.permute(0, 2, 3, 1)
    assert torch.equal(dst.cpu(), ref.half())
    back = torch.empty(3, 8, 7, 9, dtype=torch.float32, device="cuda")
    ops.nhwc_to_nchw(dst, back)
    assert torch.equal(back.cpu(), ref.half().float().permute(0, 3, 1, 2))
    a, b = randn(2, 10, 16).half().cuda(), randn(3, 10, 24).half().cuda()
    c = torch.empty(10, 40, dtype=torch.float16, device="cuda")
    ops.concat_channels(a, b, c)
    assert torch.equal(c, torch.cat([a, b], 1))


def test_timestep_embedding_golden(ops):
    g = np.load(os.path.join(G, "timestep_embedding.npz"))
    t = torch.from_numpy(g["t"]).cuda()
    for dim, key in ((320, "e320"), (64, "e64")):
        out = torch.empty(len(t), dim, dtype=torch.float16, device="cuda")
        ops.timestep_embedding(t, out)
        ref = torch.from_numpy(g[key])
        # fp16 storage of an fp32 value: half an fp16 ulp, plus the sin/cos argument-reduction ulp
        assert (out.float().cpu() - ref).abs().max() < 6e-4


@pytest.mark.parametrize("shape,C2", [((2, 64, 6, 10), 0), ((3, 320, 16, 16), 0), ((2, 640, 8, 8), 320),
                                      ((1, 2560, 8, 8), 0), ((2, 960, 32, 32), 640), ((2, 32, 5, 3), 0),
                                      # bench-sized maps: the register-resident kernel (<= 8 rows per thread, norm.cu gn_res_plan) and the statistics + apply path
                                      ((2, 320, 64, 64), 0), ((1, 960, 64, 64), 320), ((2, 640, 32, 32), 0), ((1, 320, 96, 96), 0),
                                      ((1, 1920, 48, 48), 640), ((2, 1280, 16, 16), 0), ((1, 2560, 16, 16), 1280), ((1, 128, 40, 40), 0),
                                      ((1, 1280, 48, 48), 0)])
@pytest.mark.parametrize("silu,eps", [(True, 1e-5), (False, 1e-6)])
def test_groupnorm(ops, shape, C2, silu, eps):
    N, C, H, W = shape
    x = randn(11, N, C, H, W, scale=2.0) + 0.7
    gamma, beta = 1 + 0.2 * randn(12, C), 0.1 * randn(13, C)
    x16 = x.half().float()
    ref = F.group_norm(x16, 32, gamma, beta, eps)
    ref = F.silu(ref) if silu else ref
    xh = to_nhwc16(x)
    y = torch.empty_like(xh)
    ws = ops.groupnorm_workspace(N)
    if C2:
        x1, x2 = xh[..., :C - C2].contiguous(), xh[..., C - C2:].contiguous()
        ops.groupnorm(x1, gamma.cuda(), beta.cuda(), y, N, H * W, eps, silu, ws, x2=x2)
    else:
        ops.groupnorm(xh, gamma.cuda(), beta.cuda(), y, N, H * W, eps, silu, ws)
    e = rel(from_nhwc(y, N, H, W), ref)
    assert e < 1e-3, e


def test_groupnorm_batch_independent_bits(ops):
    """Every output bit of an image is independent of its position in / the size of the batch (geometry-only decomposition)."""
    for (C, H, W) in ((320, 64, 64), (640, 32, 32), (1280, 8, 8), (960, 16, 16)):
        x = to_nhwc16(randn(17, 3, C, H, W, scale=1.5) - 0.3)
        gamma, beta = (1 + 0.2 * randn(18, C)).cuda(), (0.1 * randn(19, C)).cuda()
        y3 = torch.empty_like(x)
        ops.groupnorm(x, gamma, beta, y3, 3, H * W, 1e-5, True, ops.groupnorm_workspace(3))
        for i in range(3):
            xi = x[i:i + 1].contiguous()
            y1 = torch.empty_like(xi)
            ops.groupnorm(xi, gamma, beta, y1, 1, H * W, 1e-5, True, ops.groupnorm_workspace(1))
            assert torch.equal(y1[0], y3[i]), (C, H, W, i)


def test_groupnorm_silu_golden_kat(ops):
    from oracle import weights
    g = np.load(os.path.join(G, "op_kats.npz"))
    x = torch.from_numpy(g["gn_x"])
    sd = weights.make_state_dict({"in_layers.0.weight": (64,), "in_layers.0.bias": (64,)}, 21)
    N, C, H, W = x.shape
    xh = to_nhwc16(x)
    y = torch.empty_like(xh)
    ops.groupnorm(xh, sd["in_layers.0.weight"].cuda(), sd["in_layers.0.bias"].cuda(), y, N, H * W, 1e-5, True,
                  ops.groupnorm_workspace(N))
    e = rel(from_nhwc(y, N, H, W), torch.from_numpy(g["gn_silu_out"]))
    assert e < 2e-3, e


@pytest.mark.parametrize("M,C", [(77, 320), (1000, 640), (33, 1280), (5, 64), (64, 2048)])
def test_layernorm(ops, M, C):
    x = randn(21, M, C, scale=3.0) + 0.5
    gamma, beta = 1 + 0.2 * randn(22, C), 0.1 * randn(23, C)
    xh = x.half().cuda()
    y = torch.empty_like(xh)
    ops.layernorm(xh, gamma.cuda(), beta.cuda(), y)
    ref = F.layer_norm(x.half().float(), (C,), gamma, beta)
    assert rel(y, ref) < 1e-3


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (200, 320, 320), (4096, 320, 2880 // 9), (77, 640, 768),
                                   (16, 1280, 1280), (1, 8, 8), (300, 4, 320), (513, 130, 72)])
def test_gemm_plain(ops, M, N, K):
    A, W = randn(31, M, K), randn(32, N, K, scale=K ** -0.5)
    bias = 0.1 * randn(33, N)
    A16, W16 = A.half(), W.half()
    ref = A16.float() @ W16.float().t() + bias
    for odt in (torch.float16, torch.float32):
        out = torch.empty(M, N, dtype=odt, device="cuda")
        ops.gemm(A16.cuda(), W16.cuda(), out, bias=bias.cuda())
        e = rel(out, ref)
        assert e < (1e-3 if odt == torch.float16 else 2e-5), (odt, e)


def test_gemm_epilogues(ops):
    M, N, K, HW = 384, 256, 192, 96   # 4 "images" of 96 rows
    A, W = randn(41, M, K).half(), randn(42, N, K, scale=K ** -0.5).half()
    bias, res = 0.1 * randn(43, N), randn(44, M, N).half()
    rowadd = randn(45, M // HW, N + 16)
    base = A.float() @ W.float().t() + bias
    # bias + rowadd + residual
    out = torch.empty(M, N, dtype=torch.float16, device="cuda")
    ops.gemm(A.cuda(), W.cuda(), out, bias=bias.cuda(), rowadd=rowadd.cuda()[:, 8:], rows_per_batch=HW,
             residual=res.cuda(), ld_rowadd=N + 16)
    ref = base + rowadd[:, 8:8 + N].repeat_interleave(HW, 0) + res.float()
    assert rel(out, ref) < 1e-3
    # SiLU
    ops.gemm(A.cuda(), W.cuda(), out, bias=bias.cuda(), act=1)
    assert rel(out, F.silu(base)) < 1e-3
    # GEGLU with interleaved rows
    Wg = randn(46, 2 * N, K, scale=K ** -0.5).half()
    bg = 0.1 * randn(47, 2 * N)
    full = A.float() @ Wg.float().t() + bg
    ref = full[:, :N] * F.gelu(full[:, N:])
    Wi = torch.stack([Wg[:N], Wg[N:]], 1).reshape(2 * N, K).contiguous()
    bi = torch.stack([bg[:N], bg[N:]], 1).reshape(-1).contiguous()
    og = torch.empty(M, N, dtype=torch.float16, device="cuda")
    ops.gemm(A.cuda(), Wi.cuda(), og, bias=bi.cuda(), act=2)
    assert rel(og, ref) < 1.5e-3
    # strided A (column slice) and K-sliced W
    out2 = torch.empty(M, N, dtype=torch.float32, device="cuda")
    Ac = A.cuda()
    ops.gemm(Ac[:, 64:], W.cuda()[:, 64:], out2, K=128, lda=K, ldw=K)
    assert rel(out2, A[:, 64:].float() @ W[:, 64:].float().t()) < 2e-5


@pytest.mark.parametrize("N,Cin,Cout,H,W,stride,up", [
    (2, 64, 64, 6, 10, 1, 0), (1, 8, 320, 16, 16, 1, 0), (2, 320, 4, 16, 16, 1, 0), (2, 64, 96, 9, 7, 2, 0),
    (2, 64, 64, 8, 8, 2, 0), (1, 128, 64, 5, 6, 1, 1), (3, 320, 640, 8, 8, 1, 0), (1, 640, 320, 16, 16, 1, 1)])
def test_conv3x3(ops, N, Cin, Cout, H, W, stride, up):
    x = randn(51, N, Cin, H, W)
    w = randn(52, Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5)
    b = 0.1 * randn(53, Cout)
    x16, w16 = x.half().float(), w.half().float()
    xin = F.interpolate(x16, scale_factor=2, mode="nearest") if up else x16
    ref = F.conv2d(xin, w16, b, stride=stride, padding=1)
    Ho, Wo = ref.shape[2:]
    emb = randn(54, N, Cout)
    res = randn(55, N, Cout, Ho, Wo).half()
    ref = ref + emb[:, :, None, None] + res.float()
    wp = w.permute(0, 2, 3, 1).reshape(Cout, 9 * Cin).half().contiguous().cuda()
    out = torch.empty(N * Ho * Wo, Cout, dtype=torch.float16, device="cuda")
    ho, wo = ops.conv3x3(to_nhwc16(x), wp, out, bias=b.cuda(), rowadd=emb.cuda(), residual=to_nhwc16(res.float()).view(-1, Cout),
                         stride=stride, upsample=up)
    assert (ho, wo) == (Ho, Wo)
    e = rel(from_nhwc(out, N, Ho, Wo), ref)
    assert e < 1e-3, e


def test_conv_golden_kats(ops):
    """Downsample / Upsample outputs of the reference's own modules (openaimodel.py:90-159)."""
    from oracle import weights
    g = np.load(os.path.join(G, "op_kats.npz"))
    x = torch.from_numpy(g["gn_x"])
    N, C, H, W = x.shape
    for key, names, seed, kw in (("down_out", ("dn.0.op.weight", "dn.0.op.bias"), 25, dict(stride=2)),
                                 ("up_out", ("up.0.conv.weight", "up.0.conv.bias"), 26, dict(upsample=1))):
        sd = weights.make_state_dict({names[0]: (64, 64, 3, 3), names[1]: (64,)}, seed)
        wp = sd[names[0]].permute(0, 2, 3, 1).reshape(64, -1).half().contiguous().cuda()
        ref = torch.from_numpy(g[key])
        Ho, Wo = ref.shape[2:]
        out = torch.empty(N * Ho * Wo, 64, dtype=torch.float16, device="cuda")
        ops.conv3x3(to_nhwc16(x), wp, out, bias=sd[names[1]].cuda(), **kw)
        e = rel(from_nhwc(out, N, Ho, Wo), ref)
        assert e < 2e-3, (key, e)


@pytest.mark.parametrize("B,heads,nq,nkv,d", [(2, 4, 40, 40, 16), (1, 8, 256, 256, 40), (2, 8, 100, 77, 40),
                                              (1, 8, 128, 128, 80), (1, 8, 64, 77, 160), (2, 5, 200, 257, 64),
                                              (1, 8, 16, 16, 160), (1, 2, 1024, 1024, 40), (1, 1, 70, 9, 48)])
def test_attention(ops, B, heads, nq, nkv, d):
    from oracle import unet_oracle
    C = heads * d
    q, k, v = randn(61, B, nq, C), randn(62, B, nkv, C), randn(63, B, nkv, C)
    q16, k16, v16 = q.half(), k.half(), v.half()

    def split(t):
        return t.float().reshape(B, t.shape[1], heads, d).permute(0, 2, 1, 3).reshape(B * heads, t.shape[1], d)

    ref = unet_oracle.attention_bhnd(split(q16), split(k16), split(v16))
    ref = ref.reshape(B, heads, nq, d).permute(0, 2, 1, 3).reshape(B, nq, C)
    out = torch.empty(B, nq, C, dtype=torch.float16, device="cuda")
    ops.attention(q16.cuda(), k16.cuda(), v16.cuda(), out, B, heads, nq, nkv, d, C, C, C, C)
    e = rel(out, ref)
    assert e < 2e-3, e
    # fused-projection layout: q/k/v as column slices of one [B*n, 3C] buffer (self-attention)
    if nq == nkv:
        qkv = torch.cat([q16, k16, v16], -1).cuda().contiguous()
        flat = qkv.view(B * nq, 3 * C)
        out2 = torch.empty_like(out)
        ops.attention(flat, flat[:, C:], flat[:, 2 * C:], out2, B, heads, nq, nkv, d, 3 * C, 3 * C, 3 * C, C)
        assert torch.equal(out, out2)
    # gated accumulate (router expert sum)
    gate = torch.rand(B, generator=torch.Generator().manual_seed(64))
    out3 = out.clone()
    ops.attention(q16.cuda(), k16.cuda(), v16.cuda(), out3, B, heads, nq, nkv, d, C, C, C, C, gate=gate.cuda(),
                  gate_stride=1, accumulate=True)
    ref3 = out.float().cpu() + gate[:, None, None] * ref
    assert rel(out3, ref3) < 2e-3


def test_cross_attention_module_golden(ops):
    """CrossAttention module output of the reference (attention.py:145-194), assembled from our
    GEMM + attention kernels the way anyedit_b200.unet does."""
    from oracle import weights
    g = np.load(os.path.join(G, "op_kats.npz"))
    x, ctx, ref = (torch.from_numpy(g[k]) for k in ("ca_x", "ca_ctx", "ca_out"))
    shapes = {"attn2.to_q.weight": (64, 64), "attn2.to_k.weight": (64, 48), "attn2.to_v.weight": (64, 48),
              "attn2.to_out.0.weight": (64, 64), "attn2.to_out.0.bias": (64,)}
    sd = weights.make_state_dict(shapes, 22)
    B, n, C = x.shape
    L = ctx.shape[1]
    h16 = lambda t: t.half().cuda().contiguous()
    q = torch.empty(B * n, C, dtype=torch.float16, device="cuda")
    ops.gemm(h16(x).view(B * n, C), h16(sd["attn2.to_q.weight"]), q)
    kv = torch.empty(B * L, 2 * C, dtype=torch.float16, device="cuda")
    ops.gemm(h16(ctx).view(B * L, -1), h16(torch.cat([sd["attn2.to_k.weight"], sd["attn2.to_v.weight"]], 0)), kv)
    a = torch.empty(B * n, C, dtype=torch.float16, device="cuda")
    ops.attention(q, kv, kv[:, C:], a, B, 4, n, L, 16, C, 2 * C, 2 * C, C)
    out = torch.empty(B * n, C, dtype=torch.float32, device="cuda")
    ops.gemm(a, h16(sd["attn2.to_out.0.weight"]), out, bias=sd["attn2.to_out.0.bias"].cuda())
    e = rel(out.view(B, n, C), ref)
    assert e < 3e-3, e


def test_cfg_ddim_step_bit_exact(ops):
    """The fused update reproduces the reference's fp32 tensor arithmetic bit for bit (ddim.py:211-250)."""
    from anyedit_b200.ddim import step_coefficients
    from oracle import ddim_oracle
    sched = ddim_oracle.register_schedule("linear", 1000, 0.00085, 0.012)
    ts = ddim_oracle.make_ddim_timesteps("uniform", 50, 1000)
    for eta in (0.0, 0.7):
        sig, a, ap = ddim_oracle.make_ddim_sampling_parameters(sched["alphas_cumprod"], ts, eta)
        soma = np.sqrt(1.0 - a)
        B, shape = 3, (3, 4, 8, 8)
        x, eu, ec, nz = randn(71, *shape), randn(72, *shape), randn(73, *shape), randn(74, *shape)
        for index in (0, 17, 49):
            coef = torch.tensor(step_coefficients(a, ap, sig, soma, index), dtype=torch.float32).cuda()
            full = lambda v: torch.full((B, 1, 1, 1), float(v))
            a_t, a_prev, s_t, so = full(a[index]), full(ap[index]), full(sig[index]), full(soma[index])
            e_t = eu + 7.5 * (ec - eu)
            pred = (x - so * e_t) / a_t.sqrt()
            dirx = (1.0 - a_prev - s_t ** 2).sqrt() * e_t
            ref = a_prev.sqrt() * pred + dirx + s_t * nz
            xp, p0 = torch.empty(shape, device="cuda"), torch.empty(shape, device="cuda")
            ops.cfg_ddim_step(x.cuda(), torch.cat([eu, ec]).cuda(), coef, 7.5, True, xp, p0,
                              nz.cuda() if eta else None)
            assert torch.equal(p0.cpu(), pred), (eta, index)
            assert torch.equal(xp.cpu(), ref), (eta, index)


def test_router_gate(ops):
    T, D, L, E, B = 7, 256, 5, 11, 6
    table, W, bias = randn(81, T, D, scale=0.5), randn(82, L, E, D, scale=D ** -0.5), 0.1 * randn(83, L, E)
    idx = torch.tensor([0, 6, 3, 3, 1, 5])
    gate = torch.empty(B, L, E, device="cuda")
    ops.router_gate(table.cuda(), idx.cuda(), W.half().cuda(), bias.cuda(), gate)
    ref = torch.softmax(torch.einsum("led,bd->ble", W.half().float(), table[idx]) + bias, -1)
    assert (gate.cpu() - ref).abs().max() < 1e-5


def test_errors_are_loud(ops):
    out = torch.empty(4, 4, dtype=torch.float16, device="cuda")
    with pytest.raises(ValueError):
        ops.gemm(torch.empty(4, 12, dtype=torch.float16, device="cuda"), torch.empty(4, 12, dtype=torch.float16, device="cuda"), out)
    with pytest.raises(Exception):
        ops.gemm(torch.empty(4, 8, dtype=torch.float16), torch.empty(4, 8, dtype=torch.float16), out)  # CPU tensors


@pytest.mark.parametrize("B,heads,nq,nkv,d", [(1, 8, 256, 256, 40), (2, 8, 300, 300, 40), (2, 8, 100, 77, 40),
                                              (1, 8, 1024, 1024, 40), (1, 3, 130, 513, 24)])
def test_attention_padded_heads(ops, B, heads, nq, nkv, d):
    """Head stride padded to ceil16(d) with zero columns (the layout anyedit_b200.unet packs when d % 16 != 0,
    required by the wgmma kernel): same result as the unpadded reference."""
    from anyedit_b200.unet import head_stride_for
    from oracle import unet_oracle
    hs = head_stride_for(d)
    C, Cp = heads * d, heads * hs
    q, k, v = randn(91, B, nq, C), randn(92, B, nkv, C), randn(93, B, nkv, C)
    q16, k16, v16 = q.half(), k.half(), v.half()

    def split(t):
        return t.float().reshape(B, t.shape[1], heads, d).permute(0, 2, 1, 3).reshape(B * heads, t.shape[1], d)

    def pad(t):
        o = torch.zeros(B, t.shape[1], heads, hs, dtype=torch.float16)
        o[..., :d] = t.reshape(B, t.shape[1], heads, d)
        return o.reshape(B, t.shape[1], Cp).cuda().contiguous()

    ref = unet_oracle.attention_bhnd(split(q16), split(k16), split(v16))
    ref = ref.reshape(B, heads, nq, d).permute(0, 2, 1, 3).reshape(B, nq, C)
    out = torch.empty(B, nq, C, dtype=torch.float16, device="cuda")
    ops.attention(pad(q16), pad(k16), pad(v16), out, B, heads, nq, nkv, d, Cp, Cp, Cp, C, head_stride=hs)
    e = rel(out, ref)
    assert e < 2e-3, e


@pytest.mark.parametrize("B,heads,nq,nkv,d,amp", [(1, 8, 256, 256, 40, 1.0), (2, 8, 300, 300, 40, 1.0), (2, 8, 100, 77, 40, 1.0),
                                                  (1, 8, 1024, 1024, 40, 6.0), (1, 3, 130, 513, 24, 3.0),
                                                  (1, 2, 128, 2048, 40, 12.0), (2, 4, 512, 2048, 40, 12.0), (1, 2, 256, 4096, 40, 1.0)])
def test_attention_aux_cols(ops, B, heads, nq, nkv, d, amp):
    """anysd_attn_params::aux_cols -- q pre-scaled by scale*log2(e), K carrying 1.0 in padding columns d, d+1 and V
    in column d (what anyedit_b200.unet packs for d = 40): same softmax(q k^T scale) v as the plain contract.  `amp`
    widens the score range so the running maximum moves many times; keys are sorted by growing norm in the amp = 12
    cases so the maximum keeps rising tile after tile."""
    from anyedit_b200.unet import LOG2E, aux_cols_for, head_stride_for
    from oracle import unet_oracle
    assert aux_cols_for(d)
    hs = head_stride_for(d)
    C, Cp = heads * d, heads * hs
    q, k, v = randn(191, B, nq, C) * amp, randn(192, B, nkv, C), randn(193, B, nkv, C)
    if amp >= 12.0:
        k = k * torch.linspace(0.05, 2.0, nkv).view(1, nkv, 1)
    scale = d ** -0.5
    qs16 = (q * (scale * LOG2E)).half()                      # the operand the kernel sees
    k16, v16 = k.half(), v.half()

    def split(t):
        return t.float().reshape(B, t.shape[1], heads, d).permute(0, 2, 1, 3).reshape(B * heads, t.shape[1], d)

    def pad(t, ones):
        o = torch.zeros(B, t.shape[1], heads, hs, dtype=torch.float16)
        o[..., :d] = t.reshape(B, t.shape[1], heads, d)
        o[..., d:d + ones] = 1.0
        return o.reshape(B, t.shape[1], Cp).cuda().contiguous()

    # reference on exactly the fp16 operands: softmax(q16' k16^T ln2) v16  ==  softmax over base-2 exponent
    ref = unet_oracle.attention_bhnd(split(qs16) / (scale * LOG2E), split(k16), split(v16))
    ref = ref.reshape(B, heads, nq, d).permute(0, 2, 1, 3).reshape(B, nq, C)
    out = torch.empty(B, nq, C, dtype=torch.float16, device="cuda")
    ops.attention(pad(qs16, 0), pad(k16, 2), pad(v16, 1), out, B, heads, nq, nkv, d, Cp, Cp, Cp, C, head_stride=hs,
                  aux_cols=True)
    assert torch.isfinite(out).all()
    e = rel(out, ref)
    assert e < 2e-3, e


def test_attention_aux_cols_unsupported_is_loud(ops):
    """aux_cols with a head that has no spare columns (d = 64) must fail, not silently fall back."""
    B, heads, n, d = 1, 2, 128, 64
    t = torch.zeros(B, n, heads * d, dtype=torch.float16, device="cuda")
    out = torch.empty_like(t)
    with pytest.raises(Exception):
        ops.attention(t, t, t, out, B, heads, n, n, d, heads * d, heads * d, heads * d, heads * d, aux_cols=True)


@pytest.mark.parametrize("N,Cin,Cout,H,W", [(2, 64, 320, 64, 64), (3, 128, 64, 8, 8), (2, 64, 192, 16, 32), (1, 64, 64, 96, 96)])
def test_conv_epilogue_groupnorm_statistics(ops, stats_everywhere, N, Cin, Cout, H, W):
    """anysd_gemm_params::stats: the conv epilogue's per-(image, 32-row slab, channel) {sum, sum of squares} of its fp32
    results (incl. bias, time-embedding row, residual) fold to the per-image channel moments; an odd batch on an 8x8 map
    (two images per 128-row tile) exercises the padded image slot."""
    from anyedit_b200.unet import _pack_conv3
    x, w, b = randn(11, N, Cin, H, W), randn(12, Cout, Cin, 3, 3, scale=0.05), randn(13, Cout)
    res, row = randn(14, N, Cout, H, W), randn(15, N, Cout)
    out = torch.empty(N, H, W, Cout, dtype=torch.float16, device="cuda")
    st = ops.conv3x3(to_nhwc16(x), _pack_conv3(w, "cuda"), out.view(-1, Cout), bias=b.cuda(), rowadd=row.cuda().contiguous(),
                     residual=to_nhwc16(res).view(-1, Cout), stats=True)
    assert st is not None and st.S == H * W // 32 and len(st.parts) == 1
    ref = F.conv2d(x.half().float(), w.half().float(), b, padding=1) + row[:, :, None, None] + res.half().float()
    buf = st.parts[0][0][:N].double().cpu()                              # [N, S, C, 2]
    got = buf.sum(1)
    want = torch.stack([ref.double().sum((2, 3)), (ref.double() ** 2).sum((2, 3))], -1)
    assert rel(got[..., 0], want[..., 0]) < 2e-4 and rel(got[..., 1], want[..., 1]) < 2e-4
    assert rel(from_nhwc(out, N, H, W), ref) < 1e-3


def test_gemm_epilogue_statistics_and_groupnorm_apply(ops, stats_everywhere):
    """Dense contraction (a SpatialTransformer proj_out: bias + residual) with statistics, then GroupNorm fed by them --
    single source and channel concat (two producers) -- against F.group_norm of the fp16 tensor the GEMM wrote."""
    N, HW, K, C1, C2 = 3, 256, 320, 320, 640
    ws = ops.groupnorm_workspace(N, 32, 0, "cuda")
    outs, stats = [], []
    for seed, Cc in ((21, C1), (22, C2)):
        A, Wt, b, r = randn(seed, N * HW, K), randn(seed + 5, Cc, K, scale=K ** -0.5), randn(seed + 9, Cc), randn(seed + 13, N * HW, Cc)
        o = torch.empty(N * HW, Cc, dtype=torch.float16, device="cuda")
        st = ops.gemm(A.half().cuda(), Wt.half().cuda(), o, bias=b.cuda(), residual=r.half().cuda(), rows_per_batch=HW, stats_images=N)
        assert st is not None and st.S == HW // 32
        ref = A.half().float() @ Wt.half().float().t() + b + r.half().float()
        assert rel(o, ref) < 1e-3
        outs.append(o)
        stats.append(st)
    for silu, eps in ((True, 1e-5), (False, 1e-6)):
        gam, bet = randn(31, C1) * 0.2 + 1, randn(32, C1) * 0.1
        y = torch.empty(N, HW, C1, dtype=torch.float16, device="cuda")
        ops.groupnorm(outs[0].view(N, HW, C1), gam.cuda(), bet.cuda(), y, N, HW, eps, silu, ws, stats=stats[0])
        xr = outs[0].float().cpu().view(N, HW, C1).permute(0, 2, 1)
        ref = F.group_norm(xr, 32, gam, bet, eps)
        ref = F.silu(ref) if silu else ref
        assert rel(y.float().cpu().permute(0, 2, 1), ref) < 1e-3
    # channel concat [C1 | C2] = 960 channels, 30 per group: group 10 straddles the two sources
    cat = torch.empty(N * HW, C1 + C2, dtype=torch.float16, device="cuda")
    ops.concat_channels(outs[0], outs[1], cat)
    gam, bet = randn(33, C1 + C2) * 0.2 + 1, randn(34, C1 + C2) * 0.1
    y = torch.empty(N, HW, C1 + C2, dtype=torch.float16, device="cuda")
    both = ops.GnStats(stats[0].parts + stats[1].parts, stats[0].S)
    ops.groupnorm(cat.view(N, HW, -1), gam.cuda(), bet.cuda(), y, N, HW, 1e-5, True, ws, stats=both)
    xr = cat.float().cpu().view(N, HW, -1).permute(0, 2, 1)
    ref = F.silu(F.group_norm(xr, 32, gam, bet, 1e-5))
    assert rel(y.float().cpu().permute(0, 2, 1), ref) < 1e-3
    # a shape that cannot produce statistics says so (rows of one image not a multiple of 32)
    o = torch.empty(3 * 48, C1, dtype=torch.float16, device="cuda")
    assert ops.gemm(randn(41, 3 * 48, K).half().cuda(), randn(42, C1, K).half().cuda(), o, rows_per_batch=48, stats_images=3) is None


def test_split_k_contractions(ops, stats_everywhere):
    """Few output tiles + very long K (the 8x8 level's 2560 -> 1280 convs: 40..80 tiles over K = 23040 on 132 SMs): the schedule
    splits K across CTAs; the partial sums are added in split order by whichever unit arrives last, so two runs agree bit for
    bit and the result matches the unsplit arithmetic to fp32 summation-order noise."""
    import ctypes as C
    from anyedit_b200 import _lib
    from anyedit_b200.unet import _pack_conv3
    # conv 8x8, 2560 -> 1280, batch 16 (M = 1024), bias + residual + epilogue statistics
    N, Cin, Cout, H, W = 16, 2560, 1280, 8, 8
    x, w, b, res = randn(51, N, Cin, H, W), randn(52, Cout, Cin, 3, 3, scale=0.01), randn(53, Cout), randn(54, N, Cout, H, W)
    xin, wp, rin = to_nhwc16(x), _pack_conv3(w, "cuda"), to_nhwc16(res).view(-1, Cout)
    outs = []
    for _ in range(2):
        out = torch.empty(N, H, W, Cout, dtype=torch.float16, device="cuda")
        st = ops.conv3x3(xin, wp, out.view(-1, Cout), bias=b.cuda(), residual=rin, stats=True)
        outs.append(out)
    assert torch.equal(outs[0], outs[1])
    p = _lib.GemmParams()
    p.A, p.W, p.out = xin.data_ptr(), wp.data_ptr(), outs[0].data_ptr()
    p.M, p.N, p.K, p.lda, p.ldw, p.ldo = N * H * W, Cout, 9 * Cin, Cin, 9 * Cin, Cout
    p.out_dtype, p.conv, p.Nimg, p.H, p.Wd, p.Cin, p.stride, p.rows_per_batch = _lib.F16, 1, N, H, W, Cin, 1, H * W
    assert _lib.load().anysd_gemm_splitk_workspace_bytes(C.byref(p)) > 0, "the 8x8 conv is expected to run split-K"
    ref = F.conv2d(x.half().float(), w.half().float(), b, padding=1) + res.half().float()
    assert rel(from_nhwc(outs[0], N, H, W), ref) < 1e-3
    got = st.parts[0][0][:N].double().cpu().sum(1)
    assert rel(got[..., 0], ref.double().sum((2, 3))) < 2e-4
    # dense: M = 1024, N = 1280, K = 5120 with residual (the deep level's FF output projection)
    A, Wt, bb, r = randn(61, 1024, 5120), randn(62, 1280, 5120, scale=5120 ** -0.5), randn(63, 1280), randn(64, 1024, 1280)
    o = torch.empty(1024, 1280, dtype=torch.float16, device="cuda")
    ops.gemm(A.half().cuda(), Wt.half().cuda(), o, bias=bb.cuda(), residual=r.half().cuda())
    assert rel(o, A.half().float() @ Wt.half().float().t() + bb + r.half().float()) < 1e-3


@pytest.mark.parametrize("M,C,N,act,res_mean", [(300, 320, 1152, 0, 0.0), (4096, 320, 2560, 2, 3.0), (1000, 640, 640, 0, -8.0),
                                                (256, 1280, 3840, 0, 1.0)])
def test_layernorm_folded_into_contractions(ops, M, C, N, act, res_mean):
    """nn.LayerNorm between two contractions (attention.py:262-264, 271-274) without its own pass: the producer's epilogue
    leaves per-row moments (row_stats), the consumer takes the un-normalised rows with gamma folded into W (ln_stats).
    Reference: fp32 LayerNorm of the stored fp16 rows, then the fp32 contraction (+ GEGLU).  ``res_mean`` gives the rows a
    mean of several standard deviations: the E[x^2] - mean^2 combine must survive it."""
    a = randn(1, M, 192).half()
    wp = randn(2, C, 192, scale=192 ** -0.5).half()
    bp = randn(3, C)
    res = (randn(4, M, C) + res_mean).half()
    gamma, beta = 1.0 + 0.2 * randn(5, C), 0.1 * randn(6, C)
    w = randn(7, N, C, scale=C ** -0.5)
    bias = 0.1 * randn(8, N)
    # producer: x = a wp^T + bp + res, with the row moments of x from the epilogue
    x = torch.empty(M, C, dtype=torch.float16, device="cuda")
    rs = ops.row_stats_buffer(M, C, "cuda")
    rs.fill_(float("nan"))
    ops.gemm(a.cuda(), wp.cuda(), x, bias=bp.cuda(), residual=res.cuda(), row_stats=rs)
    x32 = a.float() @ wp.float().t() + bp + res.float()
    assert rel(x, x32) < 6e-4
    s = rs.sum(0).cpu().double()
    assert torch.isfinite(s).all()
    assert float((s[:, 0] - x32.double().sum(1)).abs().max()) < 2e-3 * C ** 0.5 * (1 + abs(res_mean))
    assert rel(s[:, 1], (x32.double() ** 2).sum(1)) < 1e-5
    # consumer: LayerNorm(x) w^T + bias (+ GEGLU), gamma / beta folded on the host exactly as UNetModel._ln_folded does
    w16 = w.half()
    wf = (w16.float() * gamma[None, :]).half()
    cs = wf.float().sum(1)
    bf = w16.float() @ beta + bias
    n_out = N // 2 if act == 2 else N
    out = torch.empty(M, n_out, dtype=torch.float16, device="cuda")
    ops.gemm(x, wf.cuda(), out, bias=bf.cuda(), act=act, ln=(rs, cs.cuda(), 1e-5))
    xs = x.float().cpu()
    ref = F.layer_norm(xs, (C,), gamma, beta, 1e-5) @ w16.float().t() + bias
    if act == 2:                               # interleaved (a_j, gate_j) rows
        ref = ref[:, 0::2] * F.gelu(ref[:, 1::2])
    e = rel(out, ref)
    # the same computation through the separate LayerNorm kernel (fp16 normalised rows): the fold must not be worse
    ln = torch.empty_like(x)
    ops.layernorm(x, gamma.cuda(), beta.cuda(), ln)
    out2 = torch.empty_like(out)
    ops.gemm(ln, w16.cuda(), out2, bias=bias.cuda(), act=act)
    e2 = rel(out2, ref)
    print(f"folded LayerNorm M={M} C={C} N={N} act={act}: {e:.2e} (separate kernel {e2:.2e})")
    assert e < 6e-4 and e < 1.3 * e2 + 1e-4


def test_layernorm_fold_unsupported_is_loud(ops):
    x = torch.zeros(64, 96, dtype=torch.float16, device="cuda")          # K % 64 != 0
    w = torch.zeros(64, 96, dtype=torch.float16, device="cuda")
    out = torch.empty(64, 64, dtype=torch.float16, device="cuda")
    rs = torch.zeros(1, 64, 2, device="cuda")
    with pytest.raises(Exception):
        ops.gemm(x, w, out, bias=torch.zeros(64, device="cuda"), ln=(rs, torch.zeros(64, device="cuda"), 1e-5))


def test_gelu_epilogue_accuracy(ops):
    """The GELU of the contraction epilogues (act 2 GEGLU, act 3 nn.GELU) is the exact erf form evaluated as a fitted logistic
    (gemm_wgmma.cu: p_gelu): |x Phi(x) - kernel| <= 1.2e-5 + fp16 rounding over the whole range, including the saturated tails."""
    x = torch.cat([torch.linspace(-12, 12, 64 * 1024 - 6), torch.tensor([-1e4, -60.0, -0.0, 0.0, 60.0, 1e4])]).half()
    A = x.view(-1, 64).cuda()                                  # values pass through an identity contraction
    W = torch.eye(64, dtype=torch.float16, device="cuda")
    out = torch.empty_like(A)
    ops.gemm(A, W, out, act=3)
    ref = F.gelu(x.double()).view(-1, 64)
    got = out.double().cpu()
    assert torch.isfinite(got).all()
    err = (got - ref).abs()
    bound = 1.2e-5 + ref.abs() * 2.0 ** -11 + 6e-8            # fit + fp16 rounding of the result (+ the subnormal step)
    worst = float((err / bound).max())
    print(f"gelu epilogue: max |err| {float(err.max()):.2e}, max err / bound {worst:.3f}")
    assert worst <= 1.0
