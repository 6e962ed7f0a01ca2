"""The fused 320-channel GEGLU feed-forward (anyedit_b200/csrc/feedforward_wgmma.cu, ``ops.geglu_ff``) against the two
contractions it replaces in the UNet (``ops.gemm`` act 2 into the hidden tensor, then ``ops.gemm`` + bias + residual):

* bit-identical (``torch.equal``) at the UNet's row counts, at every residue of M mod 128 that touches a tile edge, at
  M = 64 and M = 1, for two seeds with weights at nn.Linear's init scale;
* within a float64 bound of the exact result (the bound of tests/test_gpu_contraction.py carried through both products);
* a row does not depend on the rows around it (the same rows alone give the same bits);
* shapes the kernel does not serve are refused.

The ff1 chunk order the kernel relies on is checked on the host (no GPU needed).
"""
import pytest
import torch

from anyedit_b200.unet import ff1_chunk_order

C, HID = 320, 1280
U = 2.0 ** -24
C_ACC = 4                          # tests/test_gpu_contraction.py: truncating tensor-core adds + fp32 epilogue additions
SLOPE = 1.13                       # steepest slope of GELU
P_GELU_FIT = 1.2e-5                # |x Phi(x) - p_gelu(x)| of the fp16-output GEGLU epilogue

M_CASES = (65536, 36864, 37 * 128 + 1, 37 * 128 + 63, 37 * 128 + 64, 37 * 128 + 65, 37 * 128 + 127, 64, 1)
SEEDS = (0, 1)


# ---- host: the ff1 chunk order ------------------------------------------------------------------------------------
def test_ff1_chunk_order_is_a_pair_preserving_bijection():
    perm = ff1_chunk_order(HID)
    assert perm.shape == (2 * HID,)
    assert torch.equal(perm.sort().values, torch.arange(2 * HID))
    a, g = perm[0::2], perm[1::2]
    assert torch.equal(a % 2, torch.zeros_like(a)) and torch.equal(g, a + 1)       # (a_j, gate_j) stay adjacent, in order
    assert torch.equal(a // 2 // 32, torch.arange(HID) // 32)                      # every unit stays in its chunk of 32


def test_ff1_chunk_order_gives_the_register_a_fragment():
    # S column 8 i + 2 q + e of a chunk (e = 0: a, 1: gate) holds packed pair 4 i + q; the GEGLU values of steps
    # 4 s .. 4 s + 3 become the m64k16 A fragment of k16 step s, whose registers hold columns (k) 2q, 2q + 1 (regs 0, 1) and
    # 2q + 8, 2q + 9 (regs 2, 3): the hidden unit behind each must be 16 s + that column -- natural order within the step
    unit = ff1_chunk_order(HID)[0::2] // 2
    for ch in range(HID // 32):
        for q in range(4):
            for s in range(2):
                steps = [4 * s, 4 * s + 1, 4 * s + 2, 4 * s + 3]
                got = [int(unit[32 * ch + 4 * i + q]) for i in steps]
                assert got == [32 * ch + 16 * s + k for k in (2 * q, 2 * q + 1, 2 * q + 8, 2 * q + 9)]


# ---- GPU ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from anyedit_b200 import ops as o
    return o


def _weights(seed, dev):
    """ff1 / ff2 of one 320-channel block at nn.Linear's init scale, packed as unet.py packs them."""
    g = torch.Generator().manual_seed(seed)
    u = lambda shape, fan_in: (torch.rand(shape, generator=g) * 2 - 1) / fan_in ** 0.5
    w1, b1 = u((2 * HID, C), C), u((2 * HID,), C)                   # proj of GEGLU: rows [a | gate]
    w2, b2 = u((C, HID), HID), u((C,), HID)
    ff1_w = torch.stack([w1[:HID], w1[HID:]], 1).reshape(2 * HID, C).half()
    ff1_b = torch.stack([b1[:HID], b1[HID:]], 1).reshape(-1).float()
    perm = ff1_chunk_order(HID)
    return dict(ff1_w=ff1_w.to(dev), ff1_b=ff1_b.to(dev), ff2_w=w2.half().to(dev), ff2_b=b2.float().to(dev),
                ff1p_w=ff1_w[perm].contiguous().to(dev), ff1p_b=ff1_b[perm].contiguous().to(dev),
                ff2t_w=w2.half().t().contiguous().to(dev))


def _inputs(M, seed, dev):
    g = torch.Generator().manual_seed(1000 + seed)
    x = torch.randn(M, C, generator=g).half().to(dev)              # LayerNorm output scale
    res = torch.randn(M, C, generator=g).half().to(dev)
    return x, res


def _two_launch(ops, W, x, res):
    hid = torch.empty(x.shape[0], HID, dtype=torch.float16, device=x.device)
    ops.gemm(x, W["ff1_w"], hid, bias=W["ff1_b"], act=2)
    out = torch.empty_like(res)
    ops.gemm(hid, W["ff2_w"], out, bias=W["ff2_b"], residual=res)
    return out


def _fused(ops, W, x, res):
    out = torch.empty_like(res)
    ops.geglu_ff(x, W["ff1p_w"], W["ff1p_b"], W["ff2t_w"], W["ff2_b"], res, out)
    return out


def _gelu(v):
    return 0.5 * v * (1.0 + torch.erf(v * 0.5 ** 0.5))


def _fp64_bound(W, x, res):
    """(y, e): the exact result from the fp16 operands and the bound on |out - y| -- tests/test_gpu_contraction.py's bound for
    the GEGLU contraction (fp16 output), carried through the second contraction by |W2|, plus that contraction's own."""
    xd, w1 = x.double(), W["ff1_w"].double()
    pre = xd @ w1.t() + W["ff1_b"].double()
    e_pre = C_ACC * U * (C * (xd.abs() @ w1.abs().t()) + W["ff1_b"].double().abs())
    del xd
    a, gt, ea, eg = pre[:, 0::2], pre[:, 1::2], e_pre[:, 0::2], e_pre[:, 1::2]
    h = a * _gelu(gt)
    eh = _gelu(gt).abs() * ea + (a.abs() + ea) * (SLOPE * eg + P_GELU_FIT)
    eh = eh + 2.0 ** -11 * (h.abs() + eh) + 2.0 ** -25                # the hidden tensor's fp16 rounding
    del pre, e_pre, a, gt, ea, eg
    w2 = W["ff2_w"].double()
    y = h @ w2.t() + W["ff2_b"].double() + res.double()
    e = eh @ w2.abs().t() + C_ACC * U * (HID * ((h.abs() + eh) @ w2.abs().t()) + W["ff2_b"].double().abs() + res.double().abs()
                                          + y.abs())
    return y, e + 2.0 ** -11 * (y.abs() + e) + 2.0 ** -25


@pytest.mark.gpu
@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("M", M_CASES)
def test_fused_equals_two_contractions_and_fp64_bound(ops, M, seed):
    dev = torch.device("cuda")
    W = _weights(seed, dev)
    x, res = _inputs(M, seed, dev)
    ref = _two_launch(ops, W, x, res)
    got = _fused(ops, W, x, res)
    torch.cuda.synchronize()
    assert torch.isfinite(got.float()).all()
    y, e = _fp64_bound(W, x, res)
    err = (got.double() - y).abs()
    worst = float((err / e).max())
    assert worst <= 1.0, f"M={M} seed={seed}: |out - fp64| reaches {worst:.3f} x the bound"
    diff = (got.float() - ref.float()).abs().max().item()
    assert torch.equal(got, ref), f"M={M} seed={seed}: fused differs from the two contractions (max |diff| {diff:.3g})"


@pytest.mark.gpu
def test_rows_do_not_depend_on_their_neighbours(ops):
    dev = torch.device("cuda")
    W = _weights(3, dev)
    x, res = _inputs(65536, 3, dev)
    full = _fused(ops, W, x, res)
    for r0, n in ((0, 1), (1000, 77), (40000, 128), (65536 - 65, 65)):
        part = _fused(ops, W, x[r0:r0 + n], res[r0:r0 + n])
        assert torch.equal(part, full[r0:r0 + n]), (r0, n)
    again = _fused(ops, W, x, res)
    assert torch.equal(again, full)                                   # and run to run


@pytest.mark.gpu
def test_unservable_shapes_raise(ops):
    dev = torch.device("cuda")
    lib = ops._lib.load()
    W = _weights(0, dev)
    x, res = _inputs(256, 0, dev)
    out = torch.empty_like(res)
    P = lambda t: ops._ptr(t)
    S = ops._stream()

    def call(x_, w1, b1, w2t, b2, r, o, M, Cc, hid, ldx=C, ldr=C, ldo=C):
        return lib.anysd_geglu_ff_f16(P(x_), ldx, P(w1), P(b1), P(w2t), P(b2), P(r), ldr, P(o), ldo, M, Cc, hid, S)

    args = (x, W["ff1p_w"], W["ff1p_b"], W["ff2t_w"], W["ff2_b"], res, out)
    assert call(*args, 256, C, HID) == 0
    assert call(*args, 256, 640, 4 * 640) == ops._lib.EUNSUPPORTED              # another width
    assert call(*args, 256, C, 2 * C) == ops._lib.EUNSUPPORTED                  # hidden != 4 C
    assert call(*args, 0, C, HID) == ops._lib.EINVAL
    assert call(*args, 256, C, HID, ldx=324) == ops._lib.EINVAL                 # pitch not a multiple of 8
    xm = x.view(-1)[1:1 + 255 * C].view(255, C)                                 # 2-byte offset: misaligned
    assert call(xm, *args[1:], 255, C, HID) == ops._lib.EINVAL
    assert call(x, W["ff1p_w"], W["ff1p_b"], W["ff2t_w"], W["ff2_b"], res, out.view(-1)[4:4 + 255 * C], 255, C, HID) \
        == ops._lib.EINVAL
    with pytest.raises(ValueError):
        ops.geglu_ff(xm, W["ff1p_w"], W["ff1p_b"], W["ff2t_w"], W["ff2_b"], res[:255], out[:255])
    torch.cuda.synchronize()
