"""The pipelined wgmma attention forward (attention_wgmma.cu) at the edges of its kv-tile schedule, against the fp32 CPU
reference on the same fp16 operands.

The kernel issues S_j = Q K_j^T together with P_{j-1} V_{j-1}, keeps (K, V) tiles in a ring of 3 stages, and gives each of
two consumer warpgroups 64 of a CTA's 128 query rows.  Tiles are 128 keys for ceil16(d) <= 64 and 64 keys above.  The cases
reach: a single kv tile (prologue straight into the tail), exactly 2 and 3 tiles, k tiles +- 1 key (a partial last tile of
1 or BKV - 1 keys), more tiles than ring stages (the ring wraps), and n_q % 128 <= 64 (the second consumer warpgroup of the
last CTA has no valid rows but still takes its issue turns).  Also the forward's base-2 log-sum-exp against torch.logsumexp."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from anyedit_b200 import ops as o
    sms, major, minor = o.device_info()
    assert (major, minor) == (9, 0), f"sm_90a kernels need a Hopper GPU (H100), got cc {major}.{minor}"
    return o


def randn(seed, *shape, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g) * scale


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def split(t, B, heads, d):
    return t.float().reshape(B, t.shape[1], heads, d).permute(0, 2, 1, 3).reshape(B * heads, t.shape[1], d)


def merge(t, B, heads, n, d):
    return t.reshape(B, heads, n, d).permute(0, 2, 1, 3).reshape(B, n, heads * d)


def pad_heads(t, B, heads, d, hs, ones=0):
    o = torch.zeros(B, t.shape[1], heads, hs, dtype=torch.float16)
    o[..., :d] = t.reshape(B, t.shape[1], heads, d)
    o[..., d:d + ones] = 1.0
    return o.reshape(B, t.shape[1], heads * hs).cuda().contiguous()


@pytest.mark.parametrize("B,heads,nq,nkv,d", [
    (1, 4, 130, 256, 64),      # exactly 2 tiles of 128; idle second warpgroup in the last CTA
    (1, 4, 384, 384, 32),      # exactly 3 tiles (= ring stages); fused-qkv layout
    (1, 2, 64, 383, 48),       # 3 tiles - 1 key
    (2, 3, 70, 513, 64),       # 4 tiles + 1 key: the ring wraps, a last tile of one key
    (1, 2, 100, 77, 16),       # a single partial tile
    (1, 4, 200, 129, 80),      # 64-key tiles: 2 tiles + 1 key
    (1, 2, 130, 192, 160),     # exactly 3 tiles of 64
    (1, 2, 70, 128, 112),      # exactly 2 tiles of 64
    (1, 2, 40, 255, 96),       # 4 tiles - 1 key; only the first warpgroup has rows
    (2, 2, 192, 192, 144),     # 3 tiles; fused-qkv layout
])
def test_attention_tile_edges(ops, B, heads, nq, nkv, d):
    from oracle import unet_oracle
    C = heads * d
    q, k, v = randn(361, B, nq, C), randn(362, B, nkv, C), randn(363, B, nkv, C)
    q16, k16, v16 = q.half(), k.half(), v.half()
    ref = merge(unet_oracle.attention_bhnd(split(q16, B, heads, d), split(k16, B, heads, d), split(v16, B, heads, d)),
                B, heads, nq, d)
    out = torch.empty(B, nq, C, dtype=torch.float16, device="cuda")
    ops.attention(q16.cuda(), k16.cuda(), v16.cuda(), out, B, heads, nq, nkv, d, C, C, C, C)
    e = rel(out, ref)
    assert e < 2e-3, e
    # fused-projection layout (self-attention): the same bits from column slices of one [B*n, 3C] buffer
    if nq == nkv:
        flat = torch.cat([q16, k16, v16], -1).cuda().contiguous().view(B * nq, 3 * C)
        out2 = torch.empty_like(out)
        ops.attention(flat, flat[:, C:], flat[:, 2 * C:], out2, B, heads, nq, nkv, d, 3 * C, 3 * C, 3 * C, C)
        assert torch.equal(out, out2)
    # gated accumulate
    gate = torch.rand(B, generator=torch.Generator().manual_seed(364))
    out3 = out.clone()
    ops.attention(q16.cuda(), k16.cuda(), v16.cuda(), out3, B, heads, nq, nkv, d, C, C, C, C, gate=gate.cuda(),
                  gate_stride=1, accumulate=True)
    assert rel(out3, out.float().cpu() + gate[:, None, None] * ref) < 2e-3


@pytest.mark.parametrize("B,heads,nq,nkv,d", [(1, 4, 130, 256, 40), (1, 4, 64, 385, 40), (2, 2, 130, 128, 40),
                                              (1, 3, 200, 127, 24)])
def test_attention_padded_heads_tile_edges(ops, B, heads, nq, nkv, d):
    """Head stride padded to ceil16(d) with zero columns (anyedit_b200.unet's layout for d % 16 != 0)."""
    from anyedit_b200.unet import head_stride_for
    from oracle import unet_oracle
    hs = head_stride_for(d)
    C, Cp = heads * d, heads * hs
    q, k, v = randn(371, B, nq, C), randn(372, B, nkv, C), randn(373, B, nkv, C)
    q16, k16, v16 = q.half(), k.half(), v.half()
    ref = merge(unet_oracle.attention_bhnd(split(q16, B, heads, d), split(k16, B, heads, d), split(v16, B, heads, d)),
                B, heads, nq, d)
    out = torch.empty(B, nq, C, dtype=torch.float16, device="cuda")
    ops.attention(pad_heads(q16, B, heads, d, hs), pad_heads(k16, B, heads, d, hs), pad_heads(v16, B, heads, d, hs), out,
                  B, heads, nq, nkv, d, Cp, Cp, Cp, C, head_stride=hs)
    e = rel(out, ref)
    assert e < 2e-3, e


@pytest.mark.parametrize("B,heads,nq,nkv,d,amp", [(1, 4, 130, 384, 40, 6.0), (1, 2, 70, 127, 40, 12.0),
                                                  (1, 2, 200, 257, 40, 12.0), (2, 8, 4096, 4096, 40, 1.0)])
def test_attention_aux_cols_tile_edges(ops, B, heads, nq, nkv, d, amp):
    """aux_cols operands (q pre-scaled by scale*log2(e), ones in K's padding columns d, d+1 and V's column d), including one
    UNet-sized self-attention of the 64x64 level.  amp = 12 sorts the keys by growing norm, so the running maximum rises
    tile after tile and the rescale of O is exercised on every step."""
    from anyedit_b200.unet import LOG2E, aux_cols_for, head_stride_for
    from oracle import unet_oracle
    assert aux_cols_for(d)
    hs = head_stride_for(d)
    C, Cp = heads * d, heads * hs
    q, k, v = randn(381, B, nq, C) * amp, randn(382, B, nkv, C), randn(383, B, nkv, C)
    if amp >= 12.0:
        k = k * torch.linspace(0.05, 2.0, nkv).view(1, nkv, 1)
    scale = d ** -0.5
    qs16 = (q * (scale * LOG2E)).half()
    k16, v16 = k.half(), v.half()
    ref = merge(unet_oracle.attention_bhnd(split(qs16, B, heads, d) / (scale * LOG2E), split(k16, B, heads, d),
                                           split(v16, B, heads, d)), B, heads, nq, d)
    out = torch.empty(B, nq, C, dtype=torch.float16, device="cuda")
    ops.attention(pad_heads(qs16, B, heads, d, hs), pad_heads(k16, B, heads, d, hs, 2), pad_heads(v16, B, heads, d, hs, 1),
                  out, B, heads, nq, nkv, d, Cp, Cp, Cp, C, head_stride=hs, aux_cols=True)
    assert torch.isfinite(out).all()
    e = rel(out, ref)
    assert e < 2e-3, e


@pytest.mark.parametrize("B,heads,nq,nkv,d", [(2, 4, 130, 333, 40), (1, 4, 200, 300, 80), (2, 2, 130, 257, 160)])
def test_attention_lse(ops, B, heads, nq, nkv, d):
    """anysd_attn_params::lse: the base-2 log-sum-exp of every score row against torch.logsumexp on the same fp16 operands.
    d = 40 runs the aux_cols contract of the UNet (q pre-scaled by scale*log2(e)); 80 and 160 the plain one."""
    from anyedit_b200.unet import LOG2E, head_stride_for
    aux = d % 16 == 8
    hs = head_stride_for(d) if aux else d
    C, Cp = heads * d, heads * hs
    q, k, v = randn(391, B, nq, C), randn(392, B, nkv, C), randn(393, B, nkv, C)
    scale = d ** -0.5
    q16 = (q * (scale * LOG2E)).half() if aux else q.half()
    k16, v16 = k.half(), v.half()
    s = torch.einsum("bhid,bhjd->bhij", split(q16, B, heads, d).double().view(B, heads, nq, d),
                     split(k16, B, heads, d).double().view(B, heads, nkv, d))
    s = s / LOG2E if aux else s * scale                      # natural-log scores
    ref = torch.logsumexp(s, -1) * LOG2E
    out = torch.empty(B, nq, C, dtype=torch.float16, device="cuda")
    lse = torch.full((B, heads, nq), float("nan"), dtype=torch.float32, device="cuda")
    ops.attention(pad_heads(q16, B, heads, d, hs), pad_heads(k16, B, heads, d, hs, 2 if aux else 0),
                  pad_heads(v16, B, heads, d, hs, 1 if aux else 0), out, B, heads, nq, nkv, d, Cp, Cp, Cp, C,
                  head_stride=hs, aux_cols=aux, lse=lse)
    assert torch.isfinite(lse).all()
    err = (lse.double().cpu() - ref).abs().max().item()
    assert err < 1e-3, err
