"""The fused cross-attention block (ops.xattn_block) against the six launches it replaces: bit for bit, within the float64
bound of the exact chain, independent of the surrounding rows, and refusing the shapes it does not serve."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))

pytestmark = pytest.mark.gpu

C, HEADS, D, HS, CTX = 320, 8, 40, 48, 768
CP = HEADS * HS


def _weights(seed, dev):
    from anyedit_b200.unet import LOG2E, aux_bias, pad_heads
    g = torch.Generator().manual_seed(seed)
    u = lambda shape, fan_in: (torch.rand(shape, generator=g) * 2 - 1) / fan_in ** 0.5
    wq = pad_heads(u((C, C), C) * (D ** -0.5 * LOG2E), HEADS, D, HS)
    wkv = torch.cat([pad_heads(u((C, CTX), CTX), HEADS, D, HS), pad_heads(u((C, CTX), CTX), HEADS, D, HS)], 0)
    kv_b = torch.cat([aux_bias(HEADS, D, HS, 2), aux_bias(HEADS, D, HS, 1)])
    h, f = (lambda t: t.half().contiguous().to(dev)), (lambda t: t.float().contiguous().to(dev))
    return g, dict(o1_w=h(u((C, C), C)), o1_b=f(u((C,), C)), ln2_w=f(1 + 0.1 * torch.randn(C, generator=g)),
                   ln2_b=f(0.1 * torch.randn(C, generator=g)), q_w=h(wq), kv_w=h(wkv), kv_b=f(kv_b),
                   o2_w=h(u((C, C), C)), o2_b=f(u((C,), C)), ln3_w=f(1 + 0.1 * torch.randn(C, generator=g)),
                   ln3_b=f(0.1 * torch.randn(C, generator=g)))


def _inputs(B, n, L, seed):
    from anyedit_b200 import ops
    dev = torch.device("cuda")
    g, W = _weights(seed, dev)
    a1 = torch.randn(B * n, C, generator=g).half().to(dev)
    t = torch.randn(B * n, C, generator=g).half().to(dev)
    ctx = torch.randn(B * L, CTX, generator=g).half().to(dev)            # a different context per image
    kv = torch.empty(B * L, 2 * CP, dtype=torch.float16, device=dev)
    ops.gemm(ctx, W["kv_w"], kv, bias=W["kv_b"])
    return W, a1, t, kv


def _chain(W, a1, t, kv, B, n, L):
    from anyedit_b200 import ops
    t2, l2, t3, l3 = (torch.empty_like(t) for _ in range(4))
    q = torch.empty(B * n, CP, dtype=torch.float16, device=t.device)
    a2 = torch.empty_like(t)
    ops.gemm(a1, W["o1_w"], t2, bias=W["o1_b"], residual=t)
    ops.layernorm(t2, W["ln2_w"], W["ln2_b"], l2)
    ops.gemm(l2, W["q_w"], q)
    ops.attention(q, kv, kv[:, CP:], a2, B, HEADS, n, L, D, CP, 2 * CP, 2 * CP, C, head_stride=HS, aux_cols=True)
    ops.gemm(a2, W["o2_w"], t3, bias=W["o2_b"], residual=t2)
    ops.layernorm(t3, W["ln3_w"], W["ln3_b"], l3)
    return t2, t3, l3


def _fused(W, a1, t, kv, n, L):
    from anyedit_b200 import ops
    t2, t3, l3 = (torch.empty_like(t) for _ in range(3))
    ops.xattn_block(a1, t, W["o1_w"], W["o1_b"], W["ln2_w"], W["ln2_b"], W["q_w"], kv, L, W["o2_w"], W["o2_b"],
                    W["ln3_w"], W["ln3_b"], t2, t3, l3, n, HEADS, D, HS)
    return t2, t3, l3


@pytest.mark.parametrize("B,n,L,seed", [(16, 4096, 77, 0), (4, 9216, 77, 1), (1, 1024, 77, 0), (2, 1024, 77, 1),
                                        (2, 1024, 1, 0), (2, 1024, 16, 1), (2, 1024, 80, 0), (2, 1024, 80, 1)])
def test_xattn_block_bit_identical_to_chain(B, n, L, seed):
    W, a1, t, kv = _inputs(B, n, L, seed)
    ref = _chain(W, a1, t, kv, B, n, L)
    got = _fused(W, a1, t, kv, n, L)
    torch.cuda.synchronize()
    for name, r, o in zip(("t2", "t3", "l3"), ref, got):
        assert torch.equal(r, o), f"{name}: {(r.float() - o.float()).abs().max().item()} max abs difference"


def test_xattn_block_float64_bound():
    """Against the exact chain in float64 (from the same fp16 operands): the fp16 roundings of the intermediates bound it."""
    B, n, L = 2, 1024, 77
    W, a1, t, kv = _inputs(B, n, L, 3)
    t2, t3, l3 = _fused(W, a1, t, kv, n, L)
    torch.cuda.synchronize()
    d = lambda x: x.double().cpu()
    ln = lambda x, w, b: torch.nn.functional.layer_norm(x, (C,), d(w), d(b), 1e-5)
    e2 = d(a1) @ d(W["o1_w"]).T + d(W["o1_b"]) + d(t)
    q = (ln(d(t2), W["ln2_w"], W["ln2_b"]) @ d(W["q_w"]).T).view(B, n, HEADS, HS)[..., :D]
    k = d(kv[:, :CP]).view(B, L, HEADS, HS)[..., :D]
    v = d(kv[:, CP:]).view(B, L, HEADS, HS)[..., :D]
    s = torch.einsum("bihd,bjhd->bhij", q, k) * torch.log(torch.tensor(2.0, dtype=torch.float64))
    o = torch.einsum("bhij,bjhd->bihd", torch.softmax(s, -1), v).reshape(B * n, C)
    e3 = o @ d(W["o2_w"]).T + d(W["o2_b"]) + d(t2)
    e_l3 = ln(d(t3), W["ln3_w"], W["ln3_b"])
    rel = lambda a, b: float((d(a) - b).norm() / b.norm())
    assert rel(t2, e2) < 1e-3 and rel(t3, e3) < 3e-3 and rel(l3, e_l3) < 1e-3, (rel(t2, e2), rel(t3, e3), rel(l3, e_l3))


def test_xattn_block_rows_independent():
    """A tile's rows give the same bits whatever rows surround them (other tiles, other images)."""
    B, n, L = 2, 1024, 77
    W, a1, t, kv = _inputs(B, n, L, 4)
    full = _fused(W, a1, t, kv, n, L)
    a1b, tb = a1.clone(), t.clone()
    a1b[:128].normal_()
    tb[:128].normal_()
    a1b[n + 256:] = 0
    other = _fused(W, a1b, tb, kv, n, L)
    torch.cuda.synchronize()
    for f, o in zip(full, other):
        assert torch.equal(f[128:n + 256], o[128:n + 256])


def test_xattn_block_refusals():
    from anyedit_b200 import ops
    B, n, L = 1, 1024, 77
    W, a1, t, kv = _inputs(B, n, L, 5)
    t2, t3, l3 = (torch.empty_like(t) for _ in range(3))
    call = lambda **kw: ops.xattn_block(a1, t, W["o1_w"], W["o1_b"], W["ln2_w"], W["ln2_b"], W["q_w"], kv,
                                        kw.get("L", L), W["o2_w"], W["o2_b"], W["ln3_w"], W["ln3_b"], t2, t3, l3,
                                        kw.get("n", n), kw.get("heads", HEADS), kw.get("d", D), kw.get("hs", HS),
                                        aux_cols=kw.get("aux", True))
    kv81 = torch.zeros(81, 2 * CP, dtype=torch.float16, device="cuda")
    with pytest.raises(ValueError):
        ops.xattn_block(a1, t, W["o1_w"], W["o1_b"], W["ln2_w"], W["ln2_b"], W["q_w"], kv81, 81, W["o2_w"], W["o2_b"],
                        W["ln3_w"], W["ln3_b"], t2, t3, l3, n, HEADS, D, HS)
    for kw in ({"heads": 4}, {"hs": 40}, {"d": 48}, {"n": 512 + 64}, {"aux": False}):
        with pytest.raises(ValueError):
            call(**kw)
    a640 = torch.zeros(n, 640, dtype=torch.float16, device="cuda")
    with pytest.raises(ValueError):
        ops.xattn_block(a640, a640, W["o1_w"], W["o1_b"], W["ln2_w"], W["ln2_b"], W["q_w"], kv, L, W["o2_w"], W["o2_b"],
                        W["ln3_w"], W["ln3_b"], a640, a640, a640, n, HEADS, D, HS)
