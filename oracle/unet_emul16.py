"""Rounding-matched restatement of the UNet forward (TEST INFRASTRUCTURE, see oracle/__init__.py).

``unet_oracle`` is the fp32 specification (the reference's arithmetic).  This module evaluates the SAME graph in
fp32 on the CPU but rounds to fp16 exactly where the CUDA path stores fp16 (DESIGN.md 2: fp16 weights, fp16
NHWC activations, fp32 accumulation / statistics / softmax / eps), so that

    |cuda - emul16|   measures implementation error (should be ~1e-4: accumulation order, ex2.approx, the
                      lazy softmax reference), while
    |emul16 - fp32|   is the irreducible cost of fp16 tensor-core operands.

``tests/test_gpu_parity_shapes.py::test_rounding_matched_oracle_config0`` uses the pair to prove that the ~2e-3
final-latent distance under CFG 7.5 is operand rounding and not a defect.

Rounding points (file:line of the kernel that rounds):
  weights                      -> fp16 once at pack time (anyedit_b200/unet.py _h / _pack_conv3); for heads with
                                  d % 16 == 8 the query weight is multiplied by d^-0.5 * log2(e) BEFORE rounding (unet.py:381-386)
  every GEMM / conv output     -> fp16 after bias + time-embedding row + activation + residual in fp32
                                  (csrc/gemm_wgmma.cu epilogue); the time-embedding linears and the output conv stay fp32
  GroupNorm(+SiLU) / LayerNorm -> fp32 statistics, fp16 output (csrc/norm.cu)
  attention                    -> fp32 scores, P rounded to fp16 before P.V, output fp16 (csrc/attention_wgmma.cu); the
                                  denominator is the sum of the unrounded fp32 P (with or without aux columns)
  GEGLU                        -> a * gelu(gate) in fp32, fp16 output
  timestep embedding, silu(emb)-> fp16 (csrc/elementwise.cu)
Reference structure: the same file:line map as oracle/unet_oracle.py.
"""
import math

import torch
import torch.nn.functional as F

from .unet_oracle import _count, timestep_embedding

LOG2E = 1.4426950408889634


# Precision-lever experiments (tests/experiments/precision_levers.py): which rounding points to drop.
#   "weights"   False = exact fp32 weights (what a hi + lo split-weight contraction, 2 passes, would give)
#   "residual"  False = the residual stream (outputs of every residual-add epilogue, conv / proj_in outputs feeding it) in fp32
#   "acts"      False = no activation rounding at all
POLICY = {"weights": True, "residual": True, "acts": True}


def r16(t):
    return t.to(torch.float16).to(torch.float32) if POLICY["acts"] else t


def rres(t):
    """Rounding of a residual-stream tensor."""
    return r16(t) if POLICY["residual"] else t


_W16 = {}


def _w(sd, k):
    """fp16-rounded weight, cached per (state dict, key): the pack happens once in the product too."""
    ck = (id(sd), k)
    t = _W16.get(ck)
    if t is None or t.shape != sd[k].shape:
        if len(_W16) > 4096:
            _W16.clear()
        t = _W16[ck] = sd[k].to(torch.float16).to(torch.float32) if POLICY["weights"] else sd[k]
    return t


def _wr(w):
    return w.to(torch.float16).to(torch.float32) if POLICY["weights"] else w


def _lin(x, w16, b=None):
    return F.linear(x, w16, b)


def _gn(x, w, b, eps, silu):
    h = F.group_norm(x, 32, w, b, eps)
    return r16(F.silu(h) if silu else h)


def _attn_core(q, k, v, heads, d, aux):
    """q, k, v: [B, n, heads*d] fp16-valued.  aux: q already carries d^-0.5 * log2(e)."""
    B, n, _ = q.shape

    def split(t):
        return t.reshape(B, t.shape[1], heads, d).permute(0, 2, 1, 3)

    qh, kh, vh = split(q), split(k), split(v)
    s = torch.matmul(qh, kh.transpose(-1, -2))                   # fp32 accumulate of fp16 products
    if not aux:
        s = s * (d ** -0.5 * LOG2E)
    s = s - s.amax(-1, keepdim=True)
    p = torch.exp2(s)
    p16 = r16(p)
    den = p.sum(-1, keepdim=True)
    o = torch.matmul(p16, vh) / den
    return r16(o.permute(0, 2, 1, 3).reshape(B, n, heads * d))


def _attention(sd, p, x, ctx, heads, residual):
    c = sd[p + "to_q.weight"].shape[0]
    d = c // heads
    aux = d % 16 == 8
    wq = sd[p + "to_q.weight"]
    wq = _wr(wq * (d ** -0.5 * LOG2E)) if aux else _wr(wq)
    src = x if ctx is None else ctx
    q = r16(_lin(x, wq))
    k = r16(_lin(src, _w(sd, p + "to_k.weight")))
    v = r16(_lin(src, _w(sd, p + "to_v.weight")))
    a = _attn_core(q, k, v, heads, d, aux)
    return rres(_lin(a, _w(sd, p + "to_out.0.weight"), sd[p + "to_out.0.bias"]) + residual)


def _block(sd, p, t, ctx, heads):
    c = t.shape[-1]
    ln = r16(F.layer_norm(t, (c,), sd[p + "norm1.weight"], sd[p + "norm1.bias"]))
    t2 = _attention(sd, p + "attn1.", ln, None, heads, t)
    ln2 = r16(F.layer_norm(t2, (c,), sd[p + "norm2.weight"], sd[p + "norm2.bias"]))
    t3 = _attention(sd, p + "attn2.", ln2, ctx, heads, t2)
    ln3 = r16(F.layer_norm(t3, (c,), sd[p + "norm3.weight"], sd[p + "norm3.bias"]))
    g = _lin(ln3, _w(sd, p + "ff.net.0.proj.weight"), sd[p + "ff.net.0.proj.bias"])
    a, gate = g.chunk(2, dim=-1)
    ffh = r16(a * F.gelu(gate))
    return rres(_lin(ffh, _w(sd, p + "ff.net.2.weight"), sd[p + "ff.net.2.bias"]) + t3)


def _spatial_transformer(sd, p, h, ctx, heads_of):
    b, c, hh, ww = h.shape
    g = _gn(h, sd[p + "norm.weight"], sd[p + "norm.bias"], 1e-6, False)
    tok = g.permute(0, 2, 3, 1).reshape(b, hh * ww, c)
    w_in = sd[p + "proj_in.weight"]
    t = rres(_lin(tok, _wr(w_in.reshape(w_in.shape[0], -1)), sd[p + "proj_in.bias"]))
    heads = heads_of(t.shape[-1])
    depth = 0
    while (p + f"transformer_blocks.{depth}.norm1.weight") in sd:
        cx = ctx[depth] if isinstance(ctx, (list, tuple)) else ctx
        t = _block(sd, p + f"transformer_blocks.{depth}.", t, cx, heads)
        depth += 1
    w_out = sd[p + "proj_out.weight"]
    res = h.permute(0, 2, 3, 1).reshape(b, hh * ww, c)
    o = rres(_lin(t, _wr(w_out.reshape(w_out.shape[0], -1)), sd[p + "proj_out.bias"]) + res)
    return o.reshape(b, hh, ww, c).permute(0, 3, 1, 2)


def _resblock(sd, p, x, emb_rows):
    a = _gn(x, sd[p + "in_layers.0.weight"], sd[p + "in_layers.0.bias"], 1e-5, True)
    h1 = r16(F.conv2d(a, _w(sd, p + "in_layers.2.weight"), sd[p + "in_layers.2.bias"], padding=1) + emb_rows[:, :, None, None])
    b = _gn(h1, sd[p + "out_layers.0.weight"], sd[p + "out_layers.0.bias"], 1e-5, True)
    if (p + "skip_connection.weight") in sd:
        w = sd[p + "skip_connection.weight"]
        res = rres(F.conv2d(x, _wr(w), sd[p + "skip_connection.bias"], padding=w.shape[-1] // 2))
    else:
        res = x
    return rres(F.conv2d(b, _w(sd, p + "out_layers.3.weight"), sd[p + "out_layers.3.bias"], padding=1) + res)


def _run_block(sd, p, h, semb, ctx, heads_of):
    j = 0
    while True:
        q = f"{p}{j}."
        if (q + "in_layers.0.weight") in sd:
            # emb_layers: Linear(SiLU(emb)) with the fp16 silu(emb) operand, fp32 result (one stacked GEMM in the product)
            rows = _lin(semb, _w(sd, q + "emb_layers.1.weight"), sd[q + "emb_layers.1.bias"])
            h = _resblock(sd, q, h, rows)
        elif (q + "transformer_blocks.0.norm1.weight") in sd:
            h = _spatial_transformer(sd, q, h, ctx, heads_of)
        elif (q + "op.weight") in sd:
            h = rres(F.conv2d(h, _w(sd, q + "op.weight"), sd[q + "op.bias"], stride=2, padding=1))
        elif (q + "conv.weight") in sd:
            h = F.interpolate(h, scale_factor=2, mode="nearest")
            h = rres(F.conv2d(h, _w(sd, q + "conv.weight"), sd[q + "conv.bias"], padding=1))
        else:
            break
        j += 1
    return h


def unet_forward(sd, x, timesteps, context=None, y=None, *, num_heads=-1, num_head_channels=-1):
    """Same signature as ``unet_oracle.unet_forward`` (no hooks / control)."""
    def heads_of(inner):
        return num_heads if num_head_channels == -1 else inner // num_head_channels

    mc = sd["time_embed.0.weight"].shape[1]
    temb = r16(timestep_embedding(timesteps, mc))
    e1 = r16(F.silu(_lin(temb, _w(sd, "time_embed.0.weight"), sd["time_embed.0.bias"])))
    emb = _lin(e1, _w(sd, "time_embed.2.weight"), sd["time_embed.2.bias"])            # fp32
    if "label_emb.weight" in sd:
        assert y is not None
        emb = emb + F.embedding(y, sd["label_emb.weight"])
    semb = r16(F.silu(emb))
    ctx = [r16(c) for c in context] if isinstance(context, (list, tuple)) else r16(context)

    n_in, n_out = _count(sd, "input_blocks"), _count(sd, "output_blocks")
    hs = []
    h = r16(x.float())
    for i in range(n_in):
        if i == 0:
            h = rres(F.conv2d(h, _w(sd, "input_blocks.0.0.weight"), sd["input_blocks.0.0.bias"], padding=1))
        else:
            h = _run_block(sd, f"input_blocks.{i}.", h, semb, ctx, heads_of)
        hs.append(h)
    h = _run_block(sd, "middle_block.", h, semb, ctx, heads_of)
    for i in range(n_out):
        h = torch.cat([h, hs.pop()], dim=1)
        h = _run_block(sd, f"output_blocks.{i}.", h, semb, ctx, heads_of)
    a = _gn(h, sd["out.0.weight"], sd["out.0.bias"], 1e-5, True)
    return F.conv2d(a, _w(sd, "out.2.weight"), sd["out.2.bias"], padding=1)           # eps stays fp32
