"""H100-native ``UNetModel`` -- drop-in for ``ldm.modules.diffusionmodules.openaimodel.UNetModel``.

Same constructor kwargs (openaimodel.py:442-472), same ``state_dict`` keys and shapes
(SURVEY.md 8b: 686 tensors for the SD-1.5 geometry) and the same call
``forward(x, timesteps, context, y) -> eps`` (openaimodel.py:754-786), so yaml ``target:``
strings, checkpoints and ``DDIMSampler`` keep working.  What differs is the execution: the
parameters are repacked once into kernel layouts (fp16, conv weights as [Cout, (ky,kx,ci)],
fused QKV / KV, interleaved GEGLU, all 22 ``emb_layers`` stacked into one matrix) and the
forward is a fixed sequence of hand-written sm_90a kernels on NHWC fp16 activations,
launched through the C ABI in ``include/anysd_b200.h``.  No eager-PyTorch math, no fallback.

Supported configuration = what the AnySD / SD-1.5 / anydoor.yaml geometries use:
``dims=2, use_spatial_transformer=True, conv_resample=True`` without ``use_scale_shift_norm``,
``resblock_updown`` or ``n_embed``; anything else raises ``NotImplementedError`` at construction.
"""
import math
import os

import torch
import torch.nn as nn

from . import ops


# ---- parameter holders (never called; they exist to own tensors under the reference's names) ---

class _Param(nn.Module):
    """weight (+bias) owner standing in for nn.Conv2d / nn.Linear / nn.GroupNorm / nn.LayerNorm."""

    def __init__(self, wshape, bias=True, kind="linear", zero=False):
        super().__init__()
        self.kind = kind
        self.weight = nn.Parameter(torch.empty(*wshape))
        if bias:
            self.bias = nn.Parameter(torch.empty(wshape[0]))
        else:
            self.register_parameter("bias", None)
        self.reset(zero)

    @torch.no_grad()
    def reset(self, zero=False):
        if self.kind == "norm":
            self.weight.fill_(1.0)
            self.bias.zero_()
            return
        if zero:                       # zero_module (util.py:177-183)
            self.weight.zero_()
            if self.bias is not None:
                self.bias.zero_()
            return
        fan_in = int(math.prod(self.weight.shape[1:]))
        bound = 1.0 / math.sqrt(fan_in)  # == kaiming_uniform(a=sqrt(5)), torch's conv/linear default
        self.weight.uniform_(-bound, bound)
        if self.bias is not None:
            self.bias.uniform_(-bound, bound)


class _Slot(nn.Module):
    """Parameter-free placeholder keeping nn.Sequential indices aligned with the reference
    (SiLU / Dropout / Identity positions)."""


def _seq(*mods):
    return nn.Sequential(*mods)


class _ResBlock(nn.Module):
    def __init__(self, ch, emb_ch, out_ch):
        super().__init__()
        self.channels, self.out_channels = ch, out_ch
        self.in_layers = _seq(_Param((ch,), kind="norm"), _Slot(), _Param((out_ch, ch, 3, 3), kind="conv"))
        self.emb_layers = _seq(_Slot(), _Param((out_ch, emb_ch)))
        self.out_layers = _seq(_Param((out_ch,), kind="norm"), _Slot(), _Slot(),
                               _Param((out_ch, out_ch, 3, 3), kind="conv", zero=True))
        if out_ch != ch:
            self.skip_connection = _Param((out_ch, ch, 1, 1), kind="conv")
        else:
            self.skip_connection = _Slot()


class _CrossAttention(nn.Module):
    def __init__(self, query_dim, context_dim, heads, dim_head):
        super().__init__()
        inner = heads * dim_head
        context_dim = query_dim if context_dim is None else context_dim
        self.heads, self.dim_head, self.context_dim = heads, dim_head, context_dim
        self.to_q = _Param((inner, query_dim), bias=False)
        self.to_k = _Param((inner, context_dim), bias=False)
        self.to_v = _Param((inner, context_dim), bias=False)
        self.to_out = _seq(_Param((query_dim, inner)), _Slot())


class _GEGLU(nn.Module):
    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.proj = _Param((dim_out * 2, dim_in))


class _FeedForward(nn.Module):
    def __init__(self, dim, mult=4):
        super().__init__()
        inner = int(dim * mult)
        self.net = _seq(_GEGLU(dim, inner), _Slot(), _Param((dim, inner)))


class _TransformerBlock(nn.Module):
    def __init__(self, dim, heads, d_head, context_dim, disable_self_attn):
        super().__init__()
        self.disable_self_attn = disable_self_attn
        self.attn1 = _CrossAttention(dim, context_dim if disable_self_attn else None, heads, d_head)
        self.ff = _FeedForward(dim)
        self.attn2 = _CrossAttention(dim, context_dim, heads, d_head)
        self.norm1 = _Param((dim,), kind="norm")
        self.norm2 = _Param((dim,), kind="norm")
        self.norm3 = _Param((dim,), kind="norm")


class _SpatialTransformer(nn.Module):
    def __init__(self, ch, heads, d_head, depth, context_dim, disable_self_attn, use_linear):
        super().__init__()
        if context_dim is not None and not isinstance(context_dim, (list, tuple)):
            context_dim = [context_dim] * depth if depth > 1 else [context_dim]
        inner = heads * d_head
        self.in_channels, self.inner, self.heads, self.d_head = ch, inner, heads, d_head
        self.use_linear = use_linear
        self.norm = _Param((ch,), kind="norm")
        self.proj_in = _Param((inner, ch) if use_linear else (inner, ch, 1, 1), kind="linear" if use_linear else "conv")
        self.transformer_blocks = nn.ModuleList(
            [_TransformerBlock(inner, heads, d_head, context_dim[d], disable_self_attn) for d in range(depth)])
        # attention.py:312-318 (note the Linear(in_channels, inner_dim) quirk, SURVEY.md B.12)
        self.proj_out = _Param((inner, ch) if use_linear else (ch, inner, 1, 1),
                               kind="linear" if use_linear else "conv", zero=True)


class _Downsample(nn.Module):
    def __init__(self, ch, out_ch):
        super().__init__()
        self.op = _Param((out_ch, ch, 3, 3), kind="conv")


class _Upsample(nn.Module):
    def __init__(self, ch, out_ch):
        super().__init__()
        self.conv = _Param((out_ch, ch, 3, 3), kind="conv")


class _Embedding(nn.Module):
    def __init__(self, n, d):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(n, d))


# ---- packed (kernel-layout) weights -------------------------------------------------------------

# LayerNorm folded into the contractions either side of it (row moments from the producer's epilogue, gamma / beta folded into the
# consumer's weights: anysd_gemm_params::row_stats / ln_stats).  OFF by default: the consumers are
# epilogue-bound contractions (K = 320 .. 1280) and the two extra FMAs + the column-sum operand per accumulator can cost them
# more than the layernorm launch they replace; ANYSD_LN_FOLD=1 switches it on.
_LN_FOLD = os.environ.get("ANYSD_LN_FOLD", "0")[:1] == "1"


FF_FUSED_C = 320                # channel width of the transformer blocks whose feed-forward runs as one kernel (ops.geglu_ff)
XATTN_MAX_CTX = 80              # longest context the fused cross-attention block (ops.xattn_block) keeps on chip


def ff1_chunk_order(hidden, chunk=32):
    """Row order of the fused feed-forward's ff1 pack (feedforward_wgmma.cu), as indices into the interleaved (a_j, gate_j)
    pack: within each chunk of ``chunk`` outputs, packed pair P (rows 2P, 2P + 1) holds hidden unit
    16 (i // 4) + (2q, 2q + 1, 2q + 8, 2q + 9)[i % 4] with i = P // 4, q = P % 4 -- the unit whose GEGLU value the kernel
    needs at that accumulator position as the register A operand of the second product.  Each (a, gate) pair stays together."""
    idx = []
    for c in range(hidden // chunk):
        for P in range(chunk):
            i, q = divmod(P, 4)
            u = c * chunk + 16 * (i // 4) + (2 * q, 2 * q + 1, 2 * q + 8, 2 * q + 9)[i % 4]
            idx += [2 * u, 2 * u + 1]
    return torch.tensor(idx, dtype=torch.long)


def _h(t, dev):
    return t.detach().to(device=dev, dtype=torch.float16).contiguous()


def _f(t, dev):
    return t.detach().to(device=dev, dtype=torch.float32).contiguous()


def head_stride_for(d):
    """Head stride of packed q/k/v projections: d, or ceil16(d) when d is not a multiple of 16 -- the wgmma
    attention kernel contracts over ceil16(d) columns and needs the extra ones to be exact zeros (d = 40 -> 48)."""
    return d if d % 16 == 0 else (d + 15) // 16 * 16


def pad_heads(w, heads, d, hs):
    """[heads*d, K] projection weight -> [heads*hs, K] with (hs - d) zero rows appended to every head."""
    if hs == d:
        return w
    k = w.shape[1]
    out = w.new_zeros(heads, hs, k)
    out[:, :d] = w.reshape(heads, d, k)
    return out.reshape(heads * hs, k)


LOG2E = 1.4426950408889634


def aux_cols_for(d):
    """True when the attention operands can carry the softmax bookkeeping (anysd_attn_params::aux_cols): the padded
    head has at least two spare columns inside the kernel's ceil16(d) contraction extent (d = 40 -> 48)."""
    return d % 16 == 8


def aux_bias(heads, d, hs, ones):
    """fp32 [heads*hs] projection bias that plants 1.0 in the first `ones` padding columns of every head
    (to_q/to_k/to_v have no bias of their own, attention.py:152-154)."""
    b = torch.zeros(heads, hs, dtype=torch.float32)
    b[:, d:d + ones] = 1.0
    return b.reshape(-1)


def _pack_conv3(w, dev, cin_pad=None):
    """OIHW -> [Cout, 9*Cin_pad] fp16 with K order (ky, kx, ci)."""
    co, ci = w.shape[0], w.shape[1]
    cp = cin_pad or ci
    w = w.detach().to(dev).float().permute(0, 2, 3, 1)            # [co, 3, 3, ci]
    if cp != ci:
        w = torch.nn.functional.pad(w, (0, cp - ci))
    return w.reshape(co, 9 * cp).to(torch.float16).contiguous()


class UNetModel(nn.Module):
    """See module docstring.  Reference: openaimodel.py:412-786."""

    def __init__(self, image_size, in_channels, model_channels, out_channels, num_res_blocks,
                 attention_resolutions, dropout=0, channel_mult=(1, 2, 4, 8), conv_resample=True, dims=2,
                 num_classes=None, use_checkpoint=False, use_fp16=False, num_heads=-1, num_head_channels=-1,
                 num_heads_upsample=-1, use_scale_shift_norm=False, resblock_updown=False,
                 use_new_attention_order=False, use_spatial_transformer=False, transformer_depth=1,
                 context_dim=None, n_embed=None, legacy=True, disable_self_attentions=None,
                 num_attention_blocks=None, disable_middle_self_attn=False, use_linear_in_transformer=False,
                 _encoder_only=False):
        super().__init__()
        self._encoder_only = _encoder_only       # ControlNet (cldm.py:47-304): input blocks + middle block only
        if use_spatial_transformer:
            assert context_dim is not None, "use_spatial_transformer needs context_dim (cross-attention conditioning)"
        if context_dim is not None:
            assert use_spatial_transformer, "context_dim needs use_spatial_transformer=True"
            if not isinstance(context_dim, int):
                context_dim = list(context_dim)
        if num_heads_upsample == -1:
            num_heads_upsample = num_heads
        if num_heads == -1:
            assert num_head_channels != -1, "Either num_heads or num_head_channels has to be set"
        if num_head_channels == -1:
            assert num_heads != -1, "Either num_heads or num_head_channels has to be set"
        unsupported = []
        if dims != 2: unsupported.append("dims != 2")
        if not use_spatial_transformer: unsupported.append("use_spatial_transformer=False (AttentionBlock)")
        if use_scale_shift_norm: unsupported.append("use_scale_shift_norm")
        if resblock_updown: unsupported.append("resblock_updown")
        if not conv_resample: unsupported.append("conv_resample=False")
        if n_embed is not None: unsupported.append("n_embed")
        if num_classes is not None and not isinstance(num_classes, int): unsupported.append(f"num_classes={num_classes!r}")
        if dropout: unsupported.append("dropout > 0 (inference path)")
        if unsupported:
            raise NotImplementedError("anyedit_b200.UNetModel does not implement: " + ", ".join(unsupported))

        self.image_size, self.in_channels, self.model_channels = image_size, in_channels, model_channels
        self.out_channels = out_channels
        if isinstance(num_res_blocks, int):
            self.num_res_blocks = len(channel_mult) * [num_res_blocks]
        else:
            if len(num_res_blocks) != len(channel_mult):
                raise ValueError("provide num_res_blocks either as an int (globally constant) or "
                                 "as a list/tuple (per-level) with the same length as channel_mult")
            self.num_res_blocks = list(num_res_blocks)
        if disable_self_attentions is not None:
            assert len(disable_self_attentions) == len(channel_mult)
        if num_attention_blocks is not None:
            assert len(num_attention_blocks) == len(self.num_res_blocks)
            assert all(self.num_res_blocks[i] >= num_attention_blocks[i] for i in range(len(num_attention_blocks)))
        self.attention_resolutions = attention_resolutions
        self.dropout, self.channel_mult, self.conv_resample = dropout, channel_mult, conv_resample
        self.num_classes, self.use_checkpoint = num_classes, use_checkpoint
        self.dtype = torch.float16 if use_fp16 else torch.float32
        self.num_heads, self.num_head_channels, self.num_heads_upsample = num_heads, num_head_channels, num_heads_upsample
        self.predict_codebook_ids = False
        self.context_dim = context_dim

        D = model_channels * 4
        self.time_embed_dim = D
        self.time_embed = _seq(_Param((D, model_channels)), _Slot(), _Param((D, D)))
        if num_classes is not None:
            self.label_emb = _Embedding(num_classes, D)

        def heads_for(ch, nh):
            if num_head_channels == -1:
                return nh, ch // nh
            return ch // num_head_channels, num_head_channels

        def transformer(ch, nh, level, middle=False):
            h, d = heads_for(ch, nh)
            if middle:
                dsa = disable_middle_self_attn
            else:
                dsa = disable_self_attentions[level] if disable_self_attentions is not None else False
            return _SpatialTransformer(ch, h, d, transformer_depth, context_dim, dsa, use_linear_in_transformer)

        self.input_blocks = nn.ModuleList([_seq(_Param((model_channels, in_channels, 3, 3), kind="conv"))])
        chans = [model_channels]
        ch, ds = model_channels, 1
        for level, mult in enumerate(channel_mult):
            for nr in range(self.num_res_blocks[level]):
                layers = [_ResBlock(ch, D, mult * model_channels)]
                ch = mult * model_channels
                if ds in attention_resolutions:
                    if num_attention_blocks is None or nr < num_attention_blocks[level]:
                        layers.append(transformer(ch, num_heads, level))
                self.input_blocks.append(_seq(*layers))
                chans.append(ch)
            if level != len(channel_mult) - 1:
                self.input_blocks.append(_seq(_Downsample(ch, ch)))
                chans.append(ch)
                ds *= 2
        self.middle_block = _seq(_ResBlock(ch, D, ch), transformer(ch, num_heads, 0, middle=True), _ResBlock(ch, D, ch))
        self.output_blocks = nn.ModuleList([])
        for level, mult in ([] if _encoder_only else list(enumerate(channel_mult))[::-1]):
            for i in range(self.num_res_blocks[level] + 1):
                ich = chans.pop()
                layers = [_ResBlock(ch + ich, D, model_channels * mult)]
                ch = model_channels * mult
                if ds in attention_resolutions:
                    if num_attention_blocks is None or i < num_attention_blocks[level]:
                        layers.append(transformer(ch, num_heads, level))  # ST takes num_heads (openaimodel.py:703-706)
                if level and i == self.num_res_blocks[level]:
                    layers.append(_Upsample(ch, ch))
                    ds //= 2
                self.output_blocks.append(_seq(*layers))
        if _encoder_only:
            del self.output_blocks
        else:
            self.out = _seq(_Param((ch,), kind="norm"), _Slot(), _Param((out_channels, model_channels, 3, 3), kind="conv", zero=True))

        self._pack = None
        self._pack_key = None
        self._epoch = 0                  # bumped by invalidate(): part of the pack key and of LatentDenoiser.graph_key

    # the reference's no-op stubs (openaimodel.py:738-752)
    def convert_to_fp16(self):
        pass

    def convert_to_fp32(self):
        pass

    # ---- weight repack --------------------------------------------------------------------------
    def _param_key(self):
        dev = None
        ver = 0
        for p in self.parameters():
            ver += p._version
            dev = p.device
        return (str(dev), ver, self._epoch)

    def invalidate(self):
        """Call after an in-place weight change that does not bump parameter versions (a ``.data`` write, a raw-pointer
        kernel): drops the packed weights and makes every sampler re-capture its CUDA graphs."""
        self._pack = None
        self._epoch += 1

    def prepare(self):
        """Repack parameters into kernel layouts on their device (done lazily, redone when any
        parameter changes in place or moves)."""
        key = self._param_key()
        if self._pack is not None and self._pack_key == key:
            return self._pack
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("anyedit_b200.UNetModel runs on CUDA only (no CPU fallback); call .cuda() first")
        P = {}
        te = self.time_embed
        P["te0_w"], P["te0_b"] = _h(te[0].weight, dev), _f(te[0].bias, dev)
        P["te2_w"], P["te2_b"] = _h(te[2].weight, dev), _f(te[2].bias, dev)
        if self.num_classes is not None:
            P["label"] = _f(self.label_emb.weight, dev)
        # input channels padded to 64 (zeros) so that the input conv runs on the wgmma implicit-GEMM kernel
        # (64-channel k-blocks); the extra MACs are on zero weights
        self._cin_pad = (self.in_channels + 63) // 64 * 64
        P["in_w"] = _pack_conv3(self.input_blocks[0][0].weight, dev, self._cin_pad)
        P["in_b"] = _f(self.input_blocks[0][0].bias, dev)
        emb_w, emb_b, off = [], [], 0

        def pack_res(rb):
            nonlocal off
            d = {"cin": rb.channels, "cout": rb.out_channels, "_mod": rb}     # _mod: source module (training.py packs dX weights from it)
            d["gn1_w"], d["gn1_b"] = _f(rb.in_layers[0].weight, dev), _f(rb.in_layers[0].bias, dev)
            d["c1_w"], d["c1_b"] = _pack_conv3(rb.in_layers[2].weight, dev), _f(rb.in_layers[2].bias, dev)
            emb_w.append(rb.emb_layers[1].weight)
            emb_b.append(rb.emb_layers[1].bias)
            d["emb_off"] = off
            off += rb.out_channels
            d["gn2_w"], d["gn2_b"] = _f(rb.out_layers[0].weight, dev), _f(rb.out_layers[0].bias, dev)
            d["c2_w"], d["c2_b"] = _pack_conv3(rb.out_layers[3].weight, dev), _f(rb.out_layers[3].bias, dev)
            if isinstance(rb.skip_connection, _Param):
                w = rb.skip_connection.weight
                d["skip_w"] = _h(w.reshape(w.shape[0], -1), dev)
                d["skip_b"] = _f(rb.skip_connection.bias, dev)
            return d

        def pack_attn(at, self_attn):
            hs = head_stride_for(at.dim_head)
            aux = aux_cols_for(at.dim_head)
            d = {"heads": at.heads, "d": at.dim_head, "hs": hs, "aux": aux, "qkv_b": None, "kv_b": None, "_mod": at}
            ph = lambda w: pad_heads(w.detach(), at.heads, at.dim_head, hs)
            wq = at.to_q.weight.detach()
            if aux:
                # softmax scale and log2(e) folded into Wq; K gets 1.0 in two padding columns, V in one: the kernel
                # keeps its running reference in q's padding and reads the denominator from column d of P.V
                wq = wq.float() * (at.dim_head ** -0.5 * LOG2E)
                ab = lambda n: aux_bias(at.heads, at.dim_head, hs, n)
                d["qkv_b"] = torch.cat([ab(0), ab(2), ab(1)]).to(dev)
                d["kv_b"] = torch.cat([ab(2), ab(1)]).to(dev)
            if self_attn:
                d["qkv_w"] = _h(torch.cat([ph(wq).float(), ph(at.to_k.weight).float(), ph(at.to_v.weight).float()], 0), dev)
            else:
                d["q_w"] = _h(ph(wq), dev)
                d["kv_w"] = _h(torch.cat([ph(at.to_k.weight), ph(at.to_v.weight)], 0), dev)
            d["o_w"], d["o_b"] = _h(at.to_out[0].weight, dev), _f(at.to_out[0].bias, dev)
            return d

        def pack_st(st):
            d = {"ch": st.in_channels, "inner": st.inner, "_mod": st}
            d["gn_w"], d["gn_b"] = _f(st.norm.weight, dev), _f(st.norm.bias, dev)
            d["pin_w"] = _h(st.proj_in.weight.reshape(st.proj_in.weight.shape[0], -1), dev)
            d["pin_b"] = _f(st.proj_in.bias, dev)
            d["pout_w"] = _h(st.proj_out.weight.reshape(st.proj_out.weight.shape[0], -1), dev)
            d["pout_b"] = _f(st.proj_out.bias, dev)
            d["blocks"] = []
            for tb in st.transformer_blocks:
                b = {"attn1": pack_attn(tb.attn1, not tb.disable_self_attn), "attn2": pack_attn(tb.attn2, False),
                     "self": not tb.disable_self_attn, "_mod": tb}
                for i, nm in enumerate((tb.norm1, tb.norm2, tb.norm3), 1):
                    b[f"ln{i}_w"], b[f"ln{i}_b"] = _f(nm.weight, dev), _f(nm.bias, dev)
                gw, gb = tb.ff.net[0].proj.weight, tb.ff.net[0].proj.bias
                inner = gw.shape[0] // 2
                # interleave (a_j, gate_j) rows so the GEGLU pair sits in adjacent accumulator columns
                b["ff1_w"] = _h(torch.stack([gw[:inner], gw[inner:]], 1).reshape(2 * inner, -1), dev)
                b["ff1_b"] = _f(torch.stack([gb[:inner], gb[inner:]], 1).reshape(-1), dev)
                b["ff2_w"], b["ff2_b"] = _h(tb.ff.net[2].weight, dev), _f(tb.ff.net[2].bias, dev)
                if st.inner == FF_FUSED_C and inner == 4 * FF_FUSED_C:
                    # the fused feed-forward's packs: ff1 rows in the kernel's chunk order, W2 transposed (hidden-major)
                    perm = ff1_chunk_order(inner).to(dev)
                    b["ff1p_w"], b["ff1p_b"] = b["ff1_w"][perm].contiguous(), b["ff1_b"][perm].contiguous()
                    b["ff2t_w"] = b["ff2_w"].t().contiguous()
                d["blocks"].append(b)
            return d

        def pack_block(seq):
            out = []
            for m in seq:
                if isinstance(m, _ResBlock):
                    out.append(("res", pack_res(m)))
                elif isinstance(m, _SpatialTransformer):
                    out.append(("st", pack_st(m)))
                elif isinstance(m, _Downsample):
                    out.append(("down", {"w": _pack_conv3(m.op.weight, dev), "b": _f(m.op.bias, dev), "_mod": m}))
                elif isinstance(m, _Upsample):
                    out.append(("up", {"w": _pack_conv3(m.conv.weight, dev), "b": _f(m.conv.bias, dev), "_mod": m}))
            return out

        P["input"] = [pack_block(b) for b in list(self.input_blocks)[1:]]
        P["middle"] = pack_block(self.middle_block)
        P["output"] = [] if self._encoder_only else [pack_block(b) for b in self.output_blocks]
        P["emb_w"] = _h(torch.cat(emb_w, 0), dev)                 # all ResBlock emb_layers stacked: one GEMM
        P["emb_b"] = _f(torch.cat(emb_b, 0), dev)
        P["emb_total"] = off
        if self._encoder_only:
            self._pack_extra(P, dev)
            self._pack, self._pack_key = P, key
            return P
        P["out_gn_w"], P["out_gn_b"] = _f(self.out[0].weight, dev), _f(self.out[0].bias, dev)
        # output conv: rows padded to a multiple of 8 (zero filters) -> wgmma kernel with fp32 output
        self._cout_pad = (self.out_channels + 7) // 8 * 8
        ow = _pack_conv3(self.out[2].weight, dev)
        ob = _f(self.out[2].bias, dev)
        if self._cout_pad != self.out_channels:
            ow = torch.cat([ow, ow.new_zeros(self._cout_pad - self.out_channels, ow.shape[1])], 0).contiguous()
            ob = torch.cat([ob, ob.new_zeros(self._cout_pad - self.out_channels)], 0).contiguous()
        P["out_w"], P["out_b"] = ow, ob
        self._pack, self._pack_key = P, key
        return P

    # ---- forward ----------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, x, timesteps=None, context=None, y=None, control=None, only_mid_control=False,
                anysd=None, **kwargs):
        """eps = UNet(x, t, context, y)  (openaimodel.py:754-786).

        ``control`` / ``only_mid_control``: the 13 additive residuals of ``ControlledUnetModel.forward``
        (AnyEdit_Collection/other_modules/cldm/cldm.py:22-44), NCHW tensors.
        ``anysd``: internal hook used by ``anyedit_b200.anysd.MoE`` (task embedding + expert stream).
        """
        assert (y is not None) == (self.num_classes is not None), \
            "must specify y if and only if the model is class-conditional"
        ctrl_nhwc = bool(getattr(control, "nhwc", False))        # anyedit_b200.cldm.ControlNet hands NHWC fp16 residuals over
        if control is not None:
            control = list(control) if ctrl_nhwc else [c if c.dtype in (torch.float32, torch.float16) else c.float() for c in control]
        add_control = (lambda c, t: ops.add_(t, c)) if ctrl_nhwc else (lambda c, t: ops.add_nchw_into_nhwc(c.contiguous(), t))
        P = self.prepare()
        dev = x.device
        if dev.type != "cuda":
            raise RuntimeError("anyedit_b200.UNetModel: input must be a CUDA tensor (no CPU fallback)")
        N, Cin, H, W = x.shape
        assert Cin == self.in_channels, f"expected {self.in_channels} input channels, got {Cin}"
        if y is not None:
            assert y.shape[0] == N
        f16 = dict(dtype=torch.float16, device=dev)
        f32 = dict(dtype=torch.float32, device=dev)
        ws = ops.groupnorm_workspace(N, 32, 0, dev)

        mc = self.model_channels
        emb_all = self._embeddings(P, N, timesteps, y, anysd, dev)
        ctx16 = self._context16(context, N, dev)
        st = {"N": N, "ws": ws, "emb_all": emb_all, "ctx": ctx16, "anysd": anysd, "layer": 0, "xl": 0,
              "kvc": getattr(self, "_ctx_kv", None)}

        # -- input conv --
        # Shared CFG halves (set by the DDIM stepper when x, c_concat, t and y of the uncond / cond halves are
        # identical, ddim.py:190-210): only the cross-attention context differs, so everything before the first
        # cross-attention K/V is computed for one half and duplicated -- bit-identical (every kernel is
        # batch-independent), ~3 % of a forward at the SD-1.5 geometry (the first self-attention is the big part).
        # (with the AnySD hook the stepper has checked that the two halves carry the same edit codes: the task-embedding add
        # is then identical too; the visual tokens only enter at the cross-attention, after the shared prefix)
        share = bool(getattr(self, "_shared_halves", False)) and N % 2 == 0 and y is None and control is None
        Nx = N // 2 if share else N
        xin = torch.zeros(Nx, H, W, self._cin_pad, **f16) if self._cin_pad != Cin else torch.empty(Nx, H, W, Cin, **f16)
        ops.nchw_to_nhwc(x[:Nx].contiguous(), xin, 0)
        h = torch.empty(Nx, H, W, mc, **f16)
        # every contraction whose output feeds a GroupNorm also emits that norm's statistics from its epilogue (h._gn)
        h._gn = ops.conv3x3(xin, P["in_w"], h.view(-1, mc), bias=P["in_b"], logical_cin=Cin, stats=True)
        hs = [self._dup_rows(h) if share else h]
        for blk in P["input"]:
            if share:
                has_st = any(kind == "st" for kind, _ in blk)
                h = self._run(blk, h, None, st, share=has_st)
                if has_st:
                    share = False
                    hs.append(h)
                else:
                    hs.append(self._dup_rows(h))
            else:
                h = self._run(blk, h, None, st)
                hs.append(h)
        if share:                                                 # no attention anywhere in the encoder
            h = self._dup_rows(h)
        h = self._run(P["middle"], h, None, st)
        if control is not None:                                   # cldm.py:33-34
            add_control(control.pop(), h)
            h._gn = None                                          # changed in place: its epilogue statistics are stale
        for blk in P["output"]:
            skip = hs.pop()
            if control is not None and not only_mid_control:      # cldm.py:36-41
                add_control(control.pop(), skip)
                skip._gn = None
            h = self._run(blk, h, skip, st)
        # -- head: GN -> SiLU -> conv3x3 (fp32 out), back to NCHW in x.dtype --
        Nn, Hh, Ww, C = h.shape
        a = torch.empty_like(h)
        ops.groupnorm(h, P["out_gn_w"], P["out_gn_b"], a, N, Hh * Ww, 1e-5, True, ws, stats=getattr(h, "_gn", None))
        o = torch.empty(N, Hh, Ww, self._cout_pad, **f32)
        ops.conv3x3(a, P["out_w"], o.view(-1, self._cout_pad), bias=P["out_b"], logical_cout=self.out_channels)
        out_dtype = x.dtype if x.dtype in (torch.float32, torch.float16) else torch.float32
        out = torch.empty(N, self.out_channels, Hh, Ww, dtype=out_dtype, device=dev)
        ops.nhwc_to_nchw(o, out)
        return out.to(x.dtype)

    def _embeddings(self, P, N, timesteps, y, anysd, dev):
        """time / class / task embedding (openaimodel.py:767-772) -> the stacked ResBlock ``emb_layers`` rows [N, sum Cout] fp32."""
        f16, f32 = dict(dtype=torch.float16, device=dev), dict(dtype=torch.float32, device=dev)
        D, mc = self.time_embed_dim, self.model_channels
        temb = torch.empty(N, mc, **f16)
        ops.timestep_embedding(timesteps.to(dev), temb)
        e1 = torch.empty(N, D, **f16)
        ops.gemm(temb, P["te0_w"], e1, bias=P["te0_b"], act=1)
        emb_lin = torch.empty(N, D, **f32)
        ops.gemm(e1, P["te2_w"], emb_lin, bias=P["te2_b"])
        semb = torch.empty(N, D, **f16)
        table, idx = None, None
        if self.num_classes is not None:
            table, idx = P["label"], y.to(device=dev, dtype=torch.int64).contiguous()
        elif anysd is not None and anysd.get("task_table") is not None:
            table, idx = anysd["task_table"], anysd["edit_code"]
        ops.emb_finalize(emb_lin, semb, table, idx)
        emb_all = torch.empty(N, P["emb_total"], **f32)
        ops.gemm(semb, P["emb_w"], emb_all, bias=P["emb_b"])
        return emb_all

    @staticmethod
    def _context16(context, N, dev):
        """context (list = one tensor per transformer depth, attention.py:323-324) as fp16."""
        ctx_list = context if isinstance(context, (list, tuple)) else [context]
        ctx16 = []
        for c in ctx_list:
            if c is None:
                ctx16.append(None)
                continue
            assert c.shape[0] == N, "context batch must match x"
            c = c.to(dev)
            if c.dtype == torch.float16 and c.is_contiguous():
                ctx16.append(c)
            else:
                c32 = c.float().contiguous()
                t = torch.empty(c32.shape, dtype=torch.float16, device=dev)
                ops.cast_f16(c32, t)
                ctx16.append(t)
        return ctx16

    # ---- block executors ----------------------------------------------------------------------------
    def _run(self, blk, h, skip, st, share=False):
        """``share``: h is one CFG half (see _transformer); the first SpatialTransformer of the block widens it."""
        for kind, d in blk:
            if kind == "res":
                h = self._resblock(d, h, skip, st)
                skip = None
            elif kind == "st":
                h = self._transformer(d, h, st, share=share)
                share = False
            elif kind == "down":
                N, H, W, C = h.shape
                o = torch.empty(N, (H - 1) // 2 + 1, (W - 1) // 2 + 1, d["w"].shape[0], dtype=h.dtype, device=h.device)
                o._gn = ops.conv3x3(h, d["w"], o.view(-1, o.shape[-1]), bias=d["b"], stride=2, stats=True)
                h = o
            elif kind == "up":
                N, H, W, C = h.shape
                o = torch.empty(N, 2 * H, 2 * W, d["w"].shape[0], dtype=h.dtype, device=h.device)
                o._gn = ops.conv3x3(h, d["w"], o.view(-1, o.shape[-1]), bias=d["b"], upsample=1, stats=True)
                h = o
        return h

    def _resblock(self, d, h, skip, st):
        """openaimodel.py:254-274.  ``skip`` (if given) is concatenated after ``h`` (:780)."""
        N, H, W, C1 = h.shape
        HW = H * W
        cin, cout = d["cin"], d["cout"]
        if skip is not None:
            x = torch.empty(N, H, W, cin, dtype=h.dtype, device=h.device)
            ops.concat_channels(h, skip, x)
            ga, gb = getattr(h, "_gn", None), getattr(skip, "_gn", None)     # statistics of a concat = its parts' statistics
            x._gn = ops.GnStats(ga.parts + gb.parts, ga.S) if (ga is not None and gb is not None and ga.S == gb.S) else None
        else:
            x = h
        assert x.shape[-1] == cin
        a = torch.empty_like(x)
        ops.groupnorm(x, d["gn1_w"], d["gn1_b"], a, N, HW, 1e-5, True, st["ws"], stats=getattr(x, "_gn", None))
        h1 = torch.empty(N, H, W, cout, dtype=h.dtype, device=h.device)
        emb = st["emb_all"]
        g1 = ops.conv3x3(a, d["c1_w"], h1.view(-1, cout), bias=d["c1_b"], rowadd=emb[:, d["emb_off"]:], ld_rowadd=emb.stride(0),
                         stats=True)
        b = torch.empty_like(h1)
        ops.groupnorm(h1, d["gn2_w"], d["gn2_b"], b, N, HW, 1e-5, True, st["ws"], stats=g1)
        if "skip_w" in d:
            res = torch.empty(N * HW, cout, dtype=h.dtype, device=h.device)
            ops.gemm(x.view(-1, cin), d["skip_w"], res, bias=d["skip_b"])
        else:
            res = x.view(-1, cin)
        out = torch.empty(N, H, W, cout, dtype=h.dtype, device=h.device)
        out._gn = ops.conv3x3(b, d["c2_w"], out.view(-1, cout), bias=d["c2_b"], residual=res, stats=True)
        return out

    def _attn(self, ad, xq, ctx, N, n_q, st, self_attn, residual, out, expert=False, q_pre=None, ln=None, out_stats=False):
        """CrossAttention.forward (attention.py:163-194) + residual add of the caller (:272-273).
        ``q_pre``: the query projection computed by the caller (shared CFG halves), ``xq`` is then unused.
        ``ln`` = (row moments of xq, folded pack): xq is the UN-normalised input of the block's LayerNorm, which is folded into
        the query (/ fused q|k|v) projection; ``out_stats``: the output projection leaves ``out._ln`` for the next LayerNorm."""
        C = ad["heads"] * ad["d"]
        hs = ad["hs"]
        Cp = ad["heads"] * hs                     # projection width with padded heads (== C unless d % 16 != 0)
        dev = residual.device
        a = torch.empty(N * n_q, C, dtype=torch.float16, device=dev)
        if self_attn:
            qkv = torch.empty(N * n_q, 3 * Cp, dtype=torch.float16, device=dev)
            if ln is not None:
                ops.gemm(xq, ln[1]["w"], qkv, bias=ln[1]["b"], ln=(ln[0], ln[1]["cs"], 1e-5))
            else:
                ops.gemm(xq, ad["qkv_w"], qkv, bias=ad["qkv_b"])
            ops.attention(qkv, qkv[:, Cp:], qkv[:, 2 * Cp:], a, N, ad["heads"], n_q, n_q, ad["d"],
                          3 * Cp, 3 * Cp, 3 * Cp, C, head_stride=hs, aux_cols=ad["aux"])
        else:
            L = ctx.shape[1]
            if q_pre is not None:
                q = q_pre
            else:
                q = torch.empty(N * n_q, Cp, dtype=torch.float16, device=dev)
                if ln is not None:
                    ops.gemm(xq, ln[1]["w"], q, bias=ln[1]["b"], ln=(ln[0], ln[1]["cs"], 1e-5))
                else:
                    ops.gemm(xq, ad["q_w"], q)
            kv = self._context_kv(ad, ctx, N, st)
            ops.attention(q, kv, kv[:, Cp:], a, N, ad["heads"], n_q, L, ad["d"], Cp, 2 * Cp, 2 * Cp, C, head_stride=hs,
                          aux_cols=ad["aux"])
            if expert and st["anysd"] is not None and st["anysd"].get("experts") is not None:
                st["anysd"]["experts"](st["layer"], q, a, N, n_q, ad["heads"], ad["d"], hs, ad["aux"])
            if expert:
                st["layer"] += 1
        if out is None:
            return a
        if out_stats:
            out._ln = ops.row_stats_buffer(N * n_q, C, dev)
        ops.gemm(a, ad["o_w"], out, bias=ad["o_b"], residual=residual, row_stats=out._ln if out_stats else None)

    @staticmethod
    def _context_kv(ad, ctx, N, st):
        """The cross-attention's context K/V [N * L, 2 Cp]: constant over the steps of one sampling run, so the DDIM stepper
        keeps them (st["kvc"]: mode "fill" computes into persistent buffers, mode "use" skips the projection)."""
        L, Cp = ctx.shape[1], ad["heads"] * ad["hs"]
        kvc, xl = st.get("kvc"), st.get("xl", 0)
        if kvc is not None and kvc["mode"] == "use":
            kv = kvc["bufs"][xl]
        else:
            have = kvc is not None and len(kvc["bufs"]) > xl
            kv = kvc["bufs"][xl] if have else torch.empty(N * L, 2 * Cp, dtype=torch.float16, device=ctx.device)
            ops.gemm(ctx.view(N * L, -1), ad["kv_w"], kv, bias=ad["kv_b"])
            if kvc is not None and not have:
                kvc["bufs"].append(kv)
        st["xl"] = xl + 1
        return kv

    @staticmethod
    def _xattn_fused(b, ctx, n, st):
        """True when the span from attn1's output projection to norm3 runs as one kernel (ops.xattn_block): 320 channels as
        8 aux_cols heads of 40, a self-attention attn1, whole 128-row tiles per image, a context of at most 80 tokens, and
        no expert stream adding into the cross-attention output before its projection."""
        a2 = b["attn2"]
        experts = st["anysd"] is not None and st["anysd"].get("experts") is not None
        return ("ff1p_w" in b and b["self"] and not experts and ctx is not None and ctx.shape[1] <= XATTN_MAX_CTX
                and n % 128 == 0 and a2["aux"] and (a2["heads"], a2["d"], a2["hs"]) == (8, 40, 48))

    @staticmethod
    def _ln_folded(b):
        """The three LayerNorms of a BasicTransformerBlock (attention.py:262-264) folded into the projections that consume them:
        W' = W diag(gamma) (fp16), colsum_n = sum_k W'[n, k] (of the fp16 values: the mean term then cancels exactly against the
        accumulator), bias' = b + W beta.  Built on first use from the kernel-layout packs, dropped with them."""
        fb = b.get("_fold")
        if fb is None:
            def fold(w16, bias, gamma, beta):
                w32 = w16.float()
                wf = (w32 * gamma[None, :]).to(torch.float16).contiguous()
                bb = w32 @ beta
                if bias is not None:
                    bb = bb + bias
                return {"w": wf, "cs": wf.float().sum(1).contiguous(), "b": bb.contiguous()}
            a1 = b["attn1"]
            fb = {"a1": fold(a1["qkv_w"], a1["qkv_b"], b["ln1_w"], b["ln1_b"]) if b["self"] else fold(a1["q_w"], None, b["ln1_w"], b["ln1_b"]),
                  "a2": fold(b["attn2"]["q_w"], None, b["ln2_w"], b["ln2_b"]),
                  "ff1": fold(b["ff1_w"], b["ff1_b"], b["ln3_w"], b["ln3_b"])}
            b["_fold"] = fb
        return fb

    @staticmethod
    def _dup_rows(t):
        """[rows, ...] -> [2*rows, ...]: both CFG halves get the same values (two device-to-device copies)."""
        out = torch.empty((2 * t.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
        out[: t.shape[0]].copy_(t)
        out[t.shape[0]:].copy_(t)
        g = getattr(t, "_gn", None)
        if g is not None:                                       # per-image epilogue statistics travel with the images
            n = t.shape[0]
            out._gn = ops.GnStats([(torch.cat([b[:n], b[:n]]), c) for b, c in g.parts], g.S)
        r = getattr(t, "_ln", None)
        if r is not None:                                       # per-row moments [slabs, rows, 2] likewise
            out._ln = torch.cat([r, r], 1).contiguous()
        return out

    def _transformer(self, d, h, st, share=False):
        """SpatialTransformer.forward (attention.py:321-340); NHWC makes both rearranges free.
        ``share``: ``h`` holds ONE half of a CFG batch whose two halves are identical up to here; everything before
        the first cross-attention's K/V (GroupNorm, proj_in, LN1, self-attention, LN2, the query projection) is
        computed once and duplicated, the rest runs on the full batch.  Returns the full batch."""
        N, H, W, C = h.shape
        n = H * W
        M = N * n
        inner = d["inner"]
        dev = h.device
        g = torch.empty_like(h)
        ops.groupnorm(h, d["gn_w"], d["gn_b"], g, N, n, 1e-6, False, st["ws"], stats=getattr(h, "_gn", None))
        t = torch.empty(M, inner, dtype=torch.float16, device=dev)
        fold0 = _LN_FOLD and inner % 64 == 0
        if fold0:
            t._ln = ops.row_stats_buffer(M, inner, dev)
        ops.gemm(g.view(M, C), d["pin_w"], t, bias=d["pin_b"], row_stats=t._ln if fold0 else None)
        for i, b in enumerate(d["blocks"]):
            ctx = st["ctx"][i] if i < len(st["ctx"]) else st["ctx"][-1]
            if share and not b["self"]:
                # disable_self_attn: attn1 already attends to the context, which differs between the CFG halves --
                # nothing more can be shared, widen to the full batch here
                t, h = self._dup_rows(t), self._dup_rows(h)
                N, M, share = 2 * N, 2 * M, False
            fold = _LN_FOLD and inner % 64 == 0
            if not fold and self._xattn_fused(b, ctx, n, st):
                # 320 channels: attn1's output projection through norm3 in one launch, then the fused feed-forward
                ln = torch.empty_like(t)
                ops.layernorm(t, b["ln1_w"], b["ln1_b"], ln)
                a1 = self._attn(b["attn1"], ln, None, N, n, st, True, t, None)
                if share:
                    # shared CFG halves: widen before attn1's output projection (identical halves, bit-identical result)
                    a1, t, h = self._dup_rows(a1), self._dup_rows(t), self._dup_rows(h)
                    N, M, share = 2 * N, 2 * M, False
                a1d, ad = b["attn1"], b["attn2"]
                kv = self._context_kv(ad, ctx, N, st)
                st["layer"] += 1
                t2, t3, ln3 = (torch.empty_like(t) for _ in range(3))
                ops.xattn_block(a1, t, a1d["o_w"], a1d["o_b"], b["ln2_w"], b["ln2_b"], ad["q_w"], kv, ctx.shape[1],
                                ad["o_w"], ad["o_b"], b["ln3_w"], b["ln3_b"], t2, t3, ln3, n, ad["heads"], ad["d"], ad["hs"],
                                aux_cols=ad["aux"])
                t = torch.empty_like(t3)
                ops.geglu_ff(ln3, b["ff1p_w"], b["ff1p_b"], b["ff2t_w"], b["ff2_b"], t3, t)
                continue
            if fold:
                # LayerNorm folded into the contractions either side of it (anysd_gemm_params::row_stats / ln_stats): the
                # producer of t / t2 / t3 has left per-row moments, the consumer takes the un-normalised rows
                fb = self._ln_folded(b)
                t2 = torch.empty_like(t)
                self._attn(b["attn1"], t, None if b["self"] else ctx, N, n, st, b["self"], t, t2, ln=(t._ln, fb["a1"]), out_stats=True)
            else:
                ln = torch.empty_like(t)
                ops.layernorm(t, b["ln1_w"], b["ln1_b"], ln)
                t2 = torch.empty_like(t)
                if b["self"]:
                    self._attn(b["attn1"], ln, None, N, n, st, True, t, t2)
                else:
                    self._attn(b["attn1"], ln, ctx, N, n, st, False, t, t2)
                ln2 = torch.empty_like(t)
                ops.layernorm(t2, b["ln2_w"], b["ln2_b"], ln2)
            if ctx is None:   # "if no context is given, cross-attention defaults to self-attention"
                raise NotImplementedError("attn2 without context (self-attention fallback) is not used on the AnySD path")
            q_pre = None
            if share:
                ad = b["attn2"]
                q_half = torch.empty(M, ad["heads"] * ad["hs"], dtype=torch.float16, device=dev)
                if fold:
                    ops.gemm(t2, fb["a2"]["w"], q_half, bias=fb["a2"]["b"], ln=(t2._ln, fb["a2"]["cs"], 1e-5))
                else:
                    ops.gemm(ln2, ad["q_w"], q_half)
                q_pre, t2, h = self._dup_rows(q_half), self._dup_rows(t2), self._dup_rows(h)
                N, M, share = 2 * N, 2 * M, False
                t = None                                        # (half-batch tensor, not used again)
            t3 = torch.empty_like(t2)
            if fold:
                self._attn(b["attn2"], t2, ctx, N, n, st, False, t2, t3, expert=True, q_pre=q_pre,
                           ln=None if q_pre is not None else (t2._ln, fb["a2"]), out_stats=True)
                ffh = torch.empty(M, b["ff2_w"].shape[1], dtype=torch.float16, device=dev)
                ops.gemm(t3, fb["ff1"]["w"], ffh, bias=fb["ff1"]["b"], act=2, ln=(t3._ln, fb["ff1"]["cs"], 1e-5))
            else:
                self._attn(b["attn2"], ln2, ctx, N, n, st, False, t2, t3, expert=True, q_pre=q_pre)
                ln3 = torch.empty_like(t3)
                ops.layernorm(t3, b["ln3_w"], b["ln3_b"], ln3)
                if "ff1p_w" in b:
                    # 320 channels: both products and GEGLU in one launch, the hidden activations never written
                    t = torch.empty_like(t3)
                    ops.geglu_ff(ln3, b["ff1p_w"], b["ff1p_b"], b["ff2t_w"], b["ff2_b"], t3, t)
                    continue
                ffh = torch.empty(M, b["ff2_w"].shape[1], dtype=torch.float16, device=dev)
                ops.gemm(ln3, b["ff1_w"], ffh, bias=b["ff1_b"], act=2)
            t4 = torch.empty_like(t3)
            nxt = fold and i + 1 < len(d["blocks"])              # depth > 1: the next block's norm1 reads this output
            if nxt:
                t4._ln = ops.row_stats_buffer(M, inner, dev)
            ops.gemm(ffh, b["ff2_w"], t4, bias=b["ff2_b"], residual=t3, row_stats=t4._ln if nxt else None)
            t = t4
        out = torch.empty(N, H, W, C, dtype=torch.float16, device=dev)
        out._gn = ops.gemm(t, d["pout_w"], out.view(M, C), bias=d["pout_b"], residual=h.view(M, C), rows_per_batch=n, stats_images=N)
        return out
