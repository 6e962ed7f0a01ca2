"""H100-native first stage: ``AutoencoderKL`` -- drop-in for ``ldm.models.autoencoder.AutoencoderKL`` (encode / decode)
with the ``Encoder`` / ``Decoder`` of ``ldm.modules.diffusionmodules.model`` (SURVEY.md 8f rank 1: the step right before /
after the denoising loop, visual_reference_tool.py:220).

Same constructor (``ddconfig``, ``embed_dim``; ``lossconfig`` accepted and ignored: inference only), same ``state_dict``
keys and shapes (``encoder.*``, ``decoder.*``, ``quant_conv``, ``post_quant_conv``), same calls
``encode(x) -> DiagonalGaussianDistribution``, ``decode(z) -> image``.  Execution reuses the UNet's kernels through the C ABI:

  ResnetBlock  (model.py:91-150)    GroupNorm(32, eps 1e-6)+swish fused -> implicit-GEMM conv3x3 (+ bias, + residual / nin_shortcut)
  AttnBlock    (model.py:152-203)   ONE head of width C: the wgmma attention kernel when C <= 160; for the C = 512 of the SD
                                    autoencoder two contractions around a row softmax (S = q k^T in fp32, P fp16, O = P v)
  Downsample   (model.py:68-88)     F.pad(x, (0,1,0,1)) + conv3x3 stride 2 pad 0 = the conv kernel's right/bottom padding mode
  Upsample     (model.py:49-65)     nearest x2 + conv3x3 (the UNet's upsample conv)
  quant_conv / post_quant_conv      1x1 convs on 4 / 8 channels: GEMMs on 64-channel zero-padded rows
  DiagonalGaussianDistribution      distributions.py:24-62: clamp / std / sample in one small kernel

No eager-PyTorch math, no CPU fallback.  Not implemented (raise): ``attn_type`` other than "vanilla", ``use_timestep``.
"""
import torch
import torch.nn as nn

from . import ops
from .unet import _Param, _pack_conv3, _f, _h


class _Block(nn.Module):
    """ResnetBlock parameter holder (model.py:91-130, temb_channels = 0)."""

    def __init__(self, cin, cout):
        super().__init__()
        self.in_channels, self.out_channels = cin, cout
        self.norm1 = _Param((cin,), kind="norm")
        self.conv1 = _Param((cout, cin, 3, 3), kind="conv")
        self.norm2 = _Param((cout,), kind="norm")
        self.conv2 = _Param((cout, cout, 3, 3), kind="conv")
        if cin != cout:
            self.nin_shortcut = _Param((cout, cin, 1, 1), kind="conv")


class _Attn(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.in_channels = c
        self.norm = _Param((c,), kind="norm")
        self.q, self.k, self.v = (_Param((c, c, 1, 1), kind="conv") for _ in range(3))
        self.proj_out = _Param((c, c, 1, 1), kind="conv")


class _Resample(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv = _Param((c, c, 3, 3), kind="conv")


def _check(attn_type, **kw):
    if attn_type != "vanilla" or kw.get("use_linear_attn"):
        raise NotImplementedError("anyedit_b200.autoencoder: only attn_type='vanilla' (the SD / AnyDoor first stage) is implemented")


class Encoder(nn.Module):
    """Parameter tree of model.py:368-545's Encoder."""

    def __init__(self, *, ch, out_ch=None, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions, dropout=0.0,
                 resamp_with_conv=True, in_channels, resolution, z_channels, double_z=True, use_linear_attn=False,
                 attn_type="vanilla", **ignore_kwargs):
        super().__init__()
        _check(attn_type, use_linear_attn=use_linear_attn)
        assert resamp_with_conv, "resamp_with_conv=False (avg-pool downsampling) is not implemented"
        self.ch, self.num_resolutions, self.num_res_blocks = ch, len(ch_mult), num_res_blocks
        self.resolution, self.in_channels = resolution, in_channels
        self.conv_in = _Param((ch, in_channels, 3, 3), kind="conv")
        curr_res, in_ch_mult = resolution, (1,) + tuple(ch_mult)
        self.down = nn.ModuleList()
        block_in = ch
        for i in range(self.num_resolutions):
            block, attn = nn.ModuleList(), nn.ModuleList()
            block_in, block_out = ch * in_ch_mult[i], ch * ch_mult[i]
            for _ in range(num_res_blocks):
                block.append(_Block(block_in, block_out))
                block_in = block_out
                if curr_res in attn_resolutions:
                    attn.append(_Attn(block_in))
            down = nn.Module()
            down.block, down.attn = block, attn
            if i != self.num_resolutions - 1:
                down.downsample = _Resample(block_in)
                curr_res //= 2
            self.down.append(down)
        self.mid = nn.Module()
        self.mid.block_1, self.mid.attn_1, self.mid.block_2 = _Block(block_in, block_in), _Attn(block_in), _Block(block_in, block_in)
        self.norm_out = _Param((block_in,), kind="norm")
        self.conv_out = _Param((2 * z_channels if double_z else z_channels, block_in, 3, 3), kind="conv")


class Decoder(nn.Module):
    """Parameter tree of model.py:546-653's Decoder."""

    def __init__(self, *, ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions, dropout=0.0, resamp_with_conv=True,
                 in_channels=None, resolution, z_channels, give_pre_end=False, tanh_out=False, use_linear_attn=False,
                 attn_type="vanilla", **ignorekwargs):
        super().__init__()
        _check(attn_type, use_linear_attn=use_linear_attn)
        assert resamp_with_conv and not give_pre_end
        self.ch, self.num_resolutions, self.num_res_blocks = ch, len(ch_mult), num_res_blocks
        self.resolution, self.tanh_out, self.out_ch = resolution, tanh_out, out_ch
        block_in = ch * ch_mult[self.num_resolutions - 1]
        curr_res = resolution // 2 ** (self.num_resolutions - 1)
        self.z_shape = (1, z_channels, curr_res, curr_res)
        self.conv_in = _Param((block_in, z_channels, 3, 3), kind="conv")
        self.mid = nn.Module()
        self.mid.block_1, self.mid.attn_1, self.mid.block_2 = _Block(block_in, block_in), _Attn(block_in), _Block(block_in, block_in)
        ups = []
        for i in reversed(range(self.num_resolutions)):
            block, attn = nn.ModuleList(), nn.ModuleList()
            block_out = ch * ch_mult[i]
            for _ in range(num_res_blocks + 1):
                block.append(_Block(block_in, block_out))
                block_in = block_out
                if curr_res in attn_resolutions:
                    attn.append(_Attn(block_in))
            up = nn.Module()
            up.block, up.attn = block, attn
            if i != 0:
                up.upsample = _Resample(block_in)
                curr_res *= 2
            ups.insert(0, up)
        self.up = nn.ModuleList(ups)
        self.norm_out = _Param((block_in,), kind="norm")
        self.conv_out = _Param((out_ch, block_in, 3, 3), kind="conv")


class DiagonalGaussianDistribution(object):
    """distributions.py:24-62.  ``parameters``: fp32 NCHW moments [B, 2Z, H, W] on the GPU."""

    def __init__(self, parameters, deterministic=False):
        self.parameters = parameters.float().contiguous()
        B, Z2, H, W = self.parameters.shape
        self.deterministic = deterministic
        self.mean = torch.empty(B, Z2 // 2, H, W, dtype=torch.float32, device=parameters.device)
        self.logvar = torch.empty_like(self.mean)
        ops.gaussian_posterior(self.parameters, None, self.mean, self.logvar)        # mean (= mode) and the clamped logvar

    @property
    def std(self):
        return torch.zeros_like(self.mean) if self.deterministic else torch.exp(0.5 * self.logvar)

    @property
    def var(self):
        return torch.zeros_like(self.mean) if self.deterministic else torch.exp(self.logvar)

    def sample(self, noise=None, scale=1.0):
        """mean + std * noise (distributions.py:37-39); ``scale``: ``get_first_stage_encoding``'s scale_factor, applied in
        the same kernel."""
        if self.deterministic:
            noise = torch.zeros_like(self.mean)
        noise = torch.randn(self.mean.shape, device=self.mean.device) if noise is None else noise.float().contiguous()
        out = torch.empty_like(self.mean)
        ops.gaussian_posterior(self.parameters, noise, out, None, scale=scale)
        return out

    def mode(self):
        return self.mean


class AutoencoderKL(nn.Module):
    """See module docstring.  Reference: ldm/models/autoencoder.py:13-91."""

    def __init__(self, ddconfig, lossconfig=None, embed_dim=4, ckpt_path=None, ignore_keys=(), image_key="image",
                 colorize_nlabels=None, monitor=None, ema_decay=None, learn_logvar=False):
        super().__init__()
        assert ddconfig["double_z"]
        self.image_key, self.embed_dim = image_key, embed_dim
        self.encoder = Encoder(**ddconfig)
        self.decoder = Decoder(**ddconfig)
        z = ddconfig["z_channels"]
        self.quant_conv = _Param((2 * embed_dim, 2 * z, 1, 1), kind="conv")
        self.post_quant_conv = _Param((z, embed_dim, 1, 1), kind="conv")
        self._pack, self._pack_key, self._epoch = None, None, 0
        if ckpt_path is not None:
            self.init_from_ckpt(ckpt_path, ignore_keys=list(ignore_keys))

    def init_from_ckpt(self, path, ignore_keys=list()):
        sd = torch.load(path, map_location="cpu")["state_dict"]
        for k in list(sd.keys()):
            if any(k.startswith(ik) for ik in ignore_keys):
                del sd[k]
        self.load_state_dict(sd, strict=False)

    def invalidate(self):
        self._pack = None
        self._epoch += 1

    # ---- packing ------------------------------------------------------------------------------------------------
    def _prepare(self):
        ps = list(self.parameters())
        dev = ps[0].device
        key = (str(dev), sum(p._version for p in ps), self._epoch)
        if self._pack is not None and self._pack_key == key:
            return self._pack
        if dev.type != "cuda":
            raise RuntimeError("anyedit_b200.AutoencoderKL runs on CUDA only (no CPU fallback); call .cuda() first")
        pad64 = lambda c: (c + 63) // 64 * 64

        def conv3(m, cin_pad=None, cout_pad=None):
            w, b = _pack_conv3(m.weight, dev, cin_pad), _f(m.bias, dev)
            if cout_pad and cout_pad != w.shape[0]:
                w = torch.cat([w, w.new_zeros(cout_pad - w.shape[0], w.shape[1])], 0).contiguous()
                b = torch.cat([b, b.new_zeros(cout_pad - b.shape[0])], 0).contiguous()
            return {"w": w, "b": b}

        def lin(m):
            return _h(m.weight.reshape(m.weight.shape[0], -1), dev), _f(m.bias, dev)

        def block(m):
            d = {"cin": m.in_channels, "cout": m.out_channels, "n1": (_f(m.norm1.weight, dev), _f(m.norm1.bias, dev)),
                 "n2": (_f(m.norm2.weight, dev), _f(m.norm2.bias, dev)), "c1": conv3(m.conv1), "c2": conv3(m.conv2)}
            if hasattr(m, "nin_shortcut"):
                d["nin"] = lin(m.nin_shortcut)
            return d

        def attn(m):
            c = m.in_channels
            d = {"c": c, "norm": (_f(m.norm.weight, dev), _f(m.norm.bias, dev)), "proj": lin(m.proj_out)}
            wq, bq = lin(m.q)
            wk, bk = lin(m.k)
            wv, bv = lin(m.v)
            d["wide"] = not (c % 16 == 0 and c <= 160)
            if d["wide"]:
                d["qk_w"], d["qk_b"] = torch.cat([wq, wk], 0).contiguous(), torch.cat([bq, bk]).contiguous()
                d["v_w"], d["v_b"] = wv, bv
            else:
                d["qkv_w"], d["qkv_b"] = torch.cat([wq, wk, wv], 0).contiguous(), torch.cat([bq, bk, bv]).contiguous()
            return d

        def level(mod, resample):
            return {"blocks": [block(b) for b in mod.block], "attns": [attn(a) for a in mod.attn],
                    "resample": conv3(getattr(mod, resample).conv) if hasattr(mod, resample) else None}

        def mid(m):
            return {"b1": block(m.block_1), "attn": attn(m.attn_1), "b2": block(m.block_2)}

        enc, dec = self.encoder, self.decoder
        P = {"enc": {"cin_pad": pad64(enc.in_channels), "conv_in": conv3(enc.conv_in, pad64(enc.in_channels)),
                     "down": [level(d, "downsample") for d in enc.down], "mid": mid(enc.mid),
                     "norm_out": (_f(enc.norm_out.weight, dev), _f(enc.norm_out.bias, dev)),
                     "conv_out": conv3(enc.conv_out, cout_pad=64)},          # 2z filters + zero filters: writes full 64-channel rows
             "dec": {"conv_in": conv3(dec.conv_in, 64), "mid": mid(dec.mid), "up": [level(u, "upsample") for u in dec.up],
                     "norm_out": (_f(dec.norm_out.weight, dev), _f(dec.norm_out.bias, dev)),
                     "conv_out": conv3(dec.conv_out, cout_pad=(dec.out_ch + 7) // 8 * 8)}}
        # 1x1 convs on 2z / embed_dim channels: [N (padded to 8), K = 64] on zero-padded 64-channel rows
        def tiny_lin(m, n_pad):
            w = m.weight.detach().to(dev).float().reshape(m.weight.shape[0], -1)
            n, k = w.shape
            assert k <= 64 and n <= n_pad
            W = torch.zeros(n_pad, 64, device=dev)
            W[:n, :k] = w
            b = torch.zeros(n_pad, device=dev)
            b[:n] = m.bias.detach().to(dev).float()
            return W.to(torch.float16).contiguous(), b.contiguous(), n
        # quant_conv writes fp32 moments (8 columns); post_quant_conv writes the fp16 64-channel rows the decoder's conv_in reads
        P["quant"] = tiny_lin(self.quant_conv, (2 * self.embed_dim + 7) // 8 * 8)
        P["post_quant"] = tiny_lin(self.post_quant_conv, 64)
        P["post_quant_scaled"] = {}
        self._pack, self._pack_key = P, key
        return P

    # ---- block executors (NHWC fp16) ------------------------------------------------------------------------------
    @staticmethod
    def _gn(x, gb, ws, silu):
        N, H, W, C = x.shape
        y = torch.empty_like(x)
        ops.groupnorm(x, gb[0], gb[1], y, N, H * W, 1e-6, silu, ws)
        return y

    def _block(self, d, x, ws):
        """ResnetBlock.forward (model.py:131-150), temb = None."""
        N, H, W, cin = x.shape
        cout = d["cout"]
        a = self._gn(x, d["n1"], ws, True)
        h = torch.empty(N, H, W, cout, dtype=torch.float16, device=x.device)
        ops.conv3x3(a, d["c1"]["w"], h.view(-1, cout), bias=d["c1"]["b"])
        b = self._gn(h, d["n2"], ws, True)
        if "nin" in d:
            res = torch.empty(N * H * W, cout, dtype=torch.float16, device=x.device)
            ops.gemm(x.view(-1, cin), d["nin"][0], res, bias=d["nin"][1])
        else:
            res = x.view(-1, cin)
        out = torch.empty(N, H, W, cout, dtype=torch.float16, device=x.device)
        ops.conv3x3(b, d["c2"]["w"], out.view(-1, cout), bias=d["c2"]["b"], residual=res)
        return out

    def _attn(self, d, x, ws):
        """AttnBlock.forward (model.py:176-203): softmax(q^T k C^-0.5) over the keys, one head of width C."""
        N, H, W, C = x.shape
        n, M, dev = H * W, N * H * W, x.device
        g = self._gn(x, d["norm"], ws, False).view(M, C)
        a = torch.empty(M, C, dtype=torch.float16, device=dev)
        if not d["wide"]:
            qkv = torch.empty(M, 3 * C, dtype=torch.float16, device=dev)
            ops.gemm(g, d["qkv_w"], qkv, bias=d["qkv_b"])
            ops.attention(qkv, qkv[:, C:], qkv[:, 2 * C:], a, N, 1, n, n, C, 3 * C, 3 * C, 3 * C, C)
        else:
            qk = torch.empty(M, 2 * C, dtype=torch.float16, device=dev)
            ops.gemm(g, d["qk_w"], qk, bias=d["qk_b"])
            n8 = (n + 7) // 8 * 8                                   # row pitch of S / P / v^T (16-byte aligned rows)
            S = torch.empty(n, n8, dtype=torch.float32, device=dev)
            Pm = torch.zeros(n, n8, dtype=torch.float16, device=dev)
            vT = torch.zeros(C, n8, dtype=torch.float16, device=dev)
            for i in range(N):
                rows = slice(i * n, (i + 1) * n)
                ops.gemm(qk[rows, :C], qk[rows, C:], S, N=n)                         # S = q k^T (fp32)
                ops.softmax_rows(S[:, :n], Pm[:, :n], C ** -0.5)
                ops.gemm(d["v_w"], g[rows], vT, N=n)                               # v^T = Wv g^T  [C, n]
                ops.gemm(Pm, vT, a[rows], bias=d["v_b"], K=n8)                      # O = P v + b_v (rows of P sum to 1)
        out = torch.empty(N, H, W, C, dtype=torch.float16, device=dev)
        ops.gemm(a, d["proj"][0], out.view(M, C), bias=d["proj"][1], residual=x.view(M, C))
        return out

    def _mid(self, d, h, ws):
        return self._block(d["b2"], self._attn(d["attn"], self._block(d["b1"], h, ws), ws), ws)

    # ---- public API -------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def encode(self, x):
        """autoencoder.py:82-86: Encoder -> quant_conv -> DiagonalGaussianDistribution(moments)."""
        P = self._prepare()
        E = P["enc"]
        dev = x.device
        if dev.type != "cuda":
            raise RuntimeError("anyedit_b200.AutoencoderKL: input must be a CUDA tensor (no CPU fallback)")
        N, Cin, H, W = x.shape
        assert Cin == self.encoder.in_channels
        f16 = dict(dtype=torch.float16, device=dev)
        ws = ops.groupnorm_workspace(N, 32, 0, dev)
        xin = torch.zeros(N, H, W, E["cin_pad"], **f16)
        ops.nchw_to_nhwc(x.float().contiguous(), xin, 0)
        ch = self.encoder.ch
        h = torch.empty(N, H, W, ch, **f16)
        ops.conv3x3(xin, E["conv_in"]["w"], h.view(-1, ch), bias=E["conv_in"]["b"], logical_cin=Cin)
        for lvl in E["down"]:
            for j, b in enumerate(lvl["blocks"]):
                h = self._block(b, h, ws)
                if lvl["attns"]:
                    h = self._attn(lvl["attns"][j], h, ws)
            if lvl["resample"] is not None:                      # Downsample: pad right/bottom, conv3x3 stride 2 (model.py:83-85)
                n_, hh, ww, c = h.shape
                o = torch.empty(n_, (hh - 2) // 2 + 1, (ww - 2) // 2 + 1, c, **f16)
                ops.conv3x3(h, lvl["resample"]["w"], o.view(-1, c), bias=lvl["resample"]["b"], stride=2, pad_rb=True)
                h = o
        h = self._mid(E["mid"], h, ws)
        a = self._gn(h, E["norm_out"], ws, True)
        n_, hh, ww, c = h.shape
        mom_pre = torch.empty(n_ * hh * ww, 64, **f16)           # 2z real channels, the rest exact zeros (zero filters)
        ops.conv3x3(a, E["conv_out"]["w"], mom_pre, bias=E["conv_out"]["b"], logical_cout=2 * self.decoder.z_shape[1])
        qw, qb, qn = P["quant"]
        mom = torch.empty(n_ * hh * ww, qw.shape[0], dtype=torch.float32, device=dev)
        ops.gemm(mom_pre, qw, mom, bias=qb)
        moments = torch.empty(n_, qn, hh, ww, dtype=torch.float32, device=dev)
        ops.nhwc_to_nchw(mom.view(n_, hh, ww, qw.shape[0]), moments)
        return DiagonalGaussianDistribution(moments)

    @torch.no_grad()
    def decode(self, z, z_scale=1.0):
        """autoencoder.py:88-91: post_quant_conv -> Decoder (model.py:617-641).  ``z_scale``: a factor applied to z first
        (``decode_first_stage``'s 1 / scale_factor, ddpm.py), folded into the 1x1 post_quant_conv weights."""
        P = self._prepare()
        D = P["dec"]
        dev = z.device
        if dev.type != "cuda":
            raise RuntimeError("anyedit_b200.AutoencoderKL: input must be a CUDA tensor (no CPU fallback)")
        N, Cz, H, W = z.shape
        f16 = dict(dtype=torch.float16, device=dev)
        ws = ops.groupnorm_workspace(N, 32, 0, dev)
        zin = torch.zeros(N, H, W, 64, **f16)
        ops.nchw_to_nhwc(z.float().contiguous(), zin, 0)
        pw, pb, pn = P["post_quant"]
        if z_scale != 1.0:
            if z_scale not in P["post_quant_scaled"]:
                P["post_quant_scaled"][z_scale] = (pw.float() * z_scale).to(torch.float16).contiguous()
            pw = P["post_quant_scaled"][z_scale]
        zq = torch.empty(N * H * W, 64, **f16)
        ops.gemm(zin.view(-1, 64), pw, zq, bias=pb)
        c0 = D["conv_in"]["w"].shape[0]
        h = torch.empty(N, H, W, c0, **f16)
        ops.conv3x3(zq.view(N, H, W, 64), D["conv_in"]["w"], h.view(-1, c0), bias=D["conv_in"]["b"], logical_cin=pn)
        h = self._mid(D["mid"], h, ws)
        for lvl in reversed(D["up"]):
            for j, b in enumerate(lvl["blocks"]):
                h = self._block(b, h, ws)
                if lvl["attns"]:
                    h = self._attn(lvl["attns"][j], h, ws)
            if lvl["resample"] is not None:
                n_, hh, ww, c = h.shape
                o = torch.empty(n_, 2 * hh, 2 * ww, c, **f16)
                ops.conv3x3(h, lvl["resample"]["w"], o.view(-1, c), bias=lvl["resample"]["b"], upsample=1)
                h = o
        a = self._gn(h, D["norm_out"], ws, True)
        n_, hh, ww, c = h.shape
        cpad = D["conv_out"]["w"].shape[0]
        o = torch.empty(n_, hh, ww, cpad, dtype=torch.float32, device=dev)
        ops.conv3x3(a, D["conv_out"]["w"], o.view(-1, cpad), bias=D["conv_out"]["b"], logical_cout=self.decoder.out_ch)
        out = torch.empty(n_, self.decoder.out_ch, hh, ww, dtype=torch.float32, device=dev)
        ops.nhwc_to_nchw(o, out)
        return torch.tanh(out) if self.decoder.tanh_out else out

    def forward(self, input, sample_posterior=True):
        posterior = self.encode(input)
        z = posterior.sample() if sample_posterior else posterior.mode()
        return self.decode(z), posterior

    def get_input(self, batch, k):
        x = batch[k]
        if len(x.shape) == 3:
            x = x[..., None]
        return x.permute(0, 3, 1, 2).to(memory_format=torch.contiguous_format).float()
