"""ControlNet branch on the H100 kernels (SURVEY.md 8f rank 3) -- the only in-tree end-to-end consumer of the ``ldm`` UNet
(AnyDoor visual reference, AnyEdit_Collection/other_modules/cldm/cldm.py).

  ``ControlNet``            cldm.py:47-304: the UNet's encoder half (input blocks + middle block), a hint stem of eight 3x3
                            convs (3 of them stride 2, SiLU between, the last one zero-initialised) and 13 zero-initialised 1x1
                            convs whose outputs are the residuals; same constructor kwargs, same ``state_dict`` keys
                            (``input_hint_block.{0,2,..,14}``, ``zero_convs.{i}.0``, ``middle_block_out.0``, ...).
                            AnyDoor quirk kept (cldm.py:291-296): the hint stem's output REPLACES the first input block's
                            output -- ``x`` itself only fixes shape and dtype.
  ``ControlledUnetModel``   cldm.py:21-44 = ``UNetModel.forward(..., control=, only_mid_control=)`` (already there).
  ``ControlDenoiser``       the ``apply_model`` of ``ControlLDM`` (cldm.py:328-340): ``c_concat`` is the hint image,
                            ``c_crossattn`` the text context, ``control_scales`` folded into the packed zero-conv weights.

Execution: the hint stem's channels (16 / 32 / 96 / 256) are zero-padded to multiples of 64 so that all eight convs run on
the wgmma implicit-GEMM kernel with the SiLU in the epilogue (SiLU(0) = 0 keeps the padding exact); the stem depends on
neither x nor t, so its output is kept for as long as the hint tensor is unchanged (a sampling run computes it once, the
reference recomputes it every step); the residuals stay NHWC fp16 and are added to the UNet's activations by one kernel each
(no NCHW round trip).  Two-call CFG of ``ddim_hacked.py:181-232`` = the batched [uncond ; cond] call of ``DDIMSampler``
(every kernel is batch-independent, so the two formulations agree bit for bit).
"""
import torch
import torch.nn as nn

from . import ops
from .diffusion import LatentDenoiser
from .unet import UNetModel, _Param, _Slot, _f, _h, _pack_conv3, _seq

ControlledUnetModel = UNetModel


class _Residuals(list):
    """The 13 residuals in NHWC fp16 (``UNetModel.forward`` adds them with one kernel each)."""
    nhwc = True


def _pad64(c):
    return (c + 63) // 64 * 64


class ControlNet(UNetModel):
    def __init__(self, image_size, in_channels, model_channels, hint_channels, num_res_blocks, attention_resolutions, dropout=0,
                 channel_mult=(1, 2, 4, 8), conv_resample=True, dims=2, use_checkpoint=False, use_fp16=False, num_heads=-1,
                 num_head_channels=-1, num_heads_upsample=-1, use_scale_shift_norm=False, resblock_updown=False,
                 use_new_attention_order=False, use_spatial_transformer=False, transformer_depth=1, context_dim=None, n_embed=None,
                 legacy=True, disable_self_attentions=None, num_attention_blocks=None, disable_middle_self_attn=False,
                 use_linear_in_transformer=False):
        super().__init__(image_size, in_channels, model_channels, 0, num_res_blocks, attention_resolutions, dropout=dropout,
                         channel_mult=channel_mult, conv_resample=conv_resample, dims=dims, use_checkpoint=use_checkpoint,
                         use_fp16=use_fp16, num_heads=num_heads, num_head_channels=num_head_channels,
                         num_heads_upsample=num_heads_upsample, use_scale_shift_norm=use_scale_shift_norm,
                         resblock_updown=resblock_updown, use_new_attention_order=use_new_attention_order,
                         use_spatial_transformer=use_spatial_transformer, transformer_depth=transformer_depth,
                         context_dim=context_dim, n_embed=n_embed, legacy=legacy, disable_self_attentions=disable_self_attentions,
                         num_attention_blocks=num_attention_blocks, disable_middle_self_attn=disable_middle_self_attn,
                         use_linear_in_transformer=use_linear_in_transformer, _encoder_only=True)
        self.hint_channels = hint_channels
        mc = model_channels
        # cldm.py:146-162: conv, SiLU, conv, SiLU, conv(s2), ... , zero conv (Sequential indices 0, 2, .., 14)
        chans = [(hint_channels, 16, 1), (16, 16, 1), (16, 32, 2), (32, 32, 1), (32, 96, 2), (96, 96, 1), (96, 256, 2), (256, mc, 1)]
        mods = []
        for i, (ci, co, _s) in enumerate(chans):
            mods.append(_Param((co, ci, 3, 3), kind="conv", zero=(i == len(chans) - 1)))
            if i != len(chans) - 1:
                mods.append(_Slot())
        self.input_hint_block = _seq(*mods)
        self._hint_strides = [s_ for _, _, s_ in chans]
        # one zero conv per input block output (+ the middle block's)
        outs = [mc]
        ch = mc
        for level, mult in enumerate(channel_mult):
            for _ in range(self.num_res_blocks[level]):
                ch = mult * mc
                outs.append(ch)
            if level != len(channel_mult) - 1:
                outs.append(ch)
        self.zero_convs = nn.ModuleList([_seq(_Param((c, c, 1, 1), kind="conv", zero=True)) for c in outs])
        self.middle_block_out = _seq(_Param((ch, ch, 1, 1), kind="conv", zero=True))
        self.control_scales = None               # set by ControlDenoiser; folded into the packed zero convs
        self._hint_cache = None

    # the encoder-only UNet pack calls this hook
    def _pack_extra(self, P, dev):
        hint = []
        convs = [m for m in self.input_hint_block if isinstance(m, _Param)]
        for i, m in enumerate(convs):
            co, ci = m.weight.shape[0], m.weight.shape[1]
            cop = co if i == len(convs) - 1 else _pad64(co)
            w = _pack_conv3(m.weight, dev, _pad64(ci))
            b = _f(m.bias, dev)
            if cop != co:                                # zero filters: SiLU(0) = 0 keeps the padded channels exact zeros
                w = torch.cat([w, w.new_zeros(cop - co, w.shape[1])], 0).contiguous()
                b = torch.cat([b, b.new_zeros(cop - co)], 0).contiguous()
            hint.append({"w": w, "b": b, "stride": self._hint_strides[i], "cin_pad": _pad64(ci), "cout": cop,
                         "act": 0 if i == len(convs) - 1 else 1, "cin": ci})
        P["hint"] = hint
        scales = self.control_scales or [1.0] * (len(self.zero_convs) + 1)
        zc = []
        for m, sc in zip(list(self.zero_convs) + [self.middle_block_out], scales):
            w = m[0].weight.detach().float().reshape(m[0].weight.shape[0], -1) * float(sc)
            zc.append((_h(w, dev), _f(m[0].bias.detach().float() * float(sc), dev)))
        P["zero"] = zc

    def set_control_scales(self, scales):
        scales = None if scales is None else [float(s_) for s_ in scales]
        if scales != self.control_scales:
            self.control_scales = scales
            self.invalidate()

    def invalidate(self):
        super().invalidate()
        self._hint_cache = None

    def _guided_hint(self, P, hint, dev):
        """input_hint_block(hint) (cldm.py:288): independent of x and t -- kept while the hint tensor is unchanged.  The
        buffers persist per hint geometry and are REFILLED IN PLACE when the hint's values change (a captured CUDA graph
        of the sampler keeps reading the same memory, like the kept context K/V of the UNet)."""
        geom = (tuple(hint.shape), str(dev))
        key = (hint.data_ptr(), hint._version, str(hint.dtype), self._pack_key)
        c = self._hint_cache
        if c is not None and c["geom"] == geom and c["key"] == key:
            return c["bufs"][-1]
        N, Ch, H, W = hint.shape
        assert Ch == self.hint_channels, f"expected {self.hint_channels} hint channels, got {Ch}"
        f16 = dict(dtype=torch.float16, device=dev)
        if c is None or c["geom"] != geom:
            bufs = [torch.zeros(N, H, W, P["hint"][0]["cin_pad"], **f16)]
            hh, ww = H, W
            for d in P["hint"]:
                hh, ww = (hh - 1) // d["stride"] + 1, (ww - 1) // d["stride"] + 1
                bufs.append(torch.empty(N, hh, ww, d["cout"], **f16))
            c = self._hint_cache = {"geom": geom, "key": None, "bufs": bufs}
        bufs = c["bufs"]
        ops.nchw_to_nhwc(hint.float().contiguous(), bufs[0], 0)
        for i, d in enumerate(P["hint"]):
            cur, out = bufs[i], bufs[i + 1]
            # the stem's output feeds the first ResBlock's GroupNorm: its epilogue statistics live in a persistent buffer too
            want = (getattr(out, "_gn", None) or True) if d["act"] == 0 else False
            st = ops.conv3x3(cur, d["w"], out.view(-1, d["cout"]), bias=d["b"], stride=d["stride"], act=d["act"],
                             logical_cin=d["cin"], stats=want)
            out._gn = st if d["act"] == 0 else None
        c["key"] = key
        return bufs[-1]

    @torch.no_grad()
    def forward(self, x, hint, timesteps, context, **kwargs):
        """-> the 13 residuals (cldm.py:283-304), NHWC fp16 (``_Residuals``)."""
        P = self.prepare()
        dev = x.device
        if dev.type != "cuda":
            raise RuntimeError("anyedit_b200.cldm.ControlNet: input must be a CUDA tensor (no CPU fallback)")
        N = x.shape[0]
        emb_all = self._embeddings(P, N, timesteps, None, None, dev)
        st = {"N": N, "ws": ops.groupnorm_workspace(N, 32, 0, dev), "emb_all": emb_all, "ctx": self._context16(context, N, dev),
              "anysd": None, "layer": 0, "xl": 0, "kvc": None}
        h = self._guided_hint(P, hint, dev)
        assert h.shape[0] == N and tuple(h.shape[1:3]) == tuple(x.shape[2:]), \
            "the hint must be 8x the latent resolution (three stride-2 convs in the stem)"
        outs = _Residuals()

        def emit(t, k):
            n_, hh, ww, c = t.shape
            o = torch.empty_like(t)
            ops.gemm(t.view(-1, c), P["zero"][k][0], o.view(-1, c), bias=P["zero"][k][1])
            outs.append(o)

        emit(h, 0)
        for k, blk in enumerate(P["input"], 1):
            h = self._run(blk, h, None, st)
            emit(h, k)
        h = self._run(P["middle"], h, None, st)
        emit(h, len(P["input"]) + 1)
        return outs


class ControlDenoiser(LatentDenoiser):
    """``ControlLDM.apply_model`` (cldm.py:328-340) for the samplers: ``cond = {"c_concat": [hint], "c_crossattn": [text]}``.
    ``cond_stage_model`` (e.g. ``encoders.FrozenDinoV2Encoder``): what ``get_learned_conditioning`` runs."""

    def __init__(self, unet, control_model, only_mid_control=False, control_scales=None, cond_stage_model=None, **kwargs):
        super().__init__(unet, "crossattn", **kwargs)
        assert isinstance(control_model, ControlNet)
        self.control_model = control_model
        self.only_mid_control = only_mid_control
        self.control_scales = list(control_scales) if control_scales is not None else [1.0] * 13
        self.cond_stage_model = cond_stage_model

    def get_learned_conditioning(self, c):
        """LatentDiffusion.get_learned_conditioning (ddpm.py) without a ``cond_stage_forward``: the model's ``encode`` when it
        has one, else its call -- visual_reference_tool.py:203-205 turns the reference image (and zeros) into c_crossattn."""
        m = self.cond_stage_model
        if m is None:
            raise RuntimeError("ControlDenoiser: constructed without a cond_stage_model")
        return m.encode(c) if callable(getattr(m, "encode", None)) else m(c)

    @property
    def graph_safe(self):
        return True

    def graph_key(self):
        ps = list(self.model.diffusion_model.parameters()) + list(self.control_model.parameters())
        return (tuple((str(p.device), p._version, p.data_ptr()) for p in ps).__hash__(), self.model.diffusion_model._epoch,
                self.control_model._epoch, tuple(self.control_scales))

    def invalidate(self):
        self.model.diffusion_model.invalidate()
        self.control_model.invalidate()

    def apply_model(self, x_noisy, t, cond, *args, **kwargs):
        assert isinstance(cond, dict)
        unet = self.model.diffusion_model
        cond_txt = torch.cat(cond["c_crossattn"], 1)
        if cond.get("c_concat") is None:
            return unet(x_noisy, timesteps=t, context=cond_txt, control=None, only_mid_control=self.only_mid_control)
        self.control_model.set_control_scales(self.control_scales)
        hint = cond["c_concat"][0] if len(cond["c_concat"]) == 1 else torch.cat(cond["c_concat"], 1)
        control = self.control_model(x=x_noisy, hint=hint, timesteps=t, context=cond_txt)
        return unet(x_noisy, timesteps=t, context=cond_txt, control=control, only_mid_control=self.only_mid_control)
