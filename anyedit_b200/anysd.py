"""AnySD task-aware router + learnable task embedding on top of the H100 UNet.

The AnySD model code is absent from the reference (empty, un-pinned submodule: .gitmodules:1-4,
SURVEY.md 0.2), so this follows the specification restated in ``oracle/anysd_oracle.py`` from the
call sites (train.py:420-424, 483-485, 694-695), the decoupled cross-attention template
(AnyEdit_Collection/other_modules/ip_adapter/attention_processor.py:82-188) and the in-tree
embedding-add slot (openaimodel.py:770-772).  PARITY UNPINNED against the real AnySD weights;
pinned against the oracle restatement and against the reduction to the plain UNet.

    te    = task_embs[edit_code]
    emb   = time_embed(t_emb) + te
    g_l   = softmax(router_l(te))                                  per cross-attention layer l
    attn2 = Attn(q, K_txt, V_txt) + sum_e g_l[:, e] * Attn(q, v @ Wk_le^T, v @ Wv_le^T)

Execution: the task-embedding add is fused into ``anysd_emb_finalize``; the router gate is a
GEMM + tiny softmax; all experts' K/V projections of a layer are ONE GEMM ([B*N_vis, E*2C]); each
expert's attention is accumulated into the text-attention output by the attention kernel's gated
epilogue (out += g[b, e] * attn).
"""
import math

import torch
import torch.nn as nn

from . import ops
from .diffusion import LatentDenoiser
from .unet import UNetModel, _Param, aux_bias, aux_cols_for, head_stride_for, pad_heads


class _Adapter(nn.Module):
    def __init__(self, ch, ctx_dim, n_exp, d_emb):
        super().__init__()
        self.router = _Param((n_exp, d_emb))
        self.to_k_ip = _Param((n_exp * ch, ctx_dim), bias=False)
        self.to_v_ip = _Param((n_exp * ch, ctx_dim), bias=False)


class _TaskEmb(nn.Module):
    def __init__(self, n, d):
        super().__init__()
        self.weight = nn.Parameter(torch.zeros(n, d))


class MoE(nn.Module):
    """``MoE(unet, image_encoder, expert_num, ckpt_path)`` (train.py:420-424).  ``image_encoder`` is
    accepted for signature compatibility; the CLIP-vision tower and the image projector are outside
    this path (SURVEY.md 8f rank 2) -- ``reference_image_embeds`` are the projected visual tokens
    [B, N_vis, context_dim] (or None / N_vis = 0)."""

    graph_safe = True

    def __init__(self, unet: UNetModel, image_encoder=None, expert_num=11, ckpt_path=None, num_tasks=25):
        super().__init__()
        assert isinstance(unet, UNetModel), "MoE needs an anyedit_b200.unet.UNetModel"
        assert unet.num_classes is None, "the task embedding uses the label_emb slot; build the UNet without num_classes"
        self.unet = unet
        self.image_encoder = image_encoder
        self.expert_num = expert_num
        d_emb = unet.time_embed_dim
        ctx_dim = unet.context_dim if isinstance(unet.context_dim, int) else unet.context_dim[0]
        self.task_embs = _TaskEmb(num_tasks, d_emb)
        sites, self._site_heads = [], []
        from .unet import _SpatialTransformer
        for blk in list(unet.input_blocks) + [unet.middle_block] + list(unet.output_blocks):
            for m in blk:
                if isinstance(m, _SpatialTransformer):
                    for _tb in m.transformer_blocks:
                        sites.append(m.inner)
                        self._site_heads.append((m.heads, m.d_head))
        self.adapter_modules = nn.ModuleList([_Adapter(c, ctx_dim, expert_num, d_emb) for c in sites])
        self.image_proj_model = nn.Identity()
        self._pack, self._pack_key, self._epoch = None, None, 0
        if ckpt_path is not None:
            self.load_state_dict(torch.load(ckpt_path, map_location="cpu"), strict=False)

    def _prepare(self, dev):
        key = (str(dev), sum(p._version for p in self.task_embs.parameters()) +
               sum(p._version for p in self.adapter_modules.parameters()), self._epoch)
        if self._pack is not None and self._pack_key == key:
            return self._pack
        E = self.expert_num
        P = {"task": self.task_embs.weight.detach().to(dev, torch.float32).contiguous(), "layers": []}
        for ad, (heads, dh) in zip(self.adapter_modules, self._site_heads):
            c = ad.to_k_ip.weight.shape[0] // E
            hs = head_stride_for(dh)
            cp = heads * hs                                   # padded-head projection width
            wk = ad.to_k_ip.weight.detach().reshape(E, c, -1)
            wv = ad.to_v_ip.weight.detach().reshape(E, c, -1)
            wk = torch.stack([pad_heads(wk[e], heads, dh, hs) for e in range(E)], 0)
            wv = torch.stack([pad_heads(wv[e], heads, dh, hs) for e in range(E)], 0)
            # rows: expert-major, [K_e ; V_e] per expert -> one GEMM gives [.., e*2Cp : e*2Cp+Cp] = K_e
            kv = torch.stack([wk, wv], 1).reshape(E * 2 * cp, -1)
            # same operand contract as the UNet's own cross attention (the experts reuse its q): see unet.aux_cols_for
            kv_b = torch.cat([aux_bias(heads, dh, hs, 2), aux_bias(heads, dh, hs, 1)]).repeat(E).to(dev) \
                if aux_cols_for(dh) else None
            P["layers"].append({"c": c, "cp": cp, "kv_w": kv.to(dev, torch.float16).contiguous(), "kv_b": kv_b})
        P["router_w"] = torch.stack([ad.router.weight.detach() for ad in self.adapter_modules], 0).to(
            dev, torch.float16).contiguous()                                   # [L, E, D]
        P["router_b"] = torch.stack([ad.router.bias.detach() for ad in self.adapter_modules], 0).to(
            dev, torch.float32).contiguous()                                   # [L, E]
        self._pack, self._pack_key = P, key
        return P

    @torch.no_grad()
    def forward(self, noisy_latents, timesteps, encoder_hidden_states, reference_image_embeds=None, edit_code=None):
        """eps = MoE(x8, t, text_ehs, visual_tokens, edit_code)  (train.py:694-695)."""
        dev = noisy_latents.device
        P = self._prepare(dev)
        N = noisy_latents.shape[0]
        E = self.expert_num
        if edit_code is None:
            edit_code = torch.zeros(N, dtype=torch.long, device=dev)
        edit_code = edit_code.to(device=dev, dtype=torch.int64).contiguous()
        vis = reference_image_embeds
        n_vis = 0 if vis is None else vis.shape[1]
        hook = {"task_table": P["task"], "edit_code": edit_code, "experts": None}
        if n_vis > 0:
            v32 = vis.to(dev).float().contiguous()
            v16 = torch.empty(v32.shape, dtype=torch.float16, device=dev)
            ops.cast_f16(v32, v16)
            nl = len(P["layers"])
            gates = torch.empty(N, nl, E, dtype=torch.float32, device=dev)
            ops.router_gate(P["task"], edit_code, P["router_w"], P["router_b"], gates)   # all layers at once

            def experts(layer, q, a, N_, n_q, heads, d, hs, aux):
                L = P["layers"][layer]
                C, Cp = L["c"], L["cp"]
                kv = torch.empty(N_ * n_vis, E * 2 * Cp, dtype=torch.float16, device=dev)
                ops.gemm(v16.view(N_ * n_vis, -1), L["kv_w"], kv, bias=L["kv_b"])
                ld = E * 2 * Cp
                qk = math.log(2.0) if aux else d ** -0.5          # aux packing: q already carries scale*log2(e)
                if n_vis <= 64:                                   # all experts of the layer in one launch
                    ops.expert_attention(q, kv, gates[:, layer], a, N_, heads, n_q, n_vis, d, E, Cp, ld, C, 2 * Cp, Cp, qk, head_stride=hs)
                else:
                    for e in range(E):
                        ops.attention(q, kv[:, e * 2 * Cp:], kv[:, e * 2 * Cp + Cp:], a, N_, heads, n_q, n_vis, d,
                                      Cp, ld, ld, C, gate=gates[:, layer, e:], gate_stride=nl * E, accumulate=True,
                                      head_stride=hs, aux_cols=aux)

            hook["experts"] = experts
        return self.unet(noisy_latents, timesteps, context=encoder_hidden_states, anysd=hook)

    def invalidate(self, unet=False):
        """Drop the packed adapter / router / task tensors (after an in-place weight change that does not bump parameter
        versions: the raw AdamW kernel, a ``.data`` broadcast); ``unet=True`` also drops the frozen UNet's packs."""
        self._pack = None
        self._epoch += 1
        if unet:
            self.unet.invalidate()

    def save_pretrained(self, path):
        import os
        os.makedirs(path, exist_ok=True)
        # clones: under AdapterTrainer the parameters are views of one flat buffer (torch.save would write all of it per view)
        sd = {k: v.detach().clone() for k, v in self.state_dict().items() if not k.startswith("unet.")}
        torch.save(sd, os.path.join(path, "anysd_adapter.pt"))


class AnySDDenoiser(LatentDenoiser):
    """The ``apply_model`` boundary (ddpm.py:854-869) for the AnySD ``MoE``: what a sampler drives when the task
    router, the task-embedding add and the visual expert stream are active (BASELINE configs[2] / configs[3]).

    ``cond`` is the ``hybrid`` dict of ``DiffusionWrapper.forward`` (ddpm.py:1344-1347) plus two optional AnySD keys,
    batched and CFG-concatenated by the samplers exactly like the others:
      ``c_task``    int64 [B] edit codes                (train.py:695 ``batch["edit_code"]``)
      ``c_visual``  list of [B, N_vis, context_dim] visual tokens, concatenated along tokens (train.py:688-694)
    """

    def __init__(self, moe: "MoE", **schedule_kwargs):
        assert isinstance(moe, MoE)
        super().__init__(moe.unet, "hybrid", **schedule_kwargs)
        self.moe = moe

    @property
    def graph_safe(self):
        return True

    def graph_key(self):
        ps = list(self.moe.unet.parameters()) + list(self.moe.task_embs.parameters()) + list(self.moe.adapter_modules.parameters())
        return (tuple((str(p.device), p._version, p.data_ptr()) for p in ps).__hash__(), self.moe._epoch, self.moe.unet._epoch)

    def invalidate(self):
        self.moe.invalidate(unet=True)

    def apply_model(self, x_noisy, t, cond, return_ids=False):
        assert isinstance(cond, dict), "AnySDDenoiser takes the hybrid conditioning dict"
        xc = torch.cat([x_noisy] + list(cond.get("c_concat") or []), dim=1)
        cc = torch.cat(cond["c_crossattn"], 1)
        vis = cond.get("c_visual")
        if isinstance(vis, (list, tuple)):
            vis = torch.cat(vis, 1) if len(vis) else None
        return self.moe(xc, t, cc, vis, cond.get("c_task"))
