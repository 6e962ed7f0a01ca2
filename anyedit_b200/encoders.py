"""Condition encoders on the H100 kernels (SURVEY.md 8f rank 2): what produces ``c_crossattn`` and the visual tokens right
before the denoising loop.

  ``FrozenCLIPEmbedder``            ldm/modules/encoders/modules.py:107-150 -- the CLIP text tower the ``ldm`` stack conditions on
                                    (``transformers.CLIPTextModel``: token + position embeddings, 12 pre-LN layers with a causal
                                    mask and QuickGELU, final LayerNorm); ``layer`` = "last" | "pooled" | "hidden".
  ``CLIPTextModel``                 the tower itself, ``transformers`` state-dict keys (``text_model.*``).
  ``CLIPVisionModelWithProjection`` the CLIP-H vision tower of train.py:688-691 (``image_encoder(..., output_hidden_states=True)
                                    .hidden_states[-2]``): patch embedding as one contraction, class token, pre-LN, 32 layers
                                    (GELU), ``vision_model.*`` / ``visual_projection`` keys.
  ``Resampler``                     AnyEdit_Collection/other_modules/ip_adapter/resampler.py:81-147 (perceiver attention of 16
                                    latent queries over [image tokens ; latents], FeedForward, proj_out + LayerNorm).
  ``ImageProjModel``                ip_adapter/ip_adapter.py:28-46.

The arithmetic of the two CLIP towers lives in a third-party dependency of the reference (``transformers``, unpinned in
requirements.txt; 5.5 is what this image has): the golden vectors are generated from that library's own modules with seeded
weights (tests/golden/make_golden_encoders.py).  Execution: LayerNorm kernel, wgmma contractions with bias / QuickGELU /
GELU / residual fused in the epilogue, the wgmma attention kernel for the vision tower and the Resampler, the short-sequence
causal attention kernel for the 77 text tokens.  Tokenisation (vocabulary files) is outside the path: the text tower takes
token ids (or a caller-supplied tokenizer).  No eager-PyTorch math, no CPU fallback.
"""
import types

import torch
import torch.nn as nn

from . import ops
from .unet import _Param, _f, _h

_ACT = {"quick_gelu": 4, "gelu": 3, "gelu_new": None}


def _cfg(config, **defaults):
    ns = types.SimpleNamespace(**defaults)
    src = config if isinstance(config, dict) else {k: getattr(config, k) for k in dir(config) if not k.startswith("_")}
    for k in defaults:
        if k in src and src[k] is not None:
            setattr(ns, k, src[k])
    return ns


class _Attn(nn.Module):
    def __init__(self, d):
        super().__init__()
        self.k_proj, self.v_proj, self.q_proj, self.out_proj = (_Param((d, d)) for _ in range(4))


class _MLP(nn.Module):
    def __init__(self, d, inner):
        super().__init__()
        self.fc1, self.fc2 = _Param((inner, d)), _Param((d, inner))


class _Layer(nn.Module):
    """CLIPEncoderLayer parameter holder (transformers modeling_clip.py)."""

    def __init__(self, d, inner):
        super().__init__()
        self.self_attn = _Attn(d)
        self.layer_norm1 = _Param((d,), kind="norm")
        self.mlp = _MLP(d, inner)
        self.layer_norm2 = _Param((d,), kind="norm")


class _Encoder(nn.Module):
    def __init__(self, d, inner, n_layers):
        super().__init__()
        self.layers = nn.ModuleList([_Layer(d, inner) for _ in range(n_layers)])


class _Emb(nn.Module):
    def __init__(self, *shape):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(*shape) * 0.02)


def _pack_layers(layers, dev):
    out = []
    for L in layers:
        a = L.self_attn
        out.append({"ln1": (_f(L.layer_norm1.weight, dev), _f(L.layer_norm1.bias, dev)),
                    "ln2": (_f(L.layer_norm2.weight, dev), _f(L.layer_norm2.bias, dev)),
                    "qkv_w": _h(torch.cat([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], 0), dev),
                    "qkv_b": _f(torch.cat([a.q_proj.bias, a.k_proj.bias, a.v_proj.bias], 0), dev),
                    "o_w": _h(a.out_proj.weight, dev), "o_b": _f(a.out_proj.bias, dev),
                    "fc1_w": _h(L.mlp.fc1.weight, dev), "fc1_b": _f(L.mlp.fc1.bias, dev),
                    "fc2_w": _h(L.mlp.fc2.weight, dev), "fc2_b": _f(L.mlp.fc2.bias, dev)})
    return out


def _run_layers(packed, h, B, n, heads, act, eps, causal, keep_hidden=False, n_run=None):
    """CLIPEncoder.forward: pre-LN residual blocks on the token matrix h [B*n, D] fp16.  Returns (h, [hidden states])."""
    M, D = h.shape
    d = D // heads
    dev = h.device
    hidden = [h] if keep_hidden else None
    for L in packed[: (len(packed) if n_run is None else n_run)]:
        ln = torch.empty_like(h)
        ops.layernorm(h, L["ln1"][0], L["ln1"][1], ln, eps)
        qkv = torch.empty(M, 3 * D, dtype=torch.float16, device=dev)
        ops.gemm(ln, L["qkv_w"], qkv, bias=L["qkv_b"])
        a = torch.empty(M, D, dtype=torch.float16, device=dev)
        if causal or n <= 128 or d % 16 != 0 or d > 160:
            ops.attention_small(qkv, qkv[:, D:], qkv[:, 2 * D:], a, B, heads, n, n, d, 3 * D, 3 * D, 3 * D, D, causal=causal)
        else:
            ops.attention(qkv, qkv[:, D:], qkv[:, 2 * D:], a, B, heads, n, n, d, 3 * D, 3 * D, 3 * D, D)
        h2 = torch.empty_like(h)
        ops.gemm(a, L["o_w"], h2, bias=L["o_b"], residual=h)
        ln2 = torch.empty_like(h)
        ops.layernorm(h2, L["ln2"][0], L["ln2"][1], ln2, eps)
        f1 = torch.empty(M, L["fc1_w"].shape[0], dtype=torch.float16, device=dev)
        ops.gemm(ln2, L["fc1_w"], f1, bias=L["fc1_b"], act=act)
        h = torch.empty_like(h2)
        ops.gemm(f1, L["fc2_w"], h, bias=L["fc2_b"], residual=h2)
        if keep_hidden:
            hidden.append(h)
    return h, hidden


class _Packable(nn.Module):
    def __init__(self):
        super().__init__()
        self._pack, self._pack_key, self._epoch = None, None, 0

    def invalidate(self):
        self._pack = None
        self._epoch += 1

    def _packed(self):
        ps = list(self.parameters())
        dev = ps[0].device
        key = (str(dev), sum(p._version for p in ps), self._epoch)
        if self._pack is None or self._pack_key != key:
            if dev.type != "cuda":
                raise RuntimeError(f"anyedit_b200.encoders.{type(self).__name__} runs on CUDA only (no CPU fallback); call .cuda() first")
            self._pack, self._pack_key = self._build_pack(dev), key
        return self._pack


# ---- CLIP text tower -------------------------------------------------------------------------------------------------------
class _TextTransformer(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.embeddings = nn.Module()
        self.embeddings.token_embedding = _Emb(c.vocab_size, c.hidden_size)
        self.embeddings.position_embedding = _Emb(c.max_position_embeddings, c.hidden_size)
        self.encoder = _Encoder(c.hidden_size, c.intermediate_size, c.num_hidden_layers)
        self.final_layer_norm = _Param((c.hidden_size,), kind="norm")


class CLIPTextModel(_Packable):
    """``transformers.CLIPTextModel`` (modeling_clip.py): ``forward(input_ids, output_hidden_states=False)`` ->
    namespace(last_hidden_state, pooler_output, hidden_states)."""

    def __init__(self, config):
        super().__init__()
        self.config = c = _cfg(config, vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=12,
                               num_attention_heads=12, max_position_embeddings=77, hidden_act="quick_gelu", layer_norm_eps=1e-5,
                               eos_token_id=2)
        if _ACT.get(c.hidden_act) is None:
            raise NotImplementedError(f"hidden_act={c.hidden_act!r}: CLIP uses quick_gelu or gelu")
        self.text_model = _TextTransformer(c)

    def _build_pack(self, dev):
        t = self.text_model
        return {"tok": _h(t.embeddings.token_embedding.weight, dev), "pos": _h(t.embeddings.position_embedding.weight, dev),
                "layers": _pack_layers(t.encoder.layers, dev),
                "final": (_f(t.final_layer_norm.weight, dev), _f(t.final_layer_norm.bias, dev))}

    @torch.no_grad()
    def forward(self, input_ids, output_hidden_states=False, **kwargs):
        P, c = self._packed(), self.config
        ids = input_ids.to(device=P["tok"].device, dtype=torch.int64).contiguous()
        B, n = ids.shape
        h = torch.empty(B * n, c.hidden_size, dtype=torch.float16, device=ids.device)
        ops.embed_tokens(ids, P["tok"], P["pos"], h)
        h, hidden = _run_layers(P["layers"], h, B, n, c.num_attention_heads, _ACT[c.hidden_act], c.layer_norm_eps, causal=True,
                                keep_hidden=output_hidden_states)
        last = torch.empty_like(h)
        ops.layernorm(h, P["final"][0], P["final"][1], last, c.layer_norm_eps)
        last = last.view(B, n, -1).float()
        # pooled = the features at the end-of-text token (modeling_clip.py: argmax of the ids for the legacy eos id 2)
        if c.eos_token_id == 2:
            pos = ids.argmax(dim=-1)
        else:
            pos = (ids == c.eos_token_id).int().argmax(dim=-1)
        pooled = last[torch.arange(B, device=ids.device), pos]
        hs = tuple(t.view(B, n, -1).float() for t in hidden) if output_hidden_states else None
        return types.SimpleNamespace(last_hidden_state=last, pooler_output=pooled, hidden_states=hs)


class FrozenCLIPEmbedder(nn.Module):
    """ldm/modules/encoders/modules.py:107-150.  ``version`` may be a ``transformers`` config (or dict) of the text tower --
    there is no hub access here, weights come through ``load_state_dict`` -- and ``tokenizer`` any callable with the
    ``CLIPTokenizer`` call signature; ``forward`` also takes ready token ids [B, max_length]."""
    LAYERS = ["last", "pooled", "hidden"]

    def __init__(self, version=None, device="cuda", max_length=77, freeze=True, layer="last", layer_idx=None, tokenizer=None):
        super().__init__()
        assert layer in self.LAYERS
        self.tokenizer = tokenizer
        self.transformer = CLIPTextModel(version if version is not None and not isinstance(version, str) else {})
        self.device, self.max_length, self.layer, self.layer_idx = device, max_length, layer, layer_idx
        if layer == "hidden":
            assert layer_idx is not None
            assert 0 <= abs(layer_idx) <= 12
        if freeze:
            self.freeze()

    def freeze(self):
        self.transformer = self.transformer.eval()
        for p in self.parameters():
            p.requires_grad = False

    def forward(self, text):
        if isinstance(text, torch.Tensor):
            tokens = text
        else:
            if self.tokenizer is None:
                raise RuntimeError("FrozenCLIPEmbedder: pass token ids, or construct it with tokenizer= (no vocabulary files in this build)")
            enc = self.tokenizer(text, truncation=True, max_length=self.max_length, return_length=True,
                                 return_overflowing_tokens=False, padding="max_length", return_tensors="pt")
            tokens = enc["input_ids"]
        out = self.transformer(input_ids=tokens.to(self.device), output_hidden_states=self.layer == "hidden")
        if self.layer == "last":
            return out.last_hidden_state
        if self.layer == "pooled":
            return out.pooler_output[:, None, :]
        return out.hidden_states[self.layer_idx]

    def encode(self, text):
        return self(text)


# ---- CLIP vision tower -----------------------------------------------------------------------------------------------------
class _VisionEmbeddings(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.class_embedding = nn.Parameter(torch.randn(c.hidden_size) * 0.02)
        self.patch_embedding = _Param((c.hidden_size, c.num_channels, c.patch_size, c.patch_size), bias=False, kind="conv")
        self.position_embedding = _Emb((c.image_size // c.patch_size) ** 2 + 1, c.hidden_size)


class _VisionTransformer(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.embeddings = _VisionEmbeddings(c)
        self.pre_layrnorm = _Param((c.hidden_size,), kind="norm")          # (sic) transformers' spelling
        self.encoder = _Encoder(c.hidden_size, c.intermediate_size, c.num_hidden_layers)
        self.post_layernorm = _Param((c.hidden_size,), kind="norm")


class CLIPVisionModelWithProjection(_Packable):
    """``transformers.CLIPVisionModelWithProjection``: ``forward(pixel_values, output_hidden_states=False)`` ->
    namespace(image_embeds, last_hidden_state, hidden_states).  train.py:688-691 consumes ``hidden_states[-2]``."""

    def __init__(self, config):
        super().__init__()
        self.config = c = _cfg(config, hidden_size=1280, intermediate_size=5120, num_hidden_layers=32, num_attention_heads=16,
                               image_size=224, patch_size=14, num_channels=3, projection_dim=1024, hidden_act="gelu", layer_norm_eps=1e-5)
        if _ACT.get(c.hidden_act) is None:
            raise NotImplementedError(f"hidden_act={c.hidden_act!r}: CLIP uses quick_gelu or gelu")
        self.vision_model = _VisionTransformer(c)
        self.visual_projection = _Param((c.projection_dim, c.hidden_size), bias=False)

    def _build_pack(self, dev):
        v, c = self.vision_model, self.config
        k = c.num_channels * c.patch_size ** 2
        kp = (k + 7) // 8 * 8
        w = torch.zeros(c.hidden_size, kp, device=dev)
        w[:, :k] = v.embeddings.patch_embedding.weight.detach().to(dev).float().reshape(c.hidden_size, k)
        pos = v.embeddings.position_embedding.weight.detach().to(dev).float()
        return {"patch_w": w.to(torch.float16).contiguous(), "kp": kp, "pos_patches": pos[1:].to(torch.float16).contiguous(),
                "cls": (v.embeddings.class_embedding.detach().to(dev).float() + pos[0]).to(torch.float16).contiguous(),
                "pre": (_f(v.pre_layrnorm.weight, dev), _f(v.pre_layrnorm.bias, dev)),
                "post": (_f(v.post_layernorm.weight, dev), _f(v.post_layernorm.bias, dev)),
                "layers": _pack_layers(v.encoder.layers, dev), "proj_w": _h(self.visual_projection.weight, dev)}

    @torch.no_grad()
    def forward(self, pixel_values, output_hidden_states=False, **kwargs):
        P, c = self._packed(), self.config
        dev = P["patch_w"].device
        x = pixel_values.to(dev)
        B, Cc, H, W = x.shape
        p = c.patch_size
        gh, gw = H // p, W // p
        npatch = gh * gw
        assert npatch + 1 == self.vision_model.embeddings.position_embedding.weight.shape[0], "image size does not match the position table"
        # non-overlapping patches -> rows (a pure permutation), zero-padded to a multiple of 8 columns, fp16
        patches = torch.zeros(B * npatch, P["kp"], dtype=torch.float16, device=dev)
        patches[:, : Cc * p * p].copy_(x.reshape(B, Cc, gh, p, gw, p).permute(0, 2, 4, 1, 3, 5).reshape(B * npatch, Cc * p * p))
        D = c.hidden_size
        emb = torch.empty(B * npatch, D, dtype=torch.float16, device=dev)
        ops.gemm(patches, P["patch_w"], emb, residual=P["pos_patches"].repeat(B, 1))      # patch conv + position embedding
        n = npatch + 1
        tok = torch.empty(B, n, D, dtype=torch.float16, device=dev)
        tok[:, 0].copy_(P["cls"])
        tok[:, 1:].copy_(emb.view(B, npatch, D))
        h = torch.empty(B * n, D, dtype=torch.float16, device=dev)
        ops.layernorm(tok.view(B * n, D), P["pre"][0], P["pre"][1], h, c.layer_norm_eps)
        h, hidden = _run_layers(P["layers"], h, B, n, c.num_attention_heads, _ACT[c.hidden_act], c.layer_norm_eps, causal=False,
                                keep_hidden=output_hidden_states)
        pooled = torch.empty(B, D, dtype=torch.float16, device=dev)
        ops.layernorm(h.view(B, n, D)[:, 0].contiguous(), P["post"][0], P["post"][1], pooled, c.layer_norm_eps)
        embeds = torch.empty(B, P["proj_w"].shape[0], dtype=torch.float32, device=dev)
        ops.gemm(pooled, P["proj_w"], embeds)
        hs = tuple(t.view(B, n, D).float() for t in hidden) if output_hidden_states else None
        return types.SimpleNamespace(image_embeds=embeds, last_hidden_state=h.view(B, n, D).float(), hidden_states=hs)


# ---- IP-Adapter projectors ---------------------------------------------------------------------------------------------------
class _Perceiver(nn.Module):
    def __init__(self, dim, dim_head, heads):
        super().__init__()
        inner = dim_head * heads
        self.dim_head, self.heads = dim_head, heads
        self.norm1, self.norm2 = _Param((dim,), kind="norm"), _Param((dim,), kind="norm")
        self.to_q, self.to_kv, self.to_out = _Param((inner, dim), bias=False), _Param((2 * inner, dim), bias=False), _Param((dim, inner), bias=False)


class Resampler(_Packable):
    """ip_adapter/resampler.py:81-147 (``apply_pos_emb`` / ``num_latents_mean_pooled`` unused by the reference's callers: raise)."""

    def __init__(self, dim=1024, depth=8, dim_head=64, heads=16, num_queries=8, embedding_dim=768, output_dim=1024, ff_mult=4,
                 max_seq_len=257, apply_pos_emb=False, num_latents_mean_pooled=0):
        super().__init__()
        if apply_pos_emb or num_latents_mean_pooled:
            raise NotImplementedError("Resampler: apply_pos_emb / num_latents_mean_pooled are not used on the AnySD path")
        self.dim, self.heads, self.dim_head, self.num_queries = dim, heads, dim_head, num_queries
        self.latents = nn.Parameter(torch.randn(1, num_queries, dim) / dim ** 0.5)
        self.proj_in, self.proj_out = _Param((dim, embedding_dim)), _Param((output_dim, dim))
        self.norm_out = _Param((output_dim,), kind="norm")
        inner = int(dim * ff_mult)
        self.layers = nn.ModuleList([nn.ModuleList([
            _Perceiver(dim, dim_head, heads),
            nn.Sequential(_Param((dim,), kind="norm"), _Param((inner, dim), bias=False), nn.Identity(), _Param((dim, inner), bias=False))])
            for _ in range(depth)])

    def _build_pack(self, dev):
        lay = []
        for attn, ff in self.layers:
            lay.append({"n1": (_f(attn.norm1.weight, dev), _f(attn.norm1.bias, dev)), "n2": (_f(attn.norm2.weight, dev), _f(attn.norm2.bias, dev)),
                        "q_w": _h(attn.to_q.weight, dev), "kv_w": _h(attn.to_kv.weight, dev), "o_w": _h(attn.to_out.weight, dev),
                        "ff_n": (_f(ff[0].weight, dev), _f(ff[0].bias, dev)), "ff1_w": _h(ff[1].weight, dev), "ff2_w": _h(ff[3].weight, dev)})
        return {"latents": _h(self.latents[0], dev), "pin": (_h(self.proj_in.weight, dev), _f(self.proj_in.bias, dev)),
                "pout": (_h(self.proj_out.weight, dev), _f(self.proj_out.bias, dev)),
                "nout": (_f(self.norm_out.weight, dev), _f(self.norm_out.bias, dev)), "layers": lay}

    @torch.no_grad()
    def forward(self, x):
        P = self._packed()
        dev = P["latents"].device
        B, n1, E = x.shape
        nq, D, H, dh = self.num_queries, self.dim, self.heads, self.dim_head
        inner = H * dh
        x16 = torch.empty(B * n1, E, dtype=torch.float16, device=dev)
        ops.cast_f16(x.to(dev).float().contiguous(), x16)
        xp = torch.empty(B * n1, D, dtype=torch.float16, device=dev)
        ops.gemm(x16, P["pin"][0], xp, bias=P["pin"][1])
        lat = P["latents"].repeat(B, 1).contiguous()                          # [B*nq, D]
        nkv = n1 + nq
        for L in P["layers"]:
            kv_in = torch.empty(B, nkv, D, dtype=torch.float16, device=dev)   # cat(norm1(x), norm2(latents)) along the tokens
            xn = torch.empty_like(xp)
            ops.layernorm(xp, L["n1"][0], L["n1"][1], xn)
            ln = torch.empty_like(lat)
            ops.layernorm(lat, L["n2"][0], L["n2"][1], ln)
            kv_in[:, :n1].copy_(xn.view(B, n1, D))
            kv_in[:, n1:].copy_(ln.view(B, nq, D))
            q = torch.empty(B * nq, inner, dtype=torch.float16, device=dev)
            ops.gemm(ln, L["q_w"], q)
            kv = torch.empty(B * nkv, 2 * inner, dtype=torch.float16, device=dev)
            ops.gemm(kv_in.view(B * nkv, D), L["kv_w"], kv)
            a = torch.empty(B * nq, inner, dtype=torch.float16, device=dev)
            if dh % 16 == 0 and dh <= 160:
                ops.attention(q, kv, kv[:, inner:], a, B, H, nq, nkv, dh, inner, 2 * inner, 2 * inner, inner)
            else:
                ops.attention_small(q, kv, kv[:, inner:], a, B, H, nq, nkv, dh, inner, 2 * inner, 2 * inner, inner)
            lat2 = torch.empty_like(lat)
            ops.gemm(a, L["o_w"], lat2, residual=lat)
            fn = torch.empty_like(lat2)
            ops.layernorm(lat2, L["ff_n"][0], L["ff_n"][1], fn)
            f1 = torch.empty(B * nq, L["ff1_w"].shape[0], dtype=torch.float16, device=dev)
            ops.gemm(fn, L["ff1_w"], f1, act=3)
            lat = torch.empty_like(lat2)
            ops.gemm(f1, L["ff2_w"], lat, residual=lat2)
        out = torch.empty(B * nq, P["pout"][0].shape[0], dtype=torch.float16, device=dev)
        ops.gemm(lat, P["pout"][0], out, bias=P["pout"][1])
        y = torch.empty_like(out)
        ops.layernorm(out, P["nout"][0], P["nout"][1], y)
        return y.view(B, nq, -1).float()


class ImageProjModel(_Packable):
    """ip_adapter/ip_adapter.py:28-46: Linear(clip_embeddings_dim -> tokens * cross_attention_dim), reshape, LayerNorm."""

    def __init__(self, cross_attention_dim=1024, clip_embeddings_dim=1024, clip_extra_context_tokens=4):
        super().__init__()
        self.generator = None
        self.cross_attention_dim, self.clip_extra_context_tokens = cross_attention_dim, clip_extra_context_tokens
        self.proj = _Param((clip_extra_context_tokens * cross_attention_dim, clip_embeddings_dim))
        self.norm = _Param((cross_attention_dim,), kind="norm")

    def _build_pack(self, dev):
        return {"w": _h(self.proj.weight, dev), "b": _f(self.proj.bias, dev), "n": (_f(self.norm.weight, dev), _f(self.norm.bias, dev))}

    @torch.no_grad()
    def forward(self, image_embeds):
        P = self._packed()
        dev = P["w"].device
        B = image_embeds.shape[0]
        e16 = torch.empty(B, image_embeds.shape[1], dtype=torch.float16, device=dev)
        ops.cast_f16(image_embeds.to(dev).float().contiguous(), e16)
        t = torch.empty(B, P["w"].shape[0], dtype=torch.float16, device=dev)
        ops.gemm(e16, P["w"], t, bias=P["b"])
        y = torch.empty_like(t)
        ops.layernorm(t.view(B * self.clip_extra_context_tokens, -1), P["n"][0], P["n"][1], y.view(B * self.clip_extra_context_tokens, -1))
        return y.view(B, self.clip_extra_context_tokens, self.cross_attention_dim).float()
