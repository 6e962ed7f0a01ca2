"""Condition encoders on the H100 kernels (SURVEY.md 8f rank 2): what produces ``c_crossattn`` and the visual tokens right
before the denoising loop.

  ``FrozenCLIPEmbedder``            ldm/modules/encoders/modules.py:107-150 -- the CLIP text tower the ``ldm`` stack conditions on
                                    (``transformers.CLIPTextModel``: token + position embeddings, 12 pre-LN layers with a causal
                                    mask and QuickGELU, final LayerNorm); ``layer`` = "last" | "pooled" | "hidden".
  ``CLIPTextModel``                 the tower itself, ``transformers`` state-dict keys (``text_model.*``).
  ``CLIPVisionModelWithProjection`` the CLIP-H vision tower of train.py:688-691 (``image_encoder(..., output_hidden_states=True)
                                    .hidden_states[-2]``): patch embedding as one contraction, class token, pre-LN, 32 layers
                                    (GELU), ``vision_model.*`` / ``visual_projection`` keys.
  ``CLIPModel``                     ``transformers.CLIPModel`` (both towers, both projection heads, ``logit_scale``): the CLIP-H
                                    scorer of AnyEdit_Collection/filter_tool/utils.py; ``openai_clip_to_transformers`` maps
                                    OpenAI's ``clip.load`` layout (the ViT-B/32 of the directional score) onto it.
  ``Resampler``                     AnyEdit_Collection/other_modules/ip_adapter/resampler.py:81-147 (perceiver attention of 16
                                    latent queries over [image tokens ; latents], FeedForward, proj_out + LayerNorm).
  ``ImageProjModel``                ip_adapter/ip_adapter.py:28-46.
  ``FrozenDinoV2Encoder``           ldm/modules/encoders/modules.py:279-315, AnyDoor's ``cond_stage_model``: ImageNet normalisation
                                    (folded into the patch embedding), DINOv2 ViT-g/14 (``Dinov2Model``: 40 pre-LN blocks, SwiGLU
                                    MLP and LayerScale in the contraction epilogues, hub key names), Linear(1536, 1024) projector.

The arithmetic of the two CLIP towers lives in a third-party dependency of the reference (``transformers``, unpinned in
requirements.txt; 5.5 is what this image has): the golden vectors are generated from that library's own modules with seeded
weights (tests/golden/make_golden_encoders.py).  Execution: LayerNorm kernel, wgmma contractions with bias / QuickGELU /
GELU / residual fused in the epilogue, the wgmma attention kernel for the vision tower and the Resampler, the short-sequence
causal attention kernel for the 77 text tokens.  Tokenisation (vocabulary files) is outside the path: the text tower takes
token ids (or a caller-supplied tokenizer).  No eager-PyTorch math, no CPU fallback.
"""
import re
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
    """CLIPEncoder.forward: pre-LN residual blocks on the token matrix h [B*n, D] fp16.  Returns (h, [hidden states]).
    A layer with "ls1" / "ls2" (fp32 [D]) scales its attention / MLP branch by them (LayerScale) in the epilogue that adds
    the residual; act 5 (SwiGLU) halves the width of the first MLP contraction (the DINOv2 blocks)."""
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
        ops.gemm(a, L["o_w"], h2, bias=L["o_b"], residual=h, col_scale=L.get("ls1"))
        ln2 = torch.empty_like(h)
        ops.layernorm(h2, L["ln2"][0], L["ln2"][1], ln2, eps)
        f1 = torch.empty(M, L["fc1_w"].shape[0] // (2 if act == 5 else 1), dtype=torch.float16, device=dev)
        ops.gemm(ln2, L["fc1_w"], f1, bias=L["fc1_b"], act=act)
        h = torch.empty_like(h2)
        ops.gemm(f1, L["fc2_w"], h, bias=L["fc2_b"], residual=h2, col_scale=L.get("ls2"))
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


def _text_pack(t, dev):
    return {"tok": _h(t.embeddings.token_embedding.weight, dev), "pos": _h(t.embeddings.position_embedding.weight, dev),
            "layers": _pack_layers(t.encoder.layers, dev),
            "final": (_f(t.final_layer_norm.weight, dev), _f(t.final_layer_norm.bias, dev))}


def _text_forward(P, c, input_ids, keep_hidden=False):
    """The text tower -> (final LayerNorm fp16 [B * n, D], end-of-text positions [B], ids, hidden states)."""
    ids = input_ids.to(device=P["tok"].device, dtype=torch.int64).contiguous()
    B, n = ids.shape
    h = torch.empty(B * n, c.hidden_size, dtype=torch.float16, device=ids.device)
    ops.embed_tokens(ids, P["tok"], P["pos"], h)
    h, hidden = _run_layers(P["layers"], h, B, n, c.num_attention_heads, _ACT[c.hidden_act], c.layer_norm_eps, causal=True,
                            keep_hidden=keep_hidden)
    last = torch.empty_like(h)
    ops.layernorm(h, P["final"][0], P["final"][1], last, c.layer_norm_eps)
    # pooled = the features at the end-of-text token (modeling_clip.py: argmax of the ids for the legacy eos id 2)
    if c.eos_token_id == 2:
        pos = ids.argmax(dim=-1)
    else:
        pos = (ids == c.eos_token_id).int().argmax(dim=-1)
    return last, pos, ids, hidden


_TEXT_DEFAULTS = dict(vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=12, num_attention_heads=12,
                      max_position_embeddings=77, hidden_act="quick_gelu", layer_norm_eps=1e-5, eos_token_id=2)
_VISION_DEFAULTS = dict(hidden_size=1280, intermediate_size=5120, num_hidden_layers=32, num_attention_heads=16, image_size=224,
                        patch_size=14, num_channels=3, projection_dim=1024, hidden_act="gelu", layer_norm_eps=1e-5)


def _check_act(c):
    if _ACT.get(c.hidden_act) is None:
        raise NotImplementedError(f"hidden_act={c.hidden_act!r}: CLIP uses quick_gelu or gelu")
    return c


class CLIPTextModel(_Packable):
    """``transformers.CLIPTextModel`` (modeling_clip.py): ``forward(input_ids, output_hidden_states=False)`` ->
    namespace(last_hidden_state, pooler_output, hidden_states)."""

    def __init__(self, config):
        super().__init__()
        self.config = c = _check_act(_cfg(config, **_TEXT_DEFAULTS))
        self.text_model = _TextTransformer(c)

    def _build_pack(self, dev):
        return _text_pack(self.text_model, dev)

    @torch.no_grad()
    def forward(self, input_ids, output_hidden_states=False, **kwargs):
        P, c = self._packed(), self.config
        last, pos, ids, hidden = _text_forward(P, c, input_ids, output_hidden_states)
        B, n = ids.shape
        last = last.view(B, n, -1).float()
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


def _vision_pack(v, c, dev):
    k = c.num_channels * c.patch_size ** 2
    kp = (k + 7) // 8 * 8
    w = torch.zeros(c.hidden_size, kp, device=dev)
    w[:, :k] = v.embeddings.patch_embedding.weight.detach().to(dev).float().reshape(c.hidden_size, k)
    pos = v.embeddings.position_embedding.weight.detach().to(dev).float()
    return {"patch_w": w.to(torch.float16).contiguous(), "kp": kp, "pos_patches": pos[1:].to(torch.float16).contiguous(),
            "cls": (v.embeddings.class_embedding.detach().to(dev).float() + pos[0]).to(torch.float16).contiguous(),
            "pre": (_f(v.pre_layrnorm.weight, dev), _f(v.pre_layrnorm.bias, dev)),
            "post": (_f(v.post_layernorm.weight, dev), _f(v.post_layernorm.bias, dev)),
            "layers": _pack_layers(v.encoder.layers, dev)}


def _patch_rows(P, c, pixel_values, npos):
    """pixel_values [B, C, H, W] -> fp16 patch rows [B * patches, kp] (a pure permutation, zero-padded to kp columns)."""
    dev = P["patch_w"].device
    x = pixel_values.to(dev)
    B, Cc, H, W = x.shape
    p = c.patch_size
    gh, gw = H // p, W // p
    assert gh * gw + 1 == npos, "image size does not match the position table"
    patches = torch.zeros(B * gh * gw, P["kp"], dtype=torch.float16, device=dev)
    patches[:, : Cc * p * p].copy_(x.reshape(B, Cc, gh, p, gw, p).permute(0, 2, 4, 1, 3, 5).reshape(B * gh * gw, Cc * p * p))
    return patches


def _vision_forward(P, c, patches, keep_hidden=False):
    """The vision tower from its patch rows [B * patches, kp] fp16 -> (tokens fp16 [B * n, D], post-LayerNorm class token fp16
    [B, D], hidden states, B, n)."""
    dev = P["patch_w"].device
    npatch = P["pos_patches"].shape[0]
    B = patches.shape[0] // npatch
    assert tuple(patches.shape) == (B * npatch, P["kp"]) and patches.dtype == torch.float16, "patch rows [B * patches, kp] fp16"
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
                            keep_hidden=keep_hidden)
    pooled = torch.empty(B, D, dtype=torch.float16, device=dev)
    ops.layernorm(h.view(B, n, D)[:, 0].contiguous(), P["post"][0], P["post"][1], pooled, c.layer_norm_eps)
    return h, pooled, hidden, B, n


def _project(x16, w):
    out = torch.empty(x16.shape[0], w.shape[0], dtype=torch.float32, device=x16.device)
    ops.gemm(x16, w, out)
    return out


class CLIPVisionModelWithProjection(_Packable):
    """``transformers.CLIPVisionModelWithProjection``: ``forward(pixel_values, output_hidden_states=False)`` ->
    namespace(image_embeds, last_hidden_state, hidden_states).  train.py:688-691 consumes ``hidden_states[-2]``."""

    def __init__(self, config):
        super().__init__()
        self.config = c = _check_act(_cfg(config, **_VISION_DEFAULTS))
        self.vision_model = _VisionTransformer(c)
        self.visual_projection = _Param((c.projection_dim, c.hidden_size), bias=False)

    def _build_pack(self, dev):
        P = _vision_pack(self.vision_model, self.config, dev)
        P["proj_w"] = _h(self.visual_projection.weight, dev)
        return P

    @torch.no_grad()
    def forward(self, pixel_values, output_hidden_states=False, **kwargs):
        P, c = self._packed(), self.config
        patches = _patch_rows(P, c, pixel_values, self.vision_model.embeddings.position_embedding.weight.shape[0])
        h, pooled, hidden, B, n = _vision_forward(P, c, patches, output_hidden_states)
        D = c.hidden_size
        embeds = _project(pooled, P["proj_w"])
        hs = tuple(t.view(B, n, D).float() for t in hidden) if output_hidden_states else None
        return types.SimpleNamespace(image_embeds=embeds, last_hidden_state=h.view(B, n, D).float(), hidden_states=hs)


class CLIPModel(_Packable):
    """``transformers.CLIPModel`` (modeling_clip.py) under its state-dict keys (``text_model.*``, ``vision_model.*``,
    ``visual_projection.weight``, ``text_projection.weight``, ``logit_scale``).  ``config``: dict or ``CLIPConfig`` with
    ``text_config`` / ``vision_config`` (dicts or configs) and ``projection_dim``.
    ``get_text_features(input_ids)`` / ``get_image_features(pixel_values)`` -> the projected, un-normalised fp32 embeddings;
    ``get_image_features(patch_rows=...)`` takes the fp16 patch rows of ``ops.clip_preprocess`` instead of pixels."""

    def __init__(self, config):
        super().__init__()
        c = _cfg(config, text_config={}, vision_config={}, projection_dim=512, logit_scale_init_value=2.6592)
        tc, vc = c.text_config, c.vision_config
        self.text_config = _check_act(_cfg(tc, **_TEXT_DEFAULTS))
        self.vision_config = _check_act(_cfg(vc, **_VISION_DEFAULTS))
        self.projection_dim = c.projection_dim
        self.text_model = _TextTransformer(self.text_config)
        self.vision_model = _VisionTransformer(self.vision_config)
        self.visual_projection = _Param((c.projection_dim, self.vision_config.hidden_size), bias=False)
        self.text_projection = _Param((c.projection_dim, self.text_config.hidden_size), bias=False)
        self.logit_scale = nn.Parameter(torch.tensor(float(c.logit_scale_init_value)))

    def _build_pack(self, dev):
        return {"text": _text_pack(self.text_model, dev), "vision": _vision_pack(self.vision_model, self.vision_config, dev),
                "vproj": _h(self.visual_projection.weight, dev), "tproj": _h(self.text_projection.weight, dev),
                "logit_scale": float(self.logit_scale.detach().float().cpu())}

    @property
    def patch_size(self):
        return self.vision_config.patch_size

    @torch.no_grad()
    def get_text_features(self, input_ids):
        P = self._packed()
        last, pos, ids, _ = _text_forward(P["text"], self.text_config, input_ids)
        B, n = ids.shape
        pooled = last.view(B, n, -1)[torch.arange(B, device=ids.device), pos].contiguous()
        return _project(pooled, P["tproj"])

    @torch.no_grad()
    def get_image_features(self, pixel_values=None, patch_rows=None):
        P = self._packed()
        if patch_rows is None:
            patch_rows = _patch_rows(P["vision"], self.vision_config, pixel_values,
                                     self.vision_model.embeddings.position_embedding.weight.shape[0])
        _, pooled, _, _, _ = _vision_forward(P["vision"], self.vision_config, patch_rows)
        return _project(pooled, P["vproj"])

    def logit_scale_value(self):
        return self._packed()["logit_scale"]


# OpenAI ``clip.load`` state dict <-> ``transformers.CLIPModel`` keys.  in_proj_* of every residual block is split into
# q / k / v; ``visual.proj`` and ``text_projection`` are stored transposed ([width, embed]).
_OA_TOP = (("visual.conv1.weight", "vision_model.embeddings.patch_embedding.weight"),
           ("visual.class_embedding", "vision_model.embeddings.class_embedding"),
           ("visual.positional_embedding", "vision_model.embeddings.position_embedding.weight"),
           ("visual.ln_pre.", "vision_model.pre_layrnorm."), ("visual.ln_post.", "vision_model.post_layernorm."),
           ("token_embedding.weight", "text_model.embeddings.token_embedding.weight"),
           ("positional_embedding", "text_model.embeddings.position_embedding.weight"),
           ("ln_final.", "text_model.final_layer_norm."), ("logit_scale", "logit_scale"))
_OA_BLOCK = (("ln_1.", "layer_norm1."), ("ln_2.", "layer_norm2."), ("attn.out_proj.", "self_attn.out_proj."),
             ("mlp.c_fc.", "mlp.fc1."), ("mlp.c_proj.", "mlp.fc2."))
_OA_TOWER = (("visual.transformer.resblocks.", "vision_model.encoder.layers."), ("transformer.resblocks.", "text_model.encoder.layers."))
_OA_META = ("input_resolution", "context_length", "vocab_size")      # integer attributes some checkpoints carry


def openai_clip_to_transformers(sd):
    """State dict of OpenAI's ``clip`` model (``clip.load(...)[0].state_dict()``) -> ``transformers.CLIPModel`` keys."""
    out = {}
    for k, v in sd.items():
        if k in _OA_META:
            continue
        if k == "visual.proj":
            out["visual_projection.weight"] = v.t().contiguous()
            continue
        if k == "text_projection":
            out["text_projection.weight"] = v.t().contiguous()
            continue
        for a, b in _OA_TOWER:
            m = re.fullmatch(re.escape(a) + r"(\d+)\.(.*)", k)
            if m:
                pre, rest = f"{b}{m.group(1)}.", m.group(2)
                if rest.startswith("attn.in_proj_"):
                    leaf = "weight" if rest.endswith("weight") else "bias"
                    for n, t in zip(("q_proj", "k_proj", "v_proj"), v.chunk(3, 0)):
                        out[f"{pre}self_attn.{n}.{leaf}"] = t.contiguous()
                else:
                    out[pre + _rename(rest, _OA_BLOCK, "CLIP")] = v
                break
        else:
            out[_rename(k, _OA_TOP, "CLIP")] = v
    return out


def transformers_to_openai_clip(sd):
    """Inverse of ``openai_clip_to_transformers``."""
    out = {}
    for k, v in sd.items():
        if k == "visual_projection.weight":
            out["visual.proj"] = v.t().contiguous()
            continue
        if k == "text_projection.weight":
            out["text_projection"] = v.t().contiguous()
            continue
        for a, b in _OA_TOWER:
            m = re.fullmatch(re.escape(b) + r"(\d+)\.(.*)", k)
            if m:
                pre, rest = f"{a}{m.group(1)}.", m.group(2)
                if rest.startswith("self_attn.q_proj."):
                    leaf = rest.rsplit(".", 1)[1]
                    base = f"{b}{m.group(1)}.self_attn."
                    out[f"{pre}attn.in_proj_{leaf}"] = torch.cat([sd[f"{base}{n}.{leaf}"] for n in ("q_proj", "k_proj", "v_proj")], 0)
                elif not rest.startswith(("self_attn.k_proj.", "self_attn.v_proj.")):
                    out[pre + _rename(rest, tuple((y, x) for x, y in _OA_BLOCK), "CLIP")] = v
                break
        else:
            out[_rename(k, tuple((y, x) for x, y in _OA_TOP), "CLIP")] = v
    return out


# ---- DINOv2 ViT-g/14: AnyDoor's reference-image encoder -------------------------------------------------------------------------
IMAGENET_MEAN, IMAGENET_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def dinov2_pos_table(pos_embed, gh, gw, interpolate_offset=0.1):
    """``DinoVisionTransformer.interpolate_pos_encoding``: the position table trained on an m x m grid ([1, 1 + m*m, D]) resized
    bicubically to gh x gw patches -> fp32 [1 + gh*gw, D] (class slot first).  Offset 0.1 is the published hub form
    (``scale_factor=((gh + 0.1) / m, (gw + 0.1) / m)``); 0.0 the ``size=(gh, gw)`` form of transformers' ``Dinov2Embeddings``.
    Both return the table unchanged on its own square grid."""
    pos = pos_embed.detach().float().cpu().reshape(-1, pos_embed.shape[-1])
    m = int(round((pos.shape[0] - 1) ** 0.5))
    assert m * m == pos.shape[0] - 1, "the position table must cover a square grid plus the class slot"
    if gh == m and gw == m:
        return pos
    grid = pos[1:].reshape(1, m, m, -1).permute(0, 3, 1, 2)
    if interpolate_offset:
        kw = {"scale_factor": ((gh + interpolate_offset) / m, (gw + interpolate_offset) / m)}
    else:
        kw = {"size": (gh, gw)}
    g = torch.nn.functional.interpolate(grid, mode="bicubic", align_corners=False, **kw)
    assert tuple(g.shape[-2:]) == (gh, gw)
    return torch.cat([pos[:1], g.permute(0, 2, 3, 1).reshape(gh * gw, -1)], 0)


# transformers ``Dinov2Model`` name -> hub name.  attention.attention.{query,key,value} are fused (rows q ; k ; v) into attn.qkv.
_HF_TOP = (("embeddings.cls_token", "cls_token"), ("embeddings.mask_token", "mask_token"),
           ("embeddings.position_embeddings", "pos_embed"), ("embeddings.patch_embeddings.projection.", "patch_embed.proj."),
           ("layernorm.", "norm."))
_HF_BLOCK = (("norm1.", "norm1."), ("attention.output.dense.", "attn.proj."), ("layer_scale1.lambda1", "ls1.gamma"),
             ("norm2.", "norm2."), ("mlp.weights_in.", "mlp.w12."), ("mlp.weights_out.", "mlp.w3."), ("layer_scale2.lambda1", "ls2.gamma"))
_QKV = ("query", "key", "value")


def _rename(k, table, what="DINOv2"):
    for a, b in table:
        if k.startswith(a):
            return b + k[len(a):]
    raise KeyError(f"no {what} key mapping for {k!r}")


def dinov2_from_transformers(sd):
    """State dict of transformers' ``Dinov2Model(use_swiglu_ffn=True)`` -> the hub names ``Dinov2Model`` here loads."""
    out = {}
    for k, v in sd.items():
        m = re.fullmatch(r"encoder\.layer\.(\d+)\.(.*)", k)
        if m is None:
            out[_rename(k, _HF_TOP)] = v
        elif m.group(2).startswith("attention.attention."):
            leaf = m.group(2).rsplit(".", 1)[1]
            if m.group(2).startswith("attention.attention.query."):
                pre = f"encoder.layer.{m.group(1)}.attention.attention."
                out[f"blocks.{m.group(1)}.attn.qkv.{leaf}"] = torch.cat([sd[f"{pre}{n}.{leaf}"] for n in _QKV], 0)
        else:
            out[f"blocks.{m.group(1)}.{_rename(m.group(2), _HF_BLOCK)}"] = v
    return out


def dinov2_to_transformers(sd):
    """Inverse of ``dinov2_from_transformers``."""
    out = {}
    for k, v in sd.items():
        m = re.fullmatch(r"blocks\.(\d+)\.(.*)", k)
        if m is None:
            out[_rename(k, tuple((b, a) for a, b in _HF_TOP))] = v
        elif m.group(2).startswith("attn.qkv."):
            leaf = m.group(2).rsplit(".", 1)[1]
            for n, t in zip(_QKV, v.chunk(3, 0)):
                out[f"encoder.layer.{m.group(1)}.attention.attention.{n}.{leaf}"] = t
        else:
            out[f"encoder.layer.{m.group(1)}.{_rename(m.group(2), tuple((b, a) for a, b in _HF_BLOCK))}"] = v
    return out


class _LayerScale(nn.Module):
    def __init__(self, d):
        super().__init__()
        self.gamma = nn.Parameter(torch.ones(d))


class _DinoBlock(nn.Module):
    """Hub ``NestedTensorBlock`` parameter holder: norm1, attn.{qkv, proj}, ls1, norm2, mlp, ls2; the MLP is
    ``mlp.{w12, w3}`` (SwiGLUFFNFused) or ``mlp.{fc1, fc2}`` (the GELU ``Mlp``)."""

    def __init__(self, d, hidden, swiglu=True):
        super().__init__()
        self.norm1 = _Param((d,), kind="norm")
        self.attn = nn.Module()
        self.attn.qkv, self.attn.proj = _Param((3 * d, d)), _Param((d, d))
        self.ls1 = _LayerScale(d)
        self.norm2 = _Param((d,), kind="norm")
        self.mlp = nn.Module()
        if swiglu:
            self.mlp.w12, self.mlp.w3 = _Param((2 * hidden, d)), _Param((d, hidden))
        else:
            self.mlp.fc1, self.mlp.fc2 = _Param((hidden, d)), _Param((d, hidden))
        self.ls2 = _LayerScale(d)


# ``depth_anything_v2/dinov2.py`` ``DINOv2(model_name)``: patch 14, a 518 x 518 position table, LayerScale, offset 0.1
DINOV2_CONFIGS = {
    "vits": dict(hidden_size=384, num_attention_heads=6, num_hidden_layers=12, use_swiglu_ffn=False),
    "vitb": dict(hidden_size=768, num_attention_heads=12, num_hidden_layers=12, use_swiglu_ffn=False),
    "vitl": dict(hidden_size=1024, num_attention_heads=16, num_hidden_layers=24, use_swiglu_ffn=False),
    "vitg": dict(hidden_size=1536, num_attention_heads=24, num_hidden_layers=40, use_swiglu_ffn=True),
}


class Dinov2Model(_Packable):
    """DINOv2 ``DinoVisionTransformer`` under the hub's parameter names, with the SwiGLU MLP (hub ``dinov2_vitg14``) or the GELU
    ``Mlp`` (``use_swiglu_ffn=False``: ViT-S/B/L, exact-erf GELU in the fc1 epilogue).
    ``config``: dict or transformers ``Dinov2Config`` (hidden_size, num_hidden_layers, num_attention_heads, mlp_ratio, image_size
    = the resolution of the position table, patch_size, layer_norm_eps, use_swiglu_ffn); the defaults are ViT-g/14; the
    configurations of ``DINOv2(model_name)`` are ``DINOV2_CONFIGS``.  ``interpolate_offset``: see ``dinov2_pos_table``.
    ``pixel_mean`` / ``pixel_std`` (per channel): an input normalisation folded into the packed patch embedding.
    ``forward_features(x)`` -> {"x_norm_clstoken": [B, D], "x_norm_patchtokens": [B, gh*gw, D]} fp32;
    ``get_intermediate_layers`` as the hub's."""

    def __init__(self, config=None, interpolate_offset=0.1, pixel_mean=None, pixel_std=None):
        super().__init__()
        self.config = c = _cfg(config if config is not None else {}, hidden_size=1536, num_hidden_layers=40, num_attention_heads=24,
                               mlp_ratio=4, image_size=518, patch_size=14, num_channels=3, layer_norm_eps=1e-6, use_swiglu_ffn=True)
        D, p = c.hidden_size, c.patch_size
        if c.use_swiglu_ffn:
            hidden = (int(int(D * c.mlp_ratio) * 2 / 3) + 7) // 8 * 8     # SwiGLUFFNFused: 6144 -> 4096 for ViT-g
        else:
            hidden = int(D * c.mlp_ratio)
        self._act = 5 if c.use_swiglu_ffn else 3
        m = c.image_size // p
        self.interpolate_offset, self.pixel_mean, self.pixel_std = interpolate_offset, pixel_mean, pixel_std
        self.cls_token = nn.Parameter(torch.zeros(1, 1, D))
        self.pos_embed = nn.Parameter(torch.randn(1, m * m + 1, D) * 0.02)
        self.mask_token = nn.Parameter(torch.zeros(1, D))           # masked pre-training only; loaded, never used
        self.patch_embed = nn.Module()
        self.patch_embed.proj = _Param((D, c.num_channels, p, p), kind="conv")
        self.blocks = nn.ModuleList([_DinoBlock(D, hidden, c.use_swiglu_ffn) for _ in range(c.num_hidden_layers)])
        self.norm = _Param((D,), kind="norm")

    def _build_pack(self, dev):
        c, D, p = self.config, self.config.hidden_size, self.config.patch_size
        k = c.num_channels * p * p
        kp = (k + 7) // 8 * 8
        w = self.patch_embed.proj.weight.detach().double().cpu().reshape(D, c.num_channels, p * p)
        b = self.patch_embed.proj.bias.detach().double().cpu()
        if self.pixel_mean is not None:              # conv((x - mean) / std) = conv with W / std, bias b - sum W mean / std
            mean = torch.tensor(self.pixel_mean, dtype=torch.float64)[None, :, None]
            std = torch.tensor(self.pixel_std, dtype=torch.float64)[None, :, None]
            b = b - (w * (mean / std)).sum((1, 2))
            w = w / std
        wp = torch.zeros(D, kp, dtype=torch.float64)
        wp[:, :k] = w.reshape(D, k)
        layers = []
        for L in self.blocks:
            if self._act == 5:
                w12, b12 = L.mlp.w12.weight, L.mlp.w12.bias
                hd = w12.shape[0] // 2
                # act 5 takes rows (a_j, gate_j); the hub computes silu(x1) * x2 with x1, x2 = w12(x).chunk(2): a = x2, gate = x1
                perm = torch.stack([torch.arange(hd, 2 * hd), torch.arange(hd)], 1).reshape(-1).to(w12.device)
                fc1_w, fc1_b, fc2 = w12[perm], b12[perm], L.mlp.w3
            else:
                fc1_w, fc1_b, fc2 = L.mlp.fc1.weight, L.mlp.fc1.bias, L.mlp.fc2
            layers.append({"ln1": (_f(L.norm1.weight, dev), _f(L.norm1.bias, dev)), "ln2": (_f(L.norm2.weight, dev), _f(L.norm2.bias, dev)),
                           "qkv_w": _h(L.attn.qkv.weight, dev), "qkv_b": _f(L.attn.qkv.bias, dev),
                           "o_w": _h(L.attn.proj.weight, dev), "o_b": _f(L.attn.proj.bias, dev), "ls1": _f(L.ls1.gamma, dev),
                           "fc1_w": _h(fc1_w, dev), "fc1_b": _f(fc1_b, dev),
                           "fc2_w": _h(fc2.weight, dev), "fc2_b": _f(fc2.bias, dev), "ls2": _f(L.ls2.gamma, dev)})
        return {"patch_w": _h(wp, dev), "patch_b": _f(b, dev), "kp": kp, "layers": layers,
                "norm": (_f(self.norm.weight, dev), _f(self.norm.bias, dev)), "pos": {}}

    def _pos(self, P, gh, gw):
        """(class token + its position, fp16 [D]; patch positions, fp16 [gh*gw, D]) for one grid, built once per pack."""
        if (gh, gw) not in P["pos"]:
            dev = P["patch_w"].device
            t = dinov2_pos_table(self.pos_embed, gh, gw, self.interpolate_offset).to(dev)
            cls = self.cls_token.detach().float().reshape(-1) + t[0]
            P["pos"][(gh, gw)] = (cls.half().contiguous(), t[1:].half().contiguous())
        return P["pos"][(gh, gw)]

    def _tokens(self, x):
        """-> (fp16 [B * (1 + gh*gw), D] = class token + patch embeddings + positions, class token first per image; B; gh; gw)."""
        P, c = self._packed(), self.config
        dev = P["patch_w"].device
        x = x.to(dev)
        B, Cc, H, W = x.shape
        p, D = c.patch_size, c.hidden_size
        assert Cc == c.num_channels and H % p == 0 and W % p == 0, f"expected [B, {c.num_channels}, H, W] with H, W multiples of {p}"
        gh, gw = H // p, W // p
        npatch, n = gh * gw, gh * gw + 1
        cls, pos = self._pos(P, gh, gw)
        # non-overlapping patches -> rows (a pure permutation), zero-padded to a multiple of 8 columns, fp16
        patches = torch.zeros(B * npatch, P["kp"], dtype=torch.float16, device=dev)
        patches[:, : Cc * p * p].copy_(x.reshape(B, Cc, gh, p, gw, p).permute(0, 2, 4, 1, 3, 5).reshape(B * npatch, Cc * p * p))
        emb = torch.empty(B * npatch, D, dtype=torch.float16, device=dev)
        ops.gemm(patches, P["patch_w"], emb, bias=P["patch_b"], residual=pos.repeat(B, 1))   # normalise + patch conv + position
        tok = torch.empty(B, n, D, dtype=torch.float16, device=dev)
        tok[:, 0].copy_(cls)
        tok[:, 1:].copy_(emb.view(B, npatch, D))
        return tok.view(B * n, D), B, gh, gw

    def normed_tokens(self, x):
        """-> (fp16 [B * (1 + gh*gw), D] = the final LayerNorm of every token, class token first per image; B; 1 + gh*gw)."""
        P, c = self._packed(), self.config
        tok, B, gh, gw = self._tokens(x)
        n = gh * gw + 1
        h, _ = _run_layers(P["layers"], tok, B, n, c.num_attention_heads, self._act, c.layer_norm_eps, causal=False)
        y = torch.empty_like(h)
        ops.layernorm(h, P["norm"][0], P["norm"][1], y, c.layer_norm_eps)
        return y, B, n

    def _block_outputs(self, x, blocks):
        """Run the blocks up to the last of ``blocks`` (indices into self.blocks) -> ([fp16 [B * n, D] output of each requested
        block], B, gh, gw)."""
        P, c = self._packed(), self.config
        blocks = [b % len(P["layers"]) for b in blocks]
        tok, B, gh, gw = self._tokens(x)
        _, hidden = _run_layers(P["layers"], tok, B, gh * gw + 1, c.num_attention_heads, self._act, c.layer_norm_eps, causal=False,
                                keep_hidden=True, n_run=max(blocks) + 1)
        return [hidden[b + 1] for b in blocks], B, gh, gw

    def intermediate_patches(self, x, blocks):
        """The depth head's input: for each block in ``blocks``, the final LayerNorm of its output on the PATCH rows only, densely
        packed fp16 [B * gh * gw, D] (an image's patch rows are contiguous, so each image is normalised straight into the buffer).
        -> (list, B, gh, gw)."""
        P, c = self._packed(), self.config
        outs, B, gh, gw = self._block_outputs(x, blocks)
        n, D = gh * gw + 1, c.hidden_size
        res = []
        for h in outs:
            y = torch.empty(B, n - 1, D, dtype=torch.float16, device=h.device)
            for b in range(B):
                ops.layernorm(h.view(B, n, D)[b, 1:], P["norm"][0], P["norm"][1], y[b], c.layer_norm_eps)
            res.append(y.view(B * (n - 1), D))
        return res, B, gh, gw

    @torch.no_grad()
    def get_intermediate_layers(self, x, n=1, reshape=False, return_class_token=False, norm=True):
        """``DinoVisionTransformer.get_intermediate_layers`` (depth_anything_v2/dinov2.py:271-321): ``n`` = the number of last
        blocks or a list of block indices; the blocks run only up to the last one requested.  fp32 outputs [B, gh*gw, D]
        ([B, D, gh, gw] with ``reshape``), paired with the class tokens [B, D] when ``return_class_token``."""
        L = len(self.blocks)
        blocks = list(range(L - n, L)) if isinstance(n, int) else list(n)
        outs, B, gh, gw = self._block_outputs(x, blocks)
        P, c = self._packed(), self.config
        res = []
        for h in outs:
            if norm:
                y = torch.empty_like(h)
                ops.layernorm(h, P["norm"][0], P["norm"][1], y, c.layer_norm_eps)
                h = y
            res.append(h.view(B, gh * gw + 1, -1).float())
        cls = [t[:, 0] for t in res]
        res = [t[:, 1:] for t in res]
        if reshape:
            res = [t.reshape(B, gh, gw, -1).permute(0, 3, 1, 2).contiguous() for t in res]
        return tuple(zip(res, cls)) if return_class_token else tuple(res)

    @torch.no_grad()
    def forward_features(self, x):
        y, B, n = self.normed_tokens(x)
        y = y.view(B, n, -1).float()
        return {"x_norm_clstoken": y[:, 0], "x_norm_patchtokens": y[:, 1:]}


class FrozenDinoV2Encoder(_Packable):
    """ldm/modules/encoders/modules.py:279-315: ImageNet normalisation, DINOv2 ViT-g/14 (``model.*``, hub names; weights
    through ``load_state_dict``), ``projector`` = Linear(1536, 1024) of cat(x_norm_clstoken, x_norm_patchtokens) -> fp32
    [B, 1 + patches, 1024].  ``config``: a smaller ``Dinov2Model`` config, plus ``interpolate_offset`` and ``projection_dim``."""

    def __init__(self, device="cuda", freeze=True, config=None):
        super().__init__()
        c = _cfg(config if config is not None else {}, interpolate_offset=0.1, projection_dim=1024)
        self.model = Dinov2Model(config, c.interpolate_offset, IMAGENET_MEAN, IMAGENET_STD)
        self.device = device
        if freeze:
            self.freeze()
        self.projector = _Param((c.projection_dim, self.model.config.hidden_size))

    def freeze(self):
        self.model.eval()
        for p in self.model.parameters():
            p.requires_grad = False

    def _build_pack(self, dev):
        return {"w": _h(self.projector.weight, dev), "b": _f(self.projector.bias, dev)}

    @torch.no_grad()
    def forward(self, image):
        if isinstance(image, list):
            image = torch.cat(image, 0)
        P = self._packed()
        y, B, n = self.model.normed_tokens(image)
        out = torch.empty(B * n, P["w"].shape[0], dtype=torch.float32, device=y.device)
        ops.gemm(y, P["w"], out, bias=P["b"])
        return out.view(B, n, -1)

    def encode(self, image):
        return self(image)


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
