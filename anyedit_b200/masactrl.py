"""AnyEdit's action-change edits on the kernels: MasaCtrl's mutual self-attention in the SD-1.5 UNet.

``action_change_tool.py:15-45`` renders a source and a target prompt from one shared start code, 50 DDIM steps with CFG,
with ``MutualSelfAttentionControl(5, 12)`` registered on the UNet: from denoising step 5 and transformer block 12 on, every
self-attention query of a CFG half attends to the keys and values of the FIRST sample of that half
(AnyEdit_Collection/other_modules/masactrl/masactrl.py:41-72).  Here that is a K/V batch map handed to the attention kernel
(``anysd_attention_kvmap_f16``): query batch b reads the K/V rows of batch ``map[b]``.  Nothing is computed on the host
but the map.

Names follow the reference (``masactrl.py`` / ``masactrl_utils.py``), so the tool runs with its imports changed:
``AttentionBase``, ``MutualSelfAttentionControl`` and ``regiter_attention_editor_ldm`` (the reference's spelling).  The
editors here are descriptions of the edit -- which (step, block) pairs are active -- not attention functions: the UNet
reads them once per forward.  ``action_pairs`` runs P source / target pairs in one sampler run.
"""
import numpy as np
import torch

from . import ops

# the reference's editor classes this module does not implement (masactrl.py, masactrl_utils.py)
_NOT_IMPLEMENTED = ("AttentionStore", "MutualSelfAttentionControlMask", "MutualSelfAttentionControlMaskAuto",
                    "MutualSelfAttentionControlUnion")


class AttentionBase:
    """masactrl_utils.py:14-40: the step / layer counters of an attention editor, and no edit.

    ``cur_step`` counts UNet forwards (one per sampler step); ``cur_att_layer`` is always 0 between forwards, which is the
    only time it can be read here; ``num_att_layers`` is set by ``regiter_attention_editor_ldm`` (2 per transformer
    block).  ``reset()`` starts the count again."""

    def __init__(self):
        self.cur_step = 0
        self.num_att_layers = -1
        self.cur_att_layer = 0
        self._kv_group = None            # rows per K/V group of a CFG half; None = the whole half (the reference's editor)

    def after_step(self):
        pass

    def reset(self):
        self.cur_step = 0
        self.cur_att_layer = 0

    def active_blocks(self, step):
        """Transformer blocks (forward order) whose self-attention is edited at denoising step ``step``: none."""
        return ()


class MutualSelfAttentionControl(AttentionBase):
    """masactrl.py:14-72.  Self-attention of transformer block l at step s is edited when ``s in step_idx`` and
    ``l in layer_idx`` (the reference's ``cur_att_layer // 2``: attn1 and attn2 of a block count as two layers).  The
    edit: every query row of a CFG half attends to the K/V of the first sample of that half."""
    MODEL_TYPE = {"SD": 16, "SDXL": 70}

    def __init__(self, start_step=4, start_layer=10, layer_idx=None, step_idx=None, total_steps=50, model_type="SD"):
        super().__init__()
        self.total_steps = total_steps
        self.total_layers = self.MODEL_TYPE.get(model_type, 16)
        self.start_step = start_step
        self.start_layer = start_layer
        self.layer_idx = layer_idx if layer_idx is not None else list(range(start_layer, self.total_layers))
        self.step_idx = step_idx if step_idx is not None else list(range(start_step, total_steps))

    def active_blocks(self, step):
        return tuple(self.layer_idx) if step in self.step_idx else ()


def check_editor(editor):
    """Refuse every editor whose edit this module cannot express as a K/V batch map."""
    t = type(editor)
    if t in (AttentionBase, MutualSelfAttentionControl):
        return
    if t.__name__ in _NOT_IMPLEMENTED:
        raise NotImplementedError(f"anyedit_b200.masactrl: the {t.__name__} attention editor is not implemented on the kernels "
                                  "(AttentionBase and MutualSelfAttentionControl are)")
    raise TypeError(f"anyedit_b200.masactrl: cannot register an editor of type {t.__module__}.{t.__qualname__}; use "
                    "anyedit_b200.masactrl.AttentionBase or MutualSelfAttentionControl (the attention runs in CUDA kernels, "
                    "not in the editor's forward)")


def kv_batch_map(N, group=None):
    """K/V row of every query row of a model batch of N rows, int32 [N].

    The batch is two CFG halves ``[uncond ; cond]`` (ldm ddim.py:190-210) and the reference splits it with ``chunk(2)``
    (masactrl.py:63-70): row b reads row 0 when b < N/2, else row N/2.  ``group`` g splits each half further into groups
    of g rows, each reading its first row: ``action_pairs`` orders a half as (s0, t0, s1, t1, ...) and uses g = 2,
    ``b -> b & ~1``.  Every map satisfies map[b + N/2] = map[b] + N/2, which is what lets the UNet run a shared CFG prefix
    on the first half of it."""
    N = int(N)
    if N < 2 or N % 2:
        raise ValueError(f"MasaCtrl splits the model batch into two CFG halves: it needs an even batch of at least 2 rows, got {N}")
    half = N // 2
    g = half if group is None else int(group)
    if g < 1 or half % g:
        raise ValueError(f"K/V groups of {g} rows do not tile a CFG half of {half} rows")
    m = (np.arange(N) // g) * g
    assert np.array_equal(m[half:], m[:half] + half)
    return m.astype(np.int32)


def kv_table(editor, blocks, N, step0, steps):
    """int32 [steps, blocks, N]: the K/V map of every transformer block at denoising steps step0 .. step0 + steps - 1.
    Inactive (step, block) pairs get the identity.  The batch is only checked when some pair is active."""
    table = np.broadcast_to(np.arange(N, dtype=np.int32), (steps, blocks, N)).copy()
    m = None
    for s in range(steps):
        for blk in editor.active_blocks(step0 + s):
            if 0 <= blk < blocks:
                if m is None:
                    m = kv_batch_map(N, editor._kv_group)
                table[s, blk] = m
    return table


def _diffusion_unet(model):
    from .unet import UNetModel
    unet = getattr(getattr(model, "model", None), "diffusion_model", None)
    if not isinstance(unet, UNetModel):
        raise TypeError("regiter_attention_editor_ldm: model.model.diffusion_model must be an anyedit_b200 UNetModel")
    return unet


def regiter_attention_editor_ldm(model, editor):
    """masactrl_utils.py:147-212 (the reference's spelling): attach ``editor`` to the UNet at ``model.model.diffusion_model``
    and set ``editor.num_att_layers`` to its attention count, 2 per transformer block (32 for SD-1.5).  ``cur_step`` is
    not reset, as in the reference.  ``editor=None`` detaches the editor (an addition: the reference cannot undo it)."""
    unet = _diffusion_unet(model)
    if editor is None:
        unet._editor = None
        return
    check_editor(editor)
    editor.num_att_layers = 2 * unet.num_transformer_blocks()
    unet._editor = editor


@torch.no_grad()
def action_pairs(model, sampler, cond, uncond, steps=50, guidance_scale=7.5, start_step=5, start_layer=12, x_T=None):
    """P action-change pairs in one sampler run (action_change_tool.py:15-45 does one per call).

    ``cond`` [P, 2, L, D]: the text embeddings of (source, target) of every pair; ``uncond`` [L, D]: the empty prompt's;
    ``x_T`` [P, 4, h, w]: one start code per pair, shared by its two rows (default: ``randn`` at 64 x 64, a 512^2 image).
    The model batch is [uncond ; cond], each half ordered (s0, t0, s1, t1, ...), and the edit maps row b to b & ~1 in
    ``MutualSelfAttentionControl(start_step, start_layer, total_steps=steps)``; without guidance (scale 1) each pair's two
    rows are the reference's two single-row halves and the edit is a no-op.  DDIM at eta 0.

    Returns (latents [P, 2, 4, h, w] fp32, images uint8 [P, 2, H, W, 3]): ``decode_first_stage`` post-processed as diffusers
    does, round(clamp(x / 2 + 1/2, 0, 1) * 255).  Pair i equals the single-pair run of that pair."""
    if not (isinstance(cond, torch.Tensor) and cond.dim() == 4 and cond.shape[1] == 2 and cond.shape[0] >= 1):
        raise ValueError(f"action_pairs: cond must be [P, 2, L, D] (source, target per pair), got {tuple(getattr(cond, 'shape', ()))}")
    P, _, L, D = cond.shape
    if not (isinstance(uncond, torch.Tensor) and tuple(uncond.shape) == (L, D)):
        raise ValueError(f"action_pairs: uncond must be [L, D] = {(L, D)}, got {tuple(getattr(uncond, 'shape', ()))}")
    dev = model.device
    if x_T is None:
        x_T = torch.randn(P, 4, 64, 64, device=dev)
    if not (isinstance(x_T, torch.Tensor) and x_T.dim() == 4 and x_T.shape[0] == P):
        raise ValueError(f"action_pairs: x_T must be [P, C, h, w] with P = {P}, got {tuple(getattr(x_T, 'shape', ()))}")
    unet = _diffusion_unet(model)
    cfg = guidance_scale != 1.0
    editor = MutualSelfAttentionControl(start_step, start_layer, total_steps=steps)
    editor._kv_group = 2 if cfg else 1
    c = cond.to(device=dev).reshape(2 * P, L, D)
    uc = uncond.to(device=dev)[None].expand(2 * P, L, D)
    x = x_T.to(device=dev, dtype=torch.float32).repeat_interleave(2, 0).contiguous()
    prev = unet._editor
    regiter_attention_editor_ldm(model, editor)
    try:
        lat, _ = sampler.sample(steps, 2 * P, tuple(x.shape[1:]), {"c_crossattn": [c]}, verbose=False, x_T=x, eta=0.0,
                                unconditional_guidance_scale=guidance_scale,
                                unconditional_conditioning={"c_crossattn": [uc]} if cfg else None)
    finally:
        unet._editor = prev
    img = model.decode_first_stage(lat).float().contiguous()
    n, C, H, W = img.shape
    u8 = torch.empty(n, H, W, C, dtype=torch.uint8, device=img.device)
    ops.image_to_u8(img, u8)
    return lat.reshape(P, 2, *lat.shape[1:]), u8.reshape(P, 2, H, W, C)
