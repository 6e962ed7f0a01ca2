"""fp32 CPU restatement of MasaCtrl's mutual self-attention over the UNet and DDIM oracles (TEST INFRASTRUCTURE).

Reference (relative to /root/reference):
  AnyEdit_Collection/other_modules/masactrl/masactrl_utils.py  AttentionBase :14-40 (one UNet forward = one step),
      regiter_attention_editor_ldm :147-212 (two attention layers per BasicTransformerBlock, in forward order)
  AnyEdit_Collection/other_modules/masactrl/masactrl.py  MutualSelfAttentionControl :14-72: self-attention of block l at
      step s is edited when s in step_idx and l in layer_idx; q/k/v.chunk(2) splits the batch into its CFG halves and every
      query row of a half attends to the keys and values of the first sample of that half

Derived independently of ``anyedit_b200.masactrl``.  Attending to the K/V of another sample is attn1 evaluated with
that sample's normalised tokens as its context: K = x[row] Wk, V = x[row] Wv.  ``unet_forward`` installs that as a hook
on ``unet_oracle``'s attention for one forward and leaves the module as it was afterwards.
"""
import torch

from oracle import ddim_oracle, unet_oracle


def active(step, block, start_step=4, start_layer=10, layer_idx=None, step_idx=None, total_steps=50, total_layers=16):
    """masactrl.py:20-36, 56-61: is the self-attention of transformer block ``block`` edited at step ``step``?"""
    layers = list(layer_idx) if layer_idx is not None else list(range(start_layer, total_layers))
    steps = list(step_idx) if step_idx is not None else list(range(start_step, total_steps))
    return step in steps and block in layers


def kv_rows(N, group=None):
    """masactrl.py:63-70: chunk(2) into halves, each half's rows read the first row of their half (or of their group of
    ``group`` rows inside the half).  Refuses what the reference cannot split."""
    if N < 2 or N % 2:
        raise ValueError(f"batch {N} has no two CFG halves")
    half = N // 2
    g = half if group is None else group
    if half % g:
        raise ValueError(f"groups of {g} do not tile a half of {half}")
    return torch.tensor([(b // g) * g for b in range(N)], dtype=torch.long)


def unet_forward(sd, x, t, context, rows_of_block, **kw):
    """``unet_oracle.unet_forward`` with attn1 of transformer block i (forward order) reading the K/V rows
    ``rows_of_block(i)`` (a LongTensor [N]) when that is not None.  Blocks whose attn1 is a cross-attention
    (disable_self_attn) are counted but never edited."""
    orig = unet_oracle._attention
    count = [0]

    def attention(sd_, p, x_, context_, heads, extra=None):
        if p.endswith("attn1."):
            blk = count[0]
            count[0] += 1
            rows = rows_of_block(blk)
            if context_ is None and rows is not None:
                return orig(sd_, p, x_, x_[rows], heads, extra)
        return orig(sd_, p, x_, context_, heads, extra)

    unet_oracle._attention = attention
    try:
        return unet_oracle.unet_forward(sd, x, t, context, **kw)
    finally:
        unet_oracle._attention = orig


def ddim_sample(sd, sched, S, x_T, cond, uncond, scale, conditioning_key="crossattn", step0=0, group=None, edit=None,
                on_eps=None, **kw):
    """DDIM (eta 0) with the edit: ``edit(step, block) -> bool`` at editor step ``step0 + i`` for loop step i (None: the plain
    run).  ``on_eps(i, eps)`` sees the model output of every step.  Returns the final latent."""
    step = [step0]
    seen = [0]

    def unet(x, t, context=None, y=None):
        s = step[0]
        rows = None
        if edit is not None:
            rows_all = [None]

            def rows_of_block(blk):
                if not edit(s, blk):
                    return None
                if rows_all[0] is None:
                    rows_all[0] = kv_rows(x.shape[0], group)
                return rows_all[0]
            rows = rows_of_block
        out = unet_forward(sd, x, t, context, rows if rows is not None else (lambda blk: None), y=y, **kw)
        step[0] += 1
        if on_eps is not None:
            on_eps(seen[0], out)
        seen[0] += 1
        return out

    model_fn = lambda x, t, c: ddim_oracle.apply_model(unet, conditioning_key, x, t, c)
    out, _ = ddim_oracle.ddim_sample(model_fn, sched, S, x_T, cond, uncond, scale, eta=0.0)
    return out
