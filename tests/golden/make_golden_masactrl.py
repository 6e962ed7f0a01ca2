#!/usr/bin/env python
"""Golden vectors of MasaCtrl's mutual self-attention (AnyEdit's action-change edits), from the reference's own modules on CPU.

Run in the build container only (needs the reference checkout):

    python tests/golden/make_golden_masactrl.py

The reference's ``UNetModel`` + CPU ``DDIMSampler`` (oracle/ref_import) run a seeded tiny UNet that keeps SD-1.5's 16
transformer blocks (4 levels, attention at 3 of them, 2 res blocks per level).  The reference's own
``regiter_attention_editor_ldm`` + ``MutualSelfAttentionControl`` (AnyEdit_Collection/other_modules/masactrl) do the
registering, through a shim exposing ``.model.diffusion_model``.  Writes ``masactrl_tiny.npz`` (inputs, final latents, the
model output of one active step) and ``masactrl_keys.json`` (config + state-dict shapes; weights come from
``oracle.weights``).

Cases, CFG 7.5 and 10 DDIM steps unless stated:
  tool     the tool's setting scaled down: MutualSelfAttentionControl(2, 12, total_steps=10)
  custom   layer_idx [0, 6, 13], step_idx [0, 3]: the shared CFG prefix, the middle block and a block of the last level
  nocfg    two prompts without guidance: two single-row halves, the edit is a no-op
  reuse    the tool's editor used again for a second run: cur_step starts at 10, nothing is edited
  plain    no editor
"""
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..", "..")))

from oracle import ddim_oracle, ref_import, weights  # noqa: E402

TINY_M = dict(image_size=16, in_channels=4, model_channels=64, out_channels=4, num_res_blocks=2,
              attention_resolutions=[4, 2, 1], channel_mult=[1, 2, 4, 4], num_heads=8,
              use_spatial_transformer=True, transformer_depth=1, context_dim=64, legacy=False)
SEED = 17
S, SCALE, EPS_STEP = 10, 7.5, 3


def randn(seed, *shape):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def main():
    UNetModel, DDIMSamplerCPU, _ = ref_import.load()
    sys.path.insert(0, ref_import.SRC_ROOT)
    from AnyEdit_Collection.other_modules.masactrl.masactrl import MutualSelfAttentionControl
    from AnyEdit_Collection.other_modules.masactrl.masactrl_utils import regiter_attention_editor_ldm
    torch.set_grad_enabled(False)

    torch.manual_seed(0)
    net = UNetModel(**TINY_M).eval()
    shapes = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    sd = weights.make_state_dict(shapes, SEED)
    net.load_state_dict(sd)
    sched = ddim_oracle.register_schedule("linear", 1000, 0.00085, 0.012)
    shim = ref_import.RefModelShim(net, sched, "crossattn")
    shim.model = types.SimpleNamespace(diffusion_model=net)        # what regiter_attention_editor_ldm walks
    eps_log = {}
    apply = shim.apply_model

    def logged(x, t, c):
        out = apply(x, t, c)
        eps_log.setdefault("calls", []).append(out.clone())
        return out
    shim.apply_model = logged
    sampler = DDIMSamplerCPU(shim)

    x1 = randn(41, 1, 4, 16, 16)
    x_T = x1.repeat(2, 1, 1, 1)                                     # start_code.expand(len(prompts), ...)
    ctx = randn(42, 2, 7, 64)                                       # [source, target]
    u = randn(43, 1, 7, 64).repeat(2, 1, 1)                         # the empty prompt for both rows
    cond, uncond = {"c_crossattn": [ctx]}, {"c_crossattn": [u]}

    def run(scale, editor=None):
        eps_log.clear()
        if editor is not None:
            regiter_attention_editor_ldm(shim, editor)
        out, _ = sampler.sample(S, 2, (4, 16, 16), cond, verbose=False, x_T=x_T.clone(), eta=0.0,
                                unconditional_guidance_scale=scale, unconditional_conditioning=uncond)
        return out, eps_log["calls"][EPS_STEP]

    res = {"x_T": x1.numpy(), "ctx": ctx.numpy(), "uctx": u[:1].numpy()}
    # the plain runs first: a registered editor cannot be removed from the reference modules
    res["final_plain"], res["eps_plain"] = (a.numpy() for a in run(SCALE))
    res["final_plain_nocfg"], _ = (a.numpy() for a in run(1.0))
    tool = MutualSelfAttentionControl(2, 12, total_steps=S)
    res["final_tool"], res["eps_tool"] = (a.numpy() for a in run(SCALE, tool))
    res["num_att_layers"] = tool.num_att_layers
    res["final_reuse"], _ = (a.numpy() for a in run(SCALE, tool))  # same editor: cur_step continues at 10
    res["reuse_cur_step"] = tool.cur_step
    custom = MutualSelfAttentionControl(layer_idx=[0, 6, 13], step_idx=[0, 3], total_steps=S)
    res["final_custom"], res["eps_custom"] = (a.numpy() for a in run(SCALE, custom))
    nocfg = MutualSelfAttentionControl(2, 12, total_steps=S)
    res["final_nocfg"], _ = (a.numpy() for a in run(1.0, nocfg))
    res.update(seed=SEED, steps=S, scale=SCALE, eps_step=EPS_STEP, wsum=weights.checksum(sd))
    np.savez(os.path.join(HERE, "masactrl_tiny.npz"), **res)
    with open(os.path.join(HERE, "masactrl_keys.json"), "w") as f:
        json.dump({"config": TINY_M, "keys": {k: list(v) for k, v in shapes.items()}}, f)
    print("num_att_layers", tool.num_att_layers, "reuse cur_step", tool.cur_step)
    print("golden vectors written to", HERE)


if __name__ == "__main__":
    main()
