"""MasaCtrl mutual self-attention (anyedit_b200.masactrl) on the host: the oracle against the reference golden, the editor's
active (step, block) set, the K/V map derivation and the editor refusals.  No GPU needed."""
import json
import os

import numpy as np
import pytest
import torch

G = os.path.join(os.path.dirname(__file__), "golden")


def _golden():
    from oracle import weights
    g = np.load(os.path.join(G, "masactrl_tiny.npz"))
    meta = json.load(open(os.path.join(G, "masactrl_keys.json")))
    sd = weights.make_state_dict({k: tuple(v) for k, v in meta["keys"].items()}, int(g["seed"]))
    assert abs(weights.checksum(sd) - float(g["wsum"])) < 1e-6 * max(1.0, abs(float(g["wsum"])))
    return g, sd, meta["config"]


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).norm() / b.norm())


@pytest.fixture(scope="module")
def golden():
    return _golden()


CASES = {   # case -> (guidance scale, editor as (step0, kwargs of the edit), golden key)
    "tool": (7.5, (0, dict(start_step=2, start_layer=12, total_steps=10)), "final_tool"),
    "custom": (7.5, (0, dict(layer_idx=[0, 6, 13], step_idx=[0, 3], total_steps=10)), "final_custom"),
    "nocfg": (1.0, (0, dict(start_step=2, start_layer=12, total_steps=10)), "final_nocfg"),
    "reuse": (7.5, (10, dict(start_step=2, start_layer=12, total_steps=10)), "final_reuse"),
    "plain": (7.5, None, "final_plain"),
}


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_matches_reference_golden(golden, case):
    from oracle import ddim_oracle, masactrl_oracle
    g, sd, cfg = golden
    scale, ed, key = CASES[case]
    sched = ddim_oracle.register_schedule("linear", 1000, 0.00085, 0.012)
    x_T = torch.from_numpy(g["x_T"]).repeat(2, 1, 1, 1)
    u = torch.from_numpy(g["uctx"]).repeat(2, 1, 1)
    eps = {}
    edit = None if ed is None else (lambda s, b, kw=ed[1]: masactrl_oracle.active(s, b, **kw))
    with torch.no_grad():
        out = masactrl_oracle.ddim_sample(sd, sched, int(g["steps"]), x_T, {"c_crossattn": [torch.from_numpy(g["ctx"])]},
                                          {"c_crossattn": [u]}, scale, step0=0 if ed is None else ed[0], edit=edit,
                                          on_eps=lambda i, e: eps.__setitem__(i, e), num_heads=cfg["num_heads"])
    e = _rel(out, g[key])
    print(f"[masactrl oracle {case}] final-latent rel-L2 vs reference golden = {e:.2e}")
    assert e < 1e-5, e
    if f"eps_{case}" in g.files:
        assert _rel(eps[int(g["eps_step"])], g[f"eps_{case}"]) < 1e-5


def test_golden_cases_differ_where_the_edit_acts(golden):
    """The edit changes the target (and not the source half's arithmetic); the no-guidance and reused-editor runs are plain."""
    g, _, _ = golden
    assert _rel(g["final_tool"][1], g["final_plain"][1]) > 1e-2
    assert _rel(g["final_custom"][1], g["final_plain"][1]) > 1e-2
    assert _rel(g["final_tool"][0], g["final_plain"][0]) < 1e-5            # sources attend to themselves
    assert _rel(g["final_nocfg"], g["final_plain_nocfg"]) < 1e-5
    assert _rel(g["final_reuse"], g["final_plain"]) < 1e-5
    assert int(g["num_att_layers"]) == 32 and int(g["reuse_cur_step"]) == 20


def _active_set(editor, steps, blocks=16, step0=0):
    from anyedit_b200.masactrl import kv_table
    t = kv_table(editor, blocks, 4, step0, steps)
    ident = np.arange(4)
    return {(step0 + s, b) for s in range(steps) for b in range(blocks) if not np.array_equal(t[s, b], ident)}


def _oracle_set(steps, step0=0, **kw):
    from oracle import masactrl_oracle
    return {(s, b) for s in range(step0, step0 + steps) for b in range(16) if masactrl_oracle.active(s, b, **kw)}


@pytest.mark.parametrize("kw", [dict(), dict(start_step=5, start_layer=12), dict(layer_idx=[0, 6, 13], step_idx=[0, 3]),
                                dict(layer_idx=[15, 3, 99], step_idx=[49, 7], total_steps=20), dict(start_step=0, start_layer=0)])
def test_active_set_equals_reference_semantics(kw):
    from anyedit_b200.masactrl import MutualSelfAttentionControl
    ed = MutualSelfAttentionControl(**kw)
    assert _active_set(ed, 50) == _oracle_set(50, **kw)
    assert ed.cur_step == 0 and ed.cur_att_layer == 0
    # the tool's (5, 12): blocks 12..15 from step 5 to 49
    if kw == dict(start_step=5, start_layer=12):
        assert _active_set(ed, 50) == {(s, b) for s in range(5, 50) for b in range(12, 16)}


def test_reused_editor_continues_counting():
    """regiter_attention_editor_ldm does not reset cur_step: a second 50-step run starts at step 50, where nothing is active."""
    from anyedit_b200.masactrl import AttentionBase, MutualSelfAttentionControl
    ed = MutualSelfAttentionControl(5, 12)
    assert _active_set(ed, 50, step0=50) == set()
    ed.cur_step = 57
    ed.reset()
    assert ed.cur_step == 0 and ed.cur_att_layer == 0
    assert _active_set(AttentionBase(), 50) == set()


def test_kv_batch_map():
    from anyedit_b200.masactrl import kv_batch_map
    from oracle import masactrl_oracle
    for N in (2, 4, 6, 8, 32):
        m = kv_batch_map(N)
        assert m.dtype == np.int32
        assert m.tolist() == [0 if b < N // 2 else N // 2 for b in range(N)]
        assert m.tolist() == masactrl_oracle.kv_rows(N).tolist()
    for P in (1, 2, 3, 8):
        m = kv_batch_map(4 * P, 2)
        assert m.tolist() == [b & ~1 for b in range(4 * P)]
        assert np.array_equal(m[2 * P:], m[:2 * P] + 2 * P)
    assert kv_batch_map(2).tolist() == [0, 1]                   # two single-row halves: no edit
    assert kv_batch_map(6, 1).tolist() == list(range(6))
    for N in (0, 1, 3, 5, 7):
        with pytest.raises(ValueError):
            kv_batch_map(N)
        with pytest.raises(ValueError):
            masactrl_oracle.kv_rows(N)
    with pytest.raises(ValueError):
        kv_batch_map(6, 2)                                      # groups of 2 do not tile a half of 3


def test_kv_table_checks_the_batch_only_when_active():
    from anyedit_b200.masactrl import AttentionBase, MutualSelfAttentionControl, kv_table
    assert kv_table(AttentionBase(), 16, 3, 0, 4).shape == (4, 16, 3)          # no edit: any batch
    assert np.array_equal(kv_table(MutualSelfAttentionControl(5, 12), 16, 3, 0, 5)[:, 0], np.broadcast_to(np.arange(3), (5, 3)))
    with pytest.raises(ValueError):
        kv_table(MutualSelfAttentionControl(5, 12), 16, 3, 0, 6)


def test_register_counts_layers_and_refuses_foreign_editors():
    from anyedit_b200 import masactrl
    from anyedit_b200.diffusion import LatentDenoiser
    from anyedit_b200.unet import UNetModel
    meta = json.load(open(os.path.join(G, "sd15_keys.json")))
    with torch.device("meta"):
        sd15 = UNetModel(**meta["config"])
    assert sd15.num_transformer_blocks() == 16
    cfg = json.load(open(os.path.join(G, "masactrl_keys.json")))["config"]
    model = LatentDenoiser(UNetModel(**cfg), conditioning_key="crossattn")
    unet = model.model.diffusion_model
    ed = masactrl.MutualSelfAttentionControl(5, 12)
    ed.cur_step = 3
    masactrl.regiter_attention_editor_ldm(model, ed)
    assert ed.num_att_layers == 32 and unet._editor is ed and ed.cur_step == 3        # no reset, as in the reference
    base = masactrl.AttentionBase()
    masactrl.regiter_attention_editor_ldm(model, base)
    assert unet._editor is base and base.num_att_layers == 32
    masactrl.regiter_attention_editor_ldm(model, None)
    assert unet._editor is None
    for name in ("AttentionStore", "MutualSelfAttentionControlMask", "MutualSelfAttentionControlMaskAuto",
                 "MutualSelfAttentionControlUnion"):
        foreign = type(name, (masactrl.MutualSelfAttentionControl,), {})()
        with pytest.raises(NotImplementedError, match=name):
            masactrl.regiter_attention_editor_ldm(model, foreign)
    # the reference's own editor object (same name, another module) and arbitrary objects
    ref_like = type("MutualSelfAttentionControl", (), {"__module__": "masactrl.masactrl"})()
    with pytest.raises(TypeError, match="masactrl.masactrl.MutualSelfAttentionControl"):
        masactrl.regiter_attention_editor_ldm(model, ref_like)
    with pytest.raises(TypeError):
        masactrl.regiter_attention_editor_ldm(model, object())
    assert unet._editor is None
    with pytest.raises(TypeError):
        masactrl.regiter_attention_editor_ldm(torch.nn.Linear(2, 2), ed)


def test_action_pairs_refuses_mismatched_shapes():
    from anyedit_b200 import masactrl
    from anyedit_b200.diffusion import LatentDenoiser
    from anyedit_b200.unet import UNetModel
    cfg = json.load(open(os.path.join(G, "masactrl_keys.json")))["config"]
    model = LatentDenoiser(UNetModel(**cfg), conditioning_key="crossattn")
    good_c, good_u = torch.zeros(2, 2, 7, 64), torch.zeros(7, 64)
    for c, u, x in ((torch.zeros(2, 3, 7, 64), good_u, None), (torch.zeros(4, 7, 64), good_u, None),
                    (good_c, torch.zeros(2, 7, 64), None), (good_c, torch.zeros(7, 32), None),
                    (good_c, good_u, torch.zeros(3, 4, 16, 16)), (good_c, good_u, torch.zeros(4, 16, 16))):
        with pytest.raises(ValueError):
            masactrl.action_pairs(model, None, c, u, x_T=x)
