"""MasaCtrl mutual self-attention (anyedit_b200.masactrl) on the GPU.

* Kernel: ``anysd_attention_kvmap_f16`` with random many-to-one K/V batch maps against a float64 bound, on the wgmma and the
  mma.sync kernel (forced in child processes, ANYSD_ATTN=wgmma|mma).  Every case also runs the plain kernel on K/V gathered
  by the map (must give the same bits), and the identity map against NULL (same bits).
  Bound per output element: fp16 P (relative 2^-11) weighted by |v|, twice over, plus the fp16 output rounding:
  |o - o64| <= |g| (2^-10 sum_j p_j |v_j| + 2^-11 |o64|) + 1e-6.
* The tiny 16-block UNet against the reference golden (tests/golden/make_golden_masactrl.py), the bit-for-bit identities of
  the sampler integration, the SD-1.5 geometry against the oracle, and the refusals.
"""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

G = os.path.join(os.path.dirname(__file__), "golden")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LATENT_TOL = 5e-3            # final-latent rel-L2 of a CFG DDIM run vs the reference golden (test_gpu_unet.test_ddim_tiny_golden)
SD15_TOL = 5e-3              # final-latent bound of a CFG DDIM run vs fp32 (test_gpu_unet); measured 3.7e-3 at 64^2, 4 steps

# (name, B, heads, n_q, n_kv, d, head stride, aux_cols, gate, lse, kernels)
KCASES = [
    ("d40_n4096_aux", 4, 8, 4096, 4096, 40, 48, True, False, False, ("wgmma",)),
    ("d40_n4096", 4, 8, 4096, 4096, 40, 40, False, False, False, ("mma",)),
    ("d80_n1024", 4, 8, 1024, 1024, 80, 80, False, False, False, ("wgmma", "mma")),
    ("d160_n256", 4, 8, 256, 256, 160, 160, False, False, False, ("wgmma", "mma")),
    ("partial_kv_tile", 3, 4, 300, 200, 64, 64, False, False, False, ("wgmma", "mma")),
    ("gate", 4, 8, 256, 333, 64, 64, False, True, False, ("wgmma", "mma")),
    ("lse_aux", 6, 8, 512, 512, 40, 48, True, False, True, ("wgmma",)),
]


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


# ---- kernel worker (runs in a child process with ANYSD_ATTN forced) ---------------------------------------------------
def _operands(B, heads, n_q, n_kv, d, hs, aux, gen):
    dev = "cuda"
    q = torch.zeros(B * n_q, heads, hs)
    k = torch.zeros(B * n_kv, heads, hs)
    v = torch.zeros(B * n_kv, heads, hs)
    q[..., :d] = torch.randn(B * n_q, heads, d, generator=gen) * 0.6
    k[..., :d] = torch.randn(B * n_kv, heads, d, generator=gen) * 0.6
    v[..., :d] = torch.randn(B * n_kv, heads, d, generator=gen)
    if aux:                                   # anysd_attn_params::aux_cols operand contract
        q[..., :d] *= d ** -0.5 * 1.4426950408889634
        k[..., d:d + 2] = 1.0
        v[..., d] = 1.0
    f = lambda t: t.reshape(t.shape[0], heads * hs).half().to(dev).contiguous()
    return f(q), f(k), f(v)


def _run(ops, q, k, v, B, heads, n_q, n_kv, d, hs, aux, gate, lse, kv_batch):
    out = torch.zeros(B * n_q, heads * d, dtype=torch.float16, device="cuda")
    ls = torch.zeros(B * heads * n_q, dtype=torch.float32, device="cuda") if lse else None
    ld = heads * hs
    ops.attention(q, k, v, out, B, heads, n_q, n_kv, d, ld, ld, ld, heads * d, head_stride=hs, aux_cols=aux,
                  gate=gate, lse=ls, kv_batch=kv_batch)
    return out, ls


def _ref64(q, k, v, B, heads, n_q, n_kv, d, hs, aux, rows, m, gate):
    """float64 attention of the query rows ``rows`` of every batch, K/V of batch m[b]; returns (o64, sum_j p_j |v_j|)."""
    qf = q.view(B, n_q, heads, hs)[:, rows, :, :d].double()
    kf = k.view(B, n_kv, heads, hs)[m][..., :d].double()
    vf = v.view(B, n_kv, heads, hs)[m][..., :d].double()
    s = torch.einsum("bihd,bjhd->bhij", qf, kf)
    s = s * math.log(2.0) if aux else s * d ** -0.5
    p = torch.softmax(s, -1)
    o = torch.einsum("bhij,bjhd->bihd", p, vf)
    sa = torch.einsum("bhij,bjhd->bihd", p, vf.abs())
    if gate is not None:
        g = gate.double().view(B, 1, 1, 1)
        o, sa = o * g, sa * g.abs()
    return o, sa


def _worker(out_path):
    from anyedit_b200 import ops
    gen = torch.Generator().manual_seed(2024)
    res = {}
    for name, B, heads, n_q, n_kv, d, hs, aux, use_gate, lse, kernels in KCASES:
        if os.environ["ANYSD_ATTN"] not in kernels:
            continue
        q, k, v = _operands(B, heads, n_q, n_kv, d, hs, aux, gen)
        gate = (torch.rand(B, generator=gen) * 1.5 + 0.25).cuda() if use_gate else None
        maps = [torch.randint(0, B, (B,), generator=gen) for _ in range(2)]
        maps[0][0] = B - 1                                          # never the identity
        maps.append(torch.arange(B) & ~1)                           # the action_pairs map
        rows = torch.cat([torch.arange(min(n_q, 256)), torch.arange(max(0, n_q - 256), n_q)]).unique()
        worst, bits = 0.0, True
        for m in maps:
            mdev = m.to(torch.int32).cuda()
            out, ls = _run(ops, q, k, v, B, heads, n_q, n_kv, d, hs, aux, gate, lse, mdev)
            # the plain kernel on K/V gathered by the map: same operands per (batch, head), same bits
            kg = k.view(B, n_kv, -1)[m.cuda()].reshape(B * n_kv, -1).contiguous()
            vg = v.view(B, n_kv, -1)[m.cuda()].reshape(B * n_kv, -1).contiguous()
            og, lg = _run(ops, q, kg, vg, B, heads, n_q, n_kv, d, hs, aux, gate, lse, None)
            bits &= torch.equal(out, og) and (ls is None or torch.equal(ls, lg))
            o64, sa = _ref64(q, k, v, B, heads, n_q, n_kv, d, hs, aux, rows.cuda(), m.cuda(), gate)
            got = out.view(B, n_q, heads, d)[:, rows.cuda()].double()
            bound = 2.0 ** -10 * sa + 2.0 ** -11 * o64.abs() + 1e-6
            worst = max(worst, float(((got - o64).abs() / bound).max()))
            if lse:
                # base-2 log-sum-exp of the K/V batch's scores: the same as the gathered run, checked above
                assert torch.isfinite(ls).all()
        ident = torch.arange(B, dtype=torch.int32).cuda()
        o_id, l_id = _run(ops, q, k, v, B, heads, n_q, n_kv, d, hs, aux, gate, lse, ident)
        o_null, l_null = _run(ops, q, k, v, B, heads, n_q, n_kv, d, hs, aux, gate, lse, None)
        identity = torch.equal(o_id, o_null) and (l_id is None or torch.equal(l_id, l_null))
        res[name] = {"worst": worst, "gathered_bits": bool(bits), "identity_bits": bool(identity)}
    torch.cuda.synchronize()
    with open(out_path, "w") as f:
        json.dump(res, f)


if __name__ == "__main__" and len(sys.argv) == 3 and sys.argv[1] == "--worker":
    sys.path.insert(0, ROOT)
    _worker(sys.argv[2])
    sys.exit(0)


pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


@pytest.mark.parametrize("kernel", ["wgmma", "mma"])
def test_kvmap_kernel_against_fp64(kernel, tmp_path):
    out = tmp_path / f"kvmap_{kernel}.json"
    env = dict(os.environ, ANYSD_ATTN=kernel)
    cmd = [sys.executable, *(["-s"] if sys.flags.no_user_site else []), os.path.abspath(__file__), "--worker", str(out)]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, f"worker failed:\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"
    res = json.load(open(out))
    want = [c[0] for c in KCASES if kernel in c[-1]]
    assert sorted(res) == sorted(want)
    for name in want:
        print(f"[kvmap {kernel}] {name:16s} worst err/bound {res[name]['worst']:.3f} gathered-K/V bits "
              f"{res[name]['gathered_bits']} identity-map bits {res[name]['identity_bits']}")
    bad = [n for n in want if not (res[n]["worst"] <= 1.0 and res[n]["gathered_bits"] and res[n]["identity_bits"])]
    assert not bad, {n: res[n] for n in bad}


# ---- the tiny 16-block UNet ------------------------------------------------------------------------------------------
def _tiny():
    from anyedit_b200.diffusion import LatentDenoiser
    from anyedit_b200.unet import UNetModel
    from oracle import weights
    g = np.load(os.path.join(G, "masactrl_tiny.npz"))
    meta = json.load(open(os.path.join(G, "masactrl_keys.json")))
    net = UNetModel(**meta["config"])
    net.load_state_dict(weights.make_state_dict({k: tuple(v) for k, v in meta["keys"].items()}, int(g["seed"])), strict=True)
    return LatentDenoiser(net.cuda(), conditioning_key="crossattn").cuda(), g


@pytest.fixture(scope="module")
def tiny():
    return _tiny()


def _inputs(g, P=1):
    f = lambda k: torch.from_numpy(g[k]).cuda()
    x_T = f("x_T").repeat(2 * P, 1, 1, 1)
    ctx = f("ctx").repeat(P, 1, 1)
    u = f("uctx").repeat(2 * P, 1, 1)
    return x_T, {"c_crossattn": [ctx]}, {"c_crossattn": [u]}


def _sample(model, g, editor=None, scale=7.5, graph=True, sampler=None, inputs=None):
    from anyedit_b200.ddim import DDIMSampler
    from anyedit_b200.masactrl import regiter_attention_editor_ldm
    x_T, c, uc = inputs if inputs is not None else _inputs(g)
    regiter_attention_editor_ldm(model, editor)
    try:
        smp = sampler or DDIMSampler(model, use_cuda_graph=graph)
        out, _ = smp.sample(int(g["steps"]), x_T.shape[0], (4, 16, 16), c, verbose=False, x_T=x_T, eta=0.0,
                            unconditional_guidance_scale=scale, unconditional_conditioning=uc)
    finally:
        regiter_attention_editor_ldm(model, None)
    return out


def test_tiny_unet_vs_reference_golden(tiny):
    """The reference's own editor on its own UNet (golden) vs the kernels: the tool's setting, custom lists reaching into the
    shared CFG prefix, no guidance, and the plain run; the edit moves the target far more than the bound."""
    from anyedit_b200.masactrl import MutualSelfAttentionControl
    model, g = tiny
    f = lambda k: torch.from_numpy(g[k])
    runs = {"tool": (MutualSelfAttentionControl(2, 12, total_steps=10), 7.5),
            "custom": (MutualSelfAttentionControl(layer_idx=[0, 6, 13], step_idx=[0, 3], total_steps=10), 7.5),
            "nocfg": (MutualSelfAttentionControl(2, 12, total_steps=10), 1.0),
            "plain": (None, 7.5)}
    outs = {}
    for case, (ed, scale) in runs.items():
        outs[case] = out = _sample(model, g, ed, scale)
        e = rel(out, f(f"final_{case}"))
        print(f"[masactrl tiny {case}] final-latent rel-L2 vs reference golden = {e:.3e}")
        assert e < LATENT_TOL, (case, e)
    for case in ("tool", "custom"):
        moved = rel(outs[case][1], f("final_plain")[1])
        print(f"[masactrl tiny {case}] target vs plain target rel-L2 = {moved:.3e}")
        assert moved > 5 * LATENT_TOL, moved                   # measured 2.9e-2 (tool) against errors of 2.5e-3
    # the editor object was not reset, and a second run with it is the plain run (golden "reuse")
    ed = runs["tool"][0]
    assert ed.cur_step == 10
    again = _sample(model, g, ed)
    assert ed.cur_step == 20
    assert rel(again, f("final_reuse")) < LATENT_TOL
    assert torch.equal(again, outs["plain"])


def test_graph_equals_eager_and_step_count(tiny):
    from anyedit_b200.masactrl import MutualSelfAttentionControl
    model, g = tiny
    outs = []
    for graph in (True, False):
        ed = MutualSelfAttentionControl(layer_idx=[0, 6, 13, 15], step_idx=[0, 3, 4, 9], total_steps=10)
        outs.append(_sample(model, g, ed, graph=graph))
        assert ed.cur_step == int(g["steps"]), (graph, ed.cur_step)
    assert torch.equal(outs[0], outs[1])


def test_source_rows_equal_plain_source_run(tiny):
    """Sources attend to themselves: the source rows of a MasaCtrl run equal a plain run of the source prompt alone."""
    from anyedit_b200.masactrl import MutualSelfAttentionControl
    model, g = tiny
    out = _sample(model, g, MutualSelfAttentionControl(layer_idx=[0, 6, 13], step_idx=list(range(10)), total_steps=10))
    x_T, c, uc = _inputs(g)
    src = _sample(model, g, None, inputs=(x_T[:1], {"c_crossattn": [c["c_crossattn"][0][:1]]}, {"c_crossattn": [uc["c_crossattn"][0][:1]]}))
    assert torch.equal(out[:1], src)
    assert not torch.equal(out[1:], _sample(model, g, None)[1:])


def test_shared_halves_on_and_off(tiny, monkeypatch):
    """An active block in the shared CFG prefix (block 0) runs on the first half of the map: same bits with sharing off."""
    from anyedit_b200.ddim import DDIMSampler
    from anyedit_b200.masactrl import MutualSelfAttentionControl
    model, g = tiny
    outs = {}
    for share in ("1", "0"):
        monkeypatch.setenv("ANYSD_SHARE_CFG", share)
        for graph in (True, False):
            smp = DDIMSampler(model, use_cuda_graph=graph)
            ed = MutualSelfAttentionControl(layer_idx=[0, 1, 13], step_idx=list(range(10)), total_steps=10)
            outs[(share, graph)] = _sample(model, g, ed, sampler=smp)
            assert next(iter(smp._graphs.values())).shared == (share == "1")
    ref = outs[("0", False)]
    for k, v in outs.items():
        assert torch.equal(v, ref), k


def test_no_op_editors_equal_plain_run(tiny):
    from anyedit_b200.masactrl import AttentionBase, MutualSelfAttentionControl
    model, g = tiny
    plain = _sample(model, g, None)
    assert torch.equal(_sample(model, g, AttentionBase()), plain)
    used = MutualSelfAttentionControl(2, 12, total_steps=10)
    used.cur_step = 10                                          # exhausted: a previous run counted its 10 steps
    assert torch.equal(_sample(model, g, used), plain)


def test_eager_forward_advances_the_editor(tiny):
    """A UNet forward outside the sampler reads the editor's active set for cur_step and advances it by one."""
    from anyedit_b200.masactrl import MutualSelfAttentionControl, regiter_attention_editor_ldm
    model, g = tiny
    unet = model.model.diffusion_model
    x_T, c, uc = _inputs(g)
    x = torch.cat([x_T, x_T])
    ctx = torch.cat([uc["c_crossattn"][0], c["c_crossattn"][0]])
    t = torch.full((4,), 501, device="cuda")
    plain = unet(x, t, context=ctx)
    ed = MutualSelfAttentionControl(1, 12, total_steps=10)
    regiter_attention_editor_ldm(model, ed)
    try:
        a = unet(x, t, context=ctx)                              # step 0: not active
        b = unet(x, t, context=ctx)                              # step 1: blocks 12..15
    finally:
        regiter_attention_editor_ldm(model, None)
    assert ed.cur_step == 2
    assert torch.equal(a, plain) and not torch.equal(b[2:], plain[2:]) and torch.equal(b[[0, 2]], plain[[0, 2]])


def _vae():
    from anyedit_b200.autoencoder import AutoencoderKL
    from oracle import weights
    meta = json.load(open(os.path.join(G, "vae_tiny_keys.json")))
    net = AutoencoderKL(meta["config"], embed_dim=4)
    net.load_state_dict(weights.make_state_dict({k: tuple(v) for k, v in meta["keys"].items()}, 5), strict=True)
    return net.cuda()


def test_action_pairs_equal_single_pair_runs(tiny):
    """action_pairs with P = 3 in one run: pair i equals the single-pair run through regiter_attention_editor_ldm (the tool's
    request), latents and decoded bytes; the bytes are diffusers' post-processing of decode_first_stage."""
    from anyedit_b200.ddim import DDIMSampler
    from anyedit_b200.masactrl import MutualSelfAttentionControl, action_pairs, regiter_attention_editor_ldm
    model, g = tiny
    model.first_stage_model, model.scale_factor = _vae(), 0.18215
    try:
        gen = torch.Generator().manual_seed(5)
        P, S = 3, int(g["steps"])
        cond = torch.randn(P, 2, 7, 64, generator=gen).cuda()
        uncond = torch.randn(7, 64, generator=gen).cuda()
        x_T = torch.randn(P, 4, 16, 16, generator=gen).cuda()
        smp = DDIMSampler(model)
        lat, img = action_pairs(model, smp, cond, uncond, steps=S, guidance_scale=7.5, start_step=2, start_layer=12, x_T=x_T)
        assert tuple(lat.shape) == (P, 2, 4, 16, 16) and img.dtype == torch.uint8 and img.shape[:2] == (P, 2) and img.shape[-1] == 3
        assert model.model.diffusion_model._editor is None
        for i in range(P):
            ed = MutualSelfAttentionControl(2, 12, total_steps=S)
            regiter_attention_editor_ldm(model, ed)
            try:
                one, _ = DDIMSampler(model).sample(S, 2, (4, 16, 16), {"c_crossattn": [cond[i]]}, verbose=False,
                                                   x_T=x_T[i:i + 1].expand(2, -1, -1, -1), eta=0.0, unconditional_guidance_scale=7.5,
                                                   unconditional_conditioning={"c_crossattn": [uncond[None].expand(2, -1, -1)]})
            finally:
                regiter_attention_editor_ldm(model, None)
            assert ed.cur_step == S
            assert torch.equal(lat[i], one), i
            dec = model.decode_first_stage(one).float().cpu().numpy().transpose(0, 2, 3, 1)
            ref = (np.clip(dec / 2 + 0.5, 0, 1) * 255).round().astype(np.uint8)      # diffusers' numpy post-processing
            assert np.array_equal(img[i].cpu().numpy(), ref), i
        assert not torch.equal(lat[:, 1], action_pairs(model, smp, cond, uncond, steps=S, guidance_scale=7.5, start_step=S,
                                                      start_layer=12, x_T=x_T)[0][:, 1])
    finally:
        model.first_stage_model, model.scale_factor = None, 1.0


def test_refusals(tiny):
    from anyedit_b200.ddim import DDIMSampler
    from anyedit_b200.dpm_solver import DPMSolverSampler
    from anyedit_b200.masactrl import MutualSelfAttentionControl, regiter_attention_editor_ldm
    from anyedit_b200.plms import PLMSSampler
    model, g = tiny
    x_T, c, uc = _inputs(g)
    ctx3 = torch.cat([c["c_crossattn"][0], c["c_crossattn"][0][:1]])
    regiter_attention_editor_ldm(model, MutualSelfAttentionControl(0, 12, total_steps=10))
    try:
        with pytest.raises(ValueError, match="even batch"):          # three prompts without guidance: no two halves
            DDIMSampler(model).sample(10, 3, (4, 16, 16), {"c_crossattn": [ctx3]}, verbose=False,
                                      x_T=torch.cat([x_T, x_T[:1]]), eta=0.0)
        with pytest.raises(NotImplementedError, match="three-way"):
            DDIMSampler(model).sample(10, 2, (4, 16, 16), c, verbose=False, x_T=x_T, unconditional_guidance_scale=7.5,
                                      unconditional_conditioning=uc, image_guidance_scale=1.5, image_conditioning=uc)
        for cls in (PLMSSampler, DPMSolverSampler):
            with pytest.raises(NotImplementedError):
                cls(model).sample(10, 2, (4, 16, 16), c, verbose=False, x_T=x_T, unconditional_guidance_scale=7.5,
                                  unconditional_conditioning=uc)
        smp = DDIMSampler(model)
        smp.make_schedule(10, verbose=False)
        for call in (lambda: smp.decode(x_T, c, 3), lambda: smp.encode(x_T, c, 3),
                     lambda: smp.p_sample_ddim(x_T, c, torch.full((2,), 901, device="cuda"), 9)):
            with pytest.raises(NotImplementedError):
                call()
        foreign = type("AttentionStore", (MutualSelfAttentionControl,), {})()
        with pytest.raises(NotImplementedError, match="AttentionStore"):
            regiter_attention_editor_ldm(model, foreign)
    finally:
        regiter_attention_editor_ldm(model, None)
    # detached: the same calls run
    DDIMSampler(model).sample(2, 3, (4, 16, 16), {"c_crossattn": [ctx3]}, verbose=False, x_T=torch.cat([x_T, x_T[:1]]), eta=0.0)


def test_sd15_geometry_vs_oracle():
    """SD-1.5 at a 64^2 latent (512^2 image), seeded real-width weights: 4 DDIM steps (the ldm uniform schedule has no 3-step
    grid, util.py:46-60) with MutualSelfAttentionControl(1, 12), so blocks 12..15 (32^2 d 80 and 64^2 d 40 heads) are edited
    on 3 steps; final latent against the fp32 CPU oracle."""
    from anyedit_b200.ddim import DDIMSampler
    from anyedit_b200.diffusion import LatentDenoiser
    from anyedit_b200.masactrl import MutualSelfAttentionControl, regiter_attention_editor_ldm
    from anyedit_b200.unet import UNetModel
    from oracle import cpu, ddim_oracle, masactrl_oracle, weights
    meta = json.load(open(os.path.join(G, "sd15_keys.json")))
    cfg = dict(meta["config"], in_channels=4)
    keys = {k: tuple(v) for k, v in meta["keys"].items()}
    keys["input_blocks.0.0.weight"] = (320, 4, 3, 3)
    sd = weights.make_state_dict(keys, 3, scheme="torch")
    with torch.device("cuda"):
        net = UNetModel(**cfg)
    net.load_state_dict(sd)
    model = LatentDenoiser(net, conditioning_key="crossattn").cuda()
    gen = torch.Generator().manual_seed(4321)
    x1 = torch.randn(1, 4, 64, 64, generator=gen)
    ctx, u = torch.randn(2, 77, 768, generator=gen), torch.randn(1, 77, 768, generator=gen).repeat(2, 1, 1)
    S = 4
    runs = {}
    for name, ed in (("edit", MutualSelfAttentionControl(1, 12, total_steps=S)), ("plain", None)):
        regiter_attention_editor_ldm(model, ed)
        try:
            runs[name], _ = DDIMSampler(model).sample(S, 2, (4, 64, 64), {"c_crossattn": [ctx.cuda()]}, verbose=False,
                                                      x_T=x1.repeat(2, 1, 1, 1).cuda(), eta=0.0, unconditional_guidance_scale=7.5,
                                                      unconditional_conditioning={"c_crossattn": [u.cuda()]})
        finally:
            regiter_attention_editor_ldm(model, None)
    out = runs["edit"]
    torch.set_num_threads(cpu.usable_cores())
    sched = ddim_oracle.register_schedule("linear", 1000, 0.00085, 0.012)
    with torch.no_grad():
        ref = masactrl_oracle.ddim_sample(sd, sched, S, x1.repeat(2, 1, 1, 1), {"c_crossattn": [ctx]}, {"c_crossattn": [u]}, 7.5,
                                          edit=lambda s, b: masactrl_oracle.active(s, b, 1, 12, total_steps=S),
                                          num_heads=cfg["num_heads"])
    e = rel(out, ref)
    moved = rel(out[1], runs["plain"][1])
    print(f"[masactrl sd15 64x64, {S} steps] final-latent rel-L2 vs oracle = {e:.3e}; the edit moved the target by {moved:.3e}")
    assert torch.equal(out[0], runs["plain"][0])                    # the source attends to itself
    assert moved > 0
    assert e < SD15_TOL, e
