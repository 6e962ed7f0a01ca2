#!/usr/bin/env python
"""Timing of AnyEdit's action-change edits (MasaCtrl mutual self-attention) on one GPU -- a diagnostic, not a test.  Prints the
card and its power limit with the numbers.
  * the self-attention kernel with the identity K/V map vs the pair map (b -> b & ~1) at 64^2 d 40 (8 aux_cols heads) and
    32^2 d 80 (8 heads), model batch 4 and 32: CUDA events over repeated windows, the two maps alternated, median;
  * one 50-step CFG DDIM run (``--steps``) at the SD-1.5 geometry (64^2 latent, seeded weights) with and without
    MutualSelfAttentionControl(5, 12), P = 1 and 8 pairs (model batch 4 and 32), alternated, median of ``--reps``;
  * ``action_pairs`` end to end at 512^2 (sampler + SD VAE decode + uint8 post-processing): P = 8 in one call vs 8 calls of
    one pair, pairs/s.
Usage: python tests/diag_masactrl.py [--windows 5] [--iters 20] [--steps 50] [--reps 3]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))


def timed(fn, windows, iters):
    times = []
    for _ in range(windows):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / iters)
    return sorted(times)[len(times) // 2]


def host_s(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def kernel_leg(a):
    from anyedit_b200 import ops
    print("self-attention kernel, identity map vs pair map (ms per launch, median of windows):")
    for n, d, hs, aux in ((4096, 40, 48, True), (1024, 80, 80, False)):
        for B in (4, 32):
            heads = 8
            qkv = torch.randn(B * n, 3 * heads * hs, device="cuda").half()
            if aux:
                v = qkv.view(B * n, 3, heads, hs)
                v[..., d:] = 0
                v[:, 1, :, d:d + 2] = 1
                v[:, 2, :, d] = 1
            Cp = heads * hs
            out = torch.empty(B * n, heads * d, device="cuda", dtype=torch.float16)
            maps = {"identity": torch.arange(B, dtype=torch.int32, device="cuda"),
                    "pairs": (torch.arange(B, device="cuda") & ~1).to(torch.int32)}
            run = lambda m: ops.attention(qkv, qkv[:, Cp:], qkv[:, 2 * Cp:], out, B, heads, n, n, d, 3 * Cp, 3 * Cp, 3 * Cp,
                                          heads * d, head_stride=hs, aux_cols=aux, kv_batch=m)
            for m in maps.values():
                run(m)
            t = {k: [] for k in maps}
            for _ in range(3):
                for k, m in maps.items():
                    t[k].append(timed(lambda: run(m), a.windows, a.iters))
            ti, tp = sorted(t["identity"])[1], sorted(t["pairs"])[1]
            fl = 4.0 * B * heads * n * n * d
            print(f"  {int(n ** 0.5)}^2 d {d} B {B}: identity {ti:.3f} ms ({fl / ti / 1e9:.0f} TFLOP/s), pairs {tp:.3f} ms "
                  f"({fl / tp / 1e9:.0f} TFLOP/s), pairs / identity {tp / ti:.3f}")


def sd15(with_vae=False):
    from anyedit_b200.autoencoder import AutoencoderKL
    from anyedit_b200.diffusion import LatentDenoiser
    from anyedit_b200.unet import UNetModel
    from oracle import weights
    meta = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "sd15_keys.json")))
    cfg = dict(meta["config"], in_channels=4)
    with torch.device("cuda"):
        net = UNetModel(**cfg)
    net.load_state_dict(weights.make_state_dict({k: tuple(v.shape) for k, v in net.state_dict().items()}, 3, scheme="torch"))
    vae = None
    if with_vae:
        vae = AutoencoderKL(dict(double_z=True, z_channels=4, resolution=256, in_channels=3, out_ch=3, ch=128, ch_mult=[1, 2, 4, 4],
                                 num_res_blocks=2, attn_resolutions=[], dropout=0.0), embed_dim=4)
        vae.load_state_dict(weights.make_state_dict({k: tuple(v.shape) for k, v in vae.state_dict().items()}, 54, scheme="torch"))
        vae = vae.cuda()
    return LatentDenoiser(net, conditioning_key="crossattn", first_stage_model=vae, scale_factor=0.18215).cuda()


def run_leg(a, model):
    from anyedit_b200.ddim import DDIMSampler
    from anyedit_b200.masactrl import MutualSelfAttentionControl, regiter_attention_editor_ldm
    print(f"one {a.steps}-step CFG 7.5 DDIM run at 64^2 (s per run, median of {a.reps}):")
    smp = DDIMSampler(model)
    for P in (1, 8):
        gen = torch.Generator().manual_seed(P)
        ctx = torch.randn(2 * P, 77, 768, generator=gen).cuda()
        u = torch.randn(1, 77, 768, generator=gen).cuda().expand(2 * P, -1, -1)
        x = torch.randn(P, 4, 64, 64, generator=gen).cuda().repeat_interleave(2, 0)

        def once(editor):
            regiter_attention_editor_ldm(model, editor)
            try:
                smp.sample(a.steps, 2 * P, (4, 64, 64), {"c_crossattn": [ctx]}, verbose=False, x_T=x, eta=0.0,
                           unconditional_guidance_scale=7.5, unconditional_conditioning={"c_crossattn": [u]})
            finally:
                regiter_attention_editor_ldm(model, None)
        mk = lambda: MutualSelfAttentionControl(5, 12, total_steps=a.steps)
        once(None), once(mk())                                  # capture both graphs
        t = {"plain": [], "masactrl": []}
        for _ in range(a.reps):
            t["plain"].append(host_s(lambda: once(None)))
            t["masactrl"].append(host_s(lambda: once(mk())))
        tp, tm = sorted(t["plain"])[a.reps // 2], sorted(t["masactrl"])[a.reps // 2]
        print(f"  P = {P} (model batch {4 * P}): plain {tp:.3f} s, MasaCtrl {tm:.3f} s, ratio {tm / tp:.4f}; "
              f"spread plain {min(t['plain']):.3f}-{max(t['plain']):.3f}, MasaCtrl {min(t['masactrl']):.3f}-{max(t['masactrl']):.3f}")


def pairs_leg(a, model):
    from anyedit_b200.ddim import DDIMSampler
    from anyedit_b200.masactrl import action_pairs
    print(f"action_pairs end to end at 512^2 ({a.steps} steps, CFG 7.5, VAE decode, uint8 images):")
    smp = DDIMSampler(model)
    gen = torch.Generator().manual_seed(9)
    P = 8
    cond = torch.randn(P, 2, 77, 768, generator=gen).cuda()
    uncond = torch.randn(77, 768, generator=gen).cuda()
    x_T = torch.randn(P, 4, 64, 64, generator=gen).cuda()
    batched = lambda: action_pairs(model, smp, cond, uncond, steps=a.steps, x_T=x_T)
    single = lambda: [action_pairs(model, smp, cond[i:i + 1], uncond, steps=a.steps, x_T=x_T[i:i + 1]) for i in range(P)]
    batched(), single()
    tb = sorted(host_s(batched) for _ in range(a.reps))[a.reps // 2]
    ts = sorted(host_s(single) for _ in range(a.reps))[a.reps // 2]
    print(f"  P = 8 in one call: {tb:.3f} s = {P / tb:.3f} pairs/s ({2 * P / tb:.3f} images/s); "
          f"one pair per call: {ts:.3f} s = {P / ts:.3f} pairs/s")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "diag_masactrl needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    print(f"device: {torch.cuda.get_device_name(0)} | nvidia-smi name, power limit, max SM clock: {q[0] if q else 'n/a'}")
    torch.set_grad_enabled(False)
    kernel_leg(a)
    model = sd15(with_vae=True)
    run_leg(a, model)
    pairs_leg(a, model)


if __name__ == "__main__":
    main()
