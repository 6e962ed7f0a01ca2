"""AnyEdit's inpainting edits (anyedit_b200.inpaint, csrc/inpaint.cu) on the GPU.

* Bytes: the ragged Pillow resize against live Pillow on several hundred sizes in one launch (RGB LANCZOS, L LANCZOS, mode "1"
  NEAREST), each image equal to its own launch; the background mask and its counts against OpenCV; the prepared masked
  image against fp16 of the processors' float32 formula, bit for bit, the mask latent and the counts exactly.
* The tiny 9-channel inpainting model (seeded weights, a factor-8 first stage) end to end: prepare, encoder, posterior draw,
  PLMS with and without guidance, against the float32 CPU oracle (oracle/inpaint_oracle + vae_oracle + unet_oracle +
  plms_oracle) run here.  Bound: final-latent rel-L2 < 5e-3, the bar of every CFG sampling run against fp32 in this suite
  (test_gpu_unet.test_ddim_tiny_golden, test_gpu_masactrl).  Its origin: fp16 activations and weights carry a relative error of
  2^-11 per rounding; the UNet's relative error per eps is ~1e-3 (test_gpu_unet), guidance multiplies the eps difference by
  the scale, and the PLMS update adds the combined eps with coefficients below 1 per step, so a handful of steps stays
  within a few 1e-3.  Here the encoder's input is also fp16 (the kernels' contract), which adds 2^-12 relative to the
  masked image and thus to the posterior mean.
* Identities, bit for bit: graph replay and eager; request i of a B = 3 ragged batch and the single request; the shared
  CFG halves on and off (and that the shared path is taken).
"""
import json
import os

import numpy as np
import pytest
import torch
from PIL import Image

pytestmark = pytest.mark.gpu

cv2 = pytest.importorskip("cv2")

G = os.path.join(os.path.dirname(__file__), "golden")
LATENT_TOL = 5e-3
SD15_TOL = 5e-3
SIZE, STEPS = 128, 6


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def pil(img, size, filt=Image.LANCZOS):
    im = Image.fromarray(img)
    r = im.resize((size[1], size[0]), filt)
    return np.asarray(r.convert("L") if im.mode == "1" else r)


# ---- bytes -----------------------------------------------------------------------------------------------------------------
def _sizes():
    out = []
    for s in list(range(1, 701, 7)) + [511, 512, 513, 700]:
        out += [((s, 64), (512, 64)), ((64, s), (64, 512)), ((512, 48), (s, 48)), ((48, 512), (48, s))]
    out += [((480, 640), (512, 512)), ((512, 512), (480, 640)), ((1, 1), (512, 512)), ((512, 512), (1, 1)), ((700, 533), (333, 517))]
    return out


@pytest.mark.parametrize("kind", ["RGB", "L", "1"])
def test_ragged_resize_equals_pillow(kind):
    from anyedit_b200 import ops
    rng = np.random.default_rng({"RGB": 1, "L": 2, "1": 3}[kind])
    cases = _sizes()
    C = 3 if kind == "RGB" else 1
    srcs = []
    for (H, W), _ in cases:
        if kind == "1":
            srcs.append(rng.integers(0, 2, (H, W)).astype(bool))
        else:
            srcs.append(rng.integers(0, 256, (H, W, C) if C == 3 else (H, W), dtype=np.uint8))
    dev = [torch.from_numpy(np.ascontiguousarray(s.view(np.uint8))).cuda().reshape(*s.shape[:2], C) for s in srcs]
    outs = [torch.empty(*o, C, dtype=torch.uint8, device="cuda") for _, o in cases]
    filt = "mode1" if kind == "1" else "lanczos"
    ops.pil_resize(dev, outs, [filt] * len(cases))
    bad = []
    for s, (_, o), got in zip(srcs, cases, outs):
        ref = pil(s, o)
        if not np.array_equal(got.cpu().numpy().reshape(ref.shape), ref):
            bad.append((s.shape, o))
    assert not bad, (len(cases), bad[:10])
    for i in (0, 57, len(cases) - 1):                             # batch independence: the same bytes alone
        one = torch.empty_like(outs[i])
        ops.pil_resize([dev[i]], [one], [filt])
        assert torch.equal(one, outs[i])


def test_background_mask_equals_opencv():
    from anyedit_b200 import inpaint
    rng = np.random.default_rng(4)
    fores = []
    for H, W in [(1, 1), (2, 3), (5, 4), (37, 61), (300, 451), (480, 640), (1024, 77)]:
        f = np.zeros((H, W), np.uint8)
        f[H // 4:H // 4 + max(1, H // 2), W // 3:W // 3 + max(1, W // 3)] = 255
        f = cv2.imdecode(cv2.imencode(".jpg", np.repeat(f[..., None], 3, -1))[1], cv2.IMREAD_COLOR)
        fores.append(f)
        fores.append(rng.integers(0, 3, (H, W, 3)).astype(np.uint8))
    masks, counts = inpaint.background_mask(fores)
    for f, m, n in zip(fores, masks, counts):
        ref = cv2.cvtColor(cv2.GaussianBlur(f, (5, 5), 0), cv2.COLOR_BGR2GRAY) == 0
        assert m.dtype == torch.bool and np.array_equal(m.cpu().numpy(), ref), f.shape
        assert int(n) == int(ref.sum())


def test_prepare_bit_exact():
    from anyedit_b200 import inpaint
    from oracle import inpaint_oracle as O
    rng = np.random.default_rng(5)
    imgs = [rng.integers(0, 256, s, dtype=np.uint8) for s in ((300, 451, 3), (512, 512, 3), (97, 130, 3))]
    masks = [rng.integers(0, 2, (300, 451)).astype(bool), (rng.integers(0, 2, (64, 64)) * 255).astype(np.uint8),
             rng.integers(0, 256, (97, 130), dtype=np.uint8)]
    st = inpaint.prepare(imgs, masks, 512, 64)
    for i, (im, m) in enumerate(zip(imgs, masks)):
        masked, mb, ml, n = O.prepare(im, m, 512)
        want = masked.transpose(1, 2, 0).astype(np.float16)
        got = st["masked"][i].cpu().numpy()
        assert np.array_equal(got[..., :3].view(np.uint16), want.view(np.uint16)), i
        assert not got[..., 3:].any()
        assert np.array_equal(st["mask_latent"][i].cpu().numpy(), ml) and int(st["counts"][i]) == n


# ---- the tiny inpainting model ---------------------------------------------------------------------------------------------
def _tiny():
    """The golden's tiny model (tests/golden/make_golden_inpaint.py): its configs, its state-dict names and seeds."""
    from anyedit_b200.autoencoder import AutoencoderKL
    from anyedit_b200.diffusion import LatentInpaintDenoiser
    from anyedit_b200.unet import UNetModel
    from oracle import weights
    meta = json.load(open(os.path.join(G, "inpaint_keys.json")))
    g = np.load(os.path.join(G, "inpaint_tiny.npz"))
    net = UNetModel(**meta["unet"])
    sd_u = weights.make_state_dict({k: tuple(v) for k, v in meta["unet_keys"].items()}, int(g["seed_u"]))
    net.load_state_dict(sd_u, strict=True)
    vae = AutoencoderKL(meta["vae"], embed_dim=4)
    sd_v = weights.make_state_dict({k: tuple(v) for k, v in meta["vae_keys"].items()}, int(g["seed_v"]))
    vae.load_state_dict(sd_v, strict=True)
    model = LatentInpaintDenoiser(net.cuda(), first_stage_model=vae.cuda(), scale_factor=0.18215).cuda()
    return model, sd_u, sd_v


@pytest.fixture(scope="module")
def tiny():
    return _tiny()


def _requests(B=3, seed=9):
    gen = np.random.default_rng(seed)
    sizes = [(150, 201), (128, 128), (90, 160)][:B]
    imgs = [gen.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in sizes]
    masks = []
    for i, (h, w) in enumerate(sizes):
        m = np.zeros((h, w), np.uint8)
        m[h // 4:3 * h // 4, w // 5:w // 2] = 255
        masks.append(m > 0 if i % 2 == 0 else m)                    # mode "1" and mode "L"
    g = torch.Generator().manual_seed(seed)
    cond = torch.randn(B, 7, 32, generator=g)
    uncond = torch.randn(7, 32, generator=g)
    x_T = torch.randn(B, 4, SIZE // 8, SIZE // 8, generator=g)
    noise = torch.randn(B, 4, SIZE // 8, SIZE // 8, generator=g)
    return imgs, masks, cond, uncond, x_T, noise


def _run(model, reqs, scale=7.5, graph=True, sampler=None, idx=None):
    from anyedit_b200 import inpaint
    from anyedit_b200.plms import PLMSSampler
    imgs, masks, cond, uncond, x_T, noise = reqs
    if idx is not None:
        imgs, masks = [imgs[i] for i in idx], [masks[i] for i in idx]
        cond, x_T, noise = cond[idx], x_T[idx], noise[idx]
    smp = sampler or PLMSSampler(model, use_cuda_graph=graph)
    return inpaint.inpaint_latents(model, smp, imgs, masks, cond.cuda(), uncond.cuda(), STEPS, scale, x_T.cuda(), noise.cuda(), SIZE)


@pytest.mark.parametrize("scale", [7.5, 1.0])
def test_tiny_model_vs_reference_golden(tiny, scale):
    """The golden's two requests (a mode "1" and a JPEG'd mode "L" mask, two sizes) through prepare, the encoder, the posterior
    draw with the stored noise and PLMS, against the reference's Encoder + UNetModel(in_channels=9) + PLMSSampler."""
    model, _, _ = tiny
    g = np.load(os.path.join(G, "inpaint_tiny.npz"))
    f = lambda k: torch.from_numpy(g[k])
    reqs = ([g["img0"], g["img1"]], [g["mask0"], g["mask1"]], f("ctx"), f("uctx"), f("x_T"), f("noise"))
    assert g["mask0"].dtype == np.bool_ and g["mask1"].dtype == np.uint8
    got = _run(model, reqs, scale)
    e = rel(got, f(f"final_{scale:g}"))
    print(f"[inpaint tiny cfg {scale}] final-latent rel-L2 vs reference golden = {e:.3e}")
    assert e < LATENT_TOL, e


def test_sd15_inpainting_widths_vs_fp32_oracle():
    """SD-1.5-inpainting widths (9 input channels padded to 64 for the input conv, 320 / 640 / 1280 levels), seeded weights at
    a 64^2 latent, 4 PLMS steps (5 model calls; the ldm uniform schedule has no 3-step grid, util.py:46-60) with CFG 7.5 on the hybrid conditioning (c_concat: a binary mask latent and a
    masked-image latent, one tensor for both halves, so the shared-halves path runs), against the fp32 CPU oracle.  Bound
    SD15_TOL = 5e-3, the bar of the SD-1.5 CFG runs of test_gpu_unet / test_gpu_masactrl (measured 3.7e-3 there at 4 DDIM
    steps): the per-eps fp16 error (~1e-3) enters each update once, through combinations whose coefficients sum to 1."""
    from anyedit_b200.diffusion import LatentInpaintDenoiser
    from anyedit_b200.plms import PLMSSampler
    from anyedit_b200.unet import UNetModel
    from oracle import cpu, ddim_oracle, plms_oracle, unet_oracle, weights
    meta = json.load(open(os.path.join(G, "sd15_keys.json")))
    cfg = dict(meta["config"], in_channels=9)
    keys = {k: tuple(v) for k, v in meta["keys"].items()}
    keys["input_blocks.0.0.weight"] = (320, 9, 3, 3)
    sd = weights.make_state_dict(keys, 3, scheme="torch")
    with torch.device("cuda"):
        net = UNetModel(**cfg)
    net.load_state_dict(sd)
    model = LatentInpaintDenoiser(net).cuda()
    gen = torch.Generator().manual_seed(777)
    x_T = torch.randn(1, 4, 64, 64, generator=gen)
    ml = torch.zeros(1, 1, 64, 64)
    ml[..., 10:40, 20:50] = 1
    cc = torch.cat([ml, torch.randn(1, 4, 64, 64, generator=gen) * (1 - ml)], 1)
    ctx, u = torch.randn(1, 77, 768, generator=gen), torch.randn(1, 77, 768, generator=gen)
    S = 4
    smp = PLMSSampler(model)
    ccd = cc.cuda()
    out, _ = smp.sample(S, 1, (4, 64, 64), {"c_concat": [ccd], "c_crossattn": [ctx.cuda()]}, verbose=False, x_T=x_T.cuda(),
                        eta=0.0, unconditional_guidance_scale=7.5, unconditional_conditioning={"c_concat": [ccd], "c_crossattn": [u.cuda()]})
    assert next(iter(smp._graphs.values())).shared
    torch.set_num_threads(cpu.usable_cores())
    sched = ddim_oracle.register_schedule("linear", 1000, 0.00085, 0.012)
    fn = lambda x, t, c: unet_oracle.unet_forward(sd, torch.cat([x, cc.repeat(x.shape[0], 1, 1, 1)], 1), t, c, None,
                                                  num_heads=cfg["num_heads"])
    with torch.no_grad():
        ref, _ = plms_oracle.plms_sample(fn, sched, S, x_T, ctx, u, 7.5)
    e = rel(out, ref)
    print(f"[inpaint sd15 widths 64x64, {S} PLMS steps] final-latent rel-L2 vs fp32 oracle = {e:.3e}")
    assert e < SD15_TOL, e


def test_graph_eager_batch_and_shared_halves_bit_identical(tiny, monkeypatch):
    from anyedit_b200.plms import PLMSSampler
    model, _, _ = tiny
    reqs = _requests(3)
    outs = {}
    for share in ("1", "0"):
        monkeypatch.setenv("ANYSD_SHARE_CFG", share)
        for graph in (True, False):
            smp = PLMSSampler(model, use_cuda_graph=graph)
            outs[(share, graph)] = _run(model, reqs, sampler=smp)
            assert next(iter(smp._graphs.values())).shared == (share == "1")
    ref = outs[("0", False)]
    for k, v in outs.items():
        assert torch.equal(v, ref), k
    monkeypatch.setenv("ANYSD_SHARE_CFG", "1")
    for i in range(3):
        assert torch.equal(_run(model, reqs, idx=[i])[0], ref[i]), i


def test_inpaint_bytes_and_background_change(tiny):
    """inpaint's bytes are decode -> round(clamp(x / 2 + 1/2) * 255) -> LANCZOS to the original size; background_change skips
    a request whose background covers under 5 % and equals inpaint with its bool mask for the others."""
    from anyedit_b200 import inpaint, ops
    from anyedit_b200.plms import PLMSSampler
    model, _, _ = tiny
    imgs, masks, cond, uncond, x_T, noise = _requests(3)
    smp = PLMSSampler(model)
    outs = inpaint.inpaint(model, smp, imgs, masks, cond.cuda(), uncond.cuda(), STEPS, 7.5, x_T.cuda(), noise.cuda(), size=SIZE)
    lat = _run(model, (imgs, masks, cond, uncond, x_T, noise), sampler=smp)
    dec = model.decode_first_stage(lat).float().contiguous()
    u8 = torch.empty(3, SIZE, SIZE, 3, dtype=torch.uint8, device="cuda")
    ops.image_to_u8(dec, u8)
    for i, im in enumerate(imgs):
        assert outs[i].shape == im.shape
        assert np.array_equal(outs[i], pil(u8[i].cpu().numpy(), im.shape[:2]))
    fores = []
    for i, im in enumerate(imgs):
        f = np.zeros(im.shape, np.uint8)
        if i == 1:
            f[:] = 255
            f[:4, :4] = 0                                           # background: 16 pixels, under 5 %
        else:
            f[im.shape[0] // 3:, :] = 255
        fores.append(f)
    res = inpaint.background_change(model, smp, imgs, fores, cond.cuda(), uncond.cuda(), STEPS, 7.5, x_T.cuda(), noise.cuda(),
                                    size=SIZE)
    assert res[1] is None and res[0] is not None and res[2] is not None
    bg, _ = inpaint.background_mask(fores)
    kept = [0, 2]
    want = inpaint.inpaint(model, smp, [imgs[i] for i in kept], [bg[i] for i in kept], cond[kept].cuda(), uncond.cuda(), STEPS,
                           7.5, x_T[kept].cuda(), noise[kept].cuda(), size=SIZE)
    for j, i in enumerate(kept):
        assert np.array_equal(res[i][0], want[j]) and np.array_equal(res[i][1], bg[i].cpu().numpy())
