"""AnyEdit's inpainting edits, host side (no GPU): the numpy restatement of Pillow's LANCZOS / NEAREST resize, of the inpaint
pipeline's processors and of the background_change mask (OpenCV's 5 x 5 blur, BGR2GRAY, == 0) against the live libraries,
and the launch plan the resize kernel reads (``anysd_pil_resize_plan``, emulated here) against Pillow."""
import numpy as np
import pytest
from PIL import Image

from oracle import inpaint_oracle as O

cv2 = pytest.importorskip("cv2")


def pil(img, size, filt):
    """Image.resize to (H, W); a bool array is a mode "1" image, read back after convert("L")."""
    im = Image.fromarray(img)
    r = im.resize((size[1], size[0]), {"lanczos": Image.LANCZOS, "nearest": Image.NEAREST, "bicubic": Image.BICUBIC}[filt])
    return np.asarray(r.convert("L") if im.mode == "1" else r)


def sweep():
    """Every in-size 1..700 to 512 and 512 to every out-size 1..700, on each axis."""
    out = []
    for s in range(1, 701):
        out += [((s, 9), (512, 9)), ((9, s), (9, 512)), ((512, 9), (s, 9)), ((9, 512), (9, s))]
    return out


def test_lanczos_sweep_equals_pillow():
    rng = np.random.default_rng(3)
    bad = []
    for (H, W), size in sweep():
        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        if not np.array_equal(O.resize(img, size, "lanczos"), pil(img, size, "lanczos")):
            bad.append(((H, W), size))
    assert not bad, bad[:10]


def test_nearest_mode1_sweep_equals_pillow():
    rng = np.random.default_rng(4)
    bad = []
    for (H, W), size in sweep():
        m = rng.integers(0, 2, (H, W)).astype(bool)
        if not np.array_equal(O.resize_mask(m, size), pil(m, size, "lanczos")):       # Pillow forces NEAREST for mode "1"
            bad.append(((H, W), size))
    assert not bad, bad[:10]


def content():
    out = []
    for H, W in [(37, 61), (300, 451), (640, 480), (512, 512), (700, 533)]:
        for y, x in [(0, 0), (H // 2, W // 3), (H - 1, W - 1)]:          # impulses expose the coefficients
            im = np.zeros((H, W, 3), np.uint8)
            im[y, x] = (255, 128, 1)
            out.append(im)
        out += [np.full((H, W, 3), v, np.uint8) for v in (0, 1, 254, 255)]
        yy, xx = np.mgrid[0:H, 0:W]
        for p in (1, 2, 3):                                                  # 0/255 checkerboards: ringing and clipping
            out.append(np.repeat((((yy // p + xx // p) % 2) * 255).astype(np.uint8)[..., None], 3, -1))
    return out


@pytest.mark.parametrize("mode", ["RGB", "L"])
def test_lanczos_content_both_axes_equal_pillow(mode):
    for img in content():
        x = img if mode == "RGB" else np.ascontiguousarray(img[..., 0])
        for size in ((512, 512), (333, 700), (700, 333), (64, 48)):
            assert np.array_equal(O.resize(x, size, "lanczos"), pil(x, size, "lanczos")), (x.shape, size)


def test_masks_after_jpeg_round_trip():
    """A 0/255 mask saved as JPEG and read back (what the tool's masks go through), as mode "L" and, thresholded, mode "1"."""
    rng = np.random.default_rng(5)
    for H, W in [(480, 640), (512, 512), (333, 517)]:
        m = np.zeros((H, W), np.uint8)
        y0, x0 = rng.integers(0, H // 2), rng.integers(0, W // 2)
        m[y0:y0 + H // 3, x0:x0 + W // 4] = 255
        m = cv2.imdecode(cv2.imencode(".jpg", m)[1], cv2.IMREAD_GRAYSCALE)
        assert np.array_equal(O.resize_mask(m, (512, 512)), pil(m, (512, 512), "lanczos"))
        b = m > 127
        assert np.array_equal(O.resize_mask(b, (512, 512)), pil(b, (512, 512), "lanczos"))


def test_prepare_equals_the_processors():
    """diffusers' processors written with numpy + Pillow: image (resize LANCZOS, /255, *2-1), mask (resize, L, /255,
    binarise), masked image = image * (mask < 0.5), mask latent = nearest F.interpolate to size / 8."""
    rng = np.random.default_rng(6)
    img = rng.integers(0, 256, (300, 451, 3), dtype=np.uint8)
    for mask in (rng.integers(0, 2, (300, 451)).astype(bool), (rng.integers(0, 2, (200, 97)) * 255).astype(np.uint8)):
        masked, m, ml, n = O.prepare(img, mask, 128)
        x = np.asarray(Image.fromarray(img).resize((128, 128), Image.LANCZOS)).astype(np.float32) / 255.0
        x = (2.0 * x - 1.0).transpose(2, 0, 1)
        mm = np.asarray(Image.fromarray(mask).resize((128, 128), Image.LANCZOS).convert("L")).astype(np.float32) / 255.0
        mm = (mm >= 0.5).astype(np.float32)[None]
        assert np.array_equal(m, mm) and n == int(mm.sum())
        assert np.array_equal(masked.view(np.uint32), (x * (mm < 0.5)).view(np.uint32))           # -0.0 included
        assert np.array_equal(ml, mm[:, ::8, ::8])


def test_background_mask_equals_opencv():
    rng = np.random.default_rng(7)
    sizes = [(1, 1), (1, 5), (2, 2), (2, 3), (3, 7), (5, 4), (37, 61), (300, 451), (480, 640)]
    for H, W in sizes:
        for kind in ("noise", "jpeg", "const0", "const1"):
            if kind == "noise":
                f = rng.integers(0, 3, (H, W, 3)).astype(np.uint8)
            elif kind == "jpeg":
                f = np.zeros((H, W), np.uint8)
                f[H // 4:H // 4 + max(1, H // 2), W // 3:W // 3 + max(1, W // 3)] = 255
                f = cv2.imdecode(cv2.imencode(".jpg", np.repeat(f[..., None], 3, -1))[1], cv2.IMREAD_COLOR)
            else:
                f = np.full((H, W, 3), int(kind[-1]), np.uint8)
            ref = cv2.cvtColor(cv2.GaussianBlur(f, (5, 5), 0), cv2.COLOR_BGR2GRAY) == 0
            assert np.array_equal(O.gaussian5(f), cv2.GaussianBlur(f, (5, 5), 0)), (H, W, kind)
            assert np.array_equal(O.background_mask(f), ref), (H, W, kind)


# ---- the kernel's plan (anysd_pil_resize_plan) emulated ------------------------------------------------------------------
def _lib_or_skip():
    from anyedit_b200 import _lib
    try:
        _lib.load()
    except _lib.AnysdError as e:
        pytest.skip(str(e))


def emulate(img, size, filt):
    """What pil_resize_kernel computes from the plan: horizontal pass of every source row clipped to bytes, then vertical."""
    from anyedit_b200 import ops
    x = img[..., None] if img.ndim == 2 else img
    H, W, C = x.shape
    table, R, sm, nb = ops.pil_resize_plan([(H, W, *size)], [filt], C)
    t = table.numpy().astype(np.int64)
    OH, OW, ox, sx, oy, sy = t[2], t[3], t[4], t[5], t[6], t[7]

    def matrix(off, stride, n, n_in):
        m = np.zeros((n, n_in), np.int64)
        for i in range(n):
            e = t[off + i * stride:off + (i + 1) * stride]
            m[i, e[0]:e[0] + e[1]] = e[2:2 + e[1]]
        return m

    def run(src, m):                                              # one pass along axis 0 of src: clip((m src + 2^21) >> 22)
        return np.clip((np.einsum("oi,i...->o...", m, src.astype(np.int64)) + (1 << 21)) >> 22, 0, 255).astype(np.uint8)
    h = np.moveaxis(run(np.moveaxis(x, 1, 0), matrix(ox, sx, OW, W)), 0, 1)
    y = run(h, matrix(oy, sy, OH, H))
    return y[..., 0] if img.ndim == 2 else y


def test_kernel_plan_equals_pillow():
    """The plan of every sweep size pair, and a few where both axes change, for RGB and L LANCZOS, mode "1" and L NEAREST."""
    _lib_or_skip()
    rng = np.random.default_rng(8)
    cases = sweep() + [((1, 1), (5, 7)), ((37, 61), (512, 512)), ((512, 512), (300, 451)), ((700, 533), (512, 512)),
                       ((512, 512), (512, 512)), ((3, 512), (3, 1))]
    bad = []
    for (H, W), size in cases:
        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        g = np.ascontiguousarray(img[..., 1])
        m = rng.integers(0, 2, (H, W)).astype(bool)
        for got, want in ((emulate(img, size, "lanczos"), pil(img, size, "lanczos")),
                          (emulate(g, size, "lanczos"), pil(g, size, "lanczos")),
                          (emulate(m.view(np.uint8), size, "mode1"), pil(m, size, "nearest")),
                          (emulate(g, size, "nearest"), pil(g, size, "nearest"))):
            if not np.array_equal(got, want):
                bad.append(((H, W), size))
    assert not bad, bad[:10]


def test_kernel_plan_refusals():
    _lib_or_skip()
    from anyedit_b200 import ops
    with pytest.raises(ValueError):
        ops.pil_resize_plan([(0, 5, 5, 5)], ["lanczos"], 3)
    with pytest.raises(ValueError):
        ops.pil_resize_plan([(5, 5, 5, 5)], ["bilinear"], 3)
    with pytest.raises(ValueError):
        ops.pil_resize_plan([(5, 5, 5, 5)], ["mode1"], 3)
    with pytest.raises(ValueError):
        ops.pil_resize_plan([(5, 5, 5, 5)], ["lanczos"], 4)


# ---- the reference golden (tests/golden/make_golden_inpaint.py) ------------------------------------------------------------
def test_oracle_matches_reference_golden():
    """The restatement chain (processors, encoder, posterior draw, 9-channel UNet with hybrid conditioning, PLMS) against the
    reference's own Encoder, UNetModel(in_channels=9) and PLMSSampler: the prepared tensors exactly, the final latents of a
    CFG 7.5 and an unguided run within 1e-5."""
    import json
    import os
    import torch
    from oracle import ddim_oracle, plms_oracle, unet_oracle, vae_oracle, weights
    G = os.path.join(os.path.dirname(__file__), "golden")
    g = np.load(os.path.join(G, "inpaint_tiny.npz"))
    meta = json.load(open(os.path.join(G, "inpaint_keys.json")))
    sd_u = weights.make_state_dict({k: tuple(v) for k, v in meta["unet_keys"].items()}, int(g["seed_u"]))
    sd_v = weights.make_state_dict({k: tuple(v) for k, v in meta["vae_keys"].items()}, int(g["seed_v"]))
    assert weights.checksum(sd_u) == pytest.approx(float(g["wsum_u"]), rel=1e-12)
    assert weights.checksum(sd_v) == pytest.approx(float(g["wsum_v"]), rel=1e-12)
    size, S = int(g["size"]), int(g["steps"])
    noise = torch.from_numpy(g["noise"])
    cc = []
    for i in range(2):
        masked, _, ml, _ = O.prepare(g[f"img{i}"], g[f"mask{i}"], size)
        assert np.array_equal(masked, g["masked"][i]) and np.array_equal(ml, g["mask_latent"][i]), i
        with torch.no_grad():
            mom = vae_oracle.vae_encode_moments(sd_v, torch.from_numpy(masked)[None])
        mean, logvar = mom.chunk(2, 1)
        z = 0.18215 * (mean + torch.exp(0.5 * logvar.clamp(-30.0, 20.0)) * noise[i:i + 1])
        cc.append(torch.cat([torch.from_numpy(ml)[None], z], 1))
    cc = torch.cat(cc)
    assert float((cc - torch.from_numpy(g["c_concat"])).norm() / torch.from_numpy(g["c_concat"]).norm()) < 1e-5
    sched = ddim_oracle.register_schedule("linear", 1000, 0.00085, 0.012)
    fn = lambda x, t, c: unet_oracle.unet_forward(sd_u, torch.cat([x, cc.repeat(x.shape[0] // 2, 1, 1, 1)], 1), t, c, None,
                                                  num_heads=meta["unet"]["num_heads"])
    ctx, uctx = torch.from_numpy(g["ctx"]), torch.from_numpy(g["uctx"])
    for scale in (float(g["scale"]), 1.0):
        with torch.no_grad():
            img, _ = plms_oracle.plms_sample(fn, sched, S, torch.from_numpy(g["x_T"]), ctx,
                                             uctx[None].expand(2, -1, -1) if scale != 1.0 else None, scale)
        ref = torch.from_numpy(g[f"final_{scale:g}"])
        e = float((img - ref).norm() / ref.norm())
        assert e < 1e-5, (scale, e)


# ---- loading ---------------------------------------------------------------------------------------------------------------
def test_latent_inpaint_diffusion_alias_and_yaml_params():
    """The yaml target of ldm's v1-inpainting config resolves to LatentInpaintDenoiser; its training-only params are accepted,
    unknown ones and other concat layouts are refused."""
    from anyedit_b200.diffusion import LatentInpaintDenoiser, instantiate_from_config
    unet = {"target": "anyedit_b200.ldm.modules.diffusionmodules.openaimodel.UNetModel",
            "params": dict(image_size=8, in_channels=9, model_channels=32, out_channels=4, num_res_blocks=1,
                           attention_resolutions=[1], channel_mult=[1], num_heads=2, use_spatial_transformer=True, context_dim=32)}
    params = dict(linear_start=0.00085, linear_end=0.0120, num_timesteps_cond=1, log_every_t=200, timesteps=1000,
                  first_stage_key="jpg", cond_stage_key="txt", image_size=64, channels=4, cond_stage_trainable=False,
                  conditioning_key="hybrid", monitor="val/loss_simple_ema", scale_factor=0.18215, use_ema=False,
                  finetune_keys=None, unet_config=unet, first_stage_config={"target": "ldm.models.autoencoder.AutoencoderKL"},
                  cond_stage_config={"target": "ldm.modules.encoders.modules.FrozenCLIPEmbedder"})
    m = instantiate_from_config({"target": "anyedit_b200.ldm.models.diffusion.ddpm.LatentInpaintDiffusion", "params": params})
    assert isinstance(m, LatentInpaintDenoiser) and m.concat_keys == ("mask", "masked_image") and m.scale_factor == 0.18215
    assert m.model.conditioning_key == "hybrid" and m.model.diffusion_model.in_channels == 9
    with pytest.raises(TypeError):
        LatentInpaintDenoiser(unet, not_an_ldm_param=1)
    with pytest.raises(NotImplementedError):
        LatentInpaintDenoiser(unet, concat_keys=("masked_image",))


def test_inpainting_checkpoint_key_layout():
    """The ldm layout of sd-v1-5-inpainting: SD-1.5's UNet keys under model.diffusion_model. with the input conv widened to 9
    channels, every shape equal; a state_dict with the text encoder's keys loads with strict=False and nothing missing."""
    import json
    import os
    import torch
    from anyedit_b200.diffusion import LatentInpaintDenoiser
    from anyedit_b200.unet import UNetModel
    meta = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "sd15_keys.json")))
    want = {"model.diffusion_model." + k: tuple(v) for k, v in meta["keys"].items()}
    want["model.diffusion_model.input_blocks.0.0.weight"] = (320, 9, 3, 3)
    with torch.device("meta"):
        net = UNetModel(**dict(meta["config"], in_channels=9))
    m = LatentInpaintDenoiser(net)
    got = {k: tuple(v.shape) for k, v in m.state_dict().items() if k.startswith("model.")}
    assert got == want
    # strict=False on a small model: the encoder's keys are left over, nothing the sampler path needs is missing
    net = UNetModel(image_size=8, in_channels=9, model_channels=32, out_channels=4, num_res_blocks=1, attention_resolutions=[1],
                    channel_mult=[1], num_heads=2, use_spatial_transformer=True, context_dim=32)
    small = LatentInpaintDenoiser(net)
    sd = {k: torch.zeros(v.shape) for k, v in small.state_dict().items()}
    sd["cond_stage_model.transformer.text_model.embeddings.position_ids"] = torch.zeros(1, 77)
    r = small.load_state_dict(sd, strict=False)
    assert not r.missing_keys and r.unexpected_keys == ["cond_stage_model.transformer.text_model.embeddings.position_ids"]
