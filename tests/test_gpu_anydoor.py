"""AnyDoor's visual-reference edit on the GPU (``anyedit_b200.anydoor``, kernels in csrc/anydoor.cu).

* every stage against the reference's bytes (tests/golden/make_golden_anydoor.py): ref / jpg / hint bit for bit (SHA-256 of the
  fp32 arrays), the high-frequency map byte for byte, the integer geometry; the uint8 stages against the oracle;
* crop_back against the oracle (which equals the golden): equal except where the fp32 value lies within 1e-4 of an integer, and
  there by at most 1;
* the generic uint8 resize against live OpenCV; a batch of mixed geometries against per-pair calls; two calls alike; a CUDA-graph
  replay of the pixel kernels against eager; the refusals;
* the whole request on tiny seeded ControlNet / UNet / DINOv2 / VAE models with a fixed x_T: ``inference_single_image`` against
  the reference's composition on the host (the golden-pinned oracle's preparation -> the same models -> the oracle's crop_back),
  pixels outside the crop interior untouched, and ``edit_pairs`` pair i == ``inference_single_image`` of pair i.
"""
import hashlib
import os
import types

import numpy as np
import pytest
import torch

from oracle import anydoor_oracle as O

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.fixture(scope="module")
def A():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from anyedit_b200 import anydoor, ops
    assert tuple(ops.device_info())[1:] == (9, 0), "sm_90a kernels need a Hopper GPU (H100)"
    return anydoor


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(G, "anydoor_golden.npz"))


def batch(names):
    ins = [O.case_inputs(n) for n in names]
    return [np.stack([x[i] for x in ins]) for i in range(4)], [x[4] for x in ins]


@pytest.mark.parametrize("name", list(O.CASES))
def test_prepare_vs_reference_golden(A, gold, name):
    ri, rm, ti, tm, seed = O.case_inputs(name)
    np.random.seed(seed)
    item = A.process_pairs(ri, rm, ti, tm)
    assert item["ref"].dtype == np.float64 and item["jpg"].dtype == item["hint"].dtype == np.float32
    for k in ("ref", "jpg", "hint"):
        assert sha(item[k].astype(np.float32)) == str(gold[f"{name}/{k}"]), k
    assert np.array_equal(item["extra_sizes"], gold[f"{name}/extra_sizes"])
    assert np.array_equal(item["tar_box_yyxx_crop"], gold[f"{name}/tar_box_yyxx_crop"])
    st = {}
    np.random.seed(seed)
    O.process_pairs(ri, rm, ti, tm, stages=st)
    np.random.seed(seed)
    dev, _, _ = A._prepare(ri[None], rm[None], ti[None], tm[None])
    assert np.array_equal(dev["ref_u8"][0].cpu().numpy(), st["ref_u8"])
    assert np.array_equal(dev["mask_u8"][0].cpu().numpy(), st["ref_mask_u8"])
    assert sha(dev["hf224"][0].cpu().numpy()) == str(gold[f"{name}/hf"])
    assert np.array_equal(A.sobel(st["ref_u8"], st["ref_mask_u8"] / 255), dev["hf224"][0].cpu().numpy())
    print(f"[anydoor prepare] {name}: ref / jpg / hint and the high-frequency map equal the reference's bit for bit")


@pytest.mark.parametrize("name", list(O.CASES))
def test_crop_back_vs_golden(A, gold, name):
    ri, rm, ti, tm, seed = O.case_inputs(name)
    np.random.seed(seed)
    item = O.process_pairs(ri, rm, ti, tm)
    pred = O.decode_to_pred(O.case_pred(seed))
    want = O.crop_back(pred, ti, item["extra_sizes"], item["tar_box_yyxx_crop"])
    assert sha(want) == str(gold[f"{name}/crop_back"])
    tcopy = ti.copy()
    got = A.crop_back(pred, tcopy, item["extra_sizes"], item["tar_box_yyxx_crop"])
    assert np.array_equal(tcopy, ti), "the caller's image must be left alone"
    # the same through the decoder-output path (scale, clip and row drop in the kernel)
    g = torch.tensor([A._crop_row(item["extra_sizes"], item["tar_box_yyxx_crop"])], dtype=torch.int32, device="cuda")
    t = torch.from_numpy(ti)[None].cuda()
    out = torch.empty_like(t)
    from anyedit_b200 import ops
    ops.anydoor_crop_back(torch.from_numpy(O.case_pred(seed))[None].cuda(), t, g, out)
    H1, W1, H2, W2 = (int(v) for v in item["extra_sizes"])
    vals = O.resize_f32(pred, (W2, H2))
    near = np.abs(vals - np.rint(vals)) < 1e-4
    y1, y2, x1, x2 = (int(v) for v in item["tar_box_yyxx_crop"])
    for res in (got, out[0].cpu().numpy()):
        d = np.abs(res.astype(np.int64) - want)
        ok = np.zeros(want.shape, bool)
        qy, qx, _ = A._pad_offsets(H1, W1)
        ok[y1:y2, x1:x2] = near[qy:qy + H1, qx:qx + W1]
        print(f"[crop_back] {name}: {int((d > 0).sum())} bytes differ from the golden, all within 1e-4 of an integer")
        assert d.max() <= 1 and not (d[~ok] > 0).any()


@pytest.mark.parametrize("src,dst", [((224, 224), (256, 256)), ((256, 256), (224, 224)), ((480, 640), (512, 512)),
                                     ((417, 300), (512, 512)), ((224, 224), (112, 112)), ((61, 93), (7, 200)), ((1, 5), (3, 1))])
def test_resize_u8_vs_live_cv2(A, src, dst):
    cv2 = pytest.importorskip("cv2")
    from anyedit_b200 import ops
    img = np.random.default_rng(sum(src) + sum(dst)).integers(0, 256, (2,) + src + (3,), dtype=np.uint8)
    out = torch.empty((2,) + dst + (3,), dtype=torch.uint8, device="cuda")
    ops.resize_linear_u8(torch.from_numpy(img).cuda(), out)
    for b in range(2):
        assert np.array_equal(out[b].cpu().numpy(), cv2.resize(img[b], (dst[1], dst[0])))


def test_batch_equals_single_repeat_and_graph(A):
    names = list(O.CASES)
    (ri, rm, ti, tm), seeds = batch([n for n in names if O.CASES[n][0] == (512, 512)])
    np.random.seed(7)
    st, geoms, g = A._prepare(ri, rm, ti, tm)
    keys = ("ref_u8", "mask_u8", "hf224", "ref", "jpg", "hint")
    np.random.seed(7)
    for i in range(len(ri)):
        one, (g1,), _ = A._prepare(ri[i:i + 1], rm[i:i + 1], ti[i:i + 1], tm[i:i + 1])
        assert g1 == geoms[i]
        for k in keys:
            assert torch.equal(one[k][0], st[k][i]), (i, k)
    np.random.seed(7)
    st2, _, _ = A._prepare(ri, rm, ti, tm)
    assert all(torch.equal(st[k], st2[k]) for k in keys)
    # the pixel kernels replayed from a CUDA graph
    from anyedit_b200 import ops
    dev = [torch.from_numpy(x).cuda() for x in (ri, rm, ti)]
    outs = {k: torch.zeros_like(v) for k, v in st.items()}
    ops.anydoor_prepare(*dev, g, outs)
    torch.cuda.synchronize()
    for v in outs.values():
        v.zero_()
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            ops.anydoor_prepare(*dev, g, outs)
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(outs[k], st[k]) for k in keys)


def test_refusals(A):
    img, m = np.zeros((64, 64, 3), np.uint8), np.ones((64, 64), np.uint8)
    for bad in ((img.astype(np.float32), m, img, m), (img, m * 2, img, m), (img, m[:32], img, m), (img[..., :2], m, img, m)):
        with pytest.raises(ValueError):
            A.process_pairs(*bad)
    t, mt = torch.from_numpy(img).cuda(), torch.from_numpy(m * 3).cuda()
    with pytest.raises(ValueError, match="0 or 1"):
        A.process_pairs(t, mt, t, torch.from_numpy(m).cuda())
    with pytest.raises(RuntimeError, match="CUDA"):
        A.process_pairs(torch.from_numpy(img), torch.from_numpy(m), torch.from_numpy(img), torch.from_numpy(m))
    args = types.SimpleNamespace(H=256, W=512, num_samples=1, ddim_steps=2, guidance_scale=3.0, strength=1.0)
    with pytest.raises(ValueError, match="8 x"):
        A.inference_single_image(None, None, img, m, img, m, args)


# ---- the whole request on tiny models -----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def models(A):
    from anyedit_b200.autoencoder import AutoencoderKL
    from anyedit_b200.cldm import ControlDenoiser, ControlledUnetModel, ControlNet
    from anyedit_b200.ddim import DDIMSampler
    from anyedit_b200.encoders import FrozenDinoV2Encoder
    from oracle import weights
    import json
    meta = json.load(open(os.path.join(G, "cldm_tiny_keys.json")))
    cn = ControlNet(**dict(meta["control_config"], hint_channels=4))
    un = ControlledUnetModel(**meta["unet_config"])
    dm = json.load(open(os.path.join(G, "dinov2_tiny_keys.json")))
    enc = FrozenDinoV2Encoder(config=dict(dm["config"], image_size=224, projection_dim=meta["unet_config"]["context_dim"]))
    vm = json.load(open(os.path.join(G, "vae_tiny_keys.json")))
    vae = AutoencoderKL(dict(vm["config"], ch_mult=[1, 2, 2, 4]), embed_dim=4)
    for i, net in enumerate((cn, un, enc, vae)):
        net.load_state_dict(weights.make_state_dict({k: tuple(v.shape) for k, v in net.state_dict().items()}, 41 + i,
                                                    scheme="torch"), strict=True)
    model = ControlDenoiser(un.cuda(), cn.cuda(), cond_stage_model=enc.cuda(), first_stage_model=vae.cuda(),
                            scale_factor=0.18215).cuda()
    return model, DDIMSampler(model)


def test_inference_single_image_vs_host_composition(A, models):
    model, sampler = models
    ri, rm, ti, tm, seed = O.case_inputs("blob512")
    args = types.SimpleNamespace(H=512, W=512, num_samples=2, ddim_steps=4, guidance_scale=5.0, strength=0.8)
    x_T = torch.randn(2, 4, 64, 64, generator=torch.Generator().manual_seed(3)).cuda()
    np.random.seed(seed)
    got = A.inference_single_image(model, sampler, ri, rm, ti.copy(), tm, args, x_T=x_T)
    # the reference's composition on the host: the oracle's preparation, the same models, the oracle's crop_back
    np.random.seed(seed)
    item = O.process_pairs(ri, rm, ti, tm)
    control = torch.from_numpy(item["hint"]).cuda().permute(2, 0, 1)[None].repeat(2, 1, 1, 1).contiguous()
    clip = torch.from_numpy(item["ref"].astype(np.float32)).cuda().permute(2, 0, 1)[None].repeat(2, 1, 1, 1)
    cond = {"c_concat": [control], "c_crossattn": [model.get_learned_conditioning(torch.cat([clip, torch.zeros_like(clip)]))[:2]]}
    unc = {"c_concat": [control], "c_crossattn": [model.get_learned_conditioning(torch.cat([clip, torch.zeros_like(clip)]))[2:]]}
    model.control_scales = [0.8] * 13
    samples, _ = sampler.sample(4, 2, (4, 64, 64), cond, verbose=False, eta=0.0, unconditional_guidance_scale=5.0,
                                unconditional_conditioning=unc, x_T=x_T)
    dec = model.decode_first_stage(samples).float().cpu().numpy()
    want = O.crop_back(O.decode_to_pred(dec[0]), ti, item["extra_sizes"], item["tar_box_yyxx_crop"])
    assert np.isfinite(dec).all()
    y1, y2, x1, x2 = (int(v) for v in item["tar_box_yyxx_crop"])
    inner = np.zeros(ti.shape[:2], bool)
    inner[y1 + 5:y2 - 5, x1 + 5:x2 - 5] = True
    assert np.array_equal(got[~inner], ti[~inner])
    d = np.abs(got.astype(np.int64) - want)
    print(f"[inference_single_image] {int((d > 0).sum())} of {d.size} bytes differ from the host composition; "
          f"{int(inner.sum())} pixels pasted")
    assert d.max() == 0


def test_edit_pairs_equals_single_requests(A, models):
    model, sampler = models
    names = ["blob512", "wide", "square"]
    (ri, rm, ti, tm), _ = batch(names)
    x_T = torch.randn(3, 4, 64, 64, generator=torch.Generator().manual_seed(9)).cuda()
    np.random.seed(11)
    out = A.edit_pairs(model, sampler, ri, rm, ti, tm, steps=4, guidance_scale=5.0, strength=1.0, x_T=x_T)
    args = types.SimpleNamespace(H=512, W=512, num_samples=1, ddim_steps=4, guidance_scale=5.0, strength=1.0)
    np.random.seed(11)
    for i in range(3):
        one = A.inference_single_image(model, sampler, ri[i], rm[i], ti[i], tm[i], args, x_T=x_T[i:i + 1])
        d = int((one != out[i]).sum())
        print(f"[edit_pairs] pair {i} ({names[i]}): {d} bytes differ from its single request")
        assert d == 0
