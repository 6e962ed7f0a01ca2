"""The segmentation annotator on the GPU (``segment.UniFormerSegmentor``) and the kernels it adds:

* the depthwise conv (k 3 and 5, odd sizes, with and without a residual) against float64 ``F.conv2d(groups=C)`` within an
  element-wise bound; the adaptive average pool against float64 ``F.adaptive_avg_pool2d``, overlapping bins included; the
  half-pixel bilinear resize against float64 ``F.interpolate`` (1 x 1 sources, the identity size bit for bit, the addend, a
  channel-slice output); space-to-depth bit for bit on odd sizes, fp16 and uint8; the label kernel against torch's two resizes
  and argmax on the GPU wherever torch's top-two gap is more than a few ulps, and its palette output;
* the tiny model against the reference's golden (backbone outputs, logits, ``inference_segmentor`` labels where the stored margin
  is clear); UniFormer-S + UPerHead at the real width with seeded, BN-randomised weights against the fp32 oracle on a 480 x 640
  image rescaled to 512 x 683; the full-size model for determinism, batch independence and the strict state-dict round trip.

Element bound (terms of tests/test_gpu_depth.py): fp32 sums of n products carry <= n 2^-24 of the sum of magnitudes; one fp16
rounding adds 2^-11 |y| + 2^-25.
"""
import json
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
G = os.path.join(os.path.dirname(__file__), "golden")
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
U = 2.0 ** -24
# rel-L2 tolerances of the model tests, about 3x the values measured on the H100 (DESIGN.md §10.5)
TINY_TOL, TINY_OUT_TOL, REAL_TOL = 2.5e-3, 3.5e-3, 2.5e-3
MARGIN = 0.05               # labels must match the reference wherever its top-two gap exceeds MARGIN x the logits' rms
REAL_AGREE = 0.996          # fraction of real-width labels that agree with the fp32 oracle


def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / b.norm())


@pytest.fixture(scope="module")
def cuda_ops():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from anyedit_b200 import ops
    assert tuple(ops.device_info())[1:] == (9, 0), "sm_90a kernels need a Hopper GPU (H100)"
    return ops


def nchw(t):
    return t.permute(0, 3, 1, 2)


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


# ---- kernels -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [3, 5])
@pytest.mark.parametrize("N,H,W,Cc", [(1, 13, 17, 64), (2, 9, 31, 320), (1, 1, 5, 8)])
def test_dwconv_vs_fp64(cuda_ops, k, N, H, W, Cc):
    g = torch.Generator().manual_seed(k * 100 + H)
    x = torch.randn(N, H, W, Cc, generator=g).half()
    res = torch.randn(N, H, W, Cc, generator=g).half()
    w = torch.randn(Cc, 1, k, k, generator=g) / k
    b = torch.randn(Cc, generator=g) * 0.1
    conv = F.conv2d(nchw(x.double()), w.double(), b.double(), padding=k // 2, groups=Cc)
    mag = F.conv2d(nchw(x.double()).abs(), w.double().abs(), b.double().abs(), padding=k // 2, groups=Cc)
    for r in (None, res):
        y = torch.empty(N, H, W, Cc, dtype=torch.float16, device="cuda")
        cuda_ops.dwconv(x.cuda(), cuda_ops.pack_dwconv(w, "cuda"), b.cuda(), y, residual=r.cuda() if r is not None else None)
        want = nhwc(conv) + (r.double() if r is not None else 0)
        bound = (k * k + 2) * U * (nhwc(mag) + (r.double().abs() if r is not None else 0)) + 2.0 ** -11 * want.abs() + 2.0 ** -25
        q = float(((y.cpu().double() - want).abs() / bound).max())
        print(f"dwconv k={k} {N}x{H}x{W}x{Cc} residual={r is not None}: worst err/bound {q:.3f}")
        assert q <= 1.0


@pytest.mark.parametrize("H,W,o", [(16, 21, 1), (16, 21, 2), (16, 21, 3), (16, 21, 6), (2, 3, 6), (5, 7, 3), (32, 43, 6)])
def test_adaptive_avg_pool_vs_fp64(cuda_ops, H, W, o):
    x = torch.randn(2, H, W, 64, generator=torch.Generator().manual_seed(H * W + o)).half()
    y = torch.empty(2, o, o, 64, dtype=torch.float16, device="cuda")
    cuda_ops.adaptive_avg_pool(x.cuda(), y)
    want = nhwc(F.adaptive_avg_pool2d(nchw(x.double()), o))
    mag = nhwc(F.adaptive_avg_pool2d(nchw(x.double()).abs(), o))
    n = (-(-H // o) + 1) * (-(-W // o) + 1)
    bound = (n + 2) * U * mag + 2.0 ** -11 * want.abs() + 2.0 ** -25
    assert float(((y.cpu().double() - want).abs() / bound).max()) <= 1.0


HALF_PIXEL = [(1, 1, 16, 21), (2, 3, 16, 21), (6, 6, 16, 21), (16, 21, 32, 43), (32, 43, 128, 171), (128, 171, 512, 683),
              (64, 64, 17, 23)]


def _resize_bound(x, ref, H, W):
    m = float(x.abs().max())
    return (4 * 2.0 ** -22 * max(H, W) + 16 * U) * m + 2.0 ** -11 * ref.abs() + 2.0 ** -25


@pytest.mark.parametrize("H,W,Ho,Wo", HALF_PIXEL)
def test_resize_half_pixel_vs_fp64(cuda_ops, H, W, Ho, Wo):
    g = torch.Generator().manual_seed(H * 1000 + W + Ho)
    Cc = 64
    x = torch.randn(1, H, W, Cc, generator=g).half()
    add = torch.randn(1, Ho, Wo, Cc, generator=g).half()
    ref = nhwc(F.interpolate(nchw(x.double()), (Ho, Wo), mode="bilinear", align_corners=False))
    for addend in (None, add):
        y = torch.empty(1, Ho, Wo, Cc, dtype=torch.float16, device="cuda")
        cuda_ops.resize_bilinear(x.cuda(), y, addend=addend.cuda() if addend is not None else None, align_corners=False)
        want = ref + (addend.double() if addend is not None else 0)
        q = float(((y.cpu().double() - want).abs() / _resize_bound(x, want, H, W)).max())
        print(f"half-pixel resize {H}x{W}->{Ho}x{Wo} addend={addend is not None}: worst err/bound {q:.3f}")
        assert q <= 1.0


def test_resize_identity_exact_slice_output_and_in_place_addend(cuda_ops):
    g = torch.Generator().manual_seed(9)
    x = torch.randn(2, 16, 21, 64, generator=g).half().cuda()
    cat = torch.full((2, 16, 21, 192), 7.0, dtype=torch.float16, device="cuda")
    cuda_ops.resize_bilinear(x, cat[..., 64:128], align_corners=False)
    assert torch.equal(cat[..., 64:128], x), "the identity-size half-pixel resize must be an exact copy"
    assert bool((cat[..., :64] == 7).all() and (cat[..., 128:] == 7).all()), "the slice output wrote outside its channels"
    src = torch.randn(2, 3, 5, 64, generator=g).half().cuda()
    cuda_ops.resize_bilinear(src, cat[..., 128:], align_corners=False)
    want = F.interpolate(nchw(src.double()), (16, 21), mode="bilinear", align_corners=False)
    assert float(((cat[..., 128:].double() - nhwc(want)).abs() / _resize_bound(src.cpu(), nhwc(want).cpu(), 3, 5).cuda()).max()) <= 1.0
    cuda_ops.resize_bilinear(src, cat[..., :64], align_corners=True)          # the align-corners path takes a slice too
    want = F.interpolate(nchw(src.double()), (16, 21), mode="bilinear", align_corners=True)
    assert float((cat[..., :64].double() - nhwc(want)).abs().max()) < 1e-2
    lat = torch.randn(2, 16, 21, 64, generator=g).half().cuda()
    expect = nhwc(F.interpolate(nchw(src.double()), (16, 21), mode="bilinear", align_corners=False)) + lat.double()
    cuda_ops.resize_bilinear(src, lat, addend=lat, align_corners=False)          # laterals[i - 1] += resize(laterals[i])
    assert float(((lat.double() - expect).abs() / _resize_bound(src.cpu(), expect.cpu(), 3, 5).cuda()).max()) <= 1.0


def test_space_to_depth_bit_exact(cuda_ops):
    g = torch.Generator().manual_seed(10)
    for (B, H, W, Cc, r) in ((2, 13, 17, 64, 2), (1, 7, 9, 320, 2), (3, 5, 5, 8, 2)):
        x = torch.randn(B, H, W, Cc, generator=g).half()
        Ho, Wo = H // r, W // r
        out = torch.empty(B * Ho * Wo, r * r * Cc, dtype=torch.float16, device="cuda")
        cuda_ops.space_to_depth(x.cuda(), out, r)
        want = x[:, :Ho * r, :Wo * r].reshape(B, Ho, r, Wo, r, Cc).permute(0, 1, 3, 2, 4, 5).reshape(B * Ho * Wo, -1)
        assert torch.equal(out.cpu(), want), (B, H, W, Cc)
    img = torch.randint(0, 256, (2, 29, 35, 3), generator=g, dtype=torch.uint8)
    out = torch.empty(2 * 7 * 8, 48, dtype=torch.float16, device="cuda")
    cuda_ops.space_to_depth(img.cuda(), out, 4)
    want = img[:, :28, :32].reshape(2, 7, 4, 8, 4, 3).permute(0, 1, 3, 2, 4, 5).reshape(2 * 7 * 8, 48).half()
    assert torch.equal(out.cpu(), want)


@pytest.mark.parametrize("h,w,Hm,Wm,Ho,Wo", [(23, 31, 92, 124, 60, 90), (128, 171, 512, 683, 480, 640), (1, 1, 4, 4, 3, 5),
                                             (5, 7, 20, 28, 41, 13)])
def test_seg_labels_vs_torch(cuda_ops, h, w, Hm, Wm, Ho, Wo):
    """Labels equal torch's resize -> resize -> softmax -> argmax (on this GPU) wherever torch's top-two gap exceeds 8 ulps."""
    K, Kp = 150, 152
    g = torch.Generator().manual_seed(h * w + Ho)
    lg = torch.zeros(1, h, w, Kp)
    lg[..., :K] = torch.randn(1, h, w, K, generator=g) * 3
    lg[..., K:] = 100.0                                    # padding columns must never win
    lg = lg.cuda()
    t = F.interpolate(lg[..., :K].permute(0, 3, 1, 2).contiguous(), (Hm, Wm), mode="bilinear", align_corners=False)
    t = F.interpolate(t, (Ho, Wo), mode="bilinear", align_corners=False)
    want = torch.softmax(t, 1).argmax(1)
    top = t.topk(2, dim=1).values
    clear = (top[:, 0] - top[:, 1]) > 8 * torch.finfo(torch.float32).eps * top[:, 0].abs()
    pal = torch.randint(0, 256, (K, 3), generator=g, dtype=torch.uint8).cuda()
    lab = torch.empty(1, Ho, Wo, dtype=torch.int64, device="cuda")
    rgb = torch.empty(1, Ho, Wo, 3, dtype=torch.uint8, device="cuda")
    cuda_ops.seg_labels(lg, K, (Hm, Wm), lab, palette=pal, rgb=rgb)
    agree = lab == want
    print(f"seg_labels {h}x{w}->{Hm}x{Wm}->{Ho}x{Wo}: agree {float(agree.float().mean()):.6f}, clear {float(clear.float().mean()):.6f}")
    assert bool(agree[clear].all()) and float(agree.float().mean()) > 0.999
    assert torch.equal(rgb, pal[lab])
    lab2 = torch.empty_like(lab)
    cuda_ops.seg_labels(lg, K, (Hm, Wm), lab2)
    assert torch.equal(lab2, lab)


# ---- models ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(G, "segment_tiny.npz")), json.load(open(os.path.join(G, "segment_keys.json")))


def _tiny(meta):
    from anyedit_b200.segment import UniFormerSegmentor
    from oracle import segment_oracle as O
    m = UniFormerSegmentor(embed_dim=O.TINY_BACKBONE["embed_dim"], layers=O.TINY_BACKBONE["layers"], channels=O.TINY_HEAD["channels"])
    m.load_state_dict(O.seeded_state_dict({k: tuple(v) for k, v in meta["keys"].items()}, meta["seeds"][0]), strict=True)
    return m.cuda()


def test_tiny_vs_reference_golden(cuda_ops, gold):
    from anyedit_b200 import segment
    from oracle import segment_oracle as O
    g, meta = gold
    m = _tiny(meta)
    raw = torch.from_numpy(O.tiny_raw_images(O.TINY_SIZE, meta["seeds"][1])).cuda()
    feats = m.backbone_features(raw)
    for i, f in enumerate(feats):
        e = rel(nchw(f[:1]), g[f"out{i}"])
        print(f"[segment tiny] backbone out{i} {tuple(f.shape)} rel-L2 vs reference {e:.2e}")
        assert e <= TINY_OUT_TOL
    lg = m(raw)
    e = rel(lg[:1], g["logits"])
    print(f"[segment tiny] logits {tuple(lg.shape)} rel-L2 vs reference {e:.2e}")
    assert tuple(lg[:1].shape) == g["logits"].shape and e <= TINY_TOL

    img = O.tiny_raw_images(O.TINY_RAW, meta["seeds"][2], B=1)[0]
    res = segment.inference_segmentor(m, img)
    assert isinstance(res, list) and len(res) == 1 and res[0].dtype == np.int64 and res[0].shape == img.shape[:2]
    want, margin = g["infer_labels"], g["infer_margin"]
    rms = float(np.sqrt((g["logits"].astype(np.float64) ** 2).mean()))
    clear = margin > MARGIN * rms
    agree = res[0] == want
    print(f"[segment tiny] inference labels agree {agree.mean():.5f}; {clear.mean():.4f} of pixels have margin > {MARGIN} rms "
          f"({MARGIN * rms:.3e}), all agree there: {bool(agree[clear].all())}")
    assert bool(agree[clear].all()) and clear.mean() > 0.5
    pal = np.random.default_rng(0).integers(0, 256, size=(150, 3), dtype=np.uint8)
    shown = segment.show_result_pyplot(m, img, res, pal, opacity=1)
    assert shown.dtype == np.uint8 and shown.shape == img.shape and np.array_equal(shown, pal[res[0]])
    x = torch.from_numpy(segment.rescale(img))[None].cuda()
    lab, rgb = m.labels(x, img.shape[:2], palette=torch.from_numpy(pal).cuda())
    assert np.array_equal(lab[0].cpu().numpy(), res[0]) and np.array_equal(rgb[0].cpu().numpy(), shown)


def _real_model(seed=91):
    from anyedit_b200.segment import UniFormerSegmentor
    from oracle import segment_oracle as O
    m = UniFormerSegmentor()
    sd = O.seeded_state_dict({k: tuple(v.shape) for k, v in m.state_dict().items()}, seed)
    m.load_state_dict(sd, strict=True)
    return m, sd


def test_real_width_vs_oracle(cuda_ops):
    from anyedit_b200 import segment
    from oracle import segment_oracle as O
    m, sd = _real_model()
    m = m.cuda()
    img = O.tiny_raw_images((480, 640), 92, B=1)[0]
    r = segment.rescale(img)
    assert r.shape[:2] == (512, 683)
    with torch.no_grad():
        want = O.logits(sd, O.normalize(r))
        labels, _, _ = O.inference(sd, img)
    got = m(torch.from_numpy(r)[None].cuda())
    e = rel(got, want)
    res = segment.inference_segmentor(m, img)[0]
    agree = float((torch.from_numpy(res) == labels).float().mean())
    print(f"[segment real] logits {tuple(got.shape)} rel-L2 vs fp32 oracle {e:.2e}; labels agree on {agree:.5f} of 480 x 640 pixels")
    assert tuple(got.shape) == (1, 150, 128, 170) and e <= REAL_TOL and agree >= REAL_AGREE


def test_full_determinism_batch_independence_round_trip(cuda_ops):
    from anyedit_b200.segment import UniFormerSegmentor
    m, _ = _real_model(seed=93)
    assert len(m.state_dict()) == 414
    m = m.cuda()
    g = torch.Generator().manual_seed(34)
    x = torch.randint(0, 256, (3, 512, 683, 3), generator=g, dtype=torch.uint8).cuda()
    a = m(x)
    assert a.dtype == torch.float32 and tuple(a.shape) == (3, 150, 128, 170) and bool(a.isfinite().all())
    assert torch.equal(m(x), a), "two calls differ"
    for i in range(3):
        assert torch.equal(m(x[i:i + 1])[0], a[i]), f"image {i}: batch 1 != batch 3"
    m2 = UniFormerSegmentor()
    m2.load_state_dict({k: v.cpu() for k, v in m.state_dict().items()}, strict=True)
    assert torch.equal(m2.cuda()(x[:1])[0], a[0]), "state dict round trip changed the output"
